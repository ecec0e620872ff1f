"""ctypes binding of libka9qgpu.so (the C-ABI in include/ka9q_gpu.h).

The shipped path: every call lands in the hand-written sm_90a kernels.  There is no CPU
fallback here -- if the shared library is missing or no CUDA device is usable, import/launch
fails loudly (see load()).  torch is only used by callers for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libka9qgpu.so"

KGPU_COMPLEX, KGPU_REAL = 1, 2
KGPU_FMT_F32, KGPU_FMT_I16 = 0, 1
KGPU_CHAN_ISB = 1
KGPU_CHAN_BEAM = 4

_lib = None


class KgpuError(RuntimeError):
    pass


def build(force: bool = False) -> None:
    """Compile the CUDA library in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    if force or not LIB_PATH.exists():
        subprocess.run(["make", "-C", str(PKG / "csrc"), "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise KgpuError(
            f"{LIB_PATH} is missing: build it with `make -C ka9q_radio_b200/csrc` "
            "(python -c 'import __graft_entry__ as g; g.build()'). There is no CPU fallback."
        )
    L = C.CDLL(str(LIB_PATH))
    vp, i, d, f, l = C.c_void_p, C.c_int, C.c_double, C.c_float, C.c_long
    L.kgpu_last_error.restype = C.c_char_p
    L.kgpu_launch_count.restype = C.c_ulonglong
    L.kgpu_set_device.argtypes = [i]
    L.kgpu_master_create.restype = vp
    L.kgpu_master_create.argtypes = [i, i, i]
    L.kgpu_master_destroy.argtypes = [vp]
    L.kgpu_master_points.argtypes = [vp]
    L.kgpu_master_bins.argtypes = [vp]
    L.kgpu_master_spec_stride.argtypes = [vp]
    L.kgpu_master_spec_stride.restype = l
    L.kgpu_master_describe.argtypes = [vp, C.c_char_p, i]
    L.kgpu_forward.argtypes = [vp, vp, i, f, i, i, vp, vp, vp]
    L.kgpu_master_set_notches.argtypes = [vp, vp, vp, i]
    L.kgpu_apply_notches.argtypes = [vp, vp, i, vp]
    L.kgpu_bank_create.restype = vp
    L.kgpu_bank_create.argtypes = [vp, i]
    L.kgpu_bank_destroy.argtypes = [vp]
    L.kgpu_bank_define.argtypes = [vp, i, i]
    L.kgpu_bank_set_filter.argtypes = [vp, i, d, d, d]
    L.kgpu_bank_set_filter_on.argtypes = [vp, i, d, d, d, vp]
    L.kgpu_bank_set_response.argtypes = [vp, i, vp]
    L.kgpu_bank_get_response.argtypes = [vp, i, vp]
    L.kgpu_bank_set_shift.argtypes = [vp, i, i]
    L.kgpu_bank_set_flags.argtypes = [vp, i, i]
    L.kgpu_bank_enable.argtypes = [vp, i, i]
    L.kgpu_bank_channels.argtypes = [vp]
    L.kgpu_bank_out_stride.argtypes = [vp]
    L.kgpu_bank_out_stride.restype = l
    L.kgpu_bank_out_offset.argtypes = [vp, i]
    L.kgpu_bank_out_offset.restype = l
    L.kgpu_bank_run.argtypes = [vp, vp, i, vp, vp]
    L.kgpu_bank_run_one.argtypes = [vp, i, vp, vp, vp]
    L.kgpu_bank_commit.argtypes = [vp, vp]
    L.kgpu_unpack_airspy12.argtypes = [vp, l, vp, vp, vp]
    L.kgpu_bank_define_ex.argtypes = [vp, i, i, i]
    L.kgpu_bank_set_weights.argtypes = [vp, i, d, d, d, d]
    L.kgpu_bank_set_osc.argtypes = [vp, i, i, d, d, d, d]
    L.kgpu_bank_get_osc_phase.argtypes = [vp, i, vp]
    L.kgpu_bank_set_block_counter.argtypes = [vp, l]
    L.kgpu_bank_block_counter.argtypes = [vp]
    L.kgpu_bank_block_counter.restype = l
    L.kgpu_bank_run_ex.argtypes = [vp, vp, i, vp, l, vp, vp]
    L.kgpu_bank_run_one_ex.argtypes = [vp, i, vp, vp, vp, vp]
    L.kgpu_bank_noise.argtypes = [vp, vp, i, d, vp, vp]
    L.kgpu_bank_fm_front.argtypes = [vp, vp, l, i, vp, vp, vp]
    L.kgpu_use_static_kernels.argtypes = [i]
    L.kgpu_set_tuning.argtypes = [i, i]
    L.kgpu_set_debug_buffer.argtypes = [vp]
    L.kgpu_set_debug_buffer_rows.argtypes = [vp]
    L.kgpu_profile_enable.argtypes = [i]
    L.kgpu_profile_name.argtypes = [i]
    L.kgpu_profile_name.restype = C.c_char_p
    L.kgpu_profile_get.argtypes = [i, vp, vp]
    L.kgpu_plan_radices.argtypes = [i, vp, i]
    L.kgpu_plan_split.argtypes = [l, vp, vp]
    L.kgpu_multicast_copy.argtypes = [vp, vp, C.c_ulonglong, i, vp]
    L.kgpu_algorithmic_bytes.argtypes = [vp, vp, i]
    L.kgpu_algorithmic_bytes.restype = d
    _lib = L
    return L


def exported_symbols() -> list[str]:
    """Every function declared in include/ka9q_gpu.h (checked by the CPU test-suite)."""
    import re

    hdr = (PKG.parent / "include" / "ka9q_gpu.h").read_text()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)  # declarations only, not prose
    return sorted(set(re.findall(r"\b(kgpu_[a-z0-9_]+)\s*\(", hdr)))


def profile_snapshot() -> dict[str, tuple[float, int]]:
    """{kernel name: (total ms, launches)} since the last kgpu_profile_reset()."""
    L = load()
    out = {}
    for k in range(L.kgpu_profile_kernels()):
        ms, cnt = C.c_double(0), C.c_long(0)
        L.kgpu_profile_get(k, C.cast(C.pointer(ms), C.c_void_p), C.cast(C.pointer(cnt), C.c_void_p))
        out[L.kgpu_profile_name(k).decode()] = (ms.value, cnt.value)
    return out


def plan_radices(length: int) -> list[int]:
    out = (C.c_int * 16)()
    n = load().kgpu_plan_radices(length, C.cast(out, C.c_void_p), 16)
    if n < 0:
        raise KgpuError(f"length {length} cannot be planned")
    return [out[k] for k in range(n)]


def plan_split(n: int) -> tuple[int, int]:
    a, b = C.c_int(0), C.c_int(0)
    if load().kgpu_plan_split(n, C.cast(C.pointer(a), C.c_void_p), C.cast(C.pointer(b), C.c_void_p)) != 0:
        raise KgpuError(f"{n} points cannot be split")
    return a.value, b.value


def check(rc: int, what: str = "") -> int:
    if rc < 0:
        raise KgpuError(f"{what}: {load().kgpu_last_error().decode()}")
    return rc


class Master:
    """create_filter_input's device half (reference filter.c:186-269)."""

    def __init__(self, L: int, M: int, in_type: int):
        self.lib = load()
        self.h = self.lib.kgpu_master_create(L, M, in_type)
        if not self.h:
            raise KgpuError("kgpu_master_create: " + self.lib.kgpu_last_error().decode())
        self.L, self.M, self.in_type = L, M, in_type
        self.N = self.lib.kgpu_master_points(self.h)
        self.bins = self.lib.kgpu_master_bins(self.h)
        self.spec_stride = self.lib.kgpu_master_spec_stride(self.h)

    def describe(self) -> str:
        buf = C.create_string_buffer(512)
        self.lib.kgpu_master_describe(self.h, buf, 512)
        return buf.value.decode()

    def forward(self, d_in: int, fmt: int, scale: float, nblocks: int, d_spec: int, stream: int = 0,
                derandomize: bool = False, d_stats: int = 0) -> None:
        check(self.lib.kgpu_forward(self.h, d_in, fmt, scale, int(derandomize), nblocks, d_spec, d_stats or None,
                                    stream or None), "kgpu_forward")

    def set_notches(self, bins, alpha=0.01) -> None:
        """bins as radio.c:608-620 builds them: spur bins, DC (0) appended last."""
        bins = list(bins) + [0]
        n = len(bins)
        b = (C.c_int * n)(*bins)
        a = (C.c_double * n)(*([alpha] * n))
        check(self.lib.kgpu_master_set_notches(self.h, C.cast(b, C.c_void_p), C.cast(a, C.c_void_p), n), "set_notches")

    def apply_notches(self, d_spec: int, nblocks: int, stream: int = 0) -> None:
        check(self.lib.kgpu_apply_notches(self.h, d_spec, nblocks, stream or None), "kgpu_apply_notches")

    def close(self):
        if self.h:
            self.lib.kgpu_master_destroy(self.h)
            self.h = None


class Bank:
    """A batch of create_filter_output/set_filter/execute_filter_output slaves (filter.c:298-415, :663-1045)."""

    def __init__(self, master: Master, capacity: int):
        self.lib = load()
        self.m = master
        self.h = self.lib.kgpu_bank_create(master.h, capacity)
        if not self.h:
            raise KgpuError("kgpu_bank_create: " + self.lib.kgpu_last_error().decode())

    def define(self, idx, olen, out_type=KGPU_COMPLEX) -> int:
        return check(self.lib.kgpu_bank_define_ex(self.h, idx, olen, out_type), "kgpu_bank_define_ex")

    def set_weights(self, idx, i_weight=1.0, q_weight=0.0):
        """set_filter_weights (filter.c:922-929)"""
        a = 0.5 * complex(i_weight) - 1j * complex(q_weight)
        b = 0.5 * complex(i_weight) + 1j * complex(q_weight)
        check(self.lib.kgpu_bank_set_weights(self.h, idx, a.real, a.imag, b.real, b.imag), "kgpu_bank_set_weights")

    def set_osc(self, idx, enable, phase=0.0, freq=0.0, rate=0.0, block_adj=0.0):
        check(self.lib.kgpu_bank_set_osc(self.h, idx, int(enable), phase, freq, rate, block_adj), "kgpu_bank_set_osc")

    def osc_phase(self, idx) -> float:
        v = C.c_double(0)
        check(self.lib.kgpu_bank_get_osc_phase(self.h, idx, C.cast(C.pointer(v), C.c_void_p)), "kgpu_bank_get_osc_phase")
        return v.value

    @property
    def block_counter(self) -> int:
        return self.lib.kgpu_bank_block_counter(self.h)

    @block_counter.setter
    def block_counter(self, v: int):
        check(self.lib.kgpu_bank_set_block_counter(self.h, int(v)), "kgpu_bank_set_block_counter")

    def fm_front(self, d_out: int, nblocks: int, d_baseband: int, d_stats: int, stream: int = 0):
        check(self.lib.kgpu_bank_fm_front(self.h, d_out, 0, nblocks, d_baseband, d_stats, stream or None), "kgpu_bank_fm_front")

    def noise(self, d_spec: int, nblocks: int, samprate: float, d_n0: int, stream: int = 0):
        check(self.lib.kgpu_bank_noise(self.h, d_spec, nblocks, samprate, d_n0, stream or None), "kgpu_bank_noise")

    def set_filter(self, idx, low, high, beta):
        check(self.lib.kgpu_bank_set_filter(self.h, idx, low, high, beta), "kgpu_bank_set_filter")

    def set_response(self, idx, resp):
        import numpy as np

        r = np.ascontiguousarray(resp, np.complex64)
        check(self.lib.kgpu_bank_set_response(self.h, idx, r.ctypes.data), "kgpu_bank_set_response")

    def get_response(self, idx, points):
        import numpy as np

        r = np.empty(points, np.complex64)
        check(self.lib.kgpu_bank_get_response(self.h, idx, r.ctypes.data), "kgpu_bank_get_response")
        return r

    def set_shift(self, idx, shift):
        check(self.lib.kgpu_bank_set_shift(self.h, idx, int(shift)), "kgpu_bank_set_shift")

    def set_flags(self, idx, flags):
        check(self.lib.kgpu_bank_set_flags(self.h, idx, int(flags)), "kgpu_bank_set_flags")

    def enable(self, idx, on=True):
        check(self.lib.kgpu_bank_enable(self.h, idx, int(on)), "kgpu_bank_enable")

    @property
    def out_stride(self) -> int:
        return self.lib.kgpu_bank_out_stride(self.h)

    def out_offset(self, idx) -> int:
        return self.lib.kgpu_bank_out_offset(self.h, idx)

    def run(self, d_spec: int, nblocks: int, d_out: int, stream: int = 0, d_power: int = 0):
        check(self.lib.kgpu_bank_run_ex(self.h, d_spec, nblocks, d_out, 0, d_power or None, stream or None), "kgpu_bank_run")

    def run_one(self, idx, d_spec: int, d_out: int, stream: int = 0):
        check(self.lib.kgpu_bank_run_one(self.h, idx, d_spec, d_out, stream or None), "kgpu_bank_run_one")

    def algorithmic_bytes(self, fmt) -> float:
        return self.lib.kgpu_algorithmic_bytes(self.m.h, self.h, fmt)

    def close(self):
        if self.h:
            self.lib.kgpu_bank_destroy(self.h)
            self.h = None
