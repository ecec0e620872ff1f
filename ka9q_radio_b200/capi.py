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
KGPU_RAW_U8, KGPU_RAW_S8 = 1, 2   # kgpu_unpack8's formats, apart from kgpu_format
KGPU_RAW_S16, KGPU_RAW_U16, KGPU_RAW_SC16Q11 = 3, 4, 5   # its 16-bit formats (U16 REAL, SC16Q11 COMPLEX only)
KGPU_RAW_F32, KGPU_RAW_CF32, KGPU_RAW_CF32_CNRMF, KGPU_RAW_CF32_FSCALE = 6, 7, 8, 9   # its float formats (F32 REAL, the rest COMPLEX only)
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
    L.kgpu_master_create_ex.restype = vp
    L.kgpu_master_create_ex.argtypes = [i, i, i]
    L.kgpu_master_create_any.restype = vp
    L.kgpu_master_create_any.argtypes = [i, i, i]
    L.kgpu_master_plan.argtypes = [i, i, i, C.c_char_p, i]
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
    L.kgpu_unpack8.argtypes = [vp, i, i, l, l, i, d, vp, i, C.c_longlong, vp, vp, vp]
    L.kgpu_block_stats_i16.argtypes = [vp, i, l, l, i, i, i, vp, vp]
    ll = C.c_longlong
    L.kgpu_iq_moments.argtypes = [vp, i, ll, l, vp, i, ll, i, vp]
    L.kgpu_iq_scan.argtypes = [vp, vp, i, ll, i, vp, vp, vp]
    L.kgpu_iq_apply.argtypes = [vp, i, ll, l, vp, vp, i, ll, i, vp, vp]
    L.kgpu_siggen_create.restype = vp
    L.kgpu_siggen_create.argtypes = [i, vp]
    L.kgpu_siggen_destroy.argtypes = [vp]
    L.kgpu_siggen_generate.argtypes = [vp, ll, l, d, vp, i, vp, vp, i, l, l, vp]
    L.kgpu_siggen_set_modulation.argtypes = [vp, d]
    L.kgpu_siggen_generate_mod.argtypes = [vp, ll, l, d, vp, i, vp, vp, vp, i, l, l, vp]
    L.kgpu_siggen_state.argtypes = [vp, C.c_ulonglong, vp]
    L.kgpu_siggen_angles.argtypes = [vp, vp]
    L.filter_siggen_setup.argtypes = [vp, vp]
    L.write_genfilter.argtypes = [vp, i, d]
    L.filter_siggen_stats.argtypes = [vp, vp]
    L.filter_siggen_modulate.argtypes = [vp, d]
    L.filter_siggen_mod_pointer.restype = vp
    L.filter_siggen_mod_pointer.argtypes = [vp]
    L.kgpu_bank_define_ex.argtypes = [vp, i, i, i]
    L.kgpu_bank_define_wide.argtypes = [vp, i, i, i]
    L.kgpu_bank_define_huge.argtypes = [vp, i, i, i]
    L.kgpu_bank_define_ext.argtypes = [vp, i, i, i]
    L.kgpu_bank_define_any.argtypes = [vp, i, i, i]
    L.kgpu_chan_plan.argtypes = [i, i, C.c_char_p, i]
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
    L.kgpu_use_cols_tma.argtypes = [i]
    L.kgpu_cols_tma_fits.argtypes = [i, i, i, i, vp]
    L.kgpu_use_fused_forward.argtypes = [i]
    L.kgpu_fused_forward_fits.argtypes = [i, i, i, i, vp]
    L.kgpu_fused_forward_options.argtypes = [i, i]
    L.kgpu_fused_shape.argtypes = [vp]
    L.kgpu_fused_schedule.argtypes = [i, i, i, vp]
    L.kgpu_fused_discards.argtypes = [i, i, vp, l]
    L.kgpu_fused_discards.restype = l
    L.kgpu_profile_enable.argtypes = [i]
    L.kgpu_profile_name.argtypes = [i]
    L.kgpu_profile_name.restype = C.c_char_p
    L.kgpu_profile_get.argtypes = [i, vp, vp]
    L.kgpu_plan_radices.argtypes = [i, vp, i]
    L.kgpu_plan_split.argtypes = [l, vp, vp]
    L.kgpu_plan_radices_ex.argtypes = [i, vp, i]
    L.kgpu_plan_split_ex.argtypes = [l, vp, vp]
    L.kgpu_multicast_copy.argtypes = [vp, vp, C.c_ulonglong, i, vp]
    L.kgpu_algorithmic_bytes.argtypes = [vp, vp, i]
    L.kgpu_algorithmic_bytes.restype = d
    L.kgpu_spectrum_create.restype = vp
    L.kgpu_spectrum_create.argtypes = [i, i, i]
    L.kgpu_spectrum_set_window.argtypes = [vp, vp]
    L.kgpu_spectrum_run.argtypes = [vp, vp, l, l, i, f, vp, i, C.c_longlong, i, i, i, d, vp, vp]
    L.kgpu_spectrum_run_narrow.argtypes = [vp, vp, l, l, i, d, vp, vp, vp]
    L.kgpu_spectrum_ring_append.argtypes = [vp, l, l, vp, l, vp]
    L.kgpu_spectrum_describe.argtypes = [vp, C.c_char_p, i]
    L.kgpu_spectrum_destroy.argtypes = [vp]
    L.kgpu_spectrum_plan.argtypes = [i, i, C.c_char_p, i]
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


def plan_radices(length: int, extended: bool = False) -> list[int]:
    """extended: the radix set of kgpu_master_create_ex (also 11, 13, 17, 19, 23)"""
    out = (C.c_int * 16)()
    fn = load().kgpu_plan_radices_ex if extended else load().kgpu_plan_radices
    n = fn(length, C.cast(out, C.c_void_p), 16)
    if n < 0:
        raise KgpuError(f"length {length} cannot be planned")
    return [out[k] for k in range(n)]


def plan_split(n: int, extended: bool = False) -> tuple[int, int]:
    a, b = C.c_int(0), C.c_int(0)
    fn = load().kgpu_plan_split_ex if extended else load().kgpu_plan_split
    if fn(n, C.cast(C.pointer(a), C.c_void_p), C.cast(C.pointer(b), C.c_void_p)) != 0:
        raise KgpuError(f"{n} points cannot be split")
    return a.value, b.value


def check(rc: int, what: str = "") -> int:
    if rc < 0:
        raise KgpuError(f"{what}: {load().kgpu_last_error().decode()}")
    return rc


def unpack8(d_raw: int, fmt: int, in_type: int, history: int, L: int, nblocks: int, scale: float, d_out: int,
            d_stats: int = 0, stream: int = 0, d_chg: int = 0, nchg: int = 0, a0: int = 0) -> None:
    """8-bit, 16-bit and float ingest (kgpu_unpack8): the u8 / s8 bytes, s16 / u16 / sc16q11 words or floats of
    `history` samples then nblocks blocks of L to float32 at d_out, each (float)(scale * (double)x) (x * (float)scale for
    KGPU_RAW_CF32_FSCALE); d_stats: 0 or nblocks kgpu_block_stats (uint64 energy, or float64 fenergy for the float
    formats, uint32 overs, uint32 over_samples); d_chg: 0 or nchg kgpu_scale_change (int64 at, float64 scale), the first
    history sample being absolute sample a0."""
    check(load().kgpu_unpack8(d_raw, fmt, in_type, history, L, nblocks, scale, d_chg or None, nchg, a0, d_out,
                              d_stats or None, stream or None), "kgpu_unpack8")


def block_stats_i16(d_in: int, in_type: int, history: int, L: int, nblocks: int, d_stats: int, derandomize: bool = False,
                    limit: int = 32767, stream: int = 0) -> None:
    """Per-block statistics of int16 words on the device (kgpu_block_stats_i16): limit 32767 for the RX888's words,
    2047 for unpacked packed-12 values."""
    check(load().kgpu_block_stats_i16(d_in, in_type, history, L, nblocks, int(derandomize), limit, d_stats, stream or None),
          "kgpu_block_stats_i16")


KGPU_IQ_S8, KGPU_IQ_S16 = 1, 2   # kgpu_iq_moments / kgpu_iq_apply words
IQ_HACKRF, IQ_FUNCUBE = 1, 2     # struct kgpu_iq_params kind


class IqParams(C.Structure):
    """struct kgpu_iq_params"""
    _fields_ = [("kind", C.c_int), ("dc_alpha", C.c_double), ("gp", C.c_double)]


def iq_moments(d_raw: int, fmt: int, a0: int, count: int, d_tab: int, cap: int, w_lo: int, nw: int, stream: int = 0) -> None:
    """Moments of I/Q pairs [a0, a0 + count) into the ring table entries of writes [w_lo, w_lo + nw) (kgpu_iq_moments)."""
    check(load().kgpu_iq_moments(d_raw, fmt, a0, count, d_tab, cap, w_lo, nw, stream or None), "kgpu_iq_moments")


def iq_scan(d_tab: int, d_coef: int, cap: int, w_from: int, nw: int, kind: int, dc_alpha: float, gp: float, d_rec: int,
            stream: int = 0) -> None:
    """Records and states of the complete writes [w_from, w_from + nw), in order (kgpu_iq_scan)."""
    p = IqParams(kind, dc_alpha, gp)
    check(load().kgpu_iq_scan(d_tab, d_coef, cap, w_from, nw, C.byref(p), d_rec, stream or None), "kgpu_iq_scan")


def iq_apply(d_raw: int, fmt: int, a0: int, count: int, d_tab: int, d_coef: int, cap: int, w_lo: int, nw: int, d_out: int,
             stream: int = 0) -> None:
    """Corrected float I/Q of pairs [a0, a0 + count); pairs before 0 are 0.0 (kgpu_iq_apply)."""
    check(load().kgpu_iq_apply(d_raw, fmt, a0, count, d_tab, d_coef, cap, w_lo, nw, d_out, stream or None), "kgpu_iq_apply")


class SiggenParams(C.Structure):
    """struct kgpu_siggen_params (and filter.h's struct filter_siggen_params, the same layout)"""
    _fields_ = [("freq", C.c_double), ("rate", C.c_double), ("amplitude", C.c_double), ("noise", C.c_double),
                ("seed", C.c_uint64)]


class SiggenStats(C.Structure):
    """filter.h's struct filter_siggen_stats"""
    _fields_ = [("blocks", C.c_uint64), ("samples", C.c_uint64), ("energy", C.c_double)]


class Siggen:
    """sig_gen.c's CW source on the device (kgpu_siggen_*): carrier freq / rate in cycles per sample (per sample^2),
    amplitude, noise and the xoshiro256** seed as rand_init gives it (1); AM or DSB after modulate()."""

    def __init__(self, in_type: int, freq: float, amplitude: float, noise: float, rate: float = 0.0, seed: int = 1):
        self.cplx = in_type == KGPU_COMPLEX
        p = SiggenParams(freq, rate, amplitude, noise, seed)
        self.h = load().kgpu_siggen_create(in_type, C.byref(p))
        if not self.h:
            raise KgpuError(f"kgpu_siggen_create: {load().kgpu_last_error().decode()}")

    def generate(self, a0: int, count: int, scale: float, d_out: int, d_energy: int = 0, nblocks: int = 0, L: int = 0,
                 history: int | None = None, d_chg: int = 0, nchg: int = 0, stream: int = 0) -> None:
        """floats of samples [a0, a0 + count) at d_out; d_energy: 0 or nblocks float64 block energies of a window of
        `history` samples then nblocks blocks of L (history defaults to count - nblocks * L)"""
        if history is None:
            history = count - nblocks * L
        check(load().kgpu_siggen_generate(self.h, a0, count, scale, d_chg or None, nchg, d_out, d_energy or None, nblocks, L,
                                          history, stream or None), "kgpu_siggen_generate")

    def modulate(self, dc: float) -> None:
        """AM (dc = 1) or DSB (dc = 0): from now on generate_mod() drives the generator"""
        check(load().kgpu_siggen_set_modulation(self.h, dc), "kgpu_siggen_set_modulation")

    def generate_mod(self, a0: int, count: int, scale: float, d_out: int, d_mod: int, d_energy: int = 0, nblocks: int = 0,
                     L: int = 0, history: int | None = None, d_chg: int = 0, nchg: int = 0, stream: int = 0) -> None:
        """generate() of a modulated generator; d_mod: one float32 envelope value per sample of the window"""
        if history is None:
            history = count - nblocks * L
        check(load().kgpu_siggen_generate_mod(self.h, a0, count, scale, d_chg or None, nchg, d_out, d_mod, d_energy or None,
                                              nblocks, L, history, stream or None), "kgpu_siggen_generate_mod")

    def state(self, draw: int) -> tuple[int, int, int, int]:
        """the xoshiro256** state before draw `draw` (host jump)"""
        out = (C.c_uint64 * 4)()
        check(load().kgpu_siggen_state(self.h, draw, C.cast(out, C.c_void_p)), "kgpu_siggen_state")
        return tuple(int(v) for v in out)

    def angles(self) -> tuple[int, int]:
        """the carrier's step and sweep angles, cycles times 2^128"""
        out = (C.c_uint64 * 4)()
        check(load().kgpu_siggen_angles(self.h, C.cast(out, C.c_void_p)), "kgpu_siggen_angles")
        return int(out[0]) | int(out[1]) << 64, int(out[2]) | int(out[3]) << 64

    def close(self) -> None:
        if self.h:
            load().kgpu_siggen_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


MASTER_DIRECT, MASTER_EXTENDED, MASTER_BLUESTEIN = 0, 1, 2


def plan_master(L: int, M: int, in_type: int) -> tuple[int, str]:
    """(path, description) of the master kgpu_master_create_any would build; pure host code.  Raises when it would
    fail."""
    buf = C.create_string_buffer(512)
    return check(load().kgpu_master_plan(L, M, in_type, buf, 512), "kgpu_master_plan"), buf.value.decode()


CHAN_DIRECT, CHAN_WIDE, CHAN_HUGE, CHAN_EXTENDED, CHAN_BLUESTEIN = 0, 1, 2, 3, 4


def chan_plan(points: int, out_type: int = KGPU_COMPLEX) -> tuple[int, str]:
    """(path, description) of the channel kgpu_bank_define_any would define for `points` points; pure host code.  Raises
    when it would fail."""
    buf = C.create_string_buffer(512)
    return check(load().kgpu_chan_plan(points, out_type, buf, 512), "kgpu_chan_plan"), buf.value.decode()


class Master:
    """create_filter_input's device half (reference filter.c:186-269)."""

    def __init__(self, L: int, M: int, in_type: int, extended: bool = False, any_length: bool = False):
        """extended: create with kgpu_master_create_ex, which also serves transform lengths with prime factors 11, 13,
        17, 19 and 23 (and is kgpu_master_create for every other length).  any_length: create with
        kgpu_master_create_any, which is kgpu_master_create_ex wherever that succeeds and a Bluestein transform
        elsewhere."""
        self.lib = load()
        if any_length:
            what = "kgpu_master_create_any"
        else:
            what = "kgpu_master_create_ex" if extended else "kgpu_master_create"
        self.h = getattr(self.lib, what)(L, M, in_type)
        if not self.h:
            raise KgpuError(f"{what}: " + self.lib.kgpu_last_error().decode())
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

    def define_wide(self, idx, olen, out_type=KGPU_COMPLEX) -> int:
        """define() without its 7260-point limit: longer channels (up to 28812 points) run the four-step channel kernel."""
        return check(self.lib.kgpu_bank_define_wide(self.h, idx, olen, out_type), "kgpu_bank_define_wide")

    def define_huge(self, idx, olen, out_type=KGPU_COMPLEX) -> int:
        """define_wide() up to 1048576 points: channels longer than 28812 points run the two-kernel four-step channel
        transform through the bank's global scratch."""
        return check(self.lib.kgpu_bank_define_huge(self.h, idx, olen, out_type), "kgpu_bank_define_huge")

    def define_ext(self, idx, olen, out_type=KGPU_COMPLEX) -> int:
        """define_huge() that also serves lengths of at most 28812 points with prime factors 11, 13, 17, 19 and 23 (e.g.
        the 220 kHz and 277.2 kHz HFDL channels); their plans never take a registry slot."""
        return check(self.lib.kgpu_bank_define_ext(self.h, idx, olen, out_type), "kgpu_bank_define_ext")

    def define_any(self, idx, olen, out_type=KGPU_COMPLEX) -> int:
        """define_ext() for any point count up to 1048576: where define_ext refuses a length for its prime factors, the
        channel runs a Bluestein transform."""
        return check(self.lib.kgpu_bank_define_any(self.h, idx, olen, out_type), "kgpu_bank_define_any")

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


SPECTRUM_R2C, SPECTRUM_COMPLEX, SPECTRUM_BLUESTEIN = 0, 1, 2


def spectrum_plan(fft_n: int, in_type: int) -> tuple[int, str]:
    """(path, description) kgpu_spectrum_create would choose for fft_n; pure host code.  Raises when it would fail."""
    buf = C.create_string_buffer(256)
    return check(load().kgpu_spectrum_plan(fft_n, in_type, buf, 256), "kgpu_spectrum_plan"), buf.value.decode()


def spectrum_ring_append(ring, ring_idx: int, block, stream: int = 0) -> int:
    """Append one delivered block (a float32 CUDA tensor of (re, im) pairs, or None for a block of zeros of `block`
    samples when block is an int) to a device ring as spectrum.c:147-151 does; returns the new ring_idx."""
    import torch

    if not (ring.is_cuda and ring.is_contiguous() and ring.dtype == torch.float32 and ring.shape[-1] == 2):
        raise ValueError("ring must be a contiguous float32 CUDA tensor of (re, im) pairs")
    size = ring.numel() // 2
    if isinstance(block, int):
        src, n = None, block
    else:
        if not (block.is_cuda and block.is_contiguous() and block.dtype == torch.float32 and block.shape[-1] == 2):
            raise ValueError("block must be a contiguous float32 CUDA tensor of (re, im) pairs")
        src, n = block.data_ptr(), block.numel() // 2
    check(load().kgpu_spectrum_ring_append(ring.data_ptr(), size, int(ring_idx), src, n, stream or None),
          "kgpu_spectrum_ring_append")
    return (int(ring_idx) + n) % size


class Spectrum:
    """wideband_poll's analysis (reference spectrum.c:354-497) on a device ring of raw samples; run_narrow is
    narrowband_poll's (spectrum.c:206-306) on a ring of a COMPLEX channel's delivered blocks."""

    def __init__(self, fft_n: int, in_type: int, bin_count: int):
        self.lib = load()
        self.h = self.lib.kgpu_spectrum_create(fft_n, in_type, bin_count)
        if not self.h:
            raise KgpuError("kgpu_spectrum_create: " + self.lib.kgpu_last_error().decode())
        self.fft_n, self.in_type, self.bin_count = fft_n, in_type, bin_count

    def describe(self) -> str:
        buf = C.create_string_buffer(256)
        self.lib.kgpu_spectrum_describe(self.h, buf, 256)
        return buf.value.decode()

    def set_window(self, window) -> None:
        import numpy as np

        w = np.ascontiguousarray(window, np.float32)
        if w.shape != (self.fft_n,):
            raise ValueError(f"window needs {self.fft_n} floats")
        check(self.lib.kgpu_spectrum_set_window(self.h, w.ctypes.data), "kgpu_spectrum_set_window")

    def run(self, ring, end: int, shift: int, fft_avg: int, overlap: float, bins, scale: float = 1.0,
            derandomize: bool = False, stream: int = 0) -> None:
        """ring: a CUDA tensor of float32 / int16 samples (REAL) or of (re, im) pairs as its last dimension of 2
        (COMPLEX), any length >= fft_n; bins: a float32 CUDA tensor of at least bin_count elements."""
        import torch

        if not (ring.is_cuda and ring.is_contiguous() and bins.is_cuda and bins.dtype == torch.float32):
            raise ValueError("ring and bins must be contiguous CUDA tensors, bins float32")
        if ring.dtype == torch.float32:
            fmt = KGPU_FMT_F32
        elif ring.dtype == torch.int16:
            fmt = KGPU_FMT_I16
        else:
            raise ValueError("ring must be float32 or int16")
        samples = ring.numel() // (2 if self.in_type == KGPU_COMPLEX else 1)
        if bins.numel() < self.bin_count:
            raise ValueError(f"bins holds fewer than {self.bin_count} floats")
        check(self.lib.kgpu_spectrum_run(self.h, ring.data_ptr(), samples, int(end), fmt, float(scale), None, 0, 0,
                                         int(derandomize), int(shift), int(fft_avg), float(overlap), bins.data_ptr(), stream or None),
              "kgpu_spectrum_run")

    def run_narrow(self, ring, ring_idx: int, fft_avg: int, overlap: float, bins, stream: int = 0) -> int:
        """narrowband_poll's analysis (reference spectrum.c:206-306) of a COMPLEX analyzer: ring is a contiguous float32
        CUDA tensor of (re, im) pairs, the ring of delivered blocks; ring_idx the position its next sample would take.
        Returns the fft_avg the poll used after the reference's clamp."""
        import torch

        if not (ring.is_cuda and ring.is_contiguous() and ring.dtype == torch.float32 and ring.shape[-1] == 2):
            raise ValueError("ring must be a contiguous float32 CUDA tensor of (re, im) pairs")
        if not (bins.is_cuda and bins.dtype == torch.float32 and bins.numel() >= self.bin_count):
            raise ValueError(f"bins must be a float32 CUDA tensor of at least {self.bin_count} floats")
        used = C.c_int(0)
        check(self.lib.kgpu_spectrum_run_narrow(self.h, ring.data_ptr(), ring.numel() // 2, int(ring_idx), int(fft_avg),
                                                float(overlap), bins.data_ptr(), C.byref(used), stream or None),
              "kgpu_spectrum_run_narrow")
        return used.value

    def close(self):
        if self.h:
            self.lib.kgpu_spectrum_destroy(self.h)
            self.h = None
