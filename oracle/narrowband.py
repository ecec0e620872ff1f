"""oracle/narrowband.py -- ctypes front end to the narrowband spectrum analyzer's checkers (oracle/narrowband.mk).

TEST INFRASTRUCTURE, NOT PRODUCT.

  Restatement  oracle/libkanarrowband.so          ko_narrowband_spectrum, ko_nb_ring_step (narrowband_oracle.c)
  Reference    oracle/_ref/libka9qnarrowband.so   the reference's own narrowband_poll (ref_narrowband.c), where it was built
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REF_LIB = HERE / "_ref" / "libka9qnarrowband.so"

_lib = None
_ref = None
_POLL = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not (HERE / "libkanarrowband.so").exists():
            subprocess.run(["make", "-C", str(HERE), "-s", "-f", "narrowband.mk", "libkanarrowband.so"], check=True,
                           cwd=str(HERE))
        L = C.CDLL(str(HERE / "libkanarrowband.so"))
        L.ko_narrowband_spectrum.argtypes = _POLL
        L.ko_nb_ring_step.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                      C.c_int]
        _lib = L
    return _lib


def have_ref() -> bool:
    return REF_LIB.exists()


def ref() -> C.CDLL:
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_LIB))
        L.rs_narrowband_poll.argtypes = _POLL
        _ref = L
    return _ref


def _prep(ring, window):
    return np.ascontiguousarray(ring, np.complex64), np.ascontiguousarray(window, np.float32)


def narrowband_spectrum(fft_n, bin_count, window, fft_avg, overlap, ring, ring_idx):
    """The restatement: (bin_count float32 bins, fft_avg used) of one poll of `ring` (complex64, its whole length the
    ring size) whose next write position is ring_idx."""
    r, w = _prep(ring, window)
    out = np.empty(bin_count, np.float32)
    used = lib().ko_narrowband_spectrum(fft_n, bin_count, w.ctypes.data, int(fft_avg), float(overlap), r.ctypes.data,
                                        len(r), int(ring_idx), out.ctypes.data)
    if used < 0:
        raise ValueError("ko_narrowband_spectrum rejected the arguments")
    return out, used


def ref_narrowband_poll(fft_n, bin_count, window, fft_avg, overlap, ring, ring_idx):
    """The reference's own narrowband_poll on the same ring: (bins, the fft_avg its clamp left)."""
    r, w = _prep(ring, window)
    out = np.zeros(bin_count, np.float32)
    used = ref().rs_narrowband_poll(fft_n, bin_count, w.ctypes.data, int(fft_avg), float(overlap), r.ctypes.data,
                                    len(r), int(ring_idx), out.ctypes.data)
    return out, used


class Ring:
    """demod_spectrum's narrowband ring (spectrum.c:124-151), restated: step() is one block's upkeep and append."""

    def __init__(self, cap: int):
        self.buf = np.zeros(cap, np.complex64)
        self.size = C.c_int(0)
        self.idx = C.c_int(0)

    def step(self, fft_avg: int, fft_n: int, block=None, n: int | None = None) -> None:
        """block: complex64 samples, or None for n zeros (a lapped block)"""
        if block is not None:
            block = np.ascontiguousarray(block, np.complex64)
            n = len(block)
        if lib().ko_nb_ring_step(self.buf.ctypes.data, len(self.buf), C.byref(self.size), C.byref(self.idx), fft_avg,
                                 fft_n, None if block is None else block.ctypes.data, int(n)) != 0:
            raise ValueError("ring capacity too small")

    @property
    def ring(self) -> np.ndarray:
        return self.buf[:self.size.value].copy()

    @property
    def ring_idx(self) -> int:
        return self.idx.value
