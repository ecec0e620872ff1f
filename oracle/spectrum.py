"""oracle/spectrum.py -- ctypes front end to the wideband spectrum analyzer's checkers (oracle/spectrum.mk).

TEST INFRASTRUCTURE, NOT PRODUCT.

  Restatement  oracle/libkaspectrum.so          ko_wideband_spectrum (spectrum_oracle.c)
  Reference    oracle/_ref/libka9qspectrum.so   the reference's own wideband_poll (ref_spectrum.c), where it was built
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REF_LIB = HERE / "_ref" / "libka9qspectrum.so"

_lib = None
_ref = None
_ARGS = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_long, C.c_long, C.c_void_p]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not (HERE / "libkaspectrum.so").exists():
            subprocess.run(["make", "-C", str(HERE), "-s", "-f", "spectrum.mk", "libkaspectrum.so"], check=True,
                           cwd=str(HERE))
        L = C.CDLL(str(HERE / "libkaspectrum.so"))
        L.ko_wideband_spectrum.argtypes = _ARGS
        _lib = L
    return _lib


def have_ref() -> bool:
    return REF_LIB.exists()


def ref() -> C.CDLL:
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_LIB))
        L.rs_wideband_poll.argtypes = _ARGS
        _ref = L
    return _ref


def _prep(ring, window, is_real):
    r = np.ascontiguousarray(ring, np.float32 if is_real else np.complex64)
    w = np.ascontiguousarray(window, np.float32)
    return r, w


def wideband_spectrum(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end) -> np.ndarray:
    """The restatement: bin_count float32 bins of one poll of `ring` (float32 REAL or complex64 COMPLEX samples) whose
    newest sample ends at ring position `end`."""
    r, w = _prep(ring, window, is_real)
    out = np.empty(bin_count, np.float32)
    if lib().ko_wideband_spectrum(int(bool(is_real)), fft_n, bin_count, w.ctypes.data, int(shift), int(fft_avg),
                                  float(overlap), r.ctypes.data, len(r), int(end), out.ctypes.data) != 0:
        raise ValueError("ko_wideband_spectrum rejected the arguments")
    return out


def ref_wideband_poll(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end):
    """The reference's own wideband_poll on the same ring: (bins, the fft_avg its clamp left)."""
    r, w = _prep(ring, window, is_real)
    out = np.zeros(bin_count, np.float32)
    used = ref().rs_wideband_poll(int(bool(is_real)), fft_n, bin_count, w.ctypes.data, int(shift), int(fft_avg),
                                  float(overlap), r.ctypes.data, len(r), int(end), out.ctypes.data)
    return out, used
