"""CPU suite for raw 16-bit ingest (HydraSDR int16 / uint16, bladeRF SC16 Q11, SDRplay's planar int16): the restatement
(tests/raw16_ingest_ref.py) on hand-worked values and against the reference's own hydrasdr.c and bladerf.c compiled into
oracle/_ref/libka9qraw16.so (oracle/raw16.mk), and the raw ring sizing of write_rawfilter (pure host code)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import raw16_ingest_ref as R

ROOT = Path(__file__).resolve().parent.parent
SCALE = 1.0 / (32768 * 1.7)   # scale_AD-like double: its float products round differently


def test_hand_worked_decodes():
    assert R.values16(np.array([0x0800, 0xF7FF, 0x07FF, 0xF800, 0x0000, 0xFFFF], np.uint16), R.SC16Q11).tolist() == \
        [-2048, 2047, 2047, -2048, 0, -1]                      # bits 12-15 are ignored
    assert R.values16(np.array([0x0000, 0x8000, 0xFFFF, 0x7FFF], np.uint16), R.U16).tolist() == [-32768, 0, 32767, -1]
    assert R.values16(np.array([0x8000, 0x7FFF, 0xFFFF, 0], np.uint16), R.S16).tolist() == [-32768, 32767, -1, 0]
    assert R.unpack16(np.array([0x0000, 0x8000], np.uint16), R.U16, 0.5).tolist() == [-16384.0, 0.0]
    assert R.unpack16(np.array([0x0800, 0x17FF], np.uint16), R.SC16Q11, 1.0).tolist() == [-2048.0, 2047.0]


def test_double_rounding_differs_from_a_float_multiply():
    """(float)(scale * -32767) rounds the exact double product, which is not the float product of (float)scale and
    -32767 (the 16-bit counterpart of the 8-bit formats' case)."""
    s = 1.0 / (128 * 1.7)
    got = R.unpack16(np.array([-127], np.int16), R.S16, s)[0]
    assert got == np.float32(-0.5836396813392639)
    assert got != np.float32(np.float32(s) * np.float32(-127))


@pytest.mark.parametrize("fmt,inside,at", [
    (R.S16, [32766, -32767, 0], [32767, -32768]),
    (R.U16, [32766, -32767, 0], [32767, -32768]),
    (R.SC16Q11, [2046, -2047, 0], [2047, -2048]),
])
def test_limits_table(fmt, inside, at):
    assert not R.at_limits(fmt, np.array(inside)).any()
    assert R.at_limits(fmt, np.array(at)).all()


def test_block_stats_and_energy_are_exact():
    """both components at -32768 give 2^31 per pair, which hydrasdr.c:744's int sum overflows; the restatement (and the
    device) sums exactly"""
    x = np.array([-32768, -32768, 1, 2, 32767, 0, 3, 4], np.int64)   # I/Q, L = 2
    st = R.block_stats(x, R.S16, 2, True)
    assert st == [(2 ** 31 + 5, 2, 1), (32767 ** 2 + 25, 1, 1)]
    assert R.interleave(np.array([1, 2], np.int16), np.array([-1, -2], np.int16)).tolist() == [1, -1, 2, -2]


# ------------------------------------------------------------------ against the reference's own loops ---------------
def _oracle():
    p = ROOT / "oracle" / "_ref" / "libka9qraw16.so"
    if not p.exists():
        pytest.skip("oracle/_ref/libka9qraw16.so not built (needs the reference sources)")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.ry_open.argtypes = [i, i, i, d]
    lib.ry_set_scale.argtypes = [d]
    lib.ry_transfer.argtypes = [vp, i, vp, vp, vp]
    lib.ry_time.argtypes = [vp, i, i]
    lib.ry_time.restype = d
    lib.rb_open.argtypes = [i, i]
    lib.rb_transfer.argtypes = [vp, i, vp, vp, vp]
    lib.rb_time.argtypes = [vp, i, i]
    lib.rb_time.restype = d
    return lib


def words16(ncomp, fmt, rng, garbage=False):
    """ncomp components: a tone in noise with words at both limits now and then; for bladeRF, random bits 12-15"""
    t = np.arange(ncomp)
    if fmt == R.SC16Q11:
        v = np.clip(np.rint(1500 * np.cos(0.0123 * t) + rng.normal(0, 200, ncomp)), -2048, 2047).astype(np.int64)
        v[rng.random(ncomp) < 3e-3] = 2047
        v[rng.random(ncomp) < 3e-3] = -2048
        w = (v & 0xFFF).astype(np.uint16)
        if garbage:
            w |= (rng.integers(0, 16, ncomp) << 12).astype(np.uint16)
        return w
    v = np.clip(np.rint(20000 * np.cos(0.0123 * t) + rng.normal(0, 3000, ncomp)), -32768, 32767).astype(np.int64)
    v[rng.random(ncomp) < 3e-3] = 32767
    v[rng.random(ncomp) < 3e-3] = -32768
    if fmt == R.U16:
        return (v + 32768).astype(np.uint16)
    return v.astype(np.int16).view(np.uint16)


def no_double_min_pairs(w):
    """hydrasdr.c:744 sums x*x + y*y in int: a pair with both components at -32768 overflows it (undefined behaviour)"""
    p = w.view(np.int16).reshape(-1, 2)
    both = (p[:, 0] == -32768) & (p[:, 1] == -32768)
    p[both, 1] = -32767
    return w


def ulps(a, b):
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


L_CPU, M_CPU = 4000, 1001


@pytest.mark.parametrize("kind,fmt", [(0, R.S16), (1, R.U16), (2, R.S16)])
def test_restatement_against_ref_hydrasdr(kind, fmt):
    """rx_callback in INT16_REAL (0), UINT16_REAL (1) and INT16_IQ (2), software AGC off, over seeded transfers of
    uneven lengths with a gain change between two of them: floats bitwise, overranges and samp_since_over exactly,
    if_power within 1e-12 relative of the value from the restatement's energy."""
    lib = _oracle()
    rng = np.random.default_rng(11 + kind)
    c = 2 if kind == 2 else 1
    scales = [SCALE, SCALE, SCALE * 10 ** (6 / 20), SCALE * 10 ** (6 / 20), SCALE, SCALE * 0.7]
    assert lib.ry_open(kind, L_CPU, M_CPU, scales[0]) == 0
    drv = R.Driver("hydrasdr_iq" if kind == 2 else "hydrasdr_real")
    try:
        for k, sc in enumerate(scales):
            n = int(rng.integers(1, 3900))
            w = words16(c * n, fmt, rng)
            if kind == 2:
                w = no_double_min_pairs(w)
            lib.ry_set_scale(sc)
            fl = np.empty(c * n, np.float32)
            cnt = (C.c_uint64 * 2)()
            ifp = C.c_double(0)
            assert lib.ry_transfer(w.ctypes.data, n, fl.ctypes.data, C.cast(cnt, C.c_void_p), C.byref(ifp)) == 0
            want = R.unpack16(w, fmt, sc)
            assert np.array_equal(fl.view(np.uint32), want.view(np.uint32)), (k, int(ulps(fl, want).max()))
            drv.transfer(R.values16(w, fmt), fmt)
            assert (cnt[0], cnt[1]) == (drv.overranges, drv.since_over), k
            assert abs(ifp.value - drv.if_power) <= 1e-12 * abs(drv.if_power), k
        assert drv.overranges > 0
    finally:
        lib.ry_close()


def test_restatement_against_ref_bladerf():
    """bladerf_process over seeded buffers of uneven lengths with garbage in bits 12-15: floats bitwise (scale 1.0),
    overranges per component exactly, if_power within 1e-12 relative."""
    lib = _oracle()
    rng = np.random.default_rng(21)
    assert lib.rb_open(L_CPU, M_CPU) == 0
    drv = R.Driver("bladerf")
    try:
        for k in range(6):
            n = int(rng.integers(1, 3900))
            w = words16(2 * n, R.SC16Q11, rng, garbage=True)
            fl = np.empty(2 * n, np.float32)
            over = C.c_uint64(0)
            ifp = C.c_double(0)
            lib.rb_transfer(w.ctypes.data, n, fl.ctypes.data, C.byref(over), C.byref(ifp))
            want = R.unpack16(w, R.SC16Q11, 1.0)
            assert np.array_equal(fl.view(np.uint32), want.view(np.uint32)), k
            drv.transfer(R.values16(w, R.SC16Q11), R.SC16Q11)
            assert over.value == drv.overranges, k
            assert abs(ifp.value - drv.if_power) <= 1e-12 * abs(drv.if_power), k
        assert drv.overranges > 0
    finally:
        lib.rb_close()


def test_sdrplay_restatement():
    """sdrplay.c:1238-1242, pinned by hand: (float complex)(CMPLX(xi, xq) * scale) is each component's double product
    rounded to float, so the planar arrays interleaved and converted as S16 give the driver's floats; its energy is the
    exact sum of xi^2 + xq^2 (cnrm of integer-valued doubles)."""
    xi = np.array([-32768, 32767, 1, -1], np.int16)
    xq = np.array([-32768, 0, -127, 2], np.int16)
    s = 1.0 / (128 * 1.7)
    got = R.unpack16(R.interleave(xi, xq), R.S16, s).view(np.complex64)
    assert got[2] == np.complex64(np.float32(s * 1) + 1j * np.float32(-0.5836396813392639))
    assert got[0].real == got[0].imag == np.float32(-32768 * s)
    drv = R.Driver("sdrplay")
    e = drv.transfer(R.values16(R.interleave(xi, xq), R.S16), R.S16)
    assert e == 2 * 32768 ** 2 + 32767 ** 2 + 1 + 127 ** 2 + 5
    assert drv.overranges == 0 and drv.if_power == pytest.approx(0.05 * e / 4, rel=1e-15)


# ------------------------------------------------------------------ ring sizing ------------------------------------
def _ring_bytes(L, M, in_type, fmt):
    from ka9q_radio_b200 import capi

    fn = capi.load().filter_raw_ring_bytes
    fn.restype = C.c_long
    fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    return fn(L, M, in_type, fmt)


REAL, COMPLEX = 2, 1


@pytest.mark.parametrize("L,M,in_type,fmt", [
    (40000, 10001, COMPLEX, R.S16),          # SDRplay 2 MS/s
    (240000, 60001, COMPLEX, R.SC16Q11),     # bladeRF 12 MS/s
    (1228800, 307201, COMPLEX, R.SC16Q11),   # bladeRF 61.44 MS/s
    (400000, 100001, REAL, R.S16),           # HydraSDR int16 REAL 20 MS/s
    (400000, 100001, REAL, R.U16),
    (200000, 50001, COMPLEX, R.S16),         # HydraSDR int16 I/Q 10 MS/s
])
def test_raw16_ring_sizes(L, M, in_type, fmt):
    import os

    page = os.sysconf("SC_PAGESIZE")
    c = 2 if in_type == COMPLEX else 1
    n = _ring_bytes(L, M, in_type, fmt)
    float_ring = -(-4 * 4 * c * (L + M - 1) // page) * page // (4 * c)   # samples of the master's float ring (ND = 4)
    assert n > 0 and n % page == 0
    assert n // (2 * c) >= float_ring                 # holds the float ring's samples ...
    assert n - page < 2 * c * (float_ring + 8)        # ... in the smallest whole number of pages


def test_raw16_ring_rejections():
    assert _ring_bytes(40000, 10001, REAL, R.S16) > 0
    assert _ring_bytes(40000, 10001, COMPLEX, R.U16) == -1       # offset-binary 16-bit samples are real
    assert _ring_bytes(40000, 10001, REAL, R.SC16Q11) == -1      # SC16 Q11 samples are I/Q
    assert _ring_bytes(36000, 9001, COMPLEX, 7) == -1
    assert _ring_bytes(40000, 10001, COMPLEX, 13) == -1          # unknown format
    assert _ring_bytes(0, 10001, COMPLEX, R.S16) == -1
