"""CPU suite for raw 8-bit / packed 12-bit ingest: the restatements the GPU tests compare against, checked on hand-worked
values, and the raw ring sizing of write_rawfilter (pure host code in libka9qgpu.so)."""
import ctypes as C

import numpy as np
import pytest

import raw_ingest_ref as R


def test_excess_128_and_signed_bytes():
    assert R.values8(np.array([0, 255, 128, 127, 1], np.uint8), R.U8).tolist() == [-128, 127, 0, -1, -127]
    assert R.values8(np.array([0x80, 0x7F, 0, 0xFF], np.uint8), R.S8).tolist() == [-128, 127, 0, -1]
    assert R.unpack8(np.array([0, 255, 128], np.uint8), R.U8, 0.5).tolist() == [-64.0, 63.5, 0.0]


def test_double_rounding_differs_from_a_float_multiply():
    """scale = 1/(128 * 1.7), a scale_AD-like double: (float)(scale * -127) rounds the exact double product, which is
    not the float product of (float)scale and -127."""
    s = 1.0 / (128 * 1.7)
    got = R.unpack8(np.array([1], np.uint8), R.U8, s)[0]   # byte 1 -> x = -127
    assert got == np.float32(-0.5836396813392639)
    assert got != np.float32(np.float32(s) * np.float32(-127))


@pytest.mark.parametrize("fmt,inside,at", [
    (R.I16, [32766, -32766, 0], [32767, -32767, -32768]),
    (R.PACKED12, [2046, -2046, 0], [2047, -2047, -2048]),
    (R.U8, [126, -127, 0], [127, -128]),
    (R.S8, [126, -127, 0], [127, -128]),
])
def test_limits_table(fmt, inside, at):
    assert not R.at_limits(fmt, np.array(inside)).any()
    assert R.at_limits(fmt, np.array(at)).all()


def test_block_stats_restatement():
    x = np.array([127, 0, 3, -128, 0, 0, 1, 2], np.int64)   # I/Q, L = 2: block 0 = (127,0),(3,-128); block 1
    st = R.block_stats(x, R.U8, 2, True)
    assert st == [(127 ** 2 + 9 + 128 ** 2, 2, 2), (5, 0, 0)]
    assert R.since_over(st, 2) == 2
    assert R.derandomize(np.array([1, 2, -1], np.int16)).tolist() == [-1, 2, 1]


AIRSPY = [(400000, 100001), (200000, 50001)]   # Airspy R2 at 20 and 10 MS/s, M - 1 = L/4


def _ring_bytes(L, M, in_type, fmt):
    from ka9q_radio_b200 import capi

    fn = capi.load().filter_raw_ring_bytes
    fn.restype = C.c_long
    fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    return fn(L, M, in_type, fmt)


@pytest.mark.parametrize("L,M", AIRSPY)
def test_packed12_ring_holds_whole_groups(L, M):
    import os

    page = os.sysconf("SC_PAGESIZE")
    n = _ring_bytes(L, M, 2, R.PACKED12)           # REAL
    assert n > 0 and n % page == 0 and n % 12 == 0
    float_ring = -(-4 * 4 * (L + M - 1) // page) * page // 4   # samples of the master's float ring (ND = 4)
    assert n // 12 * 8 >= float_ring
    unit = page * 12 // np.gcd(page, 12)
    assert n - unit < float_ring * 3 // 2            # the smallest such size


def test_raw_ring_rejections_and_8bit_sizes():
    assert _ring_bytes(400004, 100001, 2, R.PACKED12) == -1    # windows would not start on a group boundary
    assert _ring_bytes(400000, 100003, 2, R.PACKED12) == -1
    assert _ring_bytes(400000, 100001, 1, R.PACKED12) == -1    # packed 12-bit samples are real
    assert _ring_bytes(36000, 9001, 1, 0) == -1                # unknown format
    n = _ring_bytes(36000, 9001, 1, R.U8)                      # RTL-SDR 1.8 MS/s I/Q: two bytes per pair
    assert n >= 2 * 4 * 45000 and n % 4096 == 0
