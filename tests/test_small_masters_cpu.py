"""Small masters (create_filter_input_small), host side: which geometries one CTA serves and what such a master allocates.

filter_small_master_bytes is pure host code; it returns -1 exactly where create_filter_input_small refuses the geometry
(and the caller keeps create_filter_input).  The callers' geometries are radio.c:1572-1583 (filter2: L = blocking x the
output rate x 20 ms, N = round2(2 L), COMPLEX), wfm.c:51-56 (the 384 kHz composite, REAL L = 7680, M = L + 1), packetd.c
(REAL 960 / 961) and ctcss.c:268-269 (REAL, L = 200 ms of samples, M = L + 1).
"""
import ctypes as C
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "tests" / "abi" / "_build" / "small_driver.so"
REAL, COMPLEX = 2, 1
MAX_WIDE = 28812   # kMaxWideChanPoints: the largest transform one CTA holds in shared memory
ND = 4


def _lib():
    if not LIB.exists():
        subprocess.run(["make", "-C", str(ROOT / "ka9q_radio_b200" / "csrc"), "-s"], check=True)
        subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-shared", "-pthread", f"-I{ROOT / 'include'}", "-o", str(LIB),
                        str(ROOT / "tests" / "abi" / "small_driver.c"), f"-L{ROOT / 'ka9q_radio_b200'}", "-lka9qgpu",
                        "-Wl,-rpath,$ORIGIN/../../../ka9q_radio_b200"], check=True)
    lib = C.CDLL(str(LIB))
    lib.small_master_bytes.restype = C.c_long
    lib.small_master_bytes.argtypes = [C.c_int] * 4
    return lib


def bytes_(L, M, t, slaves=3):
    return _lib().small_master_bytes(L, M, t, slaves)


def round2(v):
    return 1 << (v - 1).bit_length()


def smooth7(n):
    for p in (2, 3, 5, 7):
        while n % p == 0:
            n //= p
    return n == 1


FILTER2 = [(rate, blocking) for rate in (12000, 24000, 48000) for blocking in range(1, 11)]


@pytest.mark.parametrize("rate,blocking", FILTER2)
def test_filter2_geometries(rate, blocking):
    """Every filter2 master of blocking 1-10 at 12, 24 and 48 kHz: small up to N = 16384, the default path above."""
    L = blocking * rate // 50
    N = round2(2 * L)
    got = bytes_(L, N - L + 1, COMPLEX, 1)
    if N <= MAX_WIDE:
        assert got > 0
    else:   # 48 kHz, blocking 9 or 10: N = 32768
        assert (rate, blocking) in ((48000, 9), (48000, 10)) and got == -1


@pytest.mark.parametrize("L,M", [(7680, 7681), (960, 961)] + [(lrint, lrint + 1) for lrint in (1600, 2400, 3200, 4800, 9600)])
def test_composite_packetd_and_ctcss_geometries(L, M):
    """The wfm / stereod / rdsd composite, packetd, and ctcss at 8-48 kHz are all small."""
    for slaves in range(0, 9):
        assert bytes_(L, M, REAL, slaves) > 0
    assert bytes_(L, M, REAL, 9) == -1          # at most 8 slaves


def test_refused_just_outside_each_bound():
    # Nc above the one-CTA maximum: COMPLEX N = 28812 is served, the next 7-smooth length is not
    nxt = next(n for n in range(MAX_WIDE + 1, 2 * MAX_WIDE) if smooth7(n))
    assert bytes_(MAX_WIDE - 1000, 1001, COMPLEX) > 0
    assert bytes_(nxt - 1000, 1001, COMPLEX) == -1
    # REAL: Nc = N / 2 is the bound, so N = 2 x 28812 is served
    assert bytes_(2 * MAX_WIDE - 2000, 2001, REAL) > 0
    assert bytes_(2 * nxt - 2000, 2001, REAL) == -1
    # a prime factor above 7 in Nc
    assert bytes_(480, 548, COMPLEX) == -1       # N = 1027 = 13 x 79
    assert bytes_(484, 545, COMPLEX) == -1       # N = 1028 = 4 x 257
    # REAL needs L and N even
    assert bytes_(961, 960, REAL) == -1          # L odd
    assert bytes_(960, 962, REAL) == -1          # N = 1921 odd
    assert bytes_(960, 961, REAL) > 0
    # geometry and type arguments
    assert bytes_(0, 961, REAL) == -1 and bytes_(960, 0, REAL) == -1
    assert bytes_(960, 961, 0) == -1 and bytes_(960, 961, 3) == -1   # NONE, SPECTRUM
    assert bytes_(960, 961, REAL, -1) == -1


def test_bytes_are_sized_to_the_master():
    """Nothing grows with the default master's 2048 channel slots: a small master's bytes follow its own N and slaves,
    and one extra slave costs a bounded amount."""
    L, M = 7680, 7681
    N = L + M - 1
    base, per = bytes_(L, M, REAL, 0), bytes_(L, M, REAL, 1) - bytes_(L, M, REAL, 0)
    for s in range(9):
        assert bytes_(L, M, REAL, s) == base + s * per
    # per slave: ND output rows on the host and on the device, the response on both, fdomain and the own buffer, each at
    # most N complex
    assert 0 < per <= (2 * ND + 5) * 8 * N
    # without slaves: the float ring, fdomain[], the window and the spectrum slots -- about 3 ND N floats of payload
    assert base < 4 * ND * N * 8
    # a default master holds 2048-slot tables: its per-slot snapshots alone (ND x 2048 entries of more than 56 bytes) are
    # larger than a whole filter2 master of blocking 1 at 12 kHz, or a composite master's host and device bytes together
    assert bytes_(240, 273, COMPLEX, 1) < ND * 2048 * 56
    assert bytes_(L, M, REAL, 0) < 2 * ND * 2048 * 56
