"""Host-only checks of kgpu_master_create_any's path choice (kgpu_master_plan): lengths the two-pass pair serves plan
exactly as kgpu_master_create / kgpu_master_create_ex build them, every other length plans a Bluestein transform of
the smallest 7-smooth P >= 2 Nc - 1 whose split the forward pair runs, and the limits fail with a message."""
import pytest

from accuracy_cases import FORWARD
from ext_prime_cases import EXT_FORWARD, TOO_BIG_FOR_SMEM

from ka9q_radio_b200 import capi

REAL, COMPLEX = capi.KGPU_REAL, capi.KGPU_COMPLEX


def _smooth7(n):
    for p in (2, 3, 5, 7):
        while n % p == 0:
            n //= p
    return n == 1


def _rx888(rate):
    """REAL front end at `rate`, 20 ms blocks at overlap 5 (radio.c:582-587): (L, M)"""
    L = rate // 50
    return L, L // 4 + 1


@pytest.mark.parametrize("geo", FORWARD, ids=lambda g: g.id)
def test_7_smooth_lengths_plan_as_create(geo):
    path, desc = capi.plan_master(geo.L, geo.M, REAL if geo.real else COMPLEX)
    assert path == capi.MASTER_DIRECT
    n1, n2 = geo.split
    cols, rows = (",".join(map(str, r)) for r in geo.kernels)
    assert desc.startswith(f"N={geo.L + geo.M - 1} {'real' if geo.real else 'complex'}, "), desc
    assert f"two-pass {n1} x {n2}; cols radices [{cols}] rows radices [{rows}]" in desc, desc
    assert desc.endswith(f"kernels {geo.pair[0]} + {geo.pair[1]}"), desc


@pytest.mark.parametrize("geo", EXT_FORWARD, ids=lambda g: g.id)
def test_23_smooth_lengths_plan_as_create_ex(geo):
    path, desc = capi.plan_master(geo.L, geo.M, REAL if geo.real else COMPLEX)
    assert path == capi.MASTER_EXTENDED
    n1, n2 = geo.split
    cols, rows = (",".join(map(str, r)) for r in geo.plan)
    assert f"two-pass {n1} x {n2}; cols radices [{cols}] rows radices [{rows}]" in desc, desc
    assert desc.endswith("kernels fwd_cols_ext + fwd_rows_ext"), desc


BLUESTEIN = [  # (id, L, M, type, Nc, P)
    ("rx888_62m", *_rx888(62_000_000), REAL, 775_000, 1_555_200),       # 2^3 5^5 31
    ("rx888_116m", *_rx888(116_000_000), REAL, 1_450_000, 2_903_040),   # 2^4 5^5 29
    ("complex_2m9", 58_000, 14_501, COMPLEX, 72_500, 145_152),          # 2^2 5^4 29
    ("complex_7919", 63_352, 15_839, COMPLEX, 79_190, 158_760),         # 2 5 7919
    ("too_big_for_smem", TOO_BIG_FOR_SMEM[0] - 1_635_046, 1_635_047, COMPLEX, TOO_BIG_FOR_SMEM[0], None),
]


@pytest.mark.parametrize("case", BLUESTEIN, ids=lambda c: c[0])
def test_bluestein_lengths(case):
    _, L, M, in_type, nc, P = case
    N = L + M - 1
    assert nc == (N // 2 if in_type == REAL else N)
    if P is None:  # its P would exceed 3500 x 3500
        with pytest.raises(capi.KgpuError, match=f"{nc} points need a Bluestein transform of at least {2 * nc - 1} points"):
            capi.plan_master(L, M, in_type)
        return
    path, desc = capi.plan_master(L, M, in_type)
    assert path == capi.MASTER_BLUESTEIN
    assert desc.startswith(f"N={N} {'real' if in_type == REAL else 'complex'}, bluestein P={P}: {P}-point complex two-pass "), desc
    assert desc.endswith("around bluestein_in_kernel, bluestein_mul_kernel, bluestein_out_kernel"), desc
    # P is the smallest 7-smooth length >= 2 Nc - 1 whose split fits: every smaller 7-smooth candidate has no such split
    assert P >= 2 * nc - 1 and _smooth7(P)
    n1, n2 = capi.plan_split(P)
    assert f"two-pass {n1} x {n2};" in desc
    for q in range(2 * nc - 1, P):
        if _smooth7(q):
            try:
                assert capi.plan_master(q, 1, COMPLEX)[0] != capi.MASTER_DIRECT, q
            except capi.KgpuError:
                pass


def test_largest_bluestein_master():
    """Nc = 29 x 211206 needs P = 3500 x 3500, the largest the forward pair splits; Nc = 29 x 211207 fails."""
    nc = 29 * 211206
    path, desc = capi.plan_master(nc - 1000, 1001, COMPLEX)
    assert path == capi.MASTER_BLUESTEIN and "bluestein P=12250000: 12250000-point complex two-pass 3500 x 3500" in desc
    nc += 29
    with pytest.raises(capi.KgpuError, match=f"{nc} points need a Bluestein transform of at least {2 * nc - 1} points"):
        capi.plan_master(nc - 1000, 1001, COMPLEX)
    with pytest.raises(capi.KgpuError, match=f"kgpu_master_create_any: {nc} points need a Bluestein transform"):
        capi.Master(nc - 1000, 1001, COMPLEX, any_length=True)


def test_odd_real_lengths_still_fail():
    for L, M in ((4801, 1201), (1240000, 310000)):
        with pytest.raises(capi.KgpuError, match="REAL input needs even L and even N"):
            capi.plan_master(L, M, REAL)
        with pytest.raises(capi.KgpuError, match="kgpu_master_create_any: REAL input needs even L and even N"):
            capi.Master(L, M, REAL, any_length=True)


def test_bad_arguments():
    for args in ((0, 5, REAL), (100, 0, COMPLEX), (100, 5, 3)):
        with pytest.raises(capi.KgpuError, match="bad arguments"):
            capi.plan_master(*args)


def test_bluestein_symbols_declared_and_exported():
    syms = capi.exported_symbols()
    for s in ("kgpu_master_create_any", "kgpu_master_plan"):
        assert s in syms and hasattr(capi.load(), s), s
