"""Extended masters without a GPU: the prime butterflies on the host, the extended planner's splits and radices, its
agreement with today's planner on every 7-smooth length, and the rejections of kgpu_master_create_ex that happen
before any device work."""
import shutil
import subprocess
from pathlib import Path

import pytest

from accuracy_cases import FORWARD
from ext_prime_cases import EXT_FORWARD, NEW_PRIMES, TOO_BIG_FOR_SMEM

HERE = Path(__file__).resolve().parent


def _smooth7(n):
    for p in (2, 3, 5, 7):
        while n % p == 0:
            n //= p
    return n == 1


def test_prime_butterflies_on_host(tmp_path):
    """Dft<11>, <13>, <17>, <19>, <23> compiled for the host, forward and inverse, against a float64 DFT."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not available")
    exe = tmp_path / "dft_ext_host_test"
    subprocess.run([nvcc, "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-o", str(exe), str(HERE / "host" / "dft_ext_host_test.cu")], check=True, capture_output=True, timeout=600)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    print(out.stdout)
    assert out.returncode == 0 and "all prime butterflies ok" in out.stdout, out.stdout[-2000:]
    for p in NEW_PRIMES:
        assert f"radix {p:2d}" in out.stdout


@pytest.mark.parametrize("geo", EXT_FORWARD, ids=lambda g: g.id)
def test_extended_split_and_radices(geo):
    from ka9q_radio_b200 import capi

    nc = (geo.L + geo.M - 1) // (2 if geo.real else 1)
    assert capi.plan_split(nc, extended=True) == geo.split
    n1, n2 = geo.split
    assert (capi.plan_radices(n1, extended=True), capi.plan_radices(n2, extended=True)) == tuple(geo.plan)
    with pytest.raises(capi.KgpuError):  # today's planner has no split for any of them
        capi.plan_split(nc)


@pytest.mark.parametrize("geo", FORWARD, ids=lambda g: g.id)
def test_extended_planner_agrees_on_every_forward_geometry(geo):
    from ka9q_radio_b200 import capi

    nc = (geo.L + geo.M - 1) // (2 if geo.real else 1)
    split = capi.plan_split(nc)
    assert capi.plan_split(nc, extended=True) == split
    for n in split:
        assert capi.plan_radices(n, extended=True) == capi.plan_radices(n)


def test_extended_planner_agrees_on_every_7_smooth_length():
    from ka9q_radio_b200 import capi

    lengths = [n for n in range(2, 4097) if _smooth7(n)]
    assert len(lengths) == 247
    for n in lengths:
        assert capi.plan_radices(n, extended=True) == capi.plan_radices(n), n
        assert capi.plan_split(n, extended=True) == capi.plan_split(n), n


def test_extended_radices_order_and_primes():
    """even radices first, odd ones descending; every new prime is its own stage"""
    from ka9q_radio_b200 import capi

    for n in (22, 26, 34, 38, 46, 11 * 13, 17 * 19 * 4, 23 * 23 * 5, 2 * 3 * 11 * 13 * 17):
        r = capi.plan_radices(n, extended=True)
        prod = 1
        for v in r:
            prod *= v
        assert prod == n, (n, r)
        even = [v for v in r if v % 2 == 0]
        assert r == even + sorted([v for v in r if v % 2], reverse=True), (n, r)
        for p in NEW_PRIMES:
            k, m = 0, n
            while m % p == 0:
                m //= p
                k += 1
            assert r.count(p) == k, (n, r)
        with pytest.raises(capi.KgpuError):
            capi.plan_radices(n)


@pytest.mark.parametrize("n", [29, 31, 2 * 29, 37 * 8, 11 * 29, 4096 + 1])
def test_extended_planner_rejects_larger_primes(n):
    from ka9q_radio_b200 import capi

    with pytest.raises(capi.KgpuError):
        capi.plan_radices(n, extended=True)


@pytest.mark.parametrize("nc,prime", [(29 * 1000, 29), (31 * 19 * 64, 31), (8 * 9 * 5 * 1009, 1009), (2 * 7919 * 5, 7919)])
def test_create_ex_rejects_prime_factors_above_23(nc, prime):
    """COMPLEX masters: N = nc.  The rejection names the factor and the accepted set, before any device work."""
    from ka9q_radio_b200 import capi

    M = nc // 5 + 1
    with pytest.raises(capi.KgpuError, match=f"{nc} points have the prime factor {prime} "
                                             r"\(accepted factors 2, 3, 5, 7, 11, 13, 17, 19, 23\)"):
        capi.Master(nc - M + 1, M, capi.KGPU_COMPLEX, extended=True)


def test_create_ex_rejects_a_split_that_does_not_fit_shared_memory():
    from ka9q_radio_b200 import capi

    nc, (n1, n2) = TOO_BIG_FOR_SMEM
    assert capi.plan_split(nc, extended=True) == (n1, n2)
    M = nc // 5 + 1
    with pytest.raises(capi.KgpuError, match=f"{nc} points split as {n1} x {n2}, which needs .* shared memory"):
        capi.Master(nc - M + 1, M, capi.KGPU_COMPLEX, extended=True)


def test_create_ex_rejects_lengths_without_a_split():
    """2^13 19 23^2 has accepted factors only, but it is above 4096^2 points, so no split into two factors of at most
    4096 points exists."""
    from ka9q_radio_b200 import capi

    nc = 19 * 23 * 23 * 4096 * 2
    with pytest.raises(capi.KgpuError):
        capi.plan_split(nc, extended=True)
    M = nc // 5 + 1
    with pytest.raises(capi.KgpuError, match=f"{nc} points cannot be split into two plannable lengths "
                                             r"\(factors 2, 3, 5, 7, 11, 13, 17, 19, 23; <= 4096\)"):
        capi.Master(nc - M + 1, M, capi.KGPU_COMPLEX, extended=True)


def test_create_ex_keeps_the_real_parity_check():
    from ka9q_radio_b200 import capi

    with pytest.raises(capi.KgpuError, match="kgpu_master_create_ex: REAL input needs even L"):
        capi.Master(18241, 4561, capi.KGPU_REAL, extended=True)


def test_extended_symbols_declared_and_exported():
    from ka9q_radio_b200 import capi

    syms = capi.exported_symbols()
    for s in ("kgpu_master_create_ex", "kgpu_plan_radices_ex", "kgpu_plan_split_ex"):
        assert s in syms and hasattr(capi.load(), s), s
