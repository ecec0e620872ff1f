"""CPU suite for float ingest (AirspyHF+, Fobos, HydraSDR FLOAT32_REAL / FLOAT32_IQ): the restatement
(tests/float_ingest_ref.py) on hand-worked values and against the reference's own airspyhf.c, fobos.c and hydrasdr.c
compiled into oracle/_ref/libka9qfloat.so (oracle/float.mk), and the raw ring sizing of write_rawfilter (pure host code).
"""
import ctypes as C
import os
from pathlib import Path

import numpy as np
import pytest

import float_ingest_ref as R

ROOT = Path(__file__).resolve().parent.parent
SCALE = 1.0 / 1.7                     # scale_AD-like double: its float products round differently
FLT_MAX = float(np.finfo(np.float32).max)
# Bounds on |reference energy - restated energy| / restated energy per transfer (test_restatement_against_the_reference_
# loops prints the worst it meets; measured with gcc -O3 -march=native on x86-64): HydraSDR's reassociated double sums
# 4e-16; AirspyHF+'s cnrmf, which the reference's -ffp-contract=fast turns into a fused multiply-add, 1.9e-9, under the
# 2^-24 a float rounding of each term allows; fobos.c's float sum and float division by the count 1.6e-7, for transfers
# of up to 3 900 pairs.
ENERGY_BOUND = {"airspyhf": 1e-7, "hydrasdr_real": 1e-12, "hydrasdr_iq": 1e-12, "fobos": 1e-5}


def test_hand_worked_stores_and_terms():
    x = np.array([3.0, -0.5, 1e-45, -0.0], np.float32)
    assert R.store(x, R.F32, 0.5).tolist() == [1.5, -0.25, 0.0, -0.0]
    assert R.terms(x, R.F32).tolist() == [9.0, 0.25, 0.0, 0.0]
    assert R.terms(x, R.CF32).tolist() == [9.25, float(np.float32(1e-45)) ** 2]   # a denormal's square survives in double
    # a float square past FLT_MAX overflows in cnrmf and x * x, not in cnrm's doubles
    big = np.array([2e19, 0.0], np.float32)
    assert np.isinf(R.terms(big, R.CF32_CNRMF)).all() and np.isinf(R.terms(big, R.F32)[0])
    assert R.terms(big, R.CF32)[0] == pytest.approx(4e38, rel=1e-7)


def test_double_scale_and_float_scale_rules_differ():
    """(float)(scale * (double)x) rounds the exact double product once; x * (float)scale multiplies by the scale already
    rounded to float.  Over many samples the two rules disagree in the last bit somewhere, so each needs its own format."""
    rng = np.random.default_rng(5)
    x = rng.normal(0, 0.3, 100000).astype(np.float32)
    d, f = R.store(x, R.CF32, SCALE), R.store(x, R.CF32_FSCALE, SCALE)
    assert (d != f).sum() > 1000
    assert np.array_equal(f, x * np.float32(SCALE))


def test_block_energy_order_and_non_finite():
    t = np.arange(20000, dtype=np.float64)
    assert R.block_energy(t) == float(t.sum())                       # integers: exact in any order
    assert np.isnan(R.block_energy(np.r_[t, np.nan]))
    assert np.isinf(R.block_energy(np.r_[t, np.inf]))
    assert R.block_energies(np.ones(3 * 8, np.float32), R.CF32, 4) == [8.0, 8.0, 8.0]


# ------------------------------------------------------------------ against the reference's own loops ---------------
def _oracle():
    p = ROOT / "oracle" / "_ref" / "libka9qfloat.so"
    if not p.exists():
        pytest.skip("oracle/_ref/libka9qfloat.so not built (needs the reference sources)")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    for pre in ("rh", "rf", "ryf"):
        getattr(lib, f"{pre}_set_scale").argtypes = [d]
        getattr(lib, f"{pre}_transfer").argtypes = [vp, i, vp, vp, vp]
        getattr(lib, f"{pre}_time").argtypes = [vp, i, i]
        getattr(lib, f"{pre}_time").restype = d
    lib.rh_open.argtypes = [i, i, d]
    lib.rf_open.argtypes = [i, i, d, d]
    lib.ryf_open.argtypes = [i, i, i, d]
    return lib


# driver: (oracle prefix, format, complex)
DRIVERS = {
    "airspyhf": ("rh", R.CF32_CNRMF, True),
    "fobos": ("rf", R.CF32_FSCALE, True),
    "hydrasdr_real": ("ryf", R.F32, False),
    "hydrasdr_iq": ("ryf", R.CF32, True),
}


def floats(ncomp, rng, kind="noise"):
    """ncomp float components as a front end's library delivers them: a tone in noise with denormals and signed zeros
    planted; 'huge' plants values near FLT_MAX, 'nan' and 'inf' one non-finite component"""
    t = np.arange(ncomp)
    v = (0.4 * np.cos(0.0123 * t) + rng.normal(0, 0.05, ncomp)).astype(np.float32)
    k = rng.integers(0, ncomp, 8)
    v[k[:3]] = np.float32(1e-45) * rng.integers(1, 1000, 3).astype(np.float32)   # denormals
    v[k[3]], v[k[4]] = np.float32(0.0), np.float32(-0.0)
    if kind == "huge":
        v[k[5]] = np.float32(FLT_MAX)
        v[k[6]] = np.float32(-FLT_MAX * 0.75)
    elif kind == "nan":
        v[k[5]] = np.float32(np.nan)
    elif kind == "inf":
        v[k[5]] = np.float32(-np.inf)
    return v


def _open(lib, name, scale):
    pre, _, _ = DRIVERS[name]
    L, M = 4000, 1001
    if name == "airspyhf":
        return lib.rh_open(L, M, scale)
    if name == "fobos":
        return lib.rf_open(L, M, scale, 8e6)
    return lib.ryf_open(int(name == "hydrasdr_iq"), L, M, scale)


@pytest.mark.parametrize("name", list(DRIVERS))
def test_restatement_against_the_reference_loops(name):
    """Each driver's rx_callback over seeded transfers of uneven lengths, with gain changes between them, denormals,
    signed zeros, values near FLT_MAX and a NaN and an Inf transfer: floats bitwise; the energy the callback folds into
    if_power within ENERGY_BOUND of the restatement's where that energy is finite; if_power left alone where it is not."""
    lib = _oracle()
    pre, fmt, cplx = DRIVERS[name]
    c = 2 if cplx else 1
    rng = np.random.default_rng(sum(map(ord, name)))
    kinds = ["noise", "huge", "noise", "nan", "noise", "inf", "noise", "huge"]
    scales = [SCALE, SCALE, SCALE * 10 ** (6 / 20), SCALE * 10 ** (6 / 20), SCALE, SCALE * 0.7, SCALE * 1e-3, SCALE]
    assert _open(lib, name, scales[0]) == 0
    worst, skipped, checked = 0.0, 0, 0
    try:
        for k, (kind, sc) in enumerate(zip(kinds, scales)):
            n = int(rng.integers(1, 3900))
            x = floats(c * n, rng, kind)
            getattr(lib, f"{pre}_set_scale")(sc)
            fl = np.empty(c * n, np.float32)
            ifp, alpha = C.c_double(0), C.c_double(0)
            assert getattr(lib, f"{pre}_transfer")(x.ctypes.data, n, fl.ctypes.data, C.byref(ifp), C.byref(alpha)) == 0
            want = R.store(x, fmt, sc)
            assert np.array_equal(fl.view(np.uint32), want.view(np.uint32)), (k, kind)
            e = R.transfer_energy(x, fmt)
            if not np.isfinite(e):
                assert ifp.value == 0.0, (k, kind)             # the isfinite guard skipped the update
                skipped += 1
                continue
            got = ifp.value * n / alpha.value                  # if_power was 0 before the transfer
            worst = max(worst, abs(got - e) / e)
            checked += 1
        assert skipped >= 2 and checked >= 4
        print(f"{name}: worst relative energy difference {worst:.3e}")
        assert worst <= ENERGY_BOUND[name], worst
    finally:
        getattr(lib, f"{pre}_close")()


def test_fobos_power_alpha_from_first_transfer():
    """fobos.c:405-409 sets Power_alpha from the first transfer's length and keeps it: a driver that hands write_rawfilter
    the same transfers keeps its own if_power rule unchanged"""
    lib = _oracle()
    assert lib.rf_open(4000, 1001, SCALE, 8e6) == 0
    try:
        x = floats(2 * 1000, np.random.default_rng(1))
        fl = np.empty(2000, np.float32)
        ifp, a1, a2 = C.c_double(0), C.c_double(0), C.c_double(0)
        lib.rf_transfer(x.ctypes.data, 1000, fl.ctypes.data, C.byref(ifp), C.byref(a1))
        lib.rf_transfer(x.ctypes.data, 500, fl.ctypes.data, C.byref(ifp), C.byref(a2))
        assert a1.value == a2.value == pytest.approx(-np.expm1(-1000 / (20e-3 * 8e6)), rel=1e-15)
    finally:
        lib.rf_close()


# ------------------------------------------------------------------ ring sizing ------------------------------------
def _ring_bytes(L, M, in_type, fmt):
    from ka9q_radio_b200 import capi

    fn = capi.load().filter_raw_ring_bytes
    fn.restype = C.c_long
    fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    return fn(L, M, in_type, fmt)


REAL, COMPLEX = 2, 1


@pytest.mark.parametrize("L,M,in_type,fmt", [
    (18240, 4561, COMPLEX, R.CF32_CNRMF),     # AirspyHF+ 912 kS/s
    (160000, 40001, COMPLEX, R.CF32_FSCALE),  # Fobos 8 MS/s
    (400000, 100001, REAL, R.F32),            # HydraSDR FLOAT32_REAL 20 MS/s
    (200000, 50001, COMPLEX, R.CF32),         # HydraSDR FLOAT32_IQ 10 MS/s
])
def test_float_ring_sizes(L, M, in_type, fmt):
    page = os.sysconf("SC_PAGESIZE")
    c = 2 if in_type == COMPLEX else 1
    n = _ring_bytes(L, M, in_type, fmt)
    float_ring = -(-4 * 4 * c * (L + M - 1) // page) * page // (4 * c)   # samples of the master's float ring (ND = 4)
    assert n > 0 and n % page == 0
    assert n // (4 * c) >= float_ring                 # holds the float ring's samples ...
    assert n - page < 4 * c * (float_ring + 8)        # ... in the smallest whole number of pages


def test_float_ring_rejections():
    assert _ring_bytes(40000, 10001, REAL, R.F32) > 0
    assert _ring_bytes(40000, 10001, COMPLEX, R.F32) == -1          # FILTER_RAW_F32 samples are real
    for fmt in R.COMPLEX_FORMATS:
        assert _ring_bytes(40000, 10001, COMPLEX, fmt) > 0
        assert _ring_bytes(40000, 10001, REAL, fmt) == -1           # the float I/Q formats need a COMPLEX master
    assert _ring_bytes(40000, 10001, COMPLEX, 13) == -1             # unknown format
    assert _ring_bytes(0, 10001, COMPLEX, R.CF32) == -1
