"""CPU suite for the signal generator (sig_gen.c's CW source): the restatement tests/siggen_ref.py against the reference's
own proc_sig_gen loop compiled into oracle/_ref/libka9qsiggen.so (oracle/siggen.mk), and the library's host code (GF(2)
jumps, carrier angles) against plain stepping and mpmath.  None of it needs a GPU."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import siggen_ref as S

ROOT = Path(__file__).resolve().parent.parent
RATE = 1e9   # the oracle's sample rate: one clock nanosecond per sample, so each iteration's blocksize is scripted exactly
# The reference's chain and the exact phase model differ by its accumulated rounding: below 1e-13 of the full scale
# over these runs, 1.2e-12 after 8e7 samples (measured at 123.456789 MHz, COMPLEX).  A sample that close to zero has a
# float ulp smaller than that, so there the bar is this absolute one; it exempts only samples below about 1e-4 of the
# full scale.
ABS_FLOOR = 1e-11


def oracle():
    p = ROOT / "oracle" / "_ref" / "libka9qsiggen.so"
    if not p.exists():
        pytest.skip("oracle/_ref/libka9qsiggen.so not built (needs the reference sources)")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.rs_run.argtypes = [i, i, i, d, d, d, vp, vp, i, vp, vp, vp]
    lib.rs_state_after.argtypes = [C.c_uint64, C.c_uint64, vp]
    lib.rs_step_phasor.argtypes = [d, vp]
    return lib


def ref_run(lib, cplx, carrier, amplitude, noise, sizes, scales, L=20000, M=5001):
    """proc_sig_gen's floats and each iteration's in_energy"""
    sizes = np.ascontiguousarray(sizes, np.int32)
    scales = np.ascontiguousarray(scales, np.float64)
    out = np.zeros(int(sizes.sum()) * (2 if cplx else 1), np.float32)
    en = np.zeros(len(sizes))
    assert lib.rs_run(0 if cplx else 1, L, M, carrier, amplitude, noise, sizes.ctypes.data, scales.ctypes.data, len(sizes),
                      out.ctypes.data, en.ctypes.data, None) == 0
    return out, en


def script(total, seed):
    """write sizes 1, 7, 16383, 16385, then random ones, summing to total; a scale per write that changes now and then"""
    rng = np.random.default_rng(seed)
    sizes = [1, 7, 16383, 16385]
    while sum(sizes) < total:
        sizes.append(int(min(total - sum(sizes), rng.integers(1, 40000))))
    scales = 1.0 / (32768 * 1.7) * np.where(rng.random(len(sizes)) < 0.3, rng.uniform(0.2, 3.0, len(sizes)), 1.0)
    return np.array(sizes), scales


def ulp_ok(got, want, full_scale):
    """within 1 ulp of want, or within ABS_FLOOR of the full scale"""
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    return (d <= np.spacing(np.abs(want)).astype(np.float64)) | (d <= ABS_FLOOR * full_scale)


def same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_noise_is_bitwise_the_reference_loop(cplx):
    """noise only, 1.2e6 samples (pairs) in writes of 1, 7, 16383, 16385 and random sizes with scale changes between
    writes: every float bitwise proc_sig_gen's; the REAL energy per write within 1e-12 of the restatement's sum of
    samp^2, the COMPLEX one the reference's re^2 - im^2 (not a power: the one deliberate difference of the device)"""
    lib = oracle()
    sizes, scales = script(1_200_000, seed=5 + cplx)
    out, en = ref_run(lib, cplx, 0.0, 0.0, 10 ** (-30 / 20), sizes, scales)
    got, samp = S.generate(cplx, 0, int(sizes.sum()), 0.0, 10 ** (-30 / 20), np.repeat(scales, sizes))
    assert same(got, out)
    edges = np.concatenate([[0], np.cumsum(sizes)])
    for k in range(len(sizes)):
        s = samp[(2 if cplx else 1) * edges[k]:(2 if cplx else 1) * edges[k + 1]]
        want = float(np.sum(s * s)) if not cplx else float(np.sum(s[0::2] ** 2 - s[1::2] ** 2))
        assert abs(en[k] - want) <= 1e-12 * max(float(np.sum(s * s)), 1e-300), k


@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("carrier", [123456789.0, 17e6, 301.5e6])
def test_carrier_within_one_ulp(cplx, carrier):
    """carrier only, 2e6 samples at 1 GS/s: within 1 ulp of the reference's phasor chain.  Measured on REAL streams: at
    123.456789 MHz 17 samples of 2e6 differ, by one ulp; at 17 MHz and 301.5 MHz (cos has exact zeros, every 500th and
    1000th sample) the chain leaves up to 5e-14 of the full scale there, many ulps of so small a value, and no other
    sample differs by more than one ulp."""
    lib = oracle()
    n, a, sc = 2_000_000, 10 ** (-10 / 20), 0.7
    sizes = np.full(n // 16000, 16000)
    out, _ = ref_run(lib, cplx, carrier, a, 0.0, sizes, np.full(len(sizes), sc))
    got, _ = S.generate(cplx, 0, n, a, 0.0, sc, F=S.angle128(carrier / RATE))
    ok = ulp_ok(got, out, a * sc)
    assert ok.all(), (np.flatnonzero(~ok)[:5], (~ok).sum())
    assert (got != out).mean() < 5e-3


def test_carrier_with_noise_within_one_ulp():
    lib = oracle()
    n, a, sc = 600_000, 10 ** (-10 / 20), 1.3
    sizes, _ = script(n, seed=11)
    out, _ = ref_run(lib, False, 7.77e6, a, 10 ** (-40 / 20), sizes, np.full(len(sizes), sc))
    got, _ = S.generate(False, 0, n, a, 10 ** (-40 / 20), sc, F=S.angle128(7.77e6 / RATE))
    assert ulp_ok(got, out, a * sc).all()


def test_jump_ahead_equals_plain_stepping():
    """the restatement's jumps, and the library's (pure host code), against the reference's own stepping: at offsets up
    to 1e8 and across the device's 64-draw runs"""
    lib = oracle()
    from ka9q_radio_b200 import capi

    g = capi.Siggen(capi.KGPU_REAL, 0.0, 0.0, 1.0)
    for d in (0, 1, 63, 64, 65, 4095, 4096, 1 << 20, 12_345_677, 100_000_000):
        out = (C.c_uint64 * 4)()
        lib.rs_state_after(1, d, C.cast(out, C.c_void_p))
        assert S.state_at(1, d) == list(out), d
        assert g.state(d) == tuple(out), d
    s = S.state_at(1, 0)
    want = [S.step(s) for _ in range(3000)]
    assert S.draws(1, 0, 3000, log2_run=6).tolist() == want                 # lanes of 64 draws side by side
    assert S.draws(1, 1000, 2000, log2_run=4).tolist() == want[1000:]
    g.close()


@pytest.mark.parametrize("f", [0.123456789, 0.017, 0.3015, -0.25, 0.4999999, 1e-7, 0.0])
def test_carrier_angles(f):
    """the library's step angle (binary128 on the host) is mpmath's of the phasor set_osc rounds, and that phasor is the
    reference's own"""
    lib = oracle()
    from ka9q_radio_b200 import capi

    ph = (C.c_double * 2)()
    lib.rs_step_phasor(f, C.cast(ph, C.c_void_p))
    a = S.angle128(f)
    g = capi.Siggen(capi.KGPU_COMPLEX, f, 1.0, 0.0, rate=f / 1000)
    F, R = g.angles()
    assert abs(F - a) < 1 << 16 and abs(R - S.angle128(f / 1000)) < 1 << 16   # binary128 keeps 113 bits
    th = 2 * np.pi * (a / 2.0 ** 128)
    assert abs(np.cos(th) - ph[0]) < 1e-15 and abs(np.sin(th) - ph[1]) < 1e-15
    g.close()


def test_gauss_hand_worked():
    u = np.array([0, 1, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000], np.uint64)
    p = np.array([bin((int(v) * 0x2C1B3C6D) & S.M64).count("1") + bin((int(v) * 0x297A2D39) & S.M64).count("1") - 64
                  for v in u])
    want = (p + np.array([0.0, 2.0 ** -63, -(2.0 ** -63), -1.0])) * S.GAUSS_SCALE
    assert np.array_equal(S.gauss(u), want)
