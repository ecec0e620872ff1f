"""CPU suite for the modulated signal generator (sig_gen.c's AM and DSB sources): the restatement tests/siggen_mod_ref.py
against the reference's own proc_sig_gen loop compiled into oracle/_ref/libka9qsiggenmod.so (oracle/siggen_mod.mk),
whose libsamplerate stand-in hands the loop scripted envelope floats.  None of it needs a GPU."""
import ctypes as C
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

import siggen_mod_ref as SM
import siggen_ref as S
from test_siggen_cpu import ABS_FLOOR, RATE, same

ROOT = Path(__file__).resolve().parent.parent
NOISE = 10 ** (-30 / 20)
AMP = 10 ** (-10 / 20)
SCALE = 1.0 / (32768 * 1.7)
KINDS = [(False, 1), (False, 0), (True, 1), (True, 0)]   # (COMPLEX, AM): AM and DSB of both master types
KIND_IDS = ["real_am", "real_dsb", "complex_am", "complex_dsb"]


def mod_oracle():
    p = ROOT / "oracle" / "_ref" / "libka9qsiggenmod.so"
    if not p.exists():
        pytest.skip("oracle/_ref/libka9qsiggenmod.so not built (needs the reference sources)")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.rs_run_mod.argtypes = [i, i, i, d, d, d, i, vp, vp, vp, i, vp, vp, vp, vp]
    return lib


def ref_run_mod(lib, cplx, am, carrier, amplitude, noise, sizes, reads, scales, env, L=20000, M=5001):
    """proc_sig_gen's AM / DSB floats and each iteration's in_energy; iteration k has blocksize sizes[k] and takes
    reads[k] envelope floats"""
    sizes = np.ascontiguousarray(sizes, np.int32)
    reads = np.ascontiguousarray(reads, np.int32)
    scales = np.ascontiguousarray(scales, np.float64)
    env = np.ascontiguousarray(env, np.float32)
    assert len(env) == reads.sum()
    out = np.zeros(int(reads.sum()) * (2 if cplx else 1), np.float32)
    en = np.zeros(len(sizes))
    assert lib.rs_run_mod(0 if cplx else 1, L, M, carrier, amplitude, noise, am, sizes.ctypes.data, reads.ctypes.data,
                          scales.ctypes.data, len(sizes), env.ctypes.data, out.ctypes.data, en.ctypes.data, None) == 0
    return out, en


def script_mod(total, seed):
    """blocksizes 1, 7, 16383, 16385, then random ones; each iteration reads all of its blocksize, a short count or
    nothing; the reads sum to total; a scale per iteration that changes now and then"""
    rng = np.random.default_rng(seed)
    sizes, reads = [1, 7, 16383, 16385], [1, 0, 16000, 16385]
    while sum(reads) < total:
        n = int(rng.integers(1, 40000))
        u = rng.random()
        r = n if u < 0.6 else 0 if u < 0.7 else int(rng.integers(0, n + 1))
        r = min(r, total - sum(reads))
        sizes.append(n)
        reads.append(r)
    scales = SCALE * np.where(rng.random(len(sizes)) < 0.3, rng.uniform(0.2, 3.0, len(sizes)), 1.0)
    return np.array(sizes), np.array(reads), scales


def envelope(n, seed, large=True):
    """an audio-like envelope in [-1, 1] with runs of -1 (no carrier in AM), 0, +1, denormals and, if asked, large
    values"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    m = 0.8 * np.sin(2 * np.pi * t / 977.0) + 0.2 * rng.uniform(-1, 1, n)
    specials = [-1.0, 0.0, 1.0, -0.0, 1e-40, -1e-42, np.float32(1.4e-45)] + ([3.5e4, -1e6, 2.5e30] if large else [])
    for k, v in enumerate(specials):
        lo = (k + 1) * n // (len(specials) + 2)
        m[lo:lo + 300] = v
    return m.astype(np.float32)


def ulp_ok(got, want, bound):
    """within 1 ulp of want, or within the absolute bound"""
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    return (d <= np.spacing(np.abs(want)).astype(np.float64)) | (d <= bound)


def energies_ok(en, samp, reads, cplx, tol=1e-12):
    """each iteration's in_energy within tol of the restatement's sum of samp^2 (REAL) or re^2 - im^2 (COMPLEX)"""
    c = 2 if cplx else 1
    edges = np.concatenate([[0], np.cumsum(reads)])
    for k in range(len(reads)):
        s = samp[c * edges[k]:c * edges[k + 1]]
        want = float(np.sum(s * s)) if not cplx else float(np.sum(s[0::2] ** 2 - s[1::2] ** 2))
        assert abs(en[k] - want) <= tol * max(float(np.sum(s * s)), 1e-300), k


def test_fma_is_exact():
    """the restatement's fused multiply-add against exact rational arithmetic, on random and hard cases"""
    rng = np.random.default_rng(3)
    a = rng.standard_normal(3000) * 10.0 ** rng.integers(-30, 30, 3000)
    b = rng.standard_normal(3000) * 10.0 ** rng.integers(-30, 30, 3000)
    c = -(a * b) * (1 + rng.integers(-4, 5, 3000) * 2.0 ** -52)   # cancellation next to a * b
    c[::3] = rng.standard_normal(1000) * 10.0 ** rng.integers(-60, 60, 1000)
    got = SM.fma(a, b, c)
    want = np.array([float(Fraction(x) * Fraction(y) + Fraction(z)) for x, y, z in zip(a, b, c)])
    assert same(got, want)


@pytest.mark.parametrize("cplx,am", KINDS, ids=KIND_IDS)
def test_noise_only_is_bitwise_the_reference_loop(cplx, am):
    """no carrier, 6e5 samples (pairs) over uneven blocksizes with short reads, reads of nothing and scale changes: every
    float bitwise proc_sig_gen's; COMPLEX draws one Gaussian per pair (noise on I, Q a signed zero)"""
    lib = mod_oracle()
    sizes, reads, scales = script_mod(600_000, seed=21 + 2 * cplx + am)
    env = envelope(int(reads.sum()), seed=1)
    out, en = ref_run_mod(lib, cplx, am, 0.0, 0.0, NOISE, sizes, reads, scales, env)
    got, samp = SM.generate_mod(cplx, 0, int(reads.sum()), 0.0, NOISE, np.repeat(scales, reads), float(am), env)
    assert same(got, out)
    energies_ok(en, samp, reads, cplx)


@pytest.mark.parametrize("cplx,am", KINDS, ids=KIND_IDS)
def test_envelope_on_a_dc_carrier_is_bitwise_the_reference_loop(cplx, am):
    """a carrier at 0 Hz (the phasor stays exactly 1) with noise, so every product and sum of the modulation is pinned:
    the envelope's -1, 0, +-1, large values and denormals, over the scripted blocksizes and reads, bitwise"""
    lib = mod_oracle()
    sizes, reads, scales = script_mod(400_000, seed=31 + 2 * cplx + am)
    env = envelope(int(reads.sum()), seed=2)
    out, en = ref_run_mod(lib, cplx, am, 0.0, AMP, NOISE, sizes, reads, scales, env)
    got, samp = SM.generate_mod(cplx, 0, int(reads.sum()), AMP, NOISE, np.repeat(scales, reads), float(am), env)
    assert same(got, out)
    energies_ok(en, samp, reads, cplx)


@pytest.mark.parametrize("cplx,am", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("carrier", [123456789.0, 17e6])
def test_modulated_carrier_within_one_ulp(cplx, am, carrier):
    """a carrier with noise, 2e5 samples (pairs) in the scripted writes: within 1 ulp of the reference's phasor chain, or
    within ABS_FLOOR of amplitude * max|dc + m| times the scale next to zeros of the signal, where a float ulp is finer
    than the chain's own rounding (tests/test_siggen_cpu.py).  Measured: at most 2e-3 of the floats differ at all.  The
    energies within 1e-11: the chain's magnitude drifts by up to 16384 roundings between renormalisations (osc.c), a
    bias of about 1e-12 in each iteration's sum."""
    lib = mod_oracle()
    sizes, reads, scales = script_mod(200_000, seed=41 + 2 * cplx + am)
    env = envelope(int(reads.sum()), seed=3, large=False)
    out, en = ref_run_mod(lib, cplx, am, carrier, AMP, NOISE, sizes, reads, scales, env)
    sc = np.repeat(scales, reads)
    got, samp = SM.generate_mod(cplx, 0, int(reads.sum()), AMP, NOISE, sc, float(am), env, F=S.angle128(carrier / RATE))
    full = AMP * float(np.max(np.abs(am + env.astype(np.float64)))) * np.repeat(sc, 2 if cplx else 1)
    ok = ulp_ok(got, out, ABS_FLOOR * full)
    assert ok.all(), (np.flatnonzero(~ok)[:5], (~ok).sum())
    assert (got != out).mean() < 2e-3
    energies_ok(en, samp, reads, cplx, tol=1e-11)
