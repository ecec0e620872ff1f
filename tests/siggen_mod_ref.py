"""Restatement of sig_gen.c's AM and DSB sources (proc_sig_gen, sig_gen.c:297-314 and :327-344) in numpy, on
tests/siggen_ref.py's generator and carrier: the float bits the device must produce.

The reference's loop, as its compiler contracts it (the disassembly of oracle/_ref/libka9qsiggenmod.so's proc_sig_gen),
with m the envelope float libsamplerate produced for the sample and g = noise * real_gauss():
  REAL     samp = fma(amplitude * cr, dc + m, g)
  COMPLEX  k = (dc + m) * amplitude;  samp = fma(k, cr, g) + i k ci
One draw per sample, for COMPLEX pairs too: the noise is on I only.  numpy has no fused multiply-add, so fma() below
computes it exactly from error-free transformations (Boldo and Melquiond, "Emulation of FMA and correctly rounded sums:
proved algorithms using rounding to odd", IEEE Trans. Computers 57(4), 2008).
"""
import numpy as np

import siggen_ref as S


def _split(a):
    """Veltkamp's split of doubles into two halves of 26 bits"""
    t = a * 134217729.0   # 2^27 + 1
    hi = t - (t - a)
    return hi, a - hi


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _add_odd(a, b):
    """a + b rounded to odd: the exact sum, or else the neighbour of the two around it whose last bit is 1"""
    s, e = _two_sum(a, b)
    fix = (e != 0) & ((s.view(np.int64) & 1) == 0)
    return np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def fma(a, b, c):
    """a * b + c rounded once, elementwise (doubles; no overflow, no underflow in the product's error)"""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, np.float64) for v in (a, b, c)))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        ah, al = _split(a)
        bh, bl = _split(b)
        e = ((ah * bh - p) + ah * bl + al * bh) + al * bl    # p + e = a * b exactly
        th, tl = _two_sum(c, p)
        out = th + _add_odd(tl, e)
        return np.where(np.isfinite(p) & np.isfinite(c), out, p + c)


def generate_mod(cplx, n0, count, amplitude, noise, scale, dc, env, F=0, R=0, seed=1):
    """(floats, unscaled samples) of samples n0 .. n0 + count - 1, env their count envelope floats; scale a scalar or
    one per sample.  With amplitude 0 the carrier is taken as 0 (as the device does: the samples are the noise, and a
    COMPLEX Q is a zero with the sign of dc + m)."""
    c = 2 if cplx else 1
    g = S.gauss(S.draws(seed, n0, count)) * noise
    m = np.asarray(env, np.float32).astype(np.float64)
    if amplitude == 0:
        cr = ci = np.zeros(count)
    elif F == 0 and R == 0:   # the phasor of a 0 Hz carrier stays exactly 1 (and exp(0) is exact)
        cr, ci = np.ones(count), np.zeros(count)
    else:
        cr, ci = S.carrier(n0, count, F, R)
    if cplx:
        k = (m + dc) * amplitude
        samp = np.stack([fma(k, cr, g), k * ci], 1).reshape(-1)
    else:
        samp = fma(amplitude * cr, m + dc, g)
    sc = np.repeat(np.broadcast_to(np.asarray(scale, np.float64), (count,)), c)
    with np.errstate(over="ignore"):
        return (samp * sc).astype(np.float32), samp
