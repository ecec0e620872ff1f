"""Plain numpy restatements of the two per-channel steps that follow the filter on the device (noise_kernel.cuh):
estimate_noise (radio.c:1783-1866) and the front half of demod_fm (fm.c:104-131, :205-231, threshold off).  They are
written from the reference's description, independently of oracle/chan_oracle_ext.c, so that a kernel and the oracle
cannot share a mistake.  Where the reference is undefined (a REAL master smaller than the window, the bins after the
COMPLEX walk stops at the master's Nyquist bin) they state the zero fill the device documents."""
import numpy as np

NQ, N_CUTOFF, MIN_NOISE_BINS = 0.10, 1.5, 1000  # radio.c:73-76
_Z = N_CUTOFF * -np.log(1 - NQ)
CORRECTION = 1 / (1 - _Z * np.exp(-_Z) / (1 - np.exp(-_Z)))  # radio.c:1842-1843


def noise_energies(X, complex_master, s_bins, shift):
    """float32 energies of the window estimate_noise takes from master spectrum X, or None when it gives up"""
    X = np.asarray(X, np.complex64)
    m = len(X)
    nbins = max(s_bins, MIN_NOISE_BINS)
    if not complex_master:
        mbin = abs(shift) - nbins // 2
        if mbin < 0:
            mbin = 0
        elif mbin + nbins > m:
            mbin = m - nbins
        filled = nbins
        if nbins > m:  # master smaller than the window: the bins that exist, zeros after them
            mbin, filled = 0, m
        idx = mbin + np.arange(filled)
    else:
        mbin = shift - nbins // 2
        if mbin < 0:
            mbin += m
        elif mbin >= m:
            mbin -= m
        if not 0 <= mbin < m:
            return None
        to_nyq = (m // 2 - mbin) % m  # the walk stops when it reaches bin m/2; starting there it takes a full turn
        filled = min(nbins, to_nyq if to_nyq else m)
        idx = (mbin + np.arange(filled)) % m
    x = X[idx]
    e = np.zeros(nbins, np.float32)
    e[:filled] = x.real * x.real + x.imag * x.imag  # float32, each operation rounded
    return e


def estimate_noise(X, complex_master, s_bins, shift, samprate):
    """N0 in W/Hz as estimate_noise returns it: mean of the bins <= 1.5 x (10 % quantile), corrected, per master bin"""
    e = noise_energies(X, complex_master, s_bins, shift)
    if e is None:
        return 0.0
    e = e.astype(np.float64)
    q = np.quantile(e, NQ, method="linear")
    keep = e[e <= N_CUTOFF * q]
    if len(keep) == 0:
        return 0.0
    return float(np.sum(keep)) / len(keep) * CORRECTION / (len(X) * samprate)


def exact_components(rng, n, kmax=2047):
    """n complex64 values whose components are multiples of 1/16 below 128 (kmax/16): x*x + y*y is exact in float32,
    so no rounding or FMA contraction anywhere can move a bin across the quantile or the 1.5 q threshold"""
    k = rng.integers(-kmax, kmax + 1, size=(2, n))
    return (k[0] / 16 + 1j * (k[1] / 16)).astype(np.complex64)


def _on_axis(x):
    return np.asarray(x, np.float32).astype(np.complex64)  # y = 0: the energy is fl(x*x) everywhere


def order_stat_windows(rng):
    """(name, points, real_out, builder) of windows that test the order statistics of estimate_noise.  builder(rng)
    returns the window's bins (complex64, one permutation of a fixed multiset); the energies are exact in float32.
    Energies used: 1 (x=1), 1.5625 (x=1.25), 4 (x=2), 6.25 (x=2.5), 625 (x=25)."""

    def fill(nbins, parts, rest=25.0):
        v = np.concatenate([np.full(c, x, np.float64) for x, c in parts] + [np.full(nbins - sum(c for _, c in parts), rest)])
        return lambda r: _on_axis(r.permutation(v))

    x_t = np.float32(1.5309311151504517)  # fl(x_t * x_t) == 2.34375 == 1.5 * 1.5625
    assert float(x_t * x_t) == 2.34375
    x_up = np.nextafter(x_t, np.float32(2))
    out = [
        # 1200 bins: k = 119, frac 0.9; the 10 % quantile sits inside a run of 500 equal energies
        ("ties", 1200, False, fill(1200, [(1, 100), (2, 500), (2.5, 100)])),
        # 1152 bins: k = 115, frac 0.1.  cnt_le == k + 1: q2 is the next larger energy (6.25), so q = 4.225 and the
        # 6.25 bins are kept; with q2 taken as q1 they would be dropped
        ("cnt_le=k+1", 1152, False, fill(1152, [(1, 109), (2, 7), (2.5, 30)])),
        ("cnt_le=k+2", 1152, False, fill(1152, [(1, 109), (2, 8), (2.5, 30)])),  # q2 == q1 == 4: 6.25 dropped
        # REAL-output slave of 2000 points: 1001 bins, pos = 100 exactly, frac == 0: q = q1 = 4 whatever q2 is
        ("frac=0", 2000, True, fill(1001, [(1, 100), (2, 1), (2.5, 30)])),
        # q = 1.5625 (q1 == q2); 40 bins sit exactly on 1.5 q = 2.34375 (kept), 40 one ulp above it (dropped)
        ("at 1.5q", 1200, False, fill(1200, [(1, 100), (1.25, 200), (x_t, 40), (x_up, 40)])),
        ("all zero", 1000, False, fill(1000, [], rest=0.0)),
        # every energy subnormal or just above: m * 2^-74 squared is a multiple of 2^-148
        ("subnormal", 1500, False, lambda r: _on_axis(r.integers(1, 2048, 1500) * 2.0 ** -74)),
        # energies from 1e-30 to 1e30
        ("1e-30..1e30", 1800, False,
         lambda r: _on_axis(r.integers(1, 2048, 1800) * 2.0 ** r.integers(-50, 39, 1800).astype(np.float64))),
        # more than 4096 bins with heavy ties (5 distinct energies)
        ("wide ties", 9600, False, lambda r: _on_axis(r.choice([1.0, 1.25, 2.0, 2.5, 25.0], 9600, p=[.05, .03, .1, .02, .8]))),
        ("wide ties real-out", 15360, True,
         lambda r: _on_axis(r.choice([1.0, 2.0, 2.5, 25.0], 7681, p=[.09, .03, .03, .85]))),
    ]
    return out


def place_windows(X, windows, start=500, gap=37):
    """writes the windows one after another into REAL-master spectrum X -> the shift that centres each one's window"""
    shifts, pos = [], start
    for w in windows:
        X[pos:pos + len(w)] = w
        shifts.append(pos + len(w) // 2)
        pos += len(w) + gap
    assert pos <= len(X)
    return shifts


def fm_front(y, prev):
    """-> (baseband float32, mean amplitude, sum of squared amplitude deviations) of one block y (complex64) whose
    predecessor sample is prev.  The product y[n] conj(y[n-1]) is a float complex one, as in fm.c, written out so that
    every operation is rounded on its own; its argument is taken in float64."""
    y = np.asarray(y, np.complex64)
    amp = np.abs(y).astype(np.float64)  # cabsf
    mean = float(np.sum(amp)) / len(y)
    dev = float(np.sum((amp - mean) ** 2))
    p = np.concatenate([np.asarray([prev], np.complex64), y[:-1]])
    vr, vi, pr, pi = y.real, y.imag, p.real, -p.imag
    re = vr * pr - vi * pi
    im = vr * pi + vi * pr
    bb = (np.arctan2(im.astype(np.float64), re.astype(np.float64)) / np.pi).astype(np.float32)
    return bb, mean, dev
