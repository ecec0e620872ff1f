"""Restatement of sig_gen.c's CW source (proc_sig_gen, sig_gen.c:286-346) in numpy: the float bits the device must
produce.

Noise: xoshiro256** (gauss.c:32-61) seeded by splitmix64, draw d of the stream (REAL: d = sample; COMPLEX: re = 2s,
im = 2s + 1) taken by GF(2) jumps from the seeded state, and real_gauss's popcount construction (gauss.c:103-111).
Carrier: exp(2 pi i phi_n), phi_n = n F + n (n + 1) / 2 R (mod 1) with F and R the exact angles of the rounded step and
sweep phasors as 128-bit fractions of a cycle (the library's kgpu_siggen_angles, checked here against mpmath).  Each
sample is (float)(samp * scale), samp = amplitude * carrier + noise * gauss.
"""
import numpy as np

M64 = (1 << 64) - 1
GAUSS_SCALE = 0.1765469659009499


def splitmix_seed(seed):
    """xoshiro256ss_seed (gauss.c:32-44) as four words"""
    x, out = seed, []
    for _ in range(4):
        x = (x + 0x9E3779B97F4A7C15) & M64
        z = x
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        out.append(z ^ (z >> 31))
    if not any(out):
        out[0] = 1
    return out


def _rotl(x, k):
    return ((x << k) | (x >> (64 - k))) & M64


def step(s):
    """one xoshiro256ss_next state transition of a four-word list (in place); returns the output"""
    r = (_rotl((s[1] * 5) & M64, 7) * 9) & M64
    t = (s[1] << 17) & M64
    s[2] ^= s[0]
    s[3] ^= s[1]
    s[1] ^= s[2]
    s[0] ^= s[3]
    s[2] ^= t
    s[3] = _rotl(s[3], 45)
    return r


def _pack(s):
    return s[0] | s[1] << 64 | s[2] << 128 | s[3] << 192


def _unpack(v):
    return [(v >> (64 * k)) & M64 for k in range(4)]


_JUMP = []   # columns (256-bit ints) of T^(2^b)


def _apply(cols, v):
    out, j = 0, 0
    while v:
        if v & 1:
            out ^= cols[j]
        v >>= 1
        j += 1
    return out


def jump_matrix(b):
    """the columns of T^(2^b), T xoshiro256**'s state transition over GF(2)"""
    if not _JUMP:
        cols = []
        for j in range(256):
            s = _unpack(1 << j)
            step(s)
            cols.append(_pack(s))
        _JUMP.append(cols)
    while len(_JUMP) <= b:
        m = _JUMP[-1]
        _JUMP.append([_apply(m, c) for c in m])
    return _JUMP[b]


def state_at(seed, d):
    """the state before draw d, by jumps"""
    v, b = _pack(splitmix_seed(seed)), 0
    while d:
        if d & 1:
            v = _apply(jump_matrix(b), v)
        d >>= 1
        b += 1
    return _unpack(v)


def draws(seed, d0, n, log2_run=10):
    """n consecutive outputs from draw d0, as uint64: lanes of 2^log2_run draws stepped side by side"""
    R = 1 << log2_run
    lanes = max(1, -(-n // R))
    v = _pack(state_at(seed, d0))
    m = jump_matrix(log2_run)
    st = np.empty((4, lanes), np.uint64)
    for j in range(lanes):
        st[:, j] = _unpack(v)
        v = _apply(m, v)
    s0, s1, s2, s3 = (st[k].copy() for k in range(4))
    out = np.empty((R, lanes), np.uint64)
    u5, u9 = np.uint64(5), np.uint64(9)
    sh7, sh57, sh17, sh45, sh19 = (np.uint64(k) for k in (7, 57, 17, 45, 19))
    with np.errstate(over="ignore"):
        for r in range(R):
            x = s1 * u5
            out[r] = ((x << sh7) | (x >> sh57)) * u9
            t = s1 << sh17
            s2 ^= s0
            s3 ^= s1
            s1 ^= s2
            s0 ^= s3
            s2 ^= t
            s3 = (s3 << sh45) | (s3 >> sh19)
    return out.T.reshape(-1)[:n]


def gauss(u):
    """real_gauss of draws u (uint64): popcounts, then explicitly rounded doubles in the reference's order"""
    with np.errstate(over="ignore"):
        p = np.bitwise_count(u * np.uint64(0x2C1B3C6D)).astype(np.int64) + \
            np.bitwise_count(u * np.uint64(0x297A2D39)).astype(np.int64) - 64
    x = p.astype(np.float64) + u.view(np.int64).astype(np.float64) * 2.0 ** -63
    return x * GAUSS_SCALE


def angle128(f):
    """the exact angle, in cycles as a 128-bit fraction, of cispi(2 f) as the reference rounds it (sincospi.c); mpmath"""
    import math

    import mpmath

    if f == 0:
        return 0
    y = (2 * f) - math.floor((2 * f) * 0.5) * 2.0
    y = y + 2.0 if y < 0 else y
    y = y - 2.0 if y >= 2.0 else y
    q = int(2.0 * y)
    z = y - 0.5 * q
    flip = z > 0.25
    if flip:
        z = 0.5 - z
    ss, cc = math.sin(3.141592653589793 * z), math.cos(3.141592653589793 * z)
    if flip:
        ss, cc = cc, ss
    s, c = [(ss, cc), (cc, -ss), (-ss, -cc), (-cc, ss)][q]
    with mpmath.workdps(60):
        a = mpmath.atan2(mpmath.mpf(s), mpmath.mpf(c)) / (2 * mpmath.pi)
        if a < 0:
            a += 1
        return int(mpmath.floor(a * mpmath.mpf(2) ** 128))


def carrier(n0, count, F, R=0):
    """(cos, sin) of 2 pi phi_n for samples n0 .. n0 + count - 1, the phase taken to a double as the device does"""
    n = np.arange(n0, n0 + count, dtype=object)
    P = (n * F + (n * (n + 1) // 2) * R) % (1 << 128)
    hi = np.array([int(p >> 64) for p in P], np.uint64)
    phi = hi.astype(np.float64) * 2.0 ** -63            # 2 phi
    return np.cos(np.pi * phi), np.sin(np.pi * phi)


def generate(cplx, n0, count, amplitude, noise, scale, F=0, R=0, seed=1):
    """(floats, unscaled samples) of samples n0 .. n0 + count - 1; scale a scalar or one per sample"""
    c = 2 if cplx else 1
    g = gauss(draws(seed, n0 * c, count * c)) * noise
    if amplitude != 0:
        cr, ci = carrier(n0, count, F, R)
        car = np.stack([cr, ci], 1).reshape(-1) if cplx else cr
        samp = amplitude * car + g
    else:
        samp = g
    sc = np.repeat(np.broadcast_to(np.asarray(scale, np.float64), (count,)), c)
    return (samp * sc).astype(np.float32), samp
