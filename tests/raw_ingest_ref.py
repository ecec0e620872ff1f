"""Restatements of the front-end drivers' raw-sample loops, for the raw ingest tests.

rtlsdr.c:316-343 and hydrasdr.c:759-830 store (float)(scale * x) with a double scale and x the byte less 128 (u8) or the
signed byte (s8); rx888.c:753-767 and airspy-unpack.c:105-129 use a float scale.  Statistics per block cover only the
block's L new samples: the energy sum x*x over every component, the components at the format's limits and the samples
(I/Q pairs) with at least one component there.
"""
import numpy as np

PACKED12, U8, S8 = 1, 2, 3          # enum filter_raw_format
I16 = 0                              # write_i16filter's words, for the limits table


def values8(raw: np.ndarray, fmt: int) -> np.ndarray:
    """the driver's integer x of every byte"""
    b = np.asarray(raw, np.uint8)
    return b.astype(np.int64) - 128 if fmt == U8 else b.view(np.int8).astype(np.int64)


def unpack8(raw: np.ndarray, fmt: int, scale: float) -> np.ndarray:
    """(float)(scale * (double)x), component by component: a double product rounded once more to float"""
    return (np.float64(scale) * values8(raw, fmt).astype(np.float64)).astype(np.float32)


def at_limits(fmt: int, x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.int64)
    if fmt == I16:
        return (x > 32766) | (x < -32766)
    if fmt == PACKED12:
        return (x == 2047) | (x <= -2047)
    return (x >= 127) | (x <= -128)


def derandomize(x: np.ndarray) -> np.ndarray:
    """rx888.c:707-712: lsb set -> flip bits 1..15"""
    x = np.asarray(x, np.int16)
    return np.where(x & 1, x ^ np.int16(-2), x).astype(np.int16)


def block_stats(x: np.ndarray, fmt: int, L: int, complex_in: bool):
    """[(energy, overranges, overrange_samples)] per whole block of L samples of the integer stream x (components
    interleaved for I/Q)"""
    x = np.asarray(x, np.int64)
    c = 2 if complex_in else 1
    out = []
    for b in range(len(x) // (c * L)):
        v = x[b * c * L:(b + 1) * c * L]
        lim = at_limits(fmt, v).reshape(L, c)
        out.append((int((v * v).sum()), int(lim.sum()), int(lim.any(axis=1).sum())))
    return out


def since_over(stats, L: int, start: int = 0) -> int:
    """samples after the last block with an overrange (per-transfer rule of the drivers at block granularity)"""
    s = start
    for _, _, os in stats:
        s = 0 if os else s + L
    return s


def unpack12(samples12: np.ndarray) -> np.ndarray:
    """airspy-unpack.c:121: offset-binary 12-bit values -> x"""
    return np.asarray(samples12, np.int64) - 2048
