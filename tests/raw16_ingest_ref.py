"""Restatements of the 16-bit front-end drivers' sample loops, for the raw 16-bit ingest tests.

hydrasdr.c:681-716 and :729-747 (INT16_REAL, UINT16_REAL, INT16_IQ) and sdrplay.c:1234-1246 store (float)(scale * x)
with a double scale, per component; bladerf.c:215-246 (SC16_Q11) stores (float)x of the low 12 bits sign-extended from
bit 11, i.e. scale 1.0.  At the limits: x >= 32767 or x <= -32768 for the int16 and uint16 words, x == 2047 or x == -2048
(s == 0x7ff or s == 0x800 before the sign extension) for SC16_Q11.  Statistics per block cover only the block's L new
samples: the exact energy sum x*x over every component, the components at the limits and the samples (I/Q pairs) with
at least one component there.
"""
import numpy as np

S16, U16, SC16Q11 = 6, 7, 8          # enum filter_raw_format
POWER_ALPHA = 0.05                   # hydrasdr.c:116, bladerf.c:24, sdrplay.c's Power_alpha


def values16(words: np.ndarray, fmt: int) -> np.ndarray:
    """the driver's integer x of every 16-bit word"""
    w = np.ascontiguousarray(words).view(np.uint16).astype(np.int64)
    if fmt == S16:
        return np.where(w >= 32768, w - 65536, w)
    if fmt == U16:
        return w - 32768                       # offset = 1 << (bitspersample - 1), bitspersample 16 (hydrasdr.c:686)
    s = w & 0xFFF                              # bladerf.c:226-229
    return np.where(s & 0x800, s - 0x1000, s)


def unpack16(words: np.ndarray, fmt: int, scale: float) -> np.ndarray:
    """(float)(scale * (double)x), component by component: a double product rounded once more to float"""
    return (np.float64(scale) * values16(words, fmt).astype(np.float64)).astype(np.float32)


def at_limits(fmt: int, x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.int64)
    if fmt == SC16Q11:
        return (x == 2047) | (x == -2048)
    return (x >= 32767) | (x <= -32768)


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


def interleave(i: np.ndarray, q: np.ndarray) -> np.ndarray:
    """SDRplay's separate xi[], xq[] as the int16 I/Q pairs write_rawfilter_planar stores"""
    out = np.empty(2 * len(i), np.int16)
    out[0::2], out[1::2] = i, q
    return out


class Driver:
    """One front end's per-transfer counters as its loop keeps them, from the restatement's integers: overranges
    (components for bladeRF, samples for HydraSDR, none for SDRplay), samp_since_over (HydraSDR) and if_power, smoothed
    once per transfer from the transfer's energy."""

    def __init__(self, kind: str):
        assert kind in ("hydrasdr_real", "hydrasdr_iq", "bladerf", "sdrplay")
        self.kind = kind
        self.overranges = 0
        self.since_over = 0
        self.if_power = 0.0

    def transfer(self, x: np.ndarray, fmt: int) -> int:
        """x: the transfer's integers (components interleaved for I/Q); returns its exact energy"""
        x = np.asarray(x, np.int64)
        c = 1 if self.kind == "hydrasdr_real" else 2
        n = len(x) // c
        lim = at_limits(fmt, x).reshape(n, c)
        if self.kind == "bladerf":
            self.overranges += int(lim.sum())
        elif self.kind != "sdrplay":
            for over in lim.any(axis=1):       # per sample, as hydrasdr.c:706-711 and :736-741 count
                if over:
                    self.overranges += 1
                    self.since_over = 0
                else:
                    self.since_over += 1
        energy = int((x * x).sum())
        if n:
            self.if_power += POWER_ALPHA * (float(energy) / n - self.if_power)
        return energy
