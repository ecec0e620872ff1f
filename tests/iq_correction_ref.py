"""Restatement of the I/Q correction of the HackRF and FUNcube drivers (hackrf.c:297-375, funcube.c:194-310) as the
device computes it: the exact-moments algorithm.

Each write (one USB transfer, or one PortAudio block) is corrected with the coefficients the previous write left.  The
driver's sums over a write follow from five exact integer moments of its words (after HackRF's -128 -> -127 clip):
Si, Sq, Sii, Sqq, Siq.  With (DCr, DCi) the DC estimate the write was corrected with,

    i_energy = (Sii - (2 DCr) Si) + (n DCr) DCr
    q_energy = (Sqq - (2 DCi) Sq) + (n DCi) DCi
    dotprod  = (gain_i gain_q) (((Siq - DCi Si) - DCr Sq) + (n DCr) DCi)

each evaluated left to right in IEEE double without contraction, then the drivers' state update in their own
expression order.  Every sample is ((float)(scale xi), (float)(scale (secphi yq - tanphi xi))) with xi = (i - DCr) gain_i,
yq = (q - DCi) gain_q.  The kernels of csrc/iq_correct.cuh compute exactly this; samples before the first write are 0.
"""
from dataclasses import dataclass, field

import numpy as np

S8, S16 = 4, 5          # enum filter_raw_format: FILTER_RAW_S8_IQCORR, FILTER_RAW_S16_IQCORR
HACKRF, FUNCUBE = 1, 2  # how the gain/phase weight of a write is formed

STATE = ("dc_i", "dc_q", "sinphi", "imbalance", "gain_i", "gain_q", "secphi", "tanphi")


@dataclass
class Params:
    """filter_iq_correction_setup's parameters: per-sample DC weight, the gain/phase weight per write (gp_rate * n for
    HackRF, gp_alpha for FUNcube) and the driver's initial state."""
    kind: int
    dc_alpha: float
    gp: float
    state: dict = field(default_factory=dict)

    @staticmethod
    def hackrf(samprate: float) -> "Params":
        # hackrf.c:34-35 (DC_alpha, Power_tc = 1), :317 rate_factor; the sdrstate is calloc'd, then :239-241
        return Params(HACKRF, 1.0e-7, 1.0 / (samprate * 1.0),
                      dict(dc_i=0.0, dc_q=0.0, sinphi=0.0, imbalance=0.0, gain_i=1.0, gain_q=1.0, secphi=1.0, tanphi=0.0))

    @staticmethod
    def funcube(blocksize: int, samprate: int = 192000) -> "Params":
        # funcube.c:28-30 (DC_alpha, Power_tc), :201-209 (local gains, gainphase_alpha); the sdrstate is calloc'd
        return Params(FUNCUBE, 1.0e-6, blocksize / (samprate * 1.0),
                      dict(dc_i=0.0, dc_q=0.0, sinphi=0.0, imbalance=0.0, gain_i=1.0, gain_q=1.0, secphi=1.0, tanphi=0.0))


def words(raw: np.ndarray, fmt: int):
    """(i, q) int64 words of one write, HackRF's -128 clipped to -127, and the components at the limits"""
    if fmt == S8:
        v = np.asarray(raw).view(np.int8).astype(np.int64)
        over = v == -128
        v = np.where(over, -127, v)
    else:
        v = np.asarray(raw).view(np.int16).astype(np.int64)
        over = np.abs(v) >= 32767
    return v[0::2], v[1::2], over


def moments(i: np.ndarray, q: np.ndarray):
    return int(i.sum()), int(q.sum()), int((i * i).sum()), int((q * q).sum()), int((i * q).sum())


def since_over(over: np.ndarray) -> int:
    """components after the last one at the limits, or -1 if there was none"""
    idx = np.flatnonzero(over)
    return -1 if idx.size == 0 else int(over.size - 1 - idx[-1])


def step(p: Params, st: dict, n: int, m):
    """one write's record (energies, dotprod) and the state after it, from its moments m and the state it was corrected
    with; IEEE double throughout (numpy scalars: division by zero gives inf, 0/0 NaN, as in the drivers)"""
    f = np.float64
    Si, Sq, Sii, Sqq, Siq = (f(v) for v in m)
    nd = f(n)
    dcr, dci = f(st["dc_i"]), f(st["dc_q"])
    with np.errstate(all="ignore"):
        ie = (Sii - (f(2) * dcr) * Si) + (nd * dcr) * dcr
        qe = (Sqq - (f(2) * dci) * Sq) + (nd * dci) * dci
        dot = (f(st["gain_i"]) * f(st["gain_q"])) * (((Siq - dci * Si) - dcr * Sq) + (nd * dcr) * dci)
        new = {k: f(v) for k, v in st.items()}
        if n != 0 or p.kind == FUNCUBE:   # hackrf.c:359
            new["dc_i"] = dcr + f(p.dc_alpha) * (Si - nd * dcr)
            new["dc_q"] = dci + f(p.dc_alpha) * (Sq - nd * dci)
        be = f(0.5) * (ie + qe)
        if be > 0:
            w = f(p.gp) * nd if p.kind == HACKRF else f(p.gp)
            new["imbalance"] = new["imbalance"] + w * (ie / qe - new["imbalance"])
            dpn = dot / be
            new["sinphi"] = new["sinphi"] + w * (dpn - new["sinphi"])
            new["gain_q"] = np.sqrt(f(0.5) * (f(1) + new["imbalance"]))
            new["gain_i"] = np.sqrt(f(0.5) * (f(1) + f(1) / new["imbalance"]))
            new["secphi"] = f(1) / np.sqrt(f(1) - new["sinphi"] * new["sinphi"])
            new["tanphi"] = new["sinphi"] * new["secphi"]
    return (float(ie), float(qe), float(dot)), {k: float(v) for k, v in new.items()}


def apply(i: np.ndarray, q: np.ndarray, st: dict, scale: float) -> np.ndarray:
    """the corrected floats of one write (complex64), with the coefficients st"""
    f = np.float64
    x = i.astype(np.float64) - f(st["dc_i"])
    y = q.astype(np.float64) - f(st["dc_q"])
    xi = x * f(st["gain_i"])
    yq = y * f(st["gain_q"])
    y2 = f(st["secphi"]) * yq - f(st["tanphi"]) * xi
    out = np.empty(2 * i.size, np.float32)
    out[0::2] = (f(scale) * xi).astype(np.float32)
    out[1::2] = (f(scale) * y2).astype(np.float32)
    return out.view(np.complex64)


@dataclass
class Record:
    n: int
    sum_i: int
    sum_q: int
    i_energy: float
    q_energy: float
    dotprod: float
    overs: int
    since_over: int
    state: dict


def run(p: Params, fmt: int, writes, scales):
    """every write's floats and record, in order"""
    st = dict(p.state)
    floats, recs = [], []
    for raw, scale in zip(writes, scales):
        i, q, over = words(raw, fmt)
        floats.append(apply(i, q, st, scale))
        m = moments(i, q)
        (ie, qe, dot), st = step(p, st, i.size, m)
        recs.append(Record(i.size, m[0], m[1], ie, qe, dot, int(over.sum()), since_over(over), dict(st)))
    return floats, recs


def samp_since_over(prev: int, rec: Record) -> int:
    """funcube.c:256-267's samp_since_over after a write, from the record"""
    return prev + 2 * rec.n if rec.since_over < 0 else rec.since_over
