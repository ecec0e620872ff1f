"""CPU suite for the HackRF and FUNcube I/Q correction: the exact-moments restatement (tests/iq_correction_ref.py) pinned
to the reference's own hackrf.c rx_callback and funcube.c proc_funcube, compiled unmodified with the reference's flags
into oracle/_ref/libka9qiqcorr.so (oracle/iqcorr.mk), and the host-only parts of the filter.h extension.

The reference's loops sum in double with -funsafe-math-optimizations and -ffp-contract=fast, so their sums may be
reassociated and their corrections contracted to FMA; the restatement computes each write's sums exactly from integer
moments.  The bounds below were measured on these runs and are kept with some margin; the GPU suite then checks the
device bitwise against the restatement.
"""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import iq_correction_ref as R

ROOT = Path(__file__).resolve().parent.parent
HACKRF_FS = 20e6
HACKRF_SCALE = 1.0 / 128.0
FUNCUBE_SCALE = 1.0 / 32768.0


def ref_lib():
    p = ROOT / "oracle" / "_ref" / "libka9qiqcorr.so"
    if not p.exists():
        pytest.skip("oracle/_ref/libka9qiqcorr.so not built (needs the reference sources)")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.rh_open.argtypes = [d, i, i, d]
    lib.rh_set_scale.argtypes = [d]
    lib.rh_transfer.argtypes = [vp, i, vp, vp, vp, vp]
    lib.rh_time.argtypes = [vp, i, i]
    lib.rh_time.restype = d
    lib.rf_run.argtypes = [vp, i, i, d, i, i, vp, vp, vp, vp]
    return lib


def hackrf_bytes(n, seed=1, dc=(3.2, -2.1), amp=40.0, noise=6.0, clip_rate=2e-4):
    """n signed-byte I/Q pairs of a HackRF: two tones plus noise, a DC offset of a few LSB, 5 % gain imbalance, a 2 degree
    phase skew, and some -128 words"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    sig = (amp * np.exp(2j * np.pi * 0.0123 * t) + 0.5 * amp * np.exp(-2j * np.pi * 0.211 * t)
           + rng.normal(0, noise, n) + 1j * rng.normal(0, noise, n))
    ph = np.deg2rad(2.0)
    v = np.empty(2 * n)
    v[0::2] = 1.05 * sig.real + dc[0]
    v[1::2] = sig.imag * np.cos(ph) + sig.real * np.sin(ph) + dc[1]
    v = np.clip(np.rint(v), -128, 127)
    v[rng.random(2 * n) < clip_rate] = -128
    return v.astype(np.int8).view(np.uint8)


def funcube_words(n, seed=2, dc=(120.0, -80.0), amp=9000.0, noise=900.0, over_rate=3e-4):
    """n int16 I/Q pairs of a FUNcube: a tone in noise with DC, imbalance, phase skew and words at both limits"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    sig = amp * np.exp(2j * np.pi * 0.031 * t) + rng.normal(0, noise, n) + 1j * rng.normal(0, noise, n)
    ph = np.deg2rad(1.5)
    v = np.empty(2 * n)
    v[0::2] = 0.97 * sig.real + dc[0]
    v[1::2] = sig.imag * np.cos(ph) + sig.real * np.sin(ph) + dc[1]
    v = np.clip(np.rint(v), -32768, 32767)
    hit = rng.random(2 * n) < over_rate
    v[hit] = rng.choice([32767, -32767, -32768], hit.sum())
    return v.astype(np.int16)


def split(raw, sizes, comp_bytes):
    out, o = [], 0
    for s in sizes:
        out.append(raw[o:o + 2 * s * comp_bytes // raw.itemsize])
        o += 2 * s * comp_bytes // raw.itemsize
    return out


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    d = np.abs(a - b) / np.maximum(np.abs(b), 1e-300)
    d[a == b] = 0.0
    return d


def ulps(a, b):
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32).astype(np.int64))


def run_hackrf_ref(lib, writes, scales):
    """rx_callback on each transfer: floats, state, clips, if_power after each"""
    assert lib.rh_open(HACKRF_FS, 262144, 4097, scales[0]) == 0
    fl, st, clips, ifp = [], [], [], []
    try:
        for wr, sc in zip(writes, scales):
            lib.rh_set_scale(sc)
            n = wr.size // 2
            f = np.empty(n, np.complex64)
            s = np.empty(8)
            cl, ip = C.c_int(), C.c_double()
            lib.rh_transfer(wr.ctypes.data, wr.size, f.ctypes.data, s.ctypes.data, C.byref(cl), C.byref(ip))
            fl.append(f)
            st.append(s)
            clips.append(cl.value)
            ifp.append(ip.value)
    finally:
        lib.rh_close()
    return fl, np.array(st), clips, ifp


def hackrf_if_power(recs, samprate=HACKRF_FS):
    """hackrf.c:364, from the records, as a patched driver keeps it"""
    p = 0.0
    out = []
    for r in recs:
        be = 0.5 * (r.i_energy + r.q_energy)
        p += r.n * (1.0 / (samprate * 1.0)) * (be / r.n - p)
        out.append(p)
    return out


def compare_hackrf(writes, scales, state_bound, ulp_bound, power_bound):
    lib = ref_lib()
    fl_ref, st_ref, clips_ref, ifp_ref = run_hackrf_ref(lib, writes, scales)
    fl, recs = R.run(R.Params.hackrf(HACKRF_FS), R.S8, writes, scales)
    st = np.array([[r.state[k] for k in R.STATE] for r in recs])
    worst_state = rel(st, st_ref).max()
    worst_ulp = max(int(ulps(a.view(np.float32), b.view(np.float32)).max()) for a, b in zip(fl, fl_ref))
    assert np.cumsum([r.overs for r in recs]).tolist() == clips_ref
    worst_power = rel(hackrf_if_power(recs), ifp_ref).max()
    assert worst_state <= state_bound, worst_state
    assert worst_ulp <= ulp_bound, worst_ulp
    assert worst_power <= power_bound, worst_power
    return recs


def test_restatement_against_ref_hackrf():
    """250 transfers of 131 072 pairs (1.6 s at 20 MS/s: imbalance climbs from 0 and gain_i settles from its large first
    values), then odd sizes, and a scale change.  Measured: state within 4.3e-14 relative (imbalance), floats bitwise
    (0 ulp), if_power within 2.5e-14; bounds 1e-11, 1 ulp, 1e-12."""
    sizes = [131072] * 250 + [513, 100003, 131071, 4096, 65537]
    writes = split(hackrf_bytes(sum(sizes)), sizes, 1)
    scales = [HACKRF_SCALE] * 252 + [HACKRF_SCALE / 3] * 3
    recs = compare_hackrf(writes, scales, 1e-11, 1, 1e-12)
    assert recs[0].state["gain_i"] > 8 and 0.9 < recs[-1].state["gain_i"] / recs[-1].state["gain_q"] < 1.1


def test_dc_dominated_low_signal_hackrf():
    """A DC of 40 and -35 LSB over a signal of about 1 LSB: the moment expansion cancels most of Sii against the DC terms.
    Measured: state within 1.2e-12 relative (tanphi, sinphi), floats bitwise, if_power within 4.4e-13; bounds 1e-10,
    1 ulp, 1e-10."""
    sizes = [131072] * 120
    writes = split(hackrf_bytes(sum(sizes), seed=5, dc=(40.3, -35.2), amp=0.7, noise=0.6, clip_rate=0), sizes, 1)
    compare_hackrf(writes, [HACKRF_SCALE] * len(sizes), 1e-10, 1, 1e-10)


def test_zero_energy_writes_leave_the_state():
    """All-zero transfers from the initial state: block_energy is 0, so imbalance, sinphi and the gains stay as they were
    (hackrf.c:366) and DC stays 0, in the restatement and in the reference."""
    lib = ref_lib()
    writes = [np.zeros(2 * 4096, np.uint8)] * 3
    fl_ref, st_ref, clips_ref, _ = run_hackrf_ref(lib, writes, [HACKRF_SCALE] * 3)
    p = R.Params.hackrf(HACKRF_FS)
    fl, recs = R.run(p, R.S8, writes, [HACKRF_SCALE] * 3)
    init = [p.state[k] for k in R.STATE]
    for r, s in zip(recs, st_ref):
        assert [r.state[k] for k in R.STATE] == init == s.tolist()
        assert r.i_energy == r.q_energy == r.dotprod == 0.0
    assert all(np.array_equal(a, b) for a, b in zip(fl, fl_ref))


def test_restatement_against_ref_funcube():
    """2 000 blocks of 960 pairs (a 5 ms Blocktime at 192 kS/s; 10 s, so imbalance and sinphi settle), int16 words at both
    limits.  DC, sinphi and imbalance per block, the floats, overranges and samp_since_over, and if_power by
    funcube.c:293-294 from the records.  Measured: state within 1.1e-15 relative, floats at most 1 ulp apart (a
    contracted correction in the reference); bounds 1e-11, 1 ulp, and 1e-12 on if_power.  samp_since_over and the overrange count are exact."""
    lib = ref_lib()
    nb, bs = 2000, 960
    words = funcube_words(nb * bs)
    fl_ref = np.empty(nb * bs, np.complex64)
    st_ref = np.empty((nb, 8))
    counts = np.empty(2 * nb, np.uint64)
    ifp_ref = np.empty(nb)
    assert lib.rf_run(words.ctypes.data, nb, bs, FUNCUBE_SCALE, 8192, 1025, fl_ref.ctypes.data, st_ref.ctypes.data,
                      counts.ctypes.data, ifp_ref.ctypes.data) == 0
    writes = [words[2 * b * bs: 2 * (b + 1) * bs] for b in range(nb)]
    fl, recs = R.run(R.Params.funcube(bs), R.S16, writes, [FUNCUBE_SCALE] * nb)
    st = np.array([[r.state[k] for k in ("dc_i", "dc_q", "sinphi", "imbalance")] for r in recs])
    assert rel(st, st_ref[:, :4]).max() <= 1e-11
    assert ulps(np.concatenate(fl).view(np.float32), fl_ref.view(np.float32)).max() <= 1
    since, overs, p, ifp = 0, 0, 0.0, []
    for b, r in enumerate(recs):
        since = R.samp_since_over(since, r)
        overs += r.overs
        assert (overs, since) == (int(counts[2 * b]), int(counts[2 * b + 1])), b
        be = r.i_energy + r.q_energy
        if np.isfinite(be):
            p += 0.05 * (be / r.n - p)
        ifp.append(p)
    assert rel(ifp, ifp_ref).max() <= 1e-12
    assert sum(r.overs for r in recs) > 100 and any(r.since_over < 0 for r in recs)


def test_moments_and_since_over_by_hand():
    i, q, over = R.words(np.array([-128, 5, 127, -128, 0, 0], np.int8).view(np.uint8), R.S8)
    assert i.tolist() == [-127, 127, 0] and q.tolist() == [5, -127, 0] and over.tolist() == [1, 0, 0, 1, 0, 0]
    assert R.since_over(over) == 2
    assert R.moments(i, q) == (0, -122, 2 * 127 ** 2, 25 + 127 ** 2, -127 * 5 - 127 * 127)
    i, q, over = R.words(np.array([32767, -32768, 1, -32766], np.int16), R.S16)
    assert over.tolist() == [True, True, False, False] and R.since_over(over) == 2
    assert R.since_over(np.zeros(4, bool)) == -1


def test_one_division_form_serves_both_drivers():
    """hackrf.c:368 divides by 0.5 (i + q), funcube.c:301 multiplies by 2 and divides by (i + q): equal in IEEE double"""
    rng = np.random.default_rng(3)
    d = rng.normal(0, 1e6, 20000) * 10.0 ** rng.integers(-20, 20, 20000)
    e = np.abs(rng.normal(0, 1e6, 20000)) * 10.0 ** rng.integers(-20, 20, 20000)
    assert np.array_equal(d / (0.5 * e), 2 * d / e)


# ------------------------------------------------------------------ host-only parts of the extension ----------------
def _kgpu():
    p = ROOT / "ka9q_radio_b200" / "libka9qgpu.so"
    if not p.exists():
        pytest.skip("libka9qgpu.so not built")
    lib = C.CDLL(str(p))
    lib.filter_iq_table_writes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    lib.filter_iq_table_writes.restype = C.c_long
    lib.filter_raw_ring_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    lib.filter_raw_ring_bytes.restype = C.c_long
    return lib


COMPLEX, REAL = 1, 2


@pytest.mark.parametrize("L,M,fmt,word", [(400000, 100001, R.S8, 1), (3840, 961, R.S16, 2), (36000, 9001, R.S8, 1)])
def test_table_holds_every_write_of_the_raw_ring(L, M, fmt, word):
    """The table holds twice the writes of FILTER_IQ_MIN_WRITE (512) pairs the raw ring can hold, plus 2 ND + 2."""
    lib = _kgpu()
    ring = lib.filter_raw_ring_bytes(L, M, COMPLEX, fmt)
    assert ring >= 4 * (L + M - 1) * 2 * word
    cap = lib.filter_iq_table_writes(L, M, COMPLEX, fmt)
    assert cap == 2 * (ring // (2 * word) // 512) + 2 * 4 + 2


def test_table_rejects_real_masters_and_other_formats():
    lib = _kgpu()
    assert lib.filter_iq_table_writes(400000, 100001, REAL, R.S8) == -1
    assert lib.filter_raw_ring_bytes(400000, 100001, REAL, R.S16) == -1
    assert lib.filter_iq_table_writes(36000, 9001, COMPLEX, 3) == -1   # FILTER_RAW_S8 has no table
