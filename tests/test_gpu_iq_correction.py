"""HackRF and FUNcube I/Q correction on the device: the kernels through the C-ABI, and write_rawfilter with
FILTER_RAW_S8_IQCORR / FILTER_RAW_S16_IQCORR through filter.h.

The device's moments are exact integers, and its records, states and floats are bitwise those of the restatement in
tests/iq_correction_ref.py (which tests/test_iq_correction_cpu.py pins to the reference's own hackrf.c and funcube.c).
So a master fed corrected raw words is compared bitwise with the same library fed the restated floats through
write_cfilter, and within TOL with the reference's own driver loop followed by its own filter.c.
tests/abi/iqcorr_driver.c is the filter.h driver; its build against the reference's own header declares the extensions
itself, as a patched radiod would.
"""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import iq_correction_ref as R
from test_iq_correction_cpu import HACKRF_FS, HACKRF_SCALE, FUNCUBE_SCALE, funcube_words, hackrf_bytes, ref_lib

ROOT = Path(__file__).resolve().parent.parent
TOL = 1e-5
REC = np.dtype([(k, "<i8") for k in ("seq", "n", "sum_i", "sum_q")] + [(k, "<f8") for k in ("i_energy", "q_energy", "dotprod")]
               + [(k, "<i8") for k in ("overs", "since_over")] + [(k, "<f8") for k in R.STATE])
WRITE = np.dtype([("first", "<i8"), ("n", "<i8"), ("scale", "<f8"), ("m", "<i8", 5), ("overs", "<i8"), ("last_over", "<i8")])


def _driver(name="iqcorr_driver.so"):
    p = (ROOT / "oracle" / "_ref" if "refhdr" in name else ROOT / "tests" / "abi" / "_build") / name
    if not p.exists():
        pytest.skip(f"{name} not built")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.iq_open.restype = vp
    lib.iq_open.argtypes = [i, i, i, i]
    lib.iq_setup.argtypes = [vp, i, vp]
    lib.iq_add_channel.argtypes = [vp, i, d, d, d]
    lib.iq_write_raw.argtypes = [vp, vp, i, i, d]
    lib.iq_write_float.argtypes = [vp, vp, i]
    lib.iq_records.argtypes = [vp, vp, i]
    lib.iq_stats.argtypes = [vp]
    lib.iq_write_from_thread.argtypes = [vp, vp, i, i, C.c_size_t, i, i, d]
    lib.iq_execute.argtypes = [vp, i, i, vp]
    lib.iq_execute_tuned.argtypes = [vp, i, i, d, d, vp, vp]
    lib.iq_drops.argtypes = [vp, i]
    lib.iq_drops.restype = C.c_uint
    lib.iq_enable_noise.argtypes = [vp, d]
    lib.iq_noise.argtypes = [vp, i]
    lib.iq_noise.restype = d
    lib.iq_spec_setup.argtypes = [vp, i, i, vp]
    lib.iq_spec_poll.argtypes = [vp, i, i, d, vp, vp]
    lib.iq_time.argtypes = [vp, vp, i, i, C.c_size_t, i, i, d]
    lib.iq_time.restype = d
    lib.iq_close.argtypes = [vp]
    return lib


def params_array(p: R.Params):
    gp_rate, gp_alpha = (p.gp, 0.0) if p.kind == R.HACKRF else (0.0, p.gp)
    return np.array([p.dc_alpha, gp_rate, gp_alpha] + [p.state[k] for k in R.STATE], np.float64)


class Session:
    def __init__(self, lib, L, M, nworkers=0, cplx=True):
        self.lib, self.L = lib, L
        self.h = lib.iq_open(L, M, int(cplx), nworkers)
        assert self.h, "create_filter_input failed"
        self.olen = []

    def setup(self, fmt, p):
        a = params_array(p)
        return self.lib.iq_setup(self.h, fmt, a.ctypes.data)

    def add(self, olen, low, high, beta):
        i = self.lib.iq_add_channel(self.h, olen, low, high, beta)
        assert i >= 0
        self.olen.append(olen)
        return i

    def raw(self, x, fmt, scale):
        x = np.ascontiguousarray(x)
        return self.lib.iq_write_raw(self.h, x.ctypes.data, x.size // 2, fmt, scale)

    def flt(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        return self.lib.iq_write_float(self.h, x.ctypes.data, len(x))

    def records(self, cap=4096):
        out = np.zeros(cap, REC)
        n = self.lib.iq_records(self.h, out.ctypes.data, cap)
        assert n >= 0
        return out[:n]

    def exe(self, ch, shift):
        y = np.empty(self.olen[ch], np.complex64)
        assert self.lib.iq_execute(self.h, ch, shift, y.ctypes.data) == 0
        return y

    def tuned(self, ch, shift, rem, rate):
        y = np.empty(self.olen[ch], np.complex64)
        pw = C.c_double(0)
        assert self.lib.iq_execute_tuned(self.h, ch, shift, rem, rate, y.ctypes.data, C.byref(pw)) == 0
        return y, pw.value

    def spec_setup(self, fft_n, bin_count, window):
        w = np.ascontiguousarray(window, np.float32)
        assert self.lib.iq_spec_setup(self.h, fft_n, bin_count, w.ctypes.data) == 0

    def spec_poll(self, shift, fft_avg, overlap, bin_count):
        b = np.empty(bin_count, np.float32)
        end = C.c_uint64(0)
        assert self.lib.iq_spec_poll(self.h, shift, fft_avg, overlap, b.ctypes.data, C.byref(end)) == 0
        return b, end.value

    def close(self):
        if self.h:
            self.lib.iq_close(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def check_records(got, want, first=0):
    """device records against the restatement's, bitwise"""
    assert len(got) == len(want)
    for g, r in zip(got, want):
        assert int(g["seq"]) == first and int(g["n"]) == r.n and (int(g["sum_i"]), int(g["sum_q"])) == (r.sum_i, r.sum_q)
        assert (g["i_energy"], g["q_energy"], g["dotprod"]) == (r.i_energy, r.q_energy, r.dotprod) or \
            np.isnan([g["i_energy"], g["q_energy"], g["dotprod"]]).any()
        assert (int(g["overs"]), int(g["since_over"])) == (r.overs, r.since_over)
        assert np.array([g[k] for k in R.STATE]).view(np.uint64).tolist() == \
            np.array([r.state[k] for k in R.STATE]).view(np.uint64).tolist(), first
        first += 1


# ------------------------------------------------------------------ the kernels through the C-ABI --------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.S8, R.S16])
def test_kernels_exact_moments_and_bitwise_records(cuda_dev, fmt):
    """Launches of k = 1..3 blocks of L over ragged writes that straddle blocks and launches: moments exact, records and
    states bitwise the restatement's, floats bitwise, the first window's history exactly 0."""
    import torch

    from ka9q_radio_b200 import capi

    L, M1, cap = 5000, 1200, 64
    rng = np.random.default_rng(7)
    sizes = rng.integers(600, 9000, 40).tolist()
    total = sum(sizes)
    if fmt == R.S8:
        raw = hackrf_bytes(total, seed=3)
        kfmt, p, words = capi.KGPU_IQ_S8, R.Params.hackrf(HACKRF_FS), raw
    else:
        raw = funcube_words(total, over_rate=2e-3)
        kfmt, p, words = capi.KGPU_IQ_S16, R.Params.funcube(960), raw
    writes, o = [], 0
    for s in sizes:
        writes.append(words[2 * o:2 * (o + s)])
        o += s
    scales = [1.0 / (1 + (w % 3)) / 100.0 for w in range(len(sizes))]
    fl, recs = R.run(p, fmt, writes, scales)
    want = np.concatenate(fl)
    firsts = np.concatenate([[0], np.cumsum(sizes)])
    tab = np.zeros(cap, WRITE)
    for w, s in enumerate(sizes):
        tab[w % cap] = (firsts[w], s, scales[w], (0, 0, 0, 0, 0), 0, -1)
    d_tab = torch.from_numpy(tab.view(np.uint8).copy()).to(cuda_dev)
    d_coef = torch.zeros(cap * 8, dtype=torch.float64, device=cuda_dev)
    d_coef[:8] = torch.tensor([p.state[k] for k in R.STATE], dtype=torch.float64)
    d_rec = torch.zeros(cap * REC.itemsize, dtype=torch.uint8, device=cuda_dev)
    pad = np.zeros(2 * M1, words.dtype)
    stream = np.concatenate([pad, words])   # M1 pairs of history before the first write
    issued, scanned, ks = 0, 0, [1, 2, 3, 1, 3, 2, 2, 1, 3]
    kind = capi.IQ_HACKRF if fmt == R.S8 else capi.IQ_FUNCUBE

    def find(a):
        return int(np.searchsorted(firsts[:-1], a, side="right") - 1)

    for k in ks:
        a, end = issued * L, (issued + k) * L
        if end > total:
            break
        win = torch.from_numpy(stream[2 * a: 2 * (end + M1)].copy()).to(cuda_dev)   # pairs [a - M1, end)
        lo, hi = find(a), find(end - 1)
        capi.iq_moments(win.data_ptr() + 2 * M1 * words.itemsize, kfmt, a, end - a, d_tab.data_ptr(), cap, lo, hi - lo + 1)
        done = hi + 1 if firsts[hi + 1] <= end else hi
        capi.iq_scan(d_tab.data_ptr(), d_coef.data_ptr(), cap, scanned, done - scanned, kind, p.dc_alpha, p.gp, d_rec.data_ptr())
        out = torch.full((2 * (end - a + M1),), float("nan"), device=cuda_dev)
        wl = find(max(a - M1, 0))
        capi.iq_apply(win.data_ptr(), kfmt, a - M1, end - a + M1, d_tab.data_ptr(), d_coef.data_ptr(), cap, wl, hi - wl + 1,
                      out.data_ptr())
        torch.cuda.synchronize()
        t = np.frombuffer(d_tab.cpu().numpy().tobytes(), WRITE)
        for w in range(lo, hi + 1):   # the moments of writes complete by now are exact
            if firsts[w + 1] <= end:
                i, q, over = R.words(writes[w], fmt)
                assert tuple(int(v) for v in t[w % cap]["m"]) == R.moments(i, q)
                assert int(t[w % cap]["overs"]) == int(over.sum())
        got_rec = np.frombuffer(d_rec.cpu().numpy().tobytes(), REC)
        check_records([got_rec[w % cap] for w in range(scanned, done)], recs[scanned:done], scanned)
        got = out.cpu().numpy().view(np.complex64)
        if a == 0:
            assert not got[:M1].view(np.uint32).any()   # 0.0f exactly before the first write
            assert same(got[M1:], want[:end])
        else:
            assert same(got, want[a - M1:end])
        issued, scanned = issued + k, done
    assert issued >= 10


# ------------------------------------------------------------------ HackRF through filter.h ------------------------
HACKRF = dict(L=400000, M=100001)
CHANS = [(800, -0.4, 0.4, 11.0, 20000), (4000, -0.45, 0.45, 9.0, -123456), (2000, -0.3, 0.3, 11.0, 333)]


def rhackrf(writes, scales):
    """the reference's own rx_callback: its floats per transfer"""
    lib = ref_lib()
    assert lib.rh_open(HACKRF_FS, 262144, 4097, scales[0]) == 0
    out = []
    try:
        for wr, sc in zip(writes, scales):
            lib.rh_set_scale(sc)
            f, s = np.empty(wr.size // 2, np.complex64), np.empty(8)
            cl, ip = C.c_int(), C.c_double()
            lib.rh_transfer(wr.ctypes.data, wr.size, f.ctypes.data, s.ctypes.data, C.byref(cl), C.byref(ip))
            out.append(f)
    finally:
        lib.rh_close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("driver", ["iqcorr_driver.so", "iqcorr_driver_refhdr.so"])
def test_hackrf_through_filter_h(oracle, cuda_dev, driver):
    """radiod's 20 MS/s HackRF geometry (L = 400 000, M = 100 001) in 131 072-pair transfers, a scale change between two
    writes: channels, a fine-tuned channel and the noise estimates bitwise those of the same library fed the restated
    floats; channels within TOL of the reference's rx_callback followed by its filter.c; records bitwise the
    restatement's, each returned once, up to one launch late."""
    lib = _driver(driver)
    L, M = HACKRF["L"], HACKRF["M"]
    N = L + M - 1
    nw, chunk = 16, 131072
    raw = hackrf_bytes(nw * chunk, seed=11)
    writes = [raw[2 * w * chunk: 2 * (w + 1) * chunk] for w in range(nw)]
    scales = [HACKRF_SCALE] * 9 + [HACKRF_SCALE * 0.25] * (nw - 9)   # from exactly write 9's first sample
    p = R.Params.hackrf(HACKRF_FS)
    fl, recs = R.run(p, R.S8, writes, scales)
    check_ref = driver == "iqcorr_driver.so" and oracle.ref_available()
    ref = oracle.RefSession(L, M, oracle.KO_COMPLEX) if check_ref else None
    rfl = rhackrf(writes, scales) if check_ref else None
    got = []
    with Session(lib, L, M) as a, Session(lib, L, M) as b:
        assert a.setup(R.S8, p) == 0
        for s in (a, b):
            for olen, lo, hi, beta, _ in CHANS:
                s.add(olen, lo, hi, beta)
            s.add(800, -0.3, 0.3, 11.0)          # fine-tuned
            assert s.lib.iq_enable_noise(s.h, HACKRF_FS) == 0
        if ref is not None:
            for olen, lo, hi, beta, _ in CHANS:
                ref.add_channel(olen, lo, hi, beta)
        blocks = 0
        for w in range(nw):
            fa = a.raw(writes[w], R.S8, scales[w])
            assert fa == b.flt(fl[w])
            if ref is not None:
                assert ref.write(rfl[w]) == fa
            while blocks < (w + 1) * chunk // L:
                for ch, (olen, *_, shift) in enumerate(CHANS):
                    ya, yb = a.exe(ch, shift), b.exe(ch, shift)
                    assert same(ya, yb), (w, ch)
                    na = a.lib.iq_noise(a.h, ch)
                    assert na == b.lib.iq_noise(b.h, ch) or np.isnan(na)
                    if ref is not None:
                        r = ref.execute(ch, shift)
                        assert np.abs(ya - r).max() / np.abs(r).max() < TOL, (w, ch)
                _, shift, rem = oracle.compute_tuning(N, HACKRF_FS, 1_234_567.8 + 1000 * w)
                (ya, pa), (yb, pb) = a.tuned(3, shift, rem, 48000.0), b.tuned(3, shift, rem, 48000.0)
                assert same(ya, yb) and pa == pb
                blocks += 1
            got.extend(a.records())   # the launches of this write's blocks have completed: their writes' records are here
            complete = sum(1 for v in range(w + 1) if (v + 1) * chunk <= blocks * L)
            assert len(got) == complete   # every write inside a completed launch, once
        assert a.lib.iq_stats(a.h) == -1   # the records replace filter_ingest_stats
        assert blocks >= 5
    if ref is not None:
        ref.close()
    check_records(got, recs[:len(got)])


@pytest.mark.gpu
def test_hackrf_lapped_slave_and_analyzer(cuda_dev):
    """A consumer that fell ND blocks behind gets zeros and a drop, as on a float-fed master; the wideband analyzer set up
    before the first blocks and one set up after them (seeded through the table of writes) match the float-fed master's."""
    lib = _driver()
    L, M = 36000, 9001
    chunk, nw = 8192, 40
    raw = hackrf_bytes(nw * chunk, seed=4)
    writes = [raw[2 * w * chunk: 2 * (w + 1) * chunk] for w in range(nw)]
    p = R.Params.hackrf(1.8e6)
    fl, _ = R.run(p, R.S8, writes, [HACKRF_SCALE] * nw)
    with Session(lib, L, M, nworkers=1) as a, Session(lib, L, M, nworkers=1) as b:
        assert a.setup(R.S8, p) == 0
        for s in (a, b):
            s.add(480, -0.3, 0.3, 9.0)
        assert lib.iq_write_from_thread(a.h, raw.ctypes.data, chunk, 24, 2 * chunk, 1, R.S8, HACKRF_SCALE) == 0
        flo = np.ascontiguousarray(np.concatenate(fl))
        assert lib.iq_write_from_thread(b.h, flo.ctypes.data, chunk, 24, 8 * chunk, 0, 0, 0.0) == 0
        for _ in range(4):
            assert same(a.exe(0, 1500), b.exe(0, 1500))
        assert lib.iq_drops(a.h, 0) == lib.iq_drops(b.h, 0) >= 1
    fft_n, bins = 4096, 1000
    win = np.hanning(fft_n).astype(np.float32)
    for late in (False, True):
        with Session(lib, L, M) as a, Session(lib, L, M) as b:
            assert a.setup(R.S8, p) == 0
            if not late:
                a.spec_setup(fft_n, bins, win)
                b.spec_setup(fft_n, bins, win)
            for w in range(nw):
                a.raw(writes[w], R.S8, HACKRF_SCALE)
                b.flt(fl[w])
                if late and w == 20:
                    a.spec_setup(fft_n, bins, win)
                    b.spec_setup(fft_n, bins, win)
                if w % 10 == 9 and (not late or w > 20):
                    (ga, ea), (gb, eb) = a.spec_poll(0, 8, 0.5, bins), b.spec_poll(0, 8, 0.5, bins)
                    assert ea == eb and same(ga, gb), (late, w)


# ------------------------------------------------------------------ FUNcube through filter.h -----------------------
@pytest.mark.gpu
def test_funcube_through_filter_h(oracle, cuda_dev):
    """FUNcube at L = 3840 (M = 961) in 960-pair blocks with words at the limits: channels bitwise the float-fed master's
    and within TOL of the reference's proc_funcube followed by its filter.c; records bitwise, overranges and
    samp_since_over exact."""
    lib = _driver()
    L, M, bs, nb = 3840, 961, 960, 200
    words = funcube_words(nb * bs, over_rate=1e-3)
    writes = [words[2 * b * bs: 2 * (b + 1) * bs] for b in range(nb)]
    p = R.Params.funcube(bs)
    fl, recs = R.run(p, R.S16, writes, [FUNCUBE_SCALE] * nb)
    check_ref = oracle.ref_available()
    if check_ref:
        rl = ref_lib()
        rfl = np.empty(nb * bs, np.complex64)
        st, cnt, ifp = np.empty((nb, 8)), np.empty(2 * nb, np.uint64), np.empty(nb)
        assert rl.rf_run(words.ctypes.data, nb, bs, FUNCUBE_SCALE, 8192, 1025, rfl.ctypes.data, st.ctypes.data,
                         cnt.ctypes.data, ifp.ctypes.data) == 0
        ref = oracle.RefSession(L, M, oracle.KO_COMPLEX)
        ref.add_channel(480, -0.2, 0.2, 11.0)
    got = []
    with Session(lib, L, M) as a, Session(lib, L, M) as b:
        assert a.setup(R.S16, p) == 0
        for s in (a, b):
            s.add(480, -0.2, 0.2, 11.0)
        for w in range(nb):
            fa = a.raw(writes[w], R.S16, FUNCUBE_SCALE)
            assert fa == b.flt(fl[w])
            if check_ref:
                assert ref.write(rfl[w * bs:(w + 1) * bs]) == fa
            if fa == 1:
                ya, yb = a.exe(0, 100), b.exe(0, 100)
                assert same(ya, yb), w
                if check_ref:
                    r = ref.execute(0, 100)
                    assert np.abs(ya - r).max() / np.abs(r).max() < TOL, w
            got.extend(a.records())
    if check_ref:
        ref.close()
    check_records(got, recs[:len(got)])
    assert len(got) == nb
    since, overs = 0, 0
    for b, g in enumerate(got):
        since = since + 2 * int(g["n"]) if g["since_over"] < 0 else int(g["since_over"])
        overs += int(g["overs"])
        if check_ref:
            assert (overs, since) == (int(cnt[2 * b]), int(cnt[2 * b + 1]))
    assert overs > 50


# ------------------------------------------------------------------ rejections --------------------------------------
@pytest.mark.gpu
def test_rejections(cuda_dev):
    """A REAL master, a write without setup, a short write, a format mismatch, floats on a corrected master."""
    lib = _driver()
    p = R.Params.hackrf(HACKRF_FS)
    x = hackrf_bytes(4096)
    with Session(lib, 36000, 9001) as a:
        assert a.raw(x, R.S8, 1.0) == -1                         # no setup
        assert a.setup(3, p) == -1                               # FILTER_RAW_S8 has no correction
        assert a.setup(R.S8, p) == 0
        assert a.setup(R.S8, p) == -1                            # once
        assert a.raw(x[:2 * 511], R.S8, 1.0) == -1               # below FILTER_IQ_MIN_WRITE
        assert a.raw(x[:2 * 512], R.S8, 1.0) == 0
        assert a.raw(x.view(np.int16), R.S16, 1.0) == -1         # the other corrected format
        assert a.raw(x, 3, 1.0) == -1                            # an uncorrected one
        assert a.flt(np.zeros(1000, np.complex64)) == -1         # floats
        assert a.records().size == 0
    with Session(lib, 36000, 9001, cplx=False) as r:
        assert r.setup(R.S8, p) == -1                            # a REAL master
        assert r.raw(x, R.S8, 1.0) == -1
        assert r.lib.iq_stats(r.h) == 0                          # and it is left as it was
