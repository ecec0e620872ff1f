"""Channels whose inverse transform is longer than 7260 points (kgpu_bank_define_wide, chan_wide.cuh): the 384 kHz wfm
downconverter at 9600 (overlap 5) and 15360 (overlap 2) points, wide spectrum-mode slaves.

Accuracy and writes use the method and bounds of test_gpu_accuracy.py: every output sample against ifft(exact slice x R)
in float64 (max e <= 5e-6, gpu/oracle rms ratio <= 2 and max ratio <= 4), against the oracle at 1e-5 of rms, and the
output row pre-filled with a NaN pattern that must survive outside every channel's run.  Parity runs compare whole
banks (wide channels next to 600- and 1200-point ones and a REAL-output slave) with oracle.run_stream, and the filter.h
surface with the oracle and, where it is built, the reference's own filter.c.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_err
from test_gpu_accuracy import BEAM_W, MAX_E, NAN_BITS, _beam_slice, _bits, _err, _isb, _score, _sentinel, _slice
from test_filter_abi import TOL, _load

pytestmark = pytest.mark.gpu

MAX_WIDE = 28812  # kMaxWideChanPoints
WIDE = [7290, 7680, 8192, 9600, 10000, 12005, 15360, 16807, 19683, MAX_WIDE]
NW = 96000  # master of the sweep: N = L (M = 1), so a channel's points equal its output length


@pytest.fixture
def oracle(oracle, tmp_path, monkeypatch):
    """conftest's oracle bound to a private copy of its library: the copy's FFT plan cache (64 lengths per process, full after
    the rest of the suite) starts empty, so the many lengths here fit whatever ran before"""
    import shutil

    orig = oracle.lib()
    src = tmp_path / "libkaoracle_wide.so"
    shutil.copy(oracle.HERE / "libkaoracle.so", src)
    new = C.CDLL(str(src))
    for name, f in vars(orig).items():
        if isinstance(f, C._CFuncPtr):
            g = getattr(new, name)
            g.argtypes, g.restype = f.argtypes, f.restype
    monkeypatch.setattr(oracle, "_lib", new)
    return oracle


def _mk(L, M, in_type, dev, cap):
    from ka9q_radio_b200.channelizer import Channelizer

    return Channelizer(L, M, in_type, dev, capacity=cap)


def _smooth(n):
    for p in (2, 3, 5, 7):
        while n % p == 0:
            n //= p
    return n == 1


def _sweep_channels(N, ns, real, rng):
    """(points, shift, kind) for every slice class of one length"""
    h = N // 2
    inside = int(rng.integers(ns // 2 + 1, h - ns // 2 - 1))
    chans = [(ns, inside, "plain"), (ns, -inside, "plain"),            # REAL: upright / inverted (conjugate walk)
             (ns, 0, "plain"), (ns, ns // 3, "plain"),                  # across bin 0 (REAL: the part below DC is zero)
             (ns, h - ns // 4 - 1, "plain"), (ns, -(h - ns // 4 - 1), "plain"),  # across Nyquist / partly outside
             (ns, int(rng.integers(-h + 1, h)), "isb"), (ns, h - ns // 4 - 1, "isb")]
    if not real:
        chans += [(ns, int(rng.integers(-h + 1, h)), "beam"), (ns, -(h - ns // 4 - 1), "beam"), (ns, 1, "beam")]
    if ns % 2 == 0:
        chans += [(ns, 0, "real"), (ns, inside, "real"), (ns, h - ns // 4 - 1, "real")]
    return chans


@pytest.mark.parametrize("master", ["real", "complex"])
@pytest.mark.parametrize("ns", WIDE)
def test_wide_channel_per_sample_accuracy_and_writes(oracle, cuda_dev, ns, master):
    from ka9q_radio_b200 import capi

    real = master == "real"
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    rng = np.random.default_rng(ns + real)
    chans = _sweep_channels(NW, ns, real, rng)
    cz = _mk(NW, 1, in_type, cuda_dev, len(chans))
    try:
        resp = []
        for pts, s, kind in chans:
            R = (rng.standard_normal(pts) + 1j * rng.standard_normal(pts)).astype(np.complex64)
            resp.append(R)
            assert cz.add_channel(pts, s, response=R, isb=kind == "isb", beam=BEAM_W if kind == "beam" else None,
                                  out_type=capi.KGPU_REAL if kind == "real" else capi.KGPU_COMPLEX) == len(resp) - 1
        bins, nb = cz.master.bins, 2
        X = (rng.standard_normal((nb, bins)) + 1j * rng.standard_normal((nb, bins))).astype(np.complex64)
        spec = _sentinel(nb, cz.master.spec_stride, cuda_dev)
        spec[:, :bins] = torch.from_numpy(X).to(cuda_dev)
        out = _sentinel(nb, cz.bank.out_stride, cuda_dev)
        cz.channels(spec, nb, out)
        torch.cuda.synchronize()
        raw = _bits(out)
        written = np.zeros(raw.shape[1], bool)
        e_gpu, e_ora = [], []
        for i, ((pts, s, kind), R) in enumerate(zip(chans, resp)):
            olen = pts
            off = cz.bank.out_offset(i)
            written[2 * off:2 * off + (olen if kind == "real" else 2 * olen)] = True
            got = cz.channel_slice(out, i).cpu().numpy()
            for b in range(nb):
                if kind == "real":
                    sb = pts // 2 + 1
                    mi = np.arange(sb) + s
                    if real:
                        ok = (mi >= 0) & (mi < bins)
                        V = np.where(ok, X[b][np.clip(mi, 0, bins - 1)].astype(np.complex128), 0)
                    else:  # filter.c:794-809 on a COMPLEX master: X[q] + conj X[-q] inside (-m/2, m/2)
                        ok = (mi >= -(bins // 2)) & (mi < bins // 2)
                        V = np.where(ok, X[b][mi % bins].astype(np.complex128) + np.conj(X[b][(-mi) % bins]), 0)
                    V = V * R[:sb]
                    V[(sb + 1) // 2] = 0
                    truth = (np.fft.irfft(V, pts) * pts)[-olen:]
                    ora = oracle.channel_block_realout(in_type, X[b], R, s)[-olen:]
                else:
                    S = _beam_slice(oracle, X[b], pts, s) if kind == "beam" else _slice(oracle, in_type, X[b], pts, s)
                    S = S * R.astype(np.complex128)
                    if kind == "isb":
                        S = _isb(S)
                    truth = (np.fft.ifft(S) * pts)[-olen:]
                    if kind == "beam":
                        ora = oracle.channel_block_beam(X[b], R, s, *BEAM_W)[-olen:]
                    else:
                        ora = oracle.channel_block(in_type, X[b], R, s, isb=kind == "isb")[-olen:]
                what = (ns, master, s, kind, b)
                if not np.any(truth):
                    assert not np.any(got[b]) and not np.any(ora), what
                    continue
                eg, eo = _err(got[b], truth), _err(ora, truth)
                assert eg.max() <= MAX_E, (what, eg.max())
                assert np.abs(got[b] - ora).max() / np.sqrt(np.mean(np.abs(truth) ** 2)) <= 1e-5, what
                e_gpu.append(eg)
                e_ora.append(eo)
        assert (raw[:, ~written] == NAN_BITS).all(), "store outside a channel's output run"
        _score(f"wide {ns} {master}", np.concatenate(e_gpu), np.concatenate(e_ora))
    finally:
        cz.close()


def test_wide_define_accepted_range(cuda_dev):
    """Every length with factors 2, 3, 5, 7 in (7260, 28812] is accepted; the next one, a factor of 11 and the old entry
    points above 7260 are rejected with their messages; at <= 7260 define_wide is define_ex."""
    from ka9q_radio_b200 import capi

    m = capi.Master(30000, 1, capi.KGPU_COMPLEX)  # N = L: points = olen
    b = capi.Bank(m, 2)
    try:
        lengths = [n for n in range(7261, MAX_WIDE + 1) if _smooth(n)]
        assert len(lengths) == 176
        for n in lengths:
            assert b.define_wide(0, n) == n
            assert b.define_wide(1, n, capi.KGPU_REAL if n % 2 == 0 else capi.KGPU_COMPLEX) == n
        nxt = next(n for n in range(MAX_WIDE + 1, 40000) if _smooth(n))
        assert nxt == 29160
        with pytest.raises(capi.KgpuError, match=f"kgpu_bank_define_wide: {nxt}-point inverse transform exceeds the 28812-point maximum"):
            b.define_wide(0, nxt)
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define_wide: 8800-point transform cannot be split into two plannable lengths"):
            b.define_wide(0, 8800)  # 2^5 5^2 11
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define: 9600-point inverse transform exceeds the 7260-point maximum"):
            b.define(0, 9600)
        with pytest.raises(capi.KgpuError, match=r"REAL-output slaves need an even number of points \(got 7875\)"):
            b.define_wide(0, 7875, capi.KGPU_REAL)
        for n in (2, 7, 600, 1200, 4096, 4800, 7168, 7200):
            assert b.define_wide(0, n) == b.define(1, n) == n
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define: 88-point transform cannot be planned"):
            b.define_wide(0, 88)
    finally:
        b.close()
        m.close()


# (id, real, L, M, fs, [(olen, freq Hz, low, high, beta)]): every bank has 24 kHz fm (600 points at overlap 5),
# 48 kHz (1200 points) and wfm (olen 7680 = 384 kHz x 20 ms)
WFM = (-110 / 384, 110 / 384, 11.0)
MIXED = [
    ("cfg1", True, 48000, 12001, 2.4e6,
     [(7680, 600e3, *WFM), (480, 412_234.5, -1 / 3, 1 / 3, 11.0), (960, 800_000.0, -0.4, 0.4, 7.0), (7680, 150e3, *WFM)]),
    ("iq20M", False, 400000, 100001, 20e6,
     [(7680, 0.0, *WFM), (7680, 55e3, *WFM), (480, -3.1e6, -1 / 3, 1 / 3, 11.0), (960, 6.2e6, -0.4, 0.4, 7.0), (7680, -9.7e6, *WFM)]),
    ("overlap2", True, 48000, 48001, 2.4e6,
     [(7680, 600e3, *WFM), (480, 412_234.5, -1 / 3, 1 / 3, 11.0), (960, 800_000.0, -0.4, 0.4, 7.0)]),
]


@pytest.mark.parametrize("case", MIXED, ids=[c[0] for c in MIXED])
def test_wide_channels_in_a_mixed_bank(oracle, cuda_dev, case):
    """One kgpu_bank_run over wide and ordinary channels and a REAL-output slave against oracle.run_stream; run_one on a
    wide channel gives bitwise the batched output.  Slot 0 is defined at 28800 points, then at an ordinary length, before
    it gets its wfm length, so its response region is reused across the two kernels' ranges."""
    from ka9q_radio_b200 import capi

    name, real, L, M, fs, chans = case
    N = L + M - 1
    nb = 3
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.2501, 1.0) if real else oracle.siggen_complex(nb * L, 0.1, 0.02, 0.0012, 1.0)
    och = []
    for olen, f, lo, hi, beta in chans:
        _, shift, _ = oracle.compute_tuning(N, fs, f)
        och.append(dict(olen=olen, shift=shift, low=lo, high=hi, beta=beta))
    wide = [i for i, c in enumerate(och) if c["olen"] * N // L > 7260]
    assert wide and all(och[i]["olen"] * N // L in (9600, 15360) for i in wide)
    cz = _mk(L, M, in_type, cuda_dev, len(och) + 1)
    try:
        assert cz.bank.define_wide(0, 28800 * L // N) == 28800
        assert cz.bank.define_wide(0, 480) == 480 * N // L
        for c in och:
            cz.add_channel(c["olen"], c["shift"], c["low"], c["high"], c["beta"])
        ro = dict(olen=480, shift=0, low=50 / 24000, high=0.3125, beta=11.0)  # wfm.c:76-77's REAL slave, on the same bank
        cz.add_channel(ro["olen"], ro["shift"], ro["low"], ro["high"], ro["beta"], out_type=capi.KGPU_REAL)
        spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
        cz.forward(cz.stage_stream(x), nb, spec)
        cz.channels(spec, nb, out)
        torch.cuda.synchronize()
        ref, _ = oracle.run_stream(x, L, M, och)
        Rro = oracle.design_response_realout(480 * N // L, 480, N, real, ro["low"], ro["high"], ro["beta"])
        for b in range(nb):
            X = oracle.forward(oracle.block_window(x, L, M, b))
            for i in range(len(och)):
                assert rel_err(cz.channel_slice(out, i).cpu().numpy()[b], ref[b][i]) < TOL, (name, b, i)
            r = oracle.channel_block_realout(in_type, X, Rro, 0)[-480:]
            assert rel_err(cz.channel_slice(out, len(och)).cpu().numpy()[b], r) < TOL, (name, b)
        for i in wide:
            one = torch.zeros(och[i]["olen"], dtype=torch.complex64, device=cuda_dev)
            cz.bank.run_one(i, spec[1].data_ptr(), one.data_ptr())
            torch.cuda.synchronize()
            assert np.array_equal(_bits(one), _bits(cz.channel_slice(out, i)[1].contiguous())), (name, i)
    finally:
        cz.close()


def test_wide_channel_tuned_oscillator_and_power(oracle, cuda_dev):
    """The kChanOsc store of chan_wide (rotation, per-block phase, power reduced over the CTA) across retunes and launches
    of 1..3 blocks, against the oracle's restatement of radio.c:1476-1520, next to an ordinary tuned channel."""
    from ka9q_radio_b200 import capi

    L, M, fs = 48000, 12001, 2.4e6
    N = L + M - 1
    chans = [(7680, 384000.0, *WFM, False), (480, 24000.0, -1 / 3, 1 / 3, 11.0, False), (7680, 384000.0, -0.2, 0.2, 5.0, True)]
    nb = 6
    plan = [[600_017.3, 412_234.5, 250_123.4] for _ in range(nb)]
    for b in range(3, nb):
        plan[b][0] += 3_333.3
        plan[b][2] -= 17.25
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.2501, 1.0)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, len(chans))
    try:
        resp = []
        for c in chans:
            cz.add_channel(c[0], 0, c[2], c[3], c[4], isb=c[5])
            resp.append(oracle.design_response(c[0] * N // L, c[0], N, True, c[2], c[3], c[4]))
        fts = [oracle.FineTune(L, M, c[1]) for c in chans]
        d = cz.stage_stream(x)
        worst_y, worst_p, b0 = 0.0, 0.0, 0
        for nblk in (1, 2, 3):
            tun = []
            for i, c in enumerate(chans):
                rc, shift, rem = oracle.compute_tuning(N, fs, plan[b0][i])
                assert rc == 0
                cz.tune(i, shift, rem, c[1])
                tun.append((shift, rem))
            spec, out, pw = cz.alloc_spectra(nblk), cz.alloc_outputs(nblk), cz.alloc_power(nblk)
            cz.forward(d, nblk, spec, first_block=b0)
            cz.channels(spec, nblk, out, pw)
            torch.cuda.synchronize()
            pwh = pw.cpu().numpy()
            for k in range(nblk):
                X = oracle.forward(oracle.block_window(x, L, M, b0 + k))
                for i, c in enumerate(chans):
                    y = oracle.channel_block(capi.KGPU_REAL, X, resp[i], tun[i][0], c[5])[-c[0]:].copy()
                    p_ref = fts[i].block(y, tun[i][0], tun[i][1])
                    worst_y = max(worst_y, rel_err(cz.channel_slice(out, i).cpu().numpy()[k], y))
                    worst_p = max(worst_p, abs(pwh[k, i] - p_ref) / p_ref)
            b0 += nblk
        assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)
    finally:
        cz.close()


# ------------------------------------------------------------------ through filter.h ---------------
CFG1 = dict(L=48000, M=12001, fs=2.4e6)
CFG1_CHANS = [dict(olen=7680, shift=15000, low=WFM[0], high=WFM[1], beta=11.0),
              dict(olen=480, shift=-9000, low=-1 / 3, high=1 / 3, beta=11.0),
              dict(olen=7680, shift=-4100, low=WFM[0], high=WFM[1], beta=11.0, isb=True),
              dict(olen=960, shift=20000, low=-0.4, high=0.4, beta=7.0)]


@pytest.mark.parametrize("driver,zerocopy", [("driver_gpuhdr.so", "0"), ("driver_gpuhdr.so", "1"), ("driver_refhdr.so", "0")])
def test_wfm_slave_through_filter_h(oracle, cuda_dev, driver, zerocopy, monkeypatch):
    """create_filter_output at wfm's rate on cfg-1 (9600 points) through the unmodified filter.h calls, copy and
    zero-copy delivery, against the oracle and, where it is built, the reference's own filter.c."""
    monkeypatch.setenv("KA9Q_GPU_ZEROCOPY", zerocopy)
    lib = _load(driver)
    if lib is None:
        pytest.skip(f"{driver} not built")
    L, M = CFG1["L"], CFG1["M"]
    x = oracle.siggen_real(4 * L, 10 ** (-20 / 20), 10 ** (-40 / 20), 0.25, 10 ** (3 / 20))
    got, _ = oracle.ref_run_stream(x, L, M, CFG1_CHANS, lib=lib)
    ref, _ = oracle.run_stream(x, L, M, CFG1_CHANS)
    filt = oracle.ref_run_stream(x, L, M, CFG1_CHANS) if oracle.ref_available() else None
    for b in range(4):
        for c in range(len(CFG1_CHANS)):
            assert rel_err(got[b][c], ref[b][c]) < TOL, (b, c)
            if filt is not None:
                assert rel_err(filt[0][b][c], ref[b][c]) < TOL, (b, c)


def test_wfm_slave_tuned_batch_windows_and_laps_through_filter_h(oracle, cuda_dev, monkeypatch):
    """execute_filter_output_tuned (output and block power), the default spectrum windows estimate_noise reads,
    execute_filter_output_batch and the lap / drop logic, each with a wfm slave."""
    monkeypatch.delenv("KA9Q_GPU_SPECTRUM_D2H", raising=False)
    lib = _load("driver_gpuhdr.so")
    L, M, fs = CFG1["L"], CFG1["M"], CFG1["fs"]
    N = L + M - 1
    nb = 6
    x = oracle.siggen_real(8 * L, 0.1, 0.02, 0.1234, 1.0)
    freqs = [[600_017.3, 412_234.5] for _ in range(nb)]
    for b in range(3, nb):
        freqs[b][0] = 603_350.6
    olen, rate = [7680, 480], [384000.0, 24000.0]
    R = [oracle.design_response(9600, 7680, N, True, WFM[0], WFM[1], 11.0), oracle.design_response(600, 480, N, True, -1 / 3, 1 / 3, 11.0)]
    fts = [oracle.FineTune(L, M, r) for r in rate]
    with oracle.RefSession(L, M, oracle.KO_REAL, lib=lib) as s:
        ids = [s.add_channel(7680, WFM[0], WFM[1], 11.0), s.add_channel(480, -1 / 3, 1 / 3, 11.0)]
        assert lib.ref_channel_points(s.h, ids[0]) == 9600
        for b in range(nb):
            assert s.write(x[b * L:(b + 1) * L]) == 1
            X = oracle.forward(oracle.block_window(x, L, M, b))
            shifts = []
            for i in range(2):
                rc, shift, rem = oracle.compute_tuning(N, fs, freqs[b][i])
                shifts.append(shift)
                y = np.empty(olen[i], np.complex64)
                pw = C.c_double(0)
                assert lib.ref_execute_tuned(s.h, ids[i], shift, rem, rate[i], 0.0, y, C.byref(pw)) == 0
                r = oracle.channel_block(oracle.KO_REAL, X, R[i], shift)[-olen[i]:].copy()
                p_ref = fts[i].block(r, shift, rem)
                assert rel_err(y, r) < TOL, (b, i)
                assert abs(pw.value - p_ref) / p_ref < TOL, (b, i)
            if b >= 1:  # the windows follow the shifts of the previous block, which are the same from block 4 on
                host = s.spectrum()
                if b >= 4:
                    for sh, pts in zip(shifts, (9600, 600)):
                        a = oracle.estimate_noise(oracle.KO_REAL, host, pts, sh, fs)
                        ref_n0 = oracle.estimate_noise(oracle.KO_REAL, X, pts, sh, fs)
                        assert abs(a - ref_n0) / ref_n0 < 1e-5, (b, sh)
    # batch delivery, then a consumer that falls >= ND blocks behind (filter.c:690-701)
    chans = [dict(olen=7680, shift=15000 + 40 * i, low=WFM[0], high=WFM[1], beta=11.0) for i in range(3)]
    chans.append(dict(olen=480, shift=-9000, low=-1 / 3, high=1 / 3, beta=11.0))
    ref, _ = oracle.run_stream(x, L, M, chans)
    with oracle.RefSession(L, M, oracle.KO_REAL, nworkers=1, lib=lib) as s:
        for ch in chans:
            s.add_channel(ch["olen"], ch["low"], ch["high"], ch["beta"])
        shifts = (C.c_int * len(chans))(*[ch["shift"] for ch in chans])
        outs = [np.zeros(ch["olen"], np.complex64) for ch in chans]
        ptrs = (C.c_void_p * len(chans))(*[o.ctypes.data for o in outs])
        for b in range(2):
            assert lib.ref_produce_from_thread(s.h, np.ascontiguousarray(x[b * L:(b + 1) * L]), 1) == 0
            assert lib.ref_execute_batch(s.h, C.cast(shifts, C.c_void_p), C.cast(ptrs, C.c_void_p)) == 0
            for c in range(len(chans)):
                assert rel_err(outs[c], ref[b][c]) < TOL, (b, c)
        assert lib.ref_produce_from_thread(s.h, np.ascontiguousarray(x[2 * L:8 * L]), 6) == 0  # jobs 2..7, consumer at 2
        y = np.ones(7680, np.complex64)
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 1  # slot of job 2 holds job 6: zeros, a drop
        assert not y.any() and lib.ref_channel_next_job(s.h, 0) == 3
        y[:] = 1
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2  # job 3: its slot holds job 7
        assert not y.any()
        for b in (4, 5, 6, 7):
            assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2
            assert rel_err(y, ref[b][0]) < TOL, b
