"""Channels whose inverse transform length has a prime factor 11, 13, 17, 19 or 23 (kgpu_bank_define_ext,
chan_kernel_ext up to 7260 points, chan_wide_ext up to 28812): the 220 kHz (5500 points) and 277.2 kHz (6930 points)
channels of the HFDL bank at 20 ms and overlap 5, and 8800, 11088, 13860 points at other block times and overlaps.

The method and bounds are those of test_gpu_accuracy.py: every output sample against ifft(exact slice x R) in float64
(max e <= 5e-6, gpu/oracle rms ratio <= 2 and max ratio <= 4), against the oracle at 1e-5 of rms, the output row
pre-filled with a NaN pattern that must survive outside every channel's run.  Tests that transform on the CPU run in a
fresh process (see test_gpu_huge_channels._fresh: the float32 reference keeps at most 64 plan lengths per process).
"""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import rel_err
from test_gpu_accuracy import BEAM_W, MAX_E, NAN_BITS, _beam_slice, _bits, _err, _isb, _score, _sentinel, _slice
from test_filter_abi import TOL, _load
from test_gpu_wide_channels import _mk, _smooth, _sweep_channels

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
HERE = Path(__file__).resolve().parent

MAX_CHAN = 7260       # kMaxChanPoints
MAX_WIDE = 28812      # kMaxWideChanPoints
SMALL = [11, 13, 17, 19, 23, 22, 143, 323, 529, 1331, 2431, 5500, 6930, 7245, 7260]
WIDE = [7280, 8800, 11088, 13860, 28798]


def _fresh(case, *args, env=None):
    """Runs this module's `case(oracle, device, *args)` in a new Python process."""
    code = (f"import sys; sys.path[:0] = [{str(HERE)!r}, {str(ROOT)!r}]\n"
            "import torch\nfrom oracle import oracle as O\nO.lib()\n"
            f"import test_gpu_extended_channels as t\nt.{case}(O, torch.device('cuda:0'), *{args!r})\nprint('case ok')\n")
    full_env = dict(os.environ, **(env or {}))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, env=full_env, capture_output=True, text=True, timeout=1500)
    print(r.stdout)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]


def _smooth23(n):
    for p in (2, 3, 5, 7, 11, 13, 17, 19, 23):
        while n % p == 0:
            n //= p
    return n == 1


def _extended(n):
    return _smooth23(n) and not _smooth(n)


# ------------------------------------------------------------------ per-sample accuracy ------------------------------
@pytest.mark.parametrize("master", ["real", "complex"])
@pytest.mark.parametrize("lengths", [SMALL[:8], SMALL[8:], WIDE], ids=["small", "medium", "wide"])
def test_ext_channel_per_sample_accuracy_and_writes(cuda_dev, lengths, master):
    _fresh("_case_accuracy", lengths, master)


def _case_accuracy(oracle, cuda_dev, lengths, master):
    from ka9q_radio_b200 import capi

    real = master == "real"
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    N = 96000  # N = L (M = 1): a channel's points equal its output length
    for ns in lengths:
        assert _extended(ns), ns
        rng = np.random.default_rng(ns + real)
        chans = _sweep_channels(N, ns, real, rng)
        cz = _mk(N, 1, in_type, cuda_dev, len(chans))
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
                        else:
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
            _score(f"ext {ns} {master}", np.concatenate(e_gpu), np.concatenate(e_ora))
        finally:
            cz.close()


@pytest.mark.parametrize("points", [5500, 6930, 7260, 8800, 13860, 27500])
def test_ext_response_against_design_response(cuda_dev, points):
    """set_filter's forward transform (response_fft_ext / response_wide_ext) against oracle.design_response."""
    _fresh("_case_response", points)


def _case_response(oracle, cuda_dev, points):
    from ka9q_radio_b200 import capi

    L, M = 48000, 12001
    N = L + M - 1
    olen = points * L // N
    assert olen * N // L == points
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, 2)
    try:
        for idx, (lo, hi, beta) in enumerate([(-0.46, 0.46, 11.0), (0.05, 0.3, 5.0)]):
            assert cz.add_channel(olen, 0, lo, hi, beta) == idx
            got = cz.bank.get_response(idx, points)
            ref = oracle.design_response(points, olen, N, True, lo, hi, beta)
            err = np.abs(got - ref).max() / np.abs(ref).max()
            print(f"\nresponse {points} ({lo}, {hi}): max err / max |R| {err:.2e}")
            assert err <= 2e-6, (points, idx, err)
    finally:
        cz.close()


def test_ext_channel_tuned_oscillator_and_power(cuda_dev):
    """The kChanOsc store of chan_kernel_ext and chan_wide_ext across retunes and launches of 1..3 blocks, against the
    oracle's restatement of radio.c:1476-1520; run_one with power gives bitwise the batched output and power."""
    _fresh("_case_osc")


def _case_osc(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M, fs = 48000, 12001, 2.4e6
    N = L + M - 1
    # 220 kHz (5500 points), 277.2 kHz (6930), 8800 and 13860 points
    chans = [(4400, 220000.0, -104 / 220, 104 / 220, 11.0, False), (5544, 277200.0, -136 / 277.2, 136 / 277.2, 11.0, False),
             (7040, 352000.0, -0.45, 0.45, 11.0, True), (11088, 554400.0, -0.45, 0.45, 11.0, False)]
    nb = 6
    plan = [[600_017.3, 412_234.5, 250_123.4, 800_020.0] for _ in range(nb)]
    for b in range(3, nb):
        plan[b][0] += 3_333.3
        plan[b][3] -= 17.25
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.2501, 1.0)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, len(chans))
    lib = capi.load()
    try:
        resp = []
        for c in chans:
            cz.add_channel(c[0], 0, c[2], c[3], c[4], isb=c[5])
            resp.append(oracle.design_response(c[0] * N // L, c[0], N, True, c[2], c[3], c[4]))
        assert [pts for _, pts in cz._olen.values()] == [5500, 6930, 8800, 13860]
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
            if nblk == 3:  # run_one of block 1 with its block counter: bitwise the batch, power included
                for i in range(len(chans)):
                    one = torch.zeros(chans[i][0], dtype=torch.complex64, device=cuda_dev)
                    p1 = torch.zeros(1, dtype=torch.float32, device=cuda_dev)
                    cz.bank.block_counter = b0 + 1
                    capi.check(lib.kgpu_bank_run_one_ex(cz.bank.h, i, spec[1].data_ptr(), one.data_ptr(), p1.data_ptr(), None))
                    torch.cuda.synchronize()
                    assert np.array_equal(_bits(one), _bits(cz.channel_slice(out, i)[1].contiguous())), i
                    assert np.array_equal(_bits(p1), _bits(pw[1, i:i + 1].contiguous())), i
                cz.bank.block_counter = b0 + nblk
            b0 += nblk
        print(f"\nosc ext: worst rel err y {worst_y:.2e}, power {worst_p:.2e}")
        assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)
    finally:
        cz.close()


# ------------------------------------------------------------------ definition ------------------------------------
def test_ext_define_accepted_range(cuda_dev):
    """Every extended length up to 28812 is accepted, as COMPLEX and, when even, as REAL output; every 7-smooth length
    up to 28812 (and a few huge ones) gives what define_huge gives, messages included; a factor 11 above 28812, primes
    above 23 and an odd REAL output are rejected with messages that name the factor."""
    from ka9q_radio_b200 import capi

    m = capi.Master(30000, 1, capi.KGPU_COMPLEX)  # N = L: points = olen
    b = capi.Bank(m, 2)
    lib = capi.load()
    try:
        small = [n for n in range(2, MAX_CHAN + 1) if _extended(n)]
        wide = [n for n in range(MAX_CHAN + 1, MAX_WIDE + 1) if _extended(n)]
        assert len(small) == 863 and len(wide) == 1032 and wide[-1] == 28798
        for n in reversed(small + wide):  # longest first: later definitions reuse the slot's response region
            assert b.define_ext(0, n) == n
            if n % 2 == 0:
                assert b.define_ext(1, n, capi.KGPU_REAL) == n
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define_ext: 30976-point inverse transform has the prime factor 11, "
                                                 "served up to 28812 points only"):
            b.define_ext(0, 30976)  # 2^8 11^2
        for n, p in [(29 * 100, 29), (31 * 64, 31)]:
            with pytest.raises(capi.KgpuError, match=f"kgpu_bank_define_ext: {n}-point inverse transform has the prime factor {p} "):
                b.define_ext(0, n)
        with pytest.raises(capi.KgpuError, match=r"REAL-output slaves need an even number of points \(got 6875\)"):
            b.define_ext(0, 6875, capi.KGPU_REAL)  # 5^4 11
        for n in [n for n in range(1, MAX_WIDE + 1) if _smooth(n)] + [29160, 38400]:
            for ot in (capi.KGPU_COMPLEX, capi.KGPU_REAL):
                rh = lib.kgpu_bank_define_huge(b.h, 0, n, ot)
                eh = lib.kgpu_last_error().decode()
                rx = lib.kgpu_bank_define_ext(b.h, 1, n, ot)
                ex = lib.kgpu_last_error().decode()
                assert rh == rx, n
                if rh < 0:
                    assert eh == ex, (n, eh, ex)
    finally:
        b.close()
        m.close()


def test_ext_plans_take_no_registry_slot(cuda_dev):
    """After every extended length, every 7-smooth length up to 7260 through define and one more master, a bank
    defined before them still matches the oracle: no extended plan took a slot of the plan registry."""
    _fresh("_case_registry")


def _case_registry(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    N = 96000
    rng = np.random.default_rng(3)
    cz = _mk(N, 1, capi.KGPU_REAL, cuda_dev, 2)
    m = capi.Master(30000, 1, capi.KGPU_COMPLEX)
    b = capi.Bank(m, 2)
    try:
        R = [(rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64) for n in (5500, 13860)]
        cz.add_channel(5500, 12345, response=R[0])
        cz.add_channel(13860, -23456, response=R[1])
        X = (rng.standard_normal((1, cz.master.bins)) + 1j * rng.standard_normal((1, cz.master.bins))).astype(np.complex64)
        spec = cz.alloc_spectra(1)
        spec[:, :cz.master.bins] = torch.from_numpy(X).to(cuda_dev)

        def run():
            out = cz.alloc_outputs(1)
            cz.channels(spec, 1, out)
            torch.cuda.synchronize()
            return [cz.channel_slice(out, i).cpu().numpy()[0].copy() for i in range(2)]

        first = run()
        for n in [n for n in range(2, MAX_WIDE + 1) if _extended(n)]:
            assert b.define_ext(0, n) == n
        for n in [n for n in range(1, MAX_CHAN + 1) if _smooth(n)]:
            assert b.define(1, n) == n
        extra = capi.Master(2_744_000, 1, capi.KGPU_COMPLEX)
        extra.close()
        again = run()
        for i, (n, s) in enumerate([(5500, 12345), (13860, -23456)]):
            assert np.array_equal(_bits(torch.from_numpy(first[i])), _bits(torch.from_numpy(again[i]))), n
            ora = oracle.channel_block(capi.KGPU_REAL, X[0], R[i], s)[-n:]
            assert rel_err(again[i], ora) < TOL, n
    finally:
        b.close()
        m.close()
        cz.close()


# ------------------------------------------------------------------ the HFDL bank ----------------------------------
# radiod@kfs-sw.conf.d/51-hfdl.conf: (samprate, low, high, frequency) in Hz, on a 64.8 MS/s RX888 REAL master at 20 ms
# and overlap 5
RX888 = dict(L=1_296_000, M=324_001, fs=64.8e6)
HFDL = [(80e3, -36e3, 36e3, 21964e3), (100e3, -46e3, 46e3, 17944e3), (12e3, 0.0, 3e3, 15025e3),
        (100e3, -47e3, 47e3, 13310e3), (220e3, -104e3, 104e3, 11287e3), (80e3, -35e3, 35e3, 10061.5e3),
        (160e3, -78e3, 78e3, 8902.5e3), (192e3, -93e3, 93e3, 6622e3), (277.2e3, -136e3, 136e3, 5587e3),
        (40e3, -18e3, 18e3, 4672e3), (50e3, -24e3, 24e3, 3477e3), (80e3, -39e3, 39e3, 2980e3)]


def _hfdl_channels(oracle, N, fs, L):
    och, tun = [], []
    for rate, lo, hi, f in HFDL:
        olen = int(round(rate * L / fs))
        rc, shift, rem = oracle.compute_tuning(N, fs, f)
        assert rc == 0
        och.append(dict(olen=olen, shift=shift, low=lo / rate, high=hi / rate, beta=11.0))
        tun.append((shift, rem, rate))
    return och, tun


def _hfdl_stream(fs, nsamp, seed=7):
    """int16 samples: one tone inside every channel plus noise, scaled as the int16 ingest scales them"""
    rng = np.random.default_rng(seed)
    t = np.arange(nsamp) / fs
    x = rng.standard_normal(nsamp) * 300.0
    for k, (rate, lo, hi, f) in enumerate(HFDL):
        x += 2000.0 * np.cos(2 * np.pi * (f + 0.3 * hi + 17.0 * k) * t + k)
    return (np.clip(np.round(x), -32768, 32767) / 32768.0).astype(np.float32)


def test_hfdl_bank_against_the_oracle(cuda_dev):
    """The 12-channel HFDL bank (two extended channels: 5500 and 6930 points), 3 blocks in one kgpu_bank_run, against
    oracle.run_stream and, where it is built, the reference's own filter.c; with the fine-tuning oscillator on, against
    the oracle's restatement of radio.c:1476-1520 (pinned to the reference's downconvert() by test_oracle_ext_cpu.py)
    and, where it is built, against the reference's own downconvert() (the 10 061.5 kHz and 8902.5 kHz channels have a
    20 Hz remainder at 40 Hz bins); the noise estimates of the extended channels against oracle.estimate_noise."""
    _fresh("_case_hfdl_bank")


def _case_hfdl_bank(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M, fs = RX888["L"], RX888["M"], RX888["fs"]
    N = L + M - 1
    nb = 3
    x = _hfdl_stream(fs, nb * L)
    och, tun = _hfdl_channels(oracle, N, fs, L)
    pts = [c["olen"] * N // L for c in och]
    ext = [i for i, p in enumerate(pts) if not _smooth(p)]
    assert [pts[i] for i in ext] == [5500, 6930]
    assert sum(abs(r) > 0 for _, r, _ in tun) >= 2
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, len(och))
    try:
        for c in och:
            cz.add_channel(c["olen"], c["shift"], c["low"], c["high"], c["beta"])
        spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
        cz.forward(cz.stage_stream(x), nb, spec)
        cz.channels(spec, nb, out)
        torch.cuda.synchronize()
        ref, _ = oracle.run_stream(x, L, M, och)
        filt = oracle.ref_run_stream(x, L, M, och)[0] if oracle.ref_available() else None
        for b in range(nb):
            for i in range(len(och)):
                got = cz.channel_slice(out, i).cpu().numpy()[b]
                assert rel_err(got, ref[b][i]) < TOL, (b, i)
                if filt is not None:
                    assert rel_err(got, filt[b][i]) < TOL, ("filter.c", b, i)
        print(f"\nhfdl: reference filter.c {'compared' if filt is not None else 'not built'}")
        # noise of the extended channels
        n0 = torch.full((nb, cz.capacity), float("nan"), dtype=torch.float64, device=cuda_dev)
        cz.bank.noise(spec.data_ptr(), nb, fs, n0.data_ptr(), torch.cuda.current_stream(cuda_dev).cuda_stream)
        torch.cuda.synchronize()
        n0h = n0.cpu().numpy()
        for b in range(nb):
            X = oracle.forward(oracle.block_window(x, L, M, b))
            for i in ext:
                r = oracle.estimate_noise(oracle.KO_REAL, X, pts[i], och[i]["shift"], fs)
                assert abs(n0h[b, i] - r) / r < 1e-5, (b, i, n0h[b, i], r)
        # the same bank with the oscillator on, three blocks in one launch
        resp = [oracle.design_response(p, c["olen"], N, True, c["low"], c["high"], c["beta"]) for p, c in zip(pts, och)]
        fts = [oracle.FineTune(L, M, rate) for _, _, rate in tun]
        for i, (shift, rem, rate) in enumerate(tun):
            cz.tune(i, shift, rem, rate)
        spec, out, pw = cz.alloc_spectra(nb), cz.alloc_outputs(nb), cz.alloc_power(nb)
        cz.forward(cz.stage_stream(x), nb, spec)
        cz.channels(spec, nb, out, pw)
        torch.cuda.synchronize()
        pwh = pw.cpu().numpy()
        worst_y = worst_p = 0.0
        for b in range(nb):
            X = oracle.forward(oracle.block_window(x, L, M, b))
            for i, (shift, rem, rate) in enumerate(tun):
                y = oracle.channel_block(capi.KGPU_REAL, X, resp[i], shift)[-och[i]["olen"]:].copy()
                p_ref = fts[i].block(y, shift, rem)
                worst_y = max(worst_y, rel_err(cz.channel_slice(out, i).cpu().numpy()[b], y))
                worst_p = max(worst_p, abs(pwh[b, i] - p_ref) / p_ref)
        print(f"\nhfdl tuned: worst rel err y {worst_y:.2e}, power {worst_p:.2e}")
        assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)
        if _radio_ref_built():  # the reference's own downconvert(), block by block on the same stream
            worst_y = worst_p = 0.0
            with oracle.RadioRef(L, M, oracle.KO_REAL, fs) as rr:
                for (rate, lo, hi, f), c in zip(HFDL, och):
                    rr.add_channel(c["olen"], rate, f, c["low"], c["high"], c["beta"])
                for b in range(nb):
                    rr.write(x[b * L:(b + 1) * L])
                    for i, (shift, rem, rate) in enumerate(tun):
                        d = rr.downconvert(i)
                        assert d["shift"] == shift and d["remainder"] == rem, (b, i, d["shift"], d["remainder"])
                        worst_y = max(worst_y, rel_err(cz.channel_slice(out, i).cpu().numpy()[b], d["baseband"]))
                        worst_p = max(worst_p, abs(pwh[b, i] - d["bb_power"]) / d["bb_power"])
            print(f"hfdl tuned vs downconvert(): worst rel err y {worst_y:.2e}, power {worst_p:.2e}")
            assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)
        else:
            print("hfdl tuned: the reference's downconvert() is not built")
    finally:
        cz.close()


def _radio_ref_built():
    return (ROOT / "oracle" / "_ref" / "libka9qradio.so").exists()


# ------------------------------------------------------------------ through filter.h ---------------
HFDL_CH = [dict(olen=4400, shift=15000, low=-104 / 220, high=104 / 220, beta=11.0),
           dict(olen=5544, shift=-9000, low=-136 / 277.2, high=136 / 277.2, beta=11.0),
           dict(olen=480, shift=4100, low=-1 / 3, high=1 / 3, beta=11.0)]


@pytest.mark.parametrize("driver", ["driver_gpuhdr.so", "driver_refhdr.so"])
def test_hfdl_slaves_through_filter_h(cuda_dev, driver):
    """create_filter_output at 220 kHz (olen 4400, 5500 points) and 277.2 kHz (olen 5544, 6930 points) next to a 24 kHz
    channel on a 2.4 MS/s REAL master, through the unmodified filter.h calls, against the oracle and, where it is
    built, the reference's own filter.c."""
    if _load(driver) is None:
        pytest.skip(f"{driver} not built")
    _fresh("_case_through_filter_h", driver)


def _case_through_filter_h(oracle, cuda_dev, driver):
    lib = _load(driver)
    L, M, nb = 48000, 12001, 4
    x = oracle.siggen_real(nb * L, 10 ** (-20 / 20), 10 ** (-40 / 20), 0.25, 10 ** (3 / 20))
    got, _ = oracle.ref_run_stream(x, L, M, HFDL_CH, lib=lib)
    ref, _ = oracle.run_stream(x, L, M, HFDL_CH)
    filt = oracle.ref_run_stream(x, L, M, HFDL_CH) if oracle.ref_available() else None
    for b in range(nb):
        for c in range(len(HFDL_CH)):
            assert rel_err(got[b][c], ref[b][c]) < TOL, (b, c)
            if filt is not None:
                assert rel_err(filt[0][b][c], ref[b][c]) < TOL, (b, c)


# ------------------------------------------------------------------ mixed bank ----------------------------------------
def test_ext_channels_in_a_mixed_bank(cuda_dev):
    """Extended channels (5500, 6930, 8800, 11088 points) next to 600 (chan_v2), 1200 (chan_static), 9600 (chan_wide)
    and 38400 (chan_huge) points: the 7-smooth channels' outputs are bitwise those of the bank without the extended
    channels, and kgpu_use_static_kernels(0) leaves the extended channels' outputs bitwise unchanged."""
    from ka9q_radio_b200 import capi

    N, nb = 192000, 3
    rng = np.random.default_rng(21)
    smooth = [(600, 5000), (1200, -30000), (9600, 41000), (38400, -60000)]
    extended = [(5500, 17000), (6930, -21000), (8800, 70000), (11088, -80000)]
    R = {n: (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64) for n, _ in smooth + extended}
    X = (rng.standard_normal((nb, N // 2 + 1)) + 1j * rng.standard_normal((nb, N // 2 + 1))).astype(np.complex64)
    lib = capi.load()

    def run(chans):
        cz = _mk(N, 1, capi.KGPU_REAL, cuda_dev, len(chans))
        try:
            for n, s in chans:
                cz.add_channel(n, s, response=R[n])
            spec = cz.alloc_spectra(nb)
            spec[:, :N // 2 + 1] = torch.from_numpy(X).to(cuda_dev)
            out = cz.alloc_outputs(nb)
            cz.channels(spec, nb, out)
            torch.cuda.synchronize()
            return [_bits(cz.channel_slice(out, i).contiguous()) for i in range(len(chans))]
        finally:
            cz.close()

    both = run(smooth + extended)
    alone = run(smooth)
    for i in range(len(smooth)):
        assert np.array_equal(both[i], alone[i]), smooth[i]
    lib.kgpu_use_static_kernels(0)
    try:
        generic = run(smooth + extended)
    finally:
        lib.kgpu_use_static_kernels(1)
    for i in range(len(smooth), len(smooth) + len(extended)):
        assert np.array_equal(both[i], generic[i]), extended[i - len(smooth)]


# ------------------------------------------------------------------ through filter.h: tuned, batch, retune, laps ----
W220 = (-104 / 220, 104 / 220, 11.0)
W277 = (-136 / 277.2, 136 / 277.2, 11.0)


def test_hfdl_slaves_tuned_batch_retune_and_laps_through_filter_h(cuda_dev):
    """execute_filter_output_tuned (output and block power) with the 220 kHz and 277.2 kHz slaves, including a retune in
    mid-stream: the block issued before the new shift is known misses the batched launch and is recomputed alone
    (kgpu_bank_run_one_ex), and must still match; the default spectrum windows estimate_noise reads;
    execute_filter_output_batch; the lap / drop logic with an extended slave."""
    _fresh("_case_tuned_batch_retune_laps", env={"KA9Q_GPU_SPECTRUM_D2H": ""})


def _case_tuned_batch_retune_laps(oracle, cuda_dev):
    lib = _load("driver_gpuhdr.so")
    L, M, fs = 48000, 12001, 2.4e6
    N = L + M - 1
    nb = 7
    x = oracle.siggen_real(8 * L, 0.1, 0.02, 0.1234, 1.0)
    freqs = [[600_017.3, 412_234.5] for _ in range(nb)]
    for b in range(3, nb):
        freqs[b][0] = 603_350.6  # a new shift: block 3 is recomputed by run_one
    for b in range(5, nb):
        freqs[b][1] = 412_234.5 - 21_000.0  # and block 5 of the other slave
    olen, rate = [4400, 5544], [220000.0, 277200.0]
    R = [oracle.design_response(5500, 4400, N, True, *W220), oracle.design_response(6930, 5544, N, True, *W277)]
    fts = [oracle.FineTune(L, M, r) for r in rate]
    retuned = 0
    with oracle.RefSession(L, M, oracle.KO_REAL, lib=lib) as s:
        ids = [s.add_channel(4400, *W220), s.add_channel(5544, *W277)]
        assert lib.ref_channel_points(s.h, ids[0]) == 5500 and lib.ref_channel_points(s.h, ids[1]) == 6930
        prev = [None, None]
        for b in range(nb):
            assert s.write(x[b * L:(b + 1) * L]) == 1
            X = oracle.forward(oracle.block_window(x, L, M, b))
            shifts = []
            for i in range(2):
                rc, shift, rem = oracle.compute_tuning(N, fs, freqs[b][i])
                retuned += prev[i] is not None and shift != prev[i]
                prev[i] = shift
                shifts.append(shift)
                y = np.empty(olen[i], np.complex64)
                pw = C.c_double(0)
                assert lib.ref_execute_tuned(s.h, ids[i], shift, rem, rate[i], 0.0, y, C.byref(pw)) == 0
                r = oracle.channel_block(oracle.KO_REAL, X, R[i], shift)[-olen[i]:].copy()
                p_ref = fts[i].block(r, shift, rem)
                assert rel_err(y, r) < TOL, (b, i)
                assert abs(pw.value - p_ref) / p_ref < TOL, (b, i)
            if b == 4:  # the windows follow the shifts of the previous block, which block 4 repeats
                host = s.spectrum()
                for sh, pts in zip(shifts, (5500, 6930)):
                    a = oracle.estimate_noise(oracle.KO_REAL, host, pts, sh, fs)
                    ref_n0 = oracle.estimate_noise(oracle.KO_REAL, X, pts, sh, fs)
                    assert abs(a - ref_n0) / ref_n0 < 1e-5, (b, sh)
    assert retuned == 2
    # batch delivery, then a consumer that falls >= ND blocks behind (filter.c:690-701)
    chans = [dict(olen=4400, shift=15000 + 40 * i, low=W220[0], high=W220[1], beta=W220[2]) for i in range(3)]
    chans.append(dict(olen=5544, shift=-9000, low=W277[0], high=W277[1], beta=W277[2]))
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
        y = np.ones(4400, np.complex64)
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 1  # slot of job 2 holds job 6: zeros, a drop
        assert not y.any() and lib.ref_channel_next_job(s.h, 0) == 3
        y[:] = 1
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2  # job 3: its slot holds job 7
        assert not y.any()
        for b in (4, 5, 6, 7):
            assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2
            assert rel_err(y, ref[b][0]) < TOL, b


# ------------------------------------------------------------------ every length: responses and the oscillator -------
def _geometry(p):
    """A COMPLEX master on which a channel of p points has olen = p - q with q | p (q <= p / 5), so that M - 1 = 64 q
    divides L = 64 (p - q) and the oscillator's block step (shift % V) / V is the reference's: L = 64 olen, M = 64 q + 1,
    N = 64 p.  N has p's prime factors, so the master is an extended one."""
    q = max(d for d in range(1, max(1, p // 5) + 1) if p % d == 0)
    return p - q, 64 * (p - q), 64 * q + 1


def _taps(points, olen, N, real, low, high, beta):
    """set_filter's taps (kgpu.cu design_taps, filter.c:968-1030) in float64"""
    low, high = sorted((low, high))
    low, high = min(max(low, -0.5), 0.5), min(max(high, -0.5), 0.5)
    M = points - olen + 1
    half_bw = 1e-4 if high == low else abs(high - low) / 2
    centre = (high + low) / 2
    p = 2.0 / (M - 1) * np.arange(M) - 1
    win = np.i0(beta * np.sqrt(np.clip(1 - p * p, 0, None))) / np.i0(beta)
    win *= M / win.sum()
    n = np.arange(M) - (M - 1) / 2
    rr = win * 2 * half_bw * np.sinc(2 * half_bw * n)
    taps = np.zeros(points, np.complex128)
    taps[:M] = np.exp(1j * np.pi * 2 * centre * n) * rr * ((np.sqrt(2) if real else 1.0) / (rr.sum() * N))
    return taps


def test_ext_response_per_bin_accuracy_every_length(cuda_dev):
    """set_filter's response at every length of the per-sample sweep, bin by bin against the float64 DFT of its taps,
    with the bounds of test_gpu_accuracy.py (e <= 5e-6; gpu/oracle rms ratio <= 2, max ratio <= 4)."""
    _fresh("_case_response_every_length")


def _case_response_every_length(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    for p in SMALL + WIDE:
        olen, L, M = _geometry(p)
        N = L + M - 1
        cz = _mk_ext(L, M, cuda_dev, 2)
        try:
            e_gpu, e_ora = [], []
            for idx, (lo, hi, beta) in enumerate([(-0.46, 0.46, 11.0), (0.05, 0.3, 5.0)]):
                assert cz.add_channel(olen, 0, lo, hi, beta) == idx
                got = cz.bank.get_response(idx, p)
                truth = np.fft.fft(_taps(p, olen, N, False, lo, hi, beta))
                ora = oracle.design_response(p, olen, N, False, lo, hi, beta)
                e_gpu.append(_err(got, truth))
                e_ora.append(_err(ora, truth))
            _score(f"response {p}", np.concatenate(e_gpu), np.concatenate(e_ora))
        finally:
            cz.close()


def _mk_ext(L, M, dev, cap):
    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    return Channelizer(L, M, capi.KGPU_COMPLEX, dev, capacity=cap, extended=True)


def test_ext_oscillator_and_power_every_length(cuda_dev):
    """The kChanOsc store (rotation, per-block phase, block power) at every length of the per-sample sweep, over a
    retune and launches of 1 and 2 blocks, against the oracle's restatement of radio.c:1476-1520."""
    _fresh("_case_osc_every_length")


def _case_osc_every_length(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    worst_y = worst_p = 0.0
    for p in SMALL + WIDE:
        olen, L, M = _geometry(p)
        N = L + M - 1
        fs = 1000.0 * N
        rate = fs * olen / L
        rng = np.random.default_rng(p)
        R = (rng.standard_normal(p) + 1j * rng.standard_normal(p)).astype(np.complex64)
        cz = _mk_ext(L, M, cuda_dev, 1)
        try:
            cz.add_channel(olen, 0, response=R)
            ft = oracle.FineTune(L, M, rate)
            b0 = 0
            for nblk, f in ((1, 0.2345 * fs), (2, -0.3117 * fs)):
                rc, shift, rem = oracle.compute_tuning(N, fs, f)
                assert rc == 0
                cz.tune(0, shift, rem, rate)
                X = (rng.standard_normal((nblk, N)) + 1j * rng.standard_normal((nblk, N))).astype(np.complex64)
                spec, out, pw = cz.alloc_spectra(nblk), cz.alloc_outputs(nblk), cz.alloc_power(nblk)
                spec[:, :N] = torch.from_numpy(X).to(cuda_dev)
                cz.channels(spec, nblk, out, pw)
                torch.cuda.synchronize()
                pwh = pw.cpu().numpy()
                for k in range(nblk):
                    y = oracle.channel_block(capi.KGPU_COMPLEX, X[k], R, shift)[-olen:].copy()
                    p_ref = ft.block(y, shift, rem)
                    worst_y = max(worst_y, rel_err(cz.channel_slice(out, 0).cpu().numpy()[k], y))
                    worst_p = max(worst_p, abs(pwh[k, 0] - p_ref) / p_ref)
                    assert worst_y < TOL and worst_p < TOL, (p, b0 + k, worst_y, worst_p)
                b0 += nblk
        finally:
            cz.close()
    print(f"\nosc every length: worst rel err y {worst_y:.2e}, power {worst_p:.2e}")
