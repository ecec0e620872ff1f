"""Channels of any point count (kgpu_bank_define_any, bluestein_chan.cuh): lengths with a prime factor >= 29, such as the
29 kHz (725 points) and 62 kHz (1550 points) channels at 20 ms and overlap 5, and lengths above 28812 points with a
prime factor 11 .. 23, such as a 1.76 MS/s channel (44000 points), run a Bluestein transform.

Per-sample accuracy uses the metric of tests/test_gpu_bluestein_masters.py: e = |gpu - truth| / rms(truth) against
ifft(exact slice x R) in float64; max e <= 5e-6, and rms(e_gpu) <= 3 rms(e_oracle) against the float32 oracle.  Output
rows are pre-filled with a NaN pattern that must survive outside every channel's run.  Every case that transforms on
the CPU runs in a process of its own (see test_gpu_extended_channels._fresh).
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
from test_filter_abi import TOL, _load
from test_gpu_accuracy import BEAM_W, MAX_E, NAN_BITS, _beam_slice, _bits, _err, _isb, _sentinel, _slice
from test_gpu_extended_channels import _taps
from test_gpu_wide_channels import _mk, _sweep_channels

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
HERE = Path(__file__).resolve().parent
OSC = (0.123, 0.0123, 1e-9, 0.25)  # phase, freq, rate, block step of the oscillator channels (kgpu_bank_set_osc)


def _fresh(case, *args, env=None):
    """Runs this module's `case(oracle, device, *args)` in a new Python process."""
    code = (f"import sys; sys.path[:0] = [{str(HERE)!r}, {str(ROOT)!r}]\n"
            "import torch\nfrom oracle import oracle as O\nO.lib()\n"
            f"import test_gpu_bluestein_channels as t\nt.{case}(O, torch.device('cuda:0'), *{args!r})\nprint('case ok')\n")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **(env or {})), capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]


def _score(what, e_gpu, e_ora):
    r_rms = np.sqrt(np.mean(e_gpu ** 2)) / np.sqrt(np.mean(e_ora ** 2))
    print(f"accuracy {what}: max e {e_gpu.max():.2e} (oracle {e_ora.max():.2e}), gpu/oracle rms {r_rms:.2f}")
    assert e_gpu.max() <= MAX_E, (what, e_gpu.max())
    if e_gpu.size >= 4096:
        assert r_rms <= 3.0, (what, r_rms)


def _osc_phase(k, olen):
    """kgpu_bank_set_osc's phase of every sample of the k-th block after the call, in float64 cycles"""
    phase, freq, rate, adj = OSC
    m = k * olen + np.arange(olen, dtype=np.float64)
    return phase + (k + 1) * adj + m * freq + 0.5 * m * (m + 1.0) * rate


# ------------------------------------------------------------------ per-sample accuracy ------------------------------
# (lengths, master N): N > 2 points + 4 keeps every slice class of _sweep_channels in range
LENGTHS = {"primes_small": ([29, 185, 725, 1550], 96000), "primes_7919": ([7919, 15838], 96000),
           "above_28812": ([44000, 62000], 192000), "top": ([1048573], 2_400_000)}


@pytest.mark.parametrize("master", ["real", "complex"])
@pytest.mark.parametrize("lengths", list(LENGTHS))
def test_bluestein_channel_per_sample_accuracy_and_writes(cuda_dev, lengths, master):
    _fresh("_case_accuracy", lengths, master)


def _case_accuracy(oracle, cuda_dev, lengths, master):
    import scipy.fft
    from ka9q_radio_b200 import capi

    real = master == "real"
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    sizes, N = LENGTHS[lengths]
    for ns in sizes:
        assert capi.chan_plan(ns)[0] == capi.CHAN_BLUESTEIN, ns
        rng = np.random.default_rng(ns + real)
        chans = _sweep_channels(N, ns, real, rng) + [(ns, int(rng.integers(-N // 4, N // 4)), "osc")]
        cz = _mk(N, 1, in_type, cuda_dev, len(chans))
        try:
            resp = []
            for i, (pts, s, kind) in enumerate(chans):
                R = (rng.standard_normal(pts) + 1j * rng.standard_normal(pts)).astype(np.complex64)
                resp.append(R)
                assert cz.add_channel(pts, s, response=R, isb=kind == "isb", beam=BEAM_W if kind == "beam" else None,
                                      out_type=capi.KGPU_REAL if kind == "real" else capi.KGPU_COMPLEX) == i
                if kind == "osc":
                    cz.bank.set_osc(i, True, *OSC)
            bins, nb = cz.master.bins, 2
            X = (rng.standard_normal((nb, bins)) + 1j * rng.standard_normal((nb, bins))).astype(np.complex64)
            spec = _sentinel(nb, cz.master.spec_stride, cuda_dev)
            spec[:, :bins] = torch.from_numpy(X).to(cuda_dev)
            out = _sentinel(nb, cz.bank.out_stride, cuda_dev)
            pw = cz.alloc_power(nb)
            cz.channels(spec, nb, out, pw)
            torch.cuda.synchronize()
            raw, pwh = _bits(out), pw.cpu().numpy()
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
                        truth = np.fft.irfft(V, pts) * pts
                        ora = (scipy.fft.irfft(V.astype(np.complex64), pts) * np.float32(pts) if pts > 100_000
                               else oracle.channel_block_realout(in_type, X[b], R, s))
                    else:
                        S = _beam_slice(oracle, X[b], pts, s) if kind == "beam" else _slice(oracle, in_type, X[b], pts, s)
                        S = S * R.astype(np.complex128)
                        if kind == "isb":
                            S = _isb(S)
                        truth = np.fft.ifft(S) * pts
                        if pts > 100_000:  # the oracle's prime leaf is O(n^2): scipy's float32 transform instead
                            ora = scipy.fft.ifft(S.astype(np.complex64)) * np.float32(pts)
                        elif kind == "beam":
                            ora = oracle.channel_block_beam(X[b], R, s, *BEAM_W)
                        else:
                            ora = oracle.channel_block(in_type, X[b], R, s, isb=kind == "isb")
                    truth, ora = truth[-olen:], ora[-olen:]
                    if kind == "osc":
                        rot = np.exp(2j * np.pi * _osc_phase(b, olen))
                        truth, ora = truth * rot, ora * rot
                        p_ref = np.mean(np.abs(truth) ** 2)
                        assert abs(pwh[b, i] - p_ref) / p_ref < TOL, (ns, master, b, pwh[b, i], p_ref)
                    what = (ns, master, s, kind, b)
                    if not np.any(truth):
                        assert not np.any(got[b]), what
                        continue
                    eg, eo = _err(got[b], truth), _err(ora, truth)
                    assert eg.max() <= MAX_E, (what, eg.max())
                    e_gpu.append(eg)
                    e_ora.append(eo)
            assert (raw[:, ~written] == NAN_BITS).all(), "store outside a channel's output run"
            _score(f"bluestein {ns} {master}", np.concatenate(e_gpu), np.concatenate(e_ora))
        finally:
            cz.close()


# ------------------------------------------------------------------ responses ----------------------------------------
@pytest.mark.parametrize("points", [29, 185, 725, 1550, 7919, 44000, 62000])
def test_bluestein_response_per_bin_accuracy(cuda_dev, points):
    """set_filter's forward transform of a Bluestein channel, bin by bin against the float64 DFT of its taps."""
    _fresh("_case_response", points)


def _case_response(oracle, cuda_dev, points):
    from ka9q_radio_b200 import capi

    # a COMPLEX master of N = 64 points on which the channel keeps olen = points - points // 5 samples: points // 5 + 1
    # taps, as at overlap 5 (a prime point count would leave _geometry's master two taps, whose DFT is degenerate)
    olen = points - points // 5
    L, M = 64 * olen, 64 * (points - olen) + 1
    N = L + M - 1
    assert olen * N // L == points and olen * N % L == 0
    m = capi.Master(L, M, capi.KGPU_COMPLEX, any_length=True)
    b = capi.Bank(m, 2)
    try:
        e_gpu, e_ora = [], []
        for idx, (lo, hi, beta) in enumerate([(-0.46, 0.46, 11.0), (0.05, 0.3, 5.0)]):
            assert b.define_any(idx, olen) == points
            b.set_filter(idx, lo, hi, beta)
            got = b.get_response(idx, points)
            truth = np.fft.fft(_taps(points, olen, N, False, lo, hi, beta))
            e_gpu.append(_err(got, truth))
            e_ora.append(_err(oracle.design_response(points, olen, N, False, lo, hi, beta), truth))
        _score(f"response {points}", np.concatenate(e_gpu), np.concatenate(e_ora))
    finally:
        b.close()
        m.close()


# ------------------------------------------------------------------ mixed banks against the oracle -------------------
# (olen, low, high): 24 kHz (600 points, direct), 384 kHz (9600, wide), 1.536 MS/s (38400, huge), 220 kHz (5500,
# extended), then the Bluestein ones: 29 kHz (725), 62 kHz (1550), 1.76 MS/s (44000) at 20 ms and overlap 5
SMOOTH_CH = [(480, -0.4, 0.4), (7680, -110 / 384, 110 / 384), (30720, -0.45, 0.45), (4400, -104 / 220, 104 / 220)]
BLUE_CH = [(580, -13 / 29, 13 / 29), (1240, -0.45, 0.45), (35200, -0.45, 0.45)]
MASTERS = {"real": (1_296_000, 324_001, 64.8e6), "complex": (48_000, 12_001, 2.4e6)}


@pytest.mark.parametrize("master", ["real", "complex"])
def test_mixed_bank_against_the_oracle(cuda_dev, master):
    """Direct, wide, huge, extended and Bluestein channels in one bank, 3 blocks in one launch: outputs against
    oracle.run_stream and, where it is built, the reference's own filter.c; the noise estimates against
    oracle.estimate_noise; with the oscillator on, outputs and power against the oracle's restatement of
    radio.c:1476-1520 and, where it is built, the reference's own downconvert(); every non-Bluestein channel's output
    bitwise that of the bank without the Bluestein channels."""
    _fresh("_case_mixed", master)


def _case_mixed(oracle, cuda_dev, master):
    from ka9q_radio_b200 import capi

    real = master == "real"
    L, M, fs = MASTERS[master]
    N = L + M - 1
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    nb = 3
    half = fs / 2
    freqs = [0.1 * half * (k + 1) + 1234.5 * k - (0 if real else 0.5 * half) for k in range(len(SMOOTH_CH + BLUE_CH))]
    chans = []
    for (o, lo, hi), f in zip(SMOOTH_CH + BLUE_CH, freqs):
        rc, shift, rem = oracle.compute_tuning(N, fs, f)
        assert rc == 0
        chans.append(dict(olen=o, shift=shift, low=lo, high=hi, beta=11.0, rem=rem, f=f))
    pts = [c["olen"] * N // L for c in chans]
    assert pts == [600, 9600, 38400, 5500, 725, 1550, 44000], pts
    paths = [capi.chan_plan(p)[0] for p in pts]
    assert paths == [0, 1, 2, 3, 4, 4, 4], paths
    x = (oracle.siggen_real(nb * L, 0.1, 0.02, 0.2501, 1.0) if real
         else oracle.siggen_complex(nb * L, 0.1, 0.02, 0.1234, 1.0))
    nsm = len(SMOOTH_CH)

    def run(cs, tuned=False):
        cz = _mk(L, M, in_type, cuda_dev, len(cs))
        try:
            for c in cs:
                cz.add_channel(c["olen"], c["shift"], c["low"], c["high"], c["beta"])
            if tuned:
                for i, c in enumerate(cs):
                    cz.tune(i, c["shift"], c["rem"], c["olen"] * fs / L)
            spec, out, pw = cz.alloc_spectra(nb), cz.alloc_outputs(nb), cz.alloc_power(nb)
            cz.forward(cz.stage_stream(x), nb, spec)
            cz.channels(spec, nb, out, pw)
            n0 = cz.noise(spec, nb, fs)
            torch.cuda.synchronize()
            return ([cz.channel_slice(out, i).cpu().numpy().copy() for i in range(len(cs))], pw.cpu().numpy(),
                    n0.cpu().numpy())
        finally:
            cz.close()

    got, _, n0 = run(chans)
    alone, _, _ = run(chans[:nsm])
    for i in range(nsm):
        assert np.array_equal(got[i].view(np.int32), alone[i].view(np.int32)), pts[i]
    ref, spectra = oracle.run_stream(x, L, M, chans, keep_spectra=True)
    filt = oracle.ref_run_stream(x, L, M, chans)[0] if oracle.ref_available() else None
    ko = oracle.KO_REAL if real else oracle.KO_COMPLEX
    for b in range(nb):
        for i in range(len(chans)):
            assert rel_err(got[i][b], ref[b][i]) < TOL, (b, pts[i])
            if filt is not None:
                assert rel_err(got[i][b], filt[b][i]) < TOL, ("filter.c", b, pts[i])
        for i in range(nsm, len(chans)):
            r = oracle.estimate_noise(ko, spectra[b], pts[i], chans[i]["shift"], fs)
            assert abs(n0[b, i] - r) / r < 1e-5, (b, pts[i], n0[b, i], r)
    print(f"\nmixed {master}: reference filter.c {'compared' if filt is not None else 'not built'}")
    # the oscillator on: outputs and power
    tgot, pwh, _ = run(chans, tuned=True)
    resp = [oracle.design_response(p, c["olen"], N, real, c["low"], c["high"], c["beta"]) for p, c in zip(pts, chans)]
    fts = [oracle.FineTune(L, M, c["olen"] * fs / L) for c in chans]
    worst_y = worst_p = 0.0
    for b in range(nb):
        for i, c in enumerate(chans):
            y = oracle.channel_block(ko, spectra[b], resp[i], c["shift"])[-c["olen"]:].copy()
            p_ref = fts[i].block(y, c["shift"], c["rem"])
            worst_y = max(worst_y, rel_err(tgot[i][b], y))
            worst_p = max(worst_p, abs(pwh[b, i] - p_ref) / p_ref)
    print(f"mixed {master} tuned: worst rel err y {worst_y:.2e}, power {worst_p:.2e}")
    assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)
    if real and (ROOT / "oracle" / "_ref" / "libka9qradio.so").exists():
        worst_y = worst_p = 0.0
        with oracle.RadioRef(L, M, ko, fs) as rr:
            for c in chans:
                rr.add_channel(c["olen"], c["olen"] * fs / L, c["f"], c["low"], c["high"], c["beta"])
            for b in range(nb):
                rr.write(x[b * L:(b + 1) * L])
                for i, c in enumerate(chans):
                    d = rr.downconvert(i)
                    assert d["shift"] == c["shift"] and d["remainder"] == c["rem"], (b, i)
                    worst_y = max(worst_y, rel_err(tgot[i][b], d["baseband"]))
                    worst_p = max(worst_p, abs(pwh[b, i] - d["bb_power"]) / d["bb_power"])
        print(f"mixed {master} tuned vs downconvert(): worst rel err y {worst_y:.2e}, power {worst_p:.2e}")
        assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)


# ------------------------------------------------------------------ run_one, chunks and streams ----------------------
def test_run_one_chunks_and_streams_are_bitwise(cuda_dev):
    """run_one equals the batched launch bitwise (output and power); a launch of 1 048 573-point channels that runs in
    several scratch chunks equals launches of one block each; a batched launch on one stream overlapped with run_one on
    another gives what they give one after the other."""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    N, nb = 2_400_000, 4
    rng = np.random.default_rng(5)
    chans = [(1_048_573, 300_000, True), (1_048_573, -200_000, False), (725, 50_000, True), (44000, 400_000, False),
             (1_048_573, 1_100_000, False)]
    cz = _mk(N, 1, capi.KGPU_REAL, cuda_dev, len(chans))
    try:
        for i, (p, s, osc) in enumerate(chans):
            R = (rng.standard_normal(p) + 1j * rng.standard_normal(p)).astype(np.complex64)
            cz.add_channel(p, s, response=R)
            if osc:
                cz.bank.set_osc(i, True, *OSC)
        bins = cz.master.bins
        X = (rng.standard_normal((nb, bins)) + 1j * rng.standard_normal((nb, bins))).astype(np.complex64)
        spec = cz.alloc_spectra(nb)
        spec[:, :bins] = torch.from_numpy(X).to(cuda_dev)
        cz.bank.block_counter = 0
        out, pw = _sentinel(nb, cz.bank.out_stride, cuda_dev), cz.alloc_power(nb)
        cz.channels(spec, nb, out, pw)  # 3 x 4 rows of the longest length: several chunks
        torch.cuda.synchronize()
        for b in range(nb):  # one block per launch: one chunk
            cz.bank.block_counter = b
            o1, p1 = _sentinel(1, cz.bank.out_stride, cuda_dev), cz.alloc_power(1)
            cz.channels(spec[b:b + 1], 1, o1, p1)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(o1)[0], _bits(out)[b]), b
            assert np.array_equal(_bits(p1)[0], _bits(pw)[b]), b
        for i, (p, _, osc) in enumerate(chans):  # run_one of every channel and block
            for b in range(nb):
                cz.bank.block_counter = b
                one = torch.zeros(p, dtype=torch.complex64, device=cuda_dev)
                p1 = torch.zeros(1, dtype=torch.float32, device=cuda_dev)
                capi.check(lib.kgpu_bank_run_one_ex(cz.bank.h, i, spec[b].data_ptr(), one.data_ptr(), p1.data_ptr(), None))
                torch.cuda.synchronize()
                assert np.array_equal(_bits(one), _bits(cz.channel_slice(out, i)[b].contiguous())), (i, b)
                if osc:
                    assert np.array_equal(_bits(p1), _bits(pw[b, i:i + 1].contiguous())), (i, b)
        # overlapped: a batched launch on s1 and run_one of two channels on s2, enqueued together
        s1, s2 = torch.cuda.Stream(cuda_dev), torch.cuda.Stream(cuda_dev)
        cz.bank.block_counter = 0
        capi.check(lib.kgpu_bank_commit(cz.bank.h, None))
        torch.cuda.synchronize()
        o_b, p_b = _sentinel(nb, cz.bank.out_stride, cuda_dev), cz.alloc_power(nb)
        ones = [torch.zeros(p, dtype=torch.complex64, device=cuda_dev) for p in (chans[2][0], chans[0][0])]
        for rep in range(2):
            capi.check(lib.kgpu_bank_run_ex(cz.bank.h, spec.data_ptr(), nb, o_b.data_ptr(), 0, p_b.data_ptr(), s1.cuda_stream))
            cz.bank.block_counter = 1  # run_one takes block 1 of the oscillator
            for o, idx in zip(ones, (2, 0)):
                capi.check(lib.kgpu_bank_run_one(cz.bank.h, idx, spec[1].data_ptr(), o.data_ptr(), s2.cuda_stream))
            cz.bank.block_counter = 0
            torch.cuda.synchronize()
            assert np.array_equal(_bits(o_b), _bits(out)) and np.array_equal(_bits(p_b), _bits(pw)), rep
            for o, idx in zip(ones, (2, 0)):
                assert np.array_equal(_bits(o), _bits(cz.channel_slice(out, idx)[1].contiguous())), (rep, idx)
    finally:
        cz.close()


def test_define_any_matches_define_ext_and_refuses(cuda_dev):
    """define_any gives what define_ext gives (points, messages) wherever that succeeds, the Bluestein path where it
    refuses a length for its factors, and refuses above 1048576 points and odd REAL outputs."""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    m = capi.Master(30000, 1, capi.KGPU_COMPLEX)
    b = capi.Bank(m, 2)
    try:
        for n in [1, 2, 600, 5500, 6930, 7260, 9600, 28798, 38400, 29160, 1 << 20]:
            for ot in (capi.KGPU_COMPLEX, capi.KGPU_REAL):
                assert lib.kgpu_bank_define_ext(b.h, 0, n, ot) == lib.kgpu_bank_define_any(b.h, 1, n, ot), n
        for n in (29, 2900, 1984, 30976, 44000, 62000):
            assert lib.kgpu_bank_define_ext(b.h, 0, n, capi.KGPU_COMPLEX) < 0
            assert b.define_any(1, n) == n
            if n % 2 == 0:
                assert b.define_any(1, n, capi.KGPU_REAL) == n
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define_any: 1048577-point inverse transform exceeds the 1048576-point maximum"):
            b.define_any(0, (1 << 20) + 1)
        with pytest.raises(capi.KgpuError, match=r"REAL-output slaves need an even number of points \(got 725\)"):
            b.define_any(0, 725, capi.KGPU_REAL)
    finally:
        b.close()
        m.close()


# ------------------------------------------------------------------ through filter.h -------------------------------
RX888_CH = [dict(olen=580, shift=15000, low=-13 / 29, high=13 / 29, beta=11.0),     # 29 kHz, 725 points
            dict(olen=1240, shift=-9000, low=-0.45, high=0.45, beta=11.0),          # 62 kHz, 1550 points
            dict(olen=240, shift=4100, low=-5 / 12, high=5 / 12, beta=11.0),        # 12 kHz, 300 points
            dict(olen=240, shift=-7700, low=0.0, high=3 / 12, beta=11.0)]


@pytest.mark.parametrize("driver", ["driver_gpuhdr.so", "driver_refhdr.so"])
def test_bluestein_slaves_through_filter_h(cuda_dev, driver):
    """create_filter_output at 29 kHz and 62 kHz next to 12 kHz channels on a 64.8 MS/s REAL master, through the
    unmodified filter.h calls, against the oracle and, where it is built, the reference's own filter.c."""
    if _load(driver) is None:
        pytest.skip(f"{driver} not built")
    _fresh("_case_through_filter_h", driver)


def _case_through_filter_h(oracle, cuda_dev, driver):
    lib = _load(driver)
    L, M, nb = 1_296_000, 324_001, 3
    x = oracle.siggen_real(nb * L, 10 ** (-20 / 20), 10 ** (-40 / 20), 0.0123, 10 ** (3 / 20))
    got, _ = oracle.ref_run_stream(x, L, M, RX888_CH, lib=lib)
    ref, _ = oracle.run_stream(x, L, M, RX888_CH)
    filt = oracle.ref_run_stream(x, L, M, RX888_CH)[0] if oracle.ref_available() else None
    for b in range(nb):
        for c in range(len(RX888_CH)):
            assert rel_err(got[b][c], ref[b][c]) < TOL, (b, c)
            if filt is not None:
                assert rel_err(got[b][c], filt[b][c]) < TOL, ("filter.c", b, c)


W29 = (-13 / 29, 13 / 29, 11.0)
W62 = (-0.45, 0.45, 11.0)


def test_bluestein_slaves_tuned_batch_retune_and_laps_through_filter_h(cuda_dev):
    """execute_filter_output_tuned (output and block power) with the 29 kHz and 62 kHz slaves, including a retune in
    mid-stream (the block issued before the new shift is known is recomputed by kgpu_bank_run_one_ex); the noise
    estimate's spectrum; execute_filter_output_batch; the lap / drop logic with a Bluestein slave."""
    _fresh("_case_tuned_batch_retune_laps", env={"KA9Q_GPU_SPECTRUM_D2H": ""})


def _case_tuned_batch_retune_laps(oracle, cuda_dev):
    lib = _load("driver_gpuhdr.so")
    L, M, fs = 48000, 12001, 2.4e6
    N = L + M - 1
    nb = 7
    x = oracle.siggen_real(8 * L, 0.1, 0.02, 0.1234, 1.0)
    freqs = [[600_017.3, 412_234.5] for _ in range(nb)]
    for b in range(3, nb):
        freqs[b][0] = 603_350.6
    for b in range(5, nb):
        freqs[b][1] = 412_234.5 - 21_000.0
    olen, rate = [580, 1240], [29000.0, 62000.0]
    R = [oracle.design_response(725, 580, N, True, *W29), oracle.design_response(1550, 1240, N, True, *W62)]
    fts = [oracle.FineTune(L, M, r) for r in rate]
    retuned = 0
    with oracle.RefSession(L, M, oracle.KO_REAL, lib=lib) as s:
        ids = [s.add_channel(580, *W29), s.add_channel(1240, *W62)]
        assert lib.ref_channel_points(s.h, ids[0]) == 725 and lib.ref_channel_points(s.h, ids[1]) == 1550
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
            if b == 4:
                host = s.spectrum()
                for sh, pts in zip(shifts, (725, 1550)):
                    a = oracle.estimate_noise(oracle.KO_REAL, host, pts, sh, fs)
                    ref_n0 = oracle.estimate_noise(oracle.KO_REAL, X, pts, sh, fs)
                    assert abs(a - ref_n0) / ref_n0 < 1e-5, (b, sh)
    assert retuned == 2
    chans = [dict(olen=580, shift=15000 + 40 * i, low=W29[0], high=W29[1], beta=W29[2]) for i in range(3)]
    chans.append(dict(olen=1240, shift=-9000, low=W62[0], high=W62[1], beta=W62[2]))
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
        assert lib.ref_produce_from_thread(s.h, np.ascontiguousarray(x[2 * L:8 * L]), 6) == 0
        y = np.ones(580, np.complex64)
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 1
        assert not y.any() and lib.ref_channel_next_job(s.h, 0) == 3
        y[:] = 1
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2
        assert not y.any()
        for b in (4, 5, 6, 7):
            assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2
            assert rel_err(y, ref[b][0]) < TOL, b
