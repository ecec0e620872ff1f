"""Channels whose inverse transform is longer than 28812 points, up to 1048576 (kgpu_bank_define_huge, chan_huge.cuh):
the 1.536 MS/s websdr channels of an RX888 at 64.8 MS/s (38400 points at 20 ms and overlap 5, 61440 at overlap 2,
368640 at 120 ms blocks).

The method and bounds are those of test_gpu_wide_channels.py and test_gpu_accuracy.py: every output sample against
ifft(exact slice x R) in float64 (max e <= 5e-6, gpu/oracle rms ratio <= 2 and max ratio <= 4), against the oracle at
1e-5 of rms, the output row pre-filled with a NaN pattern that must survive outside every channel's run; whole banks
against oracle.run_stream; the filter.h surface against the oracle and, where it is built, the reference's own filter.c.
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


def _fresh(case, *args, env=None, unset=()):
    """Runs this module's `case(oracle, device, *args)` in a new Python process.

    The float32 reference transforms (the oracle, and the reference's filter.c behind driver_refhdr.so) keep one plan
    per transform length in a process-wide cache of 64 lengths, and a length past the 64th crashes the process.  The
    rest of the GPU suite shares one process and already uses most of those slots, so every test here that transforms
    on the CPU runs in a process of its own and leaves the suite's cache as it found it."""
    code = (f"import sys; sys.path[:0] = [{str(HERE)!r}, {str(ROOT)!r}]\n"
            "import torch\nfrom oracle import oracle as O\nO.lib()\n"
            f"import test_gpu_huge_channels as t\nt.{case}(O, torch.device('cuda:0'), *{args!r})\nprint('case ok')\n")
    full_env = {k: v for k, v in dict(os.environ, **(env or {})).items() if k not in unset}
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, env=full_env, capture_output=True, text=True, timeout=1500)
    print(r.stdout)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]

MAX_WIDE = 28812      # kMaxWideChanPoints
MAX_HUGE = 1 << 20    # kMaxHugeChanPoints
HUGE = [29160, 38400, 59049, 61440, 78125, 117649, 368640, 1048576]


def _master_for(ns):
    """a 7-smooth N (M = 1, so a channel's points equal its output length) more than twice the channel"""
    for n in (192000, 256000, 768000, 1 << 22):
        if n > 2 * ns + 2:
            return n
    raise AssertionError(ns)


@pytest.mark.parametrize("master", ["real", "complex"])
@pytest.mark.parametrize("ns", HUGE)
def test_huge_channel_per_sample_accuracy_and_writes(cuda_dev, ns, master):
    _fresh("_case_accuracy", ns, master)


def _case_accuracy(oracle, cuda_dev, ns, master):
    from ka9q_radio_b200 import capi

    real = master == "real"
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    rng = np.random.default_rng(ns + real)
    N = _master_for(ns)
    chans = _sweep_channels(N, ns, real, rng)
    cz = _mk(N, 1, in_type, cuda_dev, len(chans))
    try:
        resp = []
        for pts, s, kind in chans:
            R = (rng.standard_normal(pts) + 1j * rng.standard_normal(pts)).astype(np.complex64)
            resp.append(R)
            assert cz.add_channel(pts, s, response=R, isb=kind == "isb", beam=BEAM_W if kind == "beam" else None,
                                  out_type=capi.KGPU_REAL if kind == "real" else capi.KGPU_COMPLEX) == len(resp) - 1
        bins, nb = cz.master.bins, (2 if ns < 300000 else 1)
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
        _score(f"huge {ns} {master}", np.concatenate(e_gpu), np.concatenate(e_ora))
    finally:
        cz.close()


def test_huge_define_accepted_range(cuda_dev):
    """Every length with factors 2, 3, 5, 7 in (28812, 1048576] is accepted, as COMPLEX and, when even, as REAL output;
    the next one, a factor of 11 and an odd REAL output are rejected with their messages; up to 28812 define_huge is
    define_wide, messages included."""
    from ka9q_radio_b200 import capi

    m = capi.Master(MAX_HUGE, 1, capi.KGPU_COMPLEX)  # N = L: points = olen
    b = capi.Bank(m, 2)
    lib = capi.load()
    try:
        lengths = [n for n in range(MAX_WIDE + 1, MAX_HUGE + 1) if _smooth(n)]
        assert len(lengths) == 806 and sum(n % 2 == 0 for n in lengths) == 699
        for n in reversed(lengths):  # longest first: every later definition reuses the slot's response region
            assert b.define_huge(0, n) == n
            if n % 2 == 0:
                assert b.define_huge(1, n, capi.KGPU_REAL) == n
        nxt = next(n for n in range(MAX_HUGE + 1, 2 * MAX_HUGE) if _smooth(n))
        assert nxt == 1049760
        with pytest.raises(capi.KgpuError, match=f"kgpu_bank_define_huge: {nxt}-point inverse transform exceeds the 1048576-point maximum"):
            b.define_huge(0, nxt)
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define_huge: 30976-point transform cannot be split into two plannable lengths"):
            b.define_huge(0, 30976)  # 2^8 11^2
        with pytest.raises(capi.KgpuError, match=r"REAL-output slaves need an even number of points \(got 30375\)"):
            b.define_huge(0, 30375, capi.KGPU_REAL)
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define_wide: 29160-point inverse transform exceeds the 28812-point maximum"):
            b.define_wide(0, 29160)
        for n, ot in [(2, 0), (600, 0), (7200, 1), (7290, 0), (9600, 1), (28812, 0), (28812, 1), (88, 0), (8800, 0), (7875, 1)]:
            ot = capi.KGPU_REAL if ot else capi.KGPU_COMPLEX
            rw = lib.kgpu_bank_define_wide(b.h, 0, n, ot)
            ew = lib.kgpu_last_error().decode()
            rh = lib.kgpu_bank_define_huge(b.h, 1, n, ot)
            eh = lib.kgpu_last_error().decode()
            assert rw == rh, n
            if rw < 0:
                assert ew == eh, (n, ew, eh)
    finally:
        b.close()
        m.close()


# ------------------------------------------------------------------ the websdr bank ------------------------------
# radiod@rx888-wsprdaemon.conf's enabled channels on a 64.8 MS/s RX888 REAL master at 20 ms and overlap 5:
# (count, olen, low, high, beta): 15 WSPR at 12 kHz, 10 WWV-IQ at 16 kHz, 8 x 768 kHz, 2 x 384 kHz, 3 x 192 kHz and
# the 8 WEBSDR_TEST channels at 1.536 MS/s
RX888 = dict(L=1_296_000, M=324_001, fs=64.8e6)
WEBSDR = [(15, 240, -0.4, 0.4, 11.0), (10, 320, -0.45, 0.45, 11.0), (8, 15360, -0.45, 0.45, 11.0),
          (2, 7680, -0.45, 0.45, 11.0), (3, 3840, -0.45, 0.45, 11.0), (8, 30720, -0.46, 0.46, 11.0)]


def _websdr_channels(N, fs):
    from oracle import oracle as O

    och, f = [], 137_500.0
    for count, olen, lo, hi, beta in WEBSDR:
        for _ in range(count):  # 46 channels from 137.5 kHz to 25 MHz
            _, shift, _ = O.compute_tuning(N, fs, f)
            och.append(dict(olen=olen, shift=shift, low=lo, high=hi, beta=beta))
            f += 0.55e6 + 1234.5
    return och


def test_websdr_bank_against_the_oracle(cuda_dev):
    """The whole websdr bank plus a REAL-output huge slave, 3 blocks, one kgpu_bank_run against oracle.run_stream;
    run_one on a huge channel is bitwise the batched output."""
    _fresh("_case_websdr_bank")


def _case_websdr_bank(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M, fs = RX888["L"], RX888["M"], RX888["fs"]
    N = L + M - 1
    nb = 3
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.1234, 1.0)
    och = _websdr_channels(N, fs)
    huge = [i for i, c in enumerate(och) if c["olen"] * N // L > MAX_WIDE]
    assert len(huge) == 8 and all(och[i]["olen"] * N // L == 38400 for i in huge)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, len(och) + 1)
    try:
        for c in och:
            cz.add_channel(c["olen"], c["shift"], c["low"], c["high"], c["beta"])
        ro = dict(olen=30720, shift=200_000, low=0.01, high=0.45, beta=11.0)
        cz.add_channel(ro["olen"], ro["shift"], ro["low"], ro["high"], ro["beta"], out_type=capi.KGPU_REAL)
        spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
        cz.forward(cz.stage_stream(x), nb, spec)
        cz.channels(spec, nb, out)
        torch.cuda.synchronize()
        ref, _ = oracle.run_stream(x, L, M, och)
        Rro = oracle.design_response_realout(38400, 30720, N, True, ro["low"], ro["high"], ro["beta"])
        for b in range(nb):
            X = oracle.forward(oracle.block_window(x, L, M, b))
            for i in range(len(och)):
                assert rel_err(cz.channel_slice(out, i).cpu().numpy()[b], ref[b][i]) < TOL, (b, i)
            r = oracle.channel_block_realout(capi.KGPU_REAL, X, Rro, ro["shift"])[-30720:]
            assert rel_err(cz.channel_slice(out, len(och)).cpu().numpy()[b], r) < TOL, b
        for i in huge[:3] + [len(och)]:
            n = och[i]["olen"] if i < len(och) else (ro["olen"] + 1) // 2
            one = torch.zeros(n, dtype=torch.complex64, device=cuda_dev)
            cz.bank.run_one(i, spec[1].data_ptr(), one.data_ptr())
            torch.cuda.synchronize()
            want = out[1, cz.bank.out_offset(i):cz.bank.out_offset(i) + n].contiguous()
            if i == len(och):  # REAL output: olen floats, the last float2 half used
                assert np.array_equal(_bits(one)[: ro["olen"]], _bits(want)[: ro["olen"]]), i
            else:
                assert np.array_equal(_bits(one), _bits(want)), i
    finally:
        cz.close()


def test_huge_launch_in_scratch_chunks_is_bitwise_one_block_launches(cuda_dev):
    """8 channels of 368640 points over 6 blocks need 48 scratch slots of 2.9 MB, more than the 128 MB cap holds, so
    the launch runs in chunks of blocks; every block is bitwise what a one-block launch gives."""
    from ka9q_radio_b200 import capi

    N, ns, nb = 768000, 368640, 6
    rng = np.random.default_rng(5)
    cz = _mk(N, 1, capi.KGPU_COMPLEX, cuda_dev, 8)
    try:
        assert 8 * nb * ns * 8 > 128 << 20
        for k in range(8):
            R = (rng.standard_normal(ns) + 1j * rng.standard_normal(ns)).astype(np.complex64)
            cz.add_channel(ns, int(rng.integers(-N // 2, N // 2)), response=R, isb=k == 3, beam=BEAM_W if k == 5 else None)
        X = (rng.standard_normal((nb, N)) + 1j * rng.standard_normal((nb, N))).astype(np.complex64)
        spec = cz.alloc_spectra(nb)
        spec[:, :N] = torch.from_numpy(X).to(cuda_dev)
        out = _sentinel(nb, cz.bank.out_stride, cuda_dev)
        cz.channels(spec, nb, out)
        one = _sentinel(1, cz.bank.out_stride, cuda_dev)
        for b in range(nb):
            cz.channels(spec[b:b + 1], 1, one)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(one)[0], _bits(out)[b]), b
    finally:
        cz.close()


def test_huge_channel_tuned_oscillator_and_power(cuda_dev):
    """The kChanOsc store of chan_huge (rotation, per-block phase, power from per-CTA partial sums) across retunes and
    launches of 1..3 blocks, against the oracle's restatement of radio.c:1476-1520, next to an ordinary tuned channel;
    run_one with power gives bitwise the batched output and power."""
    _fresh("_case_osc")


def _case_osc(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M, fs = 48000, 12001, 2.4e6
    N = L + M - 1
    chans = [(30720, 1536000.0, -0.46, 0.46, 11.0, False), (480, 24000.0, -1 / 3, 1 / 3, 11.0, False),
             (49152, 2457600.0, -0.2, 0.2, 5.0, True)]
    nb = 6
    plan = [[600_017.3, 412_234.5, 250_123.4] for _ in range(nb)]
    for b in range(3, nb):
        plan[b][0] += 3_333.3
        plan[b][2] -= 17.25
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.2501, 1.0)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, len(chans))
    lib = capi.load()
    try:
        resp = []
        for c in chans:
            cz.add_channel(c[0], 0, c[2], c[3], c[4], isb=c[5])
            resp.append(oracle.design_response(c[0] * N // L, c[0], N, True, c[2], c[3], c[4]))
        assert [pts for _, pts in cz._olen.values()][::2] == [38400, 61440]
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
                for i in (0, 2):
                    one = torch.zeros(chans[i][0], dtype=torch.complex64, device=cuda_dev)
                    p1 = torch.zeros(1, dtype=torch.float32, device=cuda_dev)
                    cz.bank.block_counter = b0 + 1
                    capi.check(lib.kgpu_bank_run_one_ex(cz.bank.h, i, spec[1].data_ptr(), one.data_ptr(), p1.data_ptr(), None))
                    torch.cuda.synchronize()
                    assert np.array_equal(_bits(one), _bits(cz.channel_slice(out, i)[1].contiguous())), i
                    assert np.array_equal(_bits(p1), _bits(pw[1, i:i + 1].contiguous())), i
                cz.bank.block_counter = b0 + nblk
            b0 += nblk
        assert worst_y < TOL and worst_p < TOL, (worst_y, worst_p)
    finally:
        cz.close()


@pytest.mark.parametrize("points", [38400, 368640])
def test_huge_response_against_design_response(cuda_dev, points):
    """set_filter's forward transform (response_huge_cols / _rows) against oracle.design_response."""
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


def test_huge_channel_noise(cuda_dev):
    """kgpu_bank_noise on huge channels whose windows fit shared memory (38400 bins) and whose windows do not (61440 and
    368640, noise_kernel_gm) against oracle.estimate_noise; the ordinary channels' estimates are bitwise those of the same
    bank without the huge channels."""
    _fresh("_case_noise")


def _case_noise(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    FS = 1.536e8
    N = 768000
    rng = np.random.default_rng(11)
    bins = N // 2 + 1
    nb = 3
    sp = [((rng.standard_normal(bins) + 1j * rng.standard_normal(bins)) * (1 + np.arange(bins) / bins)).astype(np.complex64)
          for _ in range(nb)]
    ordinary = [(600, 5000, False), (9600, -120_000, False), (28812, 300_000, False), (1200, 383_900, True)]
    hugech = [(38400, 100_000, False), (61440, -250_000, False), (368640, 200_000, False), (61440, 380_000, True)]

    def run(chans):
        cz = _mk(N, 1, capi.KGPU_REAL, cuda_dev, len(chans))
        try:
            for pts, sh, ro in chans:
                cz.add_channel(pts, sh, response=np.ones(pts, np.complex64), out_type=capi.KGPU_REAL if ro else capi.KGPU_COMPLEX)
            spec = cz.alloc_spectra(nb)
            spec[:, :bins] = torch.from_numpy(np.stack(sp)).to(cuda_dev)
            n0 = torch.full((nb, cz.capacity), float("nan"), dtype=torch.float64, device=cuda_dev)
            cz.bank.noise(spec.data_ptr(), nb, FS, n0.data_ptr(), torch.cuda.current_stream(cuda_dev).cuda_stream)
            torch.cuda.synchronize()
            return n0.cpu().numpy()
        finally:
            cz.close()

    both = run(ordinary + hugech)
    alone = run(ordinary)
    assert np.array_equal(both[:, :len(ordinary)], alone), "the ordinary channels' estimates moved"
    worst = 0.0
    for b in range(nb):
        for k, (pts, sh, ro) in enumerate(ordinary + hugech):
            ref = oracle.estimate_noise(oracle.KO_REAL, sp[b], pts // 2 + 1 if ro else pts, sh, FS)
            err = abs(both[b, k] - ref) / ref
            worst = max(worst, err)
            assert err < 1e-5, (b, pts, sh, ro, both[b, k], ref)
    print(f"\nnoise huge: worst rel err {worst:.2e}")


# ------------------------------------------------------------------ through filter.h ---------------
WEBSDR_CH = [dict(olen=30720, shift=15000, low=-0.46, high=0.46, beta=11.0),
             dict(olen=480, shift=-9000, low=-1 / 3, high=1 / 3, beta=11.0),
             dict(olen=30720, shift=-4100, low=-0.3, high=0.3, beta=11.0, isb=True)]


@pytest.mark.parametrize("master", ["cfg1", "rx888"])
@pytest.mark.parametrize("driver,zerocopy", [("driver_gpuhdr.so", "0"), ("driver_gpuhdr.so", "1"), ("driver_refhdr.so", "0")])
def test_websdr_slave_through_filter_h(cuda_dev, driver, zerocopy, master):
    """create_filter_output at 1.536 MS/s (olen 30720, 38400 points) on a 2.4 MS/s and on the 64.8 MS/s REAL master
    through the unmodified filter.h calls, copy and zero-copy delivery, against the oracle and, where it is built, the
    reference's own filter.c."""
    if _load(driver) is None:
        pytest.skip(f"{driver} not built")
    _fresh("_case_through_filter_h", driver, master, env={"KA9Q_GPU_ZEROCOPY": zerocopy})


def _case_through_filter_h(oracle, cuda_dev, driver, master):
    lib = _load(driver)
    if master == "cfg1":
        L, M, chans, nb = 48000, 12001, WEBSDR_CH, 4
    else:
        L, M, nb = RX888["L"], RX888["M"], 3
        chans = [dict(c, shift=c["shift"] * 20) for c in WEBSDR_CH]
    x = oracle.siggen_real(nb * L, 10 ** (-20 / 20), 10 ** (-40 / 20), 0.25, 10 ** (3 / 20))
    got, _ = oracle.ref_run_stream(x, L, M, chans, lib=lib)
    ref, _ = oracle.run_stream(x, L, M, chans)
    filt = oracle.ref_run_stream(x, L, M, chans) if oracle.ref_available() else None
    for b in range(nb):
        for c in range(len(chans)):
            assert rel_err(got[b][c], ref[b][c]) < TOL, (b, c)
            if filt is not None:
                assert rel_err(filt[0][b][c], ref[b][c]) < TOL, (b, c)


def test_websdr_slave_tuned_batch_windows_and_laps_through_filter_h(cuda_dev):
    """execute_filter_output_tuned (output and block power), the default spectrum windows estimate_noise reads,
    execute_filter_output_batch and the lap / drop logic, each with a 1.536 MS/s slave.  The master runs at 4.8 MS/s,
    whose 60 001 bins hold the slave's 38 400-bin noise window (at 2.4 MS/s the window is wider than the spectrum, where
    the reference's estimate_noise reads past the end of it)."""
    _fresh("_case_tuned_batch_windows_laps", unset=("KA9Q_GPU_SPECTRUM_D2H",))


def _case_tuned_batch_windows_laps(oracle, cuda_dev):
    lib = _load("driver_gpuhdr.so")
    L, M, fs = 96000, 24001, 4.8e6
    N = L + M - 1
    nb = 6
    W = (-0.46, 0.46, 11.0)
    x = oracle.siggen_real(8 * L, 0.1, 0.02, 0.1234, 1.0)
    freqs = [[600_017.3, 412_234.5] for _ in range(nb)]
    for b in range(3, nb):
        freqs[b][0] = 603_350.6
    olen, rate = [30720, 480], [1536000.0, 24000.0]
    R = [oracle.design_response(38400, 30720, N, True, *W), oracle.design_response(600, 480, N, True, -1 / 3, 1 / 3, 11.0)]
    fts = [oracle.FineTune(L, M, r) for r in rate]
    with oracle.RefSession(L, M, oracle.KO_REAL, lib=lib) as s:
        ids = [s.add_channel(30720, *W), s.add_channel(480, -1 / 3, 1 / 3, 11.0)]
        assert lib.ref_channel_points(s.h, ids[0]) == 38400
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
            if b >= 4:  # the windows follow the shifts of the previous block, which are the same from block 4 on
                host = s.spectrum()
                for sh, pts in zip(shifts, (38400, 600)):
                    a = oracle.estimate_noise(oracle.KO_REAL, host, pts, sh, fs)
                    ref_n0 = oracle.estimate_noise(oracle.KO_REAL, X, pts, sh, fs)
                    assert abs(a - ref_n0) / ref_n0 < 1e-5, (b, sh)
    chans = [dict(olen=30720, shift=15000 + 40 * i, low=W[0], high=W[1], beta=W[2]) for i in range(3)]
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
        y = np.ones(30720, np.complex64)
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 1  # slot of job 2 holds job 6: zeros, a drop
        assert not y.any() and lib.ref_channel_next_job(s.h, 0) == 3
        y[:] = 1
        assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2  # job 3: its slot holds job 7
        assert not y.any()
        for b in (4, 5, 6, 7):
            assert lib.ref_lap_probe(s.h, 0, chans[0]["shift"], None, 0, y) == 2
            assert rel_err(y, ref[b][0]) < TOL, b
