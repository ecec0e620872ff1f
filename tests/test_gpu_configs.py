"""BASELINE.json's configurations at FULL size, every channel, in the launch shape bench.py times
(32 blocks per launch, first_block != 0), against the oracle at north_star's 1e-5."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _float_stream(oracle, w, xi):
    from ka9q_radio_b200 import workloads

    if w.in_type == workloads.KGPU_REAL:
        return oracle.convert_i16(xi, np.float32(w.scale))[0]
    s = np.float32(w.scale)
    return (xi[0::2].astype(np.float32) * s + 1j * (xi[1::2].astype(np.float32) * s)).astype(np.complex64)


def _run_and_check(oracle, cuda_dev, w, nstream, B, first_block, check_blocks):
    """stream of nstream blocks resident on the device, ONE launch of B blocks starting at first_block; compares every
    channel of the blocks in check_blocks (indices inside the launch) with the oracle"""
    from ka9q_radio_b200.channelizer import Channelizer

    xi = w.stream(nstream)
    xf = _float_stream(oracle, w, xi)
    cz = Channelizer(w.L, w.M, w.in_type, cuda_dev, capacity=len(w.channels))
    for c in w.channels:
        cz.add_channel(c.olen, c.shift, c.low, c.high, c.beta)
    spec, out = cz.alloc_spectra(B), cz.alloc_outputs(B)
    cz.forward(cz.stage_stream(xi), B, spec, scale=w.scale, first_block=first_block)
    cz.channels(spec, B, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    offs = [cz.bank.out_offset(i) for i in range(len(w.channels))]
    bins = cz.master.bins
    sp = spec[check_blocks[0], :bins].cpu().numpy()
    cz.close()
    resp = {}
    worst, loud = 0.0, 0.0
    items = []
    for b in check_blocks:
        X = oracle.forward(oracle.block_window(xf, w.L, w.M, first_block + b))
        if b == check_blocks[0]:
            assert np.abs(sp - X).max() / np.abs(X).max() < TOL
        for i, c in enumerate(w.channels):
            key = (c.olen, c.low, c.high, c.beta)
            if key not in resp:
                resp[key] = oracle.design_response(c.olen * w.N // w.L, c.olen, w.N, w.in_type == oracle.KO_REAL, c.low, c.high, c.beta)
            r = oracle.channel_block(w.in_type, X, resp[key], c.shift)[-c.olen:]
            items.append((got[b, offs[i]: offs[i] + c.olen], r, (b, i)))
            loud = max(loud, float(np.abs(r).max()))
    bad = None
    for g, r, tag in items:
        # Two independent float32 forward transforms differ by rounding noise of ~2e-8 of the STRONGEST channel in every
        # channel (eps * sqrt(log2 N) of the total spectral energy, gathered over the ~400 passband bins): a noise-only
        # channel 53 dB below the tones cannot agree to 1e-5 of its own level with ANY other float32 implementation, FFTW
        # included (measured here: up to 1.5e-7 of the loudest channel, peak over 1.5 M samples).  So channels more than 30 dB
        # below the loudest are measured against that -30 dB level; channels within 20 dB of the loudest must agree to 1e-5 of
        # their own peak (they agree to ~3e-7).  test_cfg2_quiet_channels_no_worse_than_the_float32_oracle shows against a
        # float64 transform that both sit on the same rounding floor (rms within 2x; the GPU's spectrum error is the smaller).
        own = float(np.abs(r).max())
        e = float(np.abs(g - r).max()) / max(own, 3e-2 * loud)
        if own >= 0.1 * loud:
            e = max(e, float(np.abs(g - r).max()) / own)
        if e > worst:
            worst, bad = e, tag
    return worst, bad, len(items)


def test_cfg2_all_channels_32_block_launch(oracle, cuda_dev):
    """cfg-2: 1024 NBFM channels + 8 inverted ones, ONE launch of 32 blocks taken from the middle of a 40-block stream
    (first_block = 5), blocks 0, 15 and 31 of the launch checked on ALL 1032 channels."""
    from ka9q_radio_b200 import workloads

    w = workloads.cfg2(with_inverted=True)
    worst, bad, n = _run_and_check(oracle, cuda_dev, w, nstream=40, B=32, first_block=5, check_blocks=[0, 15, 31])
    assert n == 3 * 1032 and worst < TOL, (worst, bad)


def test_cfg2_quiet_channels_no_worse_than_the_float32_oracle(oracle, cuda_dev):
    """The justification of the -40 dB floor above: against a float64 transform of the same block, the GPU's error on
    noise-only channels is the same rounding-noise floor as the float32 oracle's (tools/diag_floor.py prints both).
    The rms is the statistic (the max of ~4000 noise-like samples moves by +-30 % between kernel variants)."""
    from ka9q_radio_b200 import workloads
    from ka9q_radio_b200.channelizer import Channelizer

    w = workloads.cfg2()
    quiet = [9, 100, 500, 777, 1000, 33, 250, 640, 900]          # no tone within 150 kHz
    w.channels = [w.channels[i] for i in quiet] + [w.channels[3]]   # + one tone channel as the loudness reference
    xi = w.stream(2)
    xf = oracle.convert_i16(xi, np.float32(w.scale))[0]
    cz = Channelizer(w.L, w.M, w.in_type, cuda_dev, capacity=len(w.channels))
    for c in w.channels:
        cz.add_channel(c.olen, c.shift, c.low, c.high, c.beta)
    spec, out = cz.alloc_spectra(2), cz.alloc_outputs(2)
    cz.forward(cz.stage_stream(xi), 2, spec, scale=w.scale)
    cz.channels(spec, 2, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    gspec = spec.cpu().numpy()[1, : w.N // 2 + 1]
    offs = [cz.bank.out_offset(i) for i in range(len(w.channels))]
    cz.close()
    b = 1
    win = oracle.block_window(xf, w.L, w.M, b)
    X32 = oracle.forward(win)
    X64 = oracle.forward_real_f64(win.astype(np.float64))
    R = oracle.design_response(600, 480, w.N, True, w.channels[0].low, w.channels[0].high, 11.0)
    k = np.arange(-300, 300)
    eg, eo = [], []
    for i, c in enumerate(w.channels[:-1]):
        S = np.zeros(600, np.complex128)
        S[k % 600] = X64[c.shift + k] * R[k % 600].astype(np.complex128)
        S[300] = 0
        truth = (np.fft.ifft(S) * 600)[-480:]
        r32 = oracle.channel_block(oracle.KO_REAL, X32, R, c.shift)[-480:]
        g = got[b, offs[i]: offs[i] + 480]
        eg.append(np.abs(g - truth))
        eo.append(np.abs(r32 - truth))
    eg, eo = np.concatenate(eg), np.concatenate(eo)
    rms = lambda e: float(np.sqrt((e ** 2).mean()))
    assert rms(eg) < 2.0 * rms(eo), (rms(eg), rms(eo))
    assert float(eg.max()) < 3.0 * float(eo.max()), (float(eg.max()), float(eo.max()))
    nb = w.N // 2 + 1
    sg, so = np.abs(gspec - X64[:nb]), np.abs(X32[:nb] - X64[:nb])
    assert rms(sg) < 1.5 * rms(so), (rms(sg), rms(so))


def test_cfg3_all_300_channels(oracle, cuda_dev):
    """cfg-3 as surveyed: 300 SSB channels, 100 each at 12 / 24 / 48 kHz (three inverse-transform sizes in one bank)."""
    from ka9q_radio_b200 import workloads

    w = workloads.cfg3()
    worst, bad, n = _run_and_check(oracle, cuda_dev, w, nstream=6, B=4, first_block=2, check_blocks=[0, 3])
    assert n == 2 * 300 and worst < TOL, (worst, bad)


def test_cfg4_all_512_channels(oracle, cuda_dev):
    """cfg-4: complex int16 I/Q, c2c forward, all 512 channels incl. negative shifts and the wrap at +-fs/2."""
    from ka9q_radio_b200 import workloads

    w = workloads.cfg4()
    worst, bad, n = _run_and_check(oracle, cuda_dev, w, nstream=8, B=6, first_block=1, check_blocks=[0, 5])
    assert n == 2 * 512 and worst < TOL, (worst, bad)


def test_cfg5_channel_plan_one_group(oracle, cuda_dev):
    """cfg-5: the 188-bin raster of the 8192-channel plan, group 5 of 8 (channels 5120..6143), preset nfm."""
    from ka9q_radio_b200 import workloads

    w = workloads.cfg5(5, 8)
    worst, bad, n = _run_and_check(oracle, cuda_dev, w, nstream=4, B=3, first_block=1, check_blocks=[2])
    assert n == 1024 and worst < TOL, (worst, bad)
