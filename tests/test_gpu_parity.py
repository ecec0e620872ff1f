"""GPU parity: the CUDA path (through the C-ABI) against the CPU oracle on identical inputs.

Tolerance (north_star): 1e-5 relative, defined per block / per channel-block as
max|gpu - ref| / max|ref| (BASELINE.md section 3; outputs cross zero so an element-wise relative
error is meaningless).  Observed errors are ~2e-7 (two independent float32 FFTs).
"""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _mk(L, M, in_type, dev, cap=64):
    from ka9q_radio_b200.channelizer import Channelizer

    return Channelizer(L, M, in_type, dev, capacity=cap)


# ------------------------------------------------------------------ forward transform ---------
@pytest.mark.parametrize("L,M", [(4800, 1201), (48000, 12001), (1920, 481), (38400, 9601)])
def test_forward_real_float(oracle, cuda_dev, L, M):
    from ka9q_radio_b200 import capi

    nb = 3
    x = oracle.siggen_real(nb * L, 0.1, 0.01, 0.25 + 1.0 / 97, 1.4125)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
    d = cz.stage_stream(x)
    spec = cz.alloc_spectra(nb)
    cz.forward(d, nb, spec)
    torch.cuda.synchronize()
    got = spec.cpu().numpy()
    for b in range(nb):
        ref = oracle.forward(oracle.block_window(x, L, M, b))
        assert rel_err(got[b, : cz.master.bins], ref) < TOL
    cz.close()


@pytest.mark.parametrize("L,M", [(4000, 1001), (400000, 100001)])
def test_forward_complex_float(oracle, cuda_dev, L, M):
    from ka9q_radio_b200 import capi

    nb = 2
    x = oracle.siggen_complex(nb * L, 0.1, 0.01, -0.123, 1.0)
    cz = _mk(L, M, capi.KGPU_COMPLEX, cuda_dev)
    d = cz.stage_stream(x)
    spec = cz.alloc_spectra(nb)
    cz.forward(d, nb, spec)
    torch.cuda.synchronize()
    got = spec.cpu().numpy()
    for b in range(nb):
        ref = oracle.forward(oracle.block_window(x, L, M, b))
        assert rel_err(got[b, : cz.master.bins], ref) < TOL
    cz.close()


def test_forward_int16_fused_ingest(oracle, cuda_dev):
    """int16 -> float conversion fused into pass 1 == rx888.c convert() then r2c, incl. stats."""
    from ka9q_radio_b200 import capi

    L, M, nb = 48000, 12001, 2
    rng = np.random.default_rng(3)
    x = rng.integers(-32768, 32768, nb * L, dtype=np.int16)
    x[5] = 32767
    x[L + 9] = -32768
    scale = np.float32(10 ** (3 / 20) / 32768)
    for derand in (False, True):
        xf, energy, clips = oracle.convert_i16(x, scale, derand)
        cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
        d = cz.stage_stream(x)
        spec = cz.alloc_spectra(nb)
        stats = torch.zeros(nb * 2, dtype=torch.int64, device=cuda_dev)
        cz.forward(d, nb, spec, scale=float(scale), derandomize=derand, stats=stats)
        torch.cuda.synchronize()
        got = spec.cpu().numpy()
        for b in range(nb):
            ref = oracle.forward(oracle.block_window(xf, L, M, b))
            assert rel_err(got[b, : cz.master.bins], ref) < TOL
        st = stats.cpu().numpy()
        e_blocks = [oracle.convert_i16(x[b * L:(b + 1) * L], scale, derand)[1:] for b in range(nb)]
        for b in range(nb):
            assert int(st[2 * b]) == e_blocks[b][0]           # energy: exact integer arithmetic
            assert int(st[2 * b + 1] & 0xFFFFFFFF) == e_blocks[b][1]  # clip count
        cz.close()


def test_forward_linearity_and_impulse(oracle, cuda_dev):
    """Size-independent properties at the full RX888 size: DFT of an impulse is a pure phase ramp,
    and F(a+b) = F(a)+F(b)."""
    from ka9q_radio_b200 import capi

    L, M = 2592000, 648001
    N = L + M - 1
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
    x = np.zeros(L, np.float32)
    pos = 1234567
    x[pos] = 1.0
    spec = cz.alloc_spectra(1)
    cz.forward(cz.stage_stream(x), 1, spec)
    torch.cuda.synchronize()
    got = spec.cpu().numpy()[0, : cz.master.bins]
    n0 = pos + M - 1
    k = np.arange(cz.master.bins, dtype=np.float64)
    ref = np.exp(-2j * np.pi * ((k * n0) % N) / N)
    assert np.abs(got - ref).max() < 2e-6
    rng = np.random.default_rng(0)
    a = rng.standard_normal(L).astype(np.float32)
    b = rng.standard_normal(L).astype(np.float32)
    sa, sb, sab = cz.alloc_spectra(1), cz.alloc_spectra(1), cz.alloc_spectra(1)
    cz.forward(cz.stage_stream(a), 1, sa)
    cz.forward(cz.stage_stream(b), 1, sb)
    cz.forward(cz.stage_stream(a + b), 1, sab)
    torch.cuda.synchronize()
    nbin = cz.master.bins  # the rows are padded to a multiple of 4 bins: the padding is never written
    err = (sab - sa - sb)[:, :nbin].abs().max().item() / sab[:, :nbin].abs().max().item()
    assert err < 2e-6
    cz.close()


@pytest.mark.parametrize("static", [1, 0])
def test_forward_full_size_vs_oracle(oracle, cuda_dev, static):
    """cfg-2 geometry (N = 3 240 000), one block of int16 tones+noise, against the CPU oracle;
    once through the compile-time specialised kernels, once through the generic ones."""
    from ka9q_radio_b200 import capi

    capi.load().kgpu_use_static_kernels(static)

    L, M = 2592000, 648001
    fs = 129.6e6
    f = [(30.0e6 + 25e3 * k) / fs for k in (0, 100, 511, 1023)]
    x = oracle.siggen_tones_i16(L, f, [10 ** (-30 / 20)] * 4, 10 ** (-50 / 20), 1)
    scale = np.float32(10 ** (3 / 20) / 32768)
    xf, _, _ = oracle.convert_i16(x, scale)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
    spec = cz.alloc_spectra(1)
    cz.forward(cz.stage_stream(x), 1, spec, scale=float(scale))
    torch.cuda.synchronize()
    got = spec.cpu().numpy()[0, : cz.master.bins]
    ref = oracle.forward(oracle.block_window(xf, L, M, 0))
    assert rel_err(got, ref) < TOL
    # and both against float64 truth: the GPU must not be less accurate than the float oracle
    truth = oracle.forward_real_f64(oracle.block_window(xf, L, M, 0).astype(np.float64))
    e_gpu = np.sqrt(np.mean(np.abs(got - truth) ** 2))
    e_ora = np.sqrt(np.mean(np.abs(ref - truth) ** 2))
    assert e_gpu < 2.0 * e_ora
    cz.close()
    capi.load().kgpu_use_static_kernels(1)


@pytest.mark.parametrize("real,L,M,split,cols,rows", [
    (False, 400000, 100001, "800 x 625", "25,32", "25,25"),        # fwd_cols_2s + fwd_rows_2s (cfg-4)
    (True, 2592000, 648001, "1296 x 1250", "36,36", "10,25,5"),    # fwd_cols_r36 with the 1/2 of the split + fwd_rows_v2
    (False, 1296000, 324001, "1296 x 1250", "36,36", "10,25,5"),   # fwd_cols_r36 + fwd_rows_v2
    (False, 1259712, 419905, "1296 x 1296", "36,36", "12,12,9"),   # fwd_cols_r36 + generic rows
    (True, 2560000, 640001, "1280 x 1250", "16,10,8", "10,25,5"),  # generic columns + fwd_rows_v2 with the real split
    (False, 1200000, 400001, "1280 x 1250", "16,10,8", "10,25,5"), # generic columns + fwd_rows_v2
])
def test_forward_specialised_kernel_pairs(oracle, cuda_dev, real, L, M, split, cols, rows):
    """Every kernel pair kgpu_master_create can choose other than the generic one, against the oracle and against the
    generic kernels of the same master (kgpu_use_static_kernels(0) at launch time).  Two blocks, float input."""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    rng = np.random.default_rng(12)
    t = np.arange(2 * L)
    if real:
        x = (0.1 * rng.standard_normal(2 * L)).astype(np.float32)
        x += (0.5 * np.cos(2 * np.pi * ((0.2345 * t) % 1.0))).astype(np.float32)
    else:
        x = (0.1 * (rng.standard_normal(2 * L) + 1j * rng.standard_normal(2 * L))).astype(np.complex64)
        x += (0.5 * np.exp(2j * np.pi * ((0.2345 * t) % 1.0))).astype(np.complex64)
    cz = _mk(L, M, capi.KGPU_REAL if real else capi.KGPU_COMPLEX, cuda_dev)
    assert f"two-pass {split}; cols radices [{cols}] rows radices [{rows}]" in cz.master.describe()
    d = cz.stage_stream(x)
    spec, spec_gen = cz.alloc_spectra(2), cz.alloc_spectra(2)
    cz.forward(d, 2, spec)
    lib.kgpu_use_static_kernels(0)
    try:
        cz.forward(d, 2, spec_gen)
    finally:
        lib.kgpu_use_static_kernels(1)
    torch.cuda.synchronize()
    nb = cz.master.bins
    got, gen = spec.cpu().numpy()[:, :nb], spec_gen.cpu().numpy()[:, :nb]
    for b in range(2):
        ref = oracle.forward(oracle.block_window(x, L, M, b))
        assert rel_err(got[b], ref) < TOL, (b, rel_err(got[b], ref))
        assert rel_err(gen[b], ref) < TOL
    assert np.abs(got - gen).max() / np.abs(gen).max() < 2e-6
    cz.close()


def test_forward_after_a_smaller_master_is_created(oracle, cuda_dev):
    """The shared-memory limit of a kernel is one value for the whole process.  Creating a master whose generic kernels
    need less (640 000 = 800 x 800) must not take away what an existing one launches with (1 500 000 = 1250 x 1200)."""
    from ka9q_radio_b200 import capi

    L, M = 1125000, 375001
    x = oracle.siggen_complex(L, 0.1, 0.01, -0.123, 1.0)
    big = _mk(L, M, capi.KGPU_COMPLEX, cuda_dev)
    small = _mk(480000, 160001, capi.KGPU_COMPLEX, cuda_dev)
    assert "two-pass 1250 x 1200" in big.master.describe() and "two-pass 800 x 800" in small.master.describe()
    spec = big.alloc_spectra(1)
    big.forward(big.stage_stream(x), 1, spec)
    torch.cuda.synchronize()
    ref = oracle.forward(oracle.block_window(x, L, M, 0))
    assert rel_err(spec.cpu().numpy()[0, : big.master.bins], ref) < TOL
    small.close()
    big.close()


def test_notches(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M, nb = 4800, 1201, 5
    x = oracle.siggen_real(nb * L, 0.1, 0.01, 0.1, 1.0) + np.float32(0.05)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
    cz.master.set_notches([600, 77])
    spec = cz.alloc_spectra(nb)
    cz.forward(cz.stage_stream(x), nb, spec)
    cz.apply_notches(spec, nb)
    torch.cuda.synchronize()
    got = spec.cpu().numpy()
    nt = oracle.Notches([600, 77])
    for b in range(nb):
        ref = oracle.forward(oracle.block_window(x, L, M, b))
        nt.apply(ref)
        assert rel_err(got[b, : cz.master.bins], ref) < TOL
        for bn in (600, 77, 0):
            assert abs(got[b, bn] - ref[bn]) <= 2e-6 * np.abs(ref).max() + 1e-6 * abs(ref[bn])
    cz.close()


# ------------------------------------------------------------------ response design -----------
@pytest.mark.parametrize("olen,low,high,beta", [(480, -1 / 3, 1 / 3, 11.0), (240, 50 / 12000, 3000 / 12000, 11.0),
                                                (960, -0.6, 0.2, 3.0), (480, 0.1, 0.1, 11.0), (160, 0.3, -0.3, 0.0)])
def test_set_filter_matches_oracle(oracle, cuda_dev, olen, low, high, beta):
    from ka9q_radio_b200 import capi

    L, M = 48000, 12001
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
    idx = cz.add_channel(olen, 0, low, high, beta)
    pts = olen * cz.N // L
    got = cz.bank.get_response(idx, pts)
    ref = oracle.design_response(pts, olen, cz.N, True, low, high, beta)
    assert rel_err(got, ref) < 2e-6
    cz.close()


# ------------------------------------------------------------------ channel kernel ------------
def _chan_case(oracle, cuda_dev, in_type, L, M, chans, nb=3, seed=1):
    from ka9q_radio_b200 import capi

    N = L + M - 1
    if in_type == capi.KGPU_REAL:
        x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.123, 1.0)
    else:
        x = oracle.siggen_complex(nb * L, 0.1, 0.02, 0.123, 1.0)
    cz = _mk(L, M, in_type, cuda_dev, cap=len(chans))
    for ch in chans:
        cz.add_channel(ch["olen"], ch["shift"], ch["low"], ch["high"], ch["beta"], isb=ch.get("isb", False))
    spec = cz.alloc_spectra(nb)
    out = cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(x), nb, spec)
    cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    ref_out, _ = oracle.run_stream(x, L, M, chans)
    worst = 0.0
    scale_ref = max(np.abs(ref_out[b][c]).max() for b in range(nb) for c in range(len(chans)))
    for c in range(len(chans)):
        got = cz.channel_slice(out, c).cpu().numpy()
        for b in range(nb):
            r = ref_out[b][c]
            den = np.abs(r).max()
            if den < 1e-4 * scale_ref:  # silent channel: compare against the loudest one's scale
                den = scale_ref
            worst = max(worst, np.abs(got[b] - r).max() / den)
    cz.close()
    return worst


@pytest.mark.parametrize("static", [1, 0])
def test_channels_real_master_all_sizes(oracle, cuda_dev, static):
    from ka9q_radio_b200 import capi

    capi.load().kgpu_use_static_kernels(static)
    L, M = 48000, 12001
    chans = []
    for olen in (240, 480, 960, 120, 160):
        for shift in (7380, -7380, 0, 3, 29990, -29990, 30010, 120, -50):
            chans.append(dict(olen=olen, shift=shift, low=-0.3, high=0.35, beta=11.0))
    chans.append(dict(olen=480, shift=7383, low=-0.2, high=0.2, beta=5.0, isb=True))
    worst = _chan_case(oracle, cuda_dev, capi.KGPU_REAL, L, M, chans)
    capi.load().kgpu_use_static_kernels(1)
    assert worst < TOL


def test_channels_complex_master_wrap(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M = 4000, 1001  # N = 5000
    chans = []
    for olen in (80, 160, 40, 480):  # 480 -> 600 points: the specialised kernel's wrap path
        for shift in (615, -615, 0, 2499, -2499, 2450, -2480, 2490, -2500, 1, -1):
            chans.append(dict(olen=olen, shift=shift, low=-0.3, high=0.35, beta=11.0))
    chans.append(dict(olen=80, shift=600, low=-0.2, high=0.2, beta=5.0, isb=True))
    assert _chan_case(oracle, cuda_dev, capi.KGPU_COMPLEX, L, M, chans) < TOL


def test_channel_shift_sweep_exact_slices(oracle, cuda_dev):
    """Every shift in [-N/2, N/2): identity response -> the inverse transform input is exactly the
    slice the reference would build (zeros, conjugates, wrap) so outputs must match the oracle."""
    from ka9q_radio_b200 import capi

    L, M = 480, 121  # N = 600, real: 301 bins
    rng = np.random.default_rng(5)
    for in_type in (capi.KGPU_REAL, capi.KGPU_COMPLEX):
        N = L + M - 1
        shifts = list(range(-N // 2 - 5, N // 2 + 6, 1))
        cz = _mk(L, M, in_type, cuda_dev, cap=len(shifts))
        olen = 48  # points = 60
        pts = olen * N // L
        R = (rng.standard_normal(pts) + 1j * rng.standard_normal(pts)).astype(np.complex64)
        for s in shifts:
            cz.add_channel(olen, s, response=R)
        bins = cz.master.bins
        X = (rng.standard_normal(bins) + 1j * rng.standard_normal(bins)).astype(np.complex64)
        spec = cz.alloc_spectra(1)
        spec[0, :bins] = torch.from_numpy(X).to(cuda_dev)
        out = cz.alloc_outputs(1)
        cz.channels(spec, 1, out)
        torch.cuda.synchronize()
        for i, s in enumerate(shifts):
            if in_type == capi.KGPU_COMPLEX and abs(s) >= N // 2:
                continue  # outside compute_tuning's domain (radio.c:1196); documented, not compared
            y = oracle.channel_block(in_type, X, R, s)
            got = cz.channel_slice(out, i).cpu().numpy()[0]
            ref = y[pts - olen:]
            den = max(np.abs(ref).max(), 1e-3 * np.abs(X).max())
            assert np.abs(got - ref).max() / den < TOL, (in_type, s)
        cz.close()


def test_mixed_rates_cfg3_like(oracle, cuda_dev):
    """cfg-3 shape at reduced master size: 12/24/48 kHz channels side by side in one launch."""
    from ka9q_radio_b200 import capi

    L, M = 48000, 12001
    chans = []
    for i in range(12):
        olen = (240, 480, 960)[i % 3]
        chans.append(dict(olen=olen, shift=1000 + 2250 * i, low=50 / (olen * 50), high=3000 / (olen * 50), beta=11.0))
    assert _chan_case(oracle, cuda_dev, capi.KGPU_REAL, L, M, chans, nb=2) < TOL


def test_run_one_matches_batched(oracle, cuda_dev):
    from ka9q_radio_b200 import capi

    L, M = 4800, 1201
    x = oracle.siggen_real(2 * L, 0.1, 0.02, 0.2, 1.0)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev)
    for i in range(5):
        cz.add_channel(48 * (1 + i % 2), 900 + 31 * i, -0.3, 0.3, 9.0)
    spec, out = cz.alloc_spectra(2), cz.alloc_outputs(2)
    cz.forward(cz.stage_stream(x), 2, spec)
    cz.channels(spec, 2, out)
    one = torch.zeros(96, dtype=torch.complex64, device=cuda_dev)
    for i in range(5):
        cz.bank.run_one(i, spec[1].data_ptr(), one.data_ptr())
        torch.cuda.synchronize()
        ref = cz.channel_slice(out, i)[1]
        assert torch.equal(one[: ref.numel()], ref)
    cz.close()


# ------------------------------------------------------------------ BASELINE.json configs ------
def _tone_stream_i16(oracle, nsamp, fs, freqs, amp_db=-30.0, noise_db=-50.0, seed=1):
    return oracle.siggen_tones_i16(nsamp, [f / fs for f in freqs], [10 ** (amp_db / 20)] * len(freqs), 10 ** (noise_db / 20), seed)


def test_cfg2_full_size_channels_subset(oracle, cuda_dev):
    """cfg-2 at full size: 1024 NBFM channels on the 25 kHz raster + 8 inverted (negative-shift)
    channels, 2 blocks; every 37th channel and all inverted ones are checked against the oracle."""
    from ka9q_radio_b200 import capi

    L, M, fs, nb = 2592000, 648001, 129.6e6, 2
    shifts = [750_000 + 625 * k for k in range(1024)] + [-(750_000 + 625 * k) for k in (0, 3, 64, 100, 511, 700, 900, 1023)]
    tones = [30.0e6 + 25e3 * k for k in (0, 3, 37, 64, 100, 511, 700, 900, 1023, 407)]
    xi = _tone_stream_i16(oracle, nb * L, fs, tones)
    scale = np.float32(10 ** (3 / 20) / 32768)
    xf, _, _ = oracle.convert_i16(xi, scale)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, cap=len(shifts))
    for s in shifts:
        cz.add_channel(480, s, -8000 / 24000, 8000 / 24000, 11.0)
    spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(xi), nb, spec, scale=float(scale))
    cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    R = oracle.design_response(600, 480, L + M - 1, True, -1 / 3, 1 / 3, 11.0)
    check = list(range(0, 1024, 37)) + list(range(1024, len(shifts)))
    loud = 0.0
    worst = 0.0
    for b in range(nb):
        X = oracle.forward(oracle.block_window(xf, L, M, b))
        refs = {c: oracle.channel_block(oracle.KO_REAL, X, R, shifts[c])[-480:] for c in check}
        loud = max(loud, max(np.abs(r).max() for r in refs.values()))
        for c, r in refs.items():
            g = got[b, c * 480:(c + 1) * 480]
            # noise-only channels sit ~60 dB below the tones: measure against the louder of (this channel, 1e-3 of the loudest)
            worst = max(worst, np.abs(g - r).max() / max(np.abs(r).max(), 1e-3 * loud))
    cz.close()
    assert worst < TOL, worst


def test_cfg2_full_size_all_channels_tone_comb(cuda_dev):
    """Size-independent property at BASELINE.json's full cfg-2 size, ALL 1024 channels in one batched launch of
    4 blocks: a real tone A*cos at an exact bin centre whose index is a multiple of the overlap factor (V = 5)
    comes out of its channel as a CONSTANT complex sample of magnitude A/sqrt(2) from block 1 on
    (filter.c:1020-1025 gain normalisation, radio.c:1491-1497 block phase) -- checked for every channel, each
    with its own amplitude, and against leakage from the 1023 other tones.  No oracle needed at this size."""
    from ka9q_radio_b200 import capi

    L, M, nb, nch = 2592000, 648001, 4, 1024
    N = L + M - 1
    bins = [5 * (3000 + 150 * k) for k in range(nch)]          # 750-bin (30 kHz) raster, all multiples of V = 5
    amps = np.array([60.0 + 18.0 * (k % 11) for k in range(nch)])  # int16 units: rounding noise ~1e-4 of A in a channel
    rng = np.random.default_rng(5)
    ph = rng.uniform(0, 2 * np.pi, nch)
    spec = np.zeros(N // 2 + 1, np.complex128)
    spec[bins] = 0.5 * N * amps * np.exp(1j * ph)                # irfft -> sum A cos(2 pi b n / N + ph), period N
    period = np.fft.irfft(spec, N)
    reps = -(-(nb * L) // N)
    xi = np.rint(np.tile(period, reps)[: nb * L]).astype(np.int16)
    assert np.abs(xi).max() < 32000
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, cap=nch)
    for b in bins:
        cz.add_channel(480, b, -8000 / 24000, 8000 / 24000, 11.0)
    spc, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(xi), nb, spc, scale=1.0)
    cz.channels(spc, nb, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy().reshape(nb, -1)[:, : nch * 480].reshape(nb, nch, 480)
    cz.close()
    want = amps / np.sqrt(2.0)
    steady = got[1:]                                             # block 0 still contains the zero history
    mag = np.abs(steady)
    assert np.abs(mag - want[None, :, None]).max() / want.min() < 3e-3
    const = np.abs(steady - steady[:, :, :1]).max(axis=(0, 2)) / want        # constant within a block
    assert const.max() < 3e-3
    # the same complex value in every block (tone bin divisible by V: no block-to-block phase step)
    assert (np.abs(steady[1:, :, 0] - steady[:1, :, 0]) / want).max() < 3e-3


def test_cfg3_mixed_rates_full_size(oracle, cuda_dev):
    """cfg-3: RX888 input, SSB channels at 12/24/48 kHz (preset usb: +50..+3000 Hz, beta 11) in one bank."""
    from ka9q_radio_b200 import capi

    L, M, fs, nb = 2592000, 648001, 129.6e6, 1
    N = L + M - 1
    chans = []
    for i in range(30):
        olen = (240, 480, 960)[i % 3]
        rate = olen * 50
        f = 1.8e6 + i * 0.94e6
        _, shift, _ = oracle.compute_tuning(N, fs, f)
        chans.append(dict(olen=olen, shift=shift, low=50 / rate, high=3000 / rate, beta=11.0, f=f))
    xi = _tone_stream_i16(oracle, nb * L, fs, [c["f"] + 1000.0 for c in chans[::2]])
    scale = np.float32(10 ** (3 / 20) / 32768)
    xf, _, _ = oracle.convert_i16(xi, scale)
    cz = _mk(L, M, capi.KGPU_REAL, cuda_dev, cap=len(chans))
    for c in chans:
        cz.add_channel(c["olen"], c["shift"], c["low"], c["high"], c["beta"])
    spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(xi), nb, spec, scale=float(scale))
    cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    X = oracle.forward(oracle.block_window(xf, L, M, 0))
    refs = []
    for c in chans:
        pts = c["olen"] * N // L
        R = oracle.design_response(pts, c["olen"], N, True, c["low"], c["high"], c["beta"])
        refs.append(oracle.channel_block(oracle.KO_REAL, X, R, c["shift"])[-c["olen"]:])
    loud = max(np.abs(r).max() for r in refs)
    for i, r in enumerate(refs):
        g = cz.channel_slice(out, i).cpu().numpy()[0]
        assert np.abs(g - r).max() / max(np.abs(r).max(), 1e-3 * loud) < TOL, i
    cz.close()


def test_cfg4_complex_iq_int16(oracle, cuda_dev):
    """cfg-4: 20 MS/s complex int16 I/Q, N = 500 000 c2c, 512 channels on a 25 kHz raster across
    -6.4..+6.4 MHz (negative shifts and circular wrap, filter.c:728-793); every 23rd channel checked."""
    from ka9q_radio_b200 import capi

    L, M, fs, nb = 400000, 100001, 20e6, 2
    N = L + M - 1
    rng = np.random.default_rng(11)
    n = np.arange(nb * L)
    sig = sum(0.03 * np.exp(2j * np.pi * f / fs * n) for f in (-6.4e6, -1.0e6 + 25e3, 25e3 * 7, 3.2e6, 6.375e6))
    sig = sig + 0.003 * (rng.standard_normal(nb * L) + 1j * rng.standard_normal(nb * L))
    iq = np.empty(2 * nb * L, np.int16)
    iq[0::2] = np.clip(np.round(32767 * sig.real), -32767, 32767)
    iq[1::2] = np.clip(np.round(32767 * sig.imag), -32767, 32767)
    scale = np.float32(1.0 / 32768)
    xf = (iq[0::2].astype(np.float32) * scale + 1j * (iq[1::2].astype(np.float32) * scale)).astype(np.complex64)
    shifts = [int(round((-6.4e6 + 25e3 * k) / (fs / N))) for k in range(512)]
    cz = _mk(L, M, capi.KGPU_COMPLEX, cuda_dev, cap=512)
    for s in shifts:
        cz.add_channel(480, s, -1 / 3, 1 / 3, 11.0)
    spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(iq), nb, spec, scale=float(scale))
    cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    R = oracle.design_response(600, 480, N, False, -1 / 3, 1 / 3, 11.0)
    worst, loud = 0.0, 0.0
    for b in range(nb):
        X = oracle.forward(oracle.block_window(xf, L, M, b))
        assert rel_err(spec[b, :N].cpu().numpy(), X) < TOL
        refs = {c: oracle.channel_block(oracle.KO_COMPLEX, X, R, shifts[c])[-480:] for c in list(range(0, 512, 23)) + [0, 216, 263, 384, 511]}
        loud = max(loud, max(np.abs(r).max() for r in refs.values()))
        for c, r in refs.items():
            g = got[b, c * 480:(c + 1) * 480]
            worst = max(worst, np.abs(g - r).max() / max(np.abs(r).max(), 1e-3 * loud))
    cz.close()
    assert worst < TOL, worst


@pytest.mark.parametrize("name", ["real_small", "complex_small", "cfg1_siggen"])
def test_gpu_matches_golden_fixtures(oracle, cuda_dev, name):
    """The committed outputs of the reference's own filter.c (tests/golden) reproduced on the GPU."""
    from pathlib import Path

    from ka9q_radio_b200 import capi

    z = np.load(Path(__file__).resolve().parent / "golden" / f"{name}.npz")
    L, M, nb, in_type = int(z["L"]), int(z["M"]), int(z["nb"]), int(z["in_type"])
    a, n, f, s = z["sig"]
    x = oracle.siggen_real(nb * L, a, n, f, s) if in_type == oracle.KO_REAL else oracle.siggen_complex(nb * L, a, n, f, s)
    cz = _mk(L, M, in_type, cuda_dev)
    params = z["chan_params"]
    for p in params:
        cz.add_channel(int(p[0]), int(p[1]), float(p[2]), float(p[3]), float(p[4]), isb=bool(p[5]))
    if not (len(z["notch"]) == 1 and z["notch"][0] == -1):
        cz.master.set_notches([int(b) for b in z["notch"]])
    spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(x), nb, spec)
    cz.apply_notches(spec, nb)
    cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    st = int(z["spec_stride"])
    sp = spec.cpu().numpy()
    for b in range(nb):
        assert np.abs(sp[b, : cz.master.bins][::st] - z["spec_sub"][b]).max() / z["spec_absmax"][b] < TOL
        for i in range(len(params)):
            ref = z[f"out{i}"][b]
            g = cz.channel_slice(out, i).cpu().numpy()[b]
            assert np.abs(g - ref).max() / np.abs(ref).max() < TOL, (b, i)
    cz.close()
