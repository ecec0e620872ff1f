"""The two per-channel kernels that run after the filter (noise_kernel.cuh), case by case against plain references:

noise_kernel (estimate_noise, radio.c:1783-1866): every (channel, block) against oracle.estimate_noise and the numpy
restatement in noise_fm_ref.py, both fed the exact float32 spectrum the kernel read.  Spectra are written straight
into the spectrum buffer, so any window and any bin content is reachable: every slave width up to the widest channel
(28812 points), windows clamped at DC and Nyquist, the COMPLEX walk through DC and into the master's Nyquist bin, and
order statistics built from energies that are exact in float32.  n0 is prefilled with NaN; only runnable channels get
an estimate, defined but disabled ones get 0, and nothing past the bank's channels is written.

fm_front_kernel (fm.c:104-131, :205-231 without threshold): synthetic channel outputs against a float64 restatement,
across launches of 1-4 blocks with the discriminator memory carried, including a channel skipped for one launch."""
import numpy as np
import pytest
import torch

import noise_fm_ref as R
from test_filter_abi import _load
from test_gpu_wide_channels import oracle  # noqa: F401  (private oracle copy: this file needs many FFT lengths)

pytestmark = pytest.mark.gpu

FS = 4.8e6
EXACT_TOL, GAUSS_TOL = 1e-12, 1e-6


def _mk(L, M, in_type, dev, cap):
    from ka9q_radio_b200.channelizer import Channelizer

    return Channelizer(L, M, in_type, dev, capacity=cap)


def _add(cz, points, shift, real_out=False):
    """a channel of `points` points (the master has N == L, so points == olen) with a flat response"""
    from ka9q_radio_b200 import capi

    assert cz.N == cz.L
    return cz.add_channel(points, shift, response=np.ones(points, np.complex64),
                          out_type=capi.KGPU_REAL if real_out else capi.KGPU_COMPLEX)


def _run_noise(cz, spectra, dev):
    """spectra [nb][bins] -> (n0 [nb][capacity] from the device, the spectra as the device holds them)"""
    nb = len(spectra)
    spec = cz.alloc_spectra(nb)
    spec.fill_(complex(float("nan"), float("nan")))   # a read past the master's bins would show as NaN
    spec[:, : cz.master.bins] = torch.from_numpy(np.stack(spectra)).to(dev)
    n0 = torch.full((nb, cz.capacity), float("nan"), dtype=torch.float64, device=dev)
    cz.bank.noise(spec.data_ptr(), nb, FS, n0.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize()
    return n0.cpu().numpy(), spec[:, : cz.master.bins].cpu().numpy()


def _score(oracle, cz, got, sp, chans, tol, use_oracle=True, label=""):
    """chans: (idx, s_bins, shift, name).  Returns the worst relative error over every (channel, block)."""
    from ka9q_radio_b200 import capi

    cplx = cz.in_type == capi.KGPU_COMPLEX
    worst = 0.0
    for b in range(len(sp)):
        for idx, s_bins, shift, name in chans:
            refs = [R.estimate_noise(sp[b], cplx, s_bins, shift, FS)]
            if use_oracle:
                refs.append(oracle.estimate_noise(oracle.KO_COMPLEX if cplx else oracle.KO_REAL, sp[b], s_bins, shift, FS))
            for ref in refs:
                if ref == 0:
                    assert got[b, idx] == 0, (label, name, b, s_bins, shift, got[b, idx])
                    continue
                e = abs(got[b, idx] - ref) / ref
                assert e <= tol, (label, name, b, s_bins, shift, got[b, idx], ref)
                worst = max(worst, e)
    return worst


def _check_untouched(got, cz, disabled):
    assert np.isnan(got[:, cz.nchan:]).all(), "n0 written past the bank's channels"
    for idx in disabled:
        assert (got[:, idx] == 0).all(), ("disabled channel", idx)


# ------------------------------------------------------------------ noise: widths and window edges -------------------
COMPLEX_WIDTHS = [480, 1125, 2000, 3375, 4800, 7200, 7290, 9600, 15360, 28812]
REAL_OUT_WIDTHS = [1200, 9600, 28812]  # slave bins 601 (raised to 1000), 4801, 14407


def _gauss(rng, n):
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.01).astype(np.complex64)
    x[rng.integers(0, n, n // 20)] *= 40  # strong bins for the 1.5 q threshold to drop
    return x


@pytest.mark.parametrize("master", ["real", "complex"])
def test_noise_widths_and_edges(oracle, cuda_dev, master):
    """every width class (below 1000, up to 4096, 4097-7260, wide, REAL-output) at random and at edge shifts, 3 blocks
    with different Gaussian spectra, on a 96000-point master"""
    from ka9q_radio_b200 import capi

    cplx = master == "complex"
    it = capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL
    rng = np.random.default_rng(21 + cplx)
    L = 96000
    chans = []  # (points, real_out, shift)
    m = L if cplx else L // 2 + 1
    for pts, ro in [(p, False) for p in COMPLEX_WIDTHS] + [(p, True) for p in REAL_OUT_WIDTHS]:
        n = max(pts // 2 + 1 if ro else pts, 1000)
        if cplx:
            h = m // 2
            edge = [n // 2 - 5,           # window starts 5 bins below DC: wraps to the top of the master
                    h - 7 + n // 2,       # runs into bin m/2 after 7 bins: zeros after it
                    h + n // 2,           # starts exactly at m/2: a full turn
                    h + 1 + n // 2, -h, m + 100 + n // 2,
                    n // 2 - m - 1]       # start below -m: the reference gives up, 0
        else:
            edge = [0, 3, -3,                            # clamped at DC
                    n // 2, n // 2 + 1, -(n // 2) - 1,   # touching DC exactly, one bin away (negative shift: abs)
                    m - n + n // 2, m - n + n // 2 - 1,  # touching Nyquist exactly, one bin away
                    m - 1, 1 - m]                        # clamped at Nyquist
        for sh in edge + [int(s) for s in rng.integers(-(m // 2), m // 2, 2)]:
            chans.append((pts, ro, sh))
    cz = _mk(L, 1, it, cuda_dev, cap=len(chans) + 8)
    assert cz.master.bins == m
    idxs = [_add(cz, p, sh, ro) for p, ro, sh in chans]
    off = _add(cz, 9600, 1234)   # defined, then disabled: 0
    cz.bank.enable(off, False)
    got, sp = _run_noise(cz, [_gauss(rng, m) for _ in range(3)], cuda_dev)
    _check_untouched(got, cz, [off])
    sc = [(i, p // 2 + 1 if ro else p, sh, f"{p}{'r' if ro else ''}") for i, (p, ro, sh) in zip(idxs, chans)]
    worst = _score(oracle, cz, got, sp, sc, GAUSS_TOL, label=master)
    print(f"\nnoise widths/edges {master}: {len(sc)} channels x 3 blocks, worst rel err {worst:.2e}")
    cz.close()


def test_noise_real_master_smaller_than_window(oracle, cuda_dev):
    """a 301-bin REAL master under 1000-bin windows: the documented zero fill, against the numpy restatement only (the
    reference reads past its master there)"""
    from ka9q_radio_b200 import capi

    rng = np.random.default_rng(23)
    cz = _mk(480, 121, capi.KGPU_REAL, cuda_dev, cap=6)
    shifts = [0, 100, -300, 150]
    for sh in shifts:
        cz.add_channel(480, sh, response=np.ones(600, np.complex64))
    got, sp = _run_noise(cz, [_gauss(rng, cz.master.bins) for _ in range(2)], cuda_dev)
    _check_untouched(got, cz, [])
    worst = _score(oracle, cz, got, sp, [(i, 600, s, "small") for i, s in enumerate(shifts)], GAUSS_TOL, use_oracle=False)
    print(f"\nnoise small REAL master: worst rel err {worst:.2e}")
    cz.close()


# ------------------------------------------------------------------ noise: order statistics --------------------------
@pytest.mark.parametrize("nb", [1, 3])
def test_noise_order_statistics_exact(oracle, cuda_dev, nb):
    """windows whose energies are exact in float32 (noise_fm_ref.order_stat_windows): ties at the quantile,
    cnt_le == k+1 and k+2, frac == 0, bins exactly at 1.5 q, all zero, subnormal, 1e-30..1e30, wide ties.
    Only the summation order differs from the references: 1e-12."""
    from ka9q_radio_b200 import capi

    rng = np.random.default_rng(31 + nb)
    cases = R.order_stat_windows(rng)
    cz = _mk(96000, 1, capi.KGPU_REAL, cuda_dev, cap=len(cases) + 4)
    m = cz.master.bins
    spectra, shifts = [], None
    for b in range(nb):  # the same windows, permuted differently in every block
        X = R.exact_components(rng, m)
        sh = R.place_windows(X, [bld(rng) for _, _, _, bld in cases])
        assert shifts is None or sh == shifts
        shifts = sh
        spectra.append(X)
    idxs = [_add(cz, pts, s, ro) for (_, pts, ro, _), s in zip(cases, shifts)]
    got, sp = _run_noise(cz, spectra, cuda_dev)
    _check_untouched(got, cz, [])
    for (name, pts, ro, _), i, s in zip(cases, idxs, shifts):
        w = _score(oracle, cz, got, sp, [(i, pts // 2 + 1 if ro else pts, s, name)], EXACT_TOL, label=name)
        print(f"\nnoise exact {name:20s} n0 {got[0, i]:.6e} worst rel err {w:.2e}")
    assert (got[:, idxs[[c[0] for c in cases].index("all zero")]] == 0).all()
    assert (got[:, idxs[[c[0] for c in cases].index("subnormal")]] > 0).all(), "subnormal energies flushed"
    cz.close()


# ------------------------------------------------------------------ noise: from a real forward pass ------------------
@pytest.mark.parametrize("master", ["real", "complex"])
def test_noise_wide_channels_forward_pass(oracle, cuda_dev, master):
    """wfm-sized and wider channels on a spectrum from the device's own forward pass (N 60000, overlap 5)"""
    from ka9q_radio_b200 import capi

    it = capi.KGPU_REAL if master == "real" else capi.KGPU_COMPLEX
    L, M, nb, fs = 48000, 12001, 2, 2.4e6
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.0731, 1.0) if it == capi.KGPU_REAL else \
        oracle.siggen_complex(nb * L, 0.1, 0.02, 0.0731, 1.0)
    chans = [(7680, 9000), (7680, -17000), (12288, 20000), (23040, 3000), (3840, 27000), (480, 5000)]  # olen, shift
    cz = _mk(L, M, it, cuda_dev, cap=len(chans))
    for o, s in chans:
        cz.add_channel(o, s, response=np.ones(o * 5 // 4, np.complex64))
    spec = cz.alloc_spectra(nb)
    cz.forward(cz.stage_stream(x), nb, spec)
    n0 = cz.noise(spec, nb, fs)
    torch.cuda.synchronize()
    got, sp = n0.cpu().numpy(), spec[:, : cz.master.bins].cpu().numpy()
    worst = 0.0
    for b in range(nb):
        for i, (o, s) in enumerate(chans):
            cplx = it == capi.KGPU_COMPLEX
            for ref in (oracle.estimate_noise(it, sp[b], o * 5 // 4, s, fs), R.estimate_noise(sp[b], cplx, o * 5 // 4, s, fs)):
                assert ref > 0 and abs(got[b, i] - ref) / ref < GAUSS_TOL, (b, o, s, got[b, i], ref)
                worst = max(worst, abs(got[b, i] - ref) / ref)
    print(f"\nnoise forward pass {master}: worst rel err {worst:.2e}")
    cz.close()


def test_noise_wfm_through_filter_h(oracle, cuda_dev):
    """end to end: a 9600-point wfm slave (olen 7680, overlap 5) through the filter.h surface with
    filter_input_enable_noise; filter_noise_estimate against oracle.estimate_noise on each block's spectrum"""
    lib = _load("driver_gpuhdr.so")
    L, M, nb = 96000, 24001, 4
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.1234, 1.0)
    shift = 11520
    with oracle.RefSession(L, M, oracle.KO_REAL, lib=lib) as s:
        ch = s.add_channel(7680, -0.4, 0.4, 11.0)
        assert lib.ref_channel_points(s.h, ch) == 9600
        assert lib.ref_enable_noise(s.h, FS) == 0
        checked = 0
        for b in range(nb):
            assert s.write(x[b * L:(b + 1) * L]) == 1
            s.execute(ch, shift)
            n0 = lib.ref_noise(s.h, ch)
            if np.isnan(n0):  # a block recomputed alone right after the shift was set carries no estimate
                assert b == 0
                continue
            X = oracle.forward(oracle.block_window(x, L, M, b))
            ref = oracle.estimate_noise(oracle.KO_REAL, X, 9600, shift, FS)
            assert ref > 0 and abs(n0 - ref) / ref < 1e-5, (b, n0, ref)
            checked += 1
        assert checked >= nb - 1


# ------------------------------------------------------------------ FM discriminator front half ----------------------
def _fm_signal(rng, n):
    """amplitude-varying samples with exact zeros, phase steps near +-pi and exact sign flips"""
    amp = (0.5 + 0.4 * np.sin(np.linspace(0, rng.uniform(3, 30), n) + rng.uniform(0, 6))) * rng.uniform(0.5, 2)
    ph = np.cumsum(rng.uniform(-2.5, 2.5, n))
    y = (amp * np.exp(1j * ph)).astype(np.complex64)
    k = max(n // 25, 1)
    for j in np.sort(rng.choice(np.arange(1, n), min(k, n - 1), replace=False)):
        r = rng.integers(4)
        if r == 0:
            y[j] = 0
        elif r == 1:
            y[j] = -y[j - 1]
        else:  # a phase step within 1e-4 rad of +-pi
            step = np.pi - rng.uniform(1e-6, 1e-4)
            y[j] = np.complex64(y[j - 1] * np.exp(1j * (step if r == 2 else -step)) * 0.9)
    if rng.integers(2):
        y[0] = 0
    return y


def test_fm_front_blocks_launches_and_skipped_channel(cuda_dev):
    from ka9q_radio_b200 import capi

    rng = np.random.default_rng(41)
    L = 96000
    cz = _mk(L, 1, capi.KGPU_REAL, cuda_dev, cap=16)
    olens = [8, 100, 480, 1000, 7680]
    fm = [_add(cz, o, 1000 * (i + 1)) for i, o in enumerate(olens)]
    real_out = _add(cz, 480, 500, real_out=True)
    toggled = _add(cz, 480, 7000)         # disabled for the second launch only
    always_off = _add(cz, 100, 900)
    cz.bank.enable(always_off, False)
    live = fm + [toggled]
    olen = dict(zip(fm, olens)) | {toggled: 480}
    prev = {i: np.complex64(0) for i in live}
    st = torch.cuda.current_stream(cuda_dev).cuda_stream
    worst = dict(bb=0.0, mean=0.0, dev=0.0)
    for launch, nblk in enumerate((1, 2, 3, 4)):
        cz.bank.enable(toggled, launch != 1)
        active = [i for i in live if i != toggled or launch != 1]
        stride = cz.bank.out_stride
        outs = np.full((nblk, stride), np.nan + 1j * np.nan, np.complex64)
        for i in live + [always_off]:   # every row holds samples, whether its channel runs or not
            o = cz.bank.out_offset(i)
            for b in range(nblk):
                outs[b, o:o + (olen.get(i, 100))] = _fm_signal(rng, olen.get(i, 100))
        ro = cz.bank.out_offset(real_out)
        outs[:, ro:ro + 240] = (rng.standard_normal((nblk, 240)) + 1j * rng.standard_normal((nblk, 240))).astype(np.complex64)
        d_out = torch.from_numpy(outs).to(cuda_dev)
        bb = torch.full((nblk, 2 * stride), float("nan"), dtype=torch.float32, device=cuda_dev)
        stats = torch.full((nblk, cz.capacity, 2), float("nan"), dtype=torch.float64, device=cuda_dev)
        cz.bank.fm_front(d_out.data_ptr(), nblk, bb.data_ptr(), stats.data_ptr(), st)
        torch.cuda.synchronize()
        bbh, sth = bb.cpu().numpy(), stats.cpu().numpy()
        written = np.zeros(bbh.shape, bool)
        for b in range(nblk):
            for i in active:
                o, n = cz.bank.out_offset(i), olen[i]
                y = outs[b, o:o + n]
                ref_bb, ref_mean, ref_dev = R.fm_front(y, prev[i])
                prev[i] = y[-1]
                g = bbh[b, 2 * o:2 * o + n]
                written[b, 2 * o:2 * o + n] = True
                e = float(np.abs(g.astype(np.float64) - ref_bb).max())
                assert e <= 1.2e-7, (launch, b, i, n, e, int(np.abs(g - ref_bb).argmax()))
                em = abs(sth[b, i, 0] - ref_mean) / ref_mean
                assert em <= 3e-7, (launch, b, i, sth[b, i, 0], ref_mean)
                amax = float(np.abs(y).max())
                ed = abs(sth[b, i, 1] - ref_dev)
                assert ed <= 1e-6 * ref_dev + n * (4 * 2.0 ** -24 * amax) ** 2, (launch, b, i, sth[b, i, 1], ref_dev)
                worst["bb"], worst["mean"] = max(worst["bb"], e), max(worst["mean"], em)
                worst["dev"] = max(worst["dev"], ed / ref_dev)
        assert np.isnan(bbh[~written]).all(), f"launch {launch}: baseband written outside the running channels' runs"
        skipped = [i for i in range(cz.capacity) if i not in active]
        assert np.isnan(sth[:, skipped]).all(), f"launch {launch}: stats written for a skipped channel"
    print(f"\nfm front: worst baseband {worst['bb']:.2e} (units of pi), mean rel {worst['mean']:.2e}, "
          f"deviation rel {worst['dev']:.2e}")
    cz.close()
