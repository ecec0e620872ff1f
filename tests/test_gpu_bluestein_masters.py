"""Masters of any transform length (kgpu_master_create_any): Bluestein transforms on the device.

Per-bin accuracy uses the metric of tests/test_gpu_accuracy.py: e = |gpu - truth| / rms(truth), truth a float64 DFT of
exactly the float32 values the kernels saw; max e <= 5e-6, and rms(e_gpu) <= 3 rms(e_oracle) against the float32
oracle.  Spectra are pre-filled with NaN sentinels; guard rows and padding must come back bitwise unchanged.  Every
case that transforms on the CPU runs in a process of its own (see test_gpu_extended_primes._fresh).
"""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from accuracy_cases import FORWARD
from ext_prime_cases import EXT_FORWARD
from test_gpu_accuracy import MAX_E, NAN_BITS, _bits, _derandomize, _err, _sentinel, _stats_of

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
HERE = Path(__file__).resolve().parent
TOL = 1e-5  # tests/test_filter_abi.py


def _fresh(case, *args, env=None):
    code = (f"import sys; sys.path[:0] = [{str(HERE)!r}, {str(ROOT)!r}]\n"
            "import torch\nfrom oracle import oracle as O\nO.lib()\n"
            f"import test_gpu_bluestein_masters as t\nt.{case}(O, torch.device('cuda:0'), *{args!r})\nprint('case ok')\n")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **(env or {})), capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]


def _rx888(rate):
    L = rate // 50  # 20 ms blocks at overlap 5
    return L, L // 4 + 1


# (id, real, L, M, fmt, derandomize, blocks launched together, blocks checked against the float32 oracle)
GEOS = [
    ("rx888_62m_f32", True, *_rx888(62_000_000), "f32", False, 2, 2),
    ("rx888_116m_f32_chunked", True, *_rx888(116_000_000), "f32", False, 7, 1),  # 5 blocks per scratch chunk
    ("rx888_62m_i16_derand", True, *_rx888(62_000_000), "i16", True, 3, 0),
    ("complex_2m9_f32", False, 58_000, 14_501, "f32", False, 3, 3),
    ("complex_2m9_i16", False, 58_000, 14_501, "i16", False, 4, 0),
    ("complex_7919_f32", False, 63_352, 15_839, "f32", False, 1, 1),
    ("real_37_f32", True, 59_200, 14_801, "f32", False, 4, 4),                  # Nc = 37000 = 2^3 5^3 37
    ("complex_1009_i16_derand", False, 290_592, 72_649, "i16", True, 2, 0),     # N = 2^3 3^2 5 1009
]
_GEO = {g[0]: g for g in GEOS}


@pytest.mark.parametrize("gid", [g[0] for g in GEOS])
def test_bluestein_per_bin_accuracy_writes_and_stats(cuda_dev, gid):
    _fresh("_case_accuracy", gid)


def _case_accuracy(oracle, dev, gid):
    from ka9q_radio_b200 import capi

    _, real, L, M, fmt, derand, nb, n_ora = _GEO[gid]
    in_type = capi.KGPU_REAL if real else capi.KGPU_COMPLEX
    N = L + M - 1
    per = 1 if real else 2
    rng = np.random.default_rng(N)
    nsamp = (M - 1 + nb * L) * per  # history of block 0, then nb blocks of new samples
    if fmt == "i16":
        xi = rng.integers(-32768, 32768, nsamp, dtype=np.int16)
        specials = np.array([32767, -32767, -32768, 32766], np.int16)
        for b in range(nb):
            for k, pos in enumerate((M - 1 + b * L, M - 1 + b * L + L - 1, M - 2 + b * L)):
                xi[pos * per:(pos + 1) * per] = specials[(2 * b + k) % 4]
        scale = float(np.float32(10 ** (3 / 20) / 32768))
        xd = _derandomize(xi) if derand else xi
        xf = xd.astype(np.float32) * np.float32(scale)
        d_in = torch.from_numpy(xi).to(dev)
        ifmt = capi.KGPU_FMT_I16
    else:
        xf = rng.standard_normal(nsamp, dtype=np.float32)
        scale = 1.0
        d_in = torch.from_numpy(xf).to(dev)
        ifmt = capi.KGPU_FMT_F32
    z = xf if real else (xf[0::2] + 1j * xf[1::2]).astype(np.complex64)  # samples as the kernels saw them
    m = capi.Master(L, M, in_type, any_length=True)
    try:
        path, text = capi.plan_master(L, M, in_type)
        assert path == capi.MASTER_BLUESTEIN and m.describe() == text, (m.describe(), text)
        bins, stride = m.bins, m.spec_stride
        buf = _sentinel(nb + 2, stride, dev)
        spec = buf[1:nb + 1]
        st = torch.zeros(2 * nb, dtype=torch.int64, device=dev)
        stream = torch.cuda.current_stream().cuda_stream
        m.forward(d_in.data_ptr(), ifmt, scale, nb, spec.data_ptr(), stream, derandomize=derand,
                  d_stats=st.data_ptr() if fmt == "i16" else 0)
        one = _sentinel(1, stride, dev)
        if nb > 1:  # the last block launched alone (a different chunk split) gives bitwise the same spectrum
            off = (nb - 1) * L * per * d_in.element_size()
            m.forward(d_in.data_ptr() + off, ifmt, scale, 1, one.data_ptr(), stream, derandomize=derand)
        torch.cuda.synchronize()
        got = spec.cpu().numpy()[:, :bins]
    finally:
        m.close()
    raw = _bits(buf)
    assert (raw[0] == NAN_BITS).all() and (raw[nb + 1] == NAN_BITS).all(), "store outside the launched blocks' rows"
    assert (raw[1:nb + 1, 2 * bins:] == NAN_BITS).all(), "store into the row padding [bins, spec_stride)"
    assert np.isfinite(got).all(), "bin left unwritten"
    if nb > 1:
        assert np.array_equal(_bits(one)[0], raw[nb]), "a block's spectrum depends on the launch it is in"
    if fmt == "i16":
        stats = st.cpu().numpy().reshape(nb, 2)
        for b in range(nb):
            lo = (M - 1 + b * L) * per
            want = _stats_of(xd[lo:lo + L * per])
            assert (int(stats[b, 0]), int(stats[b, 1]) & 0xFFFFFFFF) == want, (gid, b)
    e_gpu, e_ora, worst = [], [], 0.0
    for b in range(nb):
        w = z[b * L:b * L + N]
        truth = np.fft.rfft(w.astype(np.float64)) if real else np.fft.fft(w.astype(np.complex128))
        e = _err(got[b], truth)
        worst = max(worst, e.max())
        if b < n_ora:
            e_gpu.append(e)
            e_ora.append(_err(oracle.forward(w), truth))
    msg = f"bluestein accuracy {gid}: max e {worst:.2e} over {nb} blocks"
    if e_gpu:
        eg, eo = np.concatenate(e_gpu), np.concatenate(e_ora)
        ratio = np.sqrt(np.mean(eg ** 2)) / np.sqrt(np.mean(eo ** 2))
        msg += f", rms {np.sqrt(np.mean(eg ** 2)):.2e} (oracle {np.sqrt(np.mean(eo ** 2)):.2e}, ratio {ratio:.2f})"
        assert ratio <= 3.0, msg
    print(msg)
    assert worst <= MAX_E, msg


# ------------------------------------------------------------------ the masters create_ex serves ----------------
SMOOTH = [g for g in FORWARD if g.id in ("c800x625", "r1296x1250", "c1296x1215", "r1280x1250")] + \
         [g for g in EXT_FORWARD if g.id in ("airspyhf_912k", "r153x135", "rx888_60m8")]


@pytest.mark.parametrize("geo", SMOOTH, ids=lambda g: g.id)
def test_create_any_is_create_ex_where_that_serves(cuda_dev, geo):
    """Same describe() (and kgpu_master_plan's string) and bitwise the same spectra of two blocks, int16 with stats."""
    from ka9q_radio_b200 import capi

    in_type = capi.KGPU_REAL if geo.real else capi.KGPU_COMPLEX
    per = 1 if geo.real else 2
    rng = np.random.default_rng(geo.L)
    x = torch.from_numpy(rng.integers(-32768, 32768, (geo.L + geo.M - 1 + geo.L) * per, dtype=np.int16)).to(cuda_dev)
    out = []
    for kw in (dict(extended=True), dict(any_length=True)):
        m = capi.Master(geo.L, geo.M, in_type, **kw)
        try:
            spec = torch.empty(2 * m.spec_stride, dtype=torch.complex64, device=cuda_dev)
            st = torch.zeros(4, dtype=torch.int64, device=cuda_dev)
            m.forward(x.data_ptr(), capi.KGPU_FMT_I16, 1e-4, 2, spec.data_ptr(), torch.cuda.current_stream().cuda_stream,
                      d_stats=st.data_ptr())
            torch.cuda.synchronize()
            out.append((m.describe(), _bits(spec.view(2, -1)[:, :m.bins]), st.cpu().numpy()))
        finally:
            m.close()
    assert out[0][0] == out[1][0] == capi.plan_master(geo.L, geo.M, in_type)[1]
    assert np.array_equal(out[0][1], out[1][1])
    assert np.array_equal(out[0][2], out[1][2])


# ------------------------------------------------------------------ through filter.h ---------------------------
def _driver(name):
    from test_filter_abi import _load

    return _load(name)


L62, M62 = _rx888(62_000_000)
N62 = L62 + M62 - 1


def _bank62():
    h = N62 // 2
    return [dict(olen=480, shift=123_457, low=-0.4, high=0.4, beta=11.0),          # NBFM, 600 points
            dict(olen=240, shift=h - 200, low=0.01, high=0.3, beta=11.0),          # usb near Nyquist, 300 points
            dict(olen=240, shift=-311_111, low=-0.3, high=-0.01, beta=11.0),       # lsb, negative shift
            dict(olen=7680, shift=250_000, low=-0.45, high=0.45, beta=11.0),       # 384 kHz, 9600 points (wide)
            dict(olen=30720, shift=400_000, low=-0.45, high=0.45, beta=11.0)]      # 1.536 MS/s, 38400 points (huge)


def _stream62(nb, seed=62):
    rng = np.random.default_rng(seed)
    n = np.arange(nb * L62)
    x = 0.3 * np.cos(2 * np.pi * 123_457.3 / N62 * n) + 0.1 * np.cos(2 * np.pi * 400_123.1 / N62 * n)
    return (x + 0.05 * rng.standard_normal(len(n))).astype(np.float32)


@pytest.mark.parametrize("driver", ["driver_gpuhdr.so", "driver_refhdr.so"])
def test_rx888_62m_through_filter_h(cuda_dev, driver):
    """create_filter_input(1240000, 310001, REAL): a mixed bank with a DC and a spur notch, three blocks, against the
    restated path and the reference's own filter.c where it is built."""
    if _driver(driver) is None:
        pytest.skip(f"{driver} not built")
    _fresh("_case_62m_through_filter_h", driver, env={"KA9Q_GPU_SPECTRUM_D2H": "all"})


def _case_62m_through_filter_h(oracle, dev, driver):
    lib = _driver(driver)
    nb = 3
    x = _stream62(nb)
    chans = _bank62()
    got, gspec = oracle.ref_run_stream(x, L62, M62, chans, notch_bins=[98_765], keep_spectra=True, lib=lib)
    refs = [("restated", *oracle.run_stream(x, L62, M62, chans, notch_bins=[98_765], keep_spectra=True))]
    if oracle.ref_available():
        refs.append(("filter.c", *oracle.ref_run_stream(x, L62, M62, chans, notch_bins=[98_765], keep_spectra=True)))
    for what, r, rs in refs:
        for b in range(nb):
            assert np.abs(gspec[b] - rs[b]).max() / np.abs(rs[b]).max() < TOL, (what, b)
            for c in range(len(chans)):
                assert np.abs(got[b][c] - r[b][c]).max() / np.abs(r[b][c]).max() < TOL, (what, b, c)


def test_rx888_62m_int16_through_filter_h(cuda_dev):
    """write_i16filter with the randomizer off and on, the same bank, against the restated path on the converted
    samples."""
    if not hasattr(_driver("driver_gpuhdr.so"), "ref_write_i16"):
        pytest.skip("driver without write_i16filter")
    _fresh("_case_62m_int16")


def _case_62m_int16(oracle, dev):
    lib = _driver("driver_gpuhdr.so")
    nb = 2
    xi = oracle.siggen_tones_i16(nb * L62, [123_457.3 / N62, 250_017.7 / N62], [0.1, 0.05], 0.01, 1)
    scale = np.float32(10 ** (3 / 20) / 32768)
    chans = _bank62()
    for derand in (0, 1):
        xf, _, _ = oracle.convert_i16(xi, scale, randomize=bool(derand))
        ref, _ = oracle.run_stream(xf, L62, M62, chans)
        with oracle.RefSession(L62, M62, oracle.KO_REAL, lib=lib) as s:
            ids = [s.add_channel(ch["olen"], ch["low"], ch["high"], ch["beta"]) for ch in chans]
            for b in range(nb):
                blk = np.ascontiguousarray(xi[b * L62:(b + 1) * L62])
                assert lib.ref_write_i16(s.h, blk, L62, float(scale), derand) == 1
                for c, (i, ch) in enumerate(zip(ids, chans)):
                    y = s.execute(i, ch["shift"])
                    r = ref[b][c]
                    assert np.abs(y - r).max() / np.abs(r).max() < TOL, (derand, b, c)


F29 = 2_900_000
L29, M29 = F29 // 50, F29 // 200 + 1
N29 = L29 + M29 - 1


def _stream29(nb):
    rng = np.random.default_rng(29)
    n = np.arange(nb * L29)
    tone = 0.3 * np.exp(2j * np.pi * 0.0917 * n) + 0.1 * np.exp(-2j * np.pi * 0.3 * n)
    return (tone + 0.05 * (rng.standard_normal(len(n)) + 1j * rng.standard_normal(len(n)))).astype(np.complex64)


@pytest.mark.parametrize("driver", ["driver_gpuhdr.so", "driver_refhdr.so"])
def test_complex_2m9_through_filter_h(cuda_dev, driver):
    """create_filter_input(58000, 14501, COMPLEX), N = 2^2 5^4 29: channels with positive, negative and wrapping shifts,
    ISB and notches, four blocks."""
    if _driver(driver) is None:
        pytest.skip(f"{driver} not built")
    _fresh("_case_2m9_through_filter_h", driver, env={"KA9Q_GPU_SPECTRUM_D2H": "all"})


def _case_2m9_through_filter_h(oracle, dev, driver):
    lib = _driver(driver)
    nb = 4
    x = _stream29(nb)
    h = N29 // 2
    chans = []
    for olen in (240, 480, 960):
        pts = olen * N29 // L29
        chans += [dict(olen=olen, shift=6649, low=-0.4, high=0.4, beta=11.0),
                  dict(olen=olen, shift=-21_750, low=-0.4, high=0.4, beta=11.0),
                  dict(olen=olen, shift=h - pts // 4, low=-0.4, high=0.4, beta=11.0),
                  dict(olen=olen, shift=pts // 8, low=-0.45, high=0.1, beta=7.0)]
    chans.append(dict(olen=480, shift=1500, low=-0.3, high=0.3, beta=9.0, isb=True))
    got, gspec = oracle.ref_run_stream(x, L29, M29, chans, notch_bins=[4321], keep_spectra=True, lib=lib)
    refs = [("restated", *oracle.run_stream(x, L29, M29, chans, notch_bins=[4321], keep_spectra=True))]
    if oracle.ref_available():
        refs.append(("filter.c", *oracle.ref_run_stream(x, L29, M29, chans, notch_bins=[4321], keep_spectra=True)))
    for what, r, rs in refs:
        for b in range(nb):
            assert np.abs(gspec[b] - rs[b]).max() / np.abs(rs[b]).max() < TOL, (what, b)
            for c in range(len(chans)):
                assert np.abs(got[b][c] - r[b][c]).max() / np.abs(r[b][c]).max() < TOL, (what, b, c)


def test_complex_2m9_tuned_output_and_noise_through_filter_h(cuda_dev):
    """execute_filter_output_tuned and filter_noise_estimate on a Bluestein master, against the restated radio.c."""
    _fresh("_case_2m9_tuned_and_noise")


def _case_2m9_tuned_and_noise(oracle, dev):
    lib = _driver("driver_gpuhdr.so")
    L, M, N, fs = L29, M29, N29, float(F29)
    nb = 6
    x = _stream29(nb)
    freqs = [[265_917.3, -870_234.5] for _ in range(nb)]
    for b in range(3, nb):
        freqs[b][0] = 270_350.6
    rate, olen = [24000.0, 12000.0], [480, 240]
    R = [oracle.design_response(o * N // L, o, N, False, lo, hi, 11.0) for o, lo, hi in ((480, -0.4, 0.4), (240, 0.01, 0.3))]
    fts = [oracle.FineTune(L, M, r) for r in rate]
    with oracle.RefSession(L, M, oracle.KO_COMPLEX, lib=lib) as s:
        ids = [s.add_channel(480, -0.4, 0.4, 11.0), s.add_channel(240, 0.01, 0.3, 11.0)]
        assert lib.ref_enable_noise(s.h, fs) == 0
        for b in range(nb):
            assert s.write(x[b * L:(b + 1) * L]) == 1
            X = oracle.forward(oracle.block_window(x, L, M, b))
            for i in range(2):
                rc, shift, rem = oracle.compute_tuning(N, fs, freqs[b][i])
                y = np.empty(olen[i], np.complex64)
                pw = C.c_double(0)
                assert lib.ref_execute_tuned(s.h, ids[i], shift, rem, rate[i], 0.0, y, C.byref(pw)) == 0
                r = oracle.channel_block(oracle.KO_COMPLEX, X, R[i], shift)[-olen[i]:].copy()
                p_ref = fts[i].block(r, shift, rem)
                assert np.abs(y - r).max() / np.abs(r).max() < TOL, (b, i)
                assert abs(pw.value - p_ref) / p_ref < TOL, (b, i)
                n0 = lib.ref_noise(s.h, ids[i])
                if not np.isnan(n0):  # NAN only for a block recomputed alone right after a (re)tune
                    ref_n0 = oracle.estimate_noise(oracle.KO_COMPLEX, X, len(R[i]), shift, fs)
                    assert abs(n0 - ref_n0) / ref_n0 < 1e-5, (b, i)
                else:
                    assert b in (0, 3)
