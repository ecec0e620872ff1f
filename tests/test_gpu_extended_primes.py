"""Masters whose transform length has prime factors 11, 13, 17, 19 or 23 (kgpu_master_create_ex) on the device.

Per-bin accuracy uses the metric and bounds of tests/test_gpu_accuracy.py: e = |gpu - truth| / rms(truth), truth a
float64 transform of exactly the float32 window, max e <= 5e-6, and with >= 4096 values gpu/oracle rms <= 2 and
max <= 4.  Spectra are pre-filled with NaN sentinels; guard rows and padding must come back bitwise unchanged.
"""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from accuracy_cases import FORWARD
from ext_prime_cases import AIRSPYHF_RATES, EXT_FORWARD, NEW_PRIMES
from test_gpu_accuracy import MAX_E, NAN_BITS, _bits, _derandomize, _err, _score, _sentinel, _stats_of

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
HERE = Path(__file__).resolve().parent
TOL = 1e-5  # tests/test_filter_abi.py


def _fresh(case, *args, env=None):
    """Runs this module's `case(oracle, device, *args)` in a new Python process.

    The float32 reference transforms keep one plan per transform length in a process-wide cache of 64 lengths, and a
    length past the 64th crashes the process.  The rest of the GPU suite shares one process and already uses most of
    those slots, so every test here that transforms on the CPU (about twenty new lengths in all) runs in a process of its
    own and leaves the suite's cache as it found it."""
    import os

    code = (f"import sys; sys.path[:0] = [{str(HERE)!r}, {str(ROOT)!r}]\n"
            "import torch\nfrom oracle import oracle as O\nO.lib()\n"
            f"import test_gpu_extended_primes as t\nt.{case}(O, torch.device('cuda:0'), *{args!r})\nprint('case ok')\n")
    full_env = dict(os.environ, **(env or {}))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, cwd=ROOT, env=full_env, capture_output=True, text=True, timeout=1200)
    print(r.stdout)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]


_BY_ID = {g.id: g for g in EXT_FORWARD}


def _cz(L, M, in_type, dev, cap=1):
    from ka9q_radio_b200.channelizer import Channelizer

    return Channelizer(L, M, in_type, dev, capacity=cap, extended=True)


def _stream(rng, n, real):
    if real:
        return rng.standard_normal(n, dtype=np.float32)
    return (rng.standard_normal(n, dtype=np.float32) + 1j * rng.standard_normal(n, dtype=np.float32)).astype(np.complex64)


@pytest.mark.parametrize("geo", EXT_FORWARD, ids=lambda g: g.id)
def test_extended_forward_per_bin_accuracy_and_writes(cuda_dev, geo):
    """White Gaussian input, blocks 1 and 2 in one launch; kgpu_use_static_kernels(0) gives bitwise the same spectra."""
    _fresh("_case_forward_accuracy", geo.id)


def _case_forward_accuracy(oracle, cuda_dev, geo_id):
    from ka9q_radio_b200 import capi

    geo = _BY_ID[geo_id]

    lib = capi.load()
    in_type = capi.KGPU_REAL if geo.real else capi.KGPU_COMPLEX
    L, M = geo.L, geo.M
    x = _stream(np.random.default_rng(L + M), 3 * L, geo.real)
    cz = _cz(L, M, in_type, cuda_dev)
    try:
        n1, n2 = geo.split
        cols, rows = (",".join(map(str, r)) for r in geo.plan)
        desc = cz.master.describe()
        assert f"two-pass {n1} x {n2}; cols radices [{cols}] rows radices [{rows}]" in desc, desc
        assert desc.endswith("kernels fwd_cols_ext + fwd_rows_ext"), desc
        bins, stride = cz.master.bins, cz.master.spec_stride
        buf = _sentinel(4, stride, cuda_dev)
        spec = buf[1:3]
        d_in = cz.stage_stream(x)
        cz.forward(d_in, 2, spec, first_block=1)
        other = _sentinel(2, stride, cuda_dev)
        lib.kgpu_use_static_kernels(0)
        try:
            cz.forward(d_in, 2, other, first_block=1)
        finally:
            lib.kgpu_use_static_kernels(1)
        torch.cuda.synchronize()
        got = spec.cpu().numpy()[:, :bins]
    finally:
        cz.close()
    raw = _bits(buf)
    assert (raw[0] == NAN_BITS).all() and (raw[3] == NAN_BITS).all(), "store outside the launched blocks' rows"
    assert (raw[1:3, 2 * bins:] == NAN_BITS).all(), "store into the row padding [bins, spec_stride)"
    assert np.isfinite(got).all(), "bin left unwritten"
    assert np.array_equal(raw[1:3], _bits(other)), "kgpu_use_static_kernels(0) changed an extended master's spectra"
    e_gpu, e_ora = [], []
    for j, b in enumerate((1, 2)):
        w = oracle.block_window(x, L, M, b)
        truth = np.fft.rfft(w.astype(np.float64)) if geo.real else np.fft.fft(w.astype(np.complex128))
        e_gpu.append(_err(got[j], truth))
        e_ora.append(_err(oracle.forward(w), truth))
    _score(f"extended forward {geo.id}", np.concatenate(e_gpu), np.concatenate(e_ora))


INGEST = [g for g in EXT_FORWARD if g.id in ("airspyhf_912k", "r153x135", "r152x138")]


@pytest.mark.parametrize("geo", INGEST, ids=lambda g: g.id)
def test_extended_int16_ingest_stats_and_derandomize(oracle, cuda_dev, geo):
    """fwd_cols_ext<1>: a 6-block int16 stream with clip values at every block's first and last new sample, 3 blocks
    launched from block 2.  Energy and clips are exact per block; derandomize + stats gives bitwise the spectra of the
    plain int16 path on a stream derandomized on the host, and that path is accurate bin by bin."""
    from ka9q_radio_b200 import capi

    specials = np.array([32767, -32767, -32768, 32766], np.int16)
    L, M, real = geo.L, geo.M, geo.real
    per = 1 if real else 2
    rng = np.random.default_rng(L)
    xi = rng.integers(-32768, 32768, 6 * L * per, dtype=np.int16)
    for b in range(6):
        for k, pos in enumerate((b * L, b * L + L - 1)):
            for c in range(per):
                xi[pos * per + c] = specials[(2 * b + k + c) % 4]
    scale = float(np.float32(10 ** (3 / 20) / 32768))
    cz = _cz(L, M, capi.KGPU_REAL if real else capi.KGPU_COMPLEX, cuda_dev)
    try:
        assert "kernels fwd_cols_ext + fwd_rows_ext" in cz.master.describe()
        bins = cz.master.bins
        for derand in (False, True):
            xd = _derandomize(xi) if derand else xi
            st = torch.zeros(3 * 2, dtype=torch.int64, device=cuda_dev)
            sp = cz.alloc_spectra(3)
            cz.forward(cz.stage_stream(xi), 3, sp, scale=scale, first_block=2, derandomize=derand, stats=st)
            plain = cz.alloc_spectra(3)
            cz.forward(cz.stage_stream(xd), 3, plain, scale=scale, first_block=2)
            torch.cuda.synchronize()
            stats = st.cpu().numpy().reshape(3, 2)
            for j in range(3):
                b = 2 + j
                want = _stats_of(xd[b * L * per:(b + 1) * L * per])
                assert (int(stats[j, 0]), int(stats[j, 1]) & 0xFFFFFFFF) == want, (geo.id, derand, j)
            assert np.array_equal(_bits(sp[:, :bins]), _bits(plain[:, :bins])), (geo.id, derand)
        xf = xd.astype(np.float32) * np.float32(scale)
        if not real:
            xf = (xf[0::2] + 1j * xf[1::2]).astype(np.complex64)
        got = plain.cpu().numpy()[:, :bins]
        e = []
        for j in range(3):
            w = oracle.block_window(xf, L, M, 2 + j)
            truth = np.fft.rfft(w.astype(np.float64)) if real else np.fft.fft(w.astype(np.complex128))
            e.append(_err(got[j], truth))
        assert np.concatenate(e).max() <= MAX_E
    finally:
        cz.close()


@pytest.mark.parametrize("geo", FORWARD, ids=lambda g: g.id)
def test_create_ex_is_create_on_7_smooth_lengths(cuda_dev, geo):
    """Same describe() and bitwise the same spectrum of one block."""
    from ka9q_radio_b200 import capi

    in_type = capi.KGPU_REAL if geo.real else capi.KGPU_COMPLEX
    x = torch.from_numpy(_stream(np.random.default_rng(geo.L), geo.L + geo.M - 1, geo.real)).to(cuda_dev)
    fmt = capi.KGPU_FMT_F32
    out = []
    for ext in (False, True):
        m = capi.Master(geo.L, geo.M, in_type, extended=ext)
        try:
            spec = torch.empty(m.spec_stride, dtype=torch.complex64, device=cuda_dev)
            m.forward(x.data_ptr(), fmt, 1.0, 1, spec.data_ptr(), torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            out.append((m.describe(), _bits(spec[:m.bins])))
        finally:
            m.close()
    assert out[0][0] == out[1][0]
    assert np.array_equal(out[0][1], out[1][1])


# ------------------------------------------------------------------ through filter.h ---------------------------
def _driver(name):
    from test_filter_abi import _load

    return _load(name)


HF = EXT_FORWARD[0]  # AirspyHF+ 912 kS/s
HF_N = HF.L + HF.M - 1


def _hf_stream(oracle, nb):
    rng = np.random.default_rng(912)
    n = np.arange(nb * HF.L)
    tone = 0.3 * np.exp(2j * np.pi * 0.0917 * n) + 0.1 * np.exp(-2j * np.pi * 0.3 * n)
    return (tone + 0.05 * (rng.standard_normal(len(n)) + 1j * rng.standard_normal(len(n)))).astype(np.complex64)


def _hf_channels():
    h = HF_N // 2
    chans = []
    for olen in (240, 480, 960):  # 12, 24 and 48 kHz
        pts = olen * HF_N // HF.L
        chans += [dict(olen=olen, shift=2091, low=-0.4, high=0.4, beta=11.0),
                  dict(olen=olen, shift=-6840, low=-0.4, high=0.4, beta=11.0),
                  dict(olen=olen, shift=h - pts // 4, low=-0.4, high=0.4, beta=11.0),      # slice wraps past N/2
                  dict(olen=olen, shift=-(h - pts // 5), low=-0.4, high=0.4, beta=11.0),
                  dict(olen=olen, shift=pts // 8, low=-0.45, high=0.1, beta=7.0)]           # slice wraps past DC
    chans += [dict(olen=480, shift=1500, low=-0.3, high=0.3, beta=9.0, isb=True),
              dict(olen=960, shift=-9000, low=0.01, high=0.35, beta=11.0, isb=True)]
    return chans


@pytest.mark.parametrize("driver", ["driver_gpuhdr.so", "driver_refhdr.so"])
def test_airspyhf_912k_through_filter_h(cuda_dev, driver):
    """create_filter_input(18240, 4561, COMPLEX) serves the master; 12, 24 and 48 kHz channels with positive, negative
    and wrapping shifts, ISB and the DC notch (plus one spur notch), five blocks, against the restated path and against
    the reference's own filter.c where it is built."""
    if _driver(driver) is None:
        pytest.skip(f"{driver} not built")
    _fresh("_case_912k_through_filter_h", driver, env={"KA9Q_GPU_SPECTRUM_D2H": "all"})


def _case_912k_through_filter_h(oracle, cuda_dev, driver):
    lib = _driver(driver)
    nb = 5
    x = _hf_stream(oracle, nb)
    chans = _hf_channels()
    got, gspec = oracle.ref_run_stream(x, HF.L, HF.M, chans, notch_bins=[4321], keep_spectra=True, lib=lib)
    ref, rspec = oracle.run_stream(x, HF.L, HF.M, chans, notch_bins=[4321], keep_spectra=True)
    refs = [("restated", ref, rspec)]
    if oracle.ref_available():
        refs.append(("filter.c", *oracle.ref_run_stream(x, HF.L, HF.M, chans, notch_bins=[4321], keep_spectra=True)))
    for what, r, rs in refs:
        for b in range(nb):
            assert np.abs(gspec[b] - rs[b]).max() / np.abs(rs[b]).max() < TOL, (what, b)
            for c in range(len(chans)):
                assert np.abs(got[b][c] - r[b][c]).max() / np.abs(r[b][c]).max() < TOL, (what, b, c)


def test_airspyhf_912k_tuned_output_and_noise_through_filter_h(cuda_dev):
    """execute_filter_output_tuned and filter_noise_estimate on the extended master, against the restated radio.c."""
    _fresh("_case_912k_tuned_and_noise")


def _case_912k_tuned_and_noise(oracle, cuda_dev):
    lib = _driver("driver_gpuhdr.so")
    L, M, N, fs = HF.L, HF.M, HF_N, 912e3
    nb = 6
    x = _hf_stream(oracle, nb)
    freqs = [[100_017.3, -212_234.5] for _ in range(nb)]
    for b in range(3, nb):
        freqs[b][0] = 103_350.6
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


def test_every_airspyhf_rate_is_accepted_by_create_filter_input(cuda_dev):
    """912, 768, 456, 384, 256 and 192 kS/s at 20 ms blocks and overlap 5: create_filter_input returns 0 and one
    24 kHz channel of one block matches the restated path."""
    _fresh("_case_every_airspyhf_rate")


def _case_every_airspyhf_rate(oracle, cuda_dev):
    lib = _driver("driver_gpuhdr.so")
    from ka9q_radio_b200 import capi

    for rate, L, M in AIRSPYHF_RATES:
        N = L + M - 1
        m = capi.Master(L, M, capi.KGPU_COMPLEX, extended=True)
        desc = m.describe()
        m.close()
        assert ("fwd_cols_ext" in desc) == any(N % p == 0 for p in NEW_PRIMES), (rate, desc)
        x = _hf_stream(oracle, 2)[: 2 * L]
        ch = [dict(olen=480, shift=N // 7, low=-0.4, high=0.4, beta=11.0)]
        got, _ = oracle.ref_run_stream(x, L, M, ch, lib=lib)  # RefSession raises if create_filter_input fails
        ref, _ = oracle.run_stream(x, L, M, ch)
        for b in range(2):
            assert np.abs(got[b][0] - ref[b][0]).max() / np.abs(ref[b][0]).max() < TOL, (rate, b)


# ------------------------------------------------------------------ plan registry isolation ----------------------
_ISOLATION_SCRIPT = r"""
import sys
import numpy as np
import torch
sys.path.insert(0, ".")
from ka9q_radio_b200 import capi

NEW = (11, 13, 17, 19, 23)

def smooth7(n):
    for p in (2, 3, 5, 7):
        while n % p == 0:
            n //= p
    return n == 1

def ext_len(n):
    try:
        capi.plan_radices(n, extended=True)
    except capi.KgpuError:
        return False
    return any(n % p == 0 for p in NEW)

# a COMPLEX master of N = l * l points splits as l x l: one distinct extended tile length per master
first = capi.Master(22800, 1, capi.KGPU_COMPLEX, extended=True)
lengths = [n for n in range(11, 4097) if ext_len(n)][:330]
for l in lengths:
    m = capi.Master(l * l, 1, capi.KGPU_COMPLEX, extended=True)
    assert f"two-pass {l} x {l};" in m.describe(), m.describe()
    m.close()
filler = capi.Bank(capi.Master(4096, 1, capi.KGPU_COMPLEX), 1)
seven = [n for n in range(2, 7261) if smooth7(n)]
for n in seven:
    assert filler.define(0, n) == n
late = capi.Master(1125000, 375001, capi.KGPU_COMPLEX)
late.close()
# the first extended master still transforms correctly
x = (np.random.default_rng(1).standard_normal(22800) + 1j * np.random.default_rng(2).standard_normal(22800)).astype(np.complex64)
d = torch.from_numpy(x).cuda()
spec = torch.empty(first.spec_stride, dtype=torch.complex64, device="cuda")
first.forward(d.data_ptr(), capi.KGPU_FMT_F32, 1.0, 1, spec.data_ptr())
torch.cuda.synchronize()
truth = np.fft.fft(x.astype(np.complex128))
e = np.abs(spec.cpu().numpy()[:22800] - truth).max() / np.sqrt(np.mean(np.abs(truth) ** 2))
assert e < 5e-6, e
first.close()
print("isolation ok,", len(set(lengths)), "extended lengths,", len(seven), "channel lengths")
"""


def test_extended_plans_stay_out_of_the_registry(cuda_dev):
    """In a fresh process: masters covering 330 distinct extended tile lengths are created and destroyed, then every
    7-smooth channel length from 2 to 7260 is defined and one more 7-smooth master is created.  All succeed, and an
    extended master created first still computes its transform."""
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _ISOLATION_SCRIPT]
    r = subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "isolation ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
