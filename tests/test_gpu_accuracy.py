"""Bin-by-bin accuracy of every forward and channel kernel path against float64 transforms, and where the kernels write.

Metric: e[k] = |gpu[k] - truth[k]| / rms(truth), on flat-spectrum inputs (white noise, flat random spectra), so the
normalisation is effectively per bin: a wrong low-energy region or a twiddle wrong in its fifth digit shows up, which
the parity tests' max|gpu - ref| / max|ref| on tone-dominated inputs cannot see.  `truth` is a float64 transform of
exactly the float32 values the kernel saw; the float32 oracle is scored against the same truth.
Bounds: max e <= 5e-6 everywhere; with >= 4096 values, rms(e_gpu) <= 2 rms(e_oracle) and max(e_gpu) <= 4 max(e_oracle).

Every spectrum and output buffer is pre-filled with a NaN pattern, and the guard rows and row padding must come back
bitwise unchanged: padding is never written, and a store past `bins`, into the next block's row or between two
channels' outputs fails here even when it overwrites nothing that is compared.
"""
import numpy as np
import pytest
import torch

from accuracy_cases import CHANNELS, FORWARD, Fwd

pytestmark = pytest.mark.gpu

MAX_E = 5e-6
NAN_BITS = 0x7FC0DEAD  # a quiet NaN no kernel computes


def _mk(L, M, in_type, dev, cap=64):
    from ka9q_radio_b200.channelizer import Channelizer

    return Channelizer(L, M, in_type, dev, capacity=cap)


def _sentinel(rows, cols, dev):
    """complex64 [rows, cols] whose every float holds NAN_BITS"""
    return torch.full((rows, 2 * cols), NAN_BITS, dtype=torch.int32, device=dev).view(torch.float32).view(torch.complex64)


def _bits(t):
    return t.view(torch.float32).view(torch.int32).cpu().numpy()


def _err(got, truth):
    return np.abs(np.asarray(got, np.complex128) - truth) / np.sqrt(np.mean(np.abs(truth) ** 2))


def _score(what, e_gpu, e_ora):
    """the bounds of the module docstring; prints the measured values (pytest -s)"""
    r_rms = np.sqrt(np.mean(e_gpu ** 2)) / np.sqrt(np.mean(e_ora ** 2))
    r_max = e_gpu.max() / e_ora.max()
    print(f"accuracy {what}: max e {e_gpu.max():.2e} (oracle {e_ora.max():.2e}), gpu/oracle rms {r_rms:.2f} max {r_max:.2f}")
    assert e_gpu.max() <= MAX_E, (what, e_gpu.max())
    if e_gpu.size >= 4096:
        assert r_rms <= 2.0, (what, r_rms)
        assert r_max <= 4.0, (what, r_max)


# ------------------------------------------------------------------ A + B: forward sweep ------------
def _forward_params():
    for f in FORWARD:
        yield pytest.param(f, 1, id=f"{f.id}-static1")
        if f.specialised:
            yield pytest.param(f, 0, id=f"{f.id}-static0")


@pytest.mark.parametrize("geo,static", list(_forward_params()))
def test_forward_per_bin_accuracy_and_writes(oracle, cuda_dev, geo: Fwd, static):
    """White Gaussian input, three blocks; blocks 1 and 2 in one launch (history and new samples both nonzero)."""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    in_type = capi.KGPU_REAL if geo.real else capi.KGPU_COMPLEX
    L, M = geo.L, geo.M
    rng = np.random.default_rng(geo.L + geo.M)
    if geo.real:
        x = rng.standard_normal(3 * L, dtype=np.float32)
    else:
        x = (rng.standard_normal(3 * L, dtype=np.float32) + 1j * rng.standard_normal(3 * L, dtype=np.float32)).astype(np.complex64)
    cz = _mk(L, M, in_type, cuda_dev, cap=1)
    try:
        n1, n2 = geo.split
        cols, rows = (",".join(map(str, r)) for r in geo.kernels)
        desc = cz.master.describe()
        assert f"two-pass {n1} x {n2}; cols radices [{cols}] rows radices [{rows}]" in desc
        assert desc.endswith(f"kernels {geo.pair[0]} + {geo.pair[1]}"), desc
        bins, stride = cz.master.bins, cz.master.spec_stride
        buf = _sentinel(4, stride, cuda_dev)
        spec = buf[1:3]
        lib.kgpu_use_static_kernels(static)
        try:
            cz.forward(cz.stage_stream(x), 2, spec, first_block=1)
        finally:
            lib.kgpu_use_static_kernels(1)
        torch.cuda.synchronize()
        got = spec.cpu().numpy()[:, :bins]
        cz.master.set_notches([bins - 1])
        cz.apply_notches(spec, 2)
        torch.cuda.synchronize()
    finally:
        cz.close()
    raw = _bits(buf)
    assert (raw[0] == NAN_BITS).all() and (raw[3] == NAN_BITS).all(), "store outside the launched blocks' rows"
    assert (raw[1:3, 2 * bins:] == NAN_BITS).all(), "store into the row padding [bins, spec_stride)"
    assert np.isfinite(buf[1:3, :bins].cpu().numpy()).all(), "bin left unwritten"
    e_gpu, e_ora = [], []
    for j, b in enumerate((1, 2)):
        w = oracle.block_window(x, L, M, b)
        truth = np.fft.rfft(w.astype(np.float64)) if geo.real else np.fft.fft(w.astype(np.complex128))
        e_gpu.append(_err(got[j], truth))
        e_ora.append(_err(oracle.forward(w), truth))
    _score(f"forward {geo.id} static={static}", np.concatenate(e_gpu), np.concatenate(e_ora))


# ------------------------------------------------------------------ C: int16 ingest on every column kernel --
INGEST = [  # (id, real, L, M, describe() substring of the split, column kernel)
    ("generic", True, 48000, 12001, "200 x 150; cols radices [20,10]", "fwd_cols_kernel"),
    ("r36_1250", True, 2592000, 648001, "1296 x 1250; cols radices [36,36]", "fwd_cols_r36"),
    ("r36_0", True, 2519424, 629857, "1296 x 1215; cols radices [36,36]", "fwd_cols_r36"),
    ("cols_2s", False, 400000, 100001, "800 x 625; cols radices [25,32]", "fwd_cols_2s"),
]
SPECIALS = np.array([32767, -32767, -32768, 32766], np.int16)  # 32766 is not a clip


def _derandomize(v):
    """rx888.c:707-712: lsb set -> flip bits 1..15"""
    return (v ^ np.where(v & 1, np.int16(-2), np.int16(0))).astype(np.int16)


def _stats_of(v):
    w = v.astype(np.int64)
    return int((w * w).sum()), int(((w > 32766) | (w < -32766)).sum())


@pytest.mark.parametrize("case", INGEST, ids=[c[0] for c in INGEST])
def test_int16_ingest_stats_and_derandomize(oracle, cuda_dev, case):
    """A 6-block int16 stream, 3 blocks launched from block 2, with clip values at the first and last new sample of every
    block (so also at every launched block's last history sample).  Energy and clip count are exact per block and the
    same on the specialised and the generic kernels; the derandomize + stats instantiation gives bitwise the spectra of
    the plain int16 one on a stream derandomized on the host."""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    name, real, L, M, desc, kernel = case
    per = 1 if real else 2  # int16 values per sample
    rng = np.random.default_rng(L)
    xi = rng.integers(-32768, 32768, 6 * L * per, dtype=np.int16)
    for b in range(6):
        for k, pos in enumerate((b * L, b * L + L - 1)):
            for c in range(per):
                xi[pos * per + c] = SPECIALS[(2 * b + k + c) % 4]
    scale = float(np.float32(10 ** (3 / 20) / 32768))
    cz = _mk(L, M, capi.KGPU_REAL if real else capi.KGPU_COMPLEX, cuda_dev, cap=1)
    try:
        assert desc in cz.master.describe() and f"kernels {kernel} + " in cz.master.describe()
        bins = cz.master.bins
        for derand in (False, True):
            xd = _derandomize(xi) if derand else xi
            stats = {}
            spec = {}
            for static in (1, 0):
                st = torch.zeros(3 * 2, dtype=torch.int64, device=cuda_dev)
                sp = cz.alloc_spectra(3)
                lib.kgpu_use_static_kernels(static)
                try:
                    cz.forward(cz.stage_stream(xi), 3, sp, scale=scale, first_block=2, derandomize=derand, stats=st)
                finally:
                    lib.kgpu_use_static_kernels(1)
                torch.cuda.synchronize()
                stats[static] = st.cpu().numpy().reshape(3, 2)
                spec[static] = sp
            plain = cz.alloc_spectra(3)
            cz.forward(cz.stage_stream(xd), 3, plain, scale=scale, first_block=2)
            torch.cuda.synchronize()
            for j in range(3):
                b = 2 + j
                new = xd[b * L * per:(b + 1) * L * per]
                want = _stats_of(new)
                if real:
                    assert oracle.convert_i16(xi[b * L:(b + 1) * L], np.float32(scale), derand)[1:] == want
                got = (int(stats[1][j, 0]), int(stats[1][j, 1]) & 0xFFFFFFFF)
                assert got == want, (name, derand, j, got, want)
            assert (stats[1] == stats[0]).all(), (name, derand)
            assert np.array_equal(_bits(spec[1][:, :bins]), _bits(plain[:, :bins])), (name, derand)
        # the plain int16 path itself, bin by bin against float64 (the scale rides on the specialised kernels' twiddles)
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


# ------------------------------------------------------------------ D: channel inverse sweep -----------
BEAM_W = (0.6 - 0.2j, 0.3 + 0.7j)


def _shifts(N, ns, rng):
    h = N // 2
    return sorted({0, 1, -1, h - 1, -(h - 1), h - ns // 4 - 1, -(h - ns // 4 - 1), ns // 4 + 1, -(ns // 4 + 1),
                   int(rng.integers(-h + 1, h)), int(rng.integers(-h + 1, h))})


def _slice(oracle, in_type, X, ns, shift):
    """the exact input of the inverse transform with an all-ones response: zeros, conjugates and wrap included"""
    return oracle.slice_multiply(in_type, X, np.ones(ns, np.complex64), shift).astype(np.complex128)


def _isb(S):
    S = S.copy()
    ns = len(S)
    for p in range(1, ns // 2):
        pos, neg = S[p], S[ns - p]
        S[p], S[ns - p] = pos + np.conj(neg), neg - np.conj(pos)
    S[0] = 0
    return S


def _beam_slice(oracle, X, ns, shift):
    """filter.c:756-775 in float64: alpha X[q] + beta conj X[m-q], at q = 0 and m/2 Re(X) alpha + Im(X) beta; the slot ->
    q map comes from slicing a spectrum that holds its own indices"""
    m = len(X)
    idx = _slice(oracle, 1, (np.arange(m) + 1).astype(np.complex64), ns, shift).real.astype(np.int64) - 1
    live = idx >= 0
    q = np.where(live, idx, 0)
    a = 0.5 * complex(BEAM_W[0]) - 1j * complex(BEAM_W[1])
    b = 0.5 * complex(BEAM_W[0]) + 1j * complex(BEAM_W[1])
    X = X.astype(np.complex128)
    v = a * X[q] + b * np.conj(X[(m - q) % m])
    edge = (q == 0) | (q == m // 2)
    v[edge] = X[q[edge]].real * a + X[q[edge]].imag * b
    return np.where(live, v, 0)


def _chan_params():
    for c in CHANNELS:
        for static in (1, 0):
            yield pytest.param(c, static, id=f"{c.id}-static{static}")


@pytest.mark.parametrize("case,static", list(_chan_params()))
def test_channel_inverse_per_sample_accuracy_and_writes(oracle, cuda_dev, case, static):
    """A flat random spectrum through every channel length and shift class, random responses; every output sample
    against ifft(slice * R) in float64, every channel also against the oracle's semantics at 1e-5 of rms."""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    in_type = capi.KGPU_REAL if case.real else capi.KGPU_COMPLEX
    L, M = case.L, case.M
    N = L + M - 1
    rng = np.random.default_rng(N + 7 * len(case.points))
    chans = []  # (points, shift, kind)
    for ns in case.points:
        chans += [(ns, s, "plain") for s in _shifts(N, ns, rng)]
    for ns in case.real_out:
        chans += [(ns, s, "real") for s in _shifts(N, ns, rng)]
    odd = [ns for ns in case.points if ns % 2][:1] + [ns for ns in case.points if ns >= 4096][-1:]
    for ns in odd:
        s = int(rng.integers(-(N // 2) + 1, N // 2))
        chans += [(ns, s, "isb"), (ns, N // 2 - ns // 4 - 1, "isb")]
        if not case.real:
            chans += [(ns, s, "beam"), (ns, -(N // 2) + ns // 4 + 1, "beam")]
    cz = _mk(L, M, in_type, cuda_dev, cap=len(chans))
    try:
        resp = []
        for ns, s, kind in chans:
            R = (rng.standard_normal(ns) + 1j * rng.standard_normal(ns)).astype(np.complex64)
            resp.append(R)
            cz.add_channel(ns * L // N, s, response=R, isb=kind == "isb", beam=BEAM_W if kind == "beam" else None,
                           out_type=capi.KGPU_REAL if kind == "real" else capi.KGPU_COMPLEX)
        bins, nb = cz.master.bins, 2
        X = (rng.standard_normal((nb, bins)) + 1j * rng.standard_normal((nb, bins))).astype(np.complex64)
        spec = _sentinel(nb, cz.master.spec_stride, cuda_dev)  # the row padding stays NaN: reading it would show
        spec[:, :bins] = torch.from_numpy(X).to(cuda_dev)
        out = _sentinel(nb, max(cz.bank.out_stride, 1), cuda_dev)
        lib.kgpu_use_static_kernels(static)
        try:
            cz.channels(spec, nb, out)
        finally:
            lib.kgpu_use_static_kernels(1)
        torch.cuda.synchronize()
        raw = _bits(out)
        written = np.zeros(raw.shape[1], bool)
        e_gpu, e_ora = [], []
        for i, ((ns, s, kind), R) in enumerate(zip(chans, resp)):
            olen = ns * L // N
            off = cz.bank.out_offset(i)
            written[2 * off:2 * off + (olen if kind == "real" else 2 * olen)] = True
            got = cz.channel_slice(out, i).cpu().numpy()
            for b in range(nb):
                if kind == "real":
                    sb = ns // 2 + 1
                    mi = np.arange(sb) + s
                    ok = (mi >= 0) & (mi < bins)
                    V = np.where(ok, X[b][np.clip(mi, 0, bins - 1)].astype(np.complex128), 0) * R[:sb]
                    V[(sb + 1) // 2] = 0
                    truth = (np.fft.irfft(V, ns) * ns)[-olen:]
                    ora = oracle.channel_block_realout(in_type, X[b], R, s)[-olen:]
                else:
                    S = _beam_slice(oracle, X[b], ns, s) if kind == "beam" else _slice(oracle, in_type, X[b], ns, s)
                    S = S * R.astype(np.complex128)
                    if kind == "isb":
                        S = _isb(S)
                    truth = (np.fft.ifft(S) * ns)[-olen:]
                    if kind == "beam":
                        ora = oracle.channel_block_beam(X[b], R, s, *BEAM_W)[-olen:]
                    else:
                        ora = oracle.channel_block(in_type, X[b], R, s, isb=kind == "isb")[-olen:]
                what = (case.id, ns, s, kind, b)
                if not np.any(truth):
                    assert not np.any(got[b]) and not np.any(ora), what  # nothing of the master in the slice
                    continue
                eg, eo = _err(got[b], truth), _err(ora, truth)
                assert eg.max() <= MAX_E, (what, eg.max())
                assert np.abs(got[b] - ora).max() / np.sqrt(np.mean(np.abs(truth) ** 2)) <= 1e-5, what
                e_gpu.append(eg)
                e_ora.append(eo)
        assert (raw[:, ~written] == NAN_BITS).all(), "store outside a channel's output run"
        _score(f"channels {case.id} static={static}", np.concatenate(e_gpu), np.concatenate(e_ora))
    finally:
        cz.close()


def test_channel_lengths_rejected_at_define(cuda_dev):
    from ka9q_radio_b200 import capi

    cz = _mk(7000, 1001, capi.KGPU_COMPLEX, cuda_dev, cap=2)  # N / L = 8 / 7
    try:
        with pytest.raises(capi.KgpuError, match="8192-point inverse transform exceeds the 7260-point maximum"):
            cz.bank.define(0, 7168)
        with pytest.raises(capi.KgpuError, match="kgpu_bank_define: 88-point transform cannot be planned"):
            cz.bank.define(1, 77)  # 88 = 8 * 11
    finally:
        cz.close()


# ------------------------------------------------------------------ plan registry ---------------------
_REGISTRY_SCRIPT = r"""
import sys
import numpy as np
import torch
sys.path.insert(0, ".")
from ka9q_radio_b200 import capi
from ka9q_radio_b200.channelizer import Channelizer
from oracle import oracle as O

lib = capi.load()
L, M, nb = 4800, 1201, 2
x = O.siggen_real(nb * L, 0.1, 0.02, 0.123, 1.0)
ch = dict(olen=480, shift=700, low=-0.3, high=0.35, beta=11.0)
cz = Channelizer(L, M, capi.KGPU_REAL, "cuda:0", capacity=1)
cz.add_channel(ch["olen"], ch["shift"], ch["low"], ch["high"], ch["beta"])
ref, _ = O.run_stream(x, L, M, [ch])

def check():
    spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
    cz.forward(cz.stage_stream(x), nb, spec)
    cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    got = cz.channel_slice(out, 0).cpu().numpy()
    for b in range(nb):
        assert np.abs(got[b] - ref[b][0]).max() / np.abs(ref[b][0]).max() < 1e-5

def plannable(n):
    for p in (2, 3, 5, 7):
        while n % p == 0:
            n //= p
    return n == 1

check()
# N == L: a slave's point count equals its output length, so a channel can ask for any length
filler = capi.Bank(capi.Master(4096, 1, capi.KGPU_COMPLEX), 1)
lengths = [n for n in range(2, 7261) if plannable(n)]
for n in lengths:
    assert filler.define(0, n) == n
late = Channelizer(1125000, 375001, capi.KGPU_COMPLEX, "cuda:0", capacity=1)  # 1250 x 1200, after every length is taken
late.close()
check()
cz.close()
print("registry ok,", len(lengths), "lengths")
"""


def test_plan_registry_holds_every_length(cuda_dev):
    """The registry is process-wide and never frees a plan, so this runs in a fresh process: after a master and a bank
    are created, every length a master or channel can ask for (2..7260, factors 2, 3, 5, 7) is registered, one more
    master is created, and the first master and bank still run and still match the oracle."""
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parent.parent
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _REGISTRY_SCRIPT]
    r = subprocess.run(args, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "registry ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
