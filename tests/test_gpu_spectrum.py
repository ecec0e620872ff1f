"""The device wideband spectrum analyzer (kgpu_spectrum_*, filter_spectrum_*; wideband_poll, reference spectrum.c:308-522):
accuracy against a float64 truth of exactly the float32 windowed samples, every bin-mapping edge against the oracle
restatement, int16 rings, polls longer than the scratch, and the filter.h path with its device ring."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from ka9q_radio_b200 import capi
from oracle import spectrum as S

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
REAL, COMPLEX = capi.KGPU_REAL, capi.KGPU_COMPLEX


def kaiser_window(n, beta=11.0):
    w = np.kaiser(n + 1, beta)[:n]
    return (w / w.sum()).astype(np.float32)


def sources(is_real, fft_n, bin_count, shift):
    """source bin of every output bin as the reference maps it, -1 where it adds nothing (or reads below its array)"""
    i = np.arange(bin_count)
    half = bin_count // 2
    if is_real:
        b0, top = (shift if shift >= 0 else fft_n // 2 + shift), fft_n // 2 + 1
        lo = np.where((b0 + i < top) & (b0 + i >= 0), b0 + i, -1)
        hi = np.where(b0 + half < top, b0 + i - bin_count, -1)
        src = np.where(i < half, lo, hi)
        return np.where(src >= 0, src, -1)
    b = shift + np.where(i < half, i, i - bin_count)
    ok = (b >= -(fft_n // 2)) & (b < (fft_n + 1) // 2)
    return np.where(ok, np.where(b >= 0, b, b + fft_n), -1)


def segments(is_real, fft_n, fft_avg, overlap, cap, end):
    adjust = int(np.rint(fft_n * (1 + (fft_avg - 1) * (1 - overlap))))
    hop = int(np.rint(fft_n * (1.0 - overlap)))
    step = hop if is_real else -hop
    return [((end - adjust + s * step) % cap + np.arange(fft_n)) % cap for s in range(fft_avg)]


def truth(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end):
    """float64 transforms of the float32 windowed segments, accumulated in float64"""
    src = sources(is_real, fft_n, bin_count, shift)
    gain = (2.0 if is_real else 1.0) / (fft_avg * fft_n * fft_n)
    acc = np.zeros(bin_count)
    for idx in segments(is_real, fft_n, fft_avg, overlap, len(ring), end):
        x = window * ring[idx]  # float32 / complex64 product, as the kernel forms it
        if is_real and shift < 0:
            x = x.copy()
            x[1::2] = -x[1::2]
            if fft_n & 1:
                x[-1] = 0
        X = np.fft.fft(x.astype(np.complex128))
        acc[src >= 0] += gain * np.abs(X[src[src >= 0]]) ** 2
    return acc


def make_ring(is_real, cap, rng, tones=()):
    n = np.arange(cap)
    if is_real:
        x = rng.standard_normal(cap)
        for f, a in tones:
            x += a * np.cos(2 * np.pi * f * n)
        return x.astype(np.float32)
    x = (rng.standard_normal(cap) + 1j * rng.standard_normal(cap)) / np.sqrt(2)
    for f, a in tones:
        x += a * np.exp(2j * np.pi * f * n)
    return x.astype(np.complex64)


def to_dev(ring):
    if np.iscomplexobj(ring):
        ring = ring.view(np.float32).reshape(-1, 2)
    return torch.from_numpy(np.ascontiguousarray(ring)).cuda()


def gpu_poll(sp, ring_dev, end, shift, fft_avg, overlap, bin_count, **kw):
    bins = torch.full((bin_count + 64,), float("nan"), device="cuda")
    sp.run(ring_dev, end, shift, fft_avg, overlap, bins, **kw)
    torch.cuda.synchronize()
    out = bins.cpu().numpy()
    assert np.isnan(out[bin_count:]).all(), "wrote past bin_count"
    return out[:bin_count]


# ------------------------------------------------------------------------------------------ 1. accuracy
ACCURACY = [6480, 22800, 129600, 518400, 6075, 7005, 104400]


@pytest.mark.parametrize("is_real", [True, False], ids=["real", "complex"])
@pytest.mark.parametrize("fft_n", ACCURACY)
def test_accuracy_against_float64_truth(is_real, fft_n):
    rng = np.random.default_rng(fft_n + is_real)
    bin_count = fft_n // 2 if is_real else fft_n
    shift = bin_count // 2 if is_real else 0
    fft_avg, overlap = 2, 0.5
    cap = 2 * fft_n + 1234
    ring = make_ring(is_real, cap, rng)
    window = kaiser_window(fft_n)
    end = 777  # the segments cross the ring end
    sp = capi.Spectrum(fft_n, REAL if is_real else COMPLEX, bin_count)
    sp.set_window(window)
    got = gpu_poll(sp, to_dev(ring), end, shift, fft_avg, overlap, bin_count)
    t = truth(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end)
    orc = S.wideband_spectrum(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end)
    m = sources(is_real, fft_n, bin_count, shift) >= 0
    scale = t[m].mean()
    e_gpu, e_orc = np.abs(got[m] - t[m]) / scale, np.abs(orc[m] - t[m]) / scale
    rms_g, rms_o = np.sqrt((e_gpu ** 2).mean()), np.sqrt((e_orc ** 2).mean())
    print(f"\n{sp.describe()}: gpu max {e_gpu.max():.2e} rms {rms_g:.2e} | float32 oracle max {e_orc.max():.2e} "
          f"rms {rms_o:.2e}")
    assert (got[~m] == 0).all()
    assert e_gpu.max() <= 1e-5
    assert rms_g <= 2 * rms_o and e_gpu.max() <= 4 * e_orc.max()
    sp.close()


# ------------------------------------------------------------------------------------------ 2. mapping edges
def check_against_oracle(is_real, fft_n, bin_count, shift, fft_avg, overlap, cap, end, tones=(), seed=1):
    rng = np.random.default_rng(seed)
    ring = make_ring(is_real, cap, rng, tones)
    window = kaiser_window(fft_n)
    sp = capi.Spectrum(fft_n, REAL if is_real else COMPLEX, bin_count)
    sp.set_window(window)
    got = gpu_poll(sp, to_dev(ring), end, shift, fft_avg, overlap, bin_count)
    sp.close()
    ref = S.wideband_spectrum(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end)
    zero = sources(is_real, fft_n, bin_count, shift) < 0
    assert (got[zero] == 0).all() and (ref[zero] == 0).all()
    tol = 1e-5 * max(ref.max(), 1e-30) + 1e-12 * ref.max()
    np.testing.assert_allclose(got, ref, rtol=0, atol=tol)
    return got


EDGES = [  # (is_real, fft_n, bin_count, shift, fft_avg, overlap)
    (True, 6480, 1000, 2900, 3, 0.5),     # REAL walk stops at fft_n/2+1
    (True, 6480, 1000, 1500, 2, 0.0),     # bin_count/2 step back onto lower bins
    (True, 6480, 1000, 100, 2, 0.25),     # step back below 0: the reference's out-of-bounds read gives 0 here
    (True, 6480, 1001, -700, 4, 0.5),     # shift < 0: sign flip
    (True, 6075, 999, -800, 3, 0.3333),   # odd fft_n, shift < 0: the last sample zeroed; odd bin_count
    (True, 7005, 1201, -900, 2, 0.5),     # Bluestein REAL with the flip
    (False, 6480, 2000, 3000, 3, 0.5),    # COMPLEX bins above coverage stay 0
    (False, 6480, 2001, -3000, 3, 0.5),   # ... and below, odd bin_count
    (False, 6075, 6075, 0, 2, 0.9),       # odd COMPLEX length, all bins
    (False, 7005, 3001, -2000, 5, 0.3333),  # Bluestein COMPLEX
]


@pytest.mark.parametrize("is_real,fft_n,bin_count,shift,fft_avg,overlap", EDGES)
def test_mapping_edges_against_oracle(is_real, fft_n, bin_count, shift, fft_avg, overlap):
    cap = 3 * fft_n + 101
    tones = [(0.123, 3.0), (0.377 if is_real else -0.301, 1.0)]
    check_against_oracle(is_real, fft_n, bin_count, shift, fft_avg, overlap, cap, end=fft_n // 3, tones=tones)


def test_complex_backward_reads_wrap_past_adjust():
    # COMPLEX segments walk backwards from end - adjust: with end small they reach around the ring's end
    fft_n, fft_avg, overlap = 6480, 6, 0.5
    check_against_oracle(False, fft_n, 4000, 500, fft_avg, overlap, cap=4 * fft_n, end=fft_n, tones=[(0.05, 2.0)])


# ------------------------------------------------------------------------------------------ 3. int16 rings
@pytest.mark.parametrize("is_real", [True, False], ids=["real", "complex"])
@pytest.mark.parametrize("derandomize", [False, True])
@pytest.mark.parametrize("fft_n", [6480, 7005])
def test_int16_ring_is_bitwise_the_float_ring(is_real, derandomize, fft_n):
    rng = np.random.default_rng(5)
    cap = 3 * fft_n + 11
    words = rng.integers(-30000, 30000, size=cap * (1 if is_real else 2)).astype(np.int16)
    scale = np.float32(1.0 / 32768)
    v = words.copy()
    if derandomize:
        v = np.where(v & 1, v ^ np.int16(-2), v).astype(np.int16)  # lsb set -> flip bits 1..15
    fl = v.astype(np.float32) * scale
    bin_count, shift = 2000, -300
    sp = capi.Spectrum(fft_n, REAL if is_real else COMPLEX, bin_count)
    sp.set_window(kaiser_window(fft_n))
    i16 = torch.from_numpy(words if is_real else words.reshape(-1, 2)).cuda()
    f32 = torch.from_numpy(fl if is_real else fl.reshape(-1, 2)).cuda()
    a = gpu_poll(sp, i16, 100, shift, 4, 0.5, bin_count, scale=float(scale), derandomize=derandomize)
    b = gpu_poll(sp, f32, 100, shift, 4, 0.5, bin_count)
    sp.close()
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------------------------------ 4. chunks
def test_poll_above_the_scratch_cap_runs_in_chunks():
    fft_n, overlap = 518400, 0.9
    cap = 6 * fft_n
    fft_avg = int(np.floor(1 + (cap // fft_n - 1) / (1 - overlap)))  # spectrum.c:359 with this ring: 51 segments
    check_against_oracle(True, fft_n, 20000, 10000, fft_avg, overlap, cap, end=12345, tones=[(0.0101, 1.0)])


# ------------------------------------------------------------------------------------------ 5. filter.h
_drv = None


def drv():
    global _drv
    if _drv is None:
        d = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "spectrum_driver.so"))
        d.sd_ring_samples.restype = C.c_long
        d.sd_write_float.argtypes = [C.c_void_p, C.c_int]
        d.sd_write_i16.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int]
        d.sd_setup.argtypes = [C.c_int, C.c_int, C.c_void_p]
        d.sd_poll.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
        d.sd_producer_start.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float]
        _drv = d
    return _drv


def restated_ring(stream, M, cap, end_sample):
    """the float ring spectrum.c reasons about once end_sample samples have been written: stream sample s sits at position
    M - 1 + s (mod cap), the positions before the stream hold zeros"""
    ring = np.zeros(cap, stream.dtype)
    q1 = M - 1 + end_sample
    q = np.arange(max(0, q1 - cap), q1)
    keep = q >= M - 1
    ring[q[keep] % cap] = stream[q[keep] - (M - 1)]
    return ring, q1 % cap


class Fh:
    def __init__(self, L, M, is_real):
        self.d = drv()
        assert self.d.sd_open(L, M, 0 if is_real else 1) == 0
        self.L, self.M, self.is_real = L, M, is_real
        self.cap = self.d.sd_ring_samples()

    def poll(self, shift, fft_avg, overlap, bin_count):
        bins = np.full(bin_count, np.nan, np.float32)
        end = C.c_uint64(0)
        assert self.d.sd_poll(shift, fft_avg, overlap, bins.ctypes.data, C.cast(C.pointer(end), C.c_void_p)) == 0
        return bins, end.value

    def close(self):
        self.d.sd_close()


def expect(fh, stream, end, fft_n, bin_count, window, shift, fft_avg, overlap):
    ring, pos = restated_ring(stream, fh.M, fh.cap, end)
    return S.wideband_spectrum(fh.is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, pos), ring, pos


def close_to(got, ref):
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-5 * ref.max() + 1e-30)


L_FH, M_FH = 20000, 4001


def test_filter_h_real_int16_master():
    fft_n, bin_count, shift, fft_avg, overlap = 6480, 1620, 810, 5, 0.5
    fh = Fh(L_FH, M_FH, True)
    window = kaiser_window(fft_n)
    assert fh.d.sd_setup(fft_n, bin_count, window.ctypes.data) == 0
    rng = np.random.default_rng(11)
    words = rng.integers(-2000, 2000, size=8 * L_FH).astype(np.int16)
    scale = np.float32(1 / 2048)
    stream = words.astype(np.float32) * scale
    for j in range(8):
        assert fh.d.sd_write_i16(words[j * L_FH:].ctypes.data, L_FH, float(scale), 0) == 1
        got, end = fh.poll(shift, fft_avg, overlap, bin_count)
        assert end == (j + 1) * L_FH
        close_to(got, expect(fh, stream, end, fft_n, bin_count, window, shift, fft_avg, overlap)[0])
    fh.close()


@pytest.mark.parametrize("is_real", [True, False], ids=["real", "complex"])
def test_filter_h_float_master_and_the_reference(is_real):
    fft_n, bin_count, fft_avg, overlap = 6480, 3000, 4, 0.5
    shift = -900 if is_real else 1200
    fh = Fh(L_FH, M_FH, is_real)
    window = kaiser_window(fft_n)
    rng = np.random.default_rng(12)
    stream = make_ring(is_real, 6 * L_FH, rng, [(0.1, 1.0)])
    assert fh.d.sd_write_float(stream.ctypes.data, L_FH) == 1
    assert fh.d.sd_setup(fft_n, bin_count, window.ctypes.data) == 0
    for j in range(1, 6):
        assert fh.d.sd_write_float(stream[j * L_FH:].ctypes.data, L_FH) == 1
        got, end = fh.poll(shift, fft_avg, overlap, bin_count)
        assert end == (j + 1) * L_FH
        ref, ring, pos = expect(fh, stream, end, fft_n, bin_count, window, shift, fft_avg, overlap)
        close_to(got, ref)
        if S.have_ref():
            own, used = S.ref_wideband_poll(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, pos)
            assert used == fft_avg
            close_to(got, own)
    fh.close()


def test_filter_h_setup_after_the_ring_has_wrapped():
    fft_n, bin_count, shift, overlap = 6480, 3240, 1620, 0.5
    fh = Fh(L_FH, M_FH, True)
    fft_avg = int(np.floor(1 + (fh.cap // fft_n - 1) / (1 - overlap)))  # the clamp: the whole ring
    rng = np.random.default_rng(13)
    blocks = fh.cap // L_FH + 3
    stream = make_ring(True, blocks * L_FH, rng)
    for j in range(blocks):
        fh.d.sd_write_float(stream[j * L_FH:].ctypes.data, L_FH)
    window = kaiser_window(fft_n)
    assert fh.d.sd_setup(fft_n, bin_count, window.ctypes.data) == 0
    got, end = fh.poll(shift, fft_avg, overlap, bin_count)
    assert end == blocks * L_FH
    close_to(got, expect(fh, stream, end, fft_n, bin_count, window, shift, fft_avg, overlap)[0])
    fh.close()


def test_filter_h_polls_beside_a_producer_thread():
    fft_n, bin_count, shift, fft_avg, overlap = 6480, 3240, 1620, 6, 0.5
    fh = Fh(L_FH, M_FH, True)
    window = kaiser_window(fft_n)
    assert fh.d.sd_setup(fft_n, bin_count, window.ctypes.data) == 0
    nblocks = 200
    stream = make_ring(True, nblocks * L_FH, np.random.default_rng(14))
    assert fh.d.sd_producer_start(stream.ctypes.data, L_FH, nblocks, 0, 1.0) == 0
    seen = []
    while len(seen) < 40:
        got, end = fh.poll(shift, fft_avg, overlap, bin_count)
        seen.append((got, end))
        if end == nblocks * L_FH:
            break
    fh.d.sd_producer_join()
    for got, end in seen:
        assert end % L_FH == 0
        close_to(got, expect(fh, stream, end, fft_n, bin_count, window, shift, fft_avg, overlap)[0])
    fh.close()


@pytest.mark.parametrize("with_spectrum", [False, True])
def test_filter_h_launches_per_block(with_spectrum):
    lib = capi.load()
    fh = Fh(L_FH, M_FH, True)
    window = kaiser_window(6480)
    if with_spectrum:
        assert fh.d.sd_setup(6480, 1000, window.ctypes.data) == 0
    x = np.zeros(L_FH, np.float32)
    fh.d.sd_write_float(x.ctypes.data, L_FH)
    before = lib.kgpu_launch_count()
    for _ in range(4):
        fh.d.sd_write_float(x.ctypes.data, L_FH)
    torch.cuda.synchronize()
    assert (lib.kgpu_launch_count() - before) == 4 * 2  # the forward pair; the ring append is a copy, not a kernel
    fh.close()
