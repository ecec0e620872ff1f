"""The device narrowband spectrum analyzer (kgpu_spectrum_run_narrow, kgpu_spectrum_ring_append, filter_spectrum_narrow_*;
narrowband_poll and its ring, reference spectrum.c:123-155 and :206-306): accuracy against a float64 truth of exactly the
float32 windowed samples, the mapping edges, clamp, hop rounding and wrap against the restatement, and the filter.h path:
the device ring bitwise equal to the ring the reference's loop builds from the blocks the slave was delivered."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from ka9q_radio_b200 import capi
from oracle import narrowband as NB
from oracle import oracle as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
COMPLEX = capi.KGPU_COMPLEX


def kaiser_window(n, beta=11.0):
    w = np.kaiser(n + 1, beta)[:n]
    return (w / w.sum()).astype(np.float32)


def make_ring(size, rng, tones=()):
    n = np.arange(size)
    x = (rng.standard_normal(size) + 1j * rng.standard_normal(size)) / np.sqrt(2)
    for f, a in tones:
        x += a * np.exp(2j * np.pi * f * n)
    return x.astype(np.complex64)


def to_dev(ring):
    return torch.from_numpy(np.ascontiguousarray(ring).view(np.float32).reshape(-1, 2)).cuda()


def sources(fft_n, bin_count):
    i = np.arange(bin_count)
    half = bin_count // 2
    src = np.where(i < half, i, fft_n - 2 * half + i)
    return np.where(src < fft_n, src, -1)


def walk(fft_n, fft_avg, overlap, size, ring_idx):
    """spectrum.c:244-281: the clamped count and the sample indices of every segment"""
    limit = np.floor(1 + ((size // fft_n) - 1) / (1 - overlap))
    avg = int(np.rint(limit)) if fft_avg > limit else fft_avg
    rp = ring_idx - int(np.rint(fft_n * (1 + (avg - 1) * (1 - overlap))))
    rp = rp + size if rp < 0 else rp
    hop = fft_n - int(np.rint(fft_n * overlap))
    return avg, [(rp + s * hop + np.arange(fft_n)) % size for s in range(avg)]


def truth(fft_n, bin_count, window, fft_avg, overlap, ring, ring_idx):
    avg, segs = walk(fft_n, fft_avg, overlap, len(ring), ring_idx)
    src = sources(fft_n, bin_count)
    acc = np.zeros(bin_count)
    for idx in segs:
        X = np.fft.fft((ring[idx] * window).astype(np.complex128))  # complex64 x float32, as the kernel forms it
        acc[src >= 0] += np.abs(X[src[src >= 0]]) ** 2 / (float(fft_n) * fft_n * avg)
    return acc


def gpu_poll(sp, ring_dev, ring_idx, fft_avg, overlap, bin_count):
    bins = torch.full((bin_count + 64,), float("nan"), device="cuda")
    used = sp.run_narrow(ring_dev, ring_idx, fft_avg, overlap, bins)
    torch.cuda.synchronize()
    out = bins.cpu().numpy()
    assert np.isnan(out[bin_count:]).all(), "wrote past bin_count"
    return out[:bin_count], used


def analyzer(fft_n, bin_count, window):
    sp = capi.Spectrum(fft_n, COMPLEX, bin_count)
    sp.set_window(window)
    return sp


def close_to(got, ref):
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-5 * ref.max() + 1e-30)


# ------------------------------------------------------------------------------------------ 1. accuracy
ACCURACY = [1620, 2000, 1575, 65536, 69629, 104400]


@pytest.mark.parametrize("fft_n", ACCURACY)
def test_accuracy_against_float64_truth(fft_n):
    rng = np.random.default_rng(fft_n)
    bin_count = fft_n - fft_n // 5
    fft_avg, overlap = 3, 0.5
    size = 2 * fft_n + 333
    ring = make_ring(size, rng)  # noise: every bin near the mean, so the bound is on every bin's rounding
    window = kaiser_window(fft_n)
    ring_idx = 100  # the segments cross the ring end
    sp = analyzer(fft_n, bin_count, window)
    got, used = gpu_poll(sp, to_dev(ring), ring_idx, fft_avg, overlap, bin_count)
    t = truth(fft_n, bin_count, window, fft_avg, overlap, ring, ring_idx)
    orc, used_o = NB.narrowband_spectrum(fft_n, bin_count, window, fft_avg, overlap, ring, ring_idx)
    assert used == used_o == fft_avg
    scale = t.mean()
    e_gpu, e_orc = np.abs(got - t) / scale, np.abs(orc - t) / scale
    print(f"\n{sp.describe()}: gpu max {e_gpu.max():.2e} | float32 oracle max {e_orc.max():.2e}")
    assert e_gpu.max() <= 1e-5
    sp.close()


# ------------------------------------------------------------------------------------------ 2. edges
EDGES = [  # (fft_n, bin_count, fft_avg, overlap, rings, ring_idx): ring_idx -1 = just before the wrap
    (2000, 1999, 3, 0.5, 3, 0),        # odd bin_count: the last bin stays 0
    (2000, 2000, 2, 0.25, 2, -1),      # every bin, ring_idx at the wrap
    (1620, 1001, 12, 0.0, 3, 17),      # fft_avg above avg_limit: clamped to 3
    (1620, 1620, 9, 0.75, 3, -1),      # the clamp with overlap: 9 segments of a 3-fft_n ring
    (1575, 1000, 4, 0.5, 3, 700),      # the walk's hop 787 where lrint(fft_n (1 - overlap)) is 788
    (69629, 50001, 3, 0.5, 2, 5),      # Bluestein, odd fft_n at overlap 0.5, odd bin_count
    (65536, 40000, 130, 0.0, 130, 9),  # more segments than one chunk of scratch holds
]


@pytest.mark.parametrize("fft_n,bin_count,fft_avg,overlap,rings,ring_idx", EDGES)
def test_edges_against_the_restatement(fft_n, bin_count, fft_avg, overlap, rings, ring_idx):
    size = rings * fft_n + (0 if rings > 100 else 41)
    ring_idx = size - 1 if ring_idx < 0 else ring_idx
    ring = make_ring(size, np.random.default_rng(fft_n + bin_count), [(0.2, 3.0), (-0.31, 1.0)])
    window = kaiser_window(fft_n)
    sp = analyzer(fft_n, bin_count, window)
    got, used = gpu_poll(sp, to_dev(ring), ring_idx, fft_avg, overlap, bin_count)
    sp.close()
    ref, used_o = NB.narrowband_spectrum(fft_n, bin_count, window, fft_avg, overlap, ring, ring_idx)
    assert used == used_o == walk(fft_n, fft_avg, overlap, size, ring_idx)[0]
    if bin_count % 2:
        assert got[-1] == 0 and ref[-1] == 0
    close_to(got, ref)


def test_hop_rounding_is_the_walks():
    # fft_n 1575, overlap 0.5: the walk steps 1575 - lrint(787.5) = 787, where lrint(fft_n (1 - overlap)) would step
    # 788.  One impulse at the first sample of segment 2 (2 hops in) lies in segments 0, 1 and 2 with the walk's hop,
    # in only 0 and 1 with the other; with a flat window every bin gets gain per segment that reads it
    fft_n, size, avg = 1575, 4 * 1575, 4
    _, segs = walk(fft_n, avg, 0.5, size, 0)
    assert segs[1][0] - segs[0][0] == 787
    ring = np.zeros(size, np.complex64)
    ring[segs[2][0]] = 1.0
    assert sum(segs[2][0] in s for s in segs) == 3
    sp = analyzer(fft_n, 1000, np.ones(fft_n, np.float32))
    got, _ = gpu_poll(sp, to_dev(ring), 0, avg, 0.5, 1000)
    sp.close()
    np.testing.assert_allclose(got, np.full(1000, 3.0 / (fft_n * fft_n * avg), np.float32), rtol=1e-5)


def test_bad_arguments():
    sp = analyzer(1000, 600, kaiser_window(1000))
    bins = torch.zeros(600, device="cuda")
    with pytest.raises(capi.KgpuError):
        sp.run_narrow(to_dev(np.zeros(999, np.complex64)), 0, 1, 0.0, bins)  # ring shorter than fft_n
    sp.close()
    sp = capi.Spectrum(1000, COMPLEX, 1001)
    with pytest.raises(capi.KgpuError):
        sp.run_narrow(to_dev(np.zeros(2000, np.complex64)), 0, 1, 0.0, torch.zeros(1001, device="cuda"))
    sp.close()
    sp = capi.Spectrum(1000, capi.KGPU_REAL, 600)
    with pytest.raises(capi.KgpuError):
        sp.run_narrow(to_dev(np.zeros(2000, np.complex64)), 0, 1, 0.0, bins)  # a REAL analyzer
    sp.close()


def test_ring_append_is_the_reference_loop():
    rng = np.random.default_rng(9)
    size, fft_n = 3000, 1000
    dev = to_dev(np.zeros(size, np.complex64))
    ref = NB.Ring(size)
    idx = 0
    for n in (700, 1300, 0, 2999, 3001, 7777, 450):
        blk = make_ring(n, rng) if n != 1300 else None
        idx = capi.spectrum_ring_append(dev, idx, to_dev(blk) if blk is not None else n)
        ref.step(3, fft_n, blk, n)
        torch.cuda.synchronize()
        assert idx == ref.ring_idx
        got = dev.cpu().numpy().view(np.complex64).ravel()
        np.testing.assert_array_equal(got.view(np.uint64), ref.ring.view(np.uint64))


# ------------------------------------------------------------------------------------------ 3. filter.h
_drv = None


def drv():
    global _drv
    if _drv is None:
        d = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "nbspectrum_driver.so"))
        vp = C.c_void_p
        d.nd_add.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double]
        d.nd_write_i16.argtypes = [vp, C.c_int, C.c_float]
        d.nd_tuned.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, vp]
        d.nd_plain.argtypes = [C.c_int, C.c_int, vp]
        d.nd_batch.argtypes = [C.c_int, vp, vp, vp]
        d.nd_drops.restype = C.c_uint
        d.nd_setup.argtypes = [C.c_int, C.c_int, C.c_int, vp]
        d.nd_reserve.argtypes = [C.c_int, C.c_long]
        d.nd_poll.argtypes = [C.c_int, C.c_int, C.c_double, vp]
        d.nd_ring.argtypes = [C.c_int, vp, C.c_long, vp]
        d.nd_ring.restype = C.c_long
        d.nd_producer_start.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_float]
        _drv = d
    return _drv


L_FH, M_FH, FS = 20000, 4001, 1.0e6  # N = 24 000: 20 ms blocks at 1 MS/s
OLEN = 1000                           # a 50 kHz narrowband slave
RATE = FS * OLEN / L_FH
SCALE = np.float32(1 / 2048)


class Fh:
    def __init__(self):
        self.d = drv()
        assert self.d.nd_open(L_FH, M_FH) == 0
        self.refs = {}

    def add(self, olen=OLEN, low=-0.4, high=0.4):
        k = self.d.nd_add(olen, low, high, 11.0)
        assert k >= 0
        return k

    def setup(self, k, fft_n, bin_count, window):
        assert self.d.nd_setup(k, fft_n, bin_count, window.ctypes.data) == 0
        self.refs[k] = NB.Ring(1 << 16)

    def tuned(self, k, freq):
        _, shift, rem = O.compute_tuning(L_FH + M_FH - 1, FS, freq)
        assert rem != 0
        y = np.zeros(OLEN, np.complex64)
        assert self.d.nd_tuned(k, shift, rem, RATE, y.ctypes.data) == 0
        return y

    def ring(self, k):
        buf = np.zeros(1 << 16, np.complex64)
        idx = C.c_long(0)
        size = self.d.nd_ring(k, buf.ctypes.data, len(buf), C.byref(idx))
        assert size > 0
        return buf[:size], idx.value

    def poll(self, k, fft_avg, overlap, bin_count):
        bins = np.full(bin_count, np.nan, np.float32)
        assert self.d.nd_poll(k, fft_avg, overlap, bins.ctypes.data) == 0
        return bins

    def check(self, k, fft_n, bin_count, window, fft_avg, overlap):
        """the device ring bitwise the reference loop's, and a poll against the restatement and the reference"""
        ring, idx = self.ring(k)
        ref = self.refs[k]
        assert idx == ref.ring_idx
        np.testing.assert_array_equal(ring.view(np.uint64), ref.ring.view(np.uint64))
        got = self.poll(k, fft_avg, overlap, bin_count)
        want, _ = NB.narrowband_spectrum(fft_n, bin_count, window, fft_avg, overlap, ref.ring, ref.ring_idx)
        close_to(got, want)
        if NB.have_ref():
            own, _ = NB.ref_narrowband_poll(fft_n, bin_count, window, fft_avg, overlap, ref.ring, ref.ring_idx)
            close_to(got, own)

    def close(self):
        self.d.nd_close()


def words(nblocks, seed):
    rng = np.random.default_rng(seed)
    n = np.arange(nblocks * L_FH)
    x = 1500 * np.cos(2 * np.pi * 0.2101 * n) + 300 * rng.standard_normal(len(n))
    return np.clip(np.rint(x), -32768, 32767).astype(np.int16)


@pytest.mark.parametrize("fft_n", [2000, 1999])  # direct and Bluestein
def test_filter_h_ring_and_polls_through_retune_and_growth(fft_n):
    bin_count, overlap = fft_n - 380, 0.5
    window = kaiser_window(fft_n)
    fh = Fh()
    k = fh.add()
    fh.setup(k, fft_n, bin_count, window)
    w = words(14, 21)
    for b in range(14):
        fft_avg = 3 if b < 9 else 5                  # the ring grows at block 9
        freq = 210_000.7 if b < 6 else 211_234.3      # a retune at block 6: that block is recomputed alone
        assert fh.d.nd_reserve(k, fft_avg * fft_n) == 0
        assert fh.d.nd_write_i16(w[b * L_FH:].ctypes.data, L_FH, float(SCALE)) == 1
        y = fh.tuned(k, freq)
        fh.refs[k].step(fft_avg, fft_n, y)
        fh.check(k, fft_n, bin_count, window, fft_avg, overlap)
    fh.close()


def test_filter_h_lapped_blocks_are_zeros_and_drops():
    fft_n, bin_count, fft_avg, overlap = 2000, 1620, 3, 0.5
    window = kaiser_window(fft_n)
    fh = Fh()
    k = fh.add()
    fh.setup(k, fft_n, bin_count, window)
    w = words(6, 22)
    assert fh.d.nd_producer_start(w.ctypes.data, L_FH, 6, 0, float(SCALE)) == 0
    fh.d.nd_producer_join()  # jobs 0..5 issued from another thread: 0 and 1 are lapped
    for _ in range(6):
        assert fh.d.nd_reserve(k, fft_avg * fft_n) == 0
        fh.refs[k].step(fft_avg, fft_n, fh.tuned(k, 210_000.7))
    assert fh.d.nd_drops(k) == 2
    assert (fh.refs[k].ring[:2 * OLEN] == 0).all()
    fh.check(k, fft_n, bin_count, window, fft_avg, overlap)
    fh.close()


def test_filter_h_polls_beside_a_producer_thread():
    fft_n, bin_count, fft_avg, overlap = 2000, 1620, 4, 0.3
    window = kaiser_window(fft_n)
    fh = Fh()
    k = fh.add()
    fh.setup(k, fft_n, bin_count, window)
    nblocks = 30
    w = words(nblocks, 23)
    assert fh.d.nd_producer_start(w.ctypes.data, L_FH, nblocks, 2, float(SCALE)) == 0
    for b in range(nblocks):
        assert fh.d.nd_reserve(k, fft_avg * fft_n) == 0
        fh.refs[k].step(fft_avg, fft_n, fh.tuned(k, 210_000.7))
        fh.d.nd_release()
        if b % 3 == 2:
            fh.check(k, fft_n, bin_count, window, fft_avg, overlap)
    fh.d.nd_producer_join()
    assert fh.d.nd_drops(k) == 0
    fh.check(k, fft_n, bin_count, window, fft_avg, overlap)
    fh.close()


def run_session(with_nb, batch, nblocks=8):
    """a plain slave and a tuned slave (with or without the analyzer); every block both are delivered, one by one or in
    one execute_filter_output_batch; returns the outputs of both and the launches per block"""
    fft_n, fft_avg = 2000, 3
    fh = Fh()
    a, k = fh.add(), fh.add()
    if with_nb:
        fh.setup(k, fft_n, 1620, kaiser_window(fft_n))
    _, sh_a, _ = O.compute_tuning(L_FH + M_FH - 1, FS, -150_000.0)
    _, sh_k, rem_k = O.compute_tuning(L_FH + M_FH - 1, FS, 210_000.7)
    w = words(nblocks, 24)
    outs, launches = [], []
    lib = capi.load()
    for b in range(nblocks):
        if with_nb:
            assert fh.d.nd_reserve(k, fft_avg * fft_n) == 0
        before = lib.kgpu_launch_count()
        assert fh.d.nd_write_i16(w[b * L_FH:].ctypes.data, L_FH, float(SCALE)) == 1
        ya, yk = np.zeros(OLEN, np.complex64), np.zeros(OLEN, np.complex64)
        if batch:
            # the tuned slave's oscillator is set by one tuned call first; the batch then delivers both
            if b == 0:
                assert fh.d.nd_tuned(k, sh_k, rem_k, RATE, yk.ctypes.data) == 0
                assert fh.d.nd_plain(a, sh_a, ya.ctypes.data) == 0
            else:
                ks = (C.c_int * 2)(a, k)
                shifts = (C.c_int * 2)(sh_a, sh_k)
                ys = (C.c_void_p * 2)(ya.ctypes.data, yk.ctypes.data)
                assert fh.d.nd_batch(2, ks, shifts, ys) == 0
        else:
            assert fh.d.nd_plain(a, sh_a, ya.ctypes.data) == 0
            assert fh.d.nd_tuned(k, sh_k, rem_k, RATE, yk.ctypes.data) == 0
        torch.cuda.synchronize()
        launches.append(lib.kgpu_launch_count() - before)
        outs.append((ya, yk))
        if with_nb:
            fh.refs[k].step(fft_avg, fft_n, yk)
    if with_nb:
        fh.check(k, fft_n, 1620, kaiser_window(fft_n), fft_avg, 0.5)
    fh.close()
    return outs, launches


@pytest.mark.parametrize("batch", [False, True], ids=["one_by_one", "batch"])
def test_filter_h_other_slaves_and_launches_unchanged(batch):
    plain, l_plain = run_session(False, batch)
    with_nb, l_nb = run_session(True, batch)
    for (a0, k0), (a1, k1) in zip(plain, with_nb):
        np.testing.assert_array_equal(a0.view(np.uint64), a1.view(np.uint64))
        np.testing.assert_array_equal(k0.view(np.uint64), k1.view(np.uint64))
    # from the third block on every block is a batch hit: the analyzer adds exactly its one append per block
    assert l_nb[2:] == [n + 1 for n in l_plain[2:]]


def test_filter_h_setup_rejects_what_the_device_cannot_serve():
    fh = Fh()
    k = fh.add()
    w = kaiser_window(2000)
    assert fh.d.nd_setup(k, 2000, 2001, w.ctypes.data) == -1  # bin_count > fft_n
    assert fh.d.nd_reserve(k, 6000) == -1                     # no analyzer
    assert fh.d.nd_poll(k, 1, 0.0, np.zeros(10, np.float32).ctypes.data) == -1
    fh.setup(k, 2000, 1620, w)
    assert fh.d.nd_poll(k, 1, 0.0, np.zeros(1620, np.float32).ctypes.data) == -1  # before the first reserve
    assert fh.d.nd_reserve(k, 6000) == 0
    assert fh.d.nd_reserve(k, 4000) == 0  # smaller: no change
    assert fh.ring(k)[0].shape == (6000,)
    assert fh.d.nd_delete(k) == 0
    fh.close()
