"""The narrowband spectrum analyzer on the host: the restatement (oracle/narrowband_oracle.c) bitwise against the
reference's own narrowband_poll (spectrum.c:206-306, built unmodified into oracle/_ref/libka9qnarrowband.so), the ring
upkeep of spectrum.c:124-151, and the transform path of every length setup_narrowband can choose."""
import numpy as np
import pytest

from ka9q_radio_b200 import capi
from oracle import narrowband as NB

need_ref = pytest.mark.skipif(not NB.have_ref(), reason="oracle/_ref/libka9qnarrowband.so not built (reference absent)")


def kaiser_window(n, beta=11.0):
    w = np.kaiser(n + 1, beta)[:n]
    return (w / w.sum()).astype(np.float32)  # normalize_windowf scales to unit sum


def ring_of(size, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(size) + 1j * rng.standard_normal(size)).astype(np.complex64)


def hop_rounding_differs(fft_n, overlap):
    return fft_n - round(fft_n * overlap) != round(fft_n * (1 - overlap))


# (fft_n, bin_count): 23-smooth lengths, 65 536 and 69 629 = 29 x 7^4 (above 65 536, a Bluestein length on the device);
# even and odd bin_count, and all bins
POLLS = [(1620, 1000), (1620, 1001), (1620, 1620), (2000, 1999), (2000, 2000), (1575, 1000), (65536, 40000),
         (65536, 65535), (69629, 50000), (69629, 69628)]
# (fft_avg, overlap, ring_size in fft_n): within the ring, above avg_limit, and overlap 0.5 with an odd fft_n, where the
# walk's hop fft_n - lrint(fft_n overlap) differs from lrint(fft_n (1 - overlap))
WALKS = [(1, 0.0, 1), (3, 0.5, 3), (4, 0.3, 4), (12, 0.0, 3), (9, 0.75, 3), (5, 0.3333, 5)]


def test_hop_rounding_case_is_exercised():
    assert hop_rounding_differs(1575, 0.5) and hop_rounding_differs(69629, 0.5)
    assert not hop_rounding_differs(2000, 0.5)


@need_ref
@pytest.mark.parametrize("fft_n,bin_count", POLLS)
@pytest.mark.parametrize("fft_avg,overlap,rings", WALKS)
def test_restatement_bitwise_equals_reference(fft_n, bin_count, fft_avg, overlap, rings):
    if fft_n > 60000 and fft_avg * rings > 12:
        pytest.skip("long CPU transforms: the shorter walks cover the same arithmetic")
    size = rings * fft_n + 37
    ring = ring_of(size, fft_n * 31 + bin_count + fft_avg)
    window = kaiser_window(fft_n)
    for idx in (0, size - 1, size // 3):  # at 0, just before the wrap, inside
        ref, used_ref = NB.ref_narrowband_poll(fft_n, bin_count, window, fft_avg, overlap, ring, idx)
        got, used = NB.narrowband_spectrum(fft_n, bin_count, window, fft_avg, overlap, ring, idx)
        assert used == used_ref
        np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))
        if bin_count % 2:
            assert got[-1] == 0  # the reference reads one past its transform there; 0 in both


def test_clamp_matches_spectrum_c():
    fft_n, window = 1000, kaiser_window(1000)
    for size, fft_avg, overlap in [(3000, 12, 0.0), (3000, 9, 0.75), (2999, 5, 0.5), (1000, 4, 0.5)]:
        limit = np.floor(1 + ((size // fft_n) - 1) / (1 - overlap))
        want = int(np.rint(limit)) if fft_avg > limit else fft_avg
        _, used = NB.narrowband_spectrum(fft_n, 600, window, fft_avg, overlap, ring_of(size, 1), 5)
        assert used == want


def test_bad_arguments_are_rejected():
    w = kaiser_window(100)
    with pytest.raises(ValueError):
        NB.narrowband_spectrum(100, 101, w, 1, 0.0, ring_of(200, 2), 0)  # bin_count > fft_n
    with pytest.raises(ValueError):
        NB.narrowband_spectrum(100, 50, w, 1, 0.0, ring_of(99, 2), 0)  # ring shorter than fft_n


def reference_ring_loop(blocks, fft_avgs, fft_n):
    """spectrum.c:124-151 written out in Python, block by block (None = a block of zeros)"""
    ring, idx = None, 0
    for blk, avg in zip(blocks, fft_avgs):
        if ring is None or len(ring) < avg * fft_n:
            if ring is None:
                idx = 0
                ring = np.zeros(0, np.complex64)
            ring = np.concatenate([ring, np.zeros(avg * fft_n - len(ring), np.complex64)])
        for s in blk:
            ring[idx] = s
            idx += 1
            if idx == len(ring):
                idx = 0
    return ring, idx


def test_ring_growth_wrap_and_zero_fill():
    fft_n, olen = 300, 250
    rng = np.random.default_rng(3)
    blocks, avgs = [], []
    for b in range(20):
        blocks.append(np.zeros(olen, np.complex64) if b in (7, 8) else
                      (rng.standard_normal(olen) + 1j * rng.standard_normal(olen)).astype(np.complex64))
        avgs.append(2 if b < 5 else 5 if b < 12 else 3)  # grows at block 5, never shrinks at 12
    r = NB.Ring(10 * fft_n)
    for b, (blk, avg) in enumerate(zip(blocks, avgs)):
        r.step(avg, fft_n, None if b in (7, 8) else blk, olen)
        want, idx = reference_ring_loop(blocks[:b + 1], avgs[:b + 1], fft_n)
        assert r.ring_idx == idx
        np.testing.assert_array_equal(r.ring.view(np.uint64), want.view(np.uint64))
    assert len(r.ring) == 5 * fft_n


def test_ring_block_longer_than_the_ring():
    r = NB.Ring(100)
    blk = (np.arange(250) + 1j).astype(np.complex64)
    r.step(1, 100, blk)
    want, idx = reference_ring_loop([blk], [1], 100)
    assert r.ring_idx == idx == 50
    np.testing.assert_array_equal(r.ring, want)


def reference_goodchoice(n):
    e = {}
    for p in (2, 3, 5, 7, 11, 13):
        while n % p == 0:
            n //= p
            e[p] = e.get(p, 0) + 1
    return n == 1 and e.get(11, 0) + e.get(13, 0) <= 1


def test_every_setup_narrowband_length_has_a_transform():
    # setup_narrowband (spectrum.c:653-656) returns a goodchoice length below 65 536 (the reference's, or the library's
    # 7-smooth one, a subset), or 65 536, or its starting length when that is larger
    lengths = [n for n in range(2, 65536) if reference_goodchoice(n)] + [65536]
    for n in lengths:
        path, text = capi.spectrum_plan(n, capi.KGPU_COMPLEX)
        assert path == capi.SPECTRUM_COMPLEX, (n, text)
    for n in (65537, 70001, 100003, 1 << 20, 1234567):
        path, _ = capi.spectrum_plan(n, capi.KGPU_COMPLEX)
        assert path in (capi.SPECTRUM_COMPLEX, capi.SPECTRUM_BLUESTEIN)
