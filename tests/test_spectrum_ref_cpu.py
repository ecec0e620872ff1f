"""The wideband spectrum restatement (oracle/spectrum_oracle.c) against the reference's own wideband_poll (spectrum.c:308-522,
built unmodified into oracle/_ref/libka9qspectrum.so): bitwise equal bins over both front-end types, shifts on both sides
and at the coverage edges, overlaps, fft_avg 1 .. 8, segments across the ring end, odd fft_n and odd bin_count.  REAL
geometries whose walk reads below the r2c output in the reference (undefined there, 0 in the restatement) are skipped."""
import numpy as np
import pytest

from oracle import spectrum as S

pytestmark = pytest.mark.skipif(not S.have_ref(), reason="oracle/_ref/libka9qspectrum.so not built (reference absent)")


def real_walk_reads_below_zero(fft_n, bin_count, shift):
    b0 = shift if shift >= 0 else fft_n // 2 + shift
    top, half = fft_n // 2 + 1, bin_count // 2
    if b0 < 0:
        return True
    return b0 + half < top and b0 + half - bin_count < 0


def kaiser_window(n, beta=11.0):
    w = np.kaiser(n + 1, beta)[:n]
    return (w / w.sum()).astype(np.float32)  # normalize_windowf scales to unit sum


GEOMS = []
for fft_n, bins in [(1000, 400), (1001, 301), (96, 96), (97, 33)]:
    for shift in (0, 5, -5, bins // 2, fft_n // 2 - bins // 2, -(fft_n // 2), fft_n // 2, -(fft_n // 2) + bins // 2 + 3,
                  fft_n // 3, -fft_n // 3):
        GEOMS.append((fft_n, bins, shift))


@pytest.mark.parametrize("is_real", [True, False], ids=["real", "complex"])
@pytest.mark.parametrize("fft_n,bin_count,shift", GEOMS)
@pytest.mark.parametrize("overlap,fft_avg", [(0.0, 1), (0.5, 3), (0.3333, 4), (0.9, 8), (0.25, 2)])
def test_restatement_bitwise_equals_reference(is_real, fft_n, bin_count, shift, overlap, fft_avg):
    if is_real and real_walk_reads_below_zero(fft_n, bin_count, shift):
        pytest.skip("the reference reads fft_out[negative] here")
    rng = np.random.default_rng(fft_n * 7919 + bin_count * 31 + shift + 1000 + int(overlap * 1e4) + fft_avg)
    cap = 4 * fft_n + 17
    if is_real:
        ring = rng.standard_normal(cap).astype(np.float32)
    else:
        ring = (rng.standard_normal(cap) + 1j * rng.standard_normal(cap)).astype(np.complex64)
    window = kaiser_window(fft_n)
    for end in (cap // 3, 5):  # segments inside the ring, and across its end (backwards for COMPLEX)
        ref, used = S.ref_wideband_poll(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end)
        assert used == fft_avg
        got = S.wideband_spectrum(is_real, fft_n, bin_count, window, shift, fft_avg, overlap, ring, end)
        np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_adjust_rounding_case_is_exercised():
    # adjust = lrint(fft_n (1 + (fft_avg-1)(1-overlap))) differs from fft_n + (fft_avg-1) hop here
    fft_n, overlap, fft_avg = 1000, 0.3333, 4
    hop = round(fft_n * (1 - overlap))
    adjust = round(fft_n * (1 + (fft_avg - 1) * (1 - overlap)))
    assert adjust != fft_n + (fft_avg - 1) * hop
