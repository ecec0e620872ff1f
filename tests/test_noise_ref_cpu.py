"""CPU suite (no GPU): pins the numpy restatement of estimate_noise in noise_fm_ref.py, which the device tests of
test_gpu_noise_fm.py score noise_kernel against, to the oracle's oracle.estimate_noise (chan_oracle_ext.c, a
line-by-line restatement of radio.c:1783-1866), on the same synthetic windows: windows of more than 4096 bins, ties at
the quantile, energies exactly at 1.5 q, and windows that clamp at DC and Nyquist or wrap through the COMPLEX master's
DC bin.  Where the reference reads outside its master (a REAL master smaller than the window) there is nothing to pin."""
import numpy as np
import pytest

import noise_fm_ref as R

FS = 1.92e6


def _check(oracle, X, complex_master, s_bins, shift):
    it = oracle.KO_COMPLEX if complex_master else oracle.KO_REAL
    ref = oracle.estimate_noise(it, X, s_bins, shift, FS)
    got = R.estimate_noise(X, complex_master, s_bins, shift, FS)
    if ref == 0:
        assert got == 0, (s_bins, shift, got)
    else:
        assert abs(got - ref) <= 1e-12 * ref, (s_bins, shift, got, ref)
    return ref


def test_order_statistic_windows_match_oracle(oracle):
    rng = np.random.default_rng(11)
    cases = R.order_stat_windows(rng)
    for blk in range(2):
        X = R.exact_components(rng, 48001)
        wins = [b(rng) for _, _, _, b in cases]
        shifts = R.place_windows(X, wins)
        for (name, pts, real_out, _), sh in zip(cases, shifts):
            s_bins = pts // 2 + 1 if real_out else pts
            ref = _check(oracle, X, False, s_bins, sh)
            assert (ref == 0) == (name == "all zero"), name


@pytest.mark.parametrize("complex_master", [False, True])
def test_widths_and_edges_match_oracle(oracle, complex_master):
    rng = np.random.default_rng(12 + complex_master)
    m = 96000 if complex_master else 48001
    X = R.exact_components(rng, m, kmax=511)
    X[rng.integers(0, m, m // 20)] *= 4  # strong bins for the threshold to drop; still exact
    for s_bins in (601, 1000, 1125, 3375, 4097, 4801, 7200, 9600, 14407, 28812):
        n = max(s_bins, 1000)
        if complex_master:
            h = m // 2
            shifts = [0, n // 2 - 5, h - 7 + n // 2, h + n // 2, h + 1 + n // 2, -h, m + 100 + n // 2, n // 2 - m - 1]
        else:
            shifts = [0, 3, -3, n // 2, n // 2 + 1, -(n // 2) - 1, m - n + n // 2, m - n + n // 2 - 1, m - 1, 1 - m]
        shifts += list(rng.integers(-m // 2, m // 2, 4))
        for sh in shifts:
            _check(oracle, X, complex_master, s_bins, int(sh))
