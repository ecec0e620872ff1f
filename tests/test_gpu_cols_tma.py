"""fwd_cols_r36 with its input tile fetched by tensor copies against the same kernel reading global memory
(kgpu_use_cols_tma 1 / 0): spectra bitwise equal, int16 statistics exactly equal.

Geometries: cfg-2 (1296 x 1250, the ragged last column group 1250 = 156 * 8 + 2) with float input, int16, and int16 with
de-randomisation and statistics, over 1 and 32 blocks; 1296 x 1280 (n2 from the arguments); COMPLEX 1296 x 1250.  Inputs
that fall back to global loads with the switch on: odd n2 (1296 x 1215), a window base 4 or 8 bytes off 16-byte alignment
and a hop whose int16 windows are not 16 bytes apart.  A misaligned input must also give what an aligned copy of the same
bytes gives through the tensor copies.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

REAL, CPLX = 2, 1


def _spectra(m, ptr, i16, nb, derand, with_stats, tma, dev):
    from ka9q_radio_b200 import capi

    lib = capi.load()
    spec = torch.zeros((nb, m.spec_stride), dtype=torch.complex64, device=dev)
    stats = torch.zeros((nb, 2), dtype=torch.int64, device=dev) if with_stats else None
    st = torch.cuda.current_stream(dev).cuda_stream
    lib.kgpu_use_cols_tma(tma)
    try:
        m.forward(ptr, capi.KGPU_FMT_I16 if i16 else capi.KGPU_FMT_F32, 1 / 3000 if i16 else 1.0, nb, spec.data_ptr(), st,
                  derandomize=derand, d_stats=stats.data_ptr() if with_stats else 0)
        torch.cuda.synchronize()
    finally:
        lib.kgpu_use_cols_tma(1)
    return spec[:, :m.bins].contiguous().view(torch.int32).cpu().numpy(), None if stats is None else stats.cpu().numpy()


def _input(L, M, real, i16, nb, b0, seed):
    rng = np.random.default_rng(seed)
    n = ((nb + b0) * L + M - 1) * (1 if real else 2) + 64  # + room for the offsets
    return rng.integers(-32768, 32768, n, dtype=np.int16) if i16 else rng.standard_normal(n, dtype=np.float32)


# (L, M, REAL, int16, derandomize, statistics, blocks, first block, byte offset, tensor copies)
CASES = {
    "cfg2_f32_32": (2592000, 648001, True, False, False, False, 32, 1, 0, 1),
    "cfg2_f32_1": (2592000, 648001, True, False, False, False, 1, 2, 0, 1),
    "cfg2_i16_32": (2592000, 648001, True, True, False, False, 32, 3, 0, 1),
    "cfg2_i16_stats_32": (2592000, 648001, True, True, True, True, 32, 3, 0, 1),
    "cfg2_i16_stats_1": (2592000, 648001, True, True, False, True, 1, 0, 0, 1),
    "r1296x1280_i16_stats": (2654208, 663553, True, True, True, True, 3, 1, 0, 1),
    "c1296x1280_f32": (1327104, 331777, False, False, False, False, 2, 1, 0, 1),
    "c1296x1250_i16": (1296000, 324001, False, True, True, True, 3, 1, 0, 1),
    "r1296x1215_i16_odd_n2": (2519424, 629857, True, True, True, True, 2, 1, 0, 0),
    "r1296x1215_f32_odd_n2": (2519424, 629857, True, False, False, False, 2, 1, 0, 0),
    "cfg2_i16_off4": (2592000, 648001, True, True, True, True, 2, 1, 4, 0),
    "cfg2_i16_off8": (2592000, 648001, True, True, False, False, 2, 1, 8, 0),
    "cfg2_f32_off8": (2592000, 648001, True, False, False, False, 2, 1, 8, 0),
    "hop_i16_unaligned": (2592004, 647997, True, True, True, True, 3, 1, 0, 0),
    "hop_f32": (2592004, 647997, True, False, False, False, 3, 1, 0, 1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_cols_tma_bitwise(cuda_dev, case):
    from ka9q_radio_b200 import capi

    L, M, real, i16, derand, with_stats, nb, b0, off, tma = CASES[case]
    lib = capi.load()
    m = capi.Master(L, M, REAL if real else CPLX)
    try:
        assert "fwd_cols_r36" in m.describe()
        host = _input(L, M, real, i16, nb, b0, seed=L + M + nb + off)
        x = torch.from_numpy(host).to(cuda_dev)
        pair = (2 if i16 else 4) * (1 if real else 2)  # bytes of one input sample (I/Q pair for COMPLEX)
        ptr = x.data_ptr() + b0 * L * pair + off
        fmt = capi.KGPU_FMT_I16 if i16 else capi.KGPU_FMT_F32
        assert lib.kgpu_cols_tma_fits(L, M, REAL if real else CPLX, fmt, ptr) == tma
        got, st_got = _spectra(m, ptr, i16, nb, derand, with_stats, 1, cuda_dev)
        ref, st_ref = _spectra(m, ptr, i16, nb, derand, with_stats, 0, cuda_dev)
        assert np.array_equal(got, ref), f"{case}: {int((got != ref).sum())} words differ"
        if with_stats:
            assert np.array_equal(st_got, st_ref)
            assert st_ref[:, 0].min() > 0  # every block has new samples
        if off:  # the same bytes at an aligned address take the tensor copies
            start = b0 * L * pair + off
            y = torch.from_numpy(host.view(np.uint8)[start:].copy()).to(cuda_dev)
            assert lib.kgpu_cols_tma_fits(L, M, REAL if real else CPLX, fmt, y.data_ptr()) == 1
            al, st_al = _spectra(m, y.data_ptr(), i16, nb, derand, with_stats, 1, cuda_dev)
            assert np.array_equal(al, ref)
            if with_stats:
                assert np.array_equal(st_al, st_ref)
    finally:
        m.close()
