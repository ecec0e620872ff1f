"""Where fwd_cols_r36 takes its input tile by tensor copies, decided on the host (kgpu_cols_tma_fits, no device needed).

A tensor map needs a 16-byte aligned base and strides that are multiples of 16 bytes: the row pitch of n2 points
(8 n2 bytes, a row of floats or a pair of int16 rows) and the hop between windows.  Every other input of a 1296-row
master runs the same kernel with global loads, and masters without fwd_cols_r36 never take tensor copies.
"""
import pytest

from ka9q_radio_b200 import capi

I16, F32 = capi.KGPU_FMT_I16, capi.KGPU_FMT_F32
REAL, CPLX = capi.KGPU_REAL, capi.KGPU_COMPLEX
BASE = 0x7F0000000000  # a 16-byte (indeed page) aligned device address; only its low bits matter


@pytest.mark.parametrize("L,M,in_type,fmt,offset,want", [
    (2592000, 648001, REAL, I16, 0, 1),    # cfg-2, 1296 x 1250
    (2592000, 648001, REAL, F32, 0, 1),
    (2592000, 648001, REAL, I16, 4, 0),    # window base off by one int16 pair
    (2592000, 648001, REAL, I16, 8, 0),
    (2592000, 648001, REAL, F32, 8, 0),    # off by one float pair
    (2592000, 648001, REAL, F32, 16, 1),
    (2592004, 647997, REAL, I16, 0, 0),    # hop 1 296 002 pairs: 4 hop is not a multiple of 16
    (2592004, 647997, REAL, F32, 0, 1),    # 8 hop is
    (2654208, 663553, REAL, I16, 0, 1),    # 1296 x 1280 (n2 from the arguments)
    (1327104, 331777, CPLX, F32, 0, 1),
    (2519424, 629857, REAL, I16, 0, 0),    # 1296 x 1215: odd n2, the row pitch is not a multiple of 16 bytes
    (2519424, 629857, REAL, F32, 0, 0),
    (1296000, 324001, CPLX, I16, 0, 1),    # COMPLEX 1296 x 1250
    (2560000, 640001, REAL, I16, 0, 0),    # 1280 x 1250: generic column kernel
    (400000, 100001, CPLX, F32, 0, 0),     # 800 x 625: fwd_cols_2s
    (1240000, 310001, REAL, I16, 0, 0),    # Bluestein master
])
def test_cols_tma_fits(L, M, in_type, fmt, offset, want):
    lib = capi.load()
    assert lib.kgpu_cols_tma_fits(L, M, in_type, fmt, BASE + offset) == want


def test_cols_tma_fits_bad_arguments():
    lib = capi.load()
    assert lib.kgpu_cols_tma_fits(0, 1, REAL, I16, BASE) == -1
    assert lib.kgpu_cols_tma_fits(2592001, 648001, REAL, I16, BASE) == -1  # REAL needs an even L
