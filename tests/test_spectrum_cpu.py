"""Host-only checks of the wideband spectrum analyzer: the transform kgpu_spectrum_create picks from fft_n alone."""
import pytest

from ka9q_radio_b200 import capi

REAL, COMPLEX = capi.KGPU_REAL, capi.KGPU_COMPLEX


@pytest.mark.parametrize("fft_n,in_type,path,text", [
    (518400, REAL, capi.SPECTRUM_R2C, "r2c fft_n=518400 real P=518400: 259200-point"),   # rbw 250 Hz at 129.6 MS/s
    (22800, REAL, capi.SPECTRUM_R2C, "r2c fft_n=22800 real P=22800: 11400-point"),       # factor 19: the extended pair
    (6075, REAL, capi.SPECTRUM_COMPLEX, "complex fft_n=6075 real P=6075"),              # odd REAL: complex transform
    (6075, COMPLEX, capi.SPECTRUM_COMPLEX, "complex fft_n=6075 complex P=6075"),
    (7005, REAL, capi.SPECTRUM_BLUESTEIN, "bluestein fft_n=7005 real P=14112"),          # 3 * 5 * 467
    (7005, COMPLEX, capi.SPECTRUM_BLUESTEIN, "bluestein fft_n=7005 complex P=14112"),
    (104400, REAL, capi.SPECTRUM_BLUESTEIN, "bluestein fft_n=104400 real P=209952"),      # factor 29
    (6125000, COMPLEX, capi.SPECTRUM_COMPLEX, "complex fft_n=6125000"),
])
def test_path_choice(fft_n, in_type, path, text):
    got, desc = capi.spectrum_plan(fft_n, in_type)
    assert got == path
    assert desc.startswith(text)


def test_bluestein_limit():
    # the largest Bluestein transform the forward pair splits within shared memory is 3500 x 3500
    _, desc = capi.spectrum_plan(29 * 211206, COMPLEX)  # 6 124 974 points
    assert "P=12250000" in desc and "3500 x 3500" in desc
    for n in (29 * 211207, 8388609):
        with pytest.raises(capi.KgpuError, match="Bluestein"):
            capi.spectrum_plan(n, REAL)


def test_bad_arguments():
    with pytest.raises(capi.KgpuError):
        capi.spectrum_plan(1, REAL)
    with pytest.raises(capi.KgpuError):
        capi.spectrum_plan(6480, 3)
