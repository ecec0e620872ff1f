"""The REAL row pass fwd_rows_v2 takes 8 mirrored row pairs per CTA: every split n1 x 1250 bin by bin, with NaN sentinels.

The geometries give item counts n1/2 + 1 of every residue mod 8, so the last CTA of a block holds 1..8 items (649 for
the halved 1296 x 1250 pass of cfg-2 leaves it one); n1 = 1323, 1575 and 1875 are odd (no k1 = n1/2 row).  Float input
is scored against float64 rfft of exactly the float32 window, with the bounds of test_gpu_accuracy.py; int16 input
against the same transform of the scaled samples.  The guard rows, the row padding [bins, spec_stride) and every bin
are checked for stray or missing stores."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_E = 5e-6
NAN_BITS = 0x7FC0DEAD
SCALE = float(np.float32(10 ** (3 / 20) / 32768))
GEOS = [  # (n1, L, M): N = 2 * 1250 * n1, overlap 5
    (1470, 2940000, 735001),  # 736 items: 0 mod 8
    (1296, 2592000, 648001),  # 649: 1, halved split on fwd_cols_r36
    (1280, 2560000, 640001),  # 641: 1
    (1875, 3750000, 937501),  # 938: 2, odd n1
    (2500, 5000000, 1250001),  # 1251: 3
    (1575, 3150000, 787501),  # 788: 4, odd n1
    (1400, 2800000, 700001),  # 701: 5
    (1323, 2646000, 661501),  # 662: 6, odd n1
    (1260, 2520000, 630001),  # 631: 7
]
CASES = [pytest.param(g, False, id=f"r{g[0]}x1250-f32") for g in GEOS] + [
    pytest.param(g, True, id=f"r{g[0]}x1250-i16") for g in GEOS if g[0] in (1296, 1323, 1260)]


def _err(got, truth):
    return np.abs(np.asarray(got, np.complex128) - truth) / np.sqrt(np.mean(np.abs(truth) ** 2))


@pytest.mark.parametrize("geo,i16", CASES)
def test_real_rows_v2_per_bin_and_writes(oracle, cuda_dev, geo, i16):
    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    n1, L, M = geo
    rng = np.random.default_rng(n1 + 7 * i16)
    if i16:
        xi = rng.integers(-32768, 32768, 3 * L, dtype=np.int16)
        x = xi.astype(np.float32) * np.float32(SCALE)
    else:
        x = rng.standard_normal(3 * L, dtype=np.float32)
    cz = Channelizer(L, M, capi.KGPU_REAL, cuda_dev, capacity=1)
    try:
        desc = cz.master.describe()
        items = n1 // 2 + 1
        assert f"two-pass {n1} x 1250; cols radices [" in desc and "rows radices [10,25,5]" in desc, desc
        assert f"/{(items + 7) // 8} CTAs per block" in desc and desc.endswith(" + fwd_rows_v2"), desc
        bins, stride = cz.master.bins, cz.master.spec_stride
        buf = torch.full((4, 2 * stride), NAN_BITS, dtype=torch.int32, device=cuda_dev).view(torch.float32)
        buf = buf.view(torch.complex64)
        spec = buf[1:3]
        cz.forward(cz.stage_stream(xi if i16 else x), 2, spec, scale=SCALE if i16 else 1.0, first_block=1)
        torch.cuda.synchronize()
        raw = buf.view(torch.float32).view(torch.int32).cpu().numpy()
        got = spec.cpu().numpy()[:, :bins]
    finally:
        cz.close()
    assert (raw[0] == NAN_BITS).all() and (raw[3] == NAN_BITS).all(), "store outside the launched blocks' rows"
    assert (raw[1:3, 2 * bins:] == NAN_BITS).all(), "store into the row padding [bins, spec_stride)"
    assert np.isfinite(got).all(), "bin left unwritten"
    e_gpu, e_ora = [], []
    for j, b in enumerate((1, 2)):
        w = oracle.block_window(x, L, M, b)
        truth = np.fft.rfft(w.astype(np.float64))
        e_gpu.append(_err(got[j], truth))
        if not i16:
            e_ora.append(_err(oracle.forward(w), truth))
    e_gpu = np.concatenate(e_gpu)
    assert e_gpu.max() <= MAX_E, e_gpu.max()
    if not i16:
        e_ora = np.concatenate(e_ora)
        r_rms = np.sqrt(np.mean(e_gpu ** 2)) / np.sqrt(np.mean(e_ora ** 2))
        r_max = e_gpu.max() / e_ora.max()
        print(f"r{n1}x1250: max e {e_gpu.max():.2e} (oracle {e_ora.max():.2e}), gpu/oracle rms {r_rms:.2f} max {r_max:.2f}")
        assert r_rms <= 2.0 and r_max <= 4.0, (r_rms, r_max)
