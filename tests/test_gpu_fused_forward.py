"""fwd_fused_r36_v2, the column and row passes of REAL 1296 x 1250 masters as one launch, against the two-kernel pair
(fwd_cols_r36_tma + fwd_rows_v2; kgpu_use_fused_forward 1 / 0) on cfg-2: spectra bitwise equal, int16 statistics exactly
equal, for float input, int16, and int16 with de-randomisation and statistics, over 2, 3, 32 and 33 blocks from a
nonzero first block (and 1 block, which runs the pair).  Each run writes into a buffer of NaN sentinels: the guard rows around the launched blocks and the
row padding [bins, spec_stride) must come back untouched.  Also: the fused form is one launch and the pair two; two
masters on two streams at once (their ticket and done counters are their own); leads other than the default and the
form without the L2 discard give the same bits; and an input the tensor copies cannot take runs the pair.
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

REAL = 2
L, M = 2592000, 648001
NAN_BITS = 0x7FC00001


def _input(nb, b0, i16, seed):
    rng = np.random.default_rng(seed)
    n = (nb + b0) * L + M - 1 + 64
    return rng.integers(-32768, 32768, n, dtype=np.int16) if i16 else rng.standard_normal(n, dtype=np.float32)


def _run(m, ptr, i16, nb, derand, with_stats, fused, dev, stream=None):
    """spectra as int32 words [nb + 2][2 * spec_stride] (guard rows 0 and nb + 1), statistics, launches made"""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    buf = torch.full((nb + 2, 2 * m.spec_stride), NAN_BITS, dtype=torch.int32, device=dev)
    spec = buf.view(torch.float32).view(torch.complex64)[1:nb + 1]
    stats = torch.zeros((nb, 2), dtype=torch.int64, device=dev) if with_stats else None
    st = (stream or torch.cuda.current_stream(dev)).cuda_stream
    lib.kgpu_use_fused_forward(fused)
    try:
        torch.cuda.synchronize()
        n0 = lib.kgpu_launch_count()
        m.forward(ptr, capi.KGPU_FMT_I16 if i16 else capi.KGPU_FMT_F32, 1 / 3000 if i16 else 1.0, nb, spec.data_ptr(), st,
                  derandomize=derand, d_stats=stats.data_ptr() if with_stats else 0)
        n = lib.kgpu_launch_count() - n0
        torch.cuda.synchronize()
    finally:
        lib.kgpu_use_fused_forward(1)
    return buf.cpu().numpy(), None if stats is None else stats.cpu().numpy(), n


def _check(raw, m, nb):
    bins = m.bins
    assert (raw[0] == NAN_BITS).all() and (raw[nb + 1] == NAN_BITS).all(), "store outside the launched blocks' rows"
    assert (raw[1:nb + 1, 2 * bins:] == NAN_BITS).all(), "store into the row padding [bins, spec_stride)"
    assert not (raw[1:nb + 1, :2 * bins] == NAN_BITS).any(), "bin left unwritten"


# (int16, derandomize, statistics)
FORMS = {"f32": (False, False, False), "i16": (True, False, False), "i16_derand_stats": (True, True, True)}


@pytest.mark.parametrize("nb", [1, 2, 3, 32, 33])
@pytest.mark.parametrize("form", list(FORMS))
def test_fused_bitwise(cuda_dev, form, nb):
    from ka9q_radio_b200 import capi

    i16, derand, with_stats = FORMS[form]
    lib = capi.load()
    m = capi.Master(L, M, REAL)
    try:
        desc = m.describe()
        assert "two-pass 1296 x 1250; cols radices [36,36] rows radices [10,25,5]" in desc and "/82 CTAs per block" in desc
        assert "kernels fwd_cols_r36 + " in desc and desc.endswith(" + fwd_rows_v2"), desc
        b0 = 1 + nb % 3
        x = torch.from_numpy(_input(nb, b0, i16, seed=nb + 100 * i16 + 1000 * derand)).to(cuda_dev)
        ptr = x.data_ptr() + b0 * L * (2 if i16 else 4)
        fmt = capi.KGPU_FMT_I16 if i16 else capi.KGPU_FMT_F32
        assert lib.kgpu_fused_forward_fits(L, M, REAL, fmt, ptr) == 1
        got, st_got, n_fused = _run(m, ptr, i16, nb, derand, with_stats, 1, cuda_dev)
        ref, st_ref, n_pair = _run(m, ptr, i16, nb, derand, with_stats, 0, cuda_dev)
        assert (n_fused, n_pair) == (1 if nb > 1 else 2, 2)  # one block runs the pair
        _check(ref, m, nb)
        _check(got, m, nb)
        assert np.array_equal(got, ref), f"{form} B={nb}: {int((got != ref).sum())} words differ"
        if with_stats:
            assert np.array_equal(st_got, st_ref)
            assert st_ref[:, 0].min() > 0
    finally:
        m.close()


def test_fused_options_same_bits(cuda_dev):
    """the lead of column items and the L2 discard change only the order and the cache, never a value"""
    from ka9q_radio_b200 import capi

    lib = capi.load()
    shape = (C.c_int * 5)()
    lib.kgpu_fused_shape(C.cast(shape, C.c_void_p))
    nc, default_lead = shape[0], shape[4]
    nb, b0 = 5, 2
    m = capi.Master(L, M, REAL)
    try:
        x = torch.from_numpy(_input(nb, b0, True, seed=7)).to(cuda_dev)
        ptr = x.data_ptr() + b0 * L * 2
        ref, st_ref, _ = _run(m, ptr, True, nb, True, True, 0, cuda_dev)
        try:
            for lead, discard in ((0, 0), (nc, 0), (default_lead, 1)):
                assert lib.kgpu_fused_forward_options(lead, discard) == 0
                got, st_got, n = _run(m, ptr, True, nb, True, True, 1, cuda_dev)
                assert n == 1
                assert np.array_equal(got, ref), f"lead {lead} discard {discard}"
                assert np.array_equal(st_got, st_ref)
        finally:
            lib.kgpu_fused_forward_options(default_lead, 0)
    finally:
        m.close()


def test_fused_two_masters_two_streams(cuda_dev):
    """two masters launched on two streams at once: each launch's counters are its master's own"""
    from ka9q_radio_b200 import capi

    nb, b0 = 6, 1
    ms = [capi.Master(L, M, REAL) for _ in range(2)]
    streams = [torch.cuda.Stream(cuda_dev) for _ in range(2)]
    try:
        xs = [torch.from_numpy(_input(nb, b0, True, seed=11 + k)).to(cuda_dev) for k in range(2)]
        ptrs = [x.data_ptr() + b0 * L * 2 for x in xs]
        refs = [_run(ms[k], ptrs[k], True, nb, False, True, 0, cuda_dev) for k in range(2)]
        specs, stats = [], []
        torch.cuda.synchronize()
        for k in range(2):
            buf = torch.full((nb, 2 * ms[k].spec_stride), NAN_BITS, dtype=torch.int32, device=cuda_dev)
            st = torch.zeros((nb, 2), dtype=torch.int64, device=cuda_dev)
            specs.append(buf)
            stats.append(st)
        for rep in range(3):  # back-to-back launches on both streams, interleaved on the host
            for k in range(2):
                ms[k].forward(ptrs[k], capi.KGPU_FMT_I16, 1 / 3000, nb, specs[k].data_ptr(), streams[k].cuda_stream,
                              derandomize=False, d_stats=stats[k].data_ptr())
        torch.cuda.synchronize()
        for k in range(2):
            got = specs[k].cpu().numpy()
            assert np.array_equal(got, refs[k][0][1:nb + 1]), f"master {k}"
            assert np.array_equal(stats[k].cpu().numpy(), refs[k][1])
    finally:
        for m in ms:
            m.close()


@pytest.mark.parametrize("off", [4, 8])
def test_unaligned_input_runs_the_pair(cuda_dev, off):
    from ka9q_radio_b200 import capi

    lib = capi.load()
    nb, b0 = 2, 1
    m = capi.Master(L, M, REAL)
    try:
        x = torch.from_numpy(_input(nb, b0, True, seed=off)).to(cuda_dev)
        ptr = x.data_ptr() + b0 * L * 2 + off
        assert lib.kgpu_fused_forward_fits(L, M, REAL, capi.KGPU_FMT_I16, ptr) == 0
        got, st_got, n = _run(m, ptr, True, nb, True, True, 1, cuda_dev)
        ref, st_ref, _ = _run(m, ptr, True, nb, True, True, 0, cuda_dev)
        assert n == 2, "an input without a tensor map must run the two-kernel pair"
        assert np.array_equal(got, ref) and np.array_equal(st_got, st_ref)
    finally:
        m.close()
