"""Which kernels each channel path launches: the kgpu_launch_count of a response (kgpu_bank_set_filter) and of a
one-block run without and with block power, for one channel of each path in a bank of its own.

The master is COMPLEX with N / L = 5 / 4 (L = 48000, M = 12001), so points = 5 olen / 4 and set_filter designs real
taps for every length.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

L, M = 48000, 12001

# (olen, points, chan_plan path, launches of: a run, a run with d_power, a response)
CASES = {
    "direct_600": (480, 600, "CHAN_DIRECT", 1, 1, 1),
    "wide_9600": (7680, 9600, "CHAN_WIDE", 1, 1, 1),
    "huge_38400": (30720, 38400, "CHAN_HUGE", 2, 3, 2),
    "extended_5500": (4400, 5500, "CHAN_EXTENDED", 1, 1, 1),
    "extended_13860": (11088, 13860, "CHAN_EXTENDED", 1, 1, 1),
    "bluestein_725": (580, 725, "CHAN_BLUESTEIN", 7, 8, 7),
    "bluestein_44000": (35200, 44000, "CHAN_BLUESTEIN", 7, 8, 7),
}


@pytest.mark.parametrize("case", list(CASES))
def test_launches_per_path(cuda_dev, case):
    from ka9q_radio_b200 import capi

    olen, points, path, run, run_power, response = CASES[case]
    assert capi.chan_plan(points)[0] == getattr(capi, path), (points, capi.chan_plan(points))
    lib = capi.load()
    m = capi.Master(L, M, capi.KGPU_COMPLEX)
    b = capi.Bank(m, 1)
    try:
        assert m.N * olen % L == 0 and b.define_any(0, olen) == points

        def launches(fn):
            before = lib.kgpu_launch_count()
            fn()
            torch.cuda.synchronize()
            return lib.kgpu_launch_count() - before

        spec = torch.zeros(m.spec_stride, dtype=torch.complex64, device=cuda_dev)
        out = torch.empty(b.out_stride, dtype=torch.complex64, device=cuda_dev)
        power = torch.empty(1, dtype=torch.float32, device=cuda_dev)
        got = (launches(lambda: b.set_filter(0, -0.1, 0.1, 11.0)),
               launches(lambda: b.run(spec.data_ptr(), 1, out.data_ptr())),
               launches(lambda: b.run(spec.data_ptr(), 1, out.data_ptr(), d_power=power.data_ptr())))
        assert got == (response, run, run_power), (case, got)
    finally:
        b.close()
        m.close()


def test_static_kernel_on_two_devices(cuda_dev):
    """A 1200-point bank (chan_static, about 77 kB of dynamic shared memory) run on device 0 and then on device 1 in one
    process: each device needs the kernel's shared-memory attribute of its own, and both compute the same output."""
    import numpy as np
    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    lib = capi.load()
    lib.kgpu_use_static_kernels(1)
    x = np.random.default_rng(1200).standard_normal(3 * L, dtype=np.float32)
    outs = []
    try:
        for dev in (torch.device("cuda:0"), torch.device("cuda:1")):
            cz = Channelizer(L, M, capi.KGPU_REAL, dev, capacity=2)
            try:
                assert cz.add_channel(960, 3000, -0.4, 0.4, 7.0) == 0 and cz._olen[0][1] == 1200
                spec, out = cz.alloc_spectra(3), cz.alloc_outputs(3)
                cz.forward(cz.stage_stream(x), 3, spec)
                out.zero_()
                cz.channels(spec, 3, out)
                torch.cuda.synchronize(dev)
                outs.append(cz.channel_slice(out, 0).cpu().numpy())
            finally:
                cz.close()
    finally:
        capi.check(lib.kgpu_set_device(0), "kgpu_set_device")
        torch.cuda.set_device(cuda_dev)
    assert np.abs(outs[0]).max() > 0
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32))
