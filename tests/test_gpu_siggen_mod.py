"""The modulated signal generator on the device: sig_gen.c's AM and DSB sources (kgpu_siggen_generate_mod) and a master
that generates them through filter.h (filter_siggen_modulate, filter_siggen_mod_pointer, write_genfilter).

The kernel is compared with the reference's own proc_sig_gen AM loop (oracle/_ref/libka9qsiggenmod.so) over more than
1e8 samples at cfg-2's geometry, in launches of 1 to 3 blocks: bitwise on a 0 Hz carrier (whose phasor stays exactly 1,
so every product of the modulation is pinned), within 1 ulp (or the absolute bound of tests/test_siggen_mod_cpu.py) on
a real one.  A modulated master is compared with the same library fed the restatement's floats (tests/siggen_mod_ref.py)
through write_rfilter / write_cfilter, bitwise on the 0 Hz carrier, and with the reference's own filter.c fed the
reference loop's floats (within TOL).  tests/abi/siggen_mod_driver.c is the filter.h driver; its build against the
reference's own header declares the extensions itself, as a patched radiod would.
"""
import ctypes as C

import numpy as np
import pytest

import siggen_mod_ref as SM
import siggen_ref as S
from test_gpu_raw_ingest import same
from test_gpu_siggen import Gen, _gdriver
from test_siggen_cpu import ABS_FLOOR, RATE
from test_siggen_mod_cpu import envelope, mod_oracle, ref_run_mod, script_mod, ulp_ok

TOL = 1e-5
NOISE = 10 ** (-30 / 20)
AMP = 10 ** (-10 / 20)
SCALE = 1.0 / (32768 * 1.7)
CFG2_L, CFG2_M = 2592000, 648001


def _mdriver(name="siggen_mod_driver.so"):
    lib = _gdriver(name)
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.sgm_modulate.argtypes = [vp, d]
    lib.sgm_has_pointer.argtypes = [vp]
    lib.sgm_write.argtypes = [vp, vp, i, d]
    lib.sgm_write_from_thread.argtypes = [vp, vp, i, i, d]
    return lib


class ModGen(Gen):
    def modulate(self, dc):
        return self.lib.sgm_modulate(self.h, dc)

    def mod(self, env, scale):
        env = np.ascontiguousarray(env, np.float32)
        return self.lib.sgm_write(self.h, env.ctypes.data, len(env), scale)


# ------------------------------------------------------------------ the kernel against the reference's loop -----------
@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("carrier", [0.0, 123456789.0], ids=["dc_carrier", "carrier"])
def test_kernel_against_reference_loop_cfg2(cuda_dev, cplx, carrier):
    """AM, 1.04e8 samples (pairs) at L = 2592000, M = 648001 in launches of 1, 2, 3, 1, ... blocks, each window generated
    from its M - 1 history samples on: bitwise proc_sig_gen's floats on the 0 Hz carrier, within 1 ulp on 123.46 MHz;
    the first window's history before the stream 0.0; the first launches' block energies within 1e-12 of the
    restatement's."""
    import torch

    from ka9q_radio_b200 import capi

    lib = mod_oracle()
    L, M, c = CFG2_L, CFG2_M, 2 if cplx else 1
    nb = 40
    total = nb * L + 17
    sizes = np.full(total // 16000 + 1, 16000)
    sizes[-1] = total - 16000 * (len(sizes) - 1)
    env = np.sin(2 * np.pi * np.arange(total) / 4801.0).astype(np.float32) * np.float32(0.9)
    env[1000:1300] = -1.0
    want, _ = ref_run_mod(lib, cplx, 1, carrier, AMP, NOISE, sizes, sizes, np.full(len(sizes), SCALE), env)
    g = capi.Siggen(capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, carrier / RATE, AMP, NOISE)
    g.modulate(1.0)
    F = g.angles()[0]
    d_env = torch.from_numpy(env).to(cuda_dev)
    span_max = 2 * L + L + M - 1
    buf = torch.empty(c * span_max, dtype=torch.float32, device=cuda_dev)
    mod = torch.zeros(span_max, dtype=torch.float32, device=cuda_dev)
    en = torch.empty(3, dtype=torch.float64, device=cuda_dev)
    blk, k = 0, 1
    while blk < nb:
        k = min(k, nb - blk)
        a0 = blk * L - (M - 1)
        span = (k - 1) * L + L + M - 1
        lo = max(a0, 0)
        mod.fill_(float("nan"))   # the entries before the stream are not read
        mod[lo - a0:span].copy_(d_env[lo:a0 + span])
        buf.fill_(float("nan"))
        g.generate_mod(a0, span, SCALE, buf.data_ptr(), mod.data_ptr(), en.data_ptr(), k, L)
        got = buf[:c * span].cpu().numpy()
        ref = np.concatenate([np.zeros(c * (lo - a0), np.float32), want[c * lo:c * (a0 + span)]])
        if carrier:
            assert ulp_ok(got, ref, ABS_FLOOR * AMP * 1.9 * SCALE).all(), blk
        else:
            assert same(got, ref), blk
        if blk < 4 and (not carrier or blk == 0):   # the restated carrier is slow: the first launches
            _, samp = SM.generate_mod(cplx, blk * L, k * L, AMP, NOISE, SCALE, 1.0, env[blk * L:(blk + k) * L], F=F)
            e = en.cpu().numpy()
            for j in range(k):
                s = samp[c * j * L:c * (j + 1) * L]
                r = float(np.sum(s * s))
                assert abs(e[j] - r) <= 1e-12 * r, (blk, j)
        blk += k
        k = k % 3 + 1
    g.close()


@pytest.mark.gpu
def test_kernel_rejections(cuda_dev):
    """a modulated generator takes kgpu_siggen_generate_mod only, a CW one kgpu_siggen_generate only; dc must be finite"""
    import torch

    from ka9q_radio_b200 import capi

    out = torch.empty(1000, device=cuda_dev)
    mod = torch.zeros(1000, device=cuda_dev)
    g = capi.Siggen(capi.KGPU_REAL, 0.0, AMP, NOISE)
    with pytest.raises(capi.KgpuError):
        g.generate_mod(0, 1000, SCALE, out.data_ptr(), mod.data_ptr())
    with pytest.raises(capi.KgpuError):
        g.modulate(float("nan"))
    g.modulate(0.0)
    with pytest.raises(capi.KgpuError):
        g.generate(0, 1000, SCALE, out.data_ptr())
    with pytest.raises(capi.KgpuError):
        g.generate_mod(0, 1000, SCALE, out.data_ptr(), 0)
    g.generate_mod(0, 1000, SCALE, out.data_ptr(), mod.data_ptr())
    want, _ = SM.generate_mod(False, 0, 1000, AMP, NOISE, SCALE, 0.0, np.zeros(1000, np.float32))
    assert same(out.cpu().numpy(), want)
    g.close()


# ------------------------------------------------------------------ a modulated master through filter.h --------------
# (name, L, M, COMPLEX): cfg-1's sig_gen (2.4 MS/s REAL) and a COMPLEX front end of the same size
MASTERS = [("real_cfg1", 48000, 12001, False), ("complex", 40000, 10001, True)]
CHANS = [(480, -0.4, 0.4, 11.0, 2000), (960, -0.3, 0.3, 9.0, -12345)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L,M,cplx", MASTERS, ids=[m[0] for m in MASTERS])
@pytest.mark.parametrize("am,carrier", [(1, 0.0), (0, 0.0), (1, 7.77e6)], ids=["am_dc", "dsb_dc", "am_carrier"])
@pytest.mark.parametrize("driver", ["siggen_mod_driver.so", "siggen_mod_driver_refhdr.so"])
def test_modulated_master_through_filter_h(oracle, cuda_dev, driver, name, L, M, cplx, am, carrier):
    """Iterations of uneven blocksizes whose reads are short or empty, with scale changes, the host float ring filled
    with NaN after setup: channel outputs, fine-tuned outputs and their powers, noise estimates, the first window's
    spectrum and the wideband analyzer are bitwise those of the same library fed the restatement's floats on the 0 Hz
    carrier (within 1e-5 on a real one), and the channels are within TOL of the reference's own filter.c fed its own AM /
    DSB loop's floats; filter_siggen_stats counts every block once with its energy within 1e-12 of the restatement's."""
    lib = _mdriver(driver)
    c = 2 if cplx else 1
    total = 9 * L + L // 3
    sizes, reads, scales = script_mod(total, seed=L + am + int(carrier))
    env = envelope(total, seed=L, large=False)   # large envelope values are the CPU suite's: here they would overflow powers
    flo, _ = ref_run_mod(mod_oracle(), cplx, am, carrier, AMP, NOISE, sizes, reads, scales, env, L=L, M=M)
    F = S.angle128(carrier / RATE) if carrier else 0
    rst, samp = SM.generate_mod(cplx, 0, total, AMP, NOISE, np.repeat(scales, reads), float(am), env, F=F)
    if cplx:
        flo, rst = flo.view(np.complex64), rst.view(np.complex64)
    check_ref = driver == "siggen_mod_driver.so" and oracle.ref_available()
    ref = oracle.RefSession(L, M, oracle.KO_COMPLEX if cplx else oracle.KO_REAL) if check_ref else None
    fft_n, bins = 4000, 1000
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    try:
        with ModGen(lib, L, M, cplx) as a, Gen(lib, L, M, cplx) as b:
            assert a.setup(carrier, AMP, NOISE) == 0
            assert lib.sgm_has_pointer(a.h) == 0
            assert a.modulate(float(am)) == 0 and lib.sgm_has_pointer(a.h) == 1
            lib.sg_fill_host_ring(a.h, float("nan"))
            assert a.gstats() == (0, 0, 0.0)
            for s in (a, b):
                for olen, lo, hi, beta, _ in CHANS:
                    s.add(olen, lo, hi, beta)
                s.lib.rd_enable_noise(s.h, 2.4e6)
                s.spec_setup(fft_n, bins, window)
            if ref is not None:
                for olen, lo, hi, beta, _ in CHANS:
                    ref.add_channel(olen, lo, hi, beta)
            pos, fired, energy = 0, 0, 0.0
            for k, n in enumerate(reads):
                n = int(n)
                fa = a.mod(env[pos:pos + n], scales[k])
                assert fa == b.flt(rst[pos:pos + n]), k
                if ref is not None:
                    assert ref.write(flo[pos:pos + n]) == fa, k
                pos += n
                if fa != 1:
                    continue
                now = pos // L
                for ch, (*_, shift) in enumerate(CHANS):
                    if ch == 0:
                        ya, pa = a.tuned(ch, shift, 1234.5, 48000.0)
                        yb, pb = b.tuned(ch, shift, 1234.5, 48000.0)
                    else:
                        ya, yb = a.exe(ch, shift), b.exe(ch, shift)
                        pa = pb = 0.0
                    assert np.isfinite(ya).all()
                    if carrier:
                        assert np.abs(ya - yb).max() <= 1e-5 * np.abs(yb).max(), (k, ch)
                    else:
                        n0 = [lib.rd_noise(s.h, ch) for s in (a, b)]   # NaN for a block recomputed alone after a retune
                        assert same(ya, yb) and pa == pb and np.array_equal(n0[:1], n0[1:], equal_nan=True), (k, ch)
                    if ref is not None and ch == 1:
                        r = ref.execute(ch, shift)
                        assert np.abs(ya - r).max() / np.abs(r).max() < TOL, (k, ch)
                (ga, ea), (gb, eb) = a.spec_poll(0 if cplx else 750, 3, 0.5, bins), b.spec_poll(0 if cplx else 750, 3, 0.5, bins)
                assert ea == eb and np.isfinite(ga).all()
                assert same(ga, gb) if not carrier else np.abs(ga - gb).max() <= 1e-4 * np.abs(gb).max()
                if fired == 0:   # the first window: M - 1 samples of zero history before the first write
                    fa_, fb_ = np.empty(L + M, np.complex64), np.empty(L + M, np.complex64)
                    na, nb_ = lib.rd_fdomain(a.h, 0, fa_.ctypes.data), lib.rd_fdomain(b.h, 0, fb_.ctypes.data)
                    assert na == nb_ and (same(fa_[:na], fb_[:na]) or carrier)
                st = a.gstats()
                assert st[0] <= now - fired and st[1] == st[0] * L
                fired += st[0]
                energy += st[2]
            while fired < pos // L:   # the last blocks' energies, once their work is done
                st = a.gstats()
                fired += st[0]
                energy += st[2]
            want = float(np.sum(samp[:c * fired * L] ** 2))
            assert fired == pos // L and abs(energy - want) <= 1e-12 * want
    finally:
        if ref is not None:
            ref.close()


@pytest.mark.gpu
def test_lapped_slave_retune_and_batch_on_a_modulated_master(cuda_dev):
    """A consumer ND blocks behind a modulated master gets zeros and a drop; a retune recomputes the block alone; the
    batch call serves it; all as on a master fed the same floats."""
    lib = _mdriver()
    L, M = 40000, 10001
    env = envelope(8 * L, seed=5, large=False)
    flo, _ = SM.generate_mod(True, 0, 8 * L, AMP, NOISE, SCALE, 0.0, env)
    flo = flo.view(np.complex64)
    with ModGen(lib, L, M, True, nworkers=1) as a, Gen(lib, L, M, True, nworkers=1) as b:
        assert a.setup(0.0, AMP, NOISE) == 0 and a.modulate(0.0) == 0
        for s in (a, b):
            s.add(480, -0.3, 0.3, 9.0)
        assert lib.sgm_write_from_thread(a.h, env.ctypes.data, L, 6, SCALE) == 0
        assert lib.rd_write_from_thread(b.h, flo.ctypes.data, L, 6, 8 * L, 0, 0, 0.0) == 0
        for shift in (1500, 1500, -700):
            assert same(a.exe(0, shift), b.exe(0, shift))
        ya, yb = np.empty(480, np.complex64), np.empty(480, np.complex64)
        assert lib.sg_execute_batch(a.h, 0, -700, ya.ctypes.data) == lib.sg_execute_batch(b.h, 0, -700, yb.ctypes.data) == 0
        assert same(ya, yb)
        assert lib.rd_drops(a.h, 0) == lib.rd_drops(b.h, 0) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
def test_analyzer_set_up_after_blocks_regenerates_its_ring(cuda_dev, cplx):
    """the wideband analyzer set up after several blocks of a modulated master: its device ring is generated again from
    the envelope ring (the host float ring holds nothing), and its bins are bitwise those of a master fed the same
    floats"""
    lib = _mdriver()
    L, M, fft_n, bins = 48000, 12001, 6000, 1500
    sizes = np.full(6 * L // 30000, 30000)
    n = int(sizes.sum())
    scales = np.where(np.arange(len(sizes)) == 3, SCALE * 2, SCALE)
    env = envelope(n, seed=7, large=False)
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    flo, _ = SM.generate_mod(cplx, 0, n, AMP, NOISE, np.repeat(scales, sizes), 1.0, env)
    if cplx:
        flo = flo.view(np.complex64)
    with ModGen(lib, L, M, cplx) as a, Gen(lib, L, M, cplx) as b:
        assert a.setup(0.0, AMP, NOISE) == 0 and a.modulate(1.0) == 0
        lib.sg_fill_host_ring(a.h, float("nan"))
        for k, m in enumerate(sizes):
            assert a.mod(env[k * 30000:(k + 1) * 30000], scales[k]) == b.flt(flo[k * 30000:(k + 1) * 30000])
            if k == 5:
                a.spec_setup(fft_n, bins, window)
                b.spec_setup(fft_n, bins, window)
            if k >= 5:
                shift = 0 if cplx else 750
                (ga, ea), (gb, eb) = a.spec_poll(shift, 3, 0.5, bins), b.spec_poll(shift, 3, 0.5, bins)
                assert ea == eb and same(ga, gb) and np.abs(ga).max() > 0, k


@pytest.mark.gpu
def test_siggen_mod_rejections(cuda_dev):
    lib = _mdriver()
    z = np.zeros(4096, np.int16)
    e = np.zeros(16, np.float32)
    with ModGen(lib, 48000, 12001, False) as s:
        assert s.modulate(1.0) == -1                            # not generated
        assert lib.sgm_has_pointer(s.h) == 0
        assert s.setup(0.0, AMP, NOISE) == 0
        assert lib.sgm_has_pointer(s.h) == 0                    # CW: no envelope
        assert s.modulate(float("inf")) == -1 and s.modulate(float("nan")) == -1
        assert s.modulate(0.0) == 0 and s.modulate(1.0) == 0    # before the first write, dc may still change
        assert s.setup(0.0, AMP, NOISE) == -1                   # set up twice
        assert s.flt(e) == -1                                   # floats on a generated master
        assert s.i16(z[:16], 1.0) == -1                         # int16
        assert s.raw(z, 16, 6) == -1                            # raw words
        assert s.stats() is None                                # filter_ingest_stats: not an ingest master
        assert s.mod(e, SCALE) == 0
        assert s.modulate(0.0) == -1                            # after the first write
        assert lib.sgm_has_pointer(s.h) == 1
    with ModGen(lib, 40000, 10001, True) as s:
        assert s.setup(0.0, AMP, NOISE) == 0 and s.gen(16, SCALE) == 0
        assert s.modulate(1.0) == -1                            # a CW master already written
        assert s.flt(e.view(np.complex64)) == -1                # write_cfilter
