"""The signal generator on the device: sig_gen.c's CW source (kgpu_siggen_generate) and a master that generates its own
input through filter.h (filter_siggen_setup, write_genfilter, filter_siggen_stats).

The kernel is compared with the reference's own proc_sig_gen loop (oracle/_ref/libka9qsiggen.so) over more than 1e8
samples at cfg-2's geometry, in launches of 1 to 3 blocks: bitwise for noise, within 1 ulp (or 1e-11 of the full scale
next to zero, see tests/test_siggen_cpu.py) for a carrier with noise.  A generated master is compared with the same
library fed that loop's floats through write_rfilter / write_cfilter (bitwise for noise) and with the reference's own
filter.c fed them (within TOL).  tests/abi/siggen_driver.c is the filter.h driver; its build against the reference's own
header declares the extensions itself, as a patched radiod would.
"""
import ctypes as C

import numpy as np
import pytest

import siggen_ref as S
from test_gpu_raw_ingest import Session, _driver, same
from test_siggen_cpu import RATE, oracle as siggen_oracle, ref_run, script, ulp_ok

TOL = 1e-5
NOISE = 10 ** (-30 / 20)
AMP = 10 ** (-10 / 20)
SCALE = 1.0 / (32768 * 1.7)
CFG2_L, CFG2_M = 2592000, 648001


def _gdriver(name="siggen_driver.so"):
    lib = _driver(name)
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.sg_setup.argtypes = [vp, d, d, d, d, C.c_uint64]
    lib.sg_write.argtypes = [vp, i, d]
    lib.sg_stats.argtypes = [vp, vp, vp]
    lib.sg_fill_host_ring.argtypes = [vp, C.c_float]
    lib.sg_write_from_thread.argtypes = [vp, i, i, d]
    lib.sg_execute_batch.argtypes = [vp, i, i, vp]
    lib.rd_fdomain.argtypes = [vp, C.c_uint, vp]
    return lib


class Gen(Session):
    def setup(self, carrier, amplitude, noise, seed=1):
        return self.lib.sg_setup(self.h, carrier / RATE, 0.0, amplitude, noise, seed)

    def gen(self, n, scale):
        return self.lib.sg_write(self.h, n, scale)

    def gstats(self):
        out, e = (C.c_uint64 * 2)(), C.c_double(0)
        if self.lib.sg_stats(self.h, C.cast(out, C.c_void_p), C.byref(e)) != 0:
            return None
        return int(out[0]), int(out[1]), e.value


# ------------------------------------------------------------------ the kernel against the reference's loop -----------
@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True], ids=["real", "complex"])
@pytest.mark.parametrize("carrier", [0.0, 123456789.0], ids=["noise", "carrier"])
def test_kernel_against_reference_loop_cfg2(cuda_dev, cplx, carrier):
    """1.04e8 samples (pairs) at L = 2592000, M = 648001 in launches of 1, 2, 3, 1, ... blocks, each window generated
    from its M - 1 history samples on: noise bitwise proc_sig_gen's floats, a carrier with noise within 1 ulp; the first
    window's history before the stream 0.0; the block energies of the first launches within 1e-12 of the restatement's."""
    import torch

    from ka9q_radio_b200 import capi

    lib = siggen_oracle()
    L, M, c = CFG2_L, CFG2_M, 2 if cplx else 1
    amp = AMP if carrier else 0.0
    nb = 40
    total = nb * L + 17
    sizes = np.full(total // 16000 + 1, 16000)
    sizes[-1] = total - 16000 * (len(sizes) - 1)
    want, _ = ref_run(lib, cplx, carrier, amp, NOISE, sizes, np.full(len(sizes), SCALE))
    g = capi.Siggen(capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, carrier / RATE, amp, NOISE)
    F = g.angles()[0]
    buf = torch.empty(c * (2 * L + L + M - 1), dtype=torch.float32, device=cuda_dev)
    en = torch.empty(3, dtype=torch.float64, device=cuda_dev)
    blk, k = 0, 1
    while blk < nb:
        k = min(k, nb - blk)
        a0 = blk * L - (M - 1)
        span = (k - 1) * L + L + M - 1
        buf.fill_(float("nan"))
        g.generate(a0, span, SCALE, buf.data_ptr(), en.data_ptr(), k, L)
        got = buf[:c * span].cpu().numpy()
        lo = max(a0, 0)
        ref = np.concatenate([np.zeros(c * (lo - a0), np.float32), want[c * lo:c * (a0 + span)]])
        if carrier:
            assert ulp_ok(got, ref, amp * SCALE).all(), blk
        else:
            assert same(got, ref), blk
        if blk < 4 and (not carrier or blk == 0):   # the restated carrier is slow: the first launch
            _, samp = S.generate(cplx, blk * L, k * L, amp, NOISE, SCALE, F=F)
            e = en.cpu().numpy()
            for j in range(k):
                s = samp[c * j * L:c * (j + 1) * L]
                r = float(np.sum(s * s))
                assert abs(e[j] - r) <= 1e-12 * r, (blk, j)
        blk += k
        k = k % 3 + 1
    g.close()


@pytest.mark.gpu
def test_kernel_scale_changes_and_rejections(cuda_dev):
    """two scale changes inside a window (one in the history) give each sample its own scale; bad arguments fail"""
    import torch

    from ka9q_radio_b200 import capi

    g = capi.Siggen(capi.KGPU_REAL, 0.0, 0.0, NOISE)
    L, hist, a0, k = 1000, 333, 5_000_000, 3
    n = hist + k * L
    chg = np.array([(a0 + hist // 2, SCALE * 0.5), (a0 + hist + L // 3, SCALE * 3)], dtype=[("at", "<i8"), ("scale", "<f8")])
    d_chg = torch.from_numpy(chg.view(np.uint8).copy()).to(cuda_dev)
    out = torch.empty(n, device=cuda_dev)
    g.generate(a0, n, SCALE, out.data_ptr(), nblocks=k, L=L, d_chg=d_chg.data_ptr(), nchg=2)
    samp = a0 + np.arange(n)
    sc = np.where(samp >= chg[1]["at"], chg[1]["scale"], np.where(samp >= chg[0]["at"], chg[0]["scale"], SCALE))
    want, _ = S.generate(False, a0, n, 0.0, NOISE, sc)
    assert same(out.cpu().numpy(), want)
    with pytest.raises(capi.KgpuError):
        g.generate(-hist - 1, n, SCALE, out.data_ptr(), nblocks=k, L=L)   # zeros reaching into a block
    with pytest.raises(capi.KgpuError):
        g.generate(0, 100, SCALE, out.data_ptr(), nblocks=1, L=50, history=50)   # L below one thread's run
    g.close()


# ------------------------------------------------------------------ a generated master through filter.h --------------
# (name, L, M, COMPLEX): cfg-1's sig_gen (2.4 MS/s REAL) and a COMPLEX front end of the same size
MASTERS = [("real_cfg1", 48000, 12001, False), ("complex", 40000, 10001, True)]
CHANS = [(480, -0.4, 0.4, 11.0, 2000), (960, -0.3, 0.3, 9.0, -12345)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L,M,cplx", MASTERS, ids=[m[0] for m in MASTERS])
@pytest.mark.parametrize("carrier", [0.0, 7.77e6], ids=["noise", "carrier"])
@pytest.mark.parametrize("driver", ["siggen_driver.so", "siggen_driver_refhdr.so"])
def test_generated_master_through_filter_h(oracle, cuda_dev, driver, name, L, M, cplx, carrier):
    """Writes of the CPU suite's scripted sizes with scale changes, the host float ring filled with NaN after setup:
    channel outputs, fine-tuned outputs and their powers, noise estimates, the first window's spectrum and the wideband
    analyzer are bitwise those of the same library fed proc_sig_gen's floats for noise, and the channels are within TOL
    of the reference's own filter.c fed them; filter_siggen_stats counts every block once with its energy within 1e-12
    of the restatement's."""
    lib = _gdriver(driver)
    c = 2 if cplx else 1
    total = 9 * L + L // 3
    sizes, scales = script(total, seed=L + int(carrier))
    amp = AMP if carrier else 0.0
    flo, _ = ref_run(siggen_oracle(), cplx, carrier, amp, NOISE, sizes, scales, L=L, M=M)
    _, samp = S.generate(cplx, 0, total, amp, NOISE, 1.0, F=S.angle128(carrier / RATE) if carrier else 0)
    if cplx:
        flo = flo.view(np.complex64)
    check_ref = driver == "siggen_driver.so" and oracle.ref_available()
    ref = oracle.RefSession(L, M, oracle.KO_COMPLEX if cplx else oracle.KO_REAL) if check_ref else None
    fft_n, bins = 4000, 1000
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    try:
        with Gen(lib, L, M, cplx) as a, Session(lib, L, M, cplx) as b:
            assert a.setup(carrier, amp, NOISE) == 0
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
            for k, n in enumerate(sizes):
                fa = a.gen(int(n), scales[k])
                assert fa == b.flt(flo[pos:pos + n]), k
                if ref is not None:
                    assert ref.write(flo[pos:pos + n]) == fa, k
                pos += int(n)
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
def test_lapped_slave_retune_and_batch_on_a_generated_master(cuda_dev):
    """A consumer ND blocks behind a generated master gets zeros and a drop; a retune recomputes the block alone; the
    batch call serves it; all as on a master fed the same floats."""
    lib = _gdriver()
    L, M = 40000, 10001
    flo, _ = ref_run(siggen_oracle(), True, 0.0, 0.0, NOISE, np.full(8, L), np.full(8, SCALE), L=L, M=M)
    flo = flo.view(np.complex64)
    with Gen(lib, L, M, True, nworkers=1) as a, Session(lib, L, M, True, nworkers=1) as b:
        assert a.setup(0.0, 0.0, NOISE) == 0
        for s in (a, b):
            s.add(480, -0.3, 0.3, 9.0)
        assert lib.sg_write_from_thread(a.h, L, 6, SCALE) == 0
        assert lib.rd_write_from_thread(b.h, flo.ctypes.data, L, 6, 8 * L, 0, 0, 0.0) == 0
        for shift in (1500, 1500, -700):
            assert same(a.exe(0, shift), b.exe(0, shift))
        ya, yb = np.empty(480, np.complex64), np.empty(480, np.complex64)
        assert lib.sg_execute_batch(a.h, 0, -700, ya.ctypes.data) == lib.sg_execute_batch(b.h, 0, -700, yb.ctypes.data) == 0
        assert same(ya, yb)
        assert lib.rd_drops(a.h, 0) == lib.rd_drops(b.h, 0) >= 1


@pytest.mark.gpu
def test_analyzer_set_up_after_blocks_regenerates_its_ring(cuda_dev):
    """the wideband analyzer set up after several blocks of a generated master: its device ring is generated again (the
    host ring holds nothing), and its bins are bitwise those of a master fed the same floats"""
    lib = _gdriver()
    L, M, fft_n, bins = 48000, 12001, 6000, 1500
    n = 6 * L
    sizes = np.full(n // 30000, 30000)
    scales = np.where(np.arange(len(sizes)) == 3, SCALE * 2, SCALE)
    flo, _ = ref_run(siggen_oracle(), False, 0.0, 0.0, NOISE, sizes, scales, L=L, M=M)
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    with Gen(lib, L, M, False) as a, Session(lib, L, M, False) as b:
        assert a.setup(0.0, 0.0, NOISE) == 0
        lib.sg_fill_host_ring(a.h, float("nan"))
        for k, m in enumerate(sizes):
            assert a.gen(int(m), scales[k]) == b.flt(flo[k * 30000:(k + 1) * 30000])
            if k == 5:
                a.spec_setup(fft_n, bins, window)
                b.spec_setup(fft_n, bins, window)
            if k >= 5:
                (ga, ea), (gb, eb) = a.spec_poll(750, 3, 0.5, bins), b.spec_poll(750, 3, 0.5, bins)
                assert ea == eb and same(ga, gb) and np.abs(ga).max() > 0, k


@pytest.mark.gpu
def test_siggen_rejections(cuda_dev):
    lib = _gdriver()
    z = np.zeros(4096, np.int16)
    with Gen(lib, 48000, 12001, False) as s:
        assert s.gstats() is None                               # not generated
        assert s.gen(16, 1.0) == -1
        assert s.setup(0.0, 0.0, NOISE) == 0
        assert s.setup(0.0, 0.0, NOISE) == -1                   # twice
        assert s.flt(np.zeros(16, np.float32)) == -1            # floats on a generated master
        assert s.i16(z[:16], 1.0) == -1                         # int16
        assert s.raw(z, 16, 6) == -1                            # raw words
        assert s.stats() is None                                # filter_ingest_stats: not an ingest master
        assert s.gen(16, 1.0) == 0
    with Gen(lib, 48000, 12001, False) as s:
        assert s.flt(np.zeros(16, np.float32)) == 0
        assert s.setup(0.0, 0.0, NOISE) == -1                   # already fed floats
    with Gen(lib, 48000, 12001, True) as s:
        assert s.raw(z, 16, 6) == 0
        assert s.setup(0.0, 0.0, NOISE) == -1                   # already fed raw words
    with Gen(lib, 48000, 12001, True) as s:
        assert s.i16(z[:32], 1.0) == 0
        assert s.setup(0.0, 0.0, NOISE) == -1                   # already fed int16
