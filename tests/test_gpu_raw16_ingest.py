"""Raw 16-bit ingest on the device: HydraSDR INT16_REAL / UINT16_REAL / INT16_IQ, bladeRF SC16 Q11 and SDRplay's planar
int16 I/Q (write_rawfilter, write_rawfilter_planar) and their A/D statistics (filter_ingest_stats).

Every format gives exactly the floats the drivers' loops store, so a master fed raw words is compared bitwise with the
same library fed the restated floats (tests/raw16_ingest_ref.py, pinned against the reference's own hydrasdr.c and
bladerf.c by tests/test_raw16_ingest_cpu.py) through write_cfilter / write_rfilter, and within TOL with the reference's
own filter.c fed the same floats.  tests/abi/raw16_driver.c is the filter.h driver; its build against the reference's
own header declares the extensions itself, as a patched radiod would.
"""
import ctypes as C

import numpy as np
import pytest

import raw16_ingest_ref as R
from test_gpu_raw_ingest import Session, _driver, same

TOL = 1e-5
SCALE = 1.0 / (32768 * 1.7)   # scale_AD-like double: its float products round differently
GAIN = 10 ** (-6 / 20)        # a gain change between two writes


def _driver16(name="raw16_driver.so"):
    lib = _driver(name)
    lib.rd_write_planar.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_double]
    lib.rd_fdomain.argtypes = [C.c_void_p, C.c_uint, C.c_void_p]
    fm = (C.c_int * 3)()
    lib.rd_raw16_formats(fm)
    assert list(fm) == [R.S16, R.U16, R.SC16Q11]
    return lib


def words16(ncomp, fmt, seed, garbage=False):
    """ncomp components of a 16-bit front end: tones in noise, at both limits now and then; for bladeRF, random bits
    12-15 that the driver ignores"""
    rng = np.random.default_rng(seed)
    t = np.arange(ncomp)
    top = 2047 if fmt == R.SC16Q11 else 32767
    v = 0.5 * top * np.cos(2 * np.pi * 0.0123 * t) + 0.2 * top * np.cos(2 * np.pi * 0.2071 * t) + rng.normal(0, top / 20, ncomp)
    v = np.clip(np.rint(v), -top - 1, top).astype(np.int64)
    v[rng.random(ncomp) < 2e-4] = top
    v[rng.random(ncomp) < 2e-4] = -top - 1
    if fmt == R.SC16Q11:
        w = (v & 0xFFF).astype(np.uint16)
        return w | (rng.integers(0, 16, ncomp) << 12).astype(np.uint16) if garbage else w
    if fmt == R.U16:
        return (v + 32768).astype(np.uint16)
    return v.astype(np.int16).view(np.uint16)


def sizes(total, L, seed):
    """uneven transfer sizes summing to total, from a fortieth of a block to over half of one"""
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while n < total:
        k = int(min(total - n, rng.integers(L // 40, L * 3 // 5)))
        out.append(k)
        n += k
    return out


# ------------------------------------------------------------------ the unpack kernel --------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt,cplx", [(R.S16, False), (R.S16, True), (R.U16, False), (R.SC16Q11, True)])
def test_unpack16_kernel_bitwise_and_block_stats(cuda_dev, fmt, cplx):
    """kgpu_unpack8 on 16-bit words: floats bitwise the restatement's with two scale changes inside the window (one in
    the history), block statistics exact over each block's new samples only (limit words planted in the history are
    never counted)."""
    import torch

    from ka9q_radio_b200 import capi

    kfmt = {R.S16: capi.KGPU_RAW_S16, R.U16: capi.KGPU_RAW_U16, R.SC16Q11: capi.KGPU_RAW_SC16Q11}[fmt]
    c = 2 if cplx else 1
    L, hist, a0 = 1000, 333, 5_000_000
    dt = np.dtype([("energy", "<u8"), ("overs", "<u4"), ("over_samples", "<u4")])
    for k in (1, 2, 3):
        n = hist + k * L
        w = words16(n * c, fmt, seed=k, garbage=fmt == R.SC16Q11)
        top = np.array([0x7FF, 0x800] if fmt == R.SC16Q11 else ([0xFFFF, 0] if fmt == R.U16 else [0x7FFF, 0x8000]), np.uint16)
        w[:64] = np.resize(top, 64)                          # limits in the history, never counted
        chg = np.array([(a0 + hist // 2, SCALE * GAIN), (a0 + hist + L // 3, SCALE * 0.3)], dtype=[("at", "<i8"), ("scale", "<f8")])
        d_w = torch.from_numpy(w.view(np.int16).copy()).to(cuda_dev)
        d_out = torch.full((n * c,), float("nan"), device=cuda_dev)
        d_st = torch.full((k * 16,), 0xA5, dtype=torch.uint8, device=cuda_dev)
        d_chg = torch.from_numpy(chg.view(np.uint8).copy()).to(cuda_dev)
        capi.unpack8(d_w.data_ptr(), kfmt, capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, hist, L, k, SCALE, d_out.data_ptr(),
                     d_st.data_ptr(), d_chg=d_chg.data_ptr(), nchg=2, a0=a0)
        torch.cuda.synchronize()
        samp = a0 + np.arange(n)
        sc = np.where(samp >= chg[1]["at"], chg[1]["scale"], np.where(samp >= chg[0]["at"], chg[0]["scale"], SCALE))
        want = (np.repeat(sc, c) * R.values16(w, fmt).astype(np.float64)).astype(np.float32)
        assert same(d_out.cpu().numpy(), want), k
        got = np.frombuffer(d_st.cpu().numpy().tobytes(), dt)
        assert [(int(g["energy"]), int(g["overs"]), int(g["over_samples"])) for g in got] == \
            R.block_stats(R.values16(w, fmt)[hist * c:], fmt, L, cplx), k


@pytest.mark.gpu
def test_unpack16_rejects_master_types(cuda_dev):
    import torch

    from ka9q_radio_b200 import capi

    d = torch.zeros(4096, dtype=torch.int16, device=cuda_dev)
    out = torch.empty(4096, device=cuda_dev)
    with pytest.raises(capi.KgpuError):
        capi.unpack8(d.data_ptr(), capi.KGPU_RAW_U16, capi.KGPU_COMPLEX, 0, 100, 1, 1.0, out.data_ptr())
    with pytest.raises(capi.KgpuError):
        capi.unpack8(d.data_ptr(), capi.KGPU_RAW_SC16Q11, capi.KGPU_REAL, 0, 100, 1, 1.0, out.data_ptr())
    with pytest.raises(capi.KgpuError):
        capi.unpack8(d.data_ptr() + 1, capi.KGPU_RAW_S16, capi.KGPU_REAL, 0, 100, 1, 1.0, out.data_ptr())


# ------------------------------------------------------------------ the front ends through filter.h ------------------
# (name, L, M, COMPLEX, format, planar): SDRplay 2 MS/s, bladeRF 12 and 61.44 MS/s, HydraSDR int16 REAL 20 MS/s (and its
# uint16 offset form), HydraSDR int16 I/Q 10 MS/s
FRONT_ENDS = [
    ("sdrplay_2m", 40000, 10001, True, R.S16, True),
    ("bladerf_12m", 240000, 60001, True, R.SC16Q11, False),
    ("bladerf_61m44", 1228800, 307201, True, R.SC16Q11, False),
    ("hydrasdr_int16_real_20m", 400000, 100001, False, R.S16, False),
    ("hydrasdr_uint16_real_20m", 400000, 100001, False, R.U16, False),
    ("hydrasdr_int16_iq_10m", 200000, 50001, True, R.S16, False),
]
CHANS = [(480, -0.4, 0.4, 11.0, 2000), (960, -0.3, 0.3, 9.0, -12345)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L,M,cplx,fmt,planar", FRONT_ENDS, ids=[f[0] for f in FRONT_ENDS])
@pytest.mark.parametrize("driver", ["raw16_driver.so", "raw16_driver_refhdr.so"])
def test_front_end_through_filter_h(oracle, cuda_dev, driver, name, L, M, cplx, fmt, planar):
    """Transfers of uneven sizes that straddle blocks and the end of the ring, with a gain change between two of them:
    the channel outputs are bitwise those of the same library fed the restated floats, and within TOL of the reference's
    own filter.c fed them; filter_ingest_stats is exact block by block; the first window's history is zero (its
    spectrum is bitwise the float master's)."""
    lib = _driver16(driver)
    c = 2 if cplx else 1
    nb = 3 if L > 1_000_000 else 7                     # past the end of the ring (ND = 4 windows) but for the largest
    total = nb * L + L // 3
    w = words16(c * total, fmt, seed=L, garbage=fmt == R.SC16Q11)
    x = R.values16(w, fmt)
    base = 1.0 if fmt == R.SC16Q11 else SCALE          # bladerf.c stores (float)x
    parts = sizes(total, L, seed=M)
    gain_at = len(parts) // 2
    check_ref = driver == "raw16_driver.so" and oracle.ref_available()
    ref = oracle.RefSession(L, M, oracle.KO_COMPLEX if cplx else oracle.KO_REAL) if check_ref else None
    want_stats = R.block_stats(x, fmt, L, cplx)
    try:
        with Session(lib, L, M, cplx) as a, Session(lib, L, M, cplx) as b:
            assert a.stats() == (0,) * 6
            for s in (a, b):
                for olen, lo, hi, beta, _ in CHANS:
                    s.add(olen, lo, hi, beta)
            if ref is not None:
                for olen, lo, hi, beta, _ in CHANS:
                    ref.add_channel(olen, lo, hi, beta)
            pos, fired, since = 0, 0, 0
            for k, n in enumerate(parts):
                sc = base * (GAIN if k >= gain_at else 1.0)
                seg = w[c * pos:c * (pos + n)]
                flo = R.unpack16(seg, fmt, sc)
                if cplx:
                    flo = flo.view(np.complex64)
                if planar:
                    iq = seg.view(np.int16)
                    xi, xq = np.ascontiguousarray(iq[0::2]), np.ascontiguousarray(iq[1::2])
                    fa = lib.rd_write_planar(a.h, xi.ctypes.data, xq.ctypes.data, n, sc)
                else:
                    fa = a.raw(seg, n, fmt, sc)
                assert fa == b.flt(flo), k
                if ref is not None:
                    assert ref.write(flo) == fa, k
                pos += n
                if fa != 1:
                    continue
                now = pos // L
                for ch, (*_, shift) in enumerate(CHANS):
                    ya, yb = a.exe(ch, shift), b.exe(ch, shift)
                    assert same(ya, yb), (k, ch)
                    if ref is not None:
                        r = ref.execute(ch, shift)
                        assert np.abs(ya - r).max() / np.abs(r).max() < TOL, (k, ch)
                if fired == 0:   # the first window: M - 1 samples of history before the first write
                    fa_, fb_ = np.empty(L + M, np.complex64), np.empty(L + M, np.complex64)
                    na, nb_ = lib.rd_fdomain(a.h, 0, fa_.ctypes.data), lib.rd_fdomain(b.h, 0, fb_.ctypes.data)
                    assert na == nb_ and same(fa_[:na], fb_[:na])
                got = a.stats()
                blk = want_stats[fired:now]
                for _, _, os in blk:
                    since = 0 if os else since + L
                assert got == (now - fired, (now - fired) * L, sum(s[0] for s in blk), sum(s[1] for s in blk),
                               sum(s[2] for s in blk), since), k
                fired = now
            assert fired == nb and sum(s[1] for s in want_stats[:nb]) > 0
    finally:
        if ref is not None:
            ref.close()


@pytest.mark.gpu
def test_lapped_slave_on_a_raw16_master(cuda_dev):
    """A consumer that fell ND blocks behind an S16-fed master gets a block of zeros and a drop, as one fed floats does."""
    lib = _driver16()
    L, M = 40000, 10001
    w = words16(2 * 8 * L, R.S16, seed=3)
    flo = R.unpack16(w, R.S16, SCALE).view(np.complex64)
    with Session(lib, L, M, True, nworkers=1) as a, Session(lib, L, M, True, nworkers=1) as b:
        for s in (a, b):
            s.add(480, -0.3, 0.3, 9.0)
        assert lib.rd_write_from_thread(a.h, w.ctypes.data, L, 6, 4 * L, 1, R.S16, SCALE) == 0
        assert lib.rd_write_from_thread(b.h, flo.ctypes.data, L, 6, 8 * L, 0, 0, 0.0) == 0
        for _ in range(4):
            assert same(a.exe(0, 1500), b.exe(0, 1500))
        assert lib.rd_drops(a.h, 0) == lib.rd_drops(b.h, 0) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.U16, R.SC16Q11])
@pytest.mark.parametrize("when", ["before", "after"])
def test_wideband_analyzer_on_raw16_master(cuda_dev, fmt, when):
    """The device ring holds the unpacked floats, so the bins are bitwise those of the analyzer on a master fed the
    restated floats; set up before the first block, or after several (the ring is then seeded by unpacking the raw host
    ring, whose U16 fill is 0x8000 = 0.0)."""
    lib = _driver16()
    if fmt == R.U16:
        L, M, cplx, fft_n, bins, shift, chunk, scale = 48000, 12001, False, 6000, 1500, 750, 40000, SCALE
    else:
        L, M, cplx, fft_n, bins, shift, chunk, scale = 40000, 10001, True, 4000, 1000, 0, 30000, 1.0
    c = 2 if cplx else 1
    w = words16(c * 6 * L, fmt, seed=9, garbage=True)
    flo = R.unpack16(w, fmt, scale)
    if cplx:
        flo = flo.view(np.complex64)
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    with Session(lib, L, M, cplx) as a, Session(lib, L, M, cplx) as b:
        if when == "before":
            a.spec_setup(fft_n, bins, window)
            b.spec_setup(fft_n, bins, window)
        for k in range(len(flo) // chunk):
            assert a.raw(w[c * k * chunk:c * (k + 1) * chunk], chunk, fmt, scale) == b.flt(flo[k * chunk:(k + 1) * chunk])
            if when == "after" and k == 3:
                a.spec_setup(fft_n, bins, window)
                b.spec_setup(fft_n, bins, window)
            if when == "before" or k >= 3:
                (ga, ea), (gb, eb) = a.spec_poll(shift, 3, 0.5, bins), b.spec_poll(shift, 3, 0.5, bins)
                assert ea == eb and same(ga, gb), k
                assert np.abs(ga).max() > 0 or ea == 0


@pytest.mark.gpu
def test_raw16_rejections(cuda_dev):
    lib = _driver16()
    z = np.zeros(4096, np.int16)
    planar = lambda s, n: lib.rd_write_planar(s.h, z.ctypes.data, z.ctypes.data, n, 1.0)  # noqa: E731
    with Session(lib, 48000, 12001, False) as s:
        assert s.raw(z, 16, R.SC16Q11) == -1                  # SC16 Q11 samples are I/Q
        assert planar(s, 16) == -1                            # planar I/Q on a REAL master
        assert s.raw(z, 16, R.S16) == 0
        assert s.raw(z, 16, R.U16) == -1                      # another format on the same master
        assert s.raw(z, 16, 2) == -1
        assert s.flt(np.zeros(16, np.float32)) == -1          # floats on a raw master
        assert s.i16(z[:16], 1.0) == -1                       # int16 ingest on a raw master
    with Session(lib, 48000, 12001, True) as s:
        assert s.raw(z, 16, R.U16) == -1                      # offset-binary 16-bit samples are real
        assert planar(s, 16) == 0                             # starts an S16 master ...
        assert s.raw(z, 16, R.S16) == 0                       # ... which takes interleaved S16 too
        assert s.raw(z, 16, R.SC16Q11) == -1
    with Session(lib, 48000, 12001, True) as s:
        assert s.raw(z, 16, R.SC16Q11) == 0
        assert planar(s, 16) == -1                            # planar on an SC16 Q11 master
        assert s.raw(z, 16, R.S16) == -1
    with Session(lib, 48000, 12001, True) as s:
        assert s.raw(np.full(64, 0x80, np.uint8), 16, 2) == 0
        assert planar(s, 16) == -1                            # planar on an 8-bit master
    with Session(lib, 48000, 12001, True) as s:
        assert s.flt(np.zeros(16, np.complex64)) == 0
        assert planar(s, 16) == -1                            # planar on a float master
        assert s.raw(z, 16, R.S16) == -1
    with Session(lib, 48000, 12001, True) as s:
        assert s.i16(z[:32], 1.0) == 0
        assert s.raw(z, 16, R.SC16Q11) == -1                  # raw16 on an int16 master
