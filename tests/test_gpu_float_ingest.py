"""Float ingest on the device: AirspyHF+ (FILTER_RAW_CF32_CNRMF), Fobos (CF32_FSCALE) and HydraSDR FLOAT32_REAL / FLOAT32_IQ
(F32, CF32) through write_rawfilter, and their A/D energy (filter_ingest_stats' fenergy).

Every format gives exactly the floats the drivers' loops store, so a master fed the library's floats is compared bitwise
with the same library fed the restated floats (tests/float_ingest_ref.py, pinned against the reference's own airspyhf.c,
fobos.c and hydrasdr.c by tests/test_float_ingest_cpu.py) through write_cfilter / write_rfilter, and within TOL with the
reference's own filter.c fed them.  The block energies are float_energy_kernel's fixed-order double sums, which the
restatement reproduces exactly.  tests/abi/float_driver.c is the filter.h driver; its build against the reference's own
header declares the extensions itself, as a patched radiod would.
"""
import ctypes as C

import numpy as np
import pytest

import float_ingest_ref as R
from test_gpu_raw_ingest import Session, _driver, same

TOL = 1e-5
SCALE = 1.0 / 1.7             # scale_AD-like double: its float products round differently
GAIN = 10 ** (-6 / 20)        # a gain change between two writes


def _driverf(name="float_driver.so"):
    lib = _driver(name)
    lib.rd_fdomain.argtypes = [C.c_void_p, C.c_uint, C.c_void_p]
    lib.rd_fstats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    fm = (C.c_int * 4)()
    lib.rd_float_formats(fm)
    assert list(fm) == [R.F32, R.CF32, R.CF32_CNRMF, R.CF32_FSCALE]
    return lib


def fstats(lib, s):
    """(blocks, samples, overranges, overrange_samples, since_over), fenergy; None on a master without statistics"""
    cnt = (C.c_uint64 * 5)()
    e = C.c_double(0)
    if lib.rd_fstats(s.h, C.cast(cnt, C.c_void_p), C.byref(e)) != 0:
        return None
    return tuple(int(v) for v in cnt), e.value


def floats(ncomp, seed, special=True):
    """ncomp float components as a front end's library delivers them: tones in noise, with denormals and signed zeros"""
    rng = np.random.default_rng(seed)
    t = np.arange(ncomp)
    v = 0.4 * np.cos(2 * np.pi * 0.0123 * t) + 0.1 * np.cos(2 * np.pi * 0.2071 * t) + rng.normal(0, 0.03, ncomp)
    v = v.astype(np.float32)
    if special:
        k = rng.integers(0, ncomp, 64)
        v[k[:32]] = np.float32(1e-45) * rng.integers(1, 1 << 20, 32).astype(np.float32)
        v[k[32:48]] = np.float32(0.0)
        v[k[48:]] = np.float32(-0.0)
    return v


def sizes(total, L, seed):
    """uneven transfer sizes summing to total, from a fortieth of a block to over half of one"""
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while n < total:
        k = int(min(total - n, rng.integers(L // 40, L * 3 // 5)))
        out.append(k)
        n += k
    return out


def stored(x, fmt, sc):
    """R.store with a scale per component"""
    x = np.asarray(x, np.float32)
    if fmt == R.CF32_FSCALE:
        return x * sc.astype(np.float32)
    return (sc * x.astype(np.float64)).astype(np.float32)


def same_or_nan(a, b):
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and same(a[~na], b[~nb])


# ------------------------------------------------------------------ the unpack kernel --------------------------------
KFMT = {R.F32: "KGPU_RAW_F32", R.CF32: "KGPU_RAW_CF32", R.CF32_CNRMF: "KGPU_RAW_CF32_CNRMF", R.CF32_FSCALE: "KGPU_RAW_CF32_FSCALE"}


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.F32, R.CF32, R.CF32_CNRMF, R.CF32_FSCALE])
def test_float_unpack_kernel_bitwise_and_block_energy(cuda_dev, fmt):
    """kgpu_unpack8 on floats: stores bitwise the restatement's with two scale changes inside the window (one in the
    history); each block's energy exactly the restated fixed-order sum over its new samples only (huge values planted in
    the history never count); a block with a NaN, an Inf or a float square past FLT_MAX has a non-finite energy."""
    import torch

    from ka9q_radio_b200 import capi

    cplx = fmt != R.F32
    c = 2 if cplx else 1
    L, hist, a0 = 30000, 3333, 5_000_000
    dt = np.dtype([("fenergy", "<f8"), ("overs", "<u4"), ("over_samples", "<u4")])
    for k in (1, 2, 3):
        n = hist + k * L
        x = floats(n * c, seed=k)
        x[:16] = np.float32(3e38)                            # in the history: never counted
        if k == 3:
            x[c * (hist + 5)] = np.float32(np.nan)           # block 0
            x[c * (hist + L + 7)] = np.float32(np.inf)       # block 1
            x[c * (hist + 2 * L + 9)] = np.float32(2e19)     # block 2: finite, but its float square is not
        chg = np.array([(a0 + hist // 2, SCALE * GAIN), (a0 + hist + L // 3, SCALE * 0.3)], dtype=[("at", "<i8"), ("scale", "<f8")])
        d_x = torch.from_numpy(x.copy()).to(cuda_dev)
        d_out = torch.full((n * c,), float("nan"), device=cuda_dev)
        d_st = torch.full((k * 16,), 0xA5, dtype=torch.uint8, device=cuda_dev)
        d_chg = torch.from_numpy(chg.view(np.uint8).copy()).to(cuda_dev)
        capi.unpack8(d_x.data_ptr(), getattr(capi, KFMT[fmt]), capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, hist, L, k,
                     SCALE, d_out.data_ptr(), d_st.data_ptr(), d_chg=d_chg.data_ptr(), nchg=2, a0=a0)
        torch.cuda.synchronize()
        samp = a0 + np.arange(n)
        sc = np.where(samp >= chg[1]["at"], chg[1]["scale"], np.where(samp >= chg[0]["at"], chg[0]["scale"], SCALE))
        assert same_or_nan(d_out.cpu().numpy(), stored(x, fmt, np.repeat(sc, c))), k
        got = np.frombuffer(d_st.cpu().numpy().tobytes(), dt)
        want = R.block_energies(x[hist * c:], fmt, L)
        assert (got["overs"] == 0).all() and (got["over_samples"] == 0).all()
        for b in range(k):
            if np.isfinite(want[b]):
                assert got["fenergy"][b] == want[b], (k, b, got["fenergy"][b], want[b])
            else:
                assert not np.isfinite(got["fenergy"][b]) and np.isnan(got["fenergy"][b]) == np.isnan(want[b]), (k, b)
        if k == 3:   # only cnrm squares in double, where 2e19 stays finite
            assert [np.isfinite(w) for w in want] == [False, False, fmt == R.CF32]


@pytest.mark.gpu
def test_float_unpack_rejects_master_types(cuda_dev):
    import torch

    from ka9q_radio_b200 import capi

    d = torch.zeros(4096, device=cuda_dev)
    out = torch.empty(4096, device=cuda_dev)
    with pytest.raises(capi.KgpuError):
        capi.unpack8(d.data_ptr(), capi.KGPU_RAW_F32, capi.KGPU_COMPLEX, 0, 100, 1, 1.0, out.data_ptr())
    for f in ("KGPU_RAW_CF32", "KGPU_RAW_CF32_CNRMF", "KGPU_RAW_CF32_FSCALE"):
        with pytest.raises(capi.KgpuError):
            capi.unpack8(d.data_ptr(), getattr(capi, f), capi.KGPU_REAL, 0, 100, 1, 1.0, out.data_ptr())
    with pytest.raises(capi.KgpuError):
        capi.unpack8(d.data_ptr() + 2, capi.KGPU_RAW_CF32, capi.KGPU_COMPLEX, 0, 100, 1, 1.0, out.data_ptr())


# ------------------------------------------------------------------ the front ends through filter.h ------------------
# (name, L, M, COMPLEX, format): AirspyHF+ 912 kS/s (N = 22 800 = 2^4 3 5^2 19, an extended 19-smooth master), Fobos
# 8 MS/s, HydraSDR FLOAT32_REAL 20 MS/s and FLOAT32_IQ 10 MS/s, 20 ms blocks, overlap factor 5
FRONT_ENDS = [
    ("airspyhf_912k", 18240, 4561, True, R.CF32_CNRMF),
    ("fobos_8m", 160000, 40001, True, R.CF32_FSCALE),
    ("hydrasdr_f32_real_20m", 400000, 100001, False, R.F32),
    ("hydrasdr_f32_iq_10m", 200000, 50001, True, R.CF32),
]
CHANS = [(480, -0.4, 0.4, 11.0, 2000), (960, -0.3, 0.3, 9.0, -1234)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,L,M,cplx,fmt", FRONT_ENDS, ids=[f[0] for f in FRONT_ENDS])
@pytest.mark.parametrize("driver", ["float_driver.so", "float_driver_refhdr.so"])
def test_front_end_through_filter_h(oracle, cuda_dev, driver, name, L, M, cplx, fmt):
    """Transfers of uneven sizes that straddle blocks and the end of the ring, with a gain change between two of them:
    the channel outputs are bitwise those of the same library fed the restated floats, and within TOL of the reference's
    own filter.c fed them; filter_ingest_stats' fenergy is exactly the restated block sums, added block by block; the
    first window's history is zero (its spectrum is bitwise the float master's)."""
    lib = _driverf(driver)
    c = 2 if cplx else 1
    nb = 7
    total = nb * L + L // 3
    x = floats(c * total, seed=L)
    parts = sizes(total, L, seed=M)
    gain_at = len(parts) // 2
    check_ref = driver == "float_driver.so" and oracle.ref_available()
    ref = oracle.RefSession(L, M, oracle.KO_COMPLEX if cplx else oracle.KO_REAL) if check_ref else None
    want_e = R.block_energies(x, fmt, L)
    try:
        with Session(lib, L, M, cplx) as a, Session(lib, L, M, cplx) as b:
            assert fstats(lib, a) == ((0,) * 5, 0.0)
            for s in (a, b):
                for olen, lo, hi, beta, _ in CHANS:
                    s.add(olen, lo, hi, beta)
            if ref is not None:
                for olen, lo, hi, beta, _ in CHANS:
                    ref.add_channel(olen, lo, hi, beta)
            pos, fired = 0, 0
            for k, n in enumerate(parts):
                sc = SCALE * (GAIN if k >= gain_at else 1.0)
                seg = x[c * pos:c * (pos + n)]
                flo = R.store(seg, fmt, sc)
                if cplx:
                    flo = flo.view(np.complex64)
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
                e = 0.0
                for be in want_e[fired:now]:
                    e += be
                assert fstats(lib, a) == ((now - fired, (now - fired) * L, 0, 0, now * L), e), k   # no limits: never over
                fired = now
            assert fired == nb
            assert b.stats() is None                          # the float-fed master: the driver counts
    finally:
        if ref is not None:
            ref.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["nan", "inf"])
def test_non_finite_block_through_filter_h(cuda_dev, bad):
    """A NaN or Inf sample in block 2 makes block 2's energy non-finite and leaves the other blocks' energies exact, so a
    driver applying its isfinite guard to each filter_ingest_stats result skips exactly the blocks it would skip."""
    lib = _driverf()
    L, M = 18240, 4561
    x = floats(2 * 5 * L, seed=4, special=False)
    x[2 * (2 * L + 123) + 1] = np.float32(np.nan if bad == "nan" else -np.inf)
    want = R.block_energies(x, R.CF32_CNRMF, L)
    with Session(lib, L, M, True) as a:
        assert fstats(lib, a)[1] == 0.0
        for b in range(5):
            assert a.raw(x[2 * b * L:2 * (b + 1) * L], L, R.CF32_CNRMF, SCALE) == 1
            cnt, e = fstats(lib, a)
            assert cnt[0] == 1, b
            if b == 2:
                assert np.isnan(e) if bad == "nan" else np.isinf(e)
            else:
                assert e == want[b], b


@pytest.mark.gpu
def test_lapped_slave_on_a_float_master(cuda_dev):
    """A consumer that fell ND blocks behind a CF32-fed master gets a block of zeros and a drop, as one fed floats does."""
    lib = _driverf()
    L, M = 40000, 10001
    x = floats(2 * 8 * L, seed=3)
    flo = R.store(x, R.CF32, SCALE).view(np.complex64)
    with Session(lib, L, M, True, nworkers=1) as a, Session(lib, L, M, True, nworkers=1) as b:
        for s in (a, b):
            s.add(480, -0.3, 0.3, 9.0)
        assert lib.rd_write_from_thread(a.h, x.ctypes.data, L, 6, 8 * L, 1, R.CF32, SCALE) == 0
        assert lib.rd_write_from_thread(b.h, flo.ctypes.data, L, 6, 8 * L, 0, 0, 0.0) == 0
        for _ in range(4):
            assert same(a.exe(0, 1500), b.exe(0, 1500))
        assert lib.rd_drops(a.h, 0) == lib.rd_drops(b.h, 0) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.CF32, R.CF32_FSCALE])
@pytest.mark.parametrize("when", ["before", "after"])
def test_wideband_analyzer_on_float_master(cuda_dev, fmt, when):
    """The device ring holds the stored floats, so the bins are bitwise those of the analyzer on a master fed the
    restated floats; set up before the first block, or after several (the ring is then seeded by converting the raw host
    ring, whose fill is 0.0f)."""
    lib = _driverf()
    L, M, fft_n, bins, shift, chunk = 40000, 10001, 4000, 1000, 0, 30000
    x = floats(2 * 6 * L, seed=9)
    flo = R.store(x, fmt, SCALE).view(np.complex64)
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    with Session(lib, L, M, True) as a, Session(lib, L, M, True) as b:
        if when == "before":
            a.spec_setup(fft_n, bins, window)
            b.spec_setup(fft_n, bins, window)
        for k in range(len(flo) // chunk):
            assert a.raw(x[2 * k * chunk:2 * (k + 1) * chunk], chunk, fmt, SCALE) == b.flt(flo[k * chunk:(k + 1) * chunk])
            if when == "after" and k == 3:
                a.spec_setup(fft_n, bins, window)
                b.spec_setup(fft_n, bins, window)
            if when == "before" or k >= 3:
                (ga, ea), (gb, eb) = a.spec_poll(shift, 3, 0.5, bins), b.spec_poll(shift, 3, 0.5, bins)
                assert ea == eb and same(ga, gb), k
                assert np.abs(ga).max() > 0 or ea == 0


@pytest.mark.gpu
def test_float_rejections(cuda_dev):
    lib = _driverf()
    z = np.zeros(4096, np.float32)
    with Session(lib, 48000, 12001, False) as s:
        for fmt in R.COMPLEX_FORMATS:
            assert s.raw(z, 16, fmt) == -1                    # the float I/Q formats need a COMPLEX master
        assert s.raw(z, 16, R.F32) == 0
        assert s.raw(z, 16, 6) == -1                          # another format on the same master
        assert s.flt(np.zeros(16, np.float32)) == -1          # floats through write_rfilter on a raw master
        assert s.i16(np.zeros(16, np.int16), 1.0) == -1       # int16 ingest on a raw master
    with Session(lib, 48000, 12001, True) as s:
        assert s.raw(z, 16, R.F32) == -1                     # FILTER_RAW_F32 samples are real
        assert s.raw(z, 16, R.CF32) == 0
        assert s.raw(z, 16, R.CF32_CNRMF) == -1               # each rule is a format of its own: no mixing
        assert s.raw(z, 16, R.CF32_FSCALE) == -1
        assert s.raw(z, 16, 13) == -1                         # unknown format
    with Session(lib, 48000, 12001, True) as s:
        assert s.flt(np.zeros(16, np.complex64)) == 0
        assert s.raw(z, 16, R.CF32) == -1                     # float raw ingest on a float master
    with Session(lib, 48000, 12001, True) as s:
        assert s.raw(np.zeros(64, np.int16), 16, 6) == 0
        assert s.raw(z, 16, R.CF32_FSCALE) == -1              # float raw ingest on an S16 master
