"""Raw 8-bit and packed 12-bit ingest through filter.h (write_rawfilter) and the A/D statistics of every raw ingest
(filter_ingest_stats), on the device.

The 8-bit formats must give exactly the floats the drivers' loops store, so a master fed raw bytes is compared bitwise
with the same library fed the restated floats through write_cfilter / write_rfilter.  Packed 12-bit runs the int16
path with the drivers' float scale and is compared with the reference's own airspy_unpack followed by its filter.c.
tests/abi/raw_driver.c is the filter.h driver; its build against the reference's own header declares the extensions
itself, as a patched radiod would.
"""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import raw_ingest_ref as R

ROOT = Path(__file__).resolve().parent.parent
TOL = 1e-5
SCALE = 1.0 / (128 * 1.7)   # scale_AD-like double (rtlsdr.c:76): its float products round differently


def _driver(name="raw_driver.so"):
    p = (ROOT / "oracle" / "_ref" if "refhdr" in name else ROOT / "tests" / "abi" / "_build") / name
    if not p.exists():
        pytest.skip(f"{name} not built")
    lib = C.CDLL(str(p))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.rd_open.restype = vp
    lib.rd_open.argtypes = [i, i, i, i]
    lib.rd_add_channel.argtypes = [vp, i, d, d, d]
    lib.rd_write_raw.argtypes = [vp, vp, i, i, d]
    lib.rd_write_i16.argtypes = [vp, vp, i, C.c_float, i]
    lib.rd_write_float.argtypes = [vp, vp, i]
    lib.rd_write_from_thread.argtypes = [vp, vp, i, i, C.c_size_t, i, i, d]
    lib.rd_execute.argtypes = [vp, i, i, vp]
    lib.rd_execute_tuned.argtypes = [vp, i, i, d, d, vp, vp]
    lib.rd_drops.argtypes = [vp, i]
    lib.rd_drops.restype = C.c_uint
    lib.rd_enable_noise.argtypes = [vp, d]
    lib.rd_noise.argtypes = [vp, i]
    lib.rd_noise.restype = d
    lib.rd_stats.argtypes = [vp, vp]
    lib.rd_spec_setup.argtypes = [vp, i, i, vp]
    lib.rd_spec_poll.argtypes = [vp, i, i, d, vp, vp]
    lib.rd_close.argtypes = [vp]
    return lib


class Session:
    def __init__(self, lib, L, M, cplx, nworkers=0):
        self.lib, self.L, self.cplx = lib, L, cplx
        self.h = lib.rd_open(L, M, int(cplx), nworkers)
        assert self.h, "create_filter_input failed"
        self.olen = []

    def add(self, olen, low, high, beta):
        i = self.lib.rd_add_channel(self.h, olen, low, high, beta)
        assert i >= 0
        self.olen.append(olen)
        return i

    def raw(self, x, n, fmt, scale=SCALE):
        x = np.ascontiguousarray(x)
        return self.lib.rd_write_raw(self.h, x.ctypes.data, n, fmt, scale)

    def i16(self, x, scale, derand=False):
        x = np.ascontiguousarray(x, np.int16)
        return self.lib.rd_write_i16(self.h, x.ctypes.data, len(x) // (2 if self.cplx else 1), scale, int(derand))

    def flt(self, x):
        x = np.ascontiguousarray(x)
        return self.lib.rd_write_float(self.h, x.ctypes.data, len(x))

    def exe(self, ch, shift):
        y = np.empty(self.olen[ch], np.complex64)
        assert self.lib.rd_execute(self.h, ch, shift, y.ctypes.data) == 0
        return y

    def tuned(self, ch, shift, rem, rate):
        y = np.empty(self.olen[ch], np.complex64)
        pw = C.c_double(0)
        assert self.lib.rd_execute_tuned(self.h, ch, shift, rem, rate, y.ctypes.data, C.byref(pw)) == 0
        return y, pw.value

    def stats(self):
        out = (C.c_uint64 * 6)()
        if self.lib.rd_stats(self.h, C.cast(out, C.c_void_p)) != 0:
            return None
        return tuple(int(v) for v in out)

    def spec_setup(self, fft_n, bin_count, window):
        w = np.ascontiguousarray(window, np.float32)
        assert self.lib.rd_spec_setup(self.h, fft_n, bin_count, w.ctypes.data) == 0

    def spec_poll(self, shift, fft_avg, overlap, bin_count):
        b = np.empty(bin_count, np.float32)
        end = C.c_uint64(0)
        assert self.lib.rd_spec_poll(self.h, shift, fft_avg, overlap, b.ctypes.data, C.byref(end)) == 0
        return b, end.value

    def close(self):
        if self.h:
            self.lib.rd_close(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def bytes8(n, fmt, seed=1, tone=0.0123):
    """n components of an 8-bit front end: a tone in noise, clipped at both ends now and then"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    v = 90 * np.cos(2 * np.pi * tone * t) + rng.normal(0, 12, n) + rng.choice([0, 0, 0, 0, 400, -400], n) * (rng.random(n) < 1e-3)
    v = np.clip(np.rint(v), -128, 127).astype(np.int64)
    return (v + 128).astype(np.uint8) if fmt == R.U8 else v.astype(np.int8).view(np.uint8)


def sum_stats(parts):
    tot = [0] * 5
    for p in parts:
        for k in range(5):
            tot[k] += p[k]
    return tot


# ------------------------------------------------------------------ the unpack kernel --------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.U8, R.S8])
@pytest.mark.parametrize("cplx", [False, True])
def test_unpack8_kernel_bitwise_and_block_stats(cuda_dev, fmt, cplx):
    import torch

    from ka9q_radio_b200 import capi

    c = 2 if cplx else 1
    L, hist = 1000, 333
    dt = np.dtype([("energy", "<u8"), ("overs", "<u4"), ("over_samples", "<u4")])
    for k in (1, 2, 3):   # 1 .. ND-1 blocks per launch
        n = hist + k * L
        raw = bytes8(n * c, fmt, seed=k)
        raw[:256] = np.arange(256, dtype=np.uint8)                 # every byte, in the history (never counted) ...
        raw[hist * c + 7: hist * c + 7 + 256] = np.arange(256)     # ... and in block 0
        d_raw = torch.from_numpy(raw).to(cuda_dev)
        d_out = torch.full((n * c,), float("nan"), device=cuda_dev)
        d_st = torch.full((k * 16,), 0xA5, dtype=torch.uint8, device=cuda_dev)
        capi.unpack8(d_raw.data_ptr(), capi.KGPU_RAW_U8 if fmt == R.U8 else capi.KGPU_RAW_S8,
                     capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, hist, L, k, SCALE, d_out.data_ptr(), d_st.data_ptr())
        torch.cuda.synchronize()
        assert same(d_out.cpu().numpy(), R.unpack8(raw, fmt, SCALE))
        got = np.frombuffer(d_st.cpu().numpy().tobytes(), dt)
        want = R.block_stats(R.values8(raw, fmt)[hist * c:], fmt, L, cplx)
        assert [(int(g["energy"]), int(g["overs"]), int(g["over_samples"])) for g in got] == want


# ------------------------------------------------------------------ RTL-SDR through filter.h -------------------------
RTL = dict(L=36000, M=9001, fs=1.8e6)
RTL_CHANS = [(240, -0.4, 0.4, 11.0, 2000), (480, -0.3, 0.3, 9.0, -7000), (1200, -0.45, 0.45, 11.0, 12345)]


@pytest.mark.gpu
@pytest.mark.parametrize("driver,drain", [("raw_driver.so", 1), ("raw_driver.so", 3), ("raw_driver.so", 0),
                                          ("raw_driver_refhdr.so", 1)])
def test_rtlsdr_through_filter_h(oracle, cuda_dev, driver, drain):
    """A COMPLEX 1.8 MS/s master fed ragged 131072-pair u8 writes (rtlsdr.c:268): a bank of channels, a fine-tuned
    channel and the noise estimates are bitwise those of the same library fed the restated floats; the plain channels
    are within TOL of the reference's own filter.c; filter_ingest_stats sums to the restatement in any drain pattern
    (every `drain` writes, 0 = once at the end)."""
    lib = _driver(driver)
    L, M, fs = RTL["L"], RTL["M"], RTL["fs"]
    N = L + M - 1
    nw, chunk = 6, 131072
    raw = bytes8(2 * nw * chunk, R.U8)
    flo = R.unpack8(raw, R.U8, SCALE).view(np.complex64)
    check_ref = driver == "raw_driver.so" and drain == 1 and oracle.ref_available()
    ref = oracle.RefSession(L, M, oracle.KO_COMPLEX) if check_ref else None
    with Session(lib, L, M, True) as a, Session(lib, L, M, True) as b:
        assert a.stats() == (0, 0, 0, 0, 0, 0)   # collection starts here
        for s in (a, b):
            for olen, lo, hi, beta, _ in RTL_CHANS:
                s.add(olen, lo, hi, beta)
            s.add(480, -0.3, 0.3, 11.0)          # fine-tuned
            assert s.lib.rd_enable_noise(s.h, fs) == 0
        if ref is not None:
            for olen, lo, hi, beta, _ in RTL_CHANS:
                ref.add_channel(olen, lo, hi, beta)
        parts, fired = [], 0
        for w in range(nw):
            fa = a.raw(raw[2 * w * chunk: 2 * (w + 1) * chunk], chunk, R.U8)
            assert fa == b.flt(flo[w * chunk:(w + 1) * chunk]) == 1
            fired = (w + 1) * chunk // L
            if ref is not None:
                assert ref.write(flo[w * chunk:(w + 1) * chunk]) == 1
            for ch, (olen, *_, shift) in enumerate(RTL_CHANS):
                ya, yb = a.exe(ch, shift), b.exe(ch, shift)
                assert same(ya, yb), (w, ch)
                assert a.lib.rd_noise(a.h, ch) == b.lib.rd_noise(b.h, ch) or np.isnan(a.lib.rd_noise(a.h, ch))
                if ref is not None:
                    r = ref.execute(ch, shift)
                    assert np.abs(ya - r).max() / np.abs(r).max() < TOL, (w, ch)
            _, shift, rem = oracle.compute_tuning(N, fs, 123_456.7 + 1000 * w)
            (ya, pa), (yb, pb) = a.tuned(3, shift, rem, 24000.0), b.tuned(3, shift, rem, 24000.0)
            assert same(ya, yb) and pa == pb
            if drain and (w + 1) % drain == 0:
                parts.append(a.stats())
        parts.append(a.stats())
        assert b.stats() is None   # fed floats: the driver counts in its own loop
    if ref is not None:
        ref.close()
    want = R.block_stats(R.values8(raw, R.U8), R.U8, L, True)[:fired]
    assert sum_stats(parts) == [fired, fired * L] + [sum(s[k] for s in want) for k in range(3)]
    assert parts[-1][5] == R.since_over(want, L)


@pytest.mark.gpu
def test_rtlsdr_lapped_slave(cuda_dev):
    """A consumer that fell ND blocks behind a raw-fed master gets a block of zeros and a drop, as one fed floats does."""
    lib = _driver()
    L, M = RTL["L"], RTL["M"]
    raw = bytes8(2 * 8 * L, R.U8)
    flo = R.unpack8(raw, R.U8, SCALE).view(np.complex64)
    with Session(lib, L, M, True, nworkers=1) as a, Session(lib, L, M, True, nworkers=1) as b:
        for s in (a, b):
            s.add(480, -0.3, 0.3, 9.0)
        assert lib.rd_write_from_thread(a.h, raw.ctypes.data, L, 6, 2 * L, 1, R.U8, SCALE) == 0
        assert lib.rd_write_from_thread(b.h, flo.ctypes.data, L, 6, 8 * L, 0, 0, 0.0) == 0
        for _ in range(4):
            ya, yb = a.exe(0, 1500), b.exe(0, 1500)
            assert same(ya, yb)
        assert lib.rd_drops(a.h, 0) == lib.rd_drops(b.h, 0) >= 1


# ------------------------------------------------------------------ Airspy R2 and HydraSDR ---------------------------
def _ref_airspy_unpack(words, count, scale):
    """the reference's own airspy_unpack (airspy-unpack.c:106-130, compiled unmodified into oracle/_ref)"""
    from oracle import oracle as O

    lib = O.ref_lib()
    fn = lib.airspy_unpack
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_uint64)]
    out = np.empty(count, np.float32)
    e = C.c_uint64(0)
    w = np.ascontiguousarray(words, np.uint32)
    over = fn(out.ctypes.data, w.ctypes.data, count, scale, C.byref(e))
    return out, int(e.value), int(over)


@pytest.mark.gpu
def test_airspy_r2_packed12_through_filter_h(oracle, cuda_dev):
    """Airspy R2 at 20 MS/s (REAL, L = 400000, M - 1 = L/4): outputs within TOL of the reference's airspy_unpack followed
    by its filter.c; statistics equal to what airspy_unpack returns over each block's new samples."""
    if not oracle.ref_available():
        pytest.skip("reference binaries not built")
    L, M, nb, chunk = 400000, 100001, 3, 131072
    scale = np.float32(1.0 / 2048)
    rng = np.random.default_rng(5)
    n = nb * L + chunk
    s12 = np.clip(np.rint(2048 + 1500 * np.cos(2 * np.pi * 0.0731 * np.arange(n)) + rng.normal(0, 100, n)), 0, 4095)
    s12[rng.random(n) < 1e-4] = 4095
    s12[rng.random(n) < 1e-4] = 0
    s12 = s12.astype(np.int64)
    words = oracle.airspy_pack(s12)
    flo, _, _ = _ref_airspy_unpack(words, n, scale)
    chans = [(960, -0.3, 0.3, 11.0, 30000), (480, -0.2, 0.4, 9.0, -123457)]
    with Session(_driver(), L, M, False) as a, oracle.RefSession(L, M, oracle.KO_REAL) as ref:
        assert a.stats() == (0,) * 6
        for olen, lo, hi, beta, _ in chans:
            a.add(olen, lo, hi, beta)
            ref.add_channel(olen, lo, hi, beta)
        fired = 0
        for w in range(n // chunk):
            seg = words[w * chunk * 3 // 8:(w + 1) * chunk * 3 // 8]
            f = a.raw(seg, chunk, R.PACKED12, float(scale))
            assert f == ref.write(flo[w * chunk:(w + 1) * chunk])
            if f == 1:
                fired = (w + 1) * chunk // L
                for ch, (*_, shift) in enumerate(chans):
                    y, r = a.exe(ch, shift), ref.execute(ch, shift)
                    assert np.abs(y - r).max() / np.abs(r).max() < TOL, (w, ch)
        got = a.stats()
    want = [_ref_airspy_unpack(words[b * L * 3 // 8:(b + 1) * L * 3 // 8], L, scale)[1:] for b in range(fired)]
    assert got[:2] == (fired, fired * L)
    assert got[2] == sum(e for e, _ in want) and got[3] == got[4] == sum(o for _, o in want)
    assert got[5] == R.since_over([(0, 0, o) for _, o in want], L)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,cplx,L,M", [(R.U8, False, 200000, 50001), (R.S8, False, 200000, 50001),
                                          (R.U8, True, 50000, 12501), (R.S8, True, 50000, 12501)])
def test_hydrasdr_8bit(cuda_dev, fmt, cplx, L, M):
    """HydraSDR UINT8 / INT8, REAL and I/Q (hydrasdr.c:759-830): bitwise the same library fed the restated floats;
    statistics (overranges per component, and per sample as the I/Q cases count them) equal to the restatement."""
    lib = _driver()
    c = 2 if cplx else 1
    chunk, nw = 65536, 8
    raw = bytes8(c * chunk * nw, fmt, seed=7)
    flo = R.unpack8(raw, fmt, SCALE)
    if cplx:
        flo = flo.view(np.complex64)
    with Session(lib, L, M, cplx) as a, Session(lib, L, M, cplx) as b:
        a.stats()
        for s in (a, b):
            s.add(400, -0.3, 0.3, 11.0)
        for w in range(nw):
            fa = a.raw(raw[c * w * chunk:c * (w + 1) * chunk], chunk, fmt)
            assert fa == b.flt(flo[w * chunk:(w + 1) * chunk])
            if fa == 1:
                assert same(a.exe(0, 4321), b.exe(0, 4321)), w
        got = a.stats()
    fired = nw * chunk // L
    want = R.block_stats(R.values8(raw, fmt), fmt, L, cplx)[:fired]
    assert list(got[:5]) == [fired, fired * L] + [sum(s[k] for s in want) for k in range(3)]
    assert got[5] == R.since_over(want, L)


# ------------------------------------------------------------------ RX888 int16 statistics ---------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("derand", [False, True])
def test_rx888_int16_statistics(oracle, cuda_dev, derand):
    """write_i16filter masters: per-block statistics equal convert()'s (rx888.c:753-767), drained block by block; the
    outputs are bitwise those of a master that never asks."""
    lib = _driver()
    L, M, nb = 48000, 12001, 7
    scale = np.float32(10 ** (3 / 20) / 32768)
    xi = oracle.siggen_tones_i16(nb * L, [0.25, 0.1], [0.3, 0.2], 0.01, 3)
    rng = np.random.default_rng(2)
    xi[rng.random(nb * L) < 2e-4] = 32767
    xi[rng.random(nb * L) < 2e-4] = -32767
    xi[rng.random(nb * L) < 2e-4] = -32768
    with Session(lib, L, M, False) as a, Session(lib, L, M, False) as b:
        assert a.stats() == (0,) * 6
        for s in (a, b):
            s.add(480, -1 / 3, 1 / 3, 11.0)
        since = 0
        for blk in range(nb):
            x = xi[blk * L:(blk + 1) * L]
            assert a.i16(x, scale, derand) == b.i16(x, scale, derand) == 1
            assert same(a.exe(0, 15000), b.exe(0, 15000))
            _, e, clips = oracle.convert_i16(x, scale, derand)
            since = 0 if clips else since + L
            assert a.stats() == (1, L, e, clips, clips, since), blk
        assert b.stats() == (0,) * 6   # first call on b
    assert any(oracle.convert_i16(xi[k * L:(k + 1) * L], scale, derand)[2] for k in range(nb))


# ------------------------------------------------------------------ wideband analyzer on raw masters ------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.U8, R.PACKED12])
@pytest.mark.parametrize("when", ["before", "after"])
def test_wideband_analyzer_on_raw_master(oracle, cuda_dev, fmt, when):
    """The device ring holds what the float path holds (floats after the 8-bit unpack, int16 for packed-12), so the bins
    are bitwise those of the analyzer on a master fed the restated floats; set up before the first block, or after
    several (the ring is then seeded by unpacking the raw host ring)."""
    lib = _driver()
    if fmt == R.U8:
        L, M, cplx, fft_n, bins, shift, chunk = 36000, 9001, True, 4000, 1000, 0, 30000
        raw = bytes8(2 * 6 * L, fmt)
        flo = R.unpack8(raw, fmt, SCALE).view(np.complex64)
        scale = SCALE
        rawchunk = lambda w: raw[2 * w * chunk:2 * (w + 1) * chunk]   # noqa: E731
    else:
        L, M, cplx, fft_n, bins, shift, chunk = 48000, 12001, False, 6000, 1500, 750, 40000
        rng = np.random.default_rng(9)
        s12 = np.clip(np.rint(2048 + 900 * np.cos(0.37 * np.arange(6 * L)) + rng.normal(0, 60, 6 * L)), 0, 4095).astype(np.int64)
        words = oracle.airspy_pack(s12)
        scale = float(np.float32(1 / 2048))
        flo = (np.float32(scale) * R.unpack12(s12).astype(np.float32)).astype(np.float32)
        rawchunk = lambda w: words[w * chunk * 3 // 8:(w + 1) * chunk * 3 // 8]   # noqa: E731
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(fft_n) / fft_n)).astype(np.float32)
    with Session(lib, L, M, cplx) as a, Session(lib, L, M, cplx) as b:
        if when == "before":
            a.spec_setup(fft_n, bins, window)
            b.spec_setup(fft_n, bins, window)
        for w in range(len(flo) // chunk):
            assert a.raw(rawchunk(w), chunk, fmt, scale) == b.flt(flo[w * chunk:(w + 1) * chunk])
            if when == "after" and w == 3:
                a.spec_setup(fft_n, bins, window)
                b.spec_setup(fft_n, bins, window)
            if when == "before" or w >= 3:
                (ga, ea), (gb, eb) = a.spec_poll(shift, 3, 0.5, bins), b.spec_poll(shift, 3, 0.5, bins)
                assert ea == eb and same(ga, gb), w
                assert np.abs(ga).max() > 0 or ea == 0


# ------------------------------------------------------------------ rejections ----------------------------------------
@pytest.mark.gpu
def test_rejections(cuda_dev):
    lib = _driver()
    x = np.full(4096, 0x80, np.uint8)
    xi = np.zeros(4096, np.int16)
    with Session(lib, 48000, 12001, False) as s:
        assert s.raw(x, 12, R.PACKED12) == -1                 # not a multiple of 8
        assert s.raw(x, 16, R.PACKED12) == 0
        assert s.raw(x, 16, R.U8) == -1                       # another format on the same master
        assert s.i16(xi[:16], 1.0) == -1
        assert s.flt(np.zeros(16, np.float32)) == -1
        assert s.raw(x, 16, -1) == -1                         # unknown format
    with Session(lib, 48000, 12001, False) as s:
        assert s.i16(xi[:16], 1.0) == 0
        assert s.raw(x, 16, R.S8) == -1
    with Session(lib, 48000, 12001, False) as s:
        assert s.flt(np.zeros(16, np.float32)) == 0
        assert s.stats() is None                              # stats on a float master
        assert s.raw(x, 16, R.U8) == -1
    with Session(lib, 48000, 12003, False) as s:
        assert s.raw(x, 16, R.PACKED12) == -1                 # M - 1 = 12002: windows off the group boundaries
    with Session(lib, 48000, 12001, True) as s:
        assert s.raw(x, 16, R.PACKED12) == -1                 # packed 12-bit samples are real
        assert s.raw(x, 16, R.S8) == 0


@pytest.mark.gpu
def test_int16_and_float_writes_exclude_each_other(cuda_dev):
    """Launches read the int16 ring of a master fed int16 words, so floats written to it would be lost: it refuses them,
    and a master fed floats refuses int16 words, through write_i16filter and through filter_i16_write_pointer."""
    from ka9q_radio_b200 import capi

    lib, kg = _driver(), capi.load()
    kg.filter_i16_write_pointer.restype = C.c_void_p
    kg.filter_i16_write_pointer.argtypes = [C.c_void_p]
    kg.write_i16filter.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_bool]
    xi, xf = np.zeros(16, np.int16), np.zeros(16, np.float32)
    # the session handle is the address of its struct filter_in
    with Session(lib, 48000, 12001, False) as s:
        assert s.i16(xi, 1.0) == 0
        assert s.flt(xf) == -1
    with Session(lib, 48000, 12001, False) as s:
        assert kg.filter_i16_write_pointer(s.h)
        assert kg.write_i16filter(s.h, None, 16, 1.0, False) == 0
        assert s.flt(xf) == -1
    with Session(lib, 48000, 12001, False) as s:
        assert s.flt(xf) == 0
        assert s.i16(xi, 1.0) == -1
        assert not kg.filter_i16_write_pointer(s.h)
    with Session(lib, 48000, 12001, False) as s:
        assert s.flt(xf[:0]) == 0                             # a write of no floats claims nothing
        assert s.i16(xi, 1.0) == 0
