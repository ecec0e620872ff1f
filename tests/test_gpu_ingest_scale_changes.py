"""Raw and int16 ingest across scale changes between writes: each write's scale covers exactly its own samples.

The drivers convert every transfer with the scale in force when it arrives (rx888.c:764, airspy.c:416-419 with
airspy-unpack.c, rtlsdr.c:338), and their gain changes (airspy.c:549 from the software AGC, rx888.c:1136 and :1159) land
between transfers.  So the floats filter.c sees keep the old scale on every sample written before a change.  Each
session here feeds one master raw words through seeded ragged write sequences whose scale changes inside a block, on a
block boundary, inside the M-1 history of the next window, twice within one launch of several blocks and back and forth,
and compares it with
  (a) the same library fed the drivers' own conversion of each write, done here in numpy, through write_rfilter /
      write_cfilter: bitwise for the channel outputs and master->fdomain[] of every launch whose window holds samples of
      more than one scale, within TOL otherwise; noise estimates, baseband power and tuned outputs within TOL;
  (b) the reference's own filter.c on the same floats, within TOL at every block, where it was built.
A launch whose window has one scale keeps the fused conversion, which kgpu_launch_count pins.  The A/D statistics are
integer moments that no scale touches; the wideband analyzer's polls match the analyzer on (a) and the restatement of
spectrum.c on the converted floats (and spectrum.c itself where it was built).
"""
import ctypes as C
import os

import numpy as np
import pytest

import raw_ingest_ref as R
from test_gpu_raw_ingest import TOL, Session, _driver, _ref_airspy_unpack, bytes8, same

ND = 4


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-30))


def close_to(got, ref):
    """the bound test_gpu_spectrum.py holds the analyzer to"""
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-5 * ref.max() + 1e-30)


def float_ring_samples(L, M, cplx):
    """the samples of the master's float ring: ND windows rounded up to a page (create_filter_input)"""
    esz = 8 if cplx else 4
    pg = os.sysconf("SC_PAGE_SIZE")
    return (ND * (L + M - 1) * esz + pg - 1) // pg * pg // esz


def launches(wcnt, job, n, L):
    """fire_ready_blocks: the (first job, k) launches a write of n samples makes, and the counters after it"""
    out = []
    wcnt += n
    while wcnt >= L:
        k = min(wcnt // L, ND - 1, ND - job % ND)
        out.append((job, k))
        wcnt -= k * L
        job += k
    return out, wcnt, job


class Dut(Session):
    def fdomain(self, job, bins):
        y = np.empty(bins, np.complex64)
        self.lib.rd_fdomain(self.h, job, y.ctypes.data)
        return y


def _lib():
    lib = _driver()
    lib.rd_fdomain.argtypes = [C.c_void_p, C.c_uint, C.c_void_p]
    lib.rd_fdomain.restype = C.c_int
    lib.rd_write_once_from_thread.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    return lib


def plan(L, M1, nb, grain, seed):
    """cut points of a write sequence over nb blocks and the points where the scale changes (all multiples of grain):
    ragged writes, two writes of several blocks (launches of k = 2 and 3), changes inside block 1, at the start of block 3,
    inside block 5's history, twice in the two-block launch of blocks 8-9, none in the three-block launch of blocks 12-14,
    and one inside block 16"""
    rng = np.random.default_rng(seed)
    g = lambda v: int(v) // grain * grain   # noqa: E731
    total = nb * L
    big = [(g(8 * L + L // 5), g(10 * L + L // 7)), (g(12 * L + L // 9), g(15 * L + L // 11))]
    changes = [g(L + L // 3), 3 * L, g(5 * L - M1 // 2), g(8 * L - M1 // 3), big[0][0], g(16 * L + L // 2)]
    cuts = {g(v) for v in rng.integers(1, total, 3 * nb)} | set(changes) | {a for a, _ in big} | {b for _, b in big}
    cuts = {c for c in cuts if 0 < c < total and not any(a < c < b for a, b in big)}
    # a few single-sample-group writes, so ragged really means ragged
    cuts |= {c + grain for c in sorted(cuts)[::5] if c + grain < total and not any(a <= c < b for a, b in big)}
    return sorted(cuts | {total}), sorted(changes)


# (id, format, complex, L, M, derandomize, when the wideband analyzer is set up, analyzer fft_n / bins / shift)
CASES = [
    ("rx888_i16", R.I16, False, 48000, 12001, False, "before", (6000, 1500, 750)),
    ("rx888_i16_derand", R.I16, False, 48000, 12001, True, "after", (6000, 1500, 750)),
    ("i16_complex_bluestein", R.I16, True, 58000, 14501, False, "before", (4000, 1000, 0)),   # N = 2^2 5^4 29
    ("rtlsdr_u8", R.U8, True, 36000, 9001, False, None, None),
    ("s8_real", R.S8, False, 48000, 12001, False, None, None),
    ("s8_complex", R.S8, True, 50000, 12501, False, None, None),
    ("airspy_packed12", R.PACKED12, False, 200000, 50001, False, "after", (8000, 2000, 1000)),
]
_CASE = {c[0]: c for c in CASES}
NB = 18
FFT_AVG, OVERLAP = 5, 0.5


def _source(fmt, cplx, n, seed):
    """integer front-end words for n samples: int16 (interleaved I/Q), bytes, or offset-binary 12-bit values"""
    rng = np.random.default_rng(seed)
    c = 2 if cplx else 1
    if fmt == R.I16:
        t = np.arange(n * c)
        x = np.rint(9000 * np.cos(2 * np.pi * 0.0713 * t) + 4000 * np.cos(2 * np.pi * 0.213 * t) + rng.normal(0, 300, n * c))
        x = np.clip(x, -32768, 32767).astype(np.int16)
        for v in (32767, -32767, -32768):
            x[rng.random(n * c) < 1e-4] = v
        return x
    if fmt == R.PACKED12:
        s = np.rint(2048 + 1500 * np.cos(2 * np.pi * 0.0731 * np.arange(n)) + rng.normal(0, 100, n))
        s[rng.random(n) < 1e-4] = 4095
        s[rng.random(n) < 1e-4] = 0
        return np.clip(s, 0, 4095).astype(np.int64)
    return bytes8(n * c, fmt, seed=seed)


def _scales(fmt):
    """two scales 1 dB apart, as a gain step leaves them: float for int16 and packed-12, double for the 8-bit formats"""
    if fmt == R.I16:
        a = np.float32(10 ** (3 / 20) / 32768)
        return float(a), float(np.float32(a * 10 ** (-1 / 20)))
    if fmt == R.PACKED12:
        return float(np.float32(1 / 2048)), float(np.float32(10 ** (-1 / 20) / 2048))
    a = 1.0 / (128 * 1.7)
    return a, a * 10 ** (1 / 20)


def _convert(fmt, words, lo, hi, scale, derand, cplx, use_ref):
    """the driver's conversion of samples [lo, hi) with one scale: float32 (REAL) or complex64 (I/Q)"""
    c = 2 if cplx else 1
    if fmt == R.I16:
        x = words[lo * c:hi * c]
        if derand:
            x = R.derandomize(x)
        y = x.astype(np.float32) * np.float32(scale)
    elif fmt == R.PACKED12:
        w = _pack(words[lo:hi])
        if use_ref:
            y = _ref_airspy_unpack(w, hi - lo, np.float32(scale))[0]
        else:
            from oracle import oracle as O
            y = O.airspy_unpack(w, hi - lo, np.float32(scale))[0]
    else:
        y = R.unpack8(words[lo * c:hi * c], fmt, scale)
    return y.view(np.complex64) if cplx else y


def _pack(s12):
    from oracle import oracle as O
    return O.airspy_pack(s12)


def _raw_write(dut, fmt, words, lo, hi, scale, derand, cplx):
    """one write from a thread of its own, so that the test's execute calls are served every block in order rather
    than the latest (the owner-thread shortcut, filter.c:681-683)"""
    c = 2 if cplx else 1
    if fmt == R.I16:
        x, kind = np.ascontiguousarray(words[lo * c:hi * c]), 3 if derand else 2
    else:
        x, kind = np.ascontiguousarray(_pack(words[lo:hi]) if fmt == R.PACKED12 else words[lo * c:hi * c]), 1
    return dut.lib.rd_write_once_from_thread(dut.h, x.ctypes.data, hi - lo, kind, fmt, scale)


def _float_write(s, y):
    y = np.ascontiguousarray(y)
    return s.lib.rd_write_once_from_thread(s.h, y.ctypes.data, len(y), 0, 0, 0.0)


def _ref_write(ref, y, start, L, shifts):
    """the floats of samples [start, start + len(y)) to the reference's filter.c in pieces that end on block boundaries,
    so that its inline execute serves each block as it fires: {job: [output of each channel]}"""
    out, pos = {}, 0
    while pos < len(y):
        nxt = min(len(y), ((start + pos) // L + 1) * L - start)
        if ref.write(y[pos:nxt]) == 1:
            out[(start + nxt) // L - 1] = [ref.execute(ch, sh) for ch, sh in enumerate(shifts)]
        pos = nxt
    return out


def _int_values(fmt, words, derand):
    if fmt == R.I16:
        return R.derandomize(words).astype(np.int64) if derand else words.astype(np.int64)
    if fmt == R.PACKED12:
        return R.unpack12(words)
    return R.values8(words, fmt)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c[0] for c in CASES])
def test_scale_changes_between_writes(oracle, cuda_dev, monkeypatch, cid):
    from oracle import spectrum as S

    from ka9q_radio_b200 import capi

    _, fmt, cplx, L, M, derand, spec_when, spec = _CASE[cid]
    lib, klib = _lib(), capi.load()
    M1, N = M - 1, L + M - 1
    fs = 50.0 * L
    grain = 8 if fmt == R.PACKED12 else 1
    cuts, changes = plan(L, M1, NB, grain, seed=[c[0] for c in CASES].index(cid))
    sA, sB = _scales(fmt)
    words = _source(fmt, cplx, NB * L, seed=3)
    use_ref = oracle.ref_available()
    bins = N if cplx else N // 2 + 1
    chans = [(L // 100, -0.4, 0.4, 11.0, N // 13), (L // 10, -0.45, 0.45, 9.0, -N // 29 if cplx else N // 5)]
    tuned_olen = L // 100
    ko = oracle.KO_COMPLEX if cplx else oracle.KO_REAL
    cap = float_ring_samples(L, M, cplx)
    # where the write plan must reach: a ring wrap inside a write, launches of 2 and 3 blocks, two changes in one
    # launch, a one-scale multi-block launch
    crossings = sum((a + M1) // cap != (b - 1 + M1) // cap for a, b in zip([0] + cuts[:-1], cuts))
    assert crossings > 0
    mixed_launches = one_scale_launches = 0
    errs = {"bitwise": [], "ref": [], "fdomain": [], "launches": [], "noise": [], "tuned": [], "spectrum": [],
            "spectrum_ref": []}
    stream = np.zeros(NB * L, np.complex64 if cplx else np.float32)
    window = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(spec[0]) / spec[0])).astype(np.float32) if spec else None
    polls_straddling = 0
    monkeypatch.setenv("KA9Q_GPU_SPECTRUM_D2H", "all")   # every bin of master->fdomain[], not the noise windows alone
    with Dut(lib, L, M, cplx) as d, Dut(lib, L, M, cplx) as a:
        ref = oracle.RefSession(L, M, ko) if use_ref else None
        for s in (d, a):
            for olen, lo, hi, beta, _ in chans:
                s.add(olen, lo, hi, beta)
            s.add(tuned_olen, -0.3, 0.3, 11.0)
            assert lib.rd_enable_noise(s.h, fs) == 0
        if ref is not None:
            for olen, lo, hi, beta, _ in chans:
                ref.add_channel(olen, lo, hi, beta)
        assert d.stats() == (0,) * 6
        if spec_when == "before":
            d.spec_setup(spec[0], spec[1], window)
            a.spec_setup(spec[0], spec[1], window)
        wcnt = job = 0
        scale, prev = sA, 0
        for w, end in enumerate(cuts):
            if prev in changes:
                scale = sB if scale == sA else sA
            y = _convert(fmt, words, prev, end, scale, derand, cplx, use_ref)
            stream[prev:end] = y
            fired, wcnt, job = launches(wcnt, job, end - prev, L)
            k0 = klib.kgpu_launch_count()
            fd = _raw_write(d, fmt, words, prev, end, scale, derand, cplx)
            k1 = klib.kgpu_launch_count()
            fa = _float_write(a, y)
            k2 = klib.kgpu_launch_count()
            assert fd == fa == (1 if fired else 0), w
            ref_out = _ref_write(ref, y, prev, L, [c[-1] for c in chans]) if ref is not None else {}
            assert sorted(ref_out) == ([j for j0, k in fired for j in range(j0, j0 + k)] if ref is not None else [])
            extra = 0
            mixed_jobs = set()
            for j0, k in fired:
                lo, hi = j0 * L - M1, (j0 + k) * L
                mixed = any(lo < c < hi for c in changes)
                mixed_launches += mixed
                one_scale_launches += (not mixed) and k > 1
                if mixed:
                    mixed_jobs |= set(range(j0, j0 + k))
                # the fused conversion costs no kernel of its own; the statistics one, the unpacks one each; a window
                # of several scales one conversion kernel for int16 and packed-12
                extra += {R.I16: 1, R.PACKED12: 2}.get(fmt, 1) + (mixed and fmt in (R.I16, R.PACKED12))
            if (k1 - k0) - (k2 - k1) != extra:
                errs["launches"].append((w, (k1 - k0) - (k2 - k1), extra))
            if spec_when == "after" and w == len(cuts) // 3:
                assert any(c < end for c in changes)   # set up after the first change
                d.spec_setup(spec[0], spec[1], window)
                a.spec_setup(spec[0], spec[1], window)
            for j0, k in fired:
                for j in range(j0, j0 + k):
                    bitwise = fmt not in (R.I16, R.PACKED12) or j in mixed_jobs
                    for ch, (*_, shift) in enumerate(chans):
                        yd, ya = d.exe(ch, shift), a.exe(ch, shift)
                        if bitwise and not same(yd, ya):
                            errs["bitwise"].append((j, ch, rel(yd, ya)))
                        elif not bitwise and rel(yd, ya) >= TOL:
                            errs["ref"].append((j, ch, "a", rel(yd, ya)))
                        if ref is not None:
                            r = ref_out[j][ch]
                            if rel(yd, r) >= TOL:
                                errs["ref"].append((j, ch, "b", rel(yd, r)))
                        nd_, na_ = lib.rd_noise(d.h, ch), lib.rd_noise(a.h, ch)
                        if not (np.isnan(nd_) and np.isnan(na_)) and not abs(nd_ - na_) <= TOL * abs(na_):
                            errs["noise"].append((j, ch, nd_, na_))
                    fdd, fda = d.fdomain(j, bins), a.fdomain(j, bins)
                    if bitwise and not same(fdd, fda):
                        errs["fdomain"].append((j, rel(fdd, fda)))
                    _, shift, rem = oracle.compute_tuning(N, fs, 0.1234 * fs + 1000 * j)
                    (yd, pd), (ya, pa) = d.tuned(2, shift, rem, fs / 100), a.tuned(2, shift, rem, fs / 100)
                    if rel(yd, ya) >= TOL or not abs(pd - pa) <= TOL * abs(pa):
                        errs["tuned"].append((j, rel(yd, ya), pd, pa))
            if fired and spec is not None and (spec_when == "before" or w >= len(cuts) // 3):
                fft_n, nbins, shift = spec
                (gd, ed), (ga, ea) = d.spec_poll(shift, FFT_AVG, OVERLAP, nbins), a.spec_poll(shift, FFT_AVG, OVERLAP, nbins)
                assert ed == ea == job * L
                adjust = round(fft_n * (1 + (FFT_AVG - 1) * (1 - OVERLAP)))
                polls_straddling += any(ed - adjust < c < ed for c in changes)
                try:
                    close_to(gd, ga)
                except AssertionError:
                    errs["spectrum"].append((w, rel(gd, ga)))
                ring = np.zeros(cap, stream.dtype)
                q = np.arange(max(0, ed - cap), ed)
                ring[(q + M1) % cap] = stream[q]
                pos = (ed + M1) % cap
                try:
                    close_to(gd, S.wideband_spectrum(not cplx, fft_n, nbins, window, shift, FFT_AVG, OVERLAP, ring, pos))
                    if S.have_ref():
                        own, used = S.ref_wideband_poll(not cplx, fft_n, nbins, window, shift, FFT_AVG, OVERLAP, ring, pos)
                        assert used == FFT_AVG
                        close_to(gd, own)
                except AssertionError:
                    errs["spectrum_ref"].append((w, rel(gd, S.wideband_spectrum(not cplx, fft_n, nbins, window, shift,
                                                                                 FFT_AVG, OVERLAP, ring, pos))))
            prev = end
        got = d.stats()
        if ref is not None:
            ref.close()
    assert mixed_launches >= 5 and one_scale_launches >= 1
    assert spec is None or polls_straddling >= 1
    fired_blocks = job
    want = R.block_stats(_int_values(fmt, words, derand), R.I16 if fmt == R.I16 else fmt, L, cplx)[:fired_blocks]
    assert list(got[:5]) == [fired_blocks, fired_blocks * L] + [sum(s[k] for s in want) for k in range(3)]
    assert got[5] == R.since_over(want, L)
    report = {k: (len(v), max(e[-1] for e in v) if k in ("bitwise", "ref", "fdomain", "spectrum", "spectrum_ref") else v[:3])
              for k, v in errs.items() if v}
    assert not any(errs.values()), f"{cid}: {mixed_launches} mixed-scale launches; failures (count, worst): {report}"


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [R.U8, R.I16], ids=["u8", "int16"])
def test_lapped_slave_across_a_scale_change(cuda_dev, fmt):
    """A consumer that fell ND blocks behind a producer thread whose scale changed gets zeros and a drop, as one fed the
    converted floats does, then the same correctly scaled blocks."""
    lib = _lib()
    L, M = 36000, 9001
    sA, sB = _scales(fmt)
    words = _source(fmt, True, 8 * L, seed=4)
    kind, c = (1, 2) if fmt == R.U8 else (2, 4)
    flo = np.concatenate([_convert(fmt, words, 0, 3 * L, sA, False, True, False),
                          _convert(fmt, words, 3 * L, 6 * L, sB, False, True, False)])
    with Dut(lib, L, M, True, nworkers=1) as d, Dut(lib, L, M, True, nworkers=1) as a:
        for s in (d, a):
            s.add(480, -0.3, 0.3, 9.0)
        w8 = np.ascontiguousarray(words)
        assert lib.rd_write_from_thread(d.h, w8.ctypes.data, L, 3, c * L, kind, fmt, sA) == 0
        assert lib.rd_write_from_thread(d.h, w8.ctypes.data + 3 * c * L, L, 3, c * L, kind, fmt, sB) == 0
        assert lib.rd_write_from_thread(a.h, flo.ctypes.data, L, 6, 8 * L, 0, 0, 0.0) == 0
        for _ in range(4):
            yd, ya = d.exe(0, 1500), a.exe(0, 1500)
            assert (same(yd, ya) if fmt == R.U8 else rel(yd, ya) < TOL or not np.abs(ya).max())
        assert lib.rd_drops(d.h, 0) == lib.rd_drops(a.h, 0) >= 1


@pytest.mark.gpu
def test_scale_table_overflow_is_rejected(cuda_dev):
    """A write whose scale change would overflow the master's table of changes returns -1 and stores nothing; the table
    holds 64 + 16 ceil(S / L) changes, S the samples of the master's float ring, and frees as the stream moves on."""
    lib = _lib()
    L, M = 48000, 12001
    S_ = float_ring_samples(L, M, False)
    cap = 64 + 16 * -(-S_ // L)
    sA, sB = _scales(R.I16)
    words = _source(R.I16, False, 12 * L, seed=6)
    with Dut(lib, L, M, False) as d, Dut(lib, L, M, False) as a:
        for s in (d, a):
            s.add(480, -0.3, 0.3, 11.0)
        pos, scale = 0, sA
        for i in range(cap + 1):            # the first write sets the scale; each later one is a change
            scale = sA if i % 2 == 0 else sB
            assert d.i16(words[pos:pos + 1], scale) == 0, i
            assert a.flt(_convert(R.I16, words, pos, pos + 1, scale, False, False, False)) == 0
            pos += 1
        other = sB if scale == sA else sA
        assert d.i16(words[pos:pos + 1], other) == -1
        for lo in range(pos, 8 * L, 4000):   # the rejected sample is written again, at the scale in force
            hi = min(lo + 4000, 8 * L)
            fd = d.i16(words[lo:hi], scale)
            assert fd == a.flt(_convert(R.I16, words, lo, hi, scale, False, False, False)) >= 0
            if fd:
                yd, ya = d.exe(0, 3000), a.exe(0, 3000)
                assert rel(yd, ya) < TOL
        assert d.i16(words[8 * L:8 * L + 1], other) == 0   # the old changes have left the table
