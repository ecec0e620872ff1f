"""Small masters (create_filter_input_small) through filter.h, against the reference's own filter.c.

tests/abi/small_driver.c opens filter_driver.c's sessions with create_filter_input_small; it is built against our header
(tests/abi/_build/small_driver.so) and against the reference's src/filter.h (oracle/_ref/small_driver_refhdr.so, where
built).  Each check runs the same calls on the reference's filter.c (oracle/_ref/libka9qref.so) and compares at TOL; the
small path is also compared with a default master fed the same samples (1e-6 relative, responses bitwise).
"""
import ctypes as C
import threading
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
TOL = 1e-5
SAME = 1e-6   # small path against a default master of the same geometry: the transforms differ in rounding only
KO_COMPLEX, KO_REAL = 1, 2
f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
c64p = np.ctypeslib.ndpointer(np.complex64, flags="C_CONTIGUOUS")
DRIVERS = ["tests/abi/_build/small_driver.so", "oracle/_ref/small_driver_refhdr.so"]


def _bind(path):
    p = ROOT / path
    if not p.exists():
        return None
    from oracle import oracle as O

    lib = O.bind_driver(C.CDLL(str(p)))
    lib.small_set_mode.argtypes = [C.c_int]
    lib.ref_execute_channel_real.argtypes = [C.c_void_p, C.c_int, C.c_int, f32p]
    lib.ref_produce_from_thread.argtypes = [C.c_void_p, f32p, C.c_int]
    lib.ref_lap_probe.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, c64p]
    lib.ref_lap_probe.restype = C.c_uint
    lib.ref_channel_next_job.argtypes = [C.c_void_p, C.c_int]
    lib.ref_channel_next_job.restype = C.c_uint
    lib.small_threads.restype = C.c_longlong
    lib.small_threads.argtypes = [C.c_int] * 5 + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
    if hasattr(lib, "small_refusals"):
        lib.small_refusals.argtypes = [C.c_void_p, C.c_int]
    return lib


def _driver(path):
    lib = _bind(path)
    if lib is None:
        pytest.skip(f"{path} not built")
    return lib


def _rel(a, b):
    return float(np.abs(a - b).max()) / max(float(np.abs(b).max()), 1e-30)


class Sess:
    """A session on `lib` (small when small=True, checked), or on the reference's filter.c when lib is None."""

    def __init__(self, oracle, lib, L, M, in_type, small=False, nworkers=0):
        if lib is not None:
            lib.small_set_mode(int(small))
        self.s = oracle.RefSession(L, M, in_type, nworkers=nworkers, lib=lib)
        if lib is not None:
            assert lib.small_last_taken() == int(small)
        self.lib = self.s.R
        self.types = []

    def add(self, olen, low, high, beta, out_type=KO_COMPLEX, isb=False):
        i = self.s.add_channel(olen, low, high, beta, out_type=out_type)
        if isb:
            self.s.set_isb(i, True)
        self.types.append(out_type)
        return i

    def execute(self, i, shift):
        if self.types[i] == KO_REAL and not hasattr(self.lib, "small_set_mode"):   # oracle/ref_driver.c: floats into dst
            return self.s.execute(i, shift).view(np.float32)[: self.s.olen[i]].copy()
        if self.types[i] == KO_REAL:
            y = np.empty(self.s.olen[i], np.float32)
            assert self.lib.ref_execute_channel_real(self.s.h, i, int(shift), y) == 0
            return y
        return self.s.execute(i, shift)

    def close(self):
        self.s.close()


def _run(oracle, lib, L, M, in_type, slaves, x, nb, small, shifts=None, events=None):
    """nb blocks written one by one; every slave read after each.  shifts[b][i]; events: {block: fn(sess)} before block b."""
    s = Sess(oracle, lib, L, M, in_type, small=small)
    ids = [s.add(*sl) for sl in slaves]
    out = []
    for b in range(nb):
        if events and b in events:
            events[b](s)
        assert s.s.write(x[b * L:(b + 1) * L]) == 1
        out.append([s.execute(i, shifts[b][i] if shifts else 0) for i in ids])
    # slave->response holds `bins` elements: points (COMPLEX output) or points / 2 + 1 (REAL output, filter.c:372-392)
    resp = [s.s.response(i)[: len(s.s.response(i)) // 2 + 1 if t == KO_REAL else None] for i, t in zip(ids, s.types)]
    s.close()
    return out, resp


def _check(oracle, lib, L, M, in_type, slaves, x, nb, shifts=None, events=None):
    """Every block of every slave against the reference and against a default master, relative to the slave's largest
    output over the stream: when M - 1 exceeds L (filter2 at blocking 10: M = 5793, L = 2400) block 0 holds only the
    filter's onset, about 1e-3 of the steady output, and both paths' float rounding is then a large part of it."""
    ref, _ = _run(oracle, None, L, M, in_type, slaves, x, nb, False, shifts, events)
    small, rs = _run(oracle, lib, L, M, in_type, slaves, x, nb, True, shifts, events)
    dflt, rd = _run(oracle, lib, L, M, in_type, slaves, x, nb, False, shifts, events)
    for i in range(len(slaves)):
        scale = max(float(np.abs(ref[b][i]).max()) for b in range(nb))
        for b in range(nb):
            assert float(np.abs(small[b][i] - ref[b][i]).max()) / scale < TOL, (b, i)
            assert float(np.abs(small[b][i] - dflt[b][i]).max()) / scale < SAME, (b, i)
    for a, d in zip(rs, rd):
        assert a.tobytes() == d.tobytes()   # slave->response: bitwise what a default master holds


@pytest.mark.gpu
@pytest.mark.parametrize("driver", DRIVERS)
@pytest.mark.parametrize("L", [240, 480, 960, 2400])
@pytest.mark.parametrize("isb", [False, True])
def test_filter2_matches_reference(oracle, cuda_dev, driver, L, isb):
    """radio.c:1572-1583: COMPLEX, N = round2(2 L), one slave of olen L read with shift 0, for 24 blocks.  L = blocking x
    240 (12 kHz, 20 ms): blockings 1, 2, 4 and 10."""
    lib = _driver(driver)
    N = 1 << (2 * L - 1).bit_length()
    nb = 24
    x = oracle.siggen_complex(nb * L, 0.1, 0.02, 0.0371, 1.0)
    _check(oracle, lib, L, N - L + 1, KO_COMPLEX, [(L, -0.21, 0.07, 7.0, KO_COMPLEX, isb)], x, nb)


@pytest.mark.gpu
def test_cascade_with_a_small_second_stage(oracle, cuda_dev):
    """test_secondary_complex_master_like_filter2 with the second stage (COMPLEX 480 / 97) made small."""
    lib = _driver(DRIVERS[0])
    L, M, nb = 48000, 12001, 6
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.25, 1.0)
    ch = dict(olen=480, shift=15000, low=-1 / 3, high=1 / 3, beta=11.0)
    first, _ = oracle.run_stream(x, L, M, [ch])
    mid = np.concatenate([first[b][0] for b in range(nb)]).astype(np.complex64)
    L2, M2 = 480, 97
    second, _ = oracle.run_stream(mid, L2, M2, [dict(olen=480, shift=0, low=-0.125, high=0.125, beta=7.0)])
    s1 = Sess(oracle, lib, L, M, KO_REAL, small=False)
    s2 = Sess(oracle, lib, L2, M2, KO_COMPLEX, small=True)
    a, b2 = s1.add(480, -1 / 3, 1 / 3, 11.0), s2.add(480, -0.125, 0.125, 7.0)
    for b in range(nb):
        assert s1.s.write(x[b * L:(b + 1) * L]) == 1
        y = s1.execute(a, 15000)
        assert _rel(y, first[b][0]) < TOL
        assert s2.s.write(y) == 1
        assert _rel(s2.execute(b2, 0), second[b][0]) < 2 * TOL, b
    s1.close()
    s2.close()


def _composite_slaves(oracle):
    """wfm.c:70-89 at 384 kHz and Blocktime 20 ms: REAL 7680 / 7681, mono REAL, pilot and L-R COMPLEX, audio_L = 960,
    the pilot and subcarrier shifts of compute_tuning."""
    _, pilot, _ = oracle.compute_tuning(15360, 384000.0, 19000.0)
    _, sub, _ = oracle.compute_tuning(15360, 384000.0, 38000.0)
    slaves = [(960, 50 / 48000, 15000 / 48000, 11.0, KO_REAL), (960, -100 / 48000, 100 / 48000, 11.0, KO_COMPLEX),
              (960, -15000 / 48000, 15000 / 48000, 11.0, KO_COMPLEX)]
    return slaves, [0, pilot, sub]


@pytest.mark.gpu
@pytest.mark.parametrize("driver", DRIVERS)
def test_wfm_composite_matches_reference(oracle, cuda_dev, driver):
    lib = _driver(driver)
    L, M, nb = 7680, 7681, 12
    slaves, shifts = _composite_slaves(oracle)
    assert shifts[1] > 0 and shifts[2] > 0
    x = (oracle.siggen_real(nb * L, 0.1, 0.01, 19000 / 384000, 1.0) + oracle.siggen_real(nb * L, 0.05, 0.01, 38000 / 384000 + 1e-3, 1.0))
    _check(oracle, lib, L, M, KO_REAL, slaves, x.astype(np.float32), nb, shifts=[shifts] * nb)


@pytest.mark.gpu
@pytest.mark.parametrize("driver", DRIVERS)
def test_retune_and_filter_swap_mid_stream(oracle, cuda_dev, driver):
    """A shift change (block 5) and a set_filter swap (block 9) take the recompute-from-stored-spectrum entry, then rejoin
    the launch; ISB is switched on at block 13."""
    lib = _driver(driver)
    L, M, nb = 4800, 1201, 18   # REAL N = 6000: Nc = 3000
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.31, 1.0)
    shifts = [[1800, 1700]] * 5 + [[1801, -1700]] * 13
    events = {9: lambda s: s.lib.ref_retune_channel(s.s.h, 1, -0.1, 0.1, 11.0),
              13: lambda s: s.s.set_isb(0, True)}
    _check(oracle, lib, L, M, KO_REAL, [(48, -0.3, 0.3, 9.0), (96, -0.2, 0.4, 5.0)], x, nb, shifts=shifts, events=events)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 3])
def test_write_that_completes_several_blocks(oracle, cuda_dev, k):
    """One write of k L samples fires one launch of k blocks; a consumer thread other than the writer then reads them in
    order (filter.c:680-707)."""
    lib = _driver(DRIVERS[0])
    L, M = 480, 545
    nb = 1 + 2 * k
    x = oracle.siggen_complex(nb * L, 0.1, 0.02, 0.0371, 1.0)
    slaves = [(L, -0.21, 0.07, 7.0)]
    ref, _ = _run(oracle, None, L, M, KO_COMPLEX, slaves, x, nb, False)
    s = Sess(oracle, lib, L, M, KO_COMPLEX, small=True, nworkers=1)
    c = s.add(*slaves[0])
    lib.ref_write_complex.argtypes = [C.c_void_p, c64p, C.c_int]
    spans = [(0, 1)] + [(1 + j * k, 1 + (j + 1) * k) for j in range(2)]
    for lo, hi in spans:
        chunk = np.ascontiguousarray(x[lo * L:hi * L])
        t = threading.Thread(target=lambda: lib.ref_write_complex(s.s.h, chunk, (hi - lo) * L))
        t.start()
        t.join()
        for b in range(lo, hi):
            assert _rel(s.execute(c, 0), ref[b][0]) < TOL, b
    assert lib.ref_channel_drops(s.s.h, c) == 0
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("driver", DRIVERS)
def test_lapped_slave_gets_zeros_and_a_drop(oracle, cuda_dev, driver):
    """test_filter_abi's lap sequence on a small master: ND blocks behind gives zeros and block_drops++, then the
    consumer catches up block by block."""
    lib = _driver(driver)
    L, M, nb = 4800, 1201, 9
    N = L + M - 1
    x = oracle.siggen_real(nb * L, 0.1, 0.02, 0.31, 1.0)
    R = oracle.design_response(60, 48, N, True, -0.3, 0.3, 9.0)
    s = Sess(oracle, lib, L, M, KO_REAL, small=True, nworkers=1)
    h = s.s.h
    a = s.add(48, -0.3, 0.3, 9.0)
    assert lib.ref_produce_from_thread(h, x[: 2 * L], 2) == 0
    y = np.empty(48, np.complex64)
    for blk in range(2):
        assert lib.ref_lap_probe(h, a, 1800, None, 0, y) == 0
        r = oracle.channel_block(oracle.KO_REAL, oracle.forward(oracle.block_window(x, L, M, blk)), R, 1800)[-48:]
        assert _rel(y, r) < TOL
    assert lib.ref_produce_from_thread(h, np.ascontiguousarray(x[2 * L: 8 * L]), 6) == 0
    y[:] = 1
    assert lib.ref_lap_probe(h, a, 1800, None, 0, y) == 1
    assert not y.any() and lib.ref_channel_next_job(h, a) == 3
    y[:] = 1
    assert lib.ref_lap_probe(h, a, 1800, None, 0, y) == 2
    assert not y.any()
    for blk in (4, 5, 6, 7):
        assert lib.ref_lap_probe(h, a, 1800, None, 0, y) == 2
        r = oracle.channel_block(oracle.KO_REAL, oracle.forward(oracle.block_window(x, L, M, blk)), R, 1800)[-48:]
        assert _rel(y, r) < TOL, blk
    s.close()


def _threads(lib, P, L, M, in_type, slaves, shifts, x, nb, small, keep=True):
    """small_threads: (slowest thread's ns, outputs [P][per] or None, masters that took the small path)"""
    n = len(slaves)
    olen = (C.c_int * n)(*[s[0] for s in slaves])
    lo, hi, beta = ((C.c_double * n)(*[s[j] for s in slaves]) for j in (1, 2, 3))
    otype = (C.c_int * n)(*[s[4] for s in slaves])
    sh = (C.c_int * n)(*shifts)
    per = nb * sum(2 * s[0] for s in slaves)
    out = np.zeros(P * per if keep else 1, np.float32)
    count = C.c_int(0)
    lib.small_set_mode(int(small))
    t = lib.small_threads(P, L, M, in_type, n, C.cast(olen, C.c_void_p), C.cast(otype, C.c_void_p), C.cast(lo, C.c_void_p),
                          C.cast(hi, C.c_void_p), C.cast(beta, C.c_void_p), C.cast(sh, C.c_void_p), nb, x.ctypes.data,
                          out.ctypes.data if keep else None, C.byref(count))
    return t, out.reshape(P, per) if keep else None, count.value


@pytest.mark.gpu
def test_64_threads_each_with_a_composite(oracle, cuda_dev):
    lib = _driver(DRIVERS[0])
    L, M, nb, P = 7680, 7681, 8, 64
    slaves, shifts = _composite_slaves(oracle)
    x = oracle.siggen_real(nb * L, 0.1, 0.01, 19000 / 384000, 1.0)
    ref, _ = _run(oracle, None, L, M, KO_REAL, slaves, x, nb, False, shifts=[shifts] * nb)
    t, out, count = _threads(lib, P, L, M, KO_REAL, slaves, shifts, x, nb, small=True)
    assert t > 0 and count == P
    for p in range(P):
        o = 0
        for b in range(nb):
            for i, sl in enumerate(slaves):
                seg = out[p, o:o + 2 * sl[0]]
                got = seg[:sl[0]] if sl[4] == KO_REAL else seg.view(np.complex64)
                assert _rel(got, ref[b][i]) < TOL, (p, b, i)
                o += 2 * sl[0]


@pytest.mark.gpu
def test_refused_extensions(oracle, cuda_dev):
    lib = _driver(DRIVERS[0])
    L, M = 960, 961
    s = Sess(oracle, lib, L, M, KO_REAL, small=True)
    a = s.add(960, -0.2, 0.2, 11.0)
    assert s.s.write(oracle.siggen_real(L, 0.1, 0.02, 0.1, 1.0)) == 1
    assert lib.small_refusals(s.s.h, a) == 0
    s.close()
    # outside the envelope the session falls back to create_filter_input, and nothing is refused
    lib.small_set_mode(1)
    s = oracle.RefSession(1000, 28, KO_COMPLEX, lib=lib)   # N = 1027 = 13 x 79
    assert lib.small_last_taken() == 0
    s.close()
