#!/usr/bin/env python3
"""Bitwise A/B of the forward spectra and channel outputs of two builds of the library (needs a GPU).

usage: spectra_ab.py --dump DIR       run the seeded cases below with the library of this tree and write every result to DIR
       spectra_ab.py --compare A B    compare two such dumps bit by bit; exit status 1 on any difference

Cases: cfg-2 (REAL int16, 32 blocks from block 3, the workload's 1024 channels), cfg-2 with float input, and REAL masters
on fwd_rows_v2 with other row counts (odd n1 included), plus the COMPLEX 1296 x 1250 master.  Then every Bluestein
transform: REAL 62 MS/s and COMPLEX 2.9 MS/s masters (kgpu_master_create_any; int16 with statistics, float), a bank of
725-, 1550- and 44 000-point channels on each (responses, outputs, oscillator channels with block power), and spectrum
polls at the REAL and COMPLEX fft_n 104 400, short and long enough to run in chunks of segments.  Then every channel
path on a REAL and a COMPLEX master (L = 48000, M = 12001): one bank with every length of PATH_POINTS in every variant
that length's path serves, run batched with and without block power, again with the specialised kernels off, and one
channel of each length alone (kgpu_bank_run_one_ex).

--lib PATH dumps with another build of libka9qgpu.so, such as the parent commit's, in place of this tree's."""
import argparse, sys
from pathlib import Path
import numpy as np

ROOT = Path(__file__).resolve().parent.parent
CASES = [  # (name, L, M, real, int16 input, blocks, first block, channels of cfg-2)
    ("cfg2_i16", 2592000, 648001, True, True, 32, 3, True),
    ("cfg2_f32", 2592000, 648001, True, False, 4, 1, True),
    ("r1280x1250_f32", 2560000, 640001, True, False, 3, 1, False),
    ("r1323x1250_f32", 2646000, 661501, True, False, 3, 1, False),
    ("r1875x1250_i16", 3750000, 937501, True, True, 3, 1, False),
    ("r1250x1250_f32", 2500000, 625001, True, False, 3, 1, False),
    ("c1296x1250_i16", 1296000, 324001, False, True, 3, 1, False),
]
BLUESTEIN_MASTERS = [  # (name, L, M, real, int16 input, blocks); N / L = 5 / 4 for both
    ("b62m_i16", 1240000, 310001, True, True, 3),
    ("b62m_f32", 1240000, 310001, True, False, 2),
    ("b2m9_c_i16", 58000, 14501, False, True, 3),
    ("b2m9_c_f32", 58000, 14501, False, False, 3),
]
BLUESTEIN_POINTS = (725, 1550, 44000)  # channels with no transform of their own: 5^2 29, 2 5^2 31, 2^5 5^3 11
BLUESTEIN_SPECTRA = [  # (name, fft_n, real, int16 ring, fft_avg); 100 segments run in chunks of 39
    ("s104400_r_i16", 104400, True, True, 3),
    ("s104400_r_i16_long", 104400, True, True, 100),
    ("s104400_c_f32", 104400, False, False, 3),
    ("s104400_c_f32_long", 104400, False, False, 100),
]
# Every channel path: chan_v2 (600, 300), chan_static (1200), chan_kernel (480: 7-smooth, no specialised kernel), wide
# (9600), huge (38 400), extended narrow and wide (5500, 8800) and Bluestein (725, 1550, 44 000); points = 5 olen / 4.
PATH_POINTS = (600, 300, 1200, 480, 9600, 38400, 5500, 8800, 725, 1550, 44000)
PATH_NB = 3


def _path_variants(real: bool, bins: int, pts: int):
    """(name, shift, flags, REAL output, oscillator) of each variant a channel path serves on this master"""
    from ka9q_radio_b200 import capi

    v = [("up", bins // 5, 0, False, False), ("isb", bins // 3, capi.KGPU_CHAN_ISB, False, False),
         ("osc", bins // 4, 0, False, True)]
    if pts % 2 == 0:  # REAL output needs an even length
        v.append(("realout", bins // 6, 0, True, False))
    if real:  # an inverted spectrum, and a channel with no overlap at all (with its zero block power)
        return v + [("inv", -(bins // 5), 0, False, True), ("none", bins + pts, 0, False, True)]
    return v + [("wrap", 17, 0, False, True), ("beam", bins // 7, capi.KGPU_CHAN_BEAM, False, False)]


def dump_paths(out: Path, dev):
    import torch
    from ka9q_radio_b200 import capi

    lib = capi.load()
    st = torch.cuda.current_stream(dev).cuda_stream
    L, M, nb = 48000, 12001, PATH_NB
    for name, real in (("paths_r", True), ("paths_c", False)):
        rng = np.random.default_rng(L + M + real)
        host = rng.standard_normal((nb * L + M - 1) * (1 if real else 2), dtype=np.float32)
        m = capi.Master(L, M, capi.KGPU_REAL if real else capi.KGPU_COMPLEX)
        chans = [(pts,) + v for pts in PATH_POINTS for v in _path_variants(real, m.bins, pts)]
        b = capi.Bank(m, len(chans))
        try:
            print(f"{name}: {m.describe()}, {len(chans)} channels")
            for i, (pts, _, shift, flags, realout, osc) in enumerate(chans):
                assert b.define_any(i, pts * 4 // 5, capi.KGPU_REAL if realout else capi.KGPU_COMPLEX) == pts
                b.set_filter(i, 0.05 if realout else -0.3, 0.4 if realout else 0.35, 11.0)
                b.set_shift(i, shift)
                if flags & capi.KGPU_CHAN_BEAM:
                    b.set_weights(i, 0.6, 0.3)
                if flags:
                    b.set_flags(i, flags)
                if osc:
                    b.set_osc(i, True, 0.1 + 0.01 * i, 1e-3, 1e-9, 0.01)
            spec = torch.empty((nb, m.spec_stride), dtype=torch.complex64, device=dev)
            m.forward(torch.from_numpy(host).to(dev).data_ptr(), capi.KGPU_FMT_F32, 1.0, nb, spec.data_ptr(), st)
            res = {"spec": spec[:, :m.bins]}
            for static in (1, 0):
                lib.kgpu_use_static_kernels(static)
                o = torch.zeros((nb, b.out_stride), dtype=torch.complex64, device=dev)
                b.run(spec.data_ptr(), nb, o.data_ptr(), st)
                res[f"chan_s{static}"] = o
                o = torch.zeros((nb, b.out_stride), dtype=torch.complex64, device=dev)
                power = torch.zeros((nb, len(chans)), dtype=torch.float32, device=dev)
                b.run(spec.data_ptr(), nb, o.data_ptr(), st, power.data_ptr())
                res[f"chan_pw_s{static}"], res[f"power_s{static}"] = o, power
            lib.kgpu_use_static_kernels(1)
            for i, (pts, vname, *_rest) in enumerate(chans):  # one channel of each length alone: its oscillator variant
                if vname != "osc":
                    continue
                o = torch.zeros(pts, dtype=torch.complex64, device=dev)
                power = torch.zeros(1, dtype=torch.float32, device=dev)
                capi.check(lib.kgpu_bank_run_one_ex(b.h, i, spec[1].data_ptr(), o.data_ptr(), power.data_ptr(), st),
                           "kgpu_bank_run_one_ex")
                res[f"one{pts}"], res[f"one{pts}_power"] = o, power
            torch.cuda.synchronize()
            for k, v in res.items():
                _save(out, f"{name}.{k}", v)
        finally:
            lib.kgpu_use_static_kernels(1)
            b.close()
            m.close()


def _save(out: Path, name: str, v):
    import torch
    a = v.contiguous().cpu().numpy() if isinstance(v, torch.Tensor) else np.ascontiguousarray(v)
    np.save(out / f"{name}.npy", a.view(np.int32))


def dump_bluestein(out: Path, dev):
    import torch
    from ka9q_radio_b200 import capi

    st = torch.cuda.current_stream(dev).cuda_stream
    for name, L, M, real, i16, nb in BLUESTEIN_MASTERS:
        rng = np.random.default_rng(L + M + nb + i16)
        per = 1 if real else 2
        n = (nb * L + M - 1) * per
        host = rng.integers(-3000, 3000, n, dtype=np.int16) if i16 else rng.standard_normal(n, dtype=np.float32)
        m = capi.Master(L, M, capi.KGPU_REAL if real else capi.KGPU_COMPLEX, any_length=True)
        b = capi.Bank(m, 8)
        try:
            print(f"{name}: {m.describe()}")
            x = torch.from_numpy(host).to(dev)
            spec = torch.empty((nb, m.spec_stride), dtype=torch.complex64, device=dev)
            stats = torch.zeros((nb, 2), dtype=torch.int64, device=dev)  # IngestStats: energy, clips
            m.forward(x.data_ptr(), capi.KGPU_FMT_I16 if i16 else capi.KGPU_FMT_F32, 1 / 3000 if i16 else 1.0, nb, spec.data_ptr(),
                      st, derandomize=i16, d_stats=stats.data_ptr() if i16 else 0)
            res = {"spec": spec[:, :m.bins]}
            if i16:
                res["stats"] = stats
            # channels 0-2 plain, 3-5 the same lengths with an oscillator
            for i in range(6):
                pts = BLUESTEIN_POINTS[i % 3]
                assert b.define_any(i, pts * L // m.N) == pts
                b.set_filter(i, -0.3 + 0.05 * i, 0.35 - 0.04 * i, 11.0)
                b.set_shift(i, (m.bins // 7) * (i + 1) * (1 if real or i % 2 else -1))
                if i >= 3:
                    b.set_osc(i, True, 0.1 * i, 1e-3 * i, 1e-9 * i, 0.01 * i)
                res[f"resp{i}"] = b.get_response(i, pts)
            o = torch.empty((nb, b.out_stride), dtype=torch.complex64, device=dev)
            b.run(spec.data_ptr(), nb, o.data_ptr(), st)
            res["chan"] = o.clone()
            power = torch.zeros((nb, 8), dtype=torch.float32, device=dev)
            b.run(spec.data_ptr(), nb, o.data_ptr(), st, power.data_ptr())
            res["chan_osc"], res["power"] = o, power
            torch.cuda.synchronize()
            for k, v in res.items():
                _save(out, f"{name}.{k}", v)
        finally:
            b.close()
            m.close()
    for name, fft_n, real, i16, avg in BLUESTEIN_SPECTRA:
        rng = np.random.default_rng(fft_n + avg + real)
        samples = 1_000_003
        n = samples * (1 if real else 2)
        ring = torch.from_numpy(rng.integers(-3000, 3000, n, dtype=np.int16) if i16 else rng.standard_normal(n, dtype=np.float32))
        s = capi.Spectrum(fft_n, capi.KGPU_REAL if real else capi.KGPU_COMPLEX, 4001)
        try:
            print(f"{name}: {s.describe()}")
            s.set_window(np.hanning(fft_n).astype(np.float32))
            bins = torch.zeros(4001, dtype=torch.float32, device=dev)
            s.run(ring.to(dev), 987_654, -1234 if real else 777, avg, 0.5, bins, scale=1 / 3000 if i16 else 1.0, derandomize=i16)
            torch.cuda.synchronize()
            _save(out, f"{name}.bins", bins)
        finally:
            s.close()


def dump(out: Path, lib: Path | None):
    import torch
    sys.path.insert(0, str(ROOT))
    from ka9q_radio_b200 import capi, workloads

    if lib:
        capi.LIB_PATH = lib.resolve()
    from ka9q_radio_b200.channelizer import Channelizer

    out.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cuda:0")
    W = workloads.by_name("cfg2")
    for name, L, M, real, i16, nb, b0, chans in CASES:
        rng = np.random.default_rng(L + M)
        per = 1 if real else 2
        n = ((nb + b0) * L + M - 1) * per
        host = rng.integers(-3000, 3000, n, dtype=np.int16) if i16 else rng.standard_normal(n, dtype=np.float32)
        cz = Channelizer(L, M, capi.KGPU_REAL if real else capi.KGPU_COMPLEX, dev, capacity=max(1, len(W.channels)))
        try:
            print(f"{name}: {cz.master.describe()}")
            if chans:
                for c in W.channels:
                    cz.add_channel(c.olen, c.shift, c.low, c.high, c.beta)
            spec = cz.alloc_spectra(nb)
            cz.forward(torch.from_numpy(host).to(dev), nb, spec, scale=W.scale if i16 else 1.0, first_block=b0)
            res = {"spec": spec[:, :cz.master.bins]}
            if chans:
                o = cz.alloc_outputs(nb)
                cz.channels(spec, nb, o)
                res["chan"] = o
            torch.cuda.synchronize()
            for k, v in res.items():
                np.save(out / f"{name}.{k}.npy", v.contiguous().view(torch.int32).cpu().numpy())
        finally:
            cz.close()
    dump_bluestein(out, dev)
    dump_paths(out, dev)


def compare(a: Path, b: Path) -> int:
    files = sorted(p.name for p in a.glob("*.npy"))
    if not files or files != sorted(p.name for p in b.glob("*.npy")):
        print("the dumps hold different files:", files, sorted(p.name for p in b.glob("*.npy")))
        return 1
    bad = 0
    for f in files:
        x, y = np.load(a / f), np.load(b / f)
        diff = int((x != y).sum()) if x.shape == y.shape else -1
        print(f"{f:28s} {x.size:11d} words  {'identical' if diff == 0 else f'DIFFERENT ({diff} words)'}")
        bad += diff != 0
    print("all identical" if not bad else f"{bad} file(s) differ")
    return 1 if bad else 0


ap = argparse.ArgumentParser()
g = ap.add_mutually_exclusive_group(required=True)
g.add_argument("--dump", type=Path)
g.add_argument("--compare", type=Path, nargs=2)
ap.add_argument("--lib", type=Path, help="with --dump: the libka9qgpu.so to dump with (default: this tree's)")
a = ap.parse_args()
if a.dump:
    dump(a.dump, a.lib)
else:
    sys.exit(compare(*a.compare))
