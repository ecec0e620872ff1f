#!/usr/bin/env python3
"""Bitwise A/B of the forward spectra and channel outputs of two builds of the library (needs a GPU).

usage: spectra_ab.py --dump DIR       run the seeded cases below with the library of this tree and write every result to DIR
       spectra_ab.py --compare A B    compare two such dumps bit by bit; exit status 1 on any difference

Cases: cfg-2 (REAL int16, 32 blocks from block 3, the workload's 1024 channels), cfg-2 with float input, and REAL masters
on fwd_rows_v2 with other row counts (odd n1 included), plus the COMPLEX 1296 x 1250 master."""
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


def dump(out: Path):
    import torch
    sys.path.insert(0, str(ROOT))
    from ka9q_radio_b200 import capi, workloads
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
a = ap.parse_args()
if a.dump:
    dump(a.dump)
else:
    sys.exit(compare(*a.compare))
