#!/usr/bin/env python3
"""Forward-pass time of the extended pair (fwd_cols_ext + fwd_rows_ext) against the generic pair (needs a GPU).

usage: ext_primes_bench.py [--blocks B] [--iters K] [--rounds R]
Masters: AirspyHF+ 912 kS/s (COMPLEX, 22 800 points), RX888 at 60.8 MS/s (REAL, 760 000 complex points), both extended,
and RX888 at 64.8 MS/s (REAL 900 x 900) on the generic pair (kgpu_use_static_kernels(0)) for comparison.  Prints us per
block and ns per complex point for each pass (per-launch CUDA events, median over rounds, masters interleaved)."""
import argparse
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from ka9q_radio_b200 import capi  # noqa: E402
from ka9q_radio_b200.channelizer import Channelizer  # noqa: E402

CASES = [  # (name, L, M, in_type, extended, static)
    ("airspyhf_912k ext", 18240, 4561, capi.KGPU_COMPLEX, True, 1),
    ("rx888_60m8 ext", 1216000, 304001, capi.KGPU_REAL, True, 1),
    ("rx888_64m8 generic", 1296000, 324001, capi.KGPU_REAL, False, 0),
]

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=8)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--rounds", type=int, default=5)
a = ap.parse_args()
lib = capi.load()
dev = torch.device("cuda:0")
B = a.blocks
setups = []
for name, L, M, in_type, ext, static in CASES:
    cz = Channelizer(L, M, in_type, dev, capacity=1, extended=ext)
    per = 2 if in_type == capi.KGPU_COMPLEX else 1
    host = np.random.default_rng(0).standard_normal(((B + 1) * L + M - 1) * per, dtype=np.float32)
    setups.append((name, cz, torch.from_numpy(host).to(dev), cz.alloc_spectra(B), static))
res = {s[0]: [] for s in setups}
for rnd in range(a.rounds + 1):
    for name, cz, d, spec, static in setups:
        lib.kgpu_use_static_kernels(static)
        lib.kgpu_profile_enable(1)
        lib.kgpu_profile_reset()
        for _ in range(a.iters):
            cz.forward(d, B, spec)
        torch.cuda.synchronize()
        p = capi.profile_snapshot()
        lib.kgpu_profile_enable(0)
        if rnd:  # round 0 warms up
            res[name].append({k: 1e3 * ms / cnt / B for k, (ms, cnt) in p.items() if cnt})
lib.kgpu_use_static_kernels(1)
print(f"{torch.cuda.get_device_name(0)}; {B} blocks per launch, median of {a.rounds} rounds of {a.iters} launches")
for name, cz, *_ in setups:
    rows = res[name]
    nc = cz.master.N // (1 if cz.in_type == capi.KGPU_COMPLEX else 2)
    cols, rws = (float(np.median([r[k] for r in rows])) for k in ("fwd_cols", "fwd_rows"))
    print(f"{name:20s} nc {nc:8d}  fwd_cols {cols:8.2f}  fwd_rows {rws:8.2f}  total {cols + rws:8.2f} us/block  "
          f"{1e3 * (cols + rws) / nc:6.3f} ns/point   {cz.master.describe()}")
    cz.close()
