#!/usr/bin/env python3
"""A/B micro-benchmark of the three kernels on cfg-2 (needs a GPU).

usage: kbench.py [--blocks B] [--iters K] variant [variant ...]
a variant is "default" (the master's own kernel pair) or "static=0" (the generic kernels, kgpu_use_static_kernels(0));
variants are interleaved round-robin to cancel drift."""
import argparse, sys, json
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from ka9q_radio_b200 import workloads
from ka9q_radio_b200 import capi
from ka9q_radio_b200.channelizer import Channelizer

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=8)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--nchan", type=int, default=0, help="0 = the workload's own channel list")
ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3", "cfg4"])
ap.add_argument("variants", nargs="+", choices=["default", "static=0"])
a = ap.parse_args()
W = workloads.by_name(a.config)
lib = capi.load()
dev = torch.device("cuda:0")
B = a.blocks
nchan = a.nchan or len(W.channels)
cz = Channelizer(W.L, W.M, W.in_type, dev, capacity=nchan)
for k in range(nchan):
    c = W.channels[k % len(W.channels)]
    cz.add_channel(c.olen, c.shift, c.low, c.high, c.beta)
nstream = max(32, 4 * B)
rng = np.random.default_rng(0)
wps = 2 if W.in_type == capi.KGPU_COMPLEX else 1
host = rng.integers(-3000, 3000, (nstream * W.L + W.M - 1) * wps, dtype=np.int16)
d_stream = torch.from_numpy(host).to(dev)
spec, out = cz.alloc_spectra(B), cz.alloc_outputs(B)
ng = nstream // B
res = {v: [] for v in a.variants}
for rnd in range(a.rounds + 1):
    for v in a.variants:
        lib.kgpu_use_static_kernels(0 if v == "static=0" else 1)
        lib.kgpu_profile_enable(1); lib.kgpu_profile_reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for i in range(a.iters):
            cz.forward(d_stream, B, spec, scale=W.scale, first_block=(i % ng) * B)
            cz.channels(spec, B, out)
        e1.record(); torch.cuda.synchronize()
        p = capi.profile_snapshot(); lib.kgpu_profile_enable(0)
        if rnd == 0: continue  # warm-up round
        row = {k: 1e3 * ms / cnt / B for k, (ms, cnt) in p.items() if cnt}
        row["wall"] = 1e3 * e0.elapsed_time(e1) / a.iters / B
        res[v].append(row)
lib.kgpu_use_static_kernels(1)
for v, rows in res.items():
    keys = rows[0].keys()
    print("%-28s" % v, "  ".join("%s %6.2f" % (k, np.median([r[k] for r in rows])) for k in keys), " us/block (median of %d)" % len(rows))
