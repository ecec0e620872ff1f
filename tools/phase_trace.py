#!/usr/bin/env python3
"""Per-CTA phase timeline of the v2 forward kernels (globaltimer stamps written by thread 0).

cols: t0 start | t1 loads arrived + stage 0 done | t2 stage 1 done | t3 stage 2 + stores issued
rows: t0 start | t1 TMA rows arrived             | t2 stages 0,1 done | t3 split + stores issued
Also, per SM, how much of the kernel's span had 0 / 1 / 2 resident CTAs past their load wait.
usage: phase_trace.py [blocks] [key=value tuning ...]"""
import sys
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench
from ka9q_radio_b200 import capi
from ka9q_radio_b200.channelizer import Channelizer
B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
lib = capi.load(); dev = torch.device("cuda:0")
for k, v in [kv.split("=") for kv in sys.argv[2:]]: lib.kgpu_set_tuning(int(k), int(v))
cz = Channelizer(bench.L, bench.M, capi.KGPU_REAL, dev, capacity=4)
host = np.random.default_rng(0).integers(-3000, 3000, 4 * B * bench.L + bench.M - 1, dtype=np.int16)
d_stream = torch.from_numpy(host).to(dev)
spec = cz.alloc_spectra(B)
n1c, n2c = 157 * B, 163 * B
dbg = torch.zeros(n1c * 6, dtype=torch.int64, device=dev)
dbg2 = torch.zeros(n2c * 6, dtype=torch.int64, device=dev)
for i in range(3): cz.forward(d_stream, B, spec, scale=bench.SCALE, first_block=i * B)
torch.cuda.synchronize()
lib.kgpu_set_debug_buffer(dbg.data_ptr()); lib.kgpu_set_debug_buffer_rows(dbg2.data_ptr())
cz.forward(d_stream, B, spec, scale=bench.SCALE, first_block=0)
torch.cuda.synchronize(); lib.kgpu_set_debug_buffer(None); lib.kgpu_set_debug_buffer_rows(None)

def report(name, raw, labels):
    t = raw.cpu().numpy().reshape(-1, 6).astype(np.float64)
    t = t[t[:, 3] > 0]
    t0 = t[:, 0].min(); span = t[:, 3].max() - t0
    print("%s: span %.1f us, %d CTAs, %.2f us/block" % (name, span / 1e3, len(t), span / 1e3 / B))
    for lab, v in zip(labels, (t[:, 1] - t[:, 0], t[:, 2] - t[:, 1], t[:, 3] - t[:, 2], t[:, 3] - t[:, 0])):
        print("  %-22s median %6.2f us  p10 %6.2f  p90 %6.2f  mean %6.2f" % (lab, np.median(v) / 1e3, np.percentile(v, 10) / 1e3, np.percentile(v, 90) / 1e3, v.mean() / 1e3))
    sm = t[:, 5].astype(int)
    occ = np.zeros(4); gaps = []
    for s in np.unique(sm):
        u = t[sm == s]
        ev = []
        for r in u:
            ev += [(r[0], 0, +1), (r[3], 0, -1), (r[1], 1, +1), (r[3], 1, -1)]
        ev.sort()
        res = comp = 0; last = t0
        for tm, kind, d in ev:
            occ[min(comp, 2)] += tm - last
            if res == 0: occ[3] += tm - last
            last = tm
            if kind == 0: res += d
            else: comp += d
        occ[min(comp, 2)] += t[:, 3].max() - last
        st = np.sort(u[:, 0]); en = np.sort(u[:, 3])
    tot = occ[:3].sum()
    print("  SM time with 0/1/2 CTAs past the load wait: %.1f %% / %.1f %% / %.1f %%   (no CTA resident: %.1f %%)" % tuple(100 * occ / tot))
    per_sm = np.bincount(sm, minlength=torch.cuda.get_device_properties(dev).multi_processor_count)
    print("  CTAs per SM: min %d max %d" % (per_sm.min(), per_sm.max()))

report("COLS v2", dbg, ("load + stage 0", "stage 1", "stage 2 + store", "total"))
report("ROWS v2", dbg2, ("TMA wait", "stages 0,1", "stage 2 + split store", "total"))
