#!/usr/bin/env python3
"""Row pass of a REAL and a COMPLEX master that move the same bytes through the same stages (needs a GPU).

REAL    L = 2592000, M = 648001 (cfg-2): nc = 1296 x 1250, fwd_cols_r36 + fwd_rows_v2<true, 1296, true>
COMPLEX L = 1296000, M = 324001:         nc = 1296 x 1250, fwd_cols_r36 + fwd_rows_v2<false, 1296, false>
Both read 13.10 MB of inter-pass rows and write 12.96 MB of spectrum per block, through the same 10 x 25 x 5 stages;
they differ in how the row pass pairs rows and how wide its stores are.  The two masters are alternated round by round
(CUDA events + the library's per-kernel profile, a warm-up round first) and the medians printed in us per block.

usage: rows_probe.py [--blocks B] [--iters K] [--rounds R]"""
import argparse, subprocess, sys
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from ka9q_radio_b200 import capi

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=32)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--rounds", type=int, default=3)
a = ap.parse_args()
MASTERS = {"real": (2592000, 648001, capi.KGPU_REAL), "complex": (1296000, 324001, capi.KGPU_COMPLEX)}

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print("gpu:", gpu)
lib = capi.load()
dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
capi.check(lib.kgpu_set_device(0), "kgpu_set_device")
B = a.blocks
nstream = max(32, 4 * B)
ng = nstream // B
rng = np.random.default_rng(0)
state = {}
for name, (L, M, typ) in MASTERS.items():
    m = capi.Master(L, M, typ)
    d = m.describe()
    assert "1296 x 1250" in d and "fwd_cols_r36 + fwd_rows_v2" in d, d
    print(f"{name}: {d}")
    wps = 2 if typ == capi.KGPU_COMPLEX else 1   # int16 words per sample
    hop = L * wps * 2                            # bytes of new input per block
    stream = torch.from_numpy(rng.integers(-3000, 3000, (nstream * L + M - 1) * wps, dtype=np.int16)).to(dev)
    spec = torch.empty((B, m.spec_stride), dtype=torch.complex64, device=dev)
    state[name] = (m, stream, spec, hop)

res = {k: [] for k in MASTERS}
for rnd in range(a.rounds + 1):
    for name, (m, stream, spec, hop) in state.items():
        st = torch.cuda.current_stream(dev).cuda_stream
        lib.kgpu_profile_enable(1); lib.kgpu_profile_reset()
        torch.cuda.synchronize()
        for i in range(a.iters):
            m.forward(stream.data_ptr() + (i % ng) * B * hop, capi.KGPU_FMT_I16, 1.0 / 32768, B, spec.data_ptr(), st)
        torch.cuda.synchronize()
        p = capi.profile_snapshot(); lib.kgpu_profile_enable(0)
        if rnd == 0:
            continue  # warm-up round
        res[name].append({k: 1e3 * ms / cnt / B for k, (ms, cnt) in p.items() if cnt})
for name, rows in res.items():
    for k in ("fwd_cols", "fwd_rows"):
        v = [r[k] for r in rows]
        print(f"{name:8s} {k:9s} median {np.median(v):6.2f}  min {min(v):6.2f}  max {max(v):6.2f} us/block ({len(v)} rounds)")
r, c = np.median([x["fwd_rows"] for x in res["real"]]), np.median([x["fwd_rows"] for x in res["complex"]])
print(f"fwd_rows real/complex = {r / c:.3f}")
for m, *_ in state.values():
    m.close()
