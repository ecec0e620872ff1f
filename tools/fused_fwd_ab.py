#!/usr/bin/env python3
"""A/B of cfg-2's forward pass as one launch (fwd_fused_r36_v2, kgpu_use_fused_forward(1)) against the two-kernel pair
fwd_cols_r36_tma + fwd_rows_v2 (kgpu_use_fused_forward(0)), on a GPU.

usage: fused_fwd_ab.py [--blocks 32] [--iters 50] [--rounds 9] [--fmt i16|i16s|f32] [--leads 0,79]

Each round runs `iters` steps (forward + the workload's 1024 channels over `blocks` blocks) with each form, the forms
alternating, after one warm-up round.  Forms: the pair; the fused launch; the fused launch with the L2 discard of each
inter-pass row once read (the gap to the fused row is what keeping those rows from being written back to DRAM saves,
net of the discards' own cost); and the fused launch at each other lead of --leads.  Per-kernel device times come from kgpu_profile_* (CUDA
events around each launch).  Prints the card, its power limit and SM clock, then per form the forward pass's median and
spread (min .. max over the rounds) in us per block, and one JSON line.  The spectra of every form are compared bitwise."""
import argparse, json, subprocess, sys
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from ka9q_radio_b200 import capi, workloads
from ka9q_radio_b200.channelizer import Channelizer

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=32)
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--rounds", type=int, default=9)
ap.add_argument("--fmt", default="i16", choices=["i16", "i16s", "f32"], help="i16s: int16 with de-randomisation and statistics")
ap.add_argument("--leads", default="", help="comma-separated leads to time besides the default one")
a = ap.parse_args()


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0)}


W = workloads.by_name("cfg2")
lib = capi.load()
dev = torch.device("cuda:0")
B = a.blocks
cz = Channelizer(W.L, W.M, W.in_type, dev, capacity=len(W.channels))
for c in W.channels:
    cz.add_channel(c.olen, c.shift, c.low, c.high, c.beta)
nstream = max(64, 2 * B)
rng = np.random.default_rng(0)
if a.fmt == "f32":
    host, scale = (1e-3 * rng.standard_normal(nstream * W.L + W.M - 1)).astype(np.float32), 1.0
else:
    host, scale = rng.integers(-3000, 3000, nstream * W.L + W.M - 1, dtype=np.int16), W.scale
d_stream = torch.from_numpy(host).to(dev)
stats = torch.zeros((B, 2), dtype=torch.int64, device=dev) if a.fmt == "i16s" else None
spec, out = cz.alloc_spectra(B), cz.alloc_outputs(B)
ng = nstream // B


def step(i):
    cz.forward(d_stream, B, spec, scale=scale, first_block=(i % ng) * B, derandomize=a.fmt == "i16s", stats=stats)
    cz.channels(spec, B, out)


import ctypes as C

shape = (C.c_int * 5)()
lib.kgpu_fused_shape(C.cast(shape, C.c_void_p))
LEAD = shape[4]
# form: (fused on, lead, discard)
forms = {"pair": (0, LEAD, 0), "fused": (1, LEAD, 0), "fused_discard": (1, LEAD, 1)}
for ld in [int(v) for v in a.leads.split(",") if v.strip()]:
    forms[f"fused_lead{ld}"] = (1, ld, 0)


def use(form):
    on, lead, discard = forms[form]
    lib.kgpu_use_fused_forward(on)
    if lib.kgpu_fused_forward_options(lead, discard):
        raise SystemExit(capi.load().kgpu_last_error().decode())


res = {f: [] for f in forms}
info = gpu_info()
for rnd in range(a.rounds + 1):
    for f in forms:
        use(f)
        lib.kgpu_profile_enable(1)
        lib.kgpu_profile_reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for i in range(a.iters):
            step(i)
        e1.record()
        torch.cuda.synchronize()
        p = capi.profile_snapshot()
        lib.kgpu_profile_enable(0)
        if rnd == 0:
            continue  # warm-up round
        row = {k: 1e3 * ms / a.iters / B for k, (ms, cnt) in p.items() if cnt}  # us per block
        row["forward"] = sum(row.get(k, 0.0) for k in ("fwd_cols", "fwd_rows", "fwd_fused"))
        row["wall"] = 1e3 * e0.elapsed_time(e1) / a.iters / B
        res[f].append(row)
info["sm_clock_after"] = gpu_info().get("clocks.sm")

# the same input through every form: spectra and statistics bitwise equal
bits = {}
for f in forms:
    use(f)
    step(3)
    torch.cuda.synchronize()
    bits[f] = (spec.clone().view(torch.int32), None if stats is None else stats.clone())
lib.kgpu_use_fused_forward(1)
lib.kgpu_fused_forward_options(LEAD, 0)
same = all(bool(torch.equal(bits[f][0], bits["pair"][0])) and (stats is None or bool(torch.equal(bits[f][1], bits["pair"][1])))
           for f in forms)

print(f"card {info.get('name')}, power limit {info.get('power.limit')}, SM clock {info.get('clocks.sm')} "
      f"(max {info.get('clocks.max.sm')}, after {info['sm_clock_after']}); cfg-2 {a.fmt}, {B} blocks, {a.iters} steps x {a.rounds} rounds")
summary = {}
for f, rows in res.items():
    summary[f] = {}
    for k in rows[0]:
        v = np.array([r[k] for r in rows])
        summary[f][k] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
        print(f"{f:18s} {k:9s} median {np.median(v):7.3f}  spread {v.min():7.3f} .. {v.max():7.3f}  us/block")
gain = 1 - summary["fused"]["forward"]["median"] / summary["pair"]["forward"]["median"]
print(f"forward pass: fused {100 * gain:.1f} % less time per block than the pair; spectra"
      f"{'' if stats is None else ' and statistics'} bitwise {'equal' if same else 'DIFFERENT'}")
print(json.dumps({"gpu": info, "fmt": a.fmt, "blocks": B, "us_per_block": summary, "forward_gain": gain, "bitwise_equal": same}))
sys.exit(0 if same else 1)
