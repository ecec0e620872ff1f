#!/usr/bin/env python3
"""Device time per block of the Bluestein forward transform (kgpu_master_create_any) on RX888 REAL masters at 62 and
116 MS/s (20 ms blocks, overlap 5: Nc = 775 000 = 2^3 5^5 31 and 1 450 000 = 2^4 5^5 29), against the direct master of
the 64.8 MS/s default (Nc = 810 000), `--blocks` int16 blocks per kgpu_forward.

Each round times every master once, in an order that alternates between rounds, with CUDA events over `--iters`
launches after `--warmup`; the result is the median over `--rounds` rounds with the min and max.  The host time of
each creation (dominated for the Bluestein masters by the chirp's transform in double) is reported too.  One JSON line
on stdout; nothing is written to the tree.

  python tools/bluestein_bench.py [--blocks 32] [--iters 20] [--warmup 3] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tools.wide_bench import gpu_info  # noqa: E402

MASTERS = [("direct_64m8", 64_800_000), ("bluestein_62m", 62_000_000), ("bluestein_116m", 116_000_000)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch

    from ka9q_radio_b200 import capi

    info = gpu_info()
    nb = args.blocks
    st = torch.cuda.current_stream().cuda_stream
    runs = {}
    for name, rate in MASTERS:
        L = rate // 50
        M = L // 4 + 1
        t0 = time.perf_counter()
        m = capi.Master(L, M, capi.KGPU_REAL, any_length=True)
        create_s = time.perf_counter() - t0
        g = torch.Generator(device="cuda:0").manual_seed(rate % 1000)
        x = torch.randint(-32768, 32768, ((nb - 1) * L + m.N,), dtype=torch.int16, device="cuda:0", generator=g)
        spec = torch.empty(nb * m.spec_stride, dtype=torch.complex64, device="cuda:0")
        stats = torch.zeros(2 * nb, dtype=torch.int64, device="cuda:0")
        runs[name] = dict(m=m, x=x, spec=spec, stats=stats, rate=rate, L=L, create_s=create_s, us=[])

    def launch(r):
        r["m"].forward(r["x"].data_ptr(), capi.KGPU_FMT_I16, 3e-5, nb, r["spec"].data_ptr(), st, d_stats=r["stats"].data_ptr())

    for r in runs.values():
        for _ in range(args.warmup):
            launch(r)
    torch.cuda.synchronize()
    names = [n for n, _ in MASTERS]
    for k in range(args.rounds):
        for name in (names if k % 2 == 0 else names[::-1]):
            r = runs[name]
            for _ in range(args.warmup):
                launch(r)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                launch(r)
            e1.record()
            torch.cuda.synchronize()
            r["us"].append(e0.elapsed_time(e1) * 1e3 / args.iters / nb)
    direct = statistics.median(runs["direct_64m8"]["us"])
    res = {"workload": f"RX888 REAL int16, 20 ms blocks at overlap 5, {nb} blocks per kgpu_forward", "rounds": args.rounds,
           "iters": args.iters}
    for name, r in runs.items():
        med = statistics.median(r["us"])
        res[name] = {"describe": r["m"].describe(), "us_per_block_median": round(med, 2),
                     "us_per_block_min": round(min(r["us"]), 2), "us_per_block_max": round(max(r["us"]), 2),
                     "ratio_to_direct": round(med / direct, 2),
                     "x_real_time": round((r["L"] / r["rate"]) / (med * 1e-6), 1),
                     "create_s": round(r["create_s"], 2)}
        r["m"].close()
    res.update(info)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
