#!/usr/bin/env python3
"""Throughput of the wide-channel kernel (chan_wide): a 20 MS/s IQ master (L = 400 000, M = 100 001, N = 500 000) with
52 wfm channels (olen 7680 = 384 kHz x 20 ms, 9600 points) on a 200 kHz raster, `--blocks` blocks per launch.

The spectra are filled once with seeded noise; only kgpu_bank_run is timed, with CUDA events over `--iters` launches
after `--warmup` launches.  Bytes are algorithmic, (2 Ns + Ls) x 8 per channel-block: the slice read, the response read
and the output write (215 kB at Ns = 9600).  The share of peak is against the H100 SXM data sheet's 3350 GB/s, which is
the data sheet's figure, not a measured one.  One JSON line on stdout; nothing is written to the tree.

  python tools/wide_bench.py [--blocks 32] [--iters 50] [--warmup 10]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HBM_GBS = 3350.0  # H100 SXM data sheet, HBM3


def gpu_info() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, power = (v.strip() for v in r.stdout.strip().split(",")[:2])
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers stand without it, but say so
        return {"gpu": None, "power_limit": None, "gpu_info_error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--channels", type=int, default=52)
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")

    import torch

    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    L, M, fs, olen = 400_000, 100_001, 20e6, 7680
    N = L + M - 1
    cz = Channelizer(L, M, capi.KGPU_COMPLEX, "cuda:0", capacity=args.channels)
    raster = round(200e3 * N / fs)  # 5000 bins
    for k in range(args.channels):
        shift = (k - args.channels // 2) * raster
        cz.add_channel(olen, shift, -110 / 384, 110 / 384, 11.0)
    ns = olen * N // L
    nb = args.blocks
    g = torch.Generator(device="cuda:0").manual_seed(1)
    spec = cz.alloc_spectra(nb)
    spec.copy_(torch.randn(spec.shape, dtype=torch.complex64, device="cuda:0", generator=g))
    out = cz.alloc_outputs(nb)
    for _ in range(args.warmup):
        cz.channels(spec, nb, out)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.iters):
        cz.channels(spec, nb, out)
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / args.iters
    bytes_per = (2 * ns + olen) * 8
    total = bytes_per * args.channels * nb
    gbs = total / (us * 1e-6) / 1e9
    res = {"workload": f"20 MS/s IQ, {args.channels} x wfm ({ns} points, olen {olen}), {nb} blocks per launch",
           "us_per_launch": round(us, 2), "us_per_channel_block": round(us / (args.channels * nb), 4),
           "bytes_per_channel_block": bytes_per, "GBps": round(gbs, 1),
           "share_of_datasheet_hbm_3350GBps": round(gbs / HBM_GBS, 4), "iters": args.iters, "warmup": args.warmup}
    res.update(gpu_info())
    cz.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
