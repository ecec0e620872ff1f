#!/usr/bin/env python3
"""Throughput of the huge-channel kernels (chan_huge): the enabled channels of radiod@rx888-wsprdaemon.conf on a
64.8 MS/s RX888 REAL master at the defaults (20 ms, overlap 5: L = 1 296 000, M = 324 001, N = 1 620 000), `--blocks`
blocks per launch: 15 WSPR channels at 12 kHz, 10 WWV-IQ at 16 kHz, 8 x 768 kHz, 2 x 384 kHz, 3 x 192 kHz and the 8
WEBSDR_TEST channels at 1.536 MS/s (olen 30 720, 38 400 points), which are the huge ones.

The spectra are filled once with seeded noise; only kgpu_bank_run is timed, with CUDA events over `--iters` launches
after `--warmup` launches, for a bank of the 8 huge channels alone and for the whole bank.  Bytes are algorithmic,
(2 Ns + Ls) x 8 per channel-block (the slice read, the response read and the output write; 860 kB at Ns = 38 400); the
scratch traffic of the two passes is not counted.  One JSON line on stdout; nothing is written to the tree.

  python tools/huge_bench.py [--blocks 32] [--iters 50] [--warmup 10]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tools.wide_bench import gpu_info  # noqa: E402

L, M, FS = 1_296_000, 324_001, 64.8e6
# (count, olen, output rate)
WSPRDAEMON = [(15, 240, 12e3), (10, 320, 16e3), (8, 15360, 768e3), (2, 7680, 384e3), (3, 3840, 192e3), (8, 30720, 1536e3)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")

    import torch

    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    N = L + M - 1
    nb = args.blocks
    info = gpu_info()

    def timed(groups):
        cz = Channelizer(L, M, capi.KGPU_REAL, "cuda:0", capacity=sum(g[0] for g in groups))
        f = 137_500.0
        for count, olen, _ in groups:
            for _ in range(count):
                cz.add_channel(olen, round(f * N / FS), -0.45, 0.45, 11.0)
                f += 0.55e6 + 1234.5
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
        cz.close()
        return t0.elapsed_time(t1) * 1e3 / args.iters

    huge = [g for g in WSPRDAEMON if g[1] * N // L > 28812]
    us_huge = timed(huge)
    us_all = timed(WSPRDAEMON)
    nh = sum(g[0] for g in huge)
    ns, olen = huge[0][1] * N // L, huge[0][1]
    bytes_huge = (2 * ns + olen) * 8 * nh * nb
    res = {"workload": f"RX888 64.8 MS/s REAL, radiod@rx888-wsprdaemon.conf channels, {nh} huge ({ns} points, olen {olen}), "
                       f"{nb} blocks per launch",
           "us_per_launch_huge": round(us_huge, 1), "us_per_launch_bank": round(us_all, 1),
           "us_per_huge_channel_block": round(us_huge / (nh * nb), 3),
           "huge_algorithmic_GBps": round(bytes_huge / (us_huge * 1e-6) / 1e9, 1),
           "signal_ms_per_launch": nb * L / FS * 1e3, "iters": args.iters, "warmup": args.warmup}
    res.update(info)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
