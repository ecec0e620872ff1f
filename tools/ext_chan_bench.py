#!/usr/bin/env python3
"""Throughput of the extended-length channel kernels (chan_kernel_ext, chan_wide_ext), `--blocks` blocks per launch:

- the 12 channels of radiod@kfs-sw.conf.d/51-hfdl.conf on a 64.8 MS/s RX888 REAL master at the defaults (20 ms, overlap
  5: L = 1 296 000, M = 324 001), whose 220 kHz and 277.2 kHz channels (5500 and 6930 points) are extended;
- banks of `--chans` channels of one length, extended lengths against 7-smooth neighbours, in us per channel-block and
  ns per channel-block point.  These run on a master of the same transform size with M = 1 (L = N = 1 620 000), on
  which every channel length is reachable (at overlap 5 only multiples of 5 are).

The spectra are filled once with seeded noise; only kgpu_bank_run is timed, with CUDA events over `--iters` launches
after `--warmup` launches.  Every bank is timed in `--rounds` rounds; within a round an extended length and its
neighbour run back to back, in alternating order from round to round.  Each figure is the median of its rounds, with
the smallest and largest beside it.  One JSON line on stdout; nothing is written to the tree.

  python tools/ext_chan_bench.py [--blocks 32] [--chans 16] [--iters 50] [--warmup 10] [--rounds 7]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tools.wide_bench import gpu_info  # noqa: E402

L, M, FS = 1_296_000, 324_001, 64.8e6
# radiod@kfs-sw.conf.d/51-hfdl.conf: (output rate, low, high, frequency) in Hz
HFDL = [(80e3, -36e3, 36e3, 21964e3), (100e3, -46e3, 46e3, 17944e3), (12e3, 0.0, 3e3, 15025e3),
        (100e3, -47e3, 47e3, 13310e3), (220e3, -104e3, 104e3, 11287e3), (80e3, -35e3, 35e3, 10061.5e3),
        (160e3, -78e3, 78e3, 8902.5e3), (192e3, -93e3, 93e3, 6622e3), (277.2e3, -136e3, 136e3, 5587e3),
        (40e3, -18e3, 18e3, 4672e3), (50e3, -24e3, 24e3, 3477e3), (80e3, -39e3, 39e3, 2980e3)]
# (extended length, 7-smooth neighbour)
PAIRS = [(5500, 5488), (6930, 7000), (8800, 8820), (11088, 11025)]


def sm_clock() -> dict:
    """SM clock right after the timed launches, and its maximum (MHz)"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        now, top = (v.strip() for v in r.stdout.strip().split(",")[:2])
        return {"sm_clock": now, "sm_clock_max": top}
    except Exception as e:
        return {"sm_clock": None, "sm_clock_error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--chans", type=int, default=16)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")

    import numpy as np
    import torch

    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    N = L + M - 1
    nb = args.blocks
    info = gpu_info()

    class Bank:  # one bank with its spectra and outputs, timed as often as asked
        def __init__(self, cz):
            g = torch.Generator(device="cuda:0").manual_seed(1)
            self.cz, self.spec, self.out = cz, cz.alloc_spectra(nb), cz.alloc_outputs(nb)
            self.spec.copy_(torch.randn(self.spec.shape, dtype=torch.complex64, device="cuda:0", generator=g))

        def time(self):  # us per launch
            for _ in range(args.warmup):
                self.cz.channels(self.spec, nb, self.out)
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                self.cz.channels(self.spec, nb, self.out)
            t1.record()
            torch.cuda.synchronize()
            return t0.elapsed_time(t1) * 1e3 / args.iters

    def stats(v, scale=1.0):
        v = sorted(x * scale for x in v)
        return {"median": round(v[len(v) // 2], 4), "min": round(v[0], 4), "max": round(v[-1], 4)}

    cz = Channelizer(L, M, capi.KGPU_REAL, "cuda:0", capacity=len(HFDL))
    for rate, lo, hi, f in HFDL:
        cz.add_channel(int(round(rate * L / FS)), round(f * N / FS), lo / rate, hi / rate, 11.0)
    hfdl = Bank(cz)
    us_hfdl = [hfdl.time() for _ in range(args.rounds)]
    cz.close()

    def one_length(points):
        cz = Channelizer(N, 1, capi.KGPU_REAL, "cuda:0", capacity=args.chans)
        for k in range(args.chans):  # M = 1 leaves set_filter no taps: a flat response instead
            cz.add_channel(points, 20_000 + k * 40_000, response=np.ones(points, np.complex64))
        return Bank(cz)

    lengths = {}
    per = 1.0 / (args.chans * nb)
    for ext, smooth in PAIRS:
        be, bs = one_length(ext), one_length(smooth)
        te, ts = [], []
        for r in range(args.rounds):
            if r % 2:
                ts.append(bs.time())
                te.append(be.time())
            else:
                te.append(be.time())
                ts.append(bs.time())
        be.cz.close()
        bs.cz.close()
        ratios = [(a / ext) / (b / smooth) for a, b in zip(te, ts)]
        lengths[str(ext)] = {"us_per_channel_block": stats(te, per), "neighbour": smooth,
                             "neighbour_us_per_channel_block": stats(ts, per), "per_point_ratio": stats(ratios)}
    res = {"workload": f"RX888 64.8 MS/s REAL, radiod@kfs-sw.conf.d/51-hfdl.conf (12 channels, 5500 and 6930 points "
                       f"extended), {nb} blocks per launch",
           "us_per_launch_hfdl": stats(us_hfdl), "signal_ms_per_launch": nb * L / FS * 1e3,
           "lengths": lengths, "chans_per_length": args.chans, "iters": args.iters, "warmup": args.warmup,
           "rounds": args.rounds}
    res.update(info)
    res.update(sm_clock())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
