#!/usr/bin/env python3
"""Throughput of the Bluestein channels (kgpu_bank_define_any, bluestein_chan.cuh), `--blocks` blocks per launch: banks of
`--chans` channels of one length, 725 (29 kHz at 20 ms and overlap 5), 1550 (62 kHz), 44 000 (1.76 MS/s) and 62 000
points (2.48 MS/s), each against a 7-smooth neighbour on the same master (720, 1536, 43 740, 61 440), in us per
channel-block.  They run on a REAL master of the 64.8 MS/s RX888's transform size with M = 1 (L = N = 1 620 000), on
which every channel length is reachable.

The spectra are filled once with seeded noise; only kgpu_bank_run is timed, with CUDA events over `--iters` launches
after `--warmup` launches.  Within a round a Bluestein length and its neighbour run back to back, in alternating order
from round to round.  Each figure is the median of `--rounds` rounds, with the smallest and largest beside it.  The card
name, power limit and SM clock are read in the same run.  One JSON line on stdout; nothing is written to the tree.

  python tools/bluestein_chan_bench.py [--blocks 32] [--chans 16] [--iters 20] [--warmup 5] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tools.ext_chan_bench import sm_clock  # noqa: E402
from tools.wide_bench import gpu_info  # noqa: E402

N = 1_620_000
# (Bluestein length, 7-smooth neighbour)
PAIRS = [(725, 720), (1550, 1536), (44000, 43740), (62000, 61440)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--chans", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    from ka9q_radio_b200 import capi
    from ka9q_radio_b200.channelizer import Channelizer

    nb = args.blocks
    info = gpu_info()

    def one_length(points):
        cz = Channelizer(N, 1, capi.KGPU_REAL, "cuda:0", capacity=args.chans)
        for k in range(args.chans):  # M = 1 leaves set_filter no taps: a flat response instead
            cz.add_channel(points, 20_000 + k * 40_000, response=np.ones(points, np.complex64))
        g = torch.Generator(device="cuda:0").manual_seed(1)
        spec, out = cz.alloc_spectra(nb), cz.alloc_outputs(nb)
        spec.copy_(torch.randn(spec.shape, dtype=torch.complex64, device="cuda:0", generator=g))
        return cz, spec, out

    def time(bank):  # us per launch
        cz, spec, out = bank
        for _ in range(args.warmup):
            cz.channels(spec, nb, out)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            cz.channels(spec, nb, out)
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) * 1e3 / args.iters

    def stats(v, scale=1.0):
        v = sorted(x * scale for x in v)
        return {"median": round(v[len(v) // 2], 4), "min": round(v[0], 4), "max": round(v[-1], 4)}

    lengths = {}
    per = 1.0 / (args.chans * nb)
    for blue, smooth in PAIRS:
        assert capi.chan_plan(blue)[0] == capi.CHAN_BLUESTEIN and capi.chan_plan(smooth)[0] != capi.CHAN_BLUESTEIN
        bb, bs = one_length(blue), one_length(smooth)
        tb, ts = [], []
        for r in range(args.rounds):
            if r % 2:
                ts.append(time(bs))
                tb.append(time(bb))
            else:
                tb.append(time(bb))
                ts.append(time(bs))
        bb[0].close()
        bs[0].close()
        lengths[str(blue)] = {"plan": capi.chan_plan(blue)[1], "us_per_channel_block": stats(tb, per), "neighbour": smooth,
                              "neighbour_us_per_channel_block": stats(ts, per),
                              "ratio": stats([a / b for a, b in zip(tb, ts)])}
    res = {"workload": f"REAL master L = N = {N}, M = 1, {args.chans} channels of one length, {nb} blocks per launch",
           "lengths": lengths, "chans_per_length": args.chans, "iters": args.iters, "warmup": args.warmup,
           "rounds": args.rounds}
    res.update(info)
    res.update(sm_clock())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
