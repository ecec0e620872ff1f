"""Narrowband spectrum analyzer timings (narrowband_poll, reference spectrum.c:206-306, on the device).

  poll    device time of one kgpu_spectrum_run_narrow (CUDA events around --reps polls, median of --rounds rounds, the
          configurations alternated round by round) on a ring of fft_avg * fft_n complex samples, for fft_n 2000, 16 200,
          65 536 (the largest length setup_narrowband searches to) and 69 629 = 29 x 7^4 (a Bluestein length), at
          fft_avg 1 and 10, overlap 0.5, bin_count = 0.8 fft_n
  append  device time of one kgpu_spectrum_ring_append of a 1000-sample block (what every delivered block adds)
  cpu     the restatement (oracle/narrowband_oracle.c) on this host: its transform is the oracle's fft_cpu (the same one
          the FFTW shim gives the reference), not FFTW with wisdom, so it gives the CPU's scale, not radiod's speed

Prints one JSON line per measurement, each with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

LENGTHS = [2000, 16200, 65536, 69629]
AVGS = [1, 10]
OVERLAP = 0.5


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power}


def window(n):
    w = np.kaiser(n + 1, 11.0)[:n]
    return (w / w.sum()).astype(np.float32)


def ring_of(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)


def bench_polls(reps: int, rounds: int, info: dict) -> None:
    import torch

    from ka9q_radio_b200 import capi

    for fft_n in LENGTHS:
        bin_count = fft_n * 4 // 5
        sp = capi.Spectrum(fft_n, capi.KGPU_COMPLEX, bin_count)
        sp.set_window(window(fft_n))
        rings = {a: torch.from_numpy(ring_of(a * fft_n, a).view(np.float32).reshape(-1, 2)).cuda() for a in AVGS}
        bins = torch.empty(bin_count, device="cuda")
        times = {a: [] for a in AVGS}
        ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for a in AVGS:  # warm-up of every shape the timed rounds use
            for _ in range(3):
                sp.run_narrow(rings[a], 17, a, OVERLAP, bins)
        for _ in range(rounds):
            for a in AVGS:
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(reps):
                    sp.run_narrow(rings[a], 17, a, OVERLAP, bins)
                ev[1].record()
                torch.cuda.synchronize()
                times[a].append(ev[0].elapsed_time(ev[1]) * 1e3 / reps)
        for a in AVGS:
            print(json.dumps({"what": "poll", "fft_n": fft_n, "path": sp.describe().split()[0], "bin_count": bin_count,
                              "fft_avg": a, "overlap": OVERLAP, "us_per_poll_median": round(float(np.median(times[a])), 1),
                              "us_spread": [round(min(times[a]), 1), round(max(times[a]), 1)], **info}), flush=True)
        sp.close()


def bench_append(reps: int, rounds: int, info: dict) -> None:
    import torch

    from ka9q_radio_b200 import capi

    ring = torch.zeros(10 * 2000, 2, device="cuda")
    blk = torch.from_numpy(ring_of(1000, 3).view(np.float32).reshape(-1, 2)).cuda()
    idx = 0
    for _ in range(3):
        idx = capi.spectrum_ring_append(ring, idx, blk)
    ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(reps):
            idx = capi.spectrum_ring_append(ring, idx, blk)
        ev[1].record()
        torch.cuda.synchronize()
        times.append(ev[0].elapsed_time(ev[1]) * 1e3 / reps)
    print(json.dumps({"what": "append", "olen": 1000, "us_per_block_median": round(float(np.median(times)), 2), **info}),
          flush=True)


def bench_cpu() -> None:
    from oracle import narrowband as NB

    for fft_n in LENGTHS:
        for a in AVGS:
            ring = ring_of(a * fft_n, a)
            t0 = time.perf_counter()
            NB.narrowband_spectrum(fft_n, fft_n * 4 // 5, window(fft_n), a, OVERLAP, ring, 17)
            ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({"what": "cpu", "transform": "oracle fft_cpu (the FFTW shim's transform), not FFTW",
                              "fft_n": fft_n, "fft_avg": a, "overlap": OVERLAP, "ms_per_poll": round(ms, 2)}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--cpu", action="store_true", help="also time the restatement's poll on the host")
    a = ap.parse_args()
    info = card()
    bench_polls(a.reps, a.rounds, info)
    bench_append(a.reps, a.rounds, info)
    if a.cpu:
        bench_cpu()


if __name__ == "__main__":
    main()
