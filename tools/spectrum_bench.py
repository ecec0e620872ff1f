"""Wideband spectrum analyzer timings on the cfg-2 front end (RX888, REAL int16, 129.6 MS/s; L = 2 592 000, M = 648 001).

  poll    device time of one kgpu_spectrum_run (CUDA events, mean of --reps) on an int16 ring with the capacity of the
          filter.h host ring, for fft_n 6480 / 129 600 / 518 400 (rbw 20 kHz / 1 kHz / 250 Hz) and one Bluestein length,
          fft_avg 1 and 10, overlap 0 and 0.5
  block   wall time per 20 ms block of the filter.h forward pipeline fed by write_i16filter, without a spectrum slave and
          with one polled at 10 Hz (every 5th block); the difference is the analyzer's cost per block
  cpu     the reference's own wideband_poll through oracle/_ref on this host: its transform is the oracle's fft_cpu
          through the FFTW shim, not FFTW with wisdom, so it gives the CPU's scale, not radiod's speed

Prints one JSON line per measurement, each with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

FS, L, M = 129.6e6, 2592000, 648001
RING = (4 * (L + M - 1) * 4 + 4095) // 4096 * 4096 // 4  # filter.h: page_round(ND * N * sizeof(float)) / sizeof(float)
LENGTHS = [6480, 129600, 518400, 104400]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power}


def window(n):
    w = np.kaiser(n + 1, 11.0)[:n]
    return (w / w.sum()).astype(np.float32)


def bench_polls(reps: int, info: dict) -> None:
    import torch

    from ka9q_radio_b200 import capi

    ring = torch.randint(-2000, 2000, (RING,), dtype=torch.int16, device="cuda")
    bins = torch.empty(65536, device="cuda")
    for fft_n in LENGTHS:
        bin_count = min(fft_n // 2, 65536)
        sp = capi.Spectrum(fft_n, capi.KGPU_REAL, bin_count)
        sp.set_window(window(fft_n))
        for fft_avg in (1, 10):
            for overlap in (0.0, 0.5):
                run = lambda: sp.run(ring, RING // 2, bin_count // 2, fft_avg, overlap, bins, scale=1 / 32768)
                for _ in range(3):
                    run()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                for _ in range(reps):
                    run()
                b.record()
                torch.cuda.synchronize()
                us = a.elapsed_time(b) * 1e3 / reps
                print(json.dumps({"what": "poll", "fft_n": fft_n, "path": sp.describe().split()[0], "fft_avg": fft_avg,
                                  "overlap": overlap, "us_per_poll": round(us, 1), **info}), flush=True)
        sp.close()


def bench_blocks(nblocks: int, info: dict) -> None:
    import torch

    d = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "spectrum_driver.so"))
    d.sd_write_i16.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int]
    d.sd_setup.argtypes = [C.c_int, C.c_int, C.c_void_p]
    d.sd_poll.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    x = np.random.default_rng(1).integers(-2000, 2000, L).astype(np.int16)
    for fft_n, fft_avg in [(None, 0), (129600, 10), (518400, 10)]:
        assert d.sd_open(L, M, 0) == 0
        bins = np.empty(65536, np.float32)
        end = C.c_uint64(0)
        if fft_n:
            w = window(fft_n)
            assert d.sd_setup(fft_n, 32768, w.ctypes.data) == 0
        for _ in range(5):
            d.sd_write_i16(x.ctypes.data, L, 1 / 32768, 0)
        t0 = time.perf_counter()
        for j in range(nblocks):
            d.sd_write_i16(x.ctypes.data, L, 1 / 32768, 0)
            if fft_n and j % 5 == 4:  # 10 Hz at 20 ms blocks
                d.sd_poll(16384, fft_avg, 0.5, bins.ctypes.data, C.cast(C.pointer(end), C.c_void_p))
        if fft_n:  # waits for every block issued so far
            d.sd_poll(16384, 1, 0.5, bins.ctypes.data, C.cast(C.pointer(end), C.c_void_p))
        else:
            torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / nblocks
        d.sd_close()
        print(json.dumps({"what": "block", "spectrum": fft_n or "none", "fft_avg": fft_avg, "ms_per_block": round(ms, 3),
                          **info}), flush=True)


def bench_cpu(info: dict) -> None:
    from oracle import spectrum as S

    if not S.have_ref():
        print(json.dumps({"what": "cpu", "skipped": "oracle/_ref/libka9qspectrum.so not built"}))
        return
    ring = np.random.default_rng(2).standard_normal(RING).astype(np.float32)
    for fft_n in LENGTHS[:3]:
        for fft_avg in (1, 10):
            t0 = time.perf_counter()
            S.ref_wideband_poll(True, fft_n, fft_n // 2, window(fft_n), fft_n // 4, fft_avg, 0.5, ring, RING // 2)
            ms = (time.perf_counter() - t0) * 1e3
            print(json.dumps({"what": "cpu", "transform": "oracle fft_cpu via the FFTW shim, not FFTW with wisdom",
                              "fft_n": fft_n, "fft_avg": fft_avg, "overlap": 0.5, "ms_per_poll": round(ms, 1)}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=100)
    ap.add_argument("--cpu", action="store_true", help="also time the reference's wideband_poll on the host")
    a = ap.parse_args()
    info = card()
    bench_polls(a.reps, info)
    bench_blocks(a.blocks, info)
    if a.cpu:
        bench_cpu(info)


if __name__ == "__main__":
    main()
