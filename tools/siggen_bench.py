"""Signal generator timings at cfg-2's geometry (129.6 MS/s, L = 2592000, M = 648001, one block = 20 ms of stream).

  generate  device time of kgpu_siggen_generate over one block's window (M - 1 history samples and L new ones, with the
            block energy), CUDA events around --reps launches, median of --rounds rounds; REAL and COMPLEX, noise only and
            carrier with noise
  filter_h  wall time per block through filter.h (tests/abi/_build/siggen_driver.so, inline: each write returns after
            its block's device work) of a generated master (write_genfilter of one block) against a master fed the
            same block of floats (write_rfilter), 16 channels executed per block, the two alternated round by round,
            median of --rounds rounds; the float figure leaves out the driver's CPU loop that makes the floats
  h2d       host-to-device copies torch.profiler records during --blocks generated blocks and during as many float-fed
            ones (the trace goes to --out)
  cpu_loop  thread CPU time per block of the reference's own proc_sig_gen CW loop (oracle/_ref/libka9qsiggen.so, where it
            was built), noise with a carrier, in writes of 100000 samples to a master too long for any block to fire

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
sys.path.insert(0, str(ROOT / "tests"))

L, M, FS = 2592000, 648001, 129.6e6
NOISE, AMP, SCALE = 10 ** (-30 / 20), 10 ** (-10 / 20), 1.0 / (32768 * 1.7)
CARRIER = 10.7e6 / FS


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power}


def emit(rec: dict, info: dict) -> None:
    print(json.dumps({**rec, **info}), flush=True)


def bench_generate(reps, rounds, info):
    import torch

    from ka9q_radio_b200 import capi

    span = L + M - 1
    for cplx in (False, True):
        for amp in (0.0, AMP):
            g = capi.Siggen(capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, CARRIER, amp, NOISE)
            out = torch.empty(span * (2 if cplx else 1), device="cuda")
            en = torch.empty(1, dtype=torch.float64, device="cuda")
            a0 = 1000 * L - (M - 1)
            g.generate(a0, span, SCALE, out.data_ptr(), en.data_ptr(), 1, L)
            torch.cuda.synchronize()
            ts = []
            for _ in range(rounds):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for r in range(reps):
                    g.generate(a0 + r * L, span, SCALE, out.data_ptr(), en.data_ptr(), 1, L)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) / reps)
            ms = float(np.median(ts))
            emit({"bench": "generate", "type": "complex" if cplx else "real", "carrier": amp != 0, "window_samples": span,
                  "ms_per_block": round(ms, 4), "stream_ms_per_block": round(1e3 * L / FS, 3),
                  "hbm_gbs": round(4 * (2 if cplx else 1) * span / (ms * 1e-3) / 1e9, 1)}, info)
            g.close()


def session(lib, gen):
    from test_gpu_siggen import Gen

    s = Gen(lib, L, M, False)
    for k in range(16):
        s.add(600, -0.2, 0.2, 11.0)
    if gen:
        assert s.setup(CARRIER * 1e9, AMP, NOISE) == 0
    return s


def bench_filter_h(rounds, blocks, out_dir, info):
    import torch

    from test_gpu_siggen import _gdriver

    lib = _gdriver()
    a, b = session(lib, True), session(lib, False)
    flo = np.random.default_rng(1).normal(0, 1e-3, L).astype(np.float32)
    shifts = [1000 + 20000 * k for k in range(16)]

    def one(s, gen):
        t = time.perf_counter()
        for _ in range(blocks):
            assert (s.gen(L, SCALE) if gen else s.flt(flo)) == 1
            for ch in range(16):
                s.exe(ch, shifts[ch])
        return (time.perf_counter() - t) / blocks

    one(a, True)
    one(b, False)
    ta, tb = [], []
    for _ in range(rounds):
        ta.append(one(a, True))
        tb.append(one(b, False))
    ga, fb = float(np.median(ta)) * 1e3, float(np.median(tb)) * 1e3
    emit({"bench": "filter_h", "channels": 16, "generated_ms_per_block": round(ga, 3), "floats_ms_per_block": round(fb, 3),
          "stream_ms_per_block": round(1e3 * L / FS, 3), "generated_x_real_time": round(1e3 * L / FS / ga, 2)}, info)
    from torch.profiler import ProfilerActivity, profile

    counts = {}
    for name, s, gen in (("generated", a, True), ("floats", b, False)):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            one(s, gen)
            torch.cuda.synchronize()
        h2d = [e for e in prof.events() if "HtoD" in e.name or "Memcpy HtoD" in e.name]
        counts[name] = len(h2d)
        if out_dir:
            prof.export_chrome_trace(str(Path(out_dir) / f"siggen_{name}.pt.trace.json"))
    emit({"bench": "h2d", "blocks": blocks, "generated_h2d_copies": counts["generated"], "floats_h2d_copies": counts["floats"]},
         info)
    a.close()
    b.close()


def bench_cpu_loop(rounds, info):
    p = ROOT / "oracle" / "_ref" / "libka9qsiggen.so"
    if not p.exists():
        emit({"bench": "cpu_loop", "skipped": "oracle/_ref/libka9qsiggen.so not built"}, info)
        return
    from test_siggen_cpu import oracle

    lib = oracle()
    n, w = 1_200_000, 100_000
    sizes = np.full(n // w, w, np.int32)
    scales = np.full(len(sizes), SCALE)
    ts = []
    for _ in range(rounds):
        cpu = C.c_double(0)
        assert lib.rs_run(1, 4_000_000, 1001, CARRIER * 1e9, AMP, NOISE, sizes.ctypes.data, scales.ctypes.data, len(sizes),
                          None, None, C.byref(cpu)) == 0
        ts.append(cpu.value / n)
    ns = float(np.median(ts)) * 1e9
    emit({"bench": "cpu_loop", "type": "real", "ns_per_sample": round(ns, 2), "ms_per_block": round(ns * L * 1e-6, 2),
          "stream_ms_per_block": round(1e3 * L / FS, 3), "cpu_seconds_per_stream_second": round(ns * 1e-9 * FS, 3)}, info)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--out", default="", help="directory for the torch.profiler traces")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("siggen_bench needs a GPU")
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
    info = card()
    bench_generate(a.reps, a.rounds, info)
    bench_filter_h(a.rounds, a.blocks, a.out, info)
    bench_cpu_loop(3, info)


if __name__ == "__main__":
    main()
