"""Modulated (AM) signal generator timings at cfg-2's geometry (REAL 129.6 MS/s, L = 2592000, M = 648001, one block =
20 ms of stream, 16 channels) and at a COMPLEX master of the same L and M.

  generate  device time of kgpu_siggen_generate_mod over one block's window (M - 1 history samples and L new ones, with
            the block energy) against kgpu_siggen_generate (CW) of the same carrier and noise, CUDA events around --reps
            launches, the two alternated, median of --rounds rounds
  filter_h  wall time per block through filter.h (tests/abi/_build/siggen_mod_driver.so, inline: each write returns after
            its block's device work) of a modulated master (the envelope written at filter_siggen_mod_pointer, then
            write_genfilter of one block) against a master fed the same block of floats (write_rfilter / write_cfilter),
            16 channels executed per block, the two alternated round by round, median of --rounds rounds
  h2d       host-to-device bytes per block torch.profiler records during --blocks blocks of each (the traces go to --out,
            or to a temporary directory)
  cpu_loop  thread CPU time per block of the reference's own proc_sig_gen AM loop (oracle/_ref/libka9qsiggenmod.so, where
            it was built), carrier with noise, in iterations of 100000 samples, EXCLUDING libsamplerate: its stand-in
            copies scripted envelope floats

Prints one JSON line per measurement, each with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import tempfile
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


def kind(cplx: bool) -> str:
    return "complex" if cplx else "real"


def bench_generate(reps, rounds, info):
    import torch

    from ka9q_radio_b200 import capi

    span = L + M - 1
    for cplx in (False, True):
        t = capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL
        cw, am = capi.Siggen(t, CARRIER, AMP, NOISE), capi.Siggen(t, CARRIER, AMP, NOISE)
        am.modulate(1.0)
        out = torch.empty(span * (2 if cplx else 1), device="cuda")
        mod = (0.5 * torch.sin(torch.arange(span, device="cuda", dtype=torch.float64) * 0.01)).float()
        en = torch.empty(1, dtype=torch.float64, device="cuda")
        a0 = 1000 * L - (M - 1)

        def run(g, r):
            if g is am:
                g.generate_mod(a0 + r * L, span, SCALE, out.data_ptr(), mod.data_ptr(), en.data_ptr(), 1, L)
            else:
                g.generate(a0 + r * L, span, SCALE, out.data_ptr(), en.data_ptr(), 1, L)

        run(cw, 0)
        run(am, 0)
        torch.cuda.synchronize()
        ts = {cw: [], am: []}
        for _ in range(rounds):
            for g in (cw, am):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for r in range(reps):
                    run(g, r)
                e1.record()
                torch.cuda.synchronize()
                ts[g].append(e0.elapsed_time(e1) / reps)
        emit({"bench": "generate", "type": kind(cplx), "window_samples": span,
              "am_ms_per_block": round(float(np.median(ts[am])), 4), "cw_ms_per_block": round(float(np.median(ts[cw])), 4),
              "stream_ms_per_block": round(1e3 * L / FS, 3)}, info)
        cw.close()
        am.close()


def session(lib, cplx, gen):
    from test_gpu_siggen_mod import ModGen

    s = ModGen(lib, L, M, cplx)
    for k in range(16):
        s.add(600, -0.2, 0.2, 11.0)
    if gen:
        assert s.setup(CARRIER * 1e9, AMP, NOISE) == 0 and s.modulate(1.0) == 0
    return s


def h2d_bytes(prof, path: Path) -> int:
    prof.export_chrome_trace(str(path))
    ev = json.loads(path.read_text()).get("traceEvents", [])
    return sum(int(e.get("args", {}).get("bytes", 0)) for e in ev if "HtoD" in str(e.get("name", "")))


def bench_filter_h(rounds, blocks, out_dir, info):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from test_gpu_siggen_mod import _mdriver

    lib = _mdriver()
    rng = np.random.default_rng(1)
    env = (0.5 * np.sin(np.arange(L) * 0.01)).astype(np.float32)
    shifts = [1000 + 20000 * k for k in range(16)]
    for cplx in (False, True):
        a, b = session(lib, cplx, True), session(lib, cplx, False)
        flo = rng.normal(0, 1e-3, L * (2 if cplx else 1)).astype(np.float32)
        if cplx:
            flo = flo.view(np.complex64)

        def one(s, gen):
            t = time.perf_counter()
            for _ in range(blocks):
                assert (s.mod(env, SCALE) if gen else s.flt(flo)) == 1
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
        emit({"bench": "filter_h", "type": kind(cplx), "channels": 16, "am_ms_per_block": round(ga, 3),
              "floats_ms_per_block": round(fb, 3), "stream_ms_per_block": round(1e3 * L / FS, 3),
              "am_x_real_time": round(1e3 * L / FS / ga, 2)}, info)
        rec = {}
        for name, s, gen in (("am", a, True), ("floats", b, False)):
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                one(s, gen)
                torch.cuda.synchronize()
            rec[f"{name}_h2d_bytes_per_block"] = h2d_bytes(prof, Path(out_dir) / f"siggen_mod_{kind(cplx)}_{name}.pt.trace.json")
            rec[f"{name}_h2d_bytes_per_block"] //= blocks
        emit({"bench": "h2d", "type": kind(cplx), "blocks": blocks, **rec}, info)
        a.close()
        b.close()


def bench_cpu_loop(rounds, info):
    p = ROOT / "oracle" / "_ref" / "libka9qsiggenmod.so"
    if not p.exists():
        emit({"bench": "cpu_loop", "skipped": "oracle/_ref/libka9qsiggenmod.so not built"}, info)
        return
    from test_siggen_mod_cpu import mod_oracle

    lib = mod_oracle()
    n, w = 1_200_000, 100_000
    sizes = np.full(n // w, w, np.int32)
    scales = np.full(len(sizes), SCALE)
    env = (0.5 * np.sin(np.arange(n) * 0.01)).astype(np.float32)
    ts = []
    for _ in range(rounds):
        cpu = C.c_double(0)
        assert lib.rs_run_mod(1, 4_000_000, 1001, CARRIER * 1e9, AMP, NOISE, 1, sizes.ctypes.data, sizes.ctypes.data,
                              scales.ctypes.data, len(sizes), env.ctypes.data, None, None, C.byref(cpu)) == 0
        ts.append(cpu.value / n)
    ns = float(np.median(ts)) * 1e9
    emit({"bench": "cpu_loop", "type": "real", "modulation": "AM", "libsamplerate": "excluded",
          "ns_per_sample": round(ns, 2), "ms_per_block": round(ns * L * 1e-6, 2),
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
        raise SystemExit("siggen_mod_bench needs a GPU")
    info = card()
    bench_generate(a.reps, a.rounds, info)
    with tempfile.TemporaryDirectory() as tmp:
        out = Path(a.out) if a.out else Path(tmp)
        out.mkdir(parents=True, exist_ok=True)
        bench_filter_h(a.rounds, a.blocks, out, info)
    bench_cpu_loop(3, info)


if __name__ == "__main__":
    main()
