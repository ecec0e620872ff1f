"""HackRF and FUNcube I/Q correction timings (filter_iq_correction_setup, write_rawfilter with *_IQCORR).

  device  device time per block of what a corrected launch runs in place of the plain unpack: kgpu_iq_moments over the
          block's new samples, kgpu_iq_scan over its writes and kgpu_iq_apply over its window, for HackRF 20 MS/s
          (L = 400 000, M = 100 001, 131 072-pair transfers) and FUNcube (L = 3840, M = 961, 960-pair blocks); CUDA
          events around --reps launches, median of --rounds rounds
  filter  wall time per block through filter.h (tests/abi/_build/iqcorr_driver.so, inline: each write returns after its
          blocks' device work) of the HackRF stream fed as corrected s8 against the same stream fed as the restated
          floats (write_cfilter), two channels, alternated round by round; the float figure leaves out the driver's loop
  driver  host CPU time per 131 072-pair transfer of the reference's own rx_callback (oracle/_ref/libka9qiqcorr.so,
          where it was built), on a master large enough that no block fires while it is timed: the driver-thread work
          a patched hackrf.c no longer does

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
sys.path.insert(0, str(ROOT / "tests"))

HACKRF = ("hackrf_20m_s8", 400000, 100001, 131072, 1)
FUNCUBE = ("funcube_192k_s16", 3840, 961, 960, 2)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power}


def timed(fn, reps, rounds):
    import torch

    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / reps)
    return float(np.median(out))


def bench_device(reps, rounds, info):
    import torch

    import iq_correction_ref as R
    from ka9q_radio_b200 import capi

    for name, L, M, chunk, fmt in (HACKRF, FUNCUBE):
        comp = np.int8 if fmt == 1 else np.int16
        win = M - 1 + L
        rng = np.random.default_rng(1)
        words = rng.integers(-100, 100, 2 * (win + chunk), dtype=np.int64).astype(comp)
        nw = (win + chunk - 1) // chunk + 1
        cap = 4 * nw
        tab = np.zeros(cap, np.dtype([("first", "<i8"), ("n", "<i8"), ("scale", "<f8"), ("m", "<i8", 5), ("overs", "<i8"),
                                      ("last_over", "<i8")]))
        for w in range(nw):
            tab[w] = (w * chunk, chunk, 1.0 / 128, (0,) * 5, 0, -1)
        d_words = torch.from_numpy(words).to("cuda:0")
        d_tab = torch.from_numpy(tab.view(np.uint8).copy()).to("cuda:0")
        p = R.Params.hackrf(20e6) if fmt == 1 else R.Params.funcube(chunk)
        d_coef = torch.zeros(cap * 8, dtype=torch.float64, device="cuda:0")
        d_coef[:8] = torch.tensor([p.state[k] for k in R.STATE], dtype=torch.float64)
        d_rec = torch.zeros(cap * 136, dtype=torch.uint8, device="cuda:0")
        d_out = torch.empty(2 * win, dtype=torch.float32, device="cuda:0")
        a0 = M - 1                      # the block's window starts at pair 0, its new pairs at M - 1
        lo, hi = (M - 1) // chunk, (win - 1) // chunk
        kfmt = capi.KGPU_IQ_S8 if fmt == 1 else capi.KGPU_IQ_S16
        kind = capi.IQ_HACKRF if fmt == 1 else capi.IQ_FUNCUBE
        new = d_words.data_ptr() + 2 * a0 * words.itemsize
        nscan = max(1, L // chunk)

        def moments():
            capi.iq_moments(new, kfmt, a0, L, d_tab.data_ptr(), cap, lo, hi - lo + 1)

        def scan():
            capi.iq_scan(d_tab.data_ptr(), d_coef.data_ptr(), cap, lo, nscan, kind, p.dc_alpha, p.gp, d_rec.data_ptr())

        def apply():
            capi.iq_apply(d_words.data_ptr(), kfmt, 0, win, d_tab.data_ptr(), d_coef.data_ptr(), cap, 0, hi + 1,
                          d_out.data_ptr())

        for fn in (moments, scan, apply):
            fn()
        torch.cuda.synchronize()
        t = {k: timed(fn, reps, rounds) for k, fn in (("moments", moments), ("scan", scan), ("apply", apply))}
        print(json.dumps({"bench": "iq_correction_device", "config": name, "L": L, "M": M, "write": chunk,
                          "moments_us": round(t["moments"], 2), "scan_us": round(t["scan"], 2),
                          "apply_us": round(t["apply"], 2), "total_us": round(sum(t.values()), 2),
                          "samples": win, **info}), flush=True)


def bench_filter(rounds, info):
    import iq_correction_ref as R
    import test_gpu_iq_correction as T
    import test_iq_correction_cpu as TC

    lib = T._driver()
    name, L, M, chunk, _ = HACKRF
    nw = 48
    raw = TC.hackrf_bytes(nw * chunk, seed=2)
    writes = [raw[2 * w * chunk: 2 * (w + 1) * chunk] for w in range(nw)]
    p = R.Params.hackrf(20e6)
    fl, _ = R.run(p, R.S8, writes, [TC.HACKRF_SCALE] * nw)
    flo = np.ascontiguousarray(np.concatenate(fl))
    blocks = nw * chunk // L
    res = {"raw": [], "float": []}
    for _ in range(rounds):
        for kind in ("raw", "float"):
            with T.Session(lib, L, M) as s:
                if kind == "raw":
                    assert s.setup(R.S8, p) == 0
                s.add(800, -0.4, 0.4, 11.0)
                s.add(4000, -0.45, 0.45, 9.0)
                if kind == "raw":
                    sec = lib.iq_time(s.h, raw.ctypes.data, chunk, nw, 2 * chunk, 1, R.S8, TC.HACKRF_SCALE)
                else:
                    sec = lib.iq_time(s.h, flo.ctypes.data, chunk, nw, 8 * chunk, 0, 0, 0.0)
                res[kind].append(sec * 1e6 / blocks)
    print(json.dumps({"bench": "iq_correction_filter_h", "config": name, "blocks_per_round": blocks,
                      "raw_us_per_block": round(float(np.median(res["raw"])), 1),
                      "float_us_per_block": round(float(np.median(res["float"])), 1), **info}), flush=True)


def bench_driver(rounds, info):
    import test_iq_correction_cpu as TC

    p = ROOT / "oracle" / "_ref" / "libka9qiqcorr.so"
    if not p.exists():
        print(json.dumps({"bench": "iq_correction_driver_cpu", "config": HACKRF[0], "us_per_transfer": "not measured",
                          "why": "oracle/_ref/libka9qiqcorr.so not built", **info}), flush=True)
        return
    lib = TC.ref_lib()
    chunk = HACKRF[3]
    buf = TC.hackrf_bytes(chunk, seed=3)
    per = []
    for _ in range(rounds):
        assert lib.rh_open(20e6, 1 << 22, 1, TC.HACKRF_SCALE) == 0   # no block fires within 24 transfers
        per.append(lib.rh_time(buf.ctypes.data, buf.size, 24) * 1e6 / 24)
        lib.rh_close()
    print(json.dumps({"bench": "iq_correction_driver_cpu", "config": HACKRF[0], "write": chunk,
                      "us_per_transfer": round(float(np.median(per)), 1),
                      "what": "reference rx_callback host CPU time, the driver-thread work the patch removes",
                      **info}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    info = card()
    t0 = time.time()
    bench_device(a.reps, a.rounds, info)
    bench_filter(a.rounds, info)
    bench_driver(a.rounds, info)
    print(json.dumps({"bench": "iq_correction_done", "seconds": round(time.time() - t0, 1)}), flush=True)


if __name__ == "__main__":
    main()
