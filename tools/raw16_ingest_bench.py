"""Raw 16-bit ingest timings (write_rawfilter with FILTER_RAW_S16 / U16 / SC16Q11, write_rawfilter_planar).

For each front end (SDRplay 2 MS/s, bladeRF 12 and 61.44 MS/s, HydraSDR int16 REAL 20 MS/s and int16 I/Q 10 MS/s):

  filter_h  wall time per block through filter.h (tests/abi/_build/raw16_driver.so, inline: each write returns after its
            blocks' device work) of a stream fed as raw words in the driver's transfer size (statistics drained after
            every write that fired a block), against the same stream fed as the restated floats (write_cfilter / write_rfilter), two channels,
            the two alternated round by round, median of --rounds rounds; the float figure leaves out the driver's CPU
            conversion loop, which raw ingest removes
  unpack    device time of kgpu_unpack8 with statistics over one block's window (M - 1 history samples and L new ones),
            CUDA events around --reps launches, median of --rounds rounds; its bytes (2 in and 4 out per component) over
            that time as a share of the H100 SXM's 3.35 TB/s
  cpu_loop  host wall time per transfer of the reference's own conversion loop (hydrasdr.c rx_callback, bladerf.c
            bladerf_process, through oracle/_ref/libka9qraw16.so where it was built; the write_*filter call that ends it
            is refused at once, so no FFT is timed), median of --rounds rounds.  SDRplay's callback is not built (its
            API has no stub), so its loop is not timed

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

import raw16_ingest_ref as R  # noqa: E402

HBM_TBS = 3.35
# name, L, M, COMPLEX, format, planar, scale, transfer (samples or pairs), reference loop: (oracle kind, hydrasdr kind)
FRONT_ENDS = [
    ("sdrplay_2m_s16_planar", 40000, 10001, True, R.S16, True, 1 / 32768, 1008, None),
    ("bladerf_12m_sc16q11", 240000, 60001, True, R.SC16Q11, False, 1.0, 240640, ("bladerf", None)),
    ("bladerf_61m44_sc16q11", 1228800, 307201, True, R.SC16Q11, False, 1.0, 1228800, ("bladerf", None)),
    ("hydrasdr_20m_int16_real", 400000, 100001, False, R.S16, False, 1 / 32768, 65536, ("hydrasdr", 0)),
    ("hydrasdr_10m_int16_iq", 200000, 50001, True, R.S16, False, 1 / 32768, 65536, ("hydrasdr", 2)),
]


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


def words(ncomp, fmt, rng):
    if fmt == R.SC16Q11:
        return rng.integers(0, 65536, ncomp).astype(np.uint16)
    v = np.clip(rng.normal(0, 6000, ncomp), -32768, 32767).astype(np.int64)
    return (v + 32768).astype(np.uint16) if fmt == R.U16 else v.astype(np.int16).view(np.uint16)


def bench_unpack(fe, reps, rounds, info):
    import torch

    from ka9q_radio_b200 import capi

    name, L, M, cplx, fmt, _, scale, _, _ = fe
    c = 2 if cplx else 1
    n = L + M - 1
    kfmt = {R.S16: capi.KGPU_RAW_S16, R.U16: capi.KGPU_RAW_U16, R.SC16Q11: capi.KGPU_RAW_SC16Q11}[fmt]
    w = torch.randint(-32768, 32768, (c * n,), dtype=torch.int16, device="cuda")
    out = torch.empty(c * n, device="cuda")
    st = torch.empty(16, dtype=torch.uint8, device="cuda")
    fn = lambda: capi.unpack8(w.data_ptr(), kfmt, capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, M - 1, L, 1, scale,  # noqa: E731
                              out.data_ptr(), st.data_ptr())
    fn()
    torch.cuda.synchronize()
    us = timed(fn, reps, rounds)
    nbytes = 6 * c * n
    print(json.dumps({"bench": "unpack", "case": name, "us_per_block": round(us, 2), "bytes": nbytes,
                      "share_of_hbm": round(nbytes / (us * 1e-6) / (HBM_TBS * 1e12), 3), **info}))


def bench_filter(fe, blocks, rounds, info):
    name, L, M, cplx, fmt, planar, scale, xfer, _ = fe
    drv = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "raw16_driver.so"))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    drv.rd_open.restype = vp
    drv.rd_open.argtypes = [i, i, i, i]
    drv.rd_add_channel.argtypes = [vp, i, d, d, d]
    drv.rd_write_raw.argtypes = [vp, vp, i, i, d]
    drv.rd_write_planar.argtypes = [vp, vp, vp, i, d]
    drv.rd_write_float.argtypes = [vp, vp, i]
    drv.rd_execute.argtypes = [vp, i, i, vp]
    drv.rd_stats.argtypes = [vp, vp]
    drv.rd_close.argtypes = [vp]
    c = 2 if cplx else 1
    n = blocks * L // xfer * xfer
    w = words(c * n, fmt, np.random.default_rng(1))
    flo = R.unpack16(w, fmt, scale)
    if cplx:
        flo = flo.view(np.complex64)
    if planar:
        xi, xq = np.ascontiguousarray(w.view(np.int16)[0::2]), np.ascontiguousarray(w.view(np.int16)[1::2])
    sessions = {}
    for kind in ("raw", "float"):
        h = drv.rd_open(L, M, int(cplx), 0)
        for olen in (480, 960):
            drv.rd_add_channel(h, olen, -0.3, 0.3, 11.0)
        sessions[kind] = h
    y = np.empty(960, np.complex64)
    st = (C.c_uint64 * 6)()
    drv.rd_stats(sessions["raw"], C.cast(st, C.c_void_p))
    times = {"raw": [], "float": []}
    for r in range(rounds + 1):
        for kind in ("raw", "float") if r % 2 == 0 else ("float", "raw"):
            h = sessions[kind]
            t0 = time.perf_counter()
            for k in range(n // xfer):
                if kind == "raw":
                    if planar:
                        rc = drv.rd_write_planar(h, xi[k * xfer:].ctypes.data, xq[k * xfer:].ctypes.data, xfer, scale)
                    else:
                        rc = drv.rd_write_raw(h, w[c * k * xfer:].ctypes.data, xfer, fmt, scale)
                    if rc == 1:   # statistics change only when blocks complete
                        drv.rd_stats(h, C.cast(st, C.c_void_p))
                else:
                    rc = drv.rd_write_float(h, flo[k * xfer:].ctypes.data, xfer)
                if rc == 1:
                    drv.rd_execute(h, 0, 1000, y.ctypes.data)
                    drv.rd_execute(h, 1, -2000, y.ctypes.data)
            if r > 0:   # round 0 warms up
                times[kind].append((time.perf_counter() - t0) * 1e6 / (n / L))
    for h in sessions.values():
        drv.rd_close(h)
    print(json.dumps({"bench": "filter_h", "case": name, "raw_us_per_block": round(float(np.median(times["raw"])), 1),
                      "float_us_per_block": round(float(np.median(times["float"])), 1), "transfer": xfer,
                      "blocks": n // L, **info}))


def bench_cpu_loop(fe, rounds, info):
    name, L, M, cplx, fmt, _, scale, xfer, loop = fe
    c = 2 if cplx else 1
    w = words(c * xfer, fmt, np.random.default_rng(2))
    lib_path = ROOT / "oracle" / "_ref" / "libka9qraw16.so"
    reps = max(5, 20_000_000 // xfer)
    if loop is not None and lib_path.exists():
        lib = C.CDLL(str(lib_path))
        lib.ry_open.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double]
        lib.ry_time.argtypes = [C.c_void_p, C.c_int, C.c_int]
        lib.ry_time.restype = C.c_double
        lib.rb_open.argtypes = [C.c_int, C.c_int]
        lib.rb_time.argtypes = [C.c_void_p, C.c_int, C.c_int]
        lib.rb_time.restype = C.c_double
        if loop[0] == "bladerf":
            assert lib.rb_open(L, M) == 0
            t = [lib.rb_time(w.ctypes.data, xfer, reps) / reps for _ in range(rounds)]
            lib.rb_close()
        else:
            assert lib.ry_open(loop[1], L, M, scale) == 0
            t = [lib.ry_time(w.ctypes.data, xfer, reps) / reps for _ in range(rounds)]
            lib.ry_close()
    else:
        print(json.dumps({"bench": "cpu_loop", "case": name, "loop": None, "transfer": xfer, **info}))
        return
    us = float(np.median(t)) * 1e6
    print(json.dumps({"bench": "cpu_loop", "case": name, "loop": "reference", "transfer": xfer, "us_per_transfer": round(us, 1),
                      "us_per_block": round(us * L / xfer, 1), **info}))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=24)
    a = ap.parse_args()
    info = card()
    for fe in FRONT_ENDS:
        bench_unpack(fe, a.reps, a.rounds, info)
        bench_filter(fe, a.blocks, a.rounds, info)
        bench_cpu_loop(fe, a.rounds, info)


if __name__ == "__main__":
    main()
