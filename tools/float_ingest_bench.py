"""Float ingest timings (write_rawfilter with FILTER_RAW_F32 / CF32 / CF32_CNRMF / CF32_FSCALE).

For each front end at its default geometry (AirspyHF+ 912 kS/s, Fobos 8 MS/s, HydraSDR FLOAT32_REAL 20 MS/s and
FLOAT32_IQ 10 MS/s, 20 ms blocks):

  filter_h  wall time per block through filter.h (tests/abi/_build/float_driver.so, inline: each write returns after its
            blocks' device work) of a stream fed as the library's floats in the driver's transfer size (statistics
            drained after every write that fired a block), against the same stream fed as the restated floats
            (write_cfilter / write_rfilter), two channels, the two alternated round by round, median of --rounds rounds;
            the float figure leaves out the driver's CPU loop, which float ingest removes.  Both send 4 bytes per
            component over PCIe
  unpack    device time of kgpu_unpack8 with statistics (the store, then float_energy_kernel) over one block's window
            (M - 1 history samples and L new ones), CUDA events around --reps launches, median of --rounds rounds
  write_host  host wall time of one write_rawfilter call that fires no block, per transfer: the admission and the
            memcpy of the transfer's floats into the raw ring, walking it, in the driver's callback thread (median over
            the filter_h run's non-firing writes).  This is what the callback runs instead of its loop
  cpu_loop  host wall time per transfer of the reference's own callback loop (airspyhf.c, fobos.c, hydrasdr.c
            rx_callback, through oracle/_ref/libka9qfloat.so where it was built; the write_cfilter / write_rfilter call
            that ends it is refused at once, so no FFT is timed, and the write pointer walks the ring between calls as it
            does in radiod), median of --rounds rounds.  Its input is the same cache-warm transfer each call, while
            write_host reads each transfer once from the stream, so cpu_loop is the lower of the two as timed
  net       cpu_loop - write_host: the callback-thread time per transfer that float ingest saves (negative: it costs)

Transfer sizes: Fobos 65 536 pairs (fobos.c:386), HydraSDR 65 536 samples, AirspyHF+ 1 024 pairs.  Prints one JSON line
per measurement, each with the card's name, power limit and SM clocks read in the same run.
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

import float_ingest_ref as R  # noqa: E402

# name, L, M, COMPLEX, format, scale, transfer (samples or pairs), reference loop: (oracle prefix, open arguments)
FRONT_ENDS = [
    ("airspyhf_912k_cf32_cnrmf", 18240, 4561, True, R.CF32_CNRMF, 1.0, 1024, ("rh", ())),
    ("fobos_8m_cf32_fscale", 160000, 40001, True, R.CF32_FSCALE, 1.0, 65536, ("rf", (8e6,))),
    ("hydrasdr_20m_f32_real", 400000, 100001, False, R.F32, 1.0, 65536, ("ryf", (0,))),
    ("hydrasdr_10m_cf32", 200000, 50001, True, R.CF32, 1.0, 65536, ("ryf", (1,))),
]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


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


def samples(ncomp, rng):
    return rng.normal(0, 0.2, ncomp).astype(np.float32)


KFMT = {R.F32: "KGPU_RAW_F32", R.CF32: "KGPU_RAW_CF32", R.CF32_CNRMF: "KGPU_RAW_CF32_CNRMF", R.CF32_FSCALE: "KGPU_RAW_CF32_FSCALE"}


def bench_unpack(fe, reps, rounds, info):
    import torch

    from ka9q_radio_b200 import capi

    name, L, M, cplx, fmt, scale, _, _ = fe
    c = 2 if cplx else 1
    n = L + M - 1
    x = torch.randn(c * n, device="cuda")
    out = torch.empty(c * n, device="cuda")
    st = torch.empty(16, dtype=torch.uint8, device="cuda")
    kf = getattr(capi, KFMT[fmt])
    fn = lambda: capi.unpack8(x.data_ptr(), kf, capi.KGPU_COMPLEX if cplx else capi.KGPU_REAL, M - 1, L, 1, scale,  # noqa: E731
                              out.data_ptr(), st.data_ptr())
    fn()
    torch.cuda.synchronize()
    us = timed(fn, reps, rounds)
    print(json.dumps({"bench": "unpack", "case": name, "us_per_block": round(us, 2), **info}))


def bench_filter(fe, blocks, rounds, info):
    name, L, M, cplx, fmt, scale, xfer, _ = fe
    drv = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "float_driver.so"))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    drv.rd_open.restype = vp
    drv.rd_open.argtypes = [i, i, i, i]
    drv.rd_add_channel.argtypes = [vp, i, d, d, d]
    drv.rd_write_raw.argtypes = [vp, vp, i, i, d]
    drv.rd_write_float.argtypes = [vp, vp, i]
    drv.rd_execute.argtypes = [vp, i, i, vp]
    drv.rd_fstats.argtypes = [vp, vp, vp]
    drv.rd_close.argtypes = [vp]
    c = 2 if cplx else 1
    n = blocks * L // xfer * xfer
    x = samples(c * n, np.random.default_rng(1))
    flo = R.store(x, fmt, scale)
    if cplx:
        flo = flo.view(np.complex64)
    sessions = {}
    for kind in ("raw", "float"):
        h = drv.rd_open(L, M, int(cplx), 0)
        for olen in (480, 960):
            drv.rd_add_channel(h, olen, -0.3, 0.3, 11.0)
        sessions[kind] = h
    y = np.empty(960, np.complex64)
    st = (C.c_uint64 * 5)()
    e = C.c_double(0)
    drv.rd_fstats(sessions["raw"], C.cast(st, C.c_void_p), C.byref(e))
    times = {"raw": [], "float": []}
    host = []   # write_rawfilter calls that fired no block: host work only
    for r in range(rounds + 1):
        for kind in ("raw", "float") if r % 2 == 0 else ("float", "raw"):
            h = sessions[kind]
            t0 = time.perf_counter()
            for k in range(n // xfer):
                if kind == "raw":
                    t1 = time.perf_counter()
                    rc = drv.rd_write_raw(h, x[c * k * xfer:].ctypes.data, xfer, fmt, scale)
                    if rc == 0 and r > 0:
                        host.append(time.perf_counter() - t1)
                    if rc == 1:   # statistics change only when blocks complete
                        drv.rd_fstats(h, C.cast(st, C.c_void_p), C.byref(e))
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
    us = float(np.median(host)) * 1e6
    print(json.dumps({"bench": "write_host", "case": name, "transfer": xfer, "us_per_transfer": round(us, 2),
                      "writes": len(host), **info}))
    return us


def bench_cpu_loop(fe, rounds, info):
    name, L, M, cplx, fmt, scale, xfer, (pre, extra) = fe
    c = 2 if cplx else 1
    x = samples(c * xfer, np.random.default_rng(2))
    lib_path = ROOT / "oracle" / "_ref" / "libka9qfloat.so"
    if not lib_path.exists():
        print(json.dumps({"bench": "cpu_loop", "case": name, "loop": None, "transfer": xfer, **info}))
        return None
    lib = C.CDLL(str(lib_path))
    i, d = C.c_int, C.c_double
    getattr(lib, f"{pre}_time").argtypes = [C.c_void_p, i, i]
    getattr(lib, f"{pre}_time").restype = d
    if pre == "rh":
        lib.rh_open.argtypes = [i, i, d]
        assert lib.rh_open(L, M, scale) == 0
    elif pre == "rf":
        lib.rf_open.argtypes = [i, i, d, d]
        assert lib.rf_open(L, M, scale, *extra) == 0
    else:
        lib.ryf_open.argtypes = [i, i, i, d]
        assert lib.ryf_open(extra[0], L, M, scale) == 0
    reps = max(5, 20_000_000 // xfer)
    t = [getattr(lib, f"{pre}_time")(x.ctypes.data, xfer, reps) / reps for _ in range(rounds)]
    getattr(lib, f"{pre}_close")()
    us = float(np.median(t)) * 1e6
    print(json.dumps({"bench": "cpu_loop", "case": name, "loop": "reference", "transfer": xfer, "us_per_transfer": round(us, 2),
                      "us_per_block": round(us * L / xfer, 1), "ns_per_sample": round(us * 1e3 / xfer, 3), **info}))
    return us


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=24)
    ap.add_argument("--cpu-only", action="store_true", help="only the reference loops' CPU time (no GPU needed)")
    a = ap.parse_args()
    info = {"gpu": None} if a.cpu_only else card()
    for fe in FRONT_ENDS:
        host = None
        if not a.cpu_only:
            bench_unpack(fe, a.reps, a.rounds, info)
            host = bench_filter(fe, a.blocks, a.rounds, info)
        loop = bench_cpu_loop(fe, a.rounds, info)
        if host is not None and loop is not None:
            name, L, xfer = fe[0], fe[1], fe[6]
            print(json.dumps({"bench": "net", "case": name, "transfer": xfer, "loop_us": round(loop, 2),
                              "write_host_us": round(host, 2), "saved_us_per_transfer": round(loop - host, 2),
                              "saved_us_per_block": round((loop - host) * L / xfer, 1), **info}))


if __name__ == "__main__":
    main()
