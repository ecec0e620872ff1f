"""Raw 8-bit / packed 12-bit ingest timings (write_rawfilter, filter_ingest_stats).

  unpack  device time per block of the conversion a raw launch adds: kgpu_unpack8 over one block's window for RTL-SDR
          1.8 MS/s u8 I/Q (L = 36 000, M = 9001), kgpu_unpack_airspy12 over one block's window for Airspy R2 20 MS/s
          packed-12 (L = 400 000, M = 100 001); CUDA events around --reps launches, median of --rounds rounds
  stats   the same for the statistics: kgpu_unpack8 with d_stats (its difference to the plain unpack is the stats'
          cost), kgpu_block_stats_i16 over the Airspy window's new samples
  filter  wall time per block through filter.h (tests/abi/_build/raw_driver.so, inline: each write returns after its
          blocks' device work) of a stream fed as raw words (write_rawfilter, statistics drained every write) against the
          same stream fed as the restated floats (write_cfilter / write_rfilter), two channels, writes alternated round
          by round; the float figure leaves out the drivers' CPU conversion loop, which raw ingest removes
  scale   wall time per block through filter.h of an RX888 int16 stream (L = 48 000, M = 12 001) whose scale changes
          every --every blocks, against the same stream at one scale, alternated round by round; the difference over
          the mixed-scale launches, counted as the extra kernel launches of the changing stream (one kgpu_scale_i16
          each), is the wall time each adds; and the device time a mixed-scale launch adds to one block's forward
          transform: kgpu_scale_i16 (two changes in the window) + kgpu_forward on floats, against kgpu_forward's fused
          int16 conversion, CUDA events around --reps launches, median of --rounds rounds

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

RTL = ("rtlsdr_1m8_u8_iq", 36000, 9001, True)
AIRSPY = ("airspy_r2_20m_packed12", 400000, 100001, False)
U8, PACKED12 = 2, 1


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


def bench_kernels(reps, rounds, info):
    import torch

    from ka9q_radio_b200 import capi

    lib = capi.load()
    _, L, M, _ = RTL
    raw = torch.randint(0, 256, (2 * (L + M - 1),), dtype=torch.uint8, device="cuda")
    out = torch.empty(2 * (L + M - 1), device="cuda")
    st = torch.empty(16, dtype=torch.uint8, device="cuda")
    plain = lambda: capi.unpack8(raw.data_ptr(), capi.KGPU_RAW_U8, capi.KGPU_COMPLEX, M - 1, L, 1, 0.0046,  # noqa: E731
                                 out.data_ptr())
    with_stats = lambda: capi.unpack8(raw.data_ptr(), capi.KGPU_RAW_U8, capi.KGPU_COMPLEX, M - 1, L, 1, 0.0046,  # noqa: E731
                                      out.data_ptr(), st.data_ptr())
    for f in (plain, with_stats):
        f()
    torch.cuda.synchronize()
    t_plain = timed(plain, reps, rounds)
    t_stats = timed(with_stats, reps, rounds)
    print(json.dumps({"bench": "unpack", "case": RTL[0], "us_per_block": round(t_plain, 2), **info}))
    print(json.dumps({"bench": "stats", "case": RTL[0], "us_per_block": round(t_stats - t_plain, 2),
                      "unpack_with_stats_us": round(t_stats, 2), **info}))
    _, L, M, _ = AIRSPY
    n = L + M - 1
    packed = torch.randint(0, 2 ** 31, (n * 3 // 8,), dtype=torch.int32, device="cuda")
    i16 = torch.empty(n, dtype=torch.int16, device="cuda")
    unpack = lambda: lib.kgpu_unpack_airspy12(packed.data_ptr(), n, i16.data_ptr(), None, None)  # noqa: E731
    stats = lambda: capi.block_stats_i16(i16.data_ptr(), capi.KGPU_REAL, M - 1, L, 1, st.data_ptr(), limit=2047)  # noqa: E731
    unpack()
    stats()
    torch.cuda.synchronize()
    print(json.dumps({"bench": "unpack", "case": AIRSPY[0], "us_per_block": round(timed(unpack, reps, rounds), 2), **info}))
    print(json.dumps({"bench": "stats", "case": AIRSPY[0], "us_per_block": round(timed(stats, reps, rounds), 2), **info}))


def bench_filter(blocks, rounds, info):
    drv = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "raw_driver.so"))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    drv.rd_open.restype = vp
    drv.rd_open.argtypes = [i, i, i, i]
    drv.rd_add_channel.argtypes = [vp, i, d, d, d]
    drv.rd_write_raw.argtypes = [vp, vp, i, i, d]
    drv.rd_write_float.argtypes = [vp, vp, i]
    drv.rd_execute.argtypes = [vp, i, i, vp]
    drv.rd_stats.argtypes = [vp, vp]
    drv.rd_close.argtypes = [vp]
    rng = np.random.default_rng(1)
    for name, L, M, cplx in (RTL, AIRSPY):
        chunk = 131072
        n = blocks * L // chunk * chunk
        if cplx:
            raw = rng.integers(0, 256, 2 * n, dtype=np.uint8)
            flo = (0.0046 * (raw.astype(np.float64) - 128)).astype(np.float32).view(np.complex64)
            fmt, rb, scale = U8, 2, 0.0046
        else:
            s12 = rng.integers(0, 4096, n)
            from oracle import oracle as O   # the packer only; the timing runs libka9qgpu.so

            raw = O.airspy_pack(s12)
            scale = float(np.float32(1 / 2048))
            flo = (np.float32(scale) * (s12 - 2048).astype(np.float32)).astype(np.float32)
            fmt, rb = PACKED12, 1.5
        rawb = raw.view(np.uint8)
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
                fired = 0
                for w in range(n // chunk):
                    if kind == "raw":
                        seg = rawb[int(w * chunk * rb):int((w + 1) * chunk * rb)]
                        rc = drv.rd_write_raw(h, seg.ctypes.data, chunk, fmt, scale)
                        drv.rd_stats(h, C.cast(st, C.c_void_p))
                    else:
                        seg = flo[w * chunk:(w + 1) * chunk]
                        rc = drv.rd_write_float(h, seg.ctypes.data, chunk)
                    if rc == 1:
                        drv.rd_execute(h, 0, 1000, y.ctypes.data)
                        drv.rd_execute(h, 1, -2000, y.ctypes.data)
                    fired += rc == 1
                dt = time.perf_counter() - t0
                if r > 0:   # round 0 warms up
                    times[kind].append(dt * 1e6 / (n / L))
        for kind in ("raw", "float"):
            drv.rd_close(sessions[kind])
        print(json.dumps({"bench": "filter_h", "case": name, "raw_us_per_block": round(float(np.median(times["raw"])), 1),
                          "float_us_per_block": round(float(np.median(times["float"])), 1), "blocks": n // L, **info}))


def bench_scale(blocks, rounds, every, info):
    from ka9q_radio_b200 import capi

    lib = capi.load()
    drv = C.CDLL(str(ROOT / "tests" / "abi" / "_build" / "raw_driver.so"))
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    drv.rd_open.restype = vp
    drv.rd_open.argtypes = [i, i, i, i]
    drv.rd_add_channel.argtypes = [vp, i, d, d, d]
    drv.rd_write_i16.argtypes = [vp, vp, i, C.c_float, i]
    drv.rd_execute.argtypes = [vp, i, i, vp]
    drv.rd_close.argtypes = [vp]
    L, M, chunk = 48000, 12001, 16000
    x = np.random.default_rng(2).integers(-3000, 3000, blocks * L).astype(np.int16)
    scales = (float(np.float32(1 / 32768)), float(np.float32(10 ** (-1 / 20) / 32768)))
    y = np.empty(960, np.complex64)
    sessions = {}
    for kind in ("one", "changing"):
        h = drv.rd_open(L, M, 0, 0)
        for olen in (480, 960):
            drv.rd_add_channel(h, olen, -0.3, 0.3, 11.0)
        sessions[kind] = h
    times = {"one": [], "changing": []}
    launches = {"one": [], "changing": []}
    for r in range(rounds + 1):
        for kind in ("one", "changing") if r % 2 == 0 else ("changing", "one"):
            h = sessions[kind]
            k0 = lib.kgpu_launch_count()
            t0 = time.perf_counter()
            for w in range(blocks * L // chunk):
                sc = scales[(w * chunk // (every * L)) % 2] if kind == "changing" else scales[0]
                if drv.rd_write_i16(h, x[w * chunk:].ctypes.data, chunk, sc, 0) == 1:
                    drv.rd_execute(h, 0, 1000, y.ctypes.data)
                    drv.rd_execute(h, 1, -2000, y.ctypes.data)
            if r > 0:
                times[kind].append((time.perf_counter() - t0) * 1e6 / blocks)
                launches[kind].append(lib.kgpu_launch_count() - k0)
    for h in sessions.values():
        drv.rd_close(h)
    one, changing = float(np.median(times["one"])), float(np.median(times["changing"]))
    mixed = float(np.median(np.subtract(launches["changing"], launches["one"])))   # mixed-scale launches per round
    import torch

    m = capi.Master(L, M, capi.KGPU_REAL)
    n = L + M - 1
    d_i16 = torch.from_numpy(x[:n].copy()).cuda()
    d_f32 = torch.empty(n, device="cuda")
    d_spec = torch.empty(2 * m.spec_stride, device="cuda")
    chg = np.array([(n // 3, scales[1]), (2 * n // 3, scales[0])], dtype=[("at", "<i8"), ("scale", "<f8")])
    d_chg = torch.from_numpy(chg.view(np.uint8).copy()).cuda()
    lib.kgpu_scale_i16.argtypes = [C.c_void_p, C.c_int, C.c_long, C.c_longlong, C.c_double, C.c_void_p, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p]
    fused = lambda: m.forward(d_i16.data_ptr(), capi.KGPU_FMT_I16, scales[0], 1, d_spec.data_ptr())  # noqa: E731

    def mixed_fwd():
        lib.kgpu_scale_i16(d_i16.data_ptr(), capi.KGPU_REAL, n, 0, scales[0], d_chg.data_ptr(), 2, 0, d_f32.data_ptr(), None)
        m.forward(d_f32.data_ptr(), capi.KGPU_FMT_F32, 1.0, 1, d_spec.data_ptr())

    for f in (fused, mixed_fwd):
        f()
    torch.cuda.synchronize()
    t_fused, t_mixed = timed(fused, 200, rounds), timed(mixed_fwd, 200, rounds)
    print(json.dumps({"bench": "scale_changes", "case": "rx888_48k_i16", "every_blocks": every,
                      "fused_forward_us": round(t_fused, 2), "mixed_scale_forward_us": round(t_mixed, 2),
                      "added_device_us_per_mixed_launch": round(t_mixed - t_fused, 2),
                      "one_scale_us_per_block": round(one, 1), "changing_us_per_block": round(changing, 1),
                      "mixed_launches_per_round": mixed,
                      "added_us_per_mixed_launch": round((changing - one) * blocks / mixed, 1) if mixed else None,
                      "blocks": blocks, **info}))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=60)
    ap.add_argument("--every", type=int, default=5, help="blocks between scale changes (the scale case)")
    a = ap.parse_args()
    info = card()
    bench_kernels(a.reps, a.rounds, info)
    bench_filter(a.blocks, a.rounds, info)
    bench_scale(a.blocks, a.rounds, a.every, info)


if __name__ == "__main__":
    main()
