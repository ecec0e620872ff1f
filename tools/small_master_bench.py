"""Small masters against default masters: P threads, each with a master of its own, written and read block by block.

Workloads (radiod's per-channel secondary masters):
  composite  wfm.c's REAL 7680 / 7681 master with mono (REAL 960), pilot and L-R (COMPLEX 960) at wfm.c's shifts; each
             thread writes 7680 floats and reads its three slaves per block
  filter2    radio.c's COMPLEX 480 / 545 master (blocking 2 at 12 kHz) with one COMPLEX 480 slave, shift 0
For P = 1, 64 and 256 the default and the small path alternate in the same process (default, small, default, small).
Each line: the wall time per block per thread (the slowest thread's write / read loop over the blocks, after every
thread has set up), the device operations per block as counted from filter_abi.c, filter_small_master_bytes, and the
default master's tables sized by its 2048 channel slots, also counted from the code.  The card's name and power limit
come first.  Run from the repository root after __graft_entry__.build(); needs a GPU.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
REAL, COMPLEX = 2, 1
ND, SLOTS = 4, 2048


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def default_ops(slave_paths, windows):
    """Device operations one block of a default master issues (execute_filter_input_n): the window H2D (1, or 2 at the
    ring's end), the two forward kernels, one channel launch per path class, the output D2H, the powers' D2H and one
    D2H per spectrum window, and four event records (the timing start, two kernel-done records, the block's event)."""
    return {"h2d": "1-2", "kernels": 2 + slave_paths, "d2h": 2 + windows, "events": 4}


def small_ops():
    return {"h2d": "1-2", "kernels": 1, "d2h": 1, "events": 1}


def default_tables_bytes():
    """Bytes of a default master sized by its 2048 channel slots alone, from filter_abi.c and kgpu.cu: pinned and device
    powers (float) and noise estimates (double) for ND x 2048, the per-slot snapshots (ND x 2048 x 64 B) and current
    parameters (2048 x 58 B), and the bank's device descriptors, order, aux, shifts and FM memory (2048 x 136 B)."""
    return 2 * ND * SLOTS * (4 + 8) + ND * SLOTS * 64 + SLOTS * 58 + SLOTS * 136


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", default="1,64,256")
    ap.add_argument("--blocks", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    from oracle import oracle as O
    sys.path.insert(0, str(ROOT / "tests"))
    from test_gpu_small_masters import _bind, _threads, _composite_slaves

    lib = _bind("tests/abi/_build/small_driver.so")
    lib.small_master_bytes.restype = C.c_long
    lib.small_master_bytes.argtypes = [C.c_int] * 4
    print(json.dumps({"card": card()}), flush=True)
    comp, shifts = _composite_slaves(O)
    work = {
        # mono (REAL out) and the two COMPLEX slaves run as two path classes on a default master; estimate_noise's
        # windows around the three shifts merge into one D2H
        "composite": (7680, 7681, REAL, comp, shifts, default_ops(2, 1)),
        "filter2": (480, 545, COMPLEX, [(480, -0.21, 0.07, 7.0, COMPLEX)], [0], default_ops(1, 1)),
    }
    for name, (L, M, t, slaves, sh, dops) in work.items():
        nb = args.blocks
        x = (O.siggen_real(nb * L, 0.1, 0.01, 0.0495, 1.0) if t == REAL else O.siggen_complex(nb * L, 0.1, 0.01, 0.0371, 1.0))
        small_bytes = lib.small_master_bytes(L, M, t, len(slaves))
        for P in [int(p) for p in args.threads.split(",")]:
            _threads(lib, P, L, M, t, slaves, sh, x[: 2 * L], 2, small=False)   # warm-up: plans, modules, allocations
            _threads(lib, P, L, M, t, slaves, sh, x[: 2 * L], 2, small=True)
            res = {False: [], True: []}
            for _ in range(args.rounds):
                for small in (False, True):
                    ns, _, count = _threads(lib, P, L, M, t, slaves, sh, x, nb, small, keep=False)
                    assert ns > 0 and count == (P if small else 0)
                    res[small].append(ns / nb / 1e3)
            for small in (False, True):
                print(json.dumps({"workload": name, "P": P, "path": "small" if small else "default",
                                  "us_per_block_per_thread": [round(v, 1) for v in res[small]],
                                  "device_ops_per_block": small_ops() if small else dops,
                                  "bytes": small_bytes if small else f"> {default_tables_bytes()} (2048-slot tables alone)"}),
                      flush=True)


if __name__ == "__main__":
    main()
