#!/usr/bin/env python3
"""Compare the spectra of two kernel variants on the same input (cfg-2 sizes, REAL int16 and COMPLEX float).
usage: ab_check.py static=0   (the generic kernels, compared with each master's default kernel pair)"""
import sys
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from ka9q_radio_b200 import workloads
W = workloads.cfg2()
from ka9q_radio_b200 import capi
from ka9q_radio_b200.channelizer import Channelizer
lib = capi.load(); dev = torch.device("cuda:0")
VARIANTS = ("default", "static=0")
for v in sys.argv[1:]:
    if v not in VARIANTS: sys.exit("variants: %s" % ", ".join(VARIANTS))
def setv(v):
    lib.kgpu_use_static_kernels(0 if v == "static=0" else 1)
B = 5
rng = np.random.default_rng(1)
W4 = workloads.cfg4()
for name, in_type, L, M in (("real-i16", capi.KGPU_REAL, W.L, W.M), ("complex-f32", capi.KGPU_COMPLEX, W.L // 2, (W.M - 1) // 2 + 1),
                            ("cfg4-complex-i16", capi.KGPU_COMPLEX, W4.L, W4.M), ("cfg4-complex-f32", capi.KGPU_COMPLEX, W4.L, W4.M)):
    cz = Channelizer(L, M, in_type, dev, capacity=64)
    nch = 43
    for k in range(nch):  # upright, inverted and band-edge channels (REAL: |shift| < N/2; COMPLEX: wraps)
        sh = (750_000 + 9_973 * k) * (1 if k % 3 else -1) if in_type == capi.KGPU_REAL else (-800_000 + 37_001 * k) * L // 1_296_000
        cz.add_channel(480, sh, -1 / 3, 1 / 3, 11.0)
    if in_type == capi.KGPU_REAL:
        x = rng.integers(-3000, 3000, B * L, dtype=np.int16)
    elif name.endswith("i16"):
        x = rng.integers(-3000, 3000, 2 * B * L, dtype=np.int16)
    else:
        x = (rng.standard_normal(B * L) + 1j * rng.standard_normal(B * L)).astype(np.complex64)
    d = cz.stage_stream(x)
    ref = cz.alloc_spectra(B); oref = cz.alloc_outputs(B); setv("default")
    cz.forward(d, B, ref, scale=W.scale); cz.channels(ref, B, oref); torch.cuda.synchronize()
    print(name, cz.master.describe())
    for v in sys.argv[1:]:
        out = cz.alloc_spectra(B); out.zero_(); oo = cz.alloc_outputs(B); oo.zero_(); setv(v)
        cz.forward(d, B, out, scale=W.scale); cz.channels(out, B, oo); torch.cuda.synchronize()
        nb = cz.master.bins
        diff = (out[:, :nb] - ref[:, :nb]).abs().max().item(); mag = ref[:, :nb].abs().max().item()
        od = (oo - oref).abs().max().item(); om = oref.abs().max().item()
        print("  variant %-10s spectrum max|diff| %.3e rel %.3e | channels max|diff| %.3e rel %.3e  %s"
              % (v, diff, diff / mag, od, od / om, "OK" if diff / mag < 1e-6 and od / om < 1e-6 else "MISMATCH"))
    setv("default"); cz.close()
