#!/usr/bin/env python3
"""Rounding floor of quiet cfg-2 channels against a float64 transform: GPU kernel variants and the float32 CPU checker.
usage: diag_floor.py [default] [static=0]   (variants as in kbench.py; test/diagnostic tool, not product code)"""
import sys
from pathlib import Path
import numpy as np, torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from ka9q_radio_b200 import workloads, capi
from ka9q_radio_b200.channelizer import Channelizer
from oracle import oracle
lib = capi.load(); dev = torch.device("cuda:0")
w = workloads.cfg2()
quiet = [9, 100, 500, 777, 1000, 33, 250, 640, 900]
w.channels = [w.channels[i] for i in quiet]
xi = w.stream(2)
xf = oracle.convert_i16(xi, np.float32(w.scale))[0]
win = oracle.block_window(xf, w.L, w.M, 1)
X32 = oracle.forward(win)
X64 = oracle.forward_real_f64(win.astype(np.float64))
R = oracle.design_response(600, 480, w.N, True, w.channels[0].low, w.channels[0].high, 11.0)
k = np.arange(-300, 300)
truth, r32 = [], []
for c in w.channels:
    S = np.zeros(600, np.complex128)
    S[k % 600] = X64[c.shift + k] * R[k % 600].astype(np.complex128)
    S[300] = 0
    truth.append((np.fft.ifft(S) * 600)[-480:])
    r32.append(oracle.channel_block(oracle.KO_REAL, X32, R, c.shift)[-480:])
truth, r32 = np.array(truth), np.array(r32)
e = r32 - truth
print("float32 CPU checker : max %.3e rms %.3e" % (np.abs(e).max(), np.sqrt((np.abs(e) ** 2).mean())))
se = np.abs(X32[:w.N // 2 + 1] - X64[:w.N // 2 + 1])
print("   spectrum: max %.3e rms %.3e (max|X| %.3e)" % (se.max(), np.sqrt((se ** 2).mean()), np.abs(X64).max()))
for v in sys.argv[1:] or ["default"]:
    if v not in ("default", "static=0"): sys.exit("variants: default, static=0")
    lib.kgpu_use_static_kernels(0 if v == "static=0" else 1)
    cz = Channelizer(w.L, w.M, w.in_type, dev, capacity=len(w.channels))
    for c in w.channels:
        cz.add_channel(c.olen, c.shift, c.low, c.high, c.beta)
    spec, out = cz.alloc_spectra(2), cz.alloc_outputs(2)
    cz.forward(cz.stage_stream(xi), 2, spec, scale=w.scale)
    cz.channels(spec, 2, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy(); sp = spec.cpu().numpy()[1, : w.N // 2 + 1]
    offs = [cz.bank.out_offset(i) for i in range(len(w.channels))]
    g = np.array([got[1, o: o + 480] for o in offs])
    cz.close()
    e = g - truth
    se = np.abs(sp - X64[: w.N // 2 + 1])
    print("%-20s: max %.3e rms %.3e | spectrum max %.3e rms %.3e" % (v, np.abs(e).max(), np.sqrt((np.abs(e) ** 2).mean()), se.max(), np.sqrt((se ** 2).mean())))
