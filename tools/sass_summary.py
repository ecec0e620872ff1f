#!/usr/bin/env python3
"""Static SASS evidence for the default kernels of libka9qgpu.so: opcode mix and the Hopper-specific mnemonics
(UBLKCP = cp.async.bulk / TMA, SYNCS = mbarrier, LDS.128).  No GPU needed."""
import collections, re, subprocess, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
so = ROOT / "ka9q_radio_b200" / "libka9qgpu.so"
names = subprocess.run(["cuobjdump", "-elf", str(so)], capture_output=True, text=True).stdout
want = {"fwd_cols_r36<int16, 1250> (column pass, default)": r"_ZN4kfft12fwd_cols_r36ILi1ELi1250ELb1EE\w+",
        "fwd_rows_r50<1296, halved> (row pass 50 x 25 + real split, tuning 10=5)": r"_ZN4kfft12fwd_rows_r50ILi1296ELb1EE\w+",
        "fwd_rows_v2<real, 1296, halved> (row pass 10 x 25 x 5, default)": r"_ZN4kfft11fwd_rows_v2ILb1ELi1296ELb1ELb0ELi0ELb1ELb0EE\w+",
        "fwd_cols_2s<int16, 25, 32> (cfg-4 column pass)": r"_ZN4kfft11fwd_cols_2sILi1ELi25ELi32EE\w+",
        "fwd_rows_2s<25, 25> (cfg-4 row pass)": r"_ZN4kfft11fwd_rows_2sILi25ELi25EE\w+",
        "chan_v2<600 = 24 x 25> (channels, default)": r"_ZN4kfft7chan_v2INS_5SPlanILi600EJLi24ELi25EEEELb0ELb0EE\w+"}
for title, pat in want.items():
    m = re.search(pat, names)
    if not m:
        print("=====", title, ": symbol not found"); continue
    sym = m.group(0)
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", sym, str(so)], capture_output=True, text=True).stdout
    ops = collections.Counter(); full = collections.Counter()
    for line in sass.splitlines():
        mm = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if mm:
            full[mm.group(2)] += 1
            ops[mm.group(2).split(".")[0]] += 1
    print("=====", title)
    print("  symbol", sym)
    print("  instructions", sum(ops.values()))
    print("  opcode mix", ", ".join(f"{k} {v}" for k, v in ops.most_common(18)))
    ev = {k: v for k, v in full.items() if k.startswith(("UBLKCP", "SYNCS", "LDS.128", "LDS.64", "STS.64", "LDG", "STG", "UTMA", "I2FP"))}
    print("  evidence", ", ".join(f"{k} {v}" for k, v in sorted(ev.items())))
