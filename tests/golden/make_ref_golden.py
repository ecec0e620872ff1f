#!/usr/bin/env python3
"""Generate tests/golden/ref_checks.npz and tests/golden/filter_h_layout.txt: what the reference's own code computes in
the comparisons of tests/test_oracle_cpu.py, tests/test_oracle_ext_cpu.py and tests/test_filter_abi.py, captured once so
that those tests run from the repository alone.

Needs oracle/_ref/ (the reference's filter.c and radio.c compiled unmodified by oracle/Makefile) and
oracle/_ref/driver_refhdr.so (the filter.h driver compiled against the reference's own header):
    python -c "import __graft_entry__ as g; g.build()"   # with the reference sources present
    python tests/golden/make_ref_golden.py
Long outputs are stored at a fixed stride (the `*_stride` entries) to keep the fixture small; the inputs are regenerated
from the seeds and parameters the tests name.
"""
import ctypes as C
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from oracle import oracle as O  # noqa: E402

OUT = Path(__file__).resolve().parent

OSC_CASES = [(0.0123, 0.0), (-0.25, 0.0), (1e-3, 1e-9), (0.0, 0.0)]
OSC_N, OSC_STRIDE = 40000, 257
BB_STRIDE = 16     # channel outputs and responses
SPEC_STRIDE = 61   # master spectra


def osc(d):
    for j, (f, r) in enumerate(OSC_CASES):
        ref = np.empty(OSC_N, np.complex128)
        O.radio_lib().rr_osc_run(f, r, OSC_N, ref.ctypes.data)
        d[f"osc{j}"] = ref[::OSC_STRIDE]
    d["osc_stride"] = OSC_STRIDE


def restatement(d):
    L, M = 4800, 1201
    x = O.ref_siggen_real(5 * L, 0.2, 0.05, 0.3123, 1.0)
    chans = [dict(olen=48, shift=s, low=-0.3, high=0.4, beta=9.0) for s in (1874, -1874, 0, 2999, -3005, 2990, 12)]
    chans.append(dict(olen=96, shift=1870, low=-0.2, high=0.2, beta=4.0, isb=True))
    o2, s2 = O.ref_run_stream(x, L, M, chans, notch_bins=[5], keep_spectra=True)
    d["rs_x_sample"], d["rs_x_sum"] = x[::BB_STRIDE].copy(), np.array([np.sum(x.astype(np.float64))])
    d["rs_spec"] = np.stack([s[::SPEC_STRIDE] for s in s2])
    d["rs_spec_absmax"] = np.array([np.abs(s).max() for s in s2])
    for c in range(len(chans)):
        d[f"rs_out{c}"] = np.stack([o2[b][c][::BB_STRIDE] for b in range(5)])
        d[f"rs_out_absmax{c}"] = np.array([np.abs(o2[b][c]).max() for b in range(5)])


def slice_sweep(d):
    """The reference's slicing as an index map: entry k of the frequency-domain slice for a shift is
    X[code - 1] * R[k] (code < 0: conjugate of bin -code - 1, code 0: zero).  Each entry is checked here to be such a
    product."""
    for tag, in_type, L, M in (("r", O.KO_REAL, 480, 121), ("c", O.KO_COMPLEX, 480, 121)):
        N = L + M - 1
        rng = np.random.default_rng(7)
        x = (rng.standard_normal(L) + (1j * rng.standard_normal(L) if in_type == O.KO_COMPLEX else 0))
        x = x.astype(np.complex64 if in_type == O.KO_COMPLEX else np.float32)
        with O.RefSession(L, M, in_type) as s:
            ids = [s.add_channel(olen, -0.3, 0.3, 8.0) for olen in (48, 24, 40)]
            s.write(x)
            X = s.spectrum()
            d[f"sw_{tag}_X"] = X
            lim = N // 2 if in_type == O.KO_COMPLEX else N
            for k, i in enumerate(ids):
                R = s.response(i)
                d[f"sw_{tag}_R{k}"] = R
                codes = []
                for shift in range(-lim + 1, lim):
                    _, fd = s.execute(i, shift, want_fdomain=True)
                    codes.append(_encode(X, R, fd))
                d[f"sw_{tag}_code{k}"] = np.stack(codes)


def _encode(X, R, fd):
    code = np.zeros(len(fd), np.int16)
    cand = np.concatenate([X, np.conj(X)])
    for k in range(len(fd)):
        if fd[k] == 0:
            continue
        prod = cand.astype(np.complex128) * complex(R[k])
        j = int(np.argmin(np.abs(prod - fd[k])))
        assert abs(prod[j] - fd[k]) <= 1e-6 * abs(fd[k]), "slice entry is not a bin times the response"
        code[k] = (j + 1) if j < len(X) else -(j - len(X) + 1)
    return code


def downconvert(d):
    cases = {
        "dr": (O.KO_REAL, 4800, 1201, 240e3, 0.0,
               [(480, 24000.0, -1 / 3, 1 / 3, 11.0), (240, 12000.0, 50 / 12000, 3000 / 12000, 11.0), (960, 48000.0, -0.4, 0.4, 7.0)], 9),
        "dc": (O.KO_COMPLEX, 4000, 1001, 200e3, 10.0e6, [(480, 24000.0, -1 / 3, 1 / 3, 11.0), (480, 24000.0, -0.3, 0.2, 9.0)], 7),
    }
    import test_oracle_ext_cpu as T
    for tag, (in_type, L, M, fs, fe, chans, nb) in cases.items():
        plan = T.downconvert_plan(tag, nb)
        x = (O.siggen_real if in_type == O.KO_REAL else O.siggen_complex)(nb * L, 0.1, 0.02, 0.1234, 1.0)
        spec, bb = [], {i: [] for i in range(len(chans))}
        scal = np.zeros((nb, len(chans), 4))   # shift, remainder, bb_power, n0
        with O.RadioRef(L, M, in_type, fs, fe) as rr:
            ids = [rr.add_channel(c[0], c[1], plan[0][i], c[2], c[3], c[4]) for i, c in enumerate(chans)]
            for b in range(nb):
                assert rr.write(x[b * L:(b + 1) * L]) == 1
                sp = rr.spectrum()
                spec.append(sp)
                for i in range(len(chans)):
                    rr.set_freq(ids[i], plan[b][i])
                    r = rr.downconvert(ids[i])
                    bb[i].append(r["baseband"][::BB_STRIDE])
                    scal[b, i] = (r["shift"], r["remainder"], r["bb_power"], r["n0"])
        d[f"{tag}_spec"] = np.stack([s[::SPEC_STRIDE] for s in spec])
        d[f"{tag}_spec_absmax"] = np.array([np.abs(s).max() for s in spec])
        d[f"{tag}_scalars"] = scal
        for i in range(len(chans)):
            d[f"{tag}_bb{i}"] = np.stack(bb[i])


def realout(d):
    import test_oracle_ext_cpu as T
    for in_type in ("real", "complex"):
        it = O.KO_REAL if in_type == "real" else O.KO_COMPLEX
        L, M, nb = 4800, 1201, 3
        x = (O.siggen_real if it == O.KO_REAL else O.siggen_complex)(nb * L, 0.1, 0.02, 0.0123, 1.0)
        with O.RefSession(L, M, it) as s:
            ids = [s.add_channel(c[0], c[1], c[2], c[3], out_type=O.KO_REAL) for c in T.REALOUT_CASES]
            full = {i: [] for i in ids}
            for b in range(nb):
                assert s.write(x[b * L:(b + 1) * L]) == 1
                for i, c in zip(ids, T.REALOUT_CASES):
                    dst, f = T._ref_exec(O, s, i, c[4], c[0], True)
                    assert np.array_equal(f[-c[0]:], dst)
                    full[i].append(f[::BB_STRIDE])
            for k, (i, c) in enumerate(zip(ids, T.REALOUT_CASES)):
                pts = c[0] * (L + M - 1) // L
                d[f"ro_{in_type}_R{k}"] = s.response(i)[: pts // 2 + 1][::BB_STRIDE]
                d[f"ro_{in_type}_out{k}"] = np.stack(full[i])


def beam(d):
    import test_oracle_ext_cpu as T
    L, M, nb = 4000, 1001, 3
    x = O.siggen_complex(nb * L, 0.1, 0.02, 0.0123, 1.0)
    with O.RefSession(L, M, O.KO_COMPLEX) as s:
        s.R.ref_set_beam.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_double] * 4
        ids = [s.add_channel(c[0], -0.3, 0.35, 11.0) for c in T.BEAM_CASES]
        for i, c in zip(ids, T.BEAM_CASES):
            s.R.ref_set_beam(s.h, i, 1, complex(c[2]).real, complex(c[2]).imag, complex(c[3]).real, complex(c[3]).imag)
        outs = {i: [] for i in ids}
        for b in range(nb):
            assert s.write(x[b * L:(b + 1) * L]) == 1
            for i, c in zip(ids, T.BEAM_CASES):
                dst, _ = T._ref_exec(O, s, i, c[1], c[0], False)
                outs[i].append(dst[::BB_STRIDE])
        for k, i in enumerate(ids):
            d[f"beam_out{k}"] = np.stack(outs[i])


def layout():
    import test_filter_abi as T
    ref = T._load("driver_refhdr.so")
    if ref is None:
        raise SystemExit("oracle/_ref/driver_refhdr.so not built (needs the reference's src/filter.h)")
    (OUT / "filter_h_layout.txt").write_text(T._report(ref) + "\n")


def main():
    d = {"bb_stride": BB_STRIDE, "spec_stride": SPEC_STRIDE}
    for f in (osc, restatement, slice_sweep, downconvert, realout, beam):
        f(d)
    np.savez_compressed(OUT / "ref_checks.npz", **d)
    layout()
    print("ref_checks.npz:", (OUT / "ref_checks.npz").stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
