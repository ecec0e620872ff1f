"""Restatements of the float front-end drivers' sample loops, for the float ingest tests.

Stores, per component:
  F32, CF32, CF32_CNRMF  (float)(scale * (double)x), a double product rounded to float: hydrasdr.c:724 (FLOAT32_REAL),
                         :753-754 (FLOAT32_IQ), airspyhf.c:315-317
  CF32_FSCALE            x * (float)scale, a float product: fobos.c:419

Energy terms, each as the loop's source computes it before adding it to its sum (the reference's -ffp-contract=fast
build contracts airspyhf.c's cnrmf into a fused multiply-add; the device, and this restatement, round both products):
  F32, CF32_FSCALE       x * x in float, per component (hydrasdr.c:725, fobos.c:418)
  CF32                   cnrm: re^2 + im^2 in double, per pair (hydrasdr.c:755)
  CF32_CNRMF             cnrmf: re^2 + im^2 in float, per pair (airspyhf.c:316)

The loops add their terms in an order their compiler chooses (-funsafe-math-optimizations vectorizes the sums), and
fobos.c adds in float.  The device adds a block's terms in double in the fixed order of float_energy_kernel
(raw_ingest.cuh), which block_energy restates exactly.  A NaN or Inf sample, or a float term past FLT_MAX, makes the sum
non-finite; each loop then leaves if_power alone (its isfinite guard).
"""
import numpy as np

F32, CF32, CF32_CNRMF, CF32_FSCALE = 9, 10, 11, 12    # enum filter_raw_format
COMPLEX_FORMATS = (CF32, CF32_CNRMF, CF32_FSCALE)
ENERGY_CLUSTER, ENERGY_THREADS = 8, 1024              # float_energy_kernel's lanes


def store(x: np.ndarray, fmt: int, scale: float) -> np.ndarray:
    """the floats the driver's loop stores for the float components x (I/Q interleaved)"""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        if fmt == CF32_FSCALE:
            return x * np.float32(scale)
        return (np.float64(scale) * x.astype(np.float64)).astype(np.float32)


def terms(x: np.ndarray, fmt: int) -> np.ndarray:
    """the loop's energy terms of the float components x (I/Q interleaved), as float64"""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        if fmt in (F32, CF32_FSCALE):
            return (x * x).astype(np.float64)
        p = x.reshape(-1, 2)
        if fmt == CF32_CNRMF:
            return (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]).astype(np.float64)
        d = p.astype(np.float64)
        return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]


def block_energy(t: np.ndarray) -> float:
    """float_energy_kernel's sum of one block's terms t: lane j adds terms j, j + K, j + 2K, ... (K = 8192 lanes) in turn,
    each CTA of 1024 lanes halves its sums pairwise, and the eight CTA sums are added in rank order"""
    lanes = ENERGY_CLUSTER * ENERGY_THREADS
    acc = np.zeros(lanes)
    with np.errstate(invalid="ignore"):
        for r in range(0, len(t), lanes):
            row = t[r:r + lanes]
            acc[:len(row)] += row
        red = acc.reshape(ENERGY_CLUSTER, ENERGY_THREADS)
        h = ENERGY_THREADS // 2
        while h:
            red[:, :h] += red[:, h:2 * h]
            h //= 2
        e = 0.0
        for r in range(ENERGY_CLUSTER):
            e += red[r, 0]
    return float(e)


def block_energies(x: np.ndarray, fmt: int, L: int) -> list:
    """block_energy of every whole block of L samples (I/Q pairs for the complex formats) of the float stream x"""
    c = 2 if fmt in COMPLEX_FORMATS else 1
    return [block_energy(terms(x[b * c * L:(b + 1) * c * L], fmt)) for b in range(len(x) // (c * L))]


def transfer_energy(x: np.ndarray, fmt: int) -> float:
    """one transfer's energy as the loop would sum its terms in order, in double (fobos.c sums in float; the bound the
    tests state covers that)"""
    with np.errstate(invalid="ignore", over="ignore"):
        return float(np.sum(terms(x, fmt)))
