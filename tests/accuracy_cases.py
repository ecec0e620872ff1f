"""The geometries tests/test_gpu_accuracy.py checks bin by bin, and the code paths each one is there to reach.

Shared with tests/test_capi_cpu.py, which asserts on a machine without a GPU that the planner still gives every row
the split and radices listed here: if the planner changes, the coverage claims fail there first."""
from typing import NamedTuple


class Fwd(NamedTuple):
    id: str
    real: bool
    L: int
    M: int
    split: tuple          # (n1, n2) of the two-pass transform
    plan: tuple           # generic tile-plan radices (columns, rows), as kgpu_plan_radices gives them
    kernels: tuple        # radices kgpu_master_describe reports for the chosen pair (specialised kernels: their own)
    pair: tuple           # names of the column and row kernels kgpu_master_create chooses
    specialised: bool     # the master's pair is not the generic one: also run with kgpu_use_static_kernels(0)
    why: str


GENERIC_COLS, GENERIC_ROWS = ("fwd_cols_kernel", None), ("fwd_rows_kernel", None)
R36, C2S = ("fwd_cols_r36", [36, 36]), ("fwd_cols_2s", [25, 32])
V2K, R2S = ("fwd_rows_v2", [10, 25, 5]), ("fwd_rows_2s", [25, 25])


def _fwd(id, real, L, M, split, cols, rows, why, kcols=GENERIC_COLS, krows=GENERIC_ROWS):
    """kcols / krows: (kernel name, radices describe() reports, None = the generic plan's) of a specialised kernel"""
    spec = kcols is not GENERIC_COLS or krows is not GENERIC_ROWS
    return Fwd(id, real, L, M, split, (cols, rows), (kcols[1] or cols, krows[1] or rows), (kcols[0], krows[0]), spec, why)


V2 = [10, 25, 5]
FORWARD = [
    # the six specialised pairs
    _fwd("c800x625", False, 400000, 100001, (800, 625), [10, 10, 8], [25, 25], "fwd_cols_2s + fwd_rows_2s (cfg-4)",
         C2S, R2S),
    _fwd("r1296x1250", True, 2592000, 648001, (1296, 1250), [12, 12, 9], V2, "r36<f,1250> with the halved split + v2 (cfg-2)",
         R36, V2K),
    _fwd("c1296x1250", False, 1296000, 324001, (1296, 1250), [12, 12, 9], V2, "r36<f,1250> + v2<false,1296>", R36, V2K),
    _fwd("c1296x1296", False, 1259712, 419905, (1296, 1296), [12, 12, 9], [12, 12, 9], "r36<f,0> + generic rows", R36),
    _fwd("r1280x1250", True, 2560000, 640001, (1280, 1250), [16, 10, 8], V2, "generic cols + v2<true,0> real split",
         GENERIC_COLS, V2K),
    _fwd("c1280x1250", False, 1200000, 400001, (1280, 1250), [16, 10, 8], V2, "generic cols + v2<false,0>", GENERIC_COLS, V2K),
    # fwd_cols_r36<f,0> with n2 != 1250: unpadded inter-pass pitch, partial last tile
    _fwd("r1296x1215", True, 2519424, 629857, (1296, 1215), [12, 12, 9], [15, 9, 9],
         "partial tile of 7, generic rows with the real split and odd n2", R36),
    _fwd("c1296x1215", False, 1259712, 314929, (1296, 1215), [12, 12, 9], [15, 9, 9], "partial tile of 7", R36),
    _fwd("c1296x1134", False, 1102248, 367417, (1296, 1134), [12, 12, 9], [6, 9, 7, 3], "partial tile of 6, radix 3", R36),
    # fwd_rows_v2 with other row counts
    _fwd("r1323x1250", True, 2646000, 661501, (1323, 1250), [9, 7, 7, 3], V2, "odd n1: odd row count of v2<true,0>",
         GENERIC_COLS, V2K),
    _fwd("r1875x1250", True, 3750000, 937501, (1875, 1250), [25, 15, 5], V2, "odd n1, 1875 rows", GENERIC_COLS, V2K),
    _fwd("r1250x1250", True, 2500000, 625001, (1250, 1250), [10, 25, 5], V2, "v2<true,0> with n1 = n2", GENERIC_COLS, V2K),
    _fwd("c1372x1250", False, 1372000, 343001, (1372, 1250), [4, 7, 7, 7], V2, "radix 4 and 7 columns", GENERIC_COLS, V2K),
    # generic REAL epilogue with odd n1 and n2: no kRowSelfMid row, odd kend
    _fwd("r75x45", True, 5400, 1351, (75, 45), [15, 5], [9, 5], "odd n1 and n2"),
    _fwd("r75x25", True, 3000, 751, (75, 25), [15, 5], [25], "odd n1 and n2, one row stage"),
    _fwd("r60x49", True, 4704, 1177, (60, 49), [10, 6], [7, 7], "odd n2, radix 7 rows"),
    # radix 2 and 7
    _fwd("c686x500", False, 274400, 68601, (686, 500), [2, 7, 7, 7], [20, 25], "radix 2 and 7 columns"),
    _fwd("c98x70", False, 5488, 1373, (98, 70), [2, 7, 7], [10, 7], "radix 2 and 7, small"),
    # the front ends radiod drives: 20 ms blocks at overlap 5
    _fwd("rtlsdr_2048k", False, 40960, 10241, (256, 200), [16, 16], [20, 10], "RTL-SDR 2.048 MS/s"),
    _fwd("airspy_r2_20m", True, 400000, 100001, (500, 500), [20, 25], [20, 25], "Airspy R2 20 MS/s"),
    _fwd("airspyhf_768k", False, 15360, 3841, (150, 128), [10, 15], [16, 8], "AirspyHF+ 768 kS/s"),
    _fwd("funcube_192k", False, 3840, 961, (75, 64), [15, 5], [8, 8], "FUNcube 192 kS/s, odd n1"),
    _fwd("rx888_64m8", True, 1296000, 324001, (900, 900), [10, 10, 9], [10, 10, 9], "RX888 64.8 MS/s"),
    _fwd("rx888_32m4", True, 648000, 162001, (648, 625), [8, 9, 9], [25, 25], "RX888 32.4 MS/s"),
    _fwd("bladerf_30m72", False, 614400, 153601, (960, 800), [12, 10, 8], [10, 10, 8], "bladeRF 30.72 MS/s"),
    _fwd("usrp_56m", False, 1120000, 280001, (1250, 1120), [10, 25, 5], [16, 10, 7], "USRP 56 MS/s, radix 7 rows"),
]

# AirspyHF+ at 912 kS/s: N = 22 800 = 2^4 * 3 * 5^2 * 19 has no plannable split
UNSERVABLE = (18240, 4561)


class Chan(NamedTuple):
    id: str
    real: bool            # master input
    L: int
    M: int
    points: list          # COMPLEX-output slaves
    real_out: list        # REAL-output slaves


CHANNELS = [
    Chan("c7_6", False, 6000, 1001, [7, 14, 49, 70, 98, 343, 686, 1029, 1372, 2401], []),
    Chan("c8_7", False, 7000, 1001, [1024, 2048, 4096], []),
    # 4800: a 192 kHz channel of a 129.6 MS/s RX888 at overlap 5 (olen 3840); 7200: near the 7260-point maximum
    Chan("c5_4", False, 4000, 1001, [75, 125, 135, 3125, 300, 600, 1200, 4800, 7200], []),
    Chan("r7_6", True, 6000, 1001, [49, 343, 2401], [14, 98, 686, 1372]),
]

# inverse-transform radices of every channel length above (kgpu_plan_radices)
CHANNEL_RADICES = {
    7: [7], 14: [2, 7], 49: [7, 7], 70: [10, 7], 98: [2, 7, 7], 343: [7, 7, 7], 686: [2, 7, 7, 7], 1029: [7, 7, 7, 3],
    1372: [4, 7, 7, 7], 2401: [7, 7, 7, 7], 1024: [16, 8, 8], 2048: [16, 16, 8], 4096: [16, 16, 16], 75: [15, 5],
    125: [25, 5], 135: [15, 9], 3125: [25, 25, 5], 300: [20, 15], 600: [24, 25], 1200: [12, 10, 10],
    4800: [20, 16, 15], 7200: [24, 20, 15],
}
