"""Masters whose transform length has prime factors 11, 13, 17, 19 or 23 (kgpu_master_create_ex), and the split and
radices the extended planner gives each.  Shared by tests/test_extended_primes_cpu.py, which pins the plans without a
GPU, and tests/test_gpu_extended_primes.py, which checks every geometry bin by bin on the device."""
from typing import NamedTuple

NEW_PRIMES = (11, 13, 17, 19, 23)


class Ext(NamedTuple):
    id: str
    real: bool
    L: int
    M: int
    split: tuple   # (n1, n2)
    plan: tuple    # (column radices, row radices), kgpu_plan_radices_ex order
    why: str


EXT_FORWARD = [
    Ext("airspyhf_912k", False, 18240, 4561, (152, 150), ([8, 19], [10, 15]), "AirspyHF+ 912 kS/s, 20 ms at overlap 5"),
    Ext("airspyhf_456k", False, 9120, 2281, (114, 100), ([6, 19], [10, 10]), "AirspyHF+ 456 kS/s"),
    Ext("rx888_60m8", True, 1216000, 304001, (950, 800), ([10, 19, 5], [10, 10, 8]), "RX888 at 60.8 MS/s, REAL"),
    Ext("c143x140", False, 16016, 4005, (143, 140), ([13, 11], [20, 7]), "11 and 13 in the column plan"),
    Ext("c144x143", False, 16474, 4119, (144, 143), ([12, 12], [13, 11]), "11 and 13 in the row plan"),
    Ext("r153x135", True, 33048, 8263, (153, 135), ([17, 9], [15, 9]), "17 in the columns, REAL with odd n1 and n2"),
    Ext("c150x136", False, 16320, 4081, (150, 136), ([10, 15], [8, 17]), "17 in the row plan"),
    Ext("r161x125", True, 32200, 8051, (161, 125), ([23, 7], [25, 5]), "23 in the columns, REAL with odd n1 and n2"),
    Ext("c147x138", False, 16230, 4057, (147, 138), ([7, 7, 3], [6, 23]), "23 in the row plan"),
    Ext("r152x138", True, 33562, 8391, (152, 138), ([8, 19], [6, 23]), "new primes in both factors, REAL"),
    Ext("c3520x2645", False, 7448320, 1862081, (3520, 2645), ([20, 16, 11], [23, 23, 5]),
        "3520: the largest column length with a new prime the generic pair fits (3536 does not)"),
]

# 3536 x 2312 = 2^4 13 17 x 2^3 17^2: plannable, but 3536 points do not fit the column kernel's shared memory
TOO_BIG_FOR_SMEM = (8175232, (3536, 2312))

# every sample rate the AirspyHF+ lists, 20 ms blocks at overlap 5 (radio.c:582-587): (rate, L, M)
AIRSPYHF_RATES = [(r, r // 50, r // 200 + 1) for r in (912000, 768000, 456000, 384000, 256000, 192000)]
