"""The work schedule of fwd_fused_r36_v2, the one-launch forward pass of REAL 1296 x 1250 masters, checked on the host
(kgpu_fused_schedule and kgpu_fused_discards run the device's own ticket map and line arithmetic; no device needed).

The kernel's CTAs take tickets in the order they become resident, so it cannot wait forever if every item waits only on
items with smaller tickets.  For every launch of 1 to 64 blocks and a range of leads: every ticket maps to one item,
every item appears exactly once, a row item R(b, *) waits for exactly the column items C(b, *), and all of those have
smaller tickets.  The lines a row item discards from L2 are exactly the 128-byte lines of its own inter-pass rows, and
the row items of a block together discard each line of that block's rows exactly once.
Also where the fused launch is chosen: REAL 1296 x 1250 masters with an input the tensor copies take, nothing else.
"""
import ctypes as C

import numpy as np
import pytest

from ka9q_radio_b200 import capi

I16, F32 = capi.KGPU_FMT_I16, capi.KGPU_FMT_F32
REAL, CPLX = capi.KGPU_REAL, capi.KGPU_COMPLEX
BASE = 0x7F0000000000


def _shape():
    out = (C.c_int * 5)()
    assert capi.load().kgpu_fused_shape(C.cast(out, C.c_void_p)) == 0
    return list(out)


def test_shape():
    nc, nr, n1, ld, lead = _shape()
    assert (nc, nr, n1, ld) == (79, 82, 1296, 1264)  # 157 column tiles in pairs, 649 row items in eights
    assert 0 <= lead <= nc


def _schedule(nb, lead):
    lib = capi.load()
    out = (C.c_int * 5)()
    nc, nr = _shape()[:2]
    items = []
    for t in range(nb * (nc + nr)):
        assert lib.kgpu_fused_schedule(nb, lead, t, C.cast(out, C.c_void_p)) == 0
        items.append(tuple(out))
    assert lib.kgpu_fused_schedule(nb, lead, nb * (nc + nr), C.cast(out, C.c_void_p)) != 0
    return items


@pytest.mark.parametrize("lead", [0, 1, 40, 78, 79, None])
def test_every_wait_is_on_smaller_tickets(lead):
    nc, nr, _, _, default_lead = _shape()
    lead = default_lead if lead is None else lead
    for nb in range(1, 65):
        items = _schedule(nb, lead)
        keys = [(k, b, i) for k, b, i, _, _ in items]
        want = {(0, b, i) for b in range(nb) for i in range(nc)} | {(1, b, i) for b in range(nb) for i in range(nr)}
        assert len(keys) == len(set(keys)) and set(keys) == want, f"B={nb} lead={lead}: not every item exactly once"
        ticket = {k: t for t, k in enumerate(keys)}
        for t, (kind, b, i, wb, wcount) in enumerate(items):
            if kind == 0:
                assert (wb, wcount) == (-1, 0), f"B={nb}: column item {b},{i} waits"
                continue
            assert (wb, wcount) == (b, nc), f"B={nb}: R({b},{i}) waits for {wcount} items of block {wb}"
            last = max(ticket[(0, b, x)] for x in range(nc))
            assert last < t, f"B={nb} lead={lead}: R({b},{i}) at ticket {t} waits for ticket {last}"


def test_discards_are_the_items_rows():
    lib = capi.load()
    nc, nr, n1, ld, _ = _shape()
    per_row = ld * 8 // 128
    assert ld * 8 % 128 == 0 and per_row == 79
    buf = (C.c_long * (16 * per_row + 1))()
    for blk in (0, 1, 31):
        seen = np.zeros(n1 * per_row, dtype=np.int64)
        for idx in range(nr):
            n = lib.kgpu_fused_discards(blk, idx, C.cast(buf, C.c_void_p), len(buf))
            lines = np.array(buf[:n], dtype=np.int64)
            # the item's rows: pairs (k, n1 - k), row 0 and row n1/2 paired with themselves
            rows = set()
            for p in range(8 * idx, 8 * idx + 8):
                if p == 0 or 2 * p == n1:
                    rows.add(p)
                elif 2 * p < n1:
                    rows |= {p, n1 - p}
            want = sorted(((blk * n1 + r) * per_row + l) for r in rows for l in range(per_row))
            assert sorted(lines.tolist()) == want, f"R({blk},{idx})"
            seen[lines - blk * n1 * per_row] += 1
        assert (seen == 1).all(), f"block {blk}: lines discarded {seen.min()} .. {seen.max()} times"


@pytest.mark.parametrize("L,M,in_type,fmt,offset,want", [
    (2592000, 648001, REAL, I16, 0, 1),    # cfg-2, 1296 x 1250
    (2592000, 648001, REAL, F32, 0, 1),
    (2592000, 648001, REAL, F32, 16, 1),
    (2592000, 648001, REAL, I16, 4, 0),    # no tensor map for the column pass: the pair
    (2592000, 648001, REAL, I16, 8, 0),
    (2592000, 648001, REAL, F32, 8, 0),
    (1296000, 324001, CPLX, I16, 0, 0),    # COMPLEX 1296 x 1250
    (2654208, 663553, REAL, I16, 0, 0),    # 1296 x 1280: no fwd_rows_v2
    (2560000, 640001, REAL, I16, 0, 0),    # 1280 x 1250: no fwd_cols_r36
    (48000, 12001, REAL, I16, 0, 0),       # cfg-1
])
def test_fused_forward_fits(L, M, in_type, fmt, offset, want):
    assert capi.load().kgpu_fused_forward_fits(L, M, in_type, fmt, BASE + offset) == want


def test_options_reject_bad_lead():
    lib = capi.load()
    nc, _, _, _, lead = _shape()
    assert lib.kgpu_fused_forward_options(nc + 1, 1) != 0
    assert lib.kgpu_fused_forward_options(-1, 1) != 0
    assert lib.kgpu_fused_forward_options(lead, 0) == 0
