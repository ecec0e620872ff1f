"""The path kgpu_bank_define_any takes for every channel length (kgpu_chan_plan), without a GPU: kgpu_bank_define_ext's
wherever that serves the length (direct, wide, huge, extended), and a Bluestein transform of a 7-smooth length
P >= 2 points - 1 for the lengths it refuses for their factors."""
import re

import pytest

from ka9q_radio_b200 import capi

MAX_CHAN, MAX_WIDE, MAX_HUGE = 7260, 28812, 1 << 20


def _rest(n, primes):
    for p in primes:
        while n % p == 0:
            n //= p
    return n


def _smooth7(n):
    return _rest(n, (2, 3, 5, 7)) == 1


def _smooth23(n):
    return _rest(n, (2, 3, 5, 7, 11, 13, 17, 19, 23)) == 1


def _bluestein_p(text):
    m = re.match(r"bluestein: (\d+) points, P=(\d+): \2-point complex two-pass (\d+) x (\d+);", text)
    assert m, text
    return int(m.group(1)), int(m.group(2)), int(m.group(3)), int(m.group(4))


def test_every_length_define_ext_serves_keeps_its_path():
    """Every length up to 28812, and every 7-smooth length up to 1048576: the path define_ext runs."""
    ext_small = ext_wide = 0
    for n in range(1, MAX_WIDE + 1):
        if not _smooth23(n):
            continue
        path, text = capi.chan_plan(n)
        if _smooth7(n):
            assert path == (capi.CHAN_DIRECT if n <= MAX_CHAN else capi.CHAN_WIDE), (n, text)
        else:
            assert path == capi.CHAN_EXTENDED, (n, text)
            ext_small += n <= MAX_CHAN
            ext_wide += n > MAX_CHAN
        assert text.split(":")[0] == {0: "direct", 1: "wide", 3: "extended"}[path], text
    assert (ext_small, ext_wide) == (863, 1032)
    huge = [a * b * c * d for a in (2 ** i for i in range(21)) for b in (3 ** i for i in range(13))
            for c in (5 ** i for i in range(9)) for d in (7 ** i for i in range(8))]
    huge = sorted(n for n in huge if MAX_WIDE < n <= MAX_HUGE)
    assert len(huge) == 806
    for n in huge:
        path, text = capi.chan_plan(n)
        assert path == capi.CHAN_HUGE and text.startswith(f"huge: {n} points, four-step"), (n, text)


def _bluestein_lengths():
    """lengths with a prime factor >= 29 (every one up to 3000, then the issue's examples and a spread up to the top), and
    23-smooth lengths above 28812 that are not 7-smooth"""
    small = [n for n in range(29, 3001) if not _smooth23(n)]
    named = [185, 580, 725, 1550, 7919, 15838, 44000, 62000, 1048573, 1048575, 30976, 28798 * 2]
    spread = [n for n in range(MAX_WIDE + 1, MAX_HUGE + 1, 9973) if not _smooth7(n) and (not _smooth23(n) or n > MAX_WIDE)]
    return small + named + spread


def test_refused_lengths_plan_a_bluestein_transform():
    for n in _bluestein_lengths():
        path, text = capi.chan_plan(n)
        assert path == capi.CHAN_BLUESTEIN, (n, text)
        pts, P, n1, n2 = _bluestein_p(text)
        assert pts == n and P >= 2 * n - 1 and _smooth7(P) and n1 * n2 == P, (n, text)
        assert n1 <= 4096 and n2 <= 4096, (n, text)
        # the smallest such P whose split exists: no 7-smooth length in [2n - 1, P) would be a shorter one that splits
        q = next(q for q in range(2 * n - 1, P + 1) if _smooth7(q))
        if q != P:  # a shorter 7-smooth length must fail to split into two factors of at most 4096
            assert not any(q % d == 0 and q // d <= 4096 and d <= 4096 for d in range(1, 4097)), (n, q, P)
        assert text.endswith("around bluestein_chan_in, bluestein_mul_kernel, bluestein_chan_out"), text


def test_issue_examples():
    for n, path in [(185, 4), (725, 4), (1550, 4), (580, 4), (44000, 4), (62000, 4), (5500, 3), (6930, 3), (38400, 2),
                    (9600, 1), (600, 0)]:
        assert capi.chan_plan(n)[0] == path, n
        if n % 2 == 0:
            assert capi.chan_plan(n, capi.KGPU_REAL)[0] == path, n


def test_refusals():
    with pytest.raises(capi.KgpuError, match="kgpu_chan_plan: 1048577-point inverse transform exceeds the 1048576-point maximum"):
        capi.chan_plan(MAX_HUGE + 1)
    assert capi.chan_plan(MAX_HUGE)[0] == capi.CHAN_HUGE
    for n in (725, 6875, 7919):
        with pytest.raises(capi.KgpuError, match=rf"REAL-output slaves need an even number of points \(got {n}\)"):
            capi.chan_plan(n, capi.KGPU_REAL)
    with pytest.raises(capi.KgpuError, match="kgpu_chan_plan: bad arguments"):
        capi.chan_plan(0)


def test_new_symbols_are_exported():
    lib = capi.load()
    for s in ("kgpu_bank_define_any", "kgpu_chan_plan"):
        assert s in capi.exported_symbols() and hasattr(lib, s), s
