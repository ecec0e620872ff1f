"""The plans of channels whose length has a prime factor 11, 13, 17, 19 or 23 (kgpu_bank_define_ext), without a GPU:
every such length up to 7260 points plans directly, and every longer one up to 28812 splits into two plannable factors
whose chan_wide_ext footprint fits the 227 KB of shared memory a block may opt into."""
from ka9q_radio_b200 import capi

MAX_CHAN, MAX_WIDE, SMEM = 7260, 28812, 227 * 1024
PRIMES = (2, 3, 5, 7, 11, 13, 17, 19, 23)


def _rest(n, primes):
    for p in primes:
        while n % p == 0:
            n //= p
    return n


def _extended(n):
    return _rest(n, PRIMES) == 1 and _rest(n, PRIMES[:4]) != 1


def _product(r):
    out = 1
    for x in r:
        out *= x
    return out


def test_every_extended_length_plans():
    small = [n for n in range(2, MAX_CHAN + 1) if _extended(n)]
    wide = [n for n in range(MAX_CHAN + 1, MAX_WIDE + 1) if _extended(n)]
    assert len(small) == 863 and len(wide) == 1032 and MAX_CHAN in small and wide[-1] == 28798
    for n in small:
        r = capi.plan_radices(n, extended=True)
        assert _product(r) == n and len(r) <= 8, (n, r)
    for n in wide:
        n1, n2 = capi.plan_split(n, extended=True)
        assert n1 * n2 == n and n1 <= 4096 and n2 <= 4096, (n, n1, n2)
        for f in (n1, n2):
            assert _product(capi.plan_radices(f, extended=True)) == f, (n, f)
        assert 8 * n1 * (n2 | 1) <= SMEM, (n, n1, n2)
