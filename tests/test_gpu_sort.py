"""GPU test of the library's own radix sort (csrc/radix_sort.cuh: one kernel per 8-bit pass, decoupled look-back) against
numpy's stable sort, through the test hook shb_test_radix_sort: sizes around the 4096-item tile, many tiles (look-back
chains), skewed digits, one and two bit ranges, with and without a payload, repeated calls (status tags)."""
import numpy as np
import pytest

from support import ctx  # noqa: F401

pytestmark = pytest.mark.gpu


def _sort(ctx, keys, vals, lo, hi):
    from shasta_b200 import capi
    k = np.ascontiguousarray(keys, np.uint64).copy()
    v = None if vals is None else np.ascontiguousarray(vals, np.uint32).copy()
    capi._check(capi.lib().shb_test_radix_sort(ctx._h, k.ctypes.data, None if v is None else v.ctypes.data, len(k),
                                               lo[0], lo[1], hi[0], hi[1]))
    return k, v


def _expected(keys, vals, lo, hi):
    def field(a, b):
        return (keys >> np.uint64(a)) & np.uint64((1 << (b - a)) - 1) if b > a else np.zeros_like(keys)
    sort_key = field(*lo) | (field(*hi) << np.uint64(lo[1] - lo[0]))
    order = np.argsort(sort_key, kind="stable")
    return keys[order], None if vals is None else vals[order]


@pytest.mark.parametrize("n", [0, 1, 31, 4095, 4096, 4097, 70001, 1 << 20, 3_000_017])
def test_sort_matches_stable_numpy_sort(ctx, n):
    rng = np.random.default_rng(n + 1)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    vals = np.arange(n, dtype=np.uint32)
    for lo, hi in (((0, 21), (32, 52)), ((32, 63), (0, 0)), ((0, 13), (0, 0)), ((5, 6), (40, 41))):
        k, v = _sort(ctx, keys, vals, lo, hi)
        ek, ev = _expected(keys, vals, lo, hi)
        assert np.array_equal(k, ek) and np.array_equal(v, ev)
        k2, _ = _sort(ctx, keys, None, lo, hi)
        assert np.array_equal(k2, ek)


def test_skewed_digits_and_long_lookback(ctx):
    # almost all keys share their digits: every tile publishes the same few digits and the look-back walks far
    rng = np.random.default_rng(7)
    n = 2_000_000
    keys = np.full(n, 0x123456789abc, np.uint64)
    idx = rng.integers(0, n, 1000)
    keys[idx] = rng.integers(0, 2**48, 1000, dtype=np.uint64)
    vals = np.arange(n, dtype=np.uint32)
    for _ in range(3):          # repeated: the status tags advance, nothing is cleared in between
        k, v = _sort(ctx, keys, vals, (0, 48), (0, 0))
        ek, ev = _expected(keys, vals, (0, 48), (0, 0))
        assert np.array_equal(k, ek) and np.array_equal(v, ev)


def test_many_sorts_wrap_the_status_tags(ctx):
    rng = np.random.default_rng(9)
    keys = rng.integers(0, 2**40, 50_000, dtype=np.uint64)
    ek, _ = _expected(keys, None, (0, 40), (0, 0))
    for _ in range(40):         # 5 passes each: the 8-bit tag space wraps several times
        k, _ = _sort(ctx, keys, None, (0, 40), (0, 0))
        assert np.array_equal(k, ek)
