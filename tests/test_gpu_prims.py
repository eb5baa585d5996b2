"""Device-wide primitives (stable LSD radix sort, multi-counter scan) against numpy, at sizes around every tile boundary."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes

pytestmark = pytest.mark.gpu


def test_scan_and_sort_match_numpy():
    g = nudge_b200.Sim(scenes.box_drop(70000))
    rng = np.random.default_rng(1)
    for n in [0, 1, 255, 256, 257, 1000, 8192, 8193, 16384, 16385, 40000, 151552, 151553, 435499, 1000000, 2200000]:
        if n <= 1000000:
            d = rng.integers(0, 5, n).astype(np.uint32)
            out, tot = g.device_scan(d)
            ref = np.concatenate([[0], np.cumsum(d)[:-1]]).astype(np.uint32) if n else d
            assert np.array_equal(out, ref) and tot == int(d.sum())
        for bits in (8, 17, 34, 48, 50, 63, 64):
            for ties in (True, False):   # heavy ties: stability, and one oversized bucket (the LSD fallback); uniform: the bucket path
                keys = rng.integers(0, 1 << bits, n, dtype=np.uint64)
                if ties and n > 10:
                    keys[: n // 3] &= np.uint64(0xff)
                vals = np.arange(n, dtype=np.uint32)
                k2, v2 = g.device_sort(keys, vals, 0, bits)
                order = np.argsort(keys, kind="stable")
                assert np.array_equal(k2, keys[order]) and np.array_equal(v2, vals[order]), (n, bits, ties)
        # keys only, two bit ranges in one call are covered by the sleeping-pair sort of the parity tests
        keys = rng.integers(0, 1 << 40, n, dtype=np.uint64)
        k2, _ = g.device_sort(keys, None, 0, 40)
        assert np.array_equal(k2, np.sort(keys)), n
