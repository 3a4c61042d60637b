"""The exact checks of scripts/pipe_left_join_timing.py on tiny host data (no GPU): they accept equal results in any row order and reject
a changed count, a moved count, a missing customer and a changed key set."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import pipe_left_join_timing as T  # noqa: E402


def q13_result(keys, counts):
    vals, dist = np.unique(np.asarray(counts), return_counts=True)
    return np.asarray(keys, np.int64), np.asarray(counts, np.int64), T.histogram(vals, dist)


def test_q13_check_accepts_equal_results_in_any_order():
    keys, counts = np.arange(1, 10, dtype=np.int64), np.array([0, 3, 1, 0, 2, 2, 0, 5, 1], np.int64)
    o = np.random.default_rng(0).permutation(9)
    s = T.check_q13(q13_result(keys, counts), q13_result(keys[o], counts[o]))
    assert s["customers"] == 9 and s["zero_order_customers"] == 3


def test_q13_check_rejects_differences():
    keys, counts = np.arange(1, 10, dtype=np.int64), np.array([0, 3, 1, 0, 2, 2, 0, 5, 1], np.int64)
    ref = q13_result(keys, counts)
    changed = counts.copy(); changed[1] = 4
    swapped = counts.copy(); swapped[[1, 7]] = swapped[[7, 1]]          # same histogram, counts moved between customers
    for bad in (q13_result(keys, changed), q13_result(keys, swapped), q13_result(keys[:-1], counts[:-1])):
        with pytest.raises(AssertionError):
            T.check_q13(ref, bad)
    with pytest.raises(AssertionError):
        T.histogram([1, 1], [2, 3])                                      # a c_count twice


def test_key_check():
    assert T.check_keys("left_semi", (3, 12), (3, 12)) == {"rows": 3, "key_sum": "0xc"}
    for bad in ((2, 12), (3, 13)):
        with pytest.raises(AssertionError):
            T.check_keys("left_anti", (3, 12), bad)
