"""The exact checks of scripts/pipe_full_join_timing.py on tiny host data (no GPU): they accept equal results in any row order and reject
a changed aggregate, a missing or extra group, a moved NULL group and a changed output summary (the NULL count of o_orderkey included:
the customers no order matched)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import pipe_full_join_timing as T  # noqa: E402


def groups(order, count=(4, 2, 7), sums=(10, -3, 2**70), nat=(3, None, 0)):
    """(nation with a NULL group, count, Decimal128 sum as words, max) in the given row order"""
    s = np.array([[v % (1 << 64), (v >> 64) % (1 << 64)] for v in sums], np.uint64)
    cols = [(np.array([0 if x is None else x for x in nat], np.int32), np.array([x is not None for x in nat])),
            (np.array(count, np.int64), None), (s, None), (np.array([5, 0, 9], np.int32), np.array([True, False, True]))]
    return T.group_rows([(v[order], None if m is None else m[order]) for v, m in cols], 1)


def test_group_check_accepts_equal_results_in_any_order():
    s = T.check_groups("a", groups([0, 1, 2]), groups([2, 0, 1]))
    assert s == {"groups": 3, "rows": 13, "null_nation_rows": 2}
    assert groups([0, 1, 2])[(None,)] == (2, -3, None)   # Decimal128 words back to a signed value, NULL max


def test_group_check_rejects_differences():
    ref = groups([0, 1, 2])
    for bad in (groups([0, 1, 2], count=(4, 3, 7)), groups([0, 1, 2], sums=(10, -3, 2**70 + 1)), groups([0, 1, 2], nat=(3, 1, 0)),
                {k: v for k, v in ref.items() if k != (0,)}):
        with pytest.raises(AssertionError):
            T.check_groups("a", ref, bad)
    with pytest.raises(AssertionError):
        T.group_rows([(np.array([1, 1]), None), (np.array([2, 3]), None)], 1)   # a group twice


def test_output_check():
    ref = T.output_summary(5, 2**64 + 7, 1, 2, 40)
    assert T.check_output(ref, T.output_summary(5, 7, 1, 2, 40)) == {"rows": 5, "key_sum": "0x7", "key_nulls": 1, "nation_nulls": 2, "nation_sum": 40}
    for bad in (T.output_summary(4, 7, 1, 2, 40), T.output_summary(5, 8, 1, 2, 40), T.output_summary(5, 7, 0, 2, 40), T.output_summary(5, 7, 1, 1, 40),
                T.output_summary(5, 7, 1, 2, 41)):
        with pytest.raises(AssertionError):
            T.check_output(ref, bad)
