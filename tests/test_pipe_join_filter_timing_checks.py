"""The exact check of scripts/pipe_join_filter_timing.py on tiny host data (no GPU): it accepts equal results and rejects a changed sum
or row count; its filter programs have the sizes the stage-filter pool admits."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import pipe_join_filter_timing as T  # noqa: E402


def test_check_accepts_equal_results():
    assert T.check_sum("q19", (123456789, 42), (123456789, 42)) == {"sum": 123456789, "rows": 42}
    assert T.check_sum("q17", (0, 0), (0, 0)) == {"sum": 0, "rows": 0}


def test_check_rejects_differences():
    for bad in ((123456788, 42), (123456789, 41), (0, 0)):
        with pytest.raises(AssertionError):
            T.check_sum("q19", (123456789, 42), bad)


def test_filter_programs_fit_the_stage_filter_pool():
    q19 = T.q19_filter(1, 6, 7, 8)
    assert len(q19) <= 128 and sum(n[0] == T.D.EXPR_COLUMN for n in q19) == 3 * (1 + 4 + 2 + 2)
    assert len(T.q17_filter(1, 3)) == 6
