"""The data of the dense aggregate sink's accumulator tests (tests/test_gpu_pipe_dense_accumulators.py) reaches the edges it was written
for: checked with the Python reference alone, so an edit that loses an edge fails here, also on a machine without a GPU."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import decimal_agg as DA
import dense_cases as C


def test_carry_case_sums_carry_out_of_the_low_word_in_every_group_and_wrap():
    for n in (60_000, 1000):
        cols, _ = C.carry_case(np.random.default_rng(31), n)
        per = C.group_values(cols, 0, 2)
        assert set(per) == set(range(C.CARRY_GROUPS)) | {None}
        for key, xs in per.items():
            assert sum(x % (1 << 64) for x in xs) >= 1 << 64, f"group {key}: no carry out of the low word"
        wrapped = [k for k, xs in per.items() if not -(1 << 127) <= sum(xs) < 1 << 127]
        assert 4 in wrapped and 5 in wrapped, "the sums of groups 4 and 5 must pass +-2^127"
        assert DA._wrap128(sum(per[4])) != sum(per[4])
        assert sum(per[1]) < 0 and all(x < 0 for x in per[7])
        assert {(1 << 63) - 1, 1 << 63} <= set(per[6]) and {-1, -(1 << 64)} <= set(per[7])


@pytest.mark.parametrize("p,s", C.AVG_TYPES)
def test_avg_case_has_negative_sums_with_remainders(p, s):
    cols, _ = C.avg_case(np.random.default_rng(41 + p), p, s)
    per = C.group_values(cols, 0, 1)
    mul = C.avg_mul(p, s)
    neg_rem = [k for k, xs in per.items() if sum(xs) < 0 and (abs(sum(xs)) * 10 ** mul) % len(xs) != 0]
    assert 0 in neg_rem and 3 in neg_rem, f"negative sums with a remainder: {neg_rem}"
    assert len(per[3]) == 7 and all(abs(x) < 10 ** p for xs in per.values() for x in xs)
    for xs in per.values():      # inside i128 and inside the target precision: no group raises
        DA.decimal_avg(sum(xs), len(xs), p, s)
    assert DA.decimal_avg(-7, 2, p, s)[0] == -(7 * 10 ** mul // 2)   # truncation toward zero, not floor


def test_word_layout_puts_the_threshold_shapes_on_both_sides_of_48k():
    one_sum = [(D.AGG_SUM, False)]
    assert C.slot_words(one_sum) == 4
    assert C.WARPS * 192 * 4 * 8 == 48 * 1024 and C.per_warp(192, one_sum) and not C.per_warp(193, one_sum)
    eight_dec = [(f, True) for f in (D.AGG_SUM, D.AGG_MIN, D.AGG_MAX, D.AGG_AVG) * 2]
    assert C.slot_words(eight_dec) == 34 and 256 * 34 * 8 == 68 * 1024
    # a Decimal128 field after an odd number of one-word fields is padded to an even word
    assert C.slot_words([(D.AGG_COUNT, False), (D.AGG_COUNT, False), (D.AGG_MIN, True)]) == 8   # 0 rows, 1-2 counts, 3 pad, 4-5, 6, 7 pad


def test_reference_agrees_with_the_oracle_on_integer_and_decimal_aggregates():
    rng = np.random.default_rng(51)
    n = 3000
    key = (rng.integers(-2, 3, n).astype(np.int16), rng.random(n) > 0.1)
    i64 = (rng.integers(C.I64_MIN, C.I64_MAX, n, endpoint=True), rng.random(n) > 0.1)
    dec = (O.Dec([int(x) << 40 for x in rng.integers(-(1 << 60), 1 << 60, n)], 38, 4), rng.random(n) > 0.1)
    cols, types = [key, i64, dec], [D.INT16, D.INT64, D.decimal128(38, 4)]
    aggs = [(D.AGG_SUM, 1), (D.AGG_MIN, 1), (D.AGG_MAX, 1), (D.AGG_COUNT, 1), (D.AGG_SUM, 2), (D.AGG_MIN, 2), (D.AGG_AVG, 2),
            (D.AGG_COUNT_STAR, None)]
    from test_gpu_pipe_dense import col, oracle_dense
    want = oracle_dense(cols, None, [0], [(f, None if c is None else [col(c)]) for f, c in aggs])
    C.check_rows(C.reference(cols, types, None, [0], [(-2, 2)], aggs), want, "reference vs oracle")
