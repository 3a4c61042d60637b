"""The tests' restatement of MIN / MAX / AVG over Decimal128 in tests/decimal_agg.py (DataFusion 55: Avg::return_type in
functions-aggregate average.rs, DecimalAverager::avg in functions-aggregate-common utils.rs), pinned by hand-worked vectors: the GPU dense aggregate sink is checked
against it."""
import numpy as np
import pytest

from oracle import oracle as O
import decimal_agg as DA


def avg(vals, p, s, valid=None):
    (v, val), = DA.scalar_aggregate([(O.A_AVG, (O.Dec(vals, p, s), valid), None)])
    return (v.p, v.s), (None if val is not None and not val[0] else int(v[0]))


def test_avg_of_one_two_two_is_one_point_six_six_six_six_six_six():
    # [1.00, 2.00, 2.00] in Decimal128(15,2): sum 500 * 10^(6-2) / 3 = 1666666 (truncated) -> 1.666666 in Decimal128(19,6)
    assert avg([100, 200, 200], 15, 2) == ((19, 6), 1666666)


def test_negative_mirror_truncates_toward_zero():
    assert avg([-100, -200, -200], 15, 2) == ((19, 6), -1666666)
    assert avg([-1, 0, 0], 10, 0) == ((14, 4), -3333)      # -10000 / 3 = -3333.33.. -> -3333, not -3334


def test_scale_and_precision_cap_at_38():
    assert avg([5, 6], 38, 36) == ((38, 38), 550)            # ts = min(38, 40): the sum is multiplied by 10^2 only
    assert avg([5, 6], 36, 38) == ((38, 38), 5)              # s = 38: no rescale, 11 / 2 = 5
    assert avg([7], 35, 2) == ((38, 6), 70000)


def test_precision_overflow_is_an_error():
    with pytest.raises(O.ArrowArithmeticOverflow, match="AvgAccumulator"):
        avg([10 ** 37, 10 ** 37], 38, 0)                      # sum * 10^4 overflows i128
    with pytest.raises(O.ArrowArithmeticOverflow, match="AvgAccumulator"):
        avg([12 * 10 ** 33], 38, 0)                            # fits i128, but 1.2e38 has 39 digits
    assert avg([99 * 10 ** 32], 38, 0) == ((38, 4), 99 * 10 ** 36)   # 9.9e37: 38 digits, fits


def test_nulls_are_skipped_and_no_value_is_null():
    assert avg([100, 999, 300], 15, 2, np.array([True, False, True])) == ((19, 6), 2000000)
    assert avg([100], 15, 2, np.array([False])) == ((19, 6), None)


def test_min_max_with_mixed_signs_grouped_and_scalar():
    d = O.Dec([5, -7, 10 ** 30, -(10 ** 30) - 1, 0, 3], 38, 2)
    g = (np.array([1, 1, 2, 2, 1, 2]), None)
    keys, res = DA.group_by([g], [(O.A_MIN, (d, None), None), (O.A_MAX, (d, None), None), (O.A_AVG, (d, None), None)])
    assert keys[0][0].tolist() == [1, 2]
    assert [int(x) for x in res[0]["dec"]] == [-7, -(10 ** 30) - 1]
    assert [int(x) for x in res[1]["dec"]] == [5, 10 ** 30]
    assert (res[2]["dec"].p, res[2]["dec"].s) == (38, 6)
    assert [int(x) for x in res[2]["dec"]] == [-6666, 6666]     # (5 - 7 + 0) * 10^4 / 3 and (10^30 - 10^30 - 1 + 3) * 10^4 / 3
    cols = DA.agg_output_columns(O.A_MIN, res[0], object, False)
    assert (cols[0][0].p, cols[0][0].s) == (38, 2) and cols[0][1] is None
    (mn, _), (mx, _) = DA.scalar_aggregate([(O.A_MIN, (d, None), None), (O.A_MAX, (d, None), None)])
    assert (int(mn[0]), int(mx[0])) == (-(10 ** 30) - 1, 10 ** 30) and (mn.p, mn.s) == (38, 2)
