"""The fusion rule's planning of MIN, MAX and AVG over Decimal128 in the join-keyed aggregate sink (no GPU needed: nothing runs).
`fuse_pipelines` fuses what dfgpu_pipeline_sink_aggregate accepts and reserves the accumulator words its placement needs (dfgpu.h):
the row counter; 2 words per Decimal128 SUM / MIN / MAX plus a non-null counter, 3 per Decimal128 AVG; one padding word in front of
the 16-byte MIN / MAX pairs; a record of an even number of words when the build carries no payload.  Plans without decimals keep the
counts they had."""
from decimal import Decimal

import pyarrow as pa
import pytest

from datafusion_b200.exec import AggregateExpr, GpuAggregateExec, GpuHashJoinExec, GpuPipelineExec, MemoryExec, _acc_words, fuse_pipelines

MONEY = pa.decimal128(15, 2)


def _mem(t):
    return MemoryExec(t.to_batches(), t.schema)


def join(payload=True, money=MONEY):
    """orders (key [+ o_d payload]) JOIN lineitem on o_orderkey = l_orderkey; l_price nullable"""
    cols = {"o_orderkey": pa.array([1, 2, 3], pa.int64())}
    if payload:
        cols["o_d"] = pa.array([9000, 9001, 9002], pa.int32()).cast(pa.date32())
    orders = pa.table(cols)
    vals = [Decimal("1.25"), None, Decimal("-3.50"), Decimal("7.00")] if pa.types.is_decimal(money) else [125, None, -350, 700]
    lineitem = pa.table({"l_orderkey": pa.array([1, 1, 2, 3], pa.int64()), "l_price": pa.array(vals, money)})
    return GpuHashJoinExec(_mem(orders), _mem(lineitem), [("o_orderkey", "l_orderkey")], "Inner")


def agg(mode, funcs, payload=True, money=MONEY):
    group = ["l_orderkey", "o_d"] if payload else ["l_orderkey"]
    return GpuAggregateExec(mode, group, [AggregateExpr(f, "l_price", f"a{i}") for i, f in enumerate(funcs)], join(payload, money))


def words(plan):
    return plan.scan.stages[-1][2].n_acc_words


@pytest.mark.parametrize("mode", ["Single", "SinglePartitioned"])
@pytest.mark.parametrize("func", ["min", "max", "avg", "sum"])
def test_rule_fuses_decimal_aggregates_in_single_modes(mode, func):
    plan = agg(mode, [func])
    fused = fuse_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.schema == plan.schema and [a[0] for a in fused.aggs] == [func]


@pytest.mark.parametrize("func", ["min", "max", "sum"])
def test_rule_fuses_decimal_min_max_sum_in_partial_mode(func):
    fused = fuse_pipelines(agg("Partial", [func]))
    assert isinstance(fused, GpuPipelineExec) and fused.mode == "Partial"


def test_rule_leaves_partial_decimal_avg_alone():
    plan = agg("Partial", ["avg"])
    assert fuse_pipelines(plan) is plan
    plan = agg("Partial", ["min", "avg"])
    assert fuse_pipelines(plan) is plan


@pytest.mark.parametrize("funcs,payload,n", [
    (["sum"], True, 1 + 3),                      # row counter, {lo, hi}, non-null counter
    (["avg"], True, 1 + 3),                      # row counter, {lo, hi}, count
    (["min"], True, 1 + 3 + 1),                  # ... and the padding word in front of the pair
    (["min", "max"], True, 1 + 3 + 3 + 1),
    (["sum", "min", "max"], True, 1 + 9 + 1),
    (["min", "avg"], True, 1 + 3 + 3 + 1),
    (["min"], False, 5),                         # key + 5 words: an even record
    (["max", "count"], False, 1 + 3 + 1 + 1 + 1),   # 6 words -> 7 (key + 7 = 8)
    (["avg"], False, 4),                         # no pair: no padding, no even-record rule
])
def test_exact_accumulator_words(funcs, payload, n):
    fused = fuse_pipelines(agg("Single", funcs, payload))
    assert isinstance(fused, GpuPipelineExec) and words(fused) == n
    if not payload and any(f in ("min", "max") for f in funcs):
        assert (1 + words(fused)) % 2 == 0


def test_plans_over_twelve_words_stay_unfused():
    # nullable SUM + MIN + MAX + AVG over Decimal128 need 1 + 9 + 3 + a padding word = 14 > 12
    plan = agg("Single", ["sum", "min", "max", "avg"])
    assert fuse_pipelines(plan) is plan
    assert _acc_words(["sum", "min", "max", "avg"], [MONEY] * 4, True) == 14


def test_timing_script_check_on_host_rows():
    """scripts/q3_decimal_aggs_timing.py's exact Int64 <-> Decimal128 check on a few hand-made groups"""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import numpy as np
    import q3_decimal_aggs_timing as T
    cols = lambda rows: [np.array(c, np.int64) for c in zip(*rows)]
    ints = [(1, 9000, 0, -7, -5, -2, 3), (2, 9001, 0, 10, 10, 10, 1), (5, 9003, 0, 8, 1, 7, 2)]
    decs = [(5, 9003, 0, 8, 1, 7, 40_000), (2, 9001, 0, 10, 10, 10, 100_000), (1, 9000, 0, -7, -5, -2, -23_333)]   # tdiv(-70000, 3) = -23333
    T.check_rows(cols(ints), cols(decs))                 # output order does not matter
    for j in range(7):                                   # every compared column is compared
        bad = [list(r) for r in decs]
        bad[2][j] += 1
        with pytest.raises(AssertionError):
            T.check_rows(cols(ints), cols(bad))
    with pytest.raises(AssertionError):                  # floor division instead of truncation toward zero
        T.check_rows(cols(ints), cols(decs[:2] + [decs[2][:6] + (-23_334,)]))
    with pytest.raises(AssertionError):
        T.check_rows(cols(ints), cols(decs[:2]))


@pytest.mark.parametrize("funcs,n", [(["sum"], 3), (["min"], 3), (["sum", "min", "max"], 7), (["avg"], 3), (["sum", "count", "avg"], 6)])
def test_int64_plans_keep_their_word_counts(funcs, n):
    money = pa.int64()
    if "avg" in funcs:                           # AVG fuses over Float64 only (the planner casts)
        money = pa.float64()
    fused = fuse_pipelines(agg("Single", funcs, money=money))
    assert isinstance(fused, GpuPipelineExec) and words(fused) == n
    # the count the rule has always reserved: row counter, 1 word per aggregate (2 per AVG), a non-null counter per SUM / MIN / MAX
    assert n == 1 + sum(2 if f == "avg" else 1 for f in funcs) + sum(1 for f in funcs if f in ("sum", "min", "max"))
    # without payload nothing is rounded up: the even-record rule concerns Decimal128 pairs only
    assert _acc_words(funcs, [money] * len(funcs), False) == n
