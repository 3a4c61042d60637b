"""MIN, MAX and AVG over Decimal128 in the fused pipeline's join-keyed aggregate sink (dfgpu_pipeline_sink_aggregate: the group is the
build row, the accumulators are words of its record).  Every result is compared exactly with tests/decimal_agg.py and the oracle
(through test_gpu_agg_decimal.reference) over the join computed here, keyed by the group tuple.  The cases cover (15,2), (38,4) and
(38,38) columns and the TPC-H Q3 revenue expression with and without NULLs; +-(10^38 - 1) and low words across bit 63; all-NULL
groups with and without a non-null counter; one million rows racing on 16 pairs; Partial MIN / MAX merged by dfgpu_agg's Final; AVG
past its precision; the record-layout rejections; and the operator twin's fused plan against the unfused dfgpu_hashjoin -> dfgpu_agg."""
from decimal import Decimal

import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from datafusion_b200.exec import AggregateExpr, GpuAggregateExec, GpuHashJoinExec, GpuPipelineExec, MemoryExec, collect, fuse_pipelines
from oracle import oracle as O
import decimal_agg as DA
from decimal_util import gpu_nodes
from test_gpu_agg_decimal import I128_MAX, as_map, assert_same, dec_values, drain_rows, push, reference
from test_gpu_pipeline import build_lookup

pytestmark = pytest.mark.gpu
TYPES = [(15, 2), (38, 4), (38, 38)]
COL = lambda i: (O.E_COLUMN, i, None, 0, 0)
BIN = lambda op: (O.E_BINARY, op, None, 0, 0)
DLIT = lambda v, p, s: (O.E_LITERAL, 0, O.decimal_dtype(p, s), 0, v)
REV = [COL(1), DLIT(1, 20, 0), COL(2), BIN(O.OP_MINUS), BIN(O.OP_MULTIPLY)]   # l_extendedprice * (1 - l_discount) -> Decimal128(38, 4)
MMA = [D.AGG_MIN, D.AGG_MAX, D.AGG_AVG, D.AGG_COUNT_STAR]


def lookup(ctx, keys, payload, n_acc):
    """the build side: unique Int64 keys, with an Int32 payload (key % 13) or key only"""
    if payload:
        return build_lookup(ctx, [(keys, None), ((keys % 13).astype(np.int32), None)], [D.INT64, D.INT32], 0, [1], n_acc_words=n_acc,
                            expected_rows=len(keys))[0]
    return build_lookup(ctx, [(keys, None)], [D.INT64], 0, [], n_acc_words=n_acc, expected_rows=len(keys))[0]


def fused(ctx, look, cols, types, aggs, mode=D.AGG_SINGLE, payload=True, batch_rows=None):
    """probe columns (0 = the join key) -> the join-keyed sink; aggs: [(func, oracle nodes or None)] -> (rows, output types)"""
    p = D.Pipeline(ctx, types, None, [(D.STAGE_INNER, 0, look)])
    try:
        p.sink_aggregate([0, len(types)] if payload else [0], [(f, None if n is None else gpu_nodes(D, n)) for f, n in aggs], mode)
        push(ctx, p, cols, types, batch_rows)
        p.finish()
        return drain_rows(p)
    finally:
        p.close()


def _take(c, idx):
    if isinstance(c[0], O.Dec):
        return (O.Dec([int(c[0][i]) for i in idx], c[0].p, c[0].s), None if c[1] is None else np.asarray(c[1])[idx])
    return (np.asarray(c[0])[idx], None if c[1] is None else np.asarray(c[1])[idx])


def expected(build_keys, cols, args, funcs, payload=True):
    """the unfused chain: inner join on column 0, the argument columns `args` (oracle columns over the probe rows), GROUP BY the key
    (and the payload) -> {group tuple: values}"""
    m = np.isin(cols[0][0], build_keys)
    if cols[0][1] is not None:
        m &= np.asarray(cols[0][1], bool)
    idx = np.nonzero(m)[0]
    k = np.asarray(cols[0][0])[idx]
    jc = [(k, None), ((k % 13).astype(np.int32), None)] + [_take(a, idx) for a in args]
    return reference(jc, [0, 1] if payload else [0], [(f, -1 if f == D.AGG_COUNT_STAR else 2, -1) for f in funcs]), jc


def probe_case(rng, n, nb, p, s, nulls):
    keys = np.arange(nb, dtype=np.int64) * 3 + 1
    pk = rng.integers(0, nb * 5 // 4, n).astype(np.int64) * 3 + 1          # a fifth of the rows have no partner
    v = (O.Dec(dec_values(rng, n, p, s), p, s), (rng.random(n) > 0.1) if nulls else None)
    return keys, [(pk, None), v], [D.INT64, D.decimal128(p, s)]


def assert_truncation_is_tested(jc, want):
    """some group's AVG is negative and its truncation toward zero differs from floor division"""
    sums, cnts = {}, {}
    v, val = jc[2]
    for i in range(len(v)):
        if val is None or val[i]:
            g = (int(jc[0][0][i]), int(jc[1][0][i]))
            sums[g] = sums.get(g, 0) + int(v[i]); cnts[g] = cnts.get(g, 0) + 1
    mul = min(38, v.s + 4) - v.s
    assert any(sums[g] < 0 and (sums[g] * 10 ** mul) % cnts[g] and want[g][2] == DA._tdiv(sums[g] * 10 ** mul, cnts[g]) for g in sums)


@pytest.mark.parametrize("nulls", [False, True], ids=["no_nulls", "nulls"])
@pytest.mark.parametrize("p,s", TYPES)
def test_min_max_avg_over_a_decimal_column(gpu_ctx, p, s, nulls):
    rng = np.random.default_rng(300 + p + s + nulls)
    keys, cols, types = probe_case(rng, 60_000, 3000, p, s, nulls)
    look = lookup(gpu_ctx, keys, True, 10)        # row counter, padding, 2 pairs, AVG {lo, hi, count}, 2 non-null counters (one the padding)
    got, ot = fused(gpu_ctx, look, cols, types, [(f, None if f == D.AGG_COUNT_STAR else [COL(1)]) for f in MMA], batch_rows=17_000)
    look.close()
    want, jc = expected(keys, cols, [cols[1]], MMA)
    assert_same(got, want, 2, f"decimal({p},{s})")
    assert ot == [D.INT64, D.INT32, D.decimal128(p, s), D.decimal128(p, s), D.decimal128(min(38, p + 4), min(38, s + 4)), D.INT64]
    assert_truncation_is_tested(jc, want)


@pytest.mark.parametrize("nulls", [False, True], ids=["no_nulls", "nulls"])
def test_min_max_avg_over_the_q3_revenue_expression(gpu_ctx, nulls):
    rng = np.random.default_rng(31 + nulls)
    n, nb = 80_000, 4000
    keys = np.arange(nb, dtype=np.int64) * 3 + 1
    pk = rng.integers(0, nb * 5 // 4, n).astype(np.int64) * 3 + 1
    price = (O.Dec(rng.integers(-10_500_000, 10_500_000, n).tolist(), 15, 2), (rng.random(n) > 0.05) if nulls else None)
    disc = (O.Dec(rng.integers(0, 11, n).tolist(), 15, 2), None)
    cols, types = [(pk, None), price, disc], [D.INT64, D.decimal128(15, 2), D.decimal128(15, 2)]
    # without NULLs SUM fits beside them (11 words); with NULLs MIN and MAX need their non-null counters (10 words with COUNT(*))
    funcs = [D.AGG_MIN, D.AGG_MAX, D.AGG_AVG, D.AGG_COUNT_STAR if nulls else D.AGG_SUM]
    look = lookup(gpu_ctx, keys, True, 10 if nulls else 11)
    got, ot = fused(gpu_ctx, look, cols, types, [(f, None if f == D.AGG_COUNT_STAR else REV) for f in funcs], batch_rows=30_000)
    look.close()
    arg = O.eval_expr(cols, REV)
    assert (arg[0].p, arg[0].s) == (38, 4)
    want, jc = expected(keys, cols, [arg], funcs)
    assert_same(got, want, 2, "revenue")
    assert ot[2:5] == [D.decimal128(38, 4), D.decimal128(38, 4), D.decimal128(38, 8)]
    assert_truncation_is_tested(jc, want)


def test_key_only_lookup_with_an_even_record(gpu_ctx):
    rng = np.random.default_rng(5)
    keys, cols, types = probe_case(rng, 40_000, 2000, 38, 4, True)
    look = lookup(gpu_ctx, keys, False, 11)       # key + 11 words: row counter, 2 pairs, AVG, 2 non-null counters, one spare
    got, _ = fused(gpu_ctx, look, cols, types, [(f, None if f == D.AGG_COUNT_STAR else [COL(1)]) for f in MMA], payload=False, batch_rows=9000)
    look.close()
    want, _ = expected(keys, cols, [cols[1]], MMA, payload=False)
    assert_same(got, want, 1, "key only")


def test_extreme_values_and_bit63_pairs(gpu_ctx):
    """+-(10^38 - 1), the largest Decimal128(38, 0) magnitudes, and pairs that differ only across bit 63 of the low word, with and
    without NULLs (group 8 has only NULL arguments: MIN and MAX are NULL, its rows are counted)"""
    big = 10 ** 38 - 1
    groups = {0: [big], 1: [-big], 2: [big, -big], 3: [(1 << 63) - 1, 1 << 63], 4: [-(1 << 64), -1],
              5: [(1 << 64) + (1 << 63), (1 << 64) + (1 << 63) - 1], 6: [-(1 << 63), -(1 << 63) - 1], 7: [0]}
    keys, vals = [], []
    for _ in range(50):
        for g, vs in groups.items():
            keys += [g] * len(vs); vals += vs
    funcs = [D.AGG_MIN, D.AGG_MAX, D.AGG_COUNT_STAR]
    for nulls in (False, True):
        k = np.array(keys + ([8] * 3 if nulls else []), np.int64)
        v = vals + ([5] * 3 if nulls else [])
        valid = np.array([True] * len(vals) + [False] * 3) if nulls else None
        cols, types = [(k, None), (O.Dec(v, 38, 0), valid)], [D.INT64, D.decimal128(38, 0)]
        look = lookup(gpu_ctx, np.arange(9, dtype=np.int64), True, 7)   # row counter, padding (= MIN's non-null counter), 2 pairs, MAX's counter
        got, _ = fused(gpu_ctx, look, cols, types, [(f, None if f == D.AGG_COUNT_STAR else [COL(1)]) for f in funcs], batch_rows=97)
        look.close()
        want, _ = expected(np.arange(9), cols, [cols[1]], funcs)
        assert_same(got, want, 2, f"extremes nulls={nulls}")
        g = as_map(got, 2)
        assert g[(0, 0)][:2] == (big, big) and g[(1, 1)][:2] == (-big, -big) and g[(2, 2)][:2] == (-big, big)
        assert g[(3, 3)][:2] == ((1 << 63) - 1, 1 << 63) and g[(4, 4)][:2] == (-(1 << 64), -1) and g[(6, 6)][:2] == (-(1 << 63) - 1, -(1 << 63))
        if nulls:
            assert g[(8, 8)] == (None, None, 3)


def test_all_null_group_with_and_without_a_non_null_counter(gpu_ctx):
    k = np.array([1, 1, 2, 2, 2], np.int64)
    cols = [(k, None), (O.Dec([5, -7, 1, 2, 3], 15, 2), np.array([True, True, False, False, False]))]
    types = [D.INT64, D.decimal128(15, 2)]
    keys = np.array([1, 2], np.int64)
    aggs = [(D.AGG_MIN, [COL(1)]), (D.AGG_MAX, [COL(1)])]
    look = lookup(gpu_ctx, keys, False, 7)          # key + row counter, 2 pairs, 2 non-null counters (+ 1 spare): 8 words
    got, _ = fused(gpu_ctx, look, cols, types, aggs, payload=False)
    look.close()
    assert as_map(got, 1) == {(1,): (-7, 5), (2,): (None, None)}
    look = lookup(gpu_ctx, keys, False, 5)          # key + row counter, 2 pairs: no word left for a non-null counter
    with pytest.raises(D.DfgpuError, match="n_acc_words") as ei:
        fused(gpu_ctx, look, cols, types, aggs, payload=False)
    assert ei.value.code == -3
    look.close()
    look = lookup(gpu_ctx, keys, False, 5)          # the same words are enough when the argument cannot be NULL
    got, _ = fused(gpu_ctx, look, [cols[0], (cols[1][0], None)], types, aggs, payload=False)
    look.close()
    assert as_map(got, 1) == {(1,): (-7, 5), (2,): (1, 3)}


def test_many_rows_race_on_few_pairs(gpu_ctx):
    """10^6 rows into 16 groups: every warp's lanes update the same few pairs (the CAS loop's retries), exact results"""
    rng = np.random.default_rng(77)
    n = 1_000_000
    keys = np.arange(16, dtype=np.int64) * 5 + 2
    pk = keys[rng.integers(0, 16, n)]
    vi = rng.integers(-10 ** 12, 10 ** 12, n)
    valid = rng.random(n) > 0.02
    cols, types = [(pk, None), (O.Dec(vi.tolist(), 15, 2), valid)], [D.INT64, D.decimal128(15, 2)]
    look = lookup(gpu_ctx, keys, True, 10)
    got, _ = fused(gpu_ctx, look, cols, types, [(f, None if f == D.AGG_COUNT_STAR else [COL(1)]) for f in MMA], batch_rows=400_000)
    look.close()
    want = {}
    for key in keys.tolist():
        sel = (pk == key)
        v = vi[sel & valid]
        total, c = int(v.sum()), len(v)
        want[(key, key % 13)] = (int(v.min()), int(v.max()), DA.decimal_avg(total, c, 15, 2)[0], int(sel.sum()))
    assert as_map(got, 2) == want


def test_partial_min_max_then_final_equals_single(gpu_ctx):
    rng = np.random.default_rng(12)
    keys, cols, types = probe_case(rng, 50_000, 2500, 38, 4, True)
    funcs = [D.AGG_MIN, D.AGG_MAX, D.AGG_COUNT_STAR]
    aggs = [(f, None if f == D.AGG_COUNT_STAR else [COL(1)]) for f in funcs]
    look = lookup(gpu_ctx, keys, True, 7)
    single, _ = fused(gpu_ctx, look, cols, types, aggs)
    look.close()
    # two Partial pipelines over the two halves of the probe side, merged by dfgpu_agg's Final
    h = None
    for part in ((0, 25_000), (25_000, 50_000)):
        look = lookup(gpu_ctx, keys, True, 7)
        p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_INNER, 0, look)])
        p.sink_aggregate([0, 2], [(f, None if n is None else gpu_nodes(D, n)) for f, n in aggs], D.AGG_PARTIAL)
        push(gpu_ctx, p, [(c[0][part[0]:part[1]], None if c[1] is None else c[1][part[0]:part[1]]) for c in cols], types)
        p.finish()
        outs = p.drain(host=True)
        st_types = [outs[0].column(i).type for i in range(5)]
        assert st_types == [D.INT64, D.INT32, D.decimal128(38, 4), D.decimal128(38, 4), D.INT64]
        if h is None:
            h = D.AggHandle(gpu_ctx, st_types, [0, 1], [(D.AGG_MIN, 2, -1), (D.AGG_MAX, 3, -1), (D.AGG_COUNT_STAR, 4, -1)], D.AGG_FINAL)
        for b in outs:
            h.push_host([D.HostColumn(*b.column_numpy(i), b.column(i).type) for i in range(5)])
        p.close(); look.close()
    h.finish()
    final, _ = drain_rows(h)
    h.close()
    assert as_map(final, 2) == as_map(single, 2)
    # AVG over Decimal128 has no pinned Partial state
    look = lookup(gpu_ctx, keys, True, 7)
    p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_INNER, 0, look)])
    with pytest.raises(D.DfgpuError, match="Single modes only") as ei:
        p.sink_aggregate([0, 2], [(D.AGG_AVG, gpu_nodes(D, [COL(1)]))], D.AGG_PARTIAL)
    assert ei.value.code == -3
    p.close(); look.close()


@pytest.mark.parametrize("p,s,inside,outside", [(36, 35, 10 ** 35 - 1, 10 ** 35), (38, 0, -(10 ** 34 - 1), -(10 ** 34))], ids=["36_35", "38_0_negative"])
def test_avg_at_and_past_the_target_precision(gpu_ctx, p, s, inside, outside):
    types = [D.INT64, D.decimal128(p, s)]
    for v, ok in ((inside, True), (outside, False)):
        cols = [(np.zeros(3, np.int64), None), (O.Dec([v, 0, 7], p, s), np.array([True, False, False]))]
        look = lookup(gpu_ctx, np.array([0], np.int64), True, 4)
        if ok:
            got, _ = fused(gpu_ctx, look, cols, types, [(D.AGG_AVG, [COL(1)]), (D.AGG_COUNT_STAR, None)])
            assert got == [(0, 0, v * 10 ** (min(38, s + 4) - s), 3)]
        else:
            with pytest.raises(O.ArrowArithmeticOverflow):
                DA.decimal_avg(v, 1, p, s)
            with pytest.raises(D.DfgpuError, match="Arithmetic Overflow in AvgAccumulator") as ei:
                fused(gpu_ctx, look, cols, types, [(D.AGG_AVG, [COL(1)]), (D.AGG_COUNT_STAR, None)])
            assert ei.value.code == -4
        look.close()


def test_record_layout_rejections(gpu_ctx):
    types = [D.INT64, D.decimal128(15, 2)]
    keys = np.array([1, 2], np.int64)
    cases = [(False, 4, [D.AGG_MIN], "n_acc_words"),          # key + 5 words: an odd record
             (False, 2, [D.AGG_MAX], "n_acc_words"),          # key + 3 words: odd as well
             (True, 3, [D.AGG_MIN], "n_acc_words"),           # row counter, padding, then one word of the pair
             (True, 5, [D.AGG_MIN, D.AGG_MAX], "n_acc_words"),   # row counter, padding, one pair and a half
             (False, 3, [D.AGG_AVG], "n_acc_words")]          # AVG takes three words besides the row counter
    for payload, n_acc, funcs, msg in cases:
        look = lookup(gpu_ctx, keys, payload, n_acc)
        p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_INNER, 0, look)])
        with pytest.raises(D.DfgpuError, match=msg) as ei:
            p.sink_aggregate([0, 2] if payload else [0], [(f, gpu_nodes(D, [COL(1)])) for f in funcs])
        assert ei.value.code == -3, (payload, n_acc, funcs)
        p.close(); look.close()


def _twin_tables(rng):
    no, nl = 5000, 60_000
    orders = pa.table({"o_orderkey": pa.array(np.arange(no, dtype=np.int64) * 4 + 1), "o_d": pa.array(rng.integers(8000, 10500, no).astype(np.int32)).cast(pa.date32())})
    lk = rng.integers(0, no * 5 // 4, nl).astype(np.int64) * 4 + 1
    # ~5 % NULL prices, and every price of one order in a hundred NULL (groups whose MIN / MAX / SUM / AVG are NULL)
    price = [None if (rng.random() < 0.05 or k % 400 == 1) else Decimal(int(x)).scaleb(-2) for k, x in zip(lk.tolist(), rng.integers(-10_500_000, 10_500_000, nl))]
    lineitem = pa.table({"l_orderkey": pa.array(lk), "l_price": pa.array(price, pa.decimal128(15, 2))})
    mem = lambda t: MemoryExec(t.to_batches(max_chunksize=20_000), t.schema)
    return mem(orders), mem(lineitem)


@pytest.mark.parametrize("funcs", [("sum", "min", "max"), ("min", "avg", "max", "count")], ids=["sum_min_max", "min_avg_max_count"])
def test_twin_fuses_and_matches_the_unfused_plan(gpu_ctx, task_ctx, funcs):
    """fuse_pipelines over join + GROUP BY with Decimal128 SUM / MIN / MAX / AVG of a nullable Decimal128(15,2) column returns a
    GpuPipelineExec whose rows and types equal those of the unfused GpuHashJoinExec -> GpuAggregateExec (dfgpu_hashjoin -> dfgpu_agg)"""
    o, l = _twin_tables(np.random.default_rng(8))
    join = GpuHashJoinExec(o, l, [("o_orderkey", "l_orderkey")], "Inner")
    plan = GpuAggregateExec("Single", ["l_orderkey", "o_d"], [AggregateExpr(f, "l_price", f"a{i}") for i, f in enumerate(funcs)], join)
    fused_plan = fuse_pipelines(plan)
    assert isinstance(fused_plan, GpuPipelineExec)
    got, ref = collect(fused_plan, task_ctx), collect(plan, task_ctx)
    assert [b.schema.types for b in got][0] == [b.schema.types for b in ref][0] == list(plan.schema.types)
    key = lambda r: (r["l_orderkey"], r["o_d"])
    rows = lambda bs: sorted(pa.Table.from_batches(bs).to_pylist(), key=key)
    g, r = rows(got), rows(ref)
    assert len(g) == len(r) > 3000 and g == r
    assert any(v is None for row in r for v in row.values())            # a group whose prices are all NULL


def test_twin_leaves_sum_min_max_avg_together_unfused():
    """nullable SUM, MIN, MAX and AVG over Decimal128 together need 14 accumulator words, more than a lookup holds"""
    o, l = _twin_tables(np.random.default_rng(9))
    join = GpuHashJoinExec(o, l, [("o_orderkey", "l_orderkey")], "Inner")
    plan = GpuAggregateExec("Single", ["l_orderkey", "o_d"], [AggregateExpr(f, "l_price", f) for f in ("sum", "min", "max", "avg")], join)
    assert fuse_pipelines(plan) is plan
