"""The fused pipeline's hash-keyed aggregate sink (dfgpu_pipeline_sink_aggregate_hash): filter [-> probe stages] -> GROUP BY keys that
the join key does not determine, packed into a 128-bit tag, in one kernel with the sink's own group table.  Every result is compared with
the unfused chain restated on the CPU (filter, the stages' joins, then decimal_agg / the oracle's group-by, or pandas for the large cases):
integers and decimals exactly, Float64 within 1e-9 relative.  The cases cover the Q15 revenue0 and Q3-by-customer shapes, SEMI and ANTI
stages, keys mixing an input column with payload fields of two INNER stages, key widths 1..8 bytes signed and unsigned with their extremes,
the side record of the one tag equal to the empty marker, the 128-bit limit, NULL groups, every aggregate over nullable and non-null
arguments, Decimal128 at (15,2) and (38,4) with +-(10^38 - 1), Single / SinglePartitioned / Partial (merged by dfgpu_agg's Final), growth
from a one-group hint within one push and across pushes, 10^7 rows racing on 16 groups, the rejections, and the operator twin."""
import math

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
from decimal_util import gpu_nodes
from test_gpu_agg_decimal import as_map, drain_rows, push, reference
from test_gpu_pipeline import build_lookup

pytestmark = pytest.mark.gpu


def col(i): return (O.E_COLUMN, i, None, 0, 0)
def lit(v, dt): return (O.E_LITERAL, 0, dt, 0, v)
def bop(op): return (O.E_BINARY, op, None, 0, 0)


NP = {D.INT8: np.int8, D.UINT8: np.uint8, D.INT16: np.int16, D.UINT16: np.uint16, D.INT32: np.int32, D.UINT32: np.uint32,
      D.INT64: np.int64, D.UINT64: np.uint64}


def _take(c, idx):
    if isinstance(c[0], O.Dec):
        return (O.Dec([int(c[0][i]) for i in idx], c[0].p, c[0].s), None if c[1] is None else np.asarray(c[1])[idx])
    return (np.asarray(c[0])[idx], None if c[1] is None else np.asarray(c[1])[idx])


def lookup(ctx, keys, pays=()):
    """a build side of unique Int64 keys and payload columns [(values, type)]"""
    cols = [(keys, None)] + [(v, None) for v, _ in pays]
    types = [D.INT64] + [t for _, t in pays]
    return build_lookup(ctx, cols, types, 0, list(range(1, len(cols))), expected_rows=len(keys))[0]


def virtual(cols, pred, stages):
    """the unfused chain on the CPU -> the virtual columns of the rows that reach the sink.  stages: [(kind, key_col, keys, pays)]"""
    n = len(cols[0][0])
    keep = np.ones(n, bool)
    if pred is not None:
        m = O.eval_expr(cols, pred)
        keep &= np.asarray(m[0], bool) & (True if m[1] is None else np.asarray(m[1], bool))
    ext = []
    for kind, kc, keys, pays in stages:
        k, kv = cols[kc]
        pos = pd.Index(keys).get_indexer(np.asarray(k))
        found = (pos >= 0) & (True if kv is None else np.asarray(kv, bool))
        keep &= ~found if kind == D.STAGE_ANTI else found
        if kind == D.STAGE_INNER:
            ext += [(np.asarray(v)[np.maximum(pos, 0)], None) for v, _ in pays]
    idx = np.nonzero(keep)[0]
    return [_take(c, idx) for c in list(cols) + ext]


def run_hash(ctx, cols, types, group_cols, aggs, pred=None, stages=(), nullable=None, mode=D.AGG_SINGLE, batch_rows=None, capacity_hint=0,
             batch_size=0):
    """the fused pipeline -> (rows, output types, metrics); aggs: [(func, oracle nodes or None)]"""
    p = D.Pipeline(ctx, types, gpu_nodes(D, pred) if pred else None, stages)
    try:
        p.sink_aggregate_hash(group_cols, [(f, None if n is None else gpu_nodes(D, n)) for f, n in aggs], mode, batch_size, capacity_hint, nullable)
        push(ctx, p, cols, types, batch_rows)
        p.finish()
        rows, ot = drain_rows(p)
        m = {k: p.metric(k) for k in ("num_groups", "sink_rows", "group_rehashes", "replayed_rows", "output_rows")}
        return rows, ot, m
    finally:
        p.close()


def expected(vcols, group_cols, aggs):
    """{group tuple: values} of the aggregates over the virtual columns; an argument program is evaluated into a column first"""
    vc, spec = list(vcols), []
    for f, nodes in aggs:
        if nodes is None:
            spec.append((f, -1, -1))
        elif len(nodes) == 1 and nodes[0][0] == O.E_COLUMN:
            spec.append((f, nodes[0][1], -1))
        else:
            vc.append(O.eval_expr(vcols, nodes))
            spec.append((f, len(vc) - 1, -1))
    return reference(vc, group_cols, spec)


def close(a, b):
    if isinstance(a, float) or isinstance(b, float):
        return a is not None and b is not None and math.isclose(a, b, rel_tol=1e-9)
    return a == b


def assert_groups(rows, want, nk, what=""):
    got = as_map(rows, nk)
    assert len(got) == len(want), f"{what}: {len(got)} groups, expected {len(want)}"
    bad = [k for k in want if k not in got or len(got[k]) != len(want[k]) or not all(close(a, b) for a, b in zip(got[k], want[k]))]
    assert not bad, f"{what}: {len(bad)} groups differ, e.g. {bad[0]}: {got.get(bad[0])} != {want[bad[0]]}"


def lineitem(rng, n, nsupp, money=D.INT64):
    """Q15-like columns: 0 l_suppkey Int64, 1 l_extendedprice, 2 l_discount (Int64 cents or Decimal128(15,2)), 3 l_shipdate Int32"""
    supp = rng.integers(1, nsupp + 1, n).astype(np.int64)
    price = rng.integers(90_000, 10_500_000, n).astype(np.int64)
    disc = rng.integers(0, 11, n).astype(np.int64)
    ship = rng.integers(8000, 10600, n).astype(np.int32)
    if money == D.INT64:
        return [(supp, None), (price, None), (disc, None), (ship, None)], [D.INT64, D.INT64, D.INT64, D.INT32]
    dt = D.decimal128(15, 2)
    return [(supp, None), (O.Dec(price.tolist(), 15, 2), None), (O.Dec(disc.tolist(), 15, 2), None), (ship, None)], [D.INT64, dt, dt, D.INT32]


WINDOW = [col(3), lit(9000, np.int32), bop(O.OP_GTEQ), col(3), lit(9090, np.int32), bop(O.OP_LT), bop(O.OP_AND)]
REV_I64 = [col(1), lit(100, np.int64), col(2), bop(O.OP_MINUS), bop(O.OP_MULTIPLY)]
REV_DEC = [col(1), (O.E_LITERAL, 0, O.decimal_dtype(20, 0), 0, 1), col(2), bop(O.OP_MINUS), bop(O.OP_MULTIPLY)]


# ---------------------------------------------------------------- shapes
@pytest.mark.parametrize("mode", [D.AGG_SINGLE, D.AGG_SINGLE_PARTITIONED], ids=["single", "single_partitioned"])
@pytest.mark.parametrize("money", [D.INT64, "dec"], ids=["int64", "decimal"])
def test_q15_revenue0_filter_then_hash_sink(gpu_ctx, money, mode):
    rng = np.random.default_rng(15)
    cols, types = lineitem(rng, 200_000, 20_000, D.INT64 if money == D.INT64 else None)
    rev = REV_I64 if money == D.INT64 else REV_DEC
    aggs = [(D.AGG_SUM, rev), (D.AGG_COUNT_STAR, None), (D.AGG_MIN, [col(1)]), (D.AGG_MAX, [col(1)])]
    rows, ot, m = run_hash(gpu_ctx, cols, types, [0], aggs, pred=WINDOW, mode=mode, batch_rows=70_000, batch_size=1000)
    vc = virtual(cols, WINDOW, [])
    want = expected(vc, [0], aggs)
    assert_groups(rows, want, 1, "revenue0")
    assert m["sink_rows"] == len(vc[0][0]) and m["num_groups"] == len(want) and m["output_rows"] == len(want)
    assert ot[0] == D.INT64


@pytest.mark.parametrize("kind", [D.STAGE_SEMI, D.STAGE_ANTI], ids=["semi", "anti"])
def test_semi_and_anti_stages_in_front_of_the_sink(gpu_ctx, kind):
    rng = np.random.default_rng(20 + kind)
    cols, types = lineitem(rng, 150_000, 5000)
    keys = np.arange(1, 5001, 3, dtype=np.int64)
    look = lookup(gpu_ctx, keys)
    aggs = [(D.AGG_SUM, [col(1)]), (D.AGG_COUNT_STAR, None)]
    rows, _, m = run_hash(gpu_ctx, cols, types, [3], aggs, pred=WINDOW, stages=[(kind, 0, look)])
    look.close()
    vc = virtual(cols, WINDOW, [(kind, 0, keys, [])])
    assert_groups(rows, expected(vc, [3], aggs), 1, "semi/anti")
    assert m["sink_rows"] == len(vc[0][0])


def q3_case(rng, nord, nline):
    okey = np.arange(nord, dtype=np.int64) * 4 + 1
    ocust = rng.integers(1, nord // 10 + 2, nord).astype(np.int32)
    oprio = rng.integers(0, 5, nord).astype(np.int32)
    odate = rng.integers(8000, 10500, nord).astype(np.int32)
    pays = [(ocust, D.INT32), (oprio, D.INT32)]
    lkey = okey[rng.integers(0, nord, nline)] + (rng.random(nline) < 0.2).astype(np.int64)   # a fifth of the rows have no partner
    price = rng.integers(90_000, 10_500_000, nline).astype(np.int64)
    disc = rng.integers(0, 11, nline).astype(np.int64)
    ship = rng.integers(8000, 10600, nline).astype(np.int32)
    return okey, odate, pays, [(lkey, None), (price, None), (disc, None), (ship, None)], [D.INT64, D.INT64, D.INT64, D.INT32]


@pytest.mark.parametrize("group", [[4], [5], [5, 4]], ids=["o_custkey", "o_shippriority", "both"])
def test_q3_grouped_by_a_build_column(gpu_ctx, group):
    rng = np.random.default_rng(3)
    okey, _, pays, cols, types = q3_case(rng, 40_000, 300_000)
    look = lookup(gpu_ctx, okey, pays)
    pred = [col(3), lit(9200, np.int32), bop(O.OP_GT)]
    aggs = [(D.AGG_SUM, REV_I64), (D.AGG_COUNT_STAR, None)]
    rows, ot, m = run_hash(gpu_ctx, cols, types, group, aggs, pred=pred, stages=[(D.STAGE_INNER, 0, look)], capacity_hint=100)
    look.close()
    vc = virtual(cols, pred, [(D.STAGE_INNER, 0, okey, pays)])
    assert_groups(rows, expected(vc, group, aggs), len(group), "q3 by build column")
    assert m["sink_rows"] == len(vc[0][0])
    assert ot[:len(group)] == [D.INT32] * len(group)


def test_key_mixing_an_input_column_with_payload_fields_of_two_inner_stages(gpu_ctx):
    rng = np.random.default_rng(7)
    n = 200_000
    k1 = rng.integers(0, 3000, n).astype(np.int64); k2 = rng.integers(0, 500, n).astype(np.int64)
    g = rng.integers(-3, 4, n).astype(np.int16); v = rng.integers(-10**6, 10**6, n).astype(np.int64)
    b1 = np.arange(0, 3000, 2, dtype=np.int64); b2 = np.arange(0, 500, dtype=np.int64)
    p1 = [((b1 % 7).astype(np.int8), D.INT8), ((b1 * 11).astype(np.int64) - 5000, D.INT64)]
    p2 = [((b2 % 13).astype(np.uint16), D.UINT16)]
    l1, l2 = lookup(gpu_ctx, b1, [(p1[0][0], D.INT8)]), lookup(gpu_ctx, b2, p2)
    cols, types = [(k1, None), (k2, None), (g, None), (v, None)], [D.INT64, D.INT64, D.INT16, D.INT64]
    aggs = [(D.AGG_SUM, [col(3)]), (D.AGG_MAX, [col(3)]), (D.AGG_COUNT_STAR, None)]
    stages = [(D.STAGE_INNER, 0, l1), (D.STAGE_INNER, 1, l2)]
    rows, ot, _ = run_hash(gpu_ctx, cols, types, [2, 4, 5], aggs, stages=stages, nullable=[False, False, True])
    l1.close(); l2.close()
    vc = virtual(cols, None, [(D.STAGE_INNER, 0, b1, p1[:1]), (D.STAGE_INNER, 1, b2, p2)])
    assert_groups(rows, expected(vc, [2, 4, 5], aggs), 3, "mixed key")
    assert ot[:3] == [D.INT16, D.INT8, D.UINT16]


# ---------------------------------------------------------------- key edges
@pytest.mark.parametrize("t", [D.INT8, D.UINT8, D.INT16, D.UINT16, D.INT32, D.UINT32, D.INT64, D.UINT64],
                         ids=["i8", "u8", "i16", "u16", "i32", "u32", "i64", "u64"])
def test_key_widths_and_extremes(gpu_ctx, t):
    rng = np.random.default_rng(40 + t)
    info = np.iinfo(NP[t])
    edges = [info.min, info.max, 0, 1, info.max - 1] + ([-1, info.min + 1] if info.min < 0 else [])
    n = 50_000
    k = np.concatenate([np.array(edges, NP[t]), rng.integers(info.min, int(info.max) + 1, n, dtype=NP[t]), np.array(edges * 3, NP[t])])
    kv = rng.random(len(k)) > 0.05
    v = rng.integers(-10**9, 10**9, len(k)).astype(np.int64)
    cols, types = [(k, kv), (v, None)], [t, D.INT64]
    aggs = [(D.AGG_SUM, [col(1)]), (D.AGG_MIN, [col(1)]), (D.AGG_COUNT_STAR, None)]
    rows, ot, _ = run_hash(gpu_ctx, cols, types, [0], aggs, nullable=[True], batch_rows=20_000)
    want = expected(cols, [0], aggs)
    assert (None,) in want and (int(info.min),) in want and (int(info.max),) in want
    assert_groups(rows, want, 1, f"key type {t}")
    assert ot[0] == t


def test_two_int64_columns_of_minus_one_take_the_side_record(gpu_ctx):
    """(-1, -1) over two non-nullable Int64 columns is the 128-bit tag {~0, ~0}: the empty marker, kept in the side record"""
    rng = np.random.default_rng(8)
    n = 100_000
    a = rng.integers(-2, 3, n).astype(np.int64); b = rng.integers(-2, 3, n).astype(np.int64)
    a[::7] = -1; b[::7] = -1
    a[:3] = [np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1]; b[:3] = [np.iinfo(np.int64).max, np.iinfo(np.int64).min, -1]
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    cols, types = [(a, None), (b, None), (v, None)], [D.INT64, D.INT64, D.INT64]
    aggs = [(D.AGG_SUM, [col(2)]), (D.AGG_COUNT_STAR, None)]
    for hint in (0, 1):   # with hint 1 the table grows, the side record moves with it
        rows, _, m = run_hash(gpu_ctx, cols, types, [0, 1], aggs, capacity_hint=hint)
        want = expected(cols, [0, 1], aggs)
        assert want[(-1, -1)][1] >= n // 7
        assert_groups(rows, want, 2, "side record")


def test_exactly_128_bits_accepted_129_rejected(gpu_ctx):
    types = [D.INT64, D.INT64, D.INT64]
    p = D.Pipeline(gpu_ctx, types)
    p.sink_aggregate_hash([0, 1], [(D.AGG_COUNT_STAR, None)])
    p.close()
    p = D.Pipeline(gpu_ctx, types)
    p.sink_aggregate_hash([0, 1], [(D.AGG_COUNT_STAR, None)], nullable=[False, False])
    p.close()
    for nul in ([True, False], [False, True]):
        p = D.Pipeline(gpu_ctx, types)
        with pytest.raises(D.DfgpuError, match="wider than 128 bits") as ei:
            p.sink_aggregate_hash([0, 1], [(D.AGG_COUNT_STAR, None)], nullable=nul)
        assert ei.value.code == -3
        p.close()
    p = D.Pipeline(gpu_ctx, [D.INT64, D.INT32, D.INT32, D.INT8])
    p.sink_aggregate_hash([0, 1, 2], [(D.AGG_COUNT_STAR, None)], nullable=[False, False, False])   # 128 bits
    p.close()
    p = D.Pipeline(gpu_ctx, [D.INT64, D.INT32, D.INT32, D.INT8])
    with pytest.raises(D.DfgpuError, match="wider than 128 bits"):
        p.sink_aggregate_hash([0, 1, 2, 3], [(D.AGG_COUNT_STAR, None)])                          # 136 bits
    p.close()


def test_null_groups_and_a_null_in_a_non_nullable_column(gpu_ctx):
    rng = np.random.default_rng(9)
    n = 80_000
    a = rng.integers(0, 50, n).astype(np.int32); av = rng.random(n) > 0.1
    b = rng.integers(0, 3, n).astype(np.int8); bv = rng.random(n) > 0.3
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    cols, types = [(a, av), (b, bv), (v, None)], [D.INT32, D.INT8, D.INT64]
    aggs = [(D.AGG_SUM, [col(2)]), (D.AGG_COUNT_STAR, None)]
    rows, _, _ = run_hash(gpu_ctx, cols, types, [0, 1], aggs, nullable=[True, True], batch_rows=30_000)
    want = expected(cols, [0, 1], aggs)
    assert (None, None) in want and (None, 1) in want and (7, None) in want
    assert_groups(rows, want, 2, "NULL groups")
    with pytest.raises(D.DfgpuError, match="declared non-nullable") as ei:
        run_hash(gpu_ctx, cols, types, [0, 1], aggs, nullable=[True, False])
    assert ei.value.code == -1


# ---------------------------------------------------------------- aggregates
@pytest.mark.parametrize("nulls", [False, True], ids=["no_nulls", "nulls"])
def test_every_aggregate(gpu_ctx, nulls):
    rng = np.random.default_rng(50 + nulls)
    n = 120_000
    g = rng.integers(0, 2000, n).astype(np.int64)
    i = rng.integers(-10**12, 10**12, n).astype(np.int64)
    u = rng.integers(0, 2**63, n, dtype=np.uint64)
    f = rng.normal(0, 1e6, n)
    iv, fv = ((rng.random(n) > 0.2), (rng.random(n) > 0.2)) if nulls else (None, None)
    cols, types = [(g, None), (i, iv), (u, iv), (f, fv)], [D.INT64, D.INT64, D.UINT64, D.FLOAT64]
    aggs = [[(D.AGG_COUNT, [col(1)]), (D.AGG_SUM, [col(1)]), (D.AGG_MIN, [col(1)]), (D.AGG_MAX, [col(1)])],
            [(D.AGG_MIN, [col(2)]), (D.AGG_MAX, [col(2)]), (D.AGG_SUM, [col(2)]), (D.AGG_COUNT_STAR, None)],
            [(D.AGG_SUM, [col(3)]), (D.AGG_MIN, [col(3)]), (D.AGG_MAX, [col(3)]), (D.AGG_AVG, [col(3)])]]
    for a in aggs:
        rows, _, _ = run_hash(gpu_ctx, cols, types, [0], a, batch_rows=50_000)
        assert_groups(rows, expected(cols, [0], a), 1, f"aggregates {a}")


@pytest.mark.parametrize("p,s", [(15, 2), (38, 4)])
def test_decimal_sum_min_max_avg(gpu_ctx, p, s):
    rng = np.random.default_rng(60 + p)
    n = 60_000
    g = rng.integers(0, 700, n).astype(np.int32)
    m = 10 ** p - 1
    vals = [int(x) * (m // 10 ** 6) for x in rng.integers(-10 ** 6, 10 ** 6, n)] if p == 15 else rng.integers(-10**15, 10**15, n).tolist()
    if p == 38:
        vals[:4] = [m, -m, m, -m]
        g[:4] = [5, 5, 6, 7]
    valid = rng.random(n) > 0.1
    valid[:4] = True
    cols, types = [(g, None), (O.Dec(vals, p, s), valid)], [D.INT32, D.decimal128(p, s)]
    aggs = [(D.AGG_MIN, [col(1)]), (D.AGG_MAX, [col(1)]), (D.AGG_SUM, [col(1)]), (D.AGG_COUNT, [col(1)])]
    rows, ot, _ = run_hash(gpu_ctx, cols, types, [0], aggs, batch_rows=25_000)
    want = expected(cols, [0], aggs)
    assert_groups(rows, want, 1, f"decimal({p},{s})")
    assert ot[1:3] == [D.decimal128(p, s)] * 2
    if p == 38:   # group 5 holds m and -m, groups 6 and 7 one of them each: MIN, MAX and the 128-bit SUM across the extremes
        assert want[(5,)][:2] == (-m, m) and want[(6,)][2] > 10 ** 37 and want[(7,)][2] < -10 ** 37
    avg = [(D.AGG_AVG, [col(1)]), (D.AGG_SUM, [col(1)])]
    small = [(g, None), (O.Dec(rng.integers(-10**15, 10**15, n).tolist(), p, s), valid)]
    rows, ot, _ = run_hash(gpu_ctx, small, types, [0], avg)
    assert_groups(rows, expected(small, [0], avg), 1, f"decimal({p},{s}) AVG")
    assert ot[1] == D.decimal128(min(38, p + 4), min(38, s + 4))


def test_decimal_avg_overflow_and_partial_avg(gpu_ctx):
    types = [D.INT64, D.decimal128(36, 35)]
    cols = [(np.zeros(3, np.int64), None), (O.Dec([10 ** 35, 0, 7], 36, 35), np.array([True, False, False]))]
    with pytest.raises(D.DfgpuError, match="Overflow") as ei:
        run_hash(gpu_ctx, cols, types, [0], [(D.AGG_AVG, [col(1)])])
    assert ei.value.code == -4
    p = D.Pipeline(gpu_ctx, types)
    with pytest.raises(D.DfgpuError, match="Single modes only") as ei:
        p.sink_aggregate_hash([0], [(D.AGG_AVG, gpu_nodes(D, [col(1)]))], D.AGG_PARTIAL)
    assert ei.value.code == -3
    p.close()


def test_divide_by_zero_in_an_argument(gpu_ctx):
    n = 10_000
    cols = [(np.arange(n, dtype=np.int64) % 10, None), (np.ones(n, np.int64), None), (np.where(np.arange(n) == 777, 0, 3).astype(np.int64), None)]
    with pytest.raises(D.DfgpuError, match="Divide by zero") as ei:
        run_hash(gpu_ctx, cols, [D.INT64] * 3, [0], [(D.AGG_SUM, [col(1), col(2), bop(O.OP_DIVIDE)])])
    assert ei.value.code == -4


# ---------------------------------------------------------------- modes
def test_partial_then_dfgpu_agg_final_equals_single(gpu_ctx):
    rng = np.random.default_rng(70)
    n = 100_000
    g = rng.integers(0, 3000, n).astype(np.int64)
    v = O.Dec(rng.integers(-10**12, 10**12, n).tolist(), 38, 4)
    f = rng.normal(0, 100, n)
    cols, types = [(g, None), (v, rng.random(n) > 0.1), (f, None)], [D.INT64, D.decimal128(38, 4), D.FLOAT64]
    aggs = [(D.AGG_MIN, [col(1)]), (D.AGG_SUM, [col(1)]), (D.AGG_AVG, [col(2)]), (D.AGG_COUNT_STAR, None)]
    single, _, _ = run_hash(gpu_ctx, cols, types, [0], aggs)
    h = None
    for lo, hi in ((0, 50_000), (50_000, n)):
        p = D.Pipeline(gpu_ctx, types)
        p.sink_aggregate_hash([0], [(fn, None if nd is None else gpu_nodes(D, nd)) for fn, nd in aggs], D.AGG_PARTIAL)
        push(gpu_ctx, p, [(c[0][lo:hi], None if c[1] is None else c[1][lo:hi]) for c in cols], types)
        p.finish()
        outs = p.drain(host=True)
        nc = outs[0].num_columns
        st = [outs[0].column(i).type for i in range(nc)]
        assert st == [D.INT64, D.decimal128(38, 4), D.decimal128(38, 4), D.UINT64, D.FLOAT64, D.INT64]
        if h is None:
            h = D.AggHandle(gpu_ctx, st, [0], [(D.AGG_MIN, 1, -1), (D.AGG_SUM, 2, -1), (D.AGG_AVG, 3, -1), (D.AGG_COUNT_STAR, 5, -1)], D.AGG_FINAL)
        for b in outs:
            h.push_host([D.HostColumn(*b.column_numpy(i), b.column(i).type) for i in range(nc)])
        p.close()
    h.finish()
    final, _ = drain_rows(h)
    h.close()
    want = as_map(single, 1)
    assert_groups(final, want, 1, "Partial + Final")


# ---------------------------------------------------------------- growth
def dec_lo(words):
    """Decimal128 words [n, 2] of values inside int64 -> int64"""
    w = np.asarray(words).reshape(-1, 2)
    lo = w[:, 0].view(np.int64)
    assert (w[:, 1].view(np.int64) == (lo >> 63)).all()
    return lo


def big_case(rng, n, ngroups):
    g = rng.permutation(n).astype(np.int64) % ngroups * 7919 - 10**9
    v = rng.integers(-10**12, 10**12, n).astype(np.int64)
    return g, v


def big_run(ctx, g, v, pushes, hint):
    """GROUP BY g: SUM(v), MIN(dec v), MAX(dec v), COUNT(*) -> DataFrame, metrics"""
    types = [D.INT64, D.INT64, D.decimal128(38, 2)]
    p = D.Pipeline(ctx, types)
    p.sink_aggregate_hash([0], [(D.AGG_SUM, gpu_nodes(D, [col(1)])), (D.AGG_MIN, gpu_nodes(D, [col(2)])), (D.AGG_MAX, gpu_nodes(D, [col(2)])),
                                (D.AGG_COUNT_STAR, None)], capacity_hint=hint)
    words = np.stack([v.view(np.uint64), (v >> 63).view(np.uint64)], axis=1)
    for s, e in pushes:
        p.push_host([D.HostColumn(g[s:e]), D.HostColumn(v[s:e]), D.HostColumn(np.ascontiguousarray(words[s:e]), None, types[2])])
    p.finish()
    parts = []
    for b in p.drain(host=True):
        c = [b.column_numpy(i)[0] for i in range(5)]
        parts.append(pd.DataFrame({"g": c[0], "sum": c[1], "min": dec_lo(c[2]), "max": dec_lo(c[3]), "cnt": c[4]}))
    m = {k: p.metric(k) for k in ("num_groups", "sink_rows", "group_rehashes", "replayed_rows")}
    p.close()
    return pd.concat(parts).sort_values("g").reset_index(drop=True), m


def big_want(g, v):
    df = pd.DataFrame({"g": g, "v": v}).groupby("g")["v"]
    return pd.DataFrame({"sum": df.sum(), "min": df.min(), "max": df.max(), "cnt": df.size()}).reset_index().sort_values("g").reset_index(drop=True)


def assert_frames(got, want):
    assert len(got) == len(want)
    for c in ("g", "sum", "min", "max", "cnt"):
        assert np.array_equal(got[c].to_numpy(np.int64), want[c].to_numpy(np.int64)), c


def test_growth_from_a_one_group_hint_in_one_push(gpu_ctx):
    rng = np.random.default_rng(80)
    n = 3_000_000
    g, v = big_case(rng, n, 2_000_000)
    got, m = big_run(gpu_ctx, g, v, [(0, n)], 1)
    assert m["group_rehashes"] > 0 and m["replayed_rows"] > 0
    assert m["sink_rows"] == n and m["num_groups"] == 2_000_000
    assert_frames(got, big_want(g, v))


def test_growth_across_several_pushes(gpu_ctx):
    rng = np.random.default_rng(81)
    n = 1_500_000
    g, v = big_case(rng, n, 600_000)
    g = np.sort(g)   # every push brings new groups
    got, m = big_run(gpu_ctx, g, v, [(s, min(n, s + 300_000)) for s in range(0, n, 300_000)], 0)
    assert m["group_rehashes"] > 0 and m["sink_rows"] == n
    assert_frames(got, big_want(g, v))


def test_ten_million_rows_racing_on_16_groups(gpu_ctx):
    rng = np.random.default_rng(82)
    n = 10_000_000
    g = rng.integers(0, 16, n).astype(np.int64) - 8
    v = rng.integers(-10**12, 10**12, n).astype(np.int64)
    got, m = big_run(gpu_ctx, g, v, [(0, n)], 0)
    assert m["group_rehashes"] == 0 and m["replayed_rows"] == 0 and m["sink_rows"] == n
    assert_frames(got, big_want(g, v))


# ---------------------------------------------------------------- rejections
def test_rejections(gpu_ctx):
    types = [D.INT64, D.INT64, D.FLOAT32, D.decimal128(15, 2)]
    maybe = D.Lookup(gpu_ctx, D.INT64, [], expected_rows=10, filter_only=True)
    p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_MAYBE, 0, maybe)])
    with pytest.raises(D.DfgpuError, match="MAYBE") as ei:
        p.sink_aggregate_hash([1], [(D.AGG_COUNT_STAR, None)])
    assert ei.value.code == -3
    p.close(); maybe.close()
    for mode in (D.AGG_FINAL, D.AGG_FINAL_PARTITIONED, D.AGG_PARTIAL_REDUCE):   # state merges are dfgpu_agg's
        p = D.Pipeline(gpu_ctx, types)
        with pytest.raises(D.DfgpuError, match="Single / SinglePartitioned / Partial") as ei:
            p.sink_aggregate_hash([1], [(D.AGG_COUNT_STAR, None)], mode)
        assert ei.value.code == -3
        p.close()
    cases = [([1], [(D.AGG_COUNT_STAR, None)] * 5, "0..4 aggregates"),
             ([1], [(D.AGG_MIN, [col(2)])], "Float32"),
             ([1], [(D.AGG_MAX, [col(2)])], "Float32"),
             ([3], [(D.AGG_COUNT_STAR, None)], "integer-like")]
    for group, aggs, msg in cases:
        p = D.Pipeline(gpu_ctx, types)
        with pytest.raises(D.DfgpuError, match=msg) as ei:
            p.sink_aggregate_hash(group, [(f, None if n is None else gpu_nodes(D, n)) for f, n in aggs])
        assert ei.value.code == -3
        p.close()


# ---------------------------------------------------------------- the operator twin
def test_twin_fuses_and_matches_the_unfused_plan(gpu_ctx):
    from datafusion_b200.exec import GpuPipelineExec, collect, fuse_hash_aggregates
    from test_fusion_rule_hash_planning import q15_plan, q3_by_customer_plan
    rng = np.random.default_rng(90)
    plans = [q15_plan(rng, n=200_000, nsupp=20_000), q15_plan(rng, mode="SinglePartitioned", n=50_000, nsupp=3000),
             q3_by_customer_plan(rng, nord=30_000, n=200_000, ncust=3000)]
    for plan in plans:
        fused = fuse_hash_aggregates(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash"
        got = pa.Table.from_batches(collect(fused)).to_pandas()
        want = pa.Table.from_batches(collect(plan)).to_pandas()
        assert len(want) > 1000
        keys = list(want.columns[:len(plan.group_by)])
        got = got.sort_values(keys).reset_index(drop=True)
        want = want.sort_values(keys).reset_index(drop=True)
        pd.testing.assert_frame_equal(got, want, check_dtype=True)
