"""The fused pipeline's dense-group aggregate sink (dfgpu_pipeline_sink_aggregate_dense): filter [-> probe stages] -> GROUP BY keys in
small declared domains, in one kernel.  Every result is compared with the oracle's UNFUSED chain (filter_batch -> eval_expr ->
group_by / scalar_aggregate, with MIN / MAX / AVG over Decimal128 from decimal_agg): integers and decimals bit-exact, Float64 within 1e-9 relative.  The shapes are TPC-H Q1 (4 SUMs, 3 AVGs,
COUNT(*) by l_returnflag, l_linestatus), Q6 (no GROUP BY) and Q4 (a semi probe feeding COUNT(*) by o_orderpriority), with Int64 and
Decimal128(15,2) money."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import decimal_agg as DA
from decimal_util import col_as_py, gpu_col_as_py, gpu_host_col, gpu_nodes
from harness import split_points

pytestmark = pytest.mark.gpu
F = {D.AGG_SUM: O.A_SUM, D.AGG_COUNT: O.A_COUNT, D.AGG_MIN: O.A_MIN, D.AGG_MAX: O.A_MAX, D.AGG_AVG: O.A_AVG, D.AGG_COUNT_STAR: O.A_COUNT_STAR}
CUT = 2300


def col(i): return (O.E_COLUMN, i, None, 0, 0)
def lit(v, dt): return (O.E_LITERAL, 0, dt, 0, v)
def dlit(v, p, s): return (O.E_LITERAL, 0, O.decimal_dtype(p, s), 0, v)
def bop(op): return (O.E_BINARY, op, None, 0, 0)
def f64(i): return [col(i), (O.E_CAST, 0, np.float64, 0, 0)]


def push_cols(ctx, p, cols, types, batch_rows, device, keep):
    for s, e in split_points(len(cols[0][0]), batch_rows):
        hc = [gpu_host_col(D, (c[0][s:e], None if c[1] is None else c[1][s:e]), t) for c, t in zip(cols, types)]
        if device:
            dc = [D.DeviceColumn.from_host(ctx, h) for h in hc]
            keep.append(dc)
            p.push_device(dc)
        else:
            p.push_host(hc)


def run_dense(ctx, cols, types, pred, group_cols, key_range, aggs, mode=D.AGG_SINGLE, batch_rows=None, device=False, stages=(), batch_size=0):
    """the fused pipeline -> (rows as tuples of Python values in output order, output type codes, metrics)"""
    p = D.Pipeline(ctx, types, gpu_nodes(D, pred) if pred else None, stages)
    p.sink_aggregate_dense(group_cols, key_range, [(f, gpu_nodes(D, n) if n else None) for f, n in aggs], mode, batch_size)
    keep = []
    if len(cols[0][0]):
        push_cols(ctx, p, cols, types, batch_rows, device, keep)
    p.finish()
    outs = p.drain(host=True)
    rows, otypes = [], []
    for b in outs:
        cs = [gpu_col_as_py(D, b, i) for i in range(b.num_columns)]
        otypes = [t for _, t in cs]
        rows += list(zip(*[v for v, _ in cs]))
    m = {k: p.metric(k) for k in ("num_groups", "input_rows", "sink_rows", "output_rows", "dense_block_launches")}
    m["batches"] = len(outs)
    p.close()
    return rows, otypes, m


def oracle_dense(cols, pred, group_cols, aggs, state=False):
    """the unfused chain -> rows in slot order (ascending keys, NULL after the values)"""
    f = O.filter_batch(cols, O.eval_expr(cols, pred)) if pred else list(cols)
    n = len(f[0][0])
    args = [O.eval_expr(f, nodes) if nodes else None for _, nodes in aggs]
    if not group_cols:
        res = DA.scalar_aggregate([(F[fn], a, None, n) for (fn, _), a in zip(aggs, args)], state=state)
        return [tuple(col_as_py(c)[0] for c in res)]
    keys, res = DA.group_by([f[g] for g in group_cols], [(F[fn], a, None) for (fn, _), a in zip(aggs, args)])
    out = list(keys)
    for (fn, _), a, r in zip(aggs, args, res):
        out += DA.agg_output_columns(F[fn], r, None if a is None else (object if isinstance(a[0], O.Dec) else np.asarray(a[0]).dtype), state)
    rows = list(zip(*[col_as_py(c) for c in out])) if out and len(out[0][0]) else []
    nk = len(group_cols)
    return sorted(rows, key=lambda r: tuple((1, 0) if v is None else (0, v) for v in r[:nk]))


def assert_rows(got, want, what=""):
    assert len(got) == len(want), f"{what}: {len(got)} rows, expected {len(want)}"
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w), what
        for j, (a, b) in enumerate(zip(g, w)):
            if isinstance(b, float) and a is not None:
                assert a == pytest.approx(b, rel=1e-9, abs=0), f"{what}: row {i} col {j}: {a} != {b}"
            else:
                assert a == b, f"{what}: row {i} col {j}: {a!r} != {b!r}"


# ---- TPC-H lineitem-shaped columns: 0 l_returnflag (code 0..2), 1 l_linestatus (0..1), 2 l_shipdate, 3 l_quantity, 4 l_extendedprice,
#      5 l_discount, 6 l_tax; money in cents (Int64) or Decimal128(15,2) ----
def lineitem(rng, n, decimal, nulls):
    rf = (rng.integers(0, 3, n).astype(np.int32), (rng.random(n) > 0.01) if nulls else None)
    ls = (rng.integers(0, 2, n).astype(np.int8), None)
    ship = (rng.integers(0, 2500, n).astype(np.int32), None)
    qty = rng.integers(1, 51, n) * 100
    price = rng.integers(90_000, 10_495_000, n)
    disc, tax = rng.integers(0, 11, n), rng.integers(0, 9, n)
    qv = (rng.random(n) > 0.02) if nulls else None
    if decimal:
        money = [(O.Dec(qty.tolist(), 15, 2), qv)] + [(O.Dec(v.tolist(), 15, 2), None) for v in (price, disc, tax)]
        mt = [D.decimal128(15, 2)] * 4
    else:
        money = [(qty, qv), (price, None), (disc, None), (tax, None)]
        mt = [D.INT64] * 4
    return [rf, ls, ship] + money, [D.INT32, D.INT8, D.DATE32] + mt


def q1_aggs(decimal):
    if decimal:   # price * (1 - disc), price * (1 - disc) * (1 + tax): Decimal128(38,4), Decimal128(38,6)
        disc_price = [col(4), dlit(1, 20, 0), col(5), bop(O.OP_MINUS), bop(O.OP_MULTIPLY)]
        charge = disc_price + [dlit(1, 20, 0), col(6), bop(O.OP_PLUS), bop(O.OP_MULTIPLY)]
        avg = lambda i: [col(i)]
    else:         # cents: price * (100 - disc), price * (100 - disc) * (100 + tax)
        disc_price = [col(4), lit(100, np.int64), col(5), bop(O.OP_MINUS), bop(O.OP_MULTIPLY)]
        charge = disc_price + [lit(100, np.int64), col(6), bop(O.OP_PLUS), bop(O.OP_MULTIPLY)]
        avg = f64
    return [(D.AGG_SUM, [col(3)]), (D.AGG_SUM, [col(4)]), (D.AGG_SUM, disc_price), (D.AGG_SUM, charge),
            (D.AGG_AVG, avg(3)), (D.AGG_AVG, avg(4)), (D.AGG_AVG, avg(5)), (D.AGG_COUNT_STAR, None)]


Q1_PRED = [col(2), lit(CUT, np.int32), bop(O.OP_LTEQ)]


@pytest.mark.parametrize("decimal", [False, True], ids=["int64_money", "decimal_money"])
@pytest.mark.parametrize("device,batch_rows", [(False, None), (True, 33_333), (False, 50_001)])
def test_q1_shape_matches_unfused_chain(gpu_ctx, decimal, device, batch_rows):
    rng = np.random.default_rng(11)
    cols, types = lineitem(rng, 120_007, decimal, nulls=True)
    aggs = q1_aggs(decimal)
    got, ot, m = run_dense(gpu_ctx, cols, types, Q1_PRED, [0, 1], [(0, 2), (0, 1)], aggs, device=device, batch_rows=batch_rows, batch_size=5)
    want = oracle_dense(cols, Q1_PRED, [0, 1], aggs)
    assert_rows(got, want, "q1")
    assert len(got) == 8 and any(r[0] is None for r in got)     # three flags and NULL x two statuses
    assert m["num_groups"] == 8 and m["output_rows"] == 8 and m["batches"] == 2 and m["input_rows"] == 120_007
    assert m["sink_rows"] == sum(r[-1] for r in got)
    if decimal:
        assert ot[2:] == [D.decimal128(25, 2), D.decimal128(25, 2), D.decimal128(38, 4), D.decimal128(38, 6),
                          D.decimal128(19, 6), D.decimal128(19, 6), D.decimal128(19, 6), D.INT64]


@pytest.mark.parametrize("decimal", [False, True], ids=["int64_money", "decimal_money"])
def test_q1_shape_partial_states(gpu_ctx, decimal):
    """Partial mode: the state columns dfgpu_agg emits (AVG over Float64 -> [count, sum]); AVG over Decimal128 is Single-only"""
    rng = np.random.default_rng(12)
    cols, types = lineitem(rng, 60_001, decimal, nulls=False)
    aggs = q1_aggs(decimal)
    if decimal:
        aggs = [a for a in aggs if a[0] != D.AGG_AVG] + [(D.AGG_MIN, [col(4)]), (D.AGG_MAX, [col(4)])]
        with pytest.raises(D.DfgpuError) as ei:
            run_dense(gpu_ctx, cols, types, Q1_PRED, [0, 1], [(0, 2), (0, 1)], q1_aggs(True), mode=D.AGG_PARTIAL)
        assert ei.value.code == -3
    got, _, _ = run_dense(gpu_ctx, cols, types, Q1_PRED, [0, 1], [(0, 2), (0, 1)], aggs, mode=D.AGG_PARTIAL, batch_rows=20_000)
    assert_rows(got, oracle_dense(cols, Q1_PRED, [0, 1], aggs, state=True), "q1 partial")


def q6(decimal):
    pred = [col(2), lit(400, np.int32), bop(O.OP_GTEQ), col(2), lit(765, np.int32), bop(O.OP_LT), bop(O.OP_AND)]
    if decimal:
        pred += [col(5), dlit(5, 15, 2), bop(O.OP_GTEQ), bop(O.OP_AND), col(5), dlit(7, 15, 2), bop(O.OP_LTEQ), bop(O.OP_AND),
                 col(3), dlit(2400, 15, 2), bop(O.OP_LT), bop(O.OP_AND)]
    else:
        pred += [col(5), lit(5, np.int64), bop(O.OP_GTEQ), bop(O.OP_AND), col(5), lit(7, np.int64), bop(O.OP_LTEQ), bop(O.OP_AND),
                 col(3), lit(2400, np.int64), bop(O.OP_LT), bop(O.OP_AND)]
    return pred, [(D.AGG_SUM, [col(4), col(5), bop(O.OP_MULTIPLY)]), (D.AGG_COUNT_STAR, None)]


@pytest.mark.parametrize("decimal", [False, True], ids=["int64_money", "decimal_money"])
def test_q6_shape_and_empty_inputs(gpu_ctx, decimal):
    rng = np.random.default_rng(13)
    cols, types = lineitem(rng, 200_003, decimal, nulls=False)
    pred, aggs = q6(decimal)
    got, _, m = run_dense(gpu_ctx, cols, types, pred, [], [], aggs, batch_rows=70_000, device=True)
    want = oracle_dense(cols, pred, [], aggs)
    assert_rows(got, want, "q6")
    assert got[0][1] > 500 and m["num_groups"] == 1 and m["output_rows"] == 1
    # empty input and a predicate that rejects every row: exactly one row, COUNT 0, SUM NULL
    empty = [(c[0][:0], None) for c in cols]
    for cs, pr in ((empty, pred), (cols, [col(2), lit(-1, np.int32), bop(O.OP_LT)])):
        got, _, m = run_dense(gpu_ctx, cs, types, pr, [], [], aggs)
        assert got == [(None, 0)] == oracle_dense(cs, pr, [], aggs)
        assert m["output_rows"] == 1


def test_q4_shape_semi_stage_and_payload_group_key(gpu_ctx):
    """orders -> RightSemi probe of the late lineitem keys -> COUNT(*) GROUP BY o_orderpriority; and an INNER stage's payload field
    (the customer's nation) as the group key"""
    rng = np.random.default_rng(14)
    no = 150_000
    okey = rng.permutation(no).astype(np.int64) + 1
    odate = rng.integers(0, 2500, no).astype(np.int32)
    prio = rng.integers(1, 6, no).astype(np.int32)
    cust = rng.integers(1, 5001, no).astype(np.int64)
    price = rng.integers(1000, 500_000, no).astype(np.int64)
    late = np.unique(rng.choice(okey, 60_000))
    lk = D.Lookup(gpu_ctx, D.INT64, [], expected_rows=len(late))
    bp = D.Pipeline(gpu_ctx, [D.INT64])
    bp.sink_build(lk, 0, [])
    bp.push_host([D.HostColumn(late, None, D.INT64)]); bp.finish(); bp.close()
    cols, types = [(okey, None), (odate, None), (prio, None), (cust, None), (price, None)], [D.INT64, D.DATE32, D.INT32, D.INT64, D.INT64]
    pred = [col(1), lit(1000, np.int32), bop(O.OP_GTEQ), col(1), lit(1092, np.int32), bop(O.OP_LT), bop(O.OP_AND)]
    got, _, _ = run_dense(gpu_ctx, cols, types, pred, [2], [(1, 5)], [(D.AGG_COUNT_STAR, None)], stages=[(D.STAGE_SEMI, 0, lk)], batch_rows=64_000)
    sel = (odate >= 1000) & (odate < 1092) & np.isin(okey, late)
    want = [(k, int((prio[sel] == k).sum())) for k in range(1, 6)]
    assert got == want and all(c > 100 for _, c in want)
    # nation of the customer: an INNER stage with an Int32 payload, grouped on the payload field (virtual column 5)
    nation = rng.integers(0, 25, 5000).astype(np.int32)
    cl = D.Lookup(gpu_ctx, D.INT64, [D.INT32], expected_rows=5000)
    bp = D.Pipeline(gpu_ctx, [D.INT64, D.INT32])
    bp.sink_build(cl, 0, [1])
    bp.push_host([D.HostColumn(np.arange(1, 5001, dtype=np.int64), None, D.INT64), D.HostColumn(nation, None, D.INT32)]); bp.finish(); bp.close()
    got, _, _ = run_dense(gpu_ctx, cols, types, pred, [5, 2], [(0, 24), (1, 5)], [(D.AGG_SUM, [col(4)]), (D.AGG_COUNT_STAR, None)],
                          stages=[(D.STAGE_INNER, 3, cl)], device=True)
    n_of = nation[cust - 1]
    sel = (odate >= 1000) & (odate < 1092)
    want = []
    for nk in range(25):
        for pk in range(1, 6):
            m = sel & (n_of == nk) & (prio == pk)
            if m.any():
                want.append((nk, pk, int(price[m].sum()), int(m.sum())))
    assert got == want
    lk.close(); cl.close()


def test_min_max_over_int64_date32_float64_decimal_with_negatives(gpu_ctx):
    rng = np.random.default_rng(15)
    n = 80_000
    g = (rng.integers(-3, 4, n).astype(np.int16), rng.random(n) > 0.05)
    i64 = (rng.integers(-10 ** 15, 10 ** 15, n), rng.random(n) > 0.1)
    d32 = (rng.integers(-20_000, 20_000, n).astype(np.int32), None)
    fl = (rng.standard_normal(n) * 1e6, rng.random(n) > 0.1)
    dec = (O.Dec([int(x) * 10 ** 18 + int(y) for x, y in zip(rng.integers(-10 ** 9, 10 ** 9, n), rng.integers(0, 10 ** 18, n))], 38, 3), rng.random(n) > 0.1)
    cols, types = [g, i64, d32, fl, dec], [D.INT16, D.INT64, D.DATE32, D.FLOAT64, D.decimal128(38, 3)]
    aggs = [(fn, [col(c)]) for c in range(1, 5) for fn in (D.AGG_MIN, D.AGG_MAX)] + [(D.AGG_COUNT, [col(4)])]
    with pytest.raises(D.DfgpuError) as ei:   # nine aggregates
        run_dense(gpu_ctx, cols, types, None, [0], [(-3, 3)], aggs)
    assert ei.value.code == -3
    aggs = aggs[:8]
    got, ot, _ = run_dense(gpu_ctx, cols, types, None, [0], [(-3, 3)], aggs, batch_rows=30_000)
    assert_rows(got, oracle_dense(cols, None, [0], aggs), "min/max")
    assert ot == [D.INT16, D.INT64, D.INT64, D.DATE32, D.DATE32, D.FLOAT64, D.FLOAT64, D.decimal128(38, 3), D.decimal128(38, 3)]
    assert len(got) == 8 and any(r[1] < 0 for r in got) and any(r[7] < 0 for r in got)


def test_domain_edges(gpu_ctx):
    rng = np.random.default_rng(16)
    n = 50_000
    a = (rng.integers(0, 15, n).astype(np.int32), rng.random(n) > 0.03)
    b = (rng.integers(100, 115, n).astype(np.int64), rng.random(n) > 0.03)
    v = (rng.integers(-1000, 1000, n), None)
    cols, types = [a, b, v], [D.INT32, D.INT64, D.INT64]
    aggs = [(D.AGG_SUM, [col(2)]), (D.AGG_COUNT_STAR, None)]
    # exactly 256 slots: 16 x 16 (15 values + NULL each)
    got, _, m = run_dense(gpu_ctx, cols, types, None, [0, 1], [(0, 14), (100, 114)], aggs)
    assert_rows(got, oracle_dense(cols, None, [0, 1], aggs), "256 slots")
    assert m["num_groups"] == 256
    # a one-value domain: the value and NULL
    one = [((a[0] * 0 + 7).astype(np.int32), a[1]), v]
    one_aggs = [(D.AGG_SUM, [col(1)]), (D.AGG_COUNT_STAR, None)]
    got, _, _ = run_dense(gpu_ctx, one, [D.INT32, D.INT64], None, [0], [(7, 7)], one_aggs)
    assert_rows(got, oracle_dense(one, None, [0], one_aggs), "one value")
    assert [r[0] for r in got] == [7, None]
    # 257 slots, a key outside its range, a MAYBE stage
    with pytest.raises(D.DfgpuError) as ei:
        run_dense(gpu_ctx, cols, types, None, [1], [(0, 255)], aggs)
    assert ei.value.code == -3
    with pytest.raises(D.DfgpuError) as ei:
        run_dense(gpu_ctx, cols, types, None, [0], [(0, 13)], aggs)
    assert ei.value.code == -1
    flt = D.Lookup(gpu_ctx, D.INT64, [], expected_rows=100, filter_only=True)
    with pytest.raises(D.DfgpuError) as ei:
        run_dense(gpu_ctx, cols, types, None, [0], [(0, 14)], aggs, stages=[(D.STAGE_MAYBE, 1, flt)])
    assert ei.value.code == -3
    flt.close()


def test_decimal_avg_overflowing_the_target_precision_is_an_error(gpu_ctx):
    """AVG(Decimal128(38,0)) -> Decimal128(38,4): sum * 10^4 overflows i128 -> "Arithmetic Overflow in AvgAccumulator" (DFGPU_ERR_ARITH);
    a value that fits i128 but not 38 digits after the division fails the precision check the same way"""
    for vals in ([10 ** 37, 10 ** 37], [12 * 10 ** 33]):
        cols = [(np.zeros(len(vals), np.int32), None), (O.Dec(vals, 38, 0), None)]
        with pytest.raises(O.ArrowArithmeticOverflow):
            oracle_dense(cols, None, [0], [(D.AGG_AVG, [col(1)])])
        with pytest.raises(D.DfgpuError) as ei:
            run_dense(gpu_ctx, cols, [D.INT32, D.decimal128(38, 0)], None, [0], [(0, 0)], [(D.AGG_AVG, [col(1)])])
        assert ei.value.code == -4


def test_fused_exec_plan_equals_the_unfused_operators(gpu_ctx):
    """exec.py: fuse_pipelines turns the Q1 plan (Int64 money) into a dense GpuPipelineExec; it returns what
    GpuAggregateExec(GpuProjectionExec(GpuFilterExec)) returns"""
    import pyarrow as pa
    import test_fusion_rule_dense_planning as P
    from datafusion_b200.exec import GpuPipelineExec, TaskContext, collect, fuse_pipelines
    agg = P.q1(False, src=P.lineitem(False, n=300_011))
    fused = fuse_pipelines(agg)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "dense"
    tctx = TaskContext(ctx=gpu_ctx)
    keys = [("l_returnflag", "ascending"), ("l_linestatus", "ascending")]
    got = pa.Table.from_batches(collect(fused, tctx), schema=agg.schema).sort_by(keys)
    want = pa.Table.from_batches(collect(agg, tctx), schema=agg.schema).sort_by(keys)
    assert got.num_rows == want.num_rows == 6 and fused.metrics()["num_groups"] == 6
    for name in agg.schema.names:
        g, w = got.column(name).to_pylist(), want.column(name).to_pylist()
        if pa.types.is_floating(agg.schema.field(name).type):
            assert g == pytest.approx(w, rel=1e-9), name
        else:
            assert g == w, name
