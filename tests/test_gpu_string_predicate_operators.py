"""String comparisons and IN lists through plan_string_predicates and the fusion rules on the GPU, each against a plain reference of its
plan: TPC-H Q3 with a real Utf8View c_mktsegment gives the integer-coded Q3 plan's rows; Q12's `l_shipmode IN ('MAIL', 'SHIP')` filter
feeds a fused aggregate; one Q19 arm's string conjuncts on both sides of the join feed a fused aggregate; the masks in collect() of a
filter over every layout and dictionary codes."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_b200.exec import (AggregateExpr, DictionaryEncodeExec, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuLikeExec, GpuPipelineExec,
                                  InListExpr, LikeExpr, MemoryExec, SessionConfig, TaskContext, col, collect, fuse_pipelines, lit,
                                  plan_string_dictionary, plan_string_predicates)
from test_gpu_tpch_q3 import gen_tables, q3_expected, q3_plan

pytestmark = pytest.mark.gpu

SEGMENTS = ["AUTOMOBILE", "BUILDING", "FURNITURE", "MACHINERY", "HOUSEHOLD"]
MODES = ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"]
INSTRUCT = ["DELIVER IN PERSON", "COLLECT COD", "NONE", "TAKE BACK RETURN"]
CONTAINERS = [f"{a} {b}" for a in ("SM", "MED", "LG", "JUMBO", "WRAP") for b in ("CASE", "BOX", "BAG", "JAR", "PKG", "PACK", "CAN", "DRUM")]


def mem(t, chunk=5000):
    return MemoryExec(t.to_batches(max_chunksize=chunk), t.schema)


def rows(plan, tc):
    return sorted(tuple(r.values()) for b in collect(plan, tc) for r in b.to_pylist())


@pytest.mark.parametrize("t", [pa.string(), pa.string_view(), "dictionary"], ids=str)
def test_q3_with_a_utf8_mktsegment(gpu_ctx, t):
    customer, orders, lineitem = gen_tables(0.02)
    seg = pa.array(np.array(SEGMENTS, object)[np.asarray(customer["c_mktsegment"])], pa.string())   # code 1 = 'BUILDING'
    text = customer.set_column(1, "c_mktsegment", seg if t == "dictionary" else seg.cast(t))
    _, coded = q3_plan(customer, orders, lineitem, 4000)
    _, plan = q3_plan(text, orders, lineitem, 4000)
    c = plan.input.input.left.input.left                                  # the customer filter
    src = DictionaryEncodeExec(c.input, plan_string_dictionary()) if t == "dictionary" else c.input
    c.predicate, c.input = col("c_mktsegment") == lit("BUILDING"), src
    tc = TaskContext(SessionConfig(), gpu_ctx)
    planned = plan_string_predicates(plan)
    fused = fuse_pipelines(planned)
    assert isinstance(fused, GpuPipelineExec) and fused.schema == plan.schema
    build = fused.scan.stages[0][2]
    assert isinstance(build.scan.stages[0][2].scan.source, GpuLikeExec)
    exp = q3_expected(customer, orders, lineitem)
    norm = lambda rs: sorted((a, b if isinstance(b, int) else (b - pd.Timestamp(0).date()).days, c_, d) for a, b, c_, d in rs)  # noqa: E731
    assert len(exp) > 0
    assert norm(rows(planned, tc)) == norm(rows(fused, tc)) == norm(rows(fuse_pipelines(coded), tc)) == exp


def lineitem_q12_q19(rng, n, n_part):
    return pa.table({"l_orderkey": rng.integers(1, 3000, n).astype(np.int64), "l_partkey": rng.integers(1, n_part + 1, n).astype(np.int64),
                     "l_quantity": rng.integers(1, 51, n).astype(np.int64), "l_price": rng.integers(100, 10000, n).astype(np.int64),
                     "l_shipmode": pa.array(np.array(MODES, object)[rng.integers(0, len(MODES), n)], pa.string()),
                     "l_shipinstruct": pa.array(np.array(INSTRUCT, object)[rng.integers(0, len(INSTRUCT), n)], pa.string_view()),
                     "l_late": rng.integers(0, 2, n).astype(np.int32)})


def test_q12_ship_mode_filter_feeds_a_fused_aggregate(gpu_ctx):
    """SUM(l_price), COUNT(*) per l_late over lineitem WHERE l_shipmode IN ('MAIL', 'SHIP') AND l_quantity < 40"""
    rng = np.random.default_rng(1)
    li = lineitem_q12_q19(rng, 60000, 100).drop(["l_shipinstruct"])     # a string column nothing reads cannot pass through a filter
    f = GpuFilterExec(InListExpr(col("l_shipmode"), ["MAIL", "SHIP"]) & (col("l_quantity") < lit(40)), mem(li), projection=[3, 5])
    agg = GpuAggregateExec("Single", ["l_late"], [AggregateExpr("sum", "l_price", "s"), AggregateExpr("count_star", None, "n")], f)
    planned = plan_string_predicates(agg)
    fused = fuse_pipelines(planned)
    assert isinstance(fused, GpuPipelineExec) and isinstance(fused.scan.source, GpuLikeExec)
    d = li.to_pandas()
    d = d[d.l_shipmode.isin(["MAIL", "SHIP"]) & (d.l_quantity < 40)]
    g = d.groupby("l_late").agg(s=("l_price", "sum"), n=("l_price", "size")).reset_index()
    exp = sorted((int(a), int(b), int(c)) for a, b, c in g.itertuples(index=False))
    tc = TaskContext(SessionConfig(), gpu_ctx)
    assert len(exp) == 2 and rows(planned, tc) == exp and rows(fused, tc) == exp


def test_q19_arm_string_conjuncts_feed_a_fused_aggregate(gpu_ctx):
    """part WHERE p_brand = 'Brand#12' AND p_container IN ('SM CASE', 'SM BOX', 'SM PACK', 'SM PKG') AND p_size <= 25, INNER JOIN lineitem
    WHERE l_shipinstruct = 'DELIVER IN PERSON' AND l_shipmode IN ('AIR', 'REG AIR') AND l_quantity <= 30, SUM(l_price) per l_partkey
    (wider size and quantity ranges than Q19's, so that the small tables leave some rows)"""
    rng = np.random.default_rng(2)
    n_part = 20000
    part = pa.table({"p_partkey": np.arange(1, n_part + 1, dtype=np.int64),
                     "p_brand": pa.array([f"Brand#{a}{b}" for a, b in rng.integers(1, 6, (n_part, 2))], pa.string_view()),
                     "p_container": pa.array(np.array(CONTAINERS, object)[rng.integers(0, len(CONTAINERS), n_part)], pa.large_string()),
                     "p_size": rng.integers(1, 51, n_part).astype(np.int32)})
    li = lineitem_q12_q19(rng, 400000, n_part)
    pf = GpuFilterExec((col("p_brand") == lit("Brand#12")) & InListExpr(col("p_container"), ["SM CASE", "SM BOX", "SM PACK", "SM PKG"])
                       & (col("p_size") <= lit(25, pa.int32())), mem(part), projection=[0])
    lf = GpuFilterExec((lit("DELIVER IN PERSON") == col("l_shipinstruct")) & InListExpr(col("l_shipmode"), ["AIR", "REG AIR"])
                       & (col("l_quantity") <= lit(30)), mem(li), projection=[1, 3])
    join = GpuHashJoinExec(pf, lf, [("p_partkey", "l_partkey")], "Inner")
    agg = GpuAggregateExec("Single", ["l_partkey"], [AggregateExpr("sum", "l_price", "revenue")], join)
    planned = plan_string_predicates(agg)
    fused = fuse_pipelines(planned)
    assert isinstance(fused, GpuPipelineExec) and isinstance(fused.scan.source, GpuLikeExec)
    assert isinstance(fused.scan.stages[0][2].scan.source, GpuLikeExec)
    p, d = part.to_pandas(), li.to_pandas()
    p = p[(p.p_brand == "Brand#12") & p.p_container.isin(["SM CASE", "SM BOX", "SM PACK", "SM PKG"]) & (p.p_size <= 25)]
    d = d[(d.l_shipinstruct == "DELIVER IN PERSON") & d.l_shipmode.isin(["AIR", "REG AIR"]) & (d.l_quantity <= 30)]
    g = d.merge(p, left_on="l_partkey", right_on="p_partkey").groupby("l_partkey").l_price.sum()
    exp = sorted((int(k), int(v)) for k, v in g.items())
    tc = TaskContext(SessionConfig(), gpu_ctx)
    assert len(exp) > 0 and rows(planned, tc) == exp and rows(fused, tc) == exp


@pytest.mark.parametrize("t", [pa.string(), pa.large_string(), pa.string_view(), "dictionary"], ids=str)
def test_collect_filter_with_string_predicates(gpu_ctx, t):
    rng = np.random.default_rng(3)
    n = 30000
    s = pa.array(np.array(MODES + [None], object)[rng.integers(0, len(MODES) + 1, n)], pa.string())
    x = rng.integers(0, 100, n).astype(np.int64)
    tab = pa.table({"k": np.arange(n, dtype=np.int64), "s": s if t == "dictionary" else s.cast(t), "x": x})
    src = mem(tab)
    if t == "dictionary":
        src = DictionaryEncodeExec(src, plan_string_dictionary())
    tc = TaskContext(SessionConfig(), gpu_ctx)
    null = pa.scalar(None, pa.bool_())
    for pred, ref in (((col("s") >= lit("RAIL")) & (col("x") > lit(30)), pc.and_kleene(pc.greater_equal(s, "RAIL"), pc.greater(tab["x"], 30))),
                      (~InListExpr(col("s"), ["MAIL", None]) | (col("x") < lit(5)),
                       pc.or_kleene(pc.invert(pc.or_kleene(pc.equal(s, "MAIL"), null)), pc.less(tab["x"], 5))),
                      (InListExpr(col("s"), ["AIR", "FOB", None], negated=True) | (col("x") < lit(5)),
                       pc.or_kleene(pc.and_kleene(pc.invert(pc.is_in(s, value_set=pa.array(["AIR", "FOB"]))), null), pc.less(tab["x"], 5))),
                      ((lit("SHIP") > col("s")) & LikeExpr(col("s"), "%AIR"), pc.and_kleene(pc.less(s, "SHIP"), pc.match_like(s, "%AIR")))):
        plan = plan_string_predicates(GpuFilterExec(pred, src, projection=[0, 2]))
        assert isinstance(plan.input, GpuLikeExec)
        got = pa.Table.from_batches(collect(plan, tc), plan.schema)
        exp = tab.select(["k", "x"]).filter(ref)
        assert got.column("k").to_pylist() == exp.column("k").to_pylist() and got.column("x").to_pylist() == exp.column("x").to_pylist()
