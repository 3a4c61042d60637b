"""The LIKE mask through the operators on the GPU: in dfgpu_filter beside an integer comparison, collect() of a twin FilterExec with
LikeExpr over every string layout and dictionary codes, TPC-H Q13 with `o_comment NOT LIKE '%special%requests%'` over Utf8 text (fused
and unfused, against pandas), and Q9's `p_name LIKE '%green%'` on the build side of an INNER stage (against pandas)."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, DictionaryEncodeExec, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuLikeExec, GpuPipelineExec,
                                  GpuProjectionExec, LikeExpr, MemoryExec, TaskContext, col, collect, fuse_pipelines, lit, plan_like_predicates,
                                  plan_string_dictionary)
from like_oracle import like

pytestmark = pytest.mark.gpu

VOCAB = ["special", "requests", "deposits", "packages", "furiously", "final", "ironic", "green", "forest", "blithely", "accounts", "pinto", "beans"]


@pytest.fixture(scope="module")
def ctx():
    c = D.Context(0)
    yield c
    c.close()


def comments(rng, n, null_p=0.0):
    out = []
    for _ in range(n):
        if rng.random() < null_p:
            out.append(None)
            continue
        words = list(rng.choice(VOCAB, int(rng.integers(3, 9))))
        out.append(" ".join(words))
    return out


def mem(t, chunk=7000):
    return MemoryExec(t.to_batches(max_chunksize=chunk), t.schema)


def test_mask_in_dfgpu_filter(ctx):
    """s NOT LIKE p AND x > c, with the mask as an ordinary UINT8 input column of dfgpu_filter"""
    rng = np.random.default_rng(1)
    s = pa.array(comments(rng, 20000, null_p=0.1))
    x = rng.integers(0, 100, 20000).astype(np.int64)
    mask = D.like(ctx, s, "%special%requests%", negated=True)
    nodes = [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.UINT8, 0, 1, 0.0), (D.EXPR_BINARY, D.OP_EQ, 0, 0, 0, 0.0),
             (D.EXPR_COLUMN, 1, 0, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.INT64, 0, 40, 0.0), (D.EXPR_BINARY, D.OP_GT, 0, 0, 0, 0.0),
             (D.EXPR_BINARY, D.OP_AND, 0, 0, 0, 0.0)]
    f = D.FilterHandle(ctx, [D.UINT8, D.INT64], nodes, [1], batch_size=0)
    f.push_device([mask, D.DeviceColumn.from_host(ctx, D.HostColumn(x))])
    f.finish()
    got = np.concatenate([b.column_numpy(0)[0] for b in f.drain(host=True)] or [np.zeros(0, np.int64)])
    f.close()
    exp = x[np.array([e is True for e in like(s.to_pylist(), "%special%requests%", True)]) & (x > 40)]
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("t", [pa.string(), pa.large_string(), pa.string_view(), "dictionary"], ids=str)
def test_collect_filter_with_like(ctx, t):
    rng = np.random.default_rng(2)
    n = 30000
    s = pa.array(comments(rng, n, null_p=0.05))
    x = rng.integers(0, 100, n).astype(np.int64)
    tab = pa.table({"k": np.arange(n, dtype=np.int64), "s": s if t == "dictionary" else s.cast(t), "x": x})
    src = mem(tab)
    if t == "dictionary":
        src = DictionaryEncodeExec(src, plan_string_dictionary())
    tc = TaskContext(ctx=ctx)
    for pred, ref in ((LikeExpr(col("s"), "%special%requests%", negated=True) & (col("x") > lit(30)),
                       pc.and_kleene(pc.invert(pc.match_like(s, "%special%requests%")), pc.greater(tab["x"], 30))),
                      (LikeExpr(col("s"), "furiously%") | ~LikeExpr(col("s"), "%green_%"),
                       pc.or_kleene(pc.match_like(s, "furiously%"), pc.invert(pc.match_like(s, "%green_%"))))):
        plan = plan_like_predicates(GpuFilterExec(pred, src, projection=[0, 2]))
        assert isinstance(plan.input, GpuLikeExec)
        got = pa.Table.from_batches(collect(plan, tc), plan.schema)
        exp = tab.select(["k", "x"]).filter(ref)
        assert got.column("k").to_pylist() == exp.column("k").to_pylist() and got.column("x").to_pylist() == exp.column("x").to_pylist()


def test_q13_with_the_real_predicate(ctx):
    """customer LEFT JOIN orders ON c_custkey = o_custkey AND o_comment NOT LIKE '%special%requests%', count(o_orderkey) per customer,
    then count(*) per c_count; o_comment is Utf8 text"""
    rng = np.random.default_rng(3)
    n_cust, n_ord = 3000, 30000
    ck = np.arange(1, n_cust + 1, dtype=np.int64)
    active = ck[ck % 3 != 0]
    ocust = active[rng.integers(0, len(active), n_ord)]
    okey = np.arange(1, n_ord + 1, dtype=np.int64)
    ocomment = comments(rng, n_ord)
    customer = pa.table({"c_custkey": pa.array(ck)}, schema=pa.schema([pa.field("c_custkey", pa.int64(), False)]))
    orders = pa.table({"o_orderkey": okey, "o_custkey": ocust, "o_comment": pa.array(ocomment, pa.string())})
    o = GpuFilterExec(LikeExpr(col("o_comment"), "%special%requests%", negated=True), mem(orders), projection=[0, 1])
    join = GpuHashJoinExec(mem(customer), o, [("c_custkey", "o_custkey")], "Left", projection=[0, 1])
    inner = plan_like_predicates(GpuAggregateExec("Single", ["c_custkey"], [AggregateExpr("count", "o_orderkey", "c_count")], join))
    fused = fuse_pipelines(inner)
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[-1][0] == D.STAGE_LEFT and isinstance(fused.scan.source, GpuLikeExec)
    outer = lambda below: GpuAggregateExec("Single", ["c_count"], [AggregateExpr("count_star", None, "custdist")],  # noqa: E731
                                           GpuProjectionExec([(col("c_count"), "c_count")], below))
    tc = TaskContext(ctx=ctx)
    rows = lambda plan: sorted(tuple(r.values()) for b in collect(plan, tc) for r in b.to_pylist())  # noqa: E731
    od = orders.to_pandas()
    od = od[~od.o_comment.str.contains("special.*requests", regex=True)]
    per = pd.DataFrame({"c_custkey": ck}).merge(od, left_on="c_custkey", right_on="o_custkey", how="left")
    per = per.groupby("c_custkey").o_orderkey.count().reset_index(name="c_count")
    hist = per.groupby("c_count").size().reset_index(name="custdist")
    exp_inner = sorted((int(a), int(b)) for a, b in per.itertuples(index=False))
    exp_outer = sorted((int(a), int(b)) for a, b in hist.itertuples(index=False))
    assert 0 < len(od) < n_ord
    assert rows(inner) == exp_inner and rows(fused) == exp_inner
    assert rows(outer(inner)) == exp_outer and rows(outer(fused)) == exp_outer


def test_q9_green_parts_on_the_build_side(ctx):
    """part (p_name LIKE '%green%') INNER JOIN lineitem ON p_partkey = l_partkey, sum(l_quantity) per part"""
    rng = np.random.default_rng(4)
    n_part, n_li = 2000, 40000
    colors = ["almond", "antique", "green", "forest", "blue", "chiffon", "dark", "greenish", "lime", "navy"]
    pname = [" ".join(rng.choice(colors, 5)) for _ in range(n_part)]
    part = pa.table({"p_partkey": np.arange(1, n_part + 1, dtype=np.int64), "p_name": pa.array(pname, pa.string_view())})
    li = pa.table({"l_partkey": rng.integers(1, n_part + 1, n_li).astype(np.int64), "l_quantity": rng.integers(1, 51, n_li).astype(np.int64)})
    build = GpuFilterExec(LikeExpr(col("p_name"), "%green%"), mem(part), projection=[0])
    join = GpuHashJoinExec(build, mem(li), [("p_partkey", "l_partkey")], "Inner")
    plan = plan_like_predicates(GpuAggregateExec("Single", ["l_partkey"], [AggregateExpr("sum", "l_quantity", "s")], join))
    fused = fuse_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[0][0] == D.STAGE_INNER
    tc = TaskContext(ctx=ctx)
    pdf, ldf = part.to_pandas(), li.to_pandas()
    green = pdf[pdf.p_name.str.contains("green", regex=False)]
    exp = ldf.merge(green, left_on="l_partkey", right_on="p_partkey").groupby("l_partkey").l_quantity.sum()
    exp = sorted((int(k), int(v)) for k, v in exp.items())
    for p in (plan, fused):
        got = sorted(tuple(r.values()) for b in collect(p, tc) for r in b.to_pylist())
        assert got == exp
