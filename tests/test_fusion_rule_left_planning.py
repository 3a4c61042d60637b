"""Planning decisions of the Left-family fusion (no GPU needed): which Left / LeftSemi / LeftAnti joins `fuse_pipelines` turns into the
join-keyed sink over a LEFT, LEFT_ANTI or INNER stage, and which it hands back unchanged."""
import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec, JoinFilter,
                                  MemoryExec, col, fuse_pipelines, lit)


def customer(nullable_key=False, with_balance=False):
    fields = [pa.field("c_custkey", pa.int64(), nullable_key)] + ([pa.field("c_acctbal", pa.int64(), False)] if with_balance else [])
    cols = [np.arange(1, 9, dtype=np.int64)] + ([np.arange(8, dtype=np.int64)] if with_balance else [])
    t = pa.Table.from_arrays(cols, schema=pa.schema(fields))
    return MemoryExec(t.to_batches(), t.schema)


def orders():
    t = pa.table({"o_orderkey": np.arange(1, 17, dtype=np.int64), "o_custkey": (np.arange(16, dtype=np.int64) % 6) + 1,
                  "o_comment": np.arange(16, dtype=np.int64), "o_price": np.arange(16, dtype=np.float64)})
    return GpuFilterExec(col("o_comment") < lit(14, pa.int64()), MemoryExec(t.to_batches(), t.schema), projection=[0, 1, 3])


def q13(group="c_custkey", aggs=(("count", "o_orderkey"),), **kw):
    join = GpuHashJoinExec(customer(**{k: v for k, v in kw.items() if k in ("nullable_key", "with_balance")}), orders(), [("c_custkey", "o_custkey")],
                           kw.get("join_type", "Left"), filter=kw.get("filter"), null_equality=kw.get("null_equality", "NullEqualsNothing"))
    below = GpuProjectionExec(kw["proj"], join) if "proj" in kw else join
    return GpuAggregateExec(kw.get("mode", "Single"), [group], [AggregateExpr(f, a, f"a{i}") for i, (f, a) in enumerate(aggs)], below)


def test_q13_aggregate_fuses_over_a_left_stage():
    for mode in ("Single", "SinglePartitioned", "Partial"):
        plan = q13(mode=mode, aggs=(("count", "o_orderkey"), ("count_star", None), ("sum", "o_price"), ("avg", "o_price")))
        fused = fuse_pipelines(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate" and fused.schema == plan.schema
        kind, pkey, build = fused.scan.stages[-1]
        assert (kind, pkey, build.key) == (D.STAGE_LEFT, "o_custkey", "c_custkey")
        assert fused.group_by == ["o_custkey"]                      # the build key, emitted from the record
        assert [a[0] for a in fused.aggs] == ["count", "count_star", "sum", "avg"]
        assert build.n_acc_words == 1 + 1 + 1 + 2 + 2


def test_left_with_a_build_column_in_the_group():
    plan = q13(with_balance=True, proj=[(col("c_custkey"), "c_custkey"), (col("c_acctbal"), "c_acctbal"), (col("o_price"), "o_price")],
               aggs=(("max", "o_price"),))
    plan = GpuAggregateExec("Single", ["c_custkey", "c_acctbal"], plan.aggr_expr, plan.input)
    fused = fuse_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.group_by == ["o_custkey", "c_acctbal"]


def test_left_shapes_that_stay_unfused():
    same = lambda p: fuse_pipelines(p) is p  # noqa: E731
    assert same(q13(group="o_custkey"))                                      # the probe key is NULL on a padded row
    assert same(q13(nullable_key=True))                                      # a NULL build key would be dropped, not emitted
    assert same(q13(with_balance=True, aggs=(("sum", "c_acctbal"),)))        # a build-only argument needs the padded row's own value
    mixed = [(col("c_custkey"), "c_custkey"), (col("o_price") + col("c_acctbal").cast(pa.float64()), "v")]
    assert same(q13(with_balance=True, proj=mixed, aggs=(("sum", "v"),)))   # reads a build column
    isnull = [(col("c_custkey"), "c_custkey"), (col("o_price").is_null(), "v")]
    assert same(q13(proj=isnull, aggs=(("count", "v"),)))                    # IS NULL is not NULL on the padded row
    both = [(col("c_custkey"), "c_custkey"), ((col("o_price") > lit(1.0)) & (col("o_price") < lit(9.0)), "v")]
    assert same(q13(proj=both, aggs=(("count", "v"),)))                      # AND does not propagate NULL
    assert same(q13(null_equality="NullEqualsNull"))
    assert same(q13(filter=JoinFilter(col("f0") > lit(3, pa.int64()), [("right", 0)])))
    for jt in ("Right", "Full"):
        assert same(q13(join_type=jt))
    part = q13(mode="Partial")
    assert same(GpuAggregateExec("Final", ["c_custkey"], [AggregateExpr("count", "o_orderkey", "a0")], part, input_schema=part.input.schema))


def test_left_semi_and_anti_joins_become_the_join_keyed_sink():
    for jt, kind in (("LeftSemi", D.STAGE_INNER), ("LeftAnti", D.STAGE_LEFT_ANTI)):
        join = GpuHashJoinExec(customer(with_balance=True), orders(), [("c_custkey", "o_custkey")], jt, projection=[1])
        fused = fuse_pipelines(join)
        assert isinstance(fused, GpuPipelineExec) and fused.schema == join.schema and fused.aggs == []
        st_kind, pkey, build = fused.scan.stages[-1]
        assert (st_kind, pkey, build.payload, build.n_acc_words) == (kind, "o_custkey", ["c_acctbal"], 1)
        assert fused.group_by == ["o_custkey", "c_acctbal"] and fused.project == [1]
        plain = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], jt)
        assert fuse_pipelines(plain).project is None
    same = lambda p: fuse_pipelines(p) is p  # noqa: E731
    assert same(GpuHashJoinExec(customer(nullable_key=True), orders(), [("c_custkey", "o_custkey")], "LeftAnti"))
    assert same(GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "LeftAnti", null_aware=True))
    for jt in ("LeftMark", "RightMark", "Left", "Inner"):
        assert same(GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], jt))
