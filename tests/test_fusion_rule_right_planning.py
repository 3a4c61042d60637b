"""Planning decisions of the Right-join fusion (no GPU needed): which HashJoinExec(Right) plans `fuse_right_joins` turns into a pipeline with
a RIGHT stage, into which sink, with which stage kinds and payloads; that the fused node's schema equals the unfused plan's, nullability
included; and which shapes it hands back unchanged.  The rules before it (fuse_output_pipelines and below) leave every Right join alone."""
import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, Column, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec,
                                  JoinFilter, MemoryExec, build_join_schema, col, fuse_output_pipelines, fuse_right_joins, lit)


def customer(extra=()):
    """the dimension (build side): c_custkey, c_mktsegment, c_nationkey in [0, 24], c_acctbal Int32, plus Int64 columns `extra`"""
    n = 40
    cols = {"c_custkey": np.arange(1, n + 1, dtype=np.int64), "c_mktsegment": (np.arange(n) % 5).astype(np.int32),
            "c_nationkey": (np.arange(n) % 25).astype(np.int32), "c_acctbal": np.arange(n, dtype=np.int32)}
    cols.update({e: np.arange(n, dtype=np.int64) * 1_000_000 for e in extra})   # too wide a domain for the dense sink
    t = pa.table(cols)
    t = t.cast(pa.schema([f.with_nullable(False) for f in t.schema]))
    return GpuFilterExec(col("c_mktsegment") == lit(1, pa.int32()), MemoryExec(t.to_batches(), t.schema))


def orders():
    n = 200
    t = pa.table({"o_orderkey": np.arange(1, n + 1, dtype=np.int64), "o_custkey": (np.arange(n, dtype=np.int64) % 60) + 1,
                  "o_orderdate": pa.array((np.arange(n) % 50).astype(np.int32)).cast(pa.date32()), "o_totalprice": np.arange(n, dtype=np.int64)})
    return GpuFilterExec(col("o_orderdate") < lit(30, pa.date32()), MemoryExec(t.to_batches(), t.schema))


def right(build=None, **kw):
    return GpuHashJoinExec(build or customer(), orders(), kw.pop("on", [("c_custkey", "o_custkey")]), "Right", **kw)


def project(plan, names):
    return GpuProjectionExec([(Column(n), n) for n in names], plan)


def agg(below, group, aggs=(("count_star", None), ("sum", "o_totalprice"), ("max", "c_acctbal")), mode="Single"):
    return GpuAggregateExec(mode, group, [AggregateExpr(f, a, f"a{i}") for i, (f, a) in enumerate(aggs)], below)


def test_output_sink_over_a_right_stage():
    plan = project(right(), ["o_orderkey", "o_totalprice", "c_acctbal", "c_nationkey"])
    assert fuse_output_pipelines(plan) is plan                               # the rules before it leave Right joins alone
    fused = fuse_right_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "output" and fused.fallback is plan
    kind, pkey, build = fused.scan.stages[-1]
    assert (kind, pkey, build.key) == (D.STAGE_RIGHT, "o_custkey", "c_custkey")
    assert build.payload == ["c_nationkey", "c_acctbal"]                    # the columns read above the join, in build order
    vs = fused.scan.virtual_schema()
    assert [vs.field(i).name for i in fused.out_cols] == ["o_orderkey", "o_totalprice", "c_acctbal", "c_nationkey"]
    assert fused.schema == plan.schema and all(f.nullable for f in vs if f.name.startswith("c_"))
    # the build key read above the join is a payload field (NULL when unmatched), never the probe key
    keyed = project(right(), ["o_orderkey", "c_custkey"])
    fused = fuse_right_joins(keyed)
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[-1][2].payload == ["c_custkey"]
    vs = fused.scan.virtual_schema()
    assert vs.field(fused.out_cols[1]).nullable and fused.out_cols[1] >= len(fused.scan.source.schema)
    # the whole join (every build column is read: 160 bits) stays unfused; with the join's projection its schema is build_join_schema's
    assert fuse_right_joins(right()) is not None and fuse_right_joins(right()).__class__ is GpuHashJoinExec
    plain = right(projection=[2, 3, 4, 7])
    fused = fuse_right_joins(plain)
    assert isinstance(fused, GpuPipelineExec) and fused.schema == plain.schema
    full, _ = build_join_schema(customer().schema, orders().schema, "Right")
    assert [f.nullable for f in fused.schema] == [full.field(i).nullable for i in (2, 3, 4, 7)] and fused.schema.field(0).nullable


def test_composite_key_and_stage_chains():
    plan = project(right(on=[("c_custkey", "o_custkey"), ("c_acctbal", "o_totalprice")]), ["o_orderkey", "c_nationkey"])
    assert fuse_right_joins(plan) is plan                                    # key types differ (Int32 / Int64): no composite key
    semi = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "RightSemi")
    top = GpuHashJoinExec(customer(), semi, [("c_custkey", "o_orderkey")], "Right")
    fused = fuse_right_joins(project(top, ["o_orderkey", "c_acctbal"]))
    assert isinstance(fused, GpuPipelineExec) and [k for k, _, _ in fused.scan.stages] == [D.STAGE_SEMI, D.STAGE_RIGHT]
    assert fused.scan.stages[-1][2].payload == ["c_acctbal"]


def test_dense_sink_grouped_on_a_right_payload_field():
    for mode in ("Single", "Partial"):
        plan = agg(right(), ["c_nationkey"], mode=mode)
        assert fuse_output_pipelines(plan) is plan
        fused = fuse_right_joins(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "dense" and fused.fallback is plan
        assert fused.key_range == [(0, 24)] and fused.schema == plan.schema
        kind, _, build = fused.scan.stages[-1]
        assert kind == D.STAGE_RIGHT and build.payload == ["c_nationkey", "c_acctbal"]


def test_hash_sink_with_a_nullable_right_group_column():
    plan = agg(right(), ["o_orderdate", "c_nationkey"])
    fused = fuse_right_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash" and fused.fallback is plan
    assert fused.group_by == ["o_orderdate", "c_nationkey"] and fused.nullable == [True, True] and fused.schema == plan.schema
    big = agg(right(build=customer(extra=("c_big",))), ["c_big"], aggs=(("count_star", None), ("sum", "o_totalprice")))   # a wide domain
    fused = fuse_right_joins(big)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash" and fused.nullable == [True]


def test_shapes_that_stay_unfused():
    same = lambda p: fuse_right_joins(p) is p  # noqa: E731
    out = ["o_orderkey", "c_nationkey"]
    assert same(project(right(filter=JoinFilter(col("f0") > lit(3, pa.int64()), [("right", 3)])), out))   # a JoinFilter
    assert same(project(right(null_equality="NullEqualsNull"), out))
    assert same(project(right(), ["o_orderkey", "o_totalprice"]))           # no build column carried: nothing enforces unique keys
    wide = right(build=customer(extra=("c_a", "c_b")))
    assert same(project(wide, ["o_orderkey", "c_a", "c_b"]))                 # 128 bits of payload
    assert same(GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Full"))
    # a Right join on a build side: its NULL payload fields cannot enter a lookup
    nested = GpuHashJoinExec(project(right(), ["o_orderkey", "c_nationkey"]), orders(), [("o_orderkey", "o_orderkey")], "Inner")
    assert same(nested)
