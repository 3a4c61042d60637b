"""Planning decisions of the Full-join fusion (no GPU needed): which HashJoinExec(Full) plans `fuse_full_joins` turns into a pipeline with
a FULL stage (a RIGHT stage whose lookup keeps visited marks), into which sink, with which payloads and lookup words; that the fused node's
schema equals the unfused plan's, nullability included, and that the probe columns are nullable in its virtual schema; and which shapes it
hands back unchanged.  The rules before it (fuse_right_joins and below) leave every Full join alone."""
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, JoinFilter, MemoryExec, build_join_schema, col, fuse_full_joins, fuse_join_filters,
                                  fuse_output_pipelines, fuse_pipelines, fuse_right_joins, lit)
from test_fusion_rule_right_planning import agg, customer, orders, project


def full(build=None, probe=None, **kw):
    return GpuHashJoinExec(build or customer(), probe or orders(), kw.pop("on", [("c_custkey", "o_custkey")]), "Full", **kw)


def orders_not_null():
    o = orders()
    t = pa.Table.from_batches(o.input.batches).cast(pa.schema([f.with_nullable(False) for f in o.input.schema]))
    return GpuFilterExec(o.predicate, MemoryExec(t.to_batches(), t.schema))


def earlier_rules_leave(plan):
    return all(rule(plan) is plan for rule in (fuse_pipelines, fuse_join_filters, fuse_output_pipelines, fuse_right_joins))


def test_output_sink_over_a_full_stage():
    plan = project(full(), ["o_orderkey", "o_totalprice", "c_acctbal", "c_nationkey"])
    assert earlier_rules_leave(plan)
    fused = fuse_full_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "output" and fused.fallback is plan
    assert fused.scan.full and len(fused.scan.stages) == 1
    kind, pkey, build = fused.scan.stages[0]
    assert (kind, pkey, build.key) == (D.STAGE_RIGHT, "o_custkey", "c_custkey")
    assert build.payload == ["c_nationkey", "c_acctbal"] and build.n_acc_words == 1   # the visited marks
    vs = fused.scan.virtual_schema()
    assert [vs.field(i).name for i in fused.out_cols] == ["o_orderkey", "o_totalprice", "c_acctbal", "c_nationkey"]
    assert fused.schema == plan.schema and all(f.nullable for f in vs)      # probe columns too: NULL on the unmatched build rows
    assert all(f.nullable for f in fused.schema)
    # the build key read above the join is a payload field (NULL on unmatched probe rows), never the probe key
    fused = fuse_full_joins(project(full(), ["o_orderkey", "c_custkey"]))
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[0][2].payload == ["c_custkey"]
    assert fused.out_cols[1] >= len(fused.scan.source.schema)
    # with the join's own projection the schema is build_join_schema(..., "Full") projected
    plain = full(projection=[2, 3, 4, 7])
    fused = fuse_full_joins(plain)
    assert isinstance(fused, GpuPipelineExec) and fused.schema == plain.schema
    whole, _ = build_join_schema(customer().schema, orders().schema, "Full")
    assert [f.nullable for f in fused.schema] == [whole.field(i).nullable for i in (2, 3, 4, 7)] == [True] * 4


def test_dense_sink():
    for mode in ("Single", "Partial"):
        for group, bounds in ((["c_nationkey"], [(0, 24)]), (["o_orderdate"], [(0, 49)]), ([], [])):
            plan = agg(full(), group, mode=mode)
            assert earlier_rules_leave(plan)
            fused = fuse_full_joins(plan)
            assert isinstance(fused, GpuPipelineExec) and fused.sink == "dense" and fused.fallback is plan, (mode, group)
            assert fused.key_range == bounds and fused.schema == plan.schema and fused.scan.full
            _, _, build = fused.scan.stages[0]
            assert build.payload == [n for n in ("c_nationkey", "c_acctbal") if n in group + ["c_acctbal"]]   # read above, in build order
            assert build.n_acc_words == 1


def test_hash_sink_declares_probe_group_columns_nullable():
    plan = agg(full(), ["o_orderdate", "c_nationkey"])
    assert earlier_rules_leave(plan)
    fused = fuse_full_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash" and fused.fallback is plan
    assert fused.group_by == ["o_orderdate", "c_nationkey"] and fused.nullable == [True, True] and fused.schema == plan.schema
    # a probe column declared non-nullable in the source is nullable above a Full join
    fused = fuse_full_joins(agg(full(probe=orders_not_null()), ["o_orderdate", "c_nationkey"]))
    assert fused.scan.source.schema.field("o_orderdate").nullable is False and fused.nullable == [True, True]
    big = agg(full(build=customer(extra=("c_big",))), ["c_big"], aggs=(("count_star", None), ("sum", "o_totalprice")))
    fused = fuse_full_joins(big)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash" and fused.nullable == [True]


def test_shapes_that_stay_unfused():
    same = lambda p: fuse_full_joins(p) is p  # noqa: E731
    out = ["o_orderkey", "c_nationkey"]
    assert same(project(full(filter=JoinFilter(col("f0") > lit(3, pa.int64()), [("right", 3)])), out))    # a JoinFilter
    assert same(project(full(null_equality="NullEqualsNull"), out))
    assert same(project(full(), ["o_orderkey", "o_totalprice"]))           # no build column carried: nothing enforces unique keys
    assert same(project(full(build=customer(extra=("c_a", "c_b"))), ["o_orderkey", "c_a", "c_b"]))   # 128 bits of payload
    # a FULL stage is the only probe stage: not above another join, and no join probes above it
    semi = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "RightSemi")
    assert same(project(full(probe=semi, on=[("c_custkey", "o_orderkey")]), ["o_orderkey", "c_acctbal"]))
    over = GpuHashJoinExec(customer(), project(full(), ["o_orderkey", "o_custkey", "c_acctbal"]), [("c_custkey", "o_orderkey")], "Right")
    assert same(project(over, ["o_orderkey", "c_nationkey"]))
    # a Full join on a build side stays unfused, and so does an aggregate that reads no build column
    nested = GpuHashJoinExec(project(full(), ["o_orderkey", "c_nationkey"]), orders(), [("o_orderkey", "o_orderkey")], "Inner")
    assert same(nested)
    assert same(agg(full(), ["o_orderdate"], aggs=(("count_star", None),)))  # no build column read above the join
