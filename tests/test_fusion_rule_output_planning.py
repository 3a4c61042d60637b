"""Planning decisions of fuse_output_pipelines (no GPU needed): which top-level join chains become one GpuPipelineExec over the ordered
output sink, which virtual column each output column comes from, what it hands back unchanged, and that it defers to the earlier rules."""
from decimal import Decimal

import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec, JoinFilter,
                                  MemoryExec, col, fuse_output_pipelines, lit)


def customer(key_type=pa.int64()):
    t = pa.Table.from_arrays([pa.array(np.arange(1, 9), key_type), np.arange(8, dtype=np.int32)],
                             schema=pa.schema([pa.field("c_custkey", key_type, False), pa.field("c_nation", pa.int32(), False)]))
    return MemoryExec(t.to_batches(), t.schema)


def extras():
    t = pa.table({"x_orderkey": np.arange(0, 16, 2, dtype=np.int64), "x_flag": np.arange(8, dtype=np.int32) % 3})
    return MemoryExec(t.to_batches(), t.schema)


def orders():
    sch = pa.schema([pa.field("o_orderkey", pa.int64(), False), pa.field("o_custkey", pa.int64()), pa.field("o_totalprice", pa.decimal128(15, 2)),
                     pa.field("o_orderdate", pa.date32())])
    t = pa.Table.from_arrays([pa.array(np.arange(16, dtype=np.int64)), pa.array(np.arange(16, dtype=np.int64) % 9, mask=np.arange(16) % 5 == 0),
                              pa.array([Decimal(i) for i in range(16)], pa.decimal128(15, 2)), pa.array(np.arange(16, dtype=np.int32)).cast(pa.date32())],
                             schema=sch)
    return GpuFilterExec(col("o_orderdate") < lit(14, pa.date32()), MemoryExec(t.to_batches(), t.schema))


def join(kind="Inner", build=None, probe=None, **kw):
    return GpuHashJoinExec(build or customer(), probe or orders(), kw.pop("on", [("c_custkey", "o_custkey")]), kind, **kw)


def test_inner_chain_becomes_the_ordered_output_sink():
    plan = join()
    fused = fuse_output_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "output" and fused.schema == plan.schema
    (kind, pkey, build), = fused.scan.stages
    assert (kind, pkey, build.key, build.payload) == (D.STAGE_INNER, "o_custkey", "c_custkey", ["c_nation"])
    vs = fused.scan.virtual_schema()
    assert [f.name for f in vs] == ["o_orderkey", "o_custkey", "o_totalprice", "o_orderdate", "c_nation"]
    # c_custkey <- the probe key o_custkey, c_nation <- the payload field, then the probe columns
    assert fused.out_cols == [1, 4, 0, 1, 2, 3]
    assert fused.fallback is plan                                # run when the build side turns out not to fuse (duplicate keys)


def test_projection_picks_and_reorders_the_emitted_columns():
    j = join()
    plan = GpuProjectionExec([(col("o_totalprice"), "o_totalprice"), (col("c_custkey"), "c_custkey"), (col("c_nation"), "c_nation")], j)
    fused = fuse_output_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.out_cols == [2, 1, 4] and fused.schema == plan.schema


def test_semi_and_anti_chains_emit_probe_columns_only():
    for kind, stage in (("RightSemi", D.STAGE_SEMI), ("RightAnti", D.STAGE_ANTI)):
        fused = fuse_output_pipelines(join(kind))
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "output"
        assert fused.scan.stages[0][0] == stage and fused.out_cols == [0, 1, 2, 3]


def test_two_stage_chain_maps_a_lower_build_key_to_its_probe_key():
    lower = join("Inner")                                        # c_custkey, c_nation, o_*
    top = GpuHashJoinExec(extras(), lower, [("x_orderkey", "o_orderkey")], "Inner")
    plan = GpuProjectionExec([(col("o_orderkey"), "o_orderkey"), (col("c_custkey"), "c_custkey"), (col("x_flag"), "x_flag"),
                              (col("x_orderkey"), "x_orderkey"), (col("c_nation"), "c_nation")], top)
    fused = fuse_output_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and [s[0] for s in fused.scan.stages] == [D.STAGE_INNER, D.STAGE_INNER]
    # virtual schema: o_orderkey, o_custkey, o_totalprice, o_orderdate, c_nation, x_flag
    assert fused.out_cols == [0, 1, 5, 0, 4]


def test_inner_stages_without_payload_get_a_row_counter_word():
    # an Inner join whose build side is its key only: the word makes the lookup refuse duplicate build keys instead of folding them
    k = MemoryExec(pa.table({"k": np.arange(4, dtype=np.int64)}).to_batches())
    fused = fuse_output_pipelines(join("Inner", build=k, on=[("k", "o_custkey")]))
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[0][2].n_acc_words == 1 and fused.out_cols == [1, 0, 1, 2, 3]
    semi = fuse_output_pipelines(join("RightSemi", build=k, on=[("k", "o_custkey")]))
    assert semi.scan.stages[0][2].n_acc_words == 0


def test_join_filters_fuse_as_stage_filters():
    f = JoinFilter(col("f0") > col("f1"), [("left", 1), ("right", 0)])
    fused = fuse_output_pipelines(join("Inner", filter=f))
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "output" and 0 in fused.scan.filters


def test_leaves_alone_what_the_output_sink_does_not_carry():
    o = orders()
    assert fuse_output_pipelines(o) is o                                                   # a bare FilterExec is one kernel already
    for kind in ("Left", "Right", "Full"):
        p = join(kind)
        assert fuse_output_pipelines(p) is p
    two = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey"), ("c_nation", "o_orderkey")], "Inner")
    assert fuse_output_pipelines(two) is two                                               # several keys
    aware = join("RightAnti", null_aware=True)
    assert fuse_output_pipelines(aware) is aware
    nen = join("Inner", null_equality="NullEqualsNull")
    assert fuse_output_pipelines(nen) is nen
    computed = GpuProjectionExec([(col("o_orderkey") + lit(1), "x")], join())
    assert fuse_output_pipelines(computed) is computed
    # the build key emitted from a probe key of another type stays unfused; without it in the output the join fuses
    other = join("Inner", build=customer(pa.int32()))
    assert fuse_output_pipelines(other) is other
    proj = GpuProjectionExec([(col("o_orderkey"), "o_orderkey"), (col("c_nation"), "c_nation")], join("Inner", build=customer(pa.int32())))
    assert isinstance(fuse_output_pipelines(proj), GpuPipelineExec)


def test_defers_to_the_earlier_rules():
    agg = GpuAggregateExec("Single", ["o_custkey", "c_nation"], [AggregateExpr("count_star", None, "n")], join())
    assert fuse_output_pipelines(agg).sink == "aggregate"
    semi = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "LeftSemi")
    fused = fuse_output_pipelines(semi)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate"
