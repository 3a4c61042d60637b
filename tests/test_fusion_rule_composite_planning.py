"""Planning decisions for joins on composite keys (no GPU needed): which two- to four-key joins each fusion rule fuses, what the stage's
probe keys, the build's keys, payload and declared key ranges become, and what stays unfused (mixed types, unknown bounds, a domain above
2^63 - 1, a key taken from an earlier stage's payload, NullEqualsNull).  One-key joins keep their string keys."""
import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec, JoinFilter,
                                  MemoryExec, col, fuse_join_filters, fuse_output_pipelines, fuse_pipelines, lit)


def mem(**cols):
    t = pa.table(cols)
    return MemoryExec(t.to_batches(), t.schema)


def partsupp(n=12, suppkey=None):
    pk = np.repeat(np.arange(1, n // 4 + 1, dtype=np.int64), 4)
    sk = np.tile(np.arange(1, 5, dtype=np.int64), n // 4) if suppkey is None else suppkey
    return mem(ps_partkey=pk, ps_suppkey=sk, ps_supplycost=np.arange(n, dtype=np.int64))


def lineitem(n=40):
    return GpuFilterExec(col("l_quantity") < lit(45), mem(l_partkey=np.arange(n, dtype=np.int64) % 3 + 1, l_suppkey=np.arange(n, dtype=np.int64) % 4 + 1,
                                                         l_quantity=np.arange(n, dtype=np.int64), l_extendedprice=np.arange(n, dtype=np.int64) * 10))


Q9_ON = [("ps_partkey", "l_partkey"), ("ps_suppkey", "l_suppkey")]


def q9_join(kind="Inner", build=None, **kw):
    return GpuHashJoinExec(build or partsupp(), lineitem(), kw.pop("on", Q9_ON), kind, **kw)


def test_two_key_inner_join_keyed_aggregate():
    j = q9_join()
    plan = GpuAggregateExec("Single", ["l_partkey", "l_suppkey", "ps_supplycost"], [AggregateExpr("sum", "l_quantity", "q")], j)
    fused = fuse_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate"
    (kind, pkey, build), = fused.scan.stages
    assert (kind, pkey, build.key, build.payload) == (D.STAGE_INNER, ["l_partkey", "l_suppkey"], ["ps_partkey", "ps_suppkey"], ["ps_supplycost"])
    assert build.key_ranges == [(1, 3), (1, 4)] and build.n_acc_words > 0
    assert fused.group_by == ["l_partkey", "l_suppkey", "ps_supplycost"]
    # the build keys name the same groups
    plan = GpuAggregateExec("Partial", ["ps_partkey", "ps_suppkey"], [AggregateExpr("count_star", None, "n")], q9_join())
    fused = fuse_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.group_by == ["l_partkey", "l_suppkey"]
    # a group key set without every component is not determined by the build row (Q9's profit by supplier): the hash-keyed sink over a
    # composite stage measured slower than the unfused join and group-by, so the plan stays unfused
    proj = GpuProjectionExec([(col("l_suppkey"), "l_suppkey"), (col("l_extendedprice") - col("ps_supplycost") * col("l_quantity"), "amount")], q9_join())
    plan = GpuAggregateExec("Single", ["l_suppkey"], [AggregateExpr("sum", "amount", "profit")], proj)
    assert fuse_pipelines(plan) is plan and fuse_output_pipelines(plan) is plan


def test_three_and_four_key_joins_fuse_onto_the_output_sink():
    for k in (3, 4):
        b = {f"b{g}": (np.arange(10, dtype=np.int32) * (g + 1)) for g in range(k)}
        b["bv"] = np.arange(10, dtype=np.int64)
        p = {f"p{g}": (np.arange(30, dtype=np.int32) % 10) for g in range(k)}
        p["pv"] = np.arange(30, dtype=np.int64)
        plan = GpuHashJoinExec(mem(**b), mem(**p), [(f"b{g}", f"p{g}") for g in range(k)], "Inner")
        fused = fuse_output_pipelines(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "output"
        (kind, pkey, build), = fused.scan.stages
        assert pkey == [f"p{g}" for g in range(k)] and build.key == [f"b{g}" for g in range(k)] and build.payload == ["bv"]
        assert build.key_ranges == [(0, 9 * (g + 1)) for g in range(k)]
        # build keys leave as their probe keys, the payload as its field
        assert fused.out_cols == list(range(k)) + [k + 1] + list(range(k + 1))
    five = GpuHashJoinExec(mem(**{f"b{g}": np.arange(3) for g in range(5)}), mem(**{f"p{g}": np.arange(3) for g in range(5)}),
                           [(f"b{g}", f"p{g}") for g in range(5)], "Inner")
    assert fuse_output_pipelines(five) is five


def test_semi_anti_and_left_joins():
    for kind, stage in (("RightSemi", D.STAGE_SEMI), ("RightAnti", D.STAGE_ANTI)):
        fused = fuse_output_pipelines(q9_join(kind))
        assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[0][:2] == (stage, ["l_partkey", "l_suppkey"])
        assert fused.scan.stages[0][2].payload == []
    ps = partsupp()
    non_null = pa.schema([pa.field(f.name, f.type, False) for f in ps.schema])
    ps = MemoryExec(ps.batches, non_null)
    for kind, stage in (("LeftSemi", D.STAGE_INNER), ("LeftAnti", D.STAGE_LEFT_ANTI)):
        fused = fuse_pipelines(q9_join(kind, build=ps))
        assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[-1][:2] == (stage, ["l_partkey", "l_suppkey"])
        assert fused.group_by == ["l_partkey", "l_suppkey", "ps_supplycost"]
    plan = GpuAggregateExec("Single", ["ps_partkey", "ps_suppkey"], [AggregateExpr("sum", "l_quantity", "q")], q9_join("Left", build=ps))
    fused = fuse_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[-1][0] == D.STAGE_LEFT and fused.group_by == ["l_partkey", "l_suppkey"]


def test_join_filter_maps_each_build_key_to_its_probe_key():
    f = JoinFilter(col("f0") < col("f1"), [("left", 1), ("right", 2)])      # ps_suppkey < l_quantity
    plan = GpuAggregateExec("Single", ["l_partkey", "l_suppkey"], [AggregateExpr("count_star", None, "n")], q9_join(filter=f))
    assert fuse_pipelines(plan) is plan
    fused = fuse_join_filters(plan)
    assert isinstance(fused, GpuPipelineExec)
    nodes = fused.scan.filters[0]
    assert [n[1] for n in nodes if n[0] == D.EXPR_COLUMN] == [1, 2]         # l_suppkey, l_quantity of the probe source


def test_refusals():
    # mixed types in a pair
    b = mem(a=np.arange(4, dtype=np.int32), b=np.arange(4, dtype=np.int64))
    p = mem(a=np.arange(8, dtype=np.int64), b=np.arange(8, dtype=np.int64))
    plan = GpuHashJoinExec(b, p, [("a", "a"), ("b", "b")], "Inner")
    assert fuse_output_pipelines(plan) is plan
    # unknown bounds: a build key column without a non-NULL value
    nulls = pa.table({"ps_partkey": pa.array([None] * 4, pa.int64()), "ps_suppkey": np.arange(4, dtype=np.int64), "ps_supplycost": np.arange(4, dtype=np.int64)})
    plan = q9_join(build=MemoryExec(nulls.to_batches(), nulls.schema))
    assert fuse_output_pipelines(plan) is plan
    # D = 2^63 stays unfused, D = 2^62 fuses
    for top, fuses in (((1 << 62) - 1, False), ((1 << 61) - 1, True)):
        plan = q9_join(build=mem(ps_partkey=np.array([0, top], np.int64), ps_suppkey=np.array([0, 1], np.int64), ps_supplycost=np.arange(2, dtype=np.int64)))
        assert isinstance(fuse_output_pipelines(plan), GpuPipelineExec) == fuses, top
    # a component that is a payload field of an earlier stage (Q5's c_nationkey)
    cust = mem(c_custkey=np.arange(1, 5, dtype=np.int64), c_nationkey=np.arange(4, dtype=np.int64))
    orders = mem(o_custkey=np.arange(1, 9, dtype=np.int64) % 4 + 1, o_suppkey=np.arange(8, dtype=np.int64) % 4)
    inner = GpuHashJoinExec(cust, orders, [("c_custkey", "o_custkey")], "Inner")
    supp = mem(s_suppkey=np.arange(4, dtype=np.int64), s_nationkey=np.arange(4, dtype=np.int64))
    plan = GpuHashJoinExec(supp, inner, [("s_suppkey", "o_suppkey"), ("s_nationkey", "c_nationkey")], "Inner")
    assert fuse_output_pipelines(plan) is plan
    # NullEqualsNull
    plan = q9_join(null_equality="NullEqualsNull")
    assert fuse_output_pipelines(plan) is plan


def test_one_key_joins_keep_their_string_keys():
    part = mem(ps_partkey=np.arange(1, 4, dtype=np.int64), ps_suppkey=np.arange(3, dtype=np.int32))
    j = GpuHashJoinExec(part, lineitem(), [("ps_partkey", "l_partkey")], "Inner")
    agg = fuse_pipelines(GpuAggregateExec("Single", ["l_partkey", "ps_suppkey"], [AggregateExpr("count_star", None, "n")], j))
    out = fuse_output_pipelines(j)
    for f in (agg, out):
        assert isinstance(f, GpuPipelineExec)
        (_, pkey, build), = f.scan.stages
        assert type(pkey) is str and type(build.key) is str and (pkey, build.key) == ("l_partkey", "ps_partkey")
        assert build.payload == ["ps_suppkey"] and build.key_ranges == []
