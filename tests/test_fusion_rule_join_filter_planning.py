"""Planning decisions of fuse_join_filters (no GPU needed): which joins with a JoinFilter it fuses, how the filter's (side, index) columns
map onto the stage filter's columns, which plans it hands back unchanged, and that GpuPipelineExec._make_pipeline passes exactly the
planned node lists to set_stage_filter."""
import types

import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200 import exec as X
from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, JoinFilter, MemoryExec, col,
                                  fuse_hash_aggregates, fuse_join_filters, fuse_pipelines, lit)

COL, LIT, BIN = D.EXPR_COLUMN, D.EXPR_LITERAL, D.EXPR_BINARY


def mem(**cols):
    t = pa.table(cols)
    return MemoryExec(t.to_batches(), t.schema)


def customer(with_balance=False):
    fields = [pa.field("c_custkey", pa.int64(), False)] + ([pa.field("c_acctbal", pa.int64(), False)] if with_balance else [])
    cols = [np.arange(1, 9, dtype=np.int64)] + ([np.arange(8, dtype=np.int64)] if with_balance else [])
    t = pa.Table.from_arrays(cols, schema=pa.schema(fields))
    return MemoryExec(t.to_batches(), t.schema)


def orders():
    t = pa.table({"o_orderkey": np.arange(1, 17, dtype=np.int64), "o_custkey": (np.arange(16, dtype=np.int64) % 6) + 1,
                  "o_comment": np.arange(16, dtype=np.int64), "o_price": np.arange(16, dtype=np.float64)})
    return GpuFilterExec(col("o_comment") < lit(14, pa.int64()), MemoryExec(t.to_batches(), t.schema), projection=[0, 1, 3])


def q13(filter, join_type="Left", **kw):
    join = GpuHashJoinExec(customer(kw.get("with_balance", False)), orders(), [("c_custkey", "o_custkey")], join_type, filter=filter,
                           null_equality=kw.get("null_equality", "NullEqualsNothing"))
    return GpuAggregateExec("Single", ["c_custkey"], [AggregateExpr("count", "o_orderkey", "a0")], join)


LEFT_FILTER = JoinFilter(col("f0") > lit(3, pa.int64()), [("right", 0)])      # o_orderkey > 3


def test_left_join_filter_fuses_only_under_the_new_rule():
    plan = q13(LEFT_FILTER)
    assert fuse_pipelines(plan) is plan and fuse_hash_aggregates(plan) is plan   # the existing rules keep their decision
    fused = fuse_join_filters(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate" and fused.schema == plan.schema
    kind, pkey, build = fused.scan.stages[-1]
    assert (kind, pkey, build.key) == (D.STAGE_LEFT, "o_custkey", "c_custkey")
    # o_orderkey is column 0 of the orders source
    assert fused.scan.filters == {0: [(COL, 0, 0, 0, 0, 0.0), (LIT, 0, D.INT64, 0, 3, 0.0), (BIN, D.OP_GT, 0, 0, 0, 0.0)]}


def test_left_family_filter_reads_build_columns_as_payload_fields():
    f = JoinFilter(col("f0") < col("f1"), [("left", 1), ("right", 0)])          # c_acctbal < o_orderkey
    for jt, kind in (("LeftSemi", D.STAGE_INNER), ("LeftAnti", D.STAGE_LEFT_ANTI)):
        join = GpuHashJoinExec(customer(with_balance=True), orders(), [("c_custkey", "o_custkey")], jt, filter=f)
        assert fuse_pipelines(join) is join
        fused = fuse_join_filters(join)
        st_kind, pkey, build = fused.scan.stages[-1]
        assert st_kind == kind and build.payload == ["c_acctbal"]
        # source: o_orderkey 0, o_custkey 1, o_comment 2, o_price 3; the stage's payload field c_acctbal is virtual column 4
        assert fused.scan.filters[0] == [(COL, 4, 0, 0, 0, 0.0), (COL, 0, 0, 0, 0, 0.0), (BIN, D.OP_LT, 0, 0, 0, 0.0)]


def lineitem():
    return mem(l_partkey=np.arange(1, 41, dtype=np.int64) % 9 + 1, l_qty=np.arange(40, dtype=np.int16), l_price=np.arange(40, dtype=np.int64),
               l_mode=(np.arange(40) % 7).astype(np.int8))


def part():
    return mem(p_partkey=np.arange(1, 11, dtype=np.int64), p_brand=(np.arange(10) % 5).astype(np.int8), p_size=(np.arange(10) % 50).astype(np.int16))


def inner(filter, join_type="Inner", probe=None, **kw):
    probe = probe if probe is not None else GpuFilterExec(col("l_mode") == lit(1, pa.int8()), lineitem())
    return GpuHashJoinExec(part(), probe, [("p_partkey", "l_partkey")], join_type, filter=filter, **kw)


def test_inner_stage_filter_maps_key_payload_and_probe_columns():
    # p_brand = 3 AND l_qty > p_size AND p_partkey < 100: build payload, probe column vs payload, the build key as the probe key
    f = JoinFilter(((col("f0") == lit(3, pa.int8())) & (col("f1") > col("f2"))) & (col("f3") < lit(100, pa.int64())),
                   [("left", 1), ("right", 1), ("left", 2), ("left", 0)])
    plan = GpuAggregateExec("Single", ["l_partkey", "p_brand"], [AggregateExpr("sum", "l_price", "rev")], inner(f))
    assert fuse_hash_aggregates(plan) is plan
    fused = fuse_join_filters(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate"
    kind, pkey, build = fused.scan.stages[0]
    assert kind == D.STAGE_INNER and pkey == "l_partkey" and build.payload == ["p_brand", "p_size"]
    # source: l_partkey 0, l_qty 1, l_price 2, l_mode 3; payload p_brand 4, p_size 5
    assert [n[:2] for n in fused.scan.filters[0] if n[0] == COL] == [(COL, 4), (COL, 1), (COL, 5), (COL, 0)]


def semi_then_inner(semi_filter, jt="RightSemi", inner_filter=None):
    semi = inner(semi_filter, jt)
    top = GpuHashJoinExec(part(), semi, [("p_partkey", "l_partkey")], "Inner", filter=inner_filter)
    return GpuAggregateExec("Single", ["l_partkey", "p_brand"], [AggregateExpr("sum", "l_price", "rev")], top)


def test_right_semi_and_anti_carry_the_build_columns_their_filter_reads():
    f = JoinFilter(col("f0") > col("f1"), [("right", 1), ("left", 2)])   # l_qty > p_size
    for jt, kind in (("RightSemi", D.STAGE_SEMI), ("RightAnti", D.STAGE_ANTI)):
        plan = semi_then_inner(f, jt)
        assert fuse_hash_aggregates(plan) is plan
        fused = fuse_join_filters(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate"
        st_kind, _, build = fused.scan.stages[0]
        assert st_kind == kind and build.payload == ["p_size"]
        # l_qty is source column 1; the stage's own p_size follows the 4 source columns (stage 1's fields come later)
        assert fused.scan.filters == {0: [(COL, 1, 0, 0, 0, 0.0), (COL, 4, 0, 0, 0, 0.0), (BIN, D.OP_GT, 0, 0, 0, 0.0)]}
        assert fused.scan.virtual_schema().names == ["l_partkey", "l_qty", "l_price", "l_mode", "p_brand", "p_size"]   # no SEMI / ANTI field


def test_shapes_that_stay_unfused():
    same = lambda p: fuse_join_filters(p) is p  # noqa: E731
    agg = lambda j: GpuAggregateExec("Single", ["l_partkey"], [AggregateExpr("count_star", None, "n")], j)  # noqa: E731
    fallible = JoinFilter((col("f0") > lit(0, pa.int64())) & ((col("f0") / col("f1")) > lit(1, pa.int64())), [("right", 2), ("right", 2)])
    assert same(agg(inner(fallible)))                                                # an AND whose right operand can raise
    castrhs = JoinFilter((col("f0") > lit(0, pa.int64())) | (col("f1").cast(pa.int64()) > lit(1, pa.int64())), [("right", 2), ("left", 2)])
    assert same(agg(inner(castrhs)))
    big = col("f0") > lit(0, pa.int64())
    for k in range(40):
        big = big | (col("f0") > lit(k, pa.int64()))                              # 4 nodes per term: beyond 128
    assert same(agg(inner(JoinFilter(big, [("right", 2)]))))
    not_bool = JoinFilter(col("f0") + lit(1, pa.int64()), [("right", 2)])
    assert same(agg(inner(not_bool)))
    ok = JoinFilter(col("f0") > lit(0, pa.int64()), [("right", 2)])
    assert not same(agg(inner(ok)))                                                  # the same plan with a fusable filter
    assert same(agg(inner(ok, null_equality="NullEqualsNull")))
    assert same(agg(inner(ok, join_type="RightAnti", null_aware=True)))
    for jt in ("Right", "Full"):
        assert same(agg(inner(ok, join_type=jt)))
    for jt in ("LeftMark", "RightMark", "Inner"):
        assert same(inner(ok, join_type=jt))
    wide = mem(p_partkey=np.arange(1, 11, dtype=np.int64), a=np.arange(10, dtype=np.int64), b=np.arange(10, dtype=np.int64))
    j = GpuHashJoinExec(wide, GpuFilterExec(col("l_mode") == lit(1, pa.int8()), lineitem()), [("p_partkey", "l_partkey")], "RightSemi",
                        filter=JoinFilter(col("f0") < col("f1"), [("left", 1), ("left", 2)]))
    assert same(agg(j))                                                              # 128 payload bits
    assert same(q13(LEFT_FILTER, null_equality="NullEqualsNull"))


class _FakePipeline:
    calls = []

    def __init__(self, ctx, types_, nodes, stages):
        self.filters = []
        _FakePipeline.calls.append(self)

    def set_stage_filter(self, stage, nodes):
        self.filters.append((stage, list(nodes)))

    def close(self):
        pass


def test_make_pipeline_passes_the_planned_filters(monkeypatch):
    plan = semi_then_inner(JoinFilter(col("f0") > col("f1"), [("right", 1), ("left", 2)]),
                           inner_filter=JoinFilter(col("f0") == lit(2, pa.int8()), [("left", 1)]))   # ... and p_brand = 2 on stage 1
    fused = fuse_join_filters(plan)
    assert isinstance(fused, GpuPipelineExec) and sorted(fused.scan.filters) == [0, 1]
    assert [n[:2] for n in fused.scan.filters[1] if n[0] == COL] == [(COL, 4)]       # stage 1's p_brand: virtual column 4
    monkeypatch.setattr(X.D, "Pipeline", _FakePipeline)
    monkeypatch.setattr(X.GpuPipelineExec, "build_lookup", lambda self, ctx: types.SimpleNamespace(close=lambda: None))
    pipe, keep = fused._make_pipeline(types.SimpleNamespace(gpu=None))
    assert pipe.filters == sorted(fused.scan.filters.items()) and len(keep) == 2
