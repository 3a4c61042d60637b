"""The hash-keyed aggregate fusion as a PLANNING decision (no GPU needed: nothing is executed).  `fuse_hash_aggregates` runs after
`fuse_pipelines`: it returns that rule's result when it fuses, and otherwise collapses an AggregateExec whose GROUP BY the join key does not
determine (TPC-H Q15's revenue0 over a FilterExec; Q3 grouped by o_custkey over the Inner join) into one GpuPipelineExec with the hash
sink.  Everything the library would refuse stays unfused.  The plan builders are shared with the GPU test that executes them."""
import datetime
from decimal import Decimal

import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec, MemoryExec,
                                  col, fuse_hash_aggregates, fuse_pipelines, lit)

CUT = datetime.date(1995, 3, 15)
LO, HI = datetime.date(1996, 1, 1), datetime.date(1996, 4, 1)


def mem(t):
    return MemoryExec(t.to_batches(max_chunksize=max(1, t.num_rows // 3)), t.schema)


def lineitem(rng, n, nsupp, norders=16, money=pa.int64()):
    price = rng.integers(90_000, 10_500_000, n).astype(np.int64)
    return pa.table({"l_orderkey": rng.integers(1, norders + 1, n).astype(np.int64), "l_suppkey": rng.integers(1, nsupp + 1, n).astype(np.int64),
                     "l_extendedprice": pa.array(price) if money == pa.int64() else pa.array([Decimal(int(x)).scaleb(-2) for x in price], money), "l_discount": rng.integers(0, 11, n).astype(np.int64),
                     "l_shipdate": pa.array(rng.integers(9000, 10300, n).astype(np.int32)).cast(pa.date32())})


def q15_plan(rng=None, mode="Single", n=40, nsupp=100_000, money=pa.int64(), agg="sum"):
    """revenue0: lineitem WHERE l_shipdate in [LO, HI) GROUP BY l_suppkey, SUM(l_extendedprice * (100 - l_discount))"""
    rng = rng if rng is not None else np.random.default_rng(0)
    l = lineitem(rng, n, nsupp, money=money)
    f = GpuFilterExec((col("l_shipdate") >= lit(LO, pa.date32())) & (col("l_shipdate") < lit(HI, pa.date32())), mem(l))
    rev = col("l_extendedprice") if agg == "avg" else col("l_extendedprice") * (lit(100, pa.int64()) - col("l_discount"))
    p = GpuProjectionExec([(col("l_suppkey"), "l_suppkey"), (rev, "rev")], f)
    return GpuAggregateExec(mode, ["l_suppkey"], [AggregateExpr(agg, "rev", "total_revenue")], p)


def q3_by_customer_plan(rng=None, mode="Single", nord=16, n=40, ncust=5, join_type="Inner"):
    """the Q3 join grouped by o_custkey: the orders build pipeline carries o_custkey as payload"""
    rng = rng if rng is not None else np.random.default_rng(0)
    orders = pa.table({"o_orderkey": np.arange(1, nord + 1, dtype=np.int64), "o_custkey": rng.integers(1, ncust + 1, nord).astype(np.int64),
                       "o_orderdate": pa.array(rng.integers(8800, 9300, nord).astype(np.int32)).cast(pa.date32())})
    o = GpuFilterExec(col("o_orderdate") < lit(CUT, pa.date32()), mem(orders), projection=[0, 1])
    l = GpuFilterExec(col("l_shipdate") > lit(CUT, pa.date32()), mem(lineitem(rng, n, 10, nord)), projection=[0, 2, 3])
    inner = GpuHashJoinExec(o, l, [("o_orderkey", "l_orderkey")], join_type)
    p = GpuProjectionExec([(col("o_custkey"), "o_custkey"), (col("l_extendedprice") * (lit(100, pa.int64()) - col("l_discount")), "rev")], inner)
    return GpuAggregateExec(mode, ["o_custkey"], [AggregateExpr("sum", "rev", "revenue"), AggregateExpr("count_star", None, "n")], p)


def test_q15_revenue0_takes_the_hash_sink():
    for mode in ("Single", "SinglePartitioned", "Partial"):
        agg = q15_plan(mode=mode)
        assert fuse_pipelines(agg) is agg                  # the join-keyed and dense sinks cannot carry it
        fused = fuse_hash_aggregates(agg)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash" and fused.mode == mode
        assert fused.group_by == ["l_suppkey"] and fused.nullable == [True] and not fused.scan.stages
        assert fused.schema == agg.schema and [a[0] for a in fused.aggs] == ["sum"]


def test_q3_grouped_by_customer_takes_the_hash_sink():
    for mode in ("Single", "SinglePartitioned", "Partial"):
        agg = q3_by_customer_plan(mode=mode)
        assert fuse_pipelines(agg) is agg
        fused = fuse_hash_aggregates(agg)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "hash" and fused.mode == mode
        assert fused.group_by == ["o_custkey"] and [a[0] for a in fused.aggs] == ["sum", "count_star"]
        (kind, pkey, build), = fused.scan.stages
        assert kind == D.STAGE_INNER and pkey == "l_orderkey" and build.key == "o_orderkey" and build.payload == ["o_custkey"]
        assert build.n_acc_words == 0                      # the hash sink owns its records


def test_shapes_fuse_pipelines_fuses_keep_its_plan():
    from test_fusion_rule_planning import q3_parts, revenue_projection
    _, _, inner = q3_parts()
    agg = GpuAggregateExec("Single", ["l_orderkey", "o_orderdate", "o_shippriority"], [AggregateExpr("sum", "rev", "revenue")], revenue_projection(inner))
    fused = fuse_hash_aggregates(agg)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "aggregate"
    # the twin of fuse_pipelines' unfused `GROUP BY o_shippriority` over the Q3 join: now the hash sink
    by_prio = GpuAggregateExec("Single", ["o_shippriority"], [AggregateExpr("sum", "rev", "revenue")], revenue_projection(inner))
    assert fuse_pipelines(by_prio) is by_prio
    fused = fuse_hash_aggregates(by_prio)
    assert fused.sink == "hash" and fused.group_by == ["o_shippriority"]


def test_what_the_hash_sink_cannot_carry_stays_unfused():
    same = lambda p: fuse_hash_aggregates(p) is p
    agg = q3_by_customer_plan()
    inner = agg.input.input
    # a computed group key
    shifted = GpuProjectionExec([(col("o_custkey") + lit(1, pa.int64()), "k"), (col("l_extendedprice"), "rev")], inner)
    assert same(GpuAggregateExec("Single", ["k"], [AggregateExpr("sum", "rev", "revenue")], shifted))
    # an aggregate FILTER clause
    flt = GpuProjectionExec([(col("o_custkey"), "o_custkey"), (col("l_extendedprice"), "rev"), (col("l_discount") > lit(3, pa.int64()), "keep")], inner)
    assert same(GpuAggregateExec("Single", ["o_custkey"], [AggregateExpr("sum", "rev", "revenue", filter="keep")], flt))
    # Final merges states
    part = q3_by_customer_plan(mode="Partial")
    assert same(GpuAggregateExec("Final", ["o_custkey"], [AggregateExpr("sum", "rev", "revenue"), AggregateExpr("count_star", None, "n")], part,
                                 input_schema=part.input.schema))
    # the topmost join is not Inner
    assert same(q3_by_customer_plan(join_type="Right"))
    # more than 128 key bits: two nullable Int64 columns take 130
    wide = GpuProjectionExec([(col("o_custkey"), "o_custkey"), (col("l_discount"), "l_discount"), (col("l_extendedprice"), "rev")], inner)
    assert same(GpuAggregateExec("Single", ["o_custkey", "l_discount"], [AggregateExpr("sum", "rev", "revenue")], wide))
    # a bare scan: nothing to fuse
    l = lineitem(np.random.default_rng(1), 30, 5)
    assert same(GpuAggregateExec("Single", ["l_suppkey"], [AggregateExpr("sum", "l_extendedprice", "s")], mem(l)))
    bare = GpuProjectionExec([(col("l_suppkey"), "l_suppkey"), (col("l_extendedprice"), "p")], mem(l))
    assert same(GpuAggregateExec("Single", ["l_suppkey"], [AggregateExpr("sum", "p", "s")], bare))
    # AVG over Decimal128 in Partial mode has no pinned state; in Single modes it fuses
    assert same(q15_plan(mode="Partial", money=pa.decimal128(15, 2), agg="avg"))
    assert fuse_hash_aggregates(q15_plan(mode="Single", money=pa.decimal128(15, 2), agg="avg")).sink == "hash"
    # no GROUP BY is fuse_pipelines' dense sink (TPC-H Q6), never the hash sink; more than four aggregates stay unfused
    f = q15_plan().input
    assert fuse_hash_aggregates(GpuAggregateExec("Single", [], [AggregateExpr("sum", "rev", "r")], f)).sink == "dense"
    assert same(GpuAggregateExec("Single", ["l_suppkey"], [AggregateExpr("sum", "rev", f"r{i}") for i in range(5)], f))
