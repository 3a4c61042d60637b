"""The fusion rule's dense branch as a PLANNING decision (no GPU needed: nothing is executed): AggregateExec over [ProjectionExec]
over FilterExec over a source, with no join, becomes a GpuPipelineExec with the dense-group aggregate sink when the GROUP BY columns
are source columns whose bounds are known and span at most DENSE_MAX_GROUPS slots (TPC-H Q1, Q6).  Everything else is handed back
untouched."""
import datetime
from decimal import Decimal

import numpy as np
import pyarrow as pa

from datafusion_b200.exec import (AggregateExpr, ExecutionPlan, GpuAggregateExec, GpuFilterExec, GpuPipelineExec, GpuProjectionExec, MemoryExec,
                                  col, fuse_pipelines, lit)

CUT = datetime.date(1998, 9, 2)
DEC = pa.decimal128(15, 2)


def lineitem(decimal=False, n=40, flag_hi=2):
    money = (lambda v: pa.array([int(x) for x in v], pa.int64())) if not decimal else (lambda v: pa.array([Decimal(int(x)).scaleb(-2) for x in v], DEC))
    r = np.arange(n)
    t = pa.table({"l_returnflag": pa.array(r % (flag_hi + 1), pa.int32()), "l_linestatus": pa.array(r % 2, pa.int8()),
                  "l_shipdate": pa.array((10_000 + r % 800).astype(np.int32)).cast(pa.date32()),
                  "l_quantity": money(100 * (r % 50 + 1)), "l_extendedprice": money(r * 100 + 90_000), "l_discount": money(r % 11),
                  "l_tax": money(r % 9)})
    return MemoryExec(t.to_batches(max_chunksize=16), t.schema)


def q1(decimal=False, mode="Single", src=None, filter_clause=None):
    src = src or lineitem(decimal)
    f = GpuFilterExec(col("l_shipdate") <= lit(CUT, pa.date32()), src)
    one = lit(1, pa.decimal128(20, 0)) if decimal else lit(100, pa.int64())
    disc_price = col("l_extendedprice") * (one - col("l_discount"))
    proj = GpuProjectionExec([(col("l_returnflag"), "l_returnflag"), (col("l_linestatus"), "l_linestatus"), (col("l_quantity"), "l_quantity"),
                              (col("l_extendedprice"), "l_extendedprice"), (disc_price, "disc_price"),
                              (disc_price * (one + col("l_tax")), "charge"),
                              ((col("l_quantity") if decimal else col("l_quantity").cast(pa.float64())), "qty_avg"),
                              ((col("l_discount") if decimal else col("l_discount").cast(pa.float64())), "disc_avg"),
                              (col("l_shipdate") > lit(CUT, pa.date32()), "late")], f)
    aggs = [AggregateExpr("sum", "l_quantity", "sum_qty"), AggregateExpr("sum", "l_extendedprice", "sum_base_price"),
            AggregateExpr("sum", "disc_price", "sum_disc_price"), AggregateExpr("sum", "charge", "sum_charge"),
            AggregateExpr("avg", "qty_avg", "avg_qty"), AggregateExpr("avg", "disc_avg", "avg_disc"),
            AggregateExpr("count_star", None, "count_order", filter=filter_clause)]
    return GpuAggregateExec(mode, ["l_returnflag", "l_linestatus"], aggs, proj)


def q6(decimal=False, mode="Single"):
    src = lineitem(decimal)
    d = (lambda v: lit(Decimal(v).scaleb(-2), DEC)) if decimal else (lambda v: lit(v, pa.int64()))
    pred = ((col("l_shipdate") >= lit(datetime.date(1994, 1, 1), pa.date32())) & (col("l_shipdate") < lit(datetime.date(1995, 1, 1), pa.date32()))
            & (col("l_discount") >= d(5)) & (col("l_discount") <= d(7)) & (col("l_quantity") < d(2400)))
    proj = GpuProjectionExec([(col("l_extendedprice") * col("l_discount"), "rev")], GpuFilterExec(pred, src))
    return GpuAggregateExec(mode, [], [AggregateExpr("sum", "rev", "revenue")], proj)


def test_rule_fuses_q1_and_q6_shapes_into_dense_pipelines():
    for decimal in (False, True):
        for mode in ("Single", "SinglePartitioned"):
            agg = q1(decimal, mode)
            fused = fuse_pipelines(agg)
            assert isinstance(fused, GpuPipelineExec) and fused.sink == "dense" and fused.schema == agg.schema
            assert fused.group_by == ["l_returnflag", "l_linestatus"] and fused.key_range == [(0, 2), (0, 1)] and not fused.scan.stages
            assert [a[0] for a in fused.aggs] == ["sum", "sum", "sum", "sum", "avg", "avg", "count_star"]
            fused = fuse_pipelines(q6(decimal, mode))
            assert isinstance(fused, GpuPipelineExec) and fused.sink == "dense" and fused.group_by == [] and fused.key_range == []
    assert fuse_pipelines(q1(False, "Partial")).sink == "dense"                 # Float64 AVG has the [count, sum] state
    assert q1(True).schema.field("avg_qty").type == pa.decimal128(19, 6)        # Avg::return_type over Decimal128(15,2)
    assert q1(True).schema.field("sum_qty").type == pa.decimal128(25, 2)


def test_rule_fuses_a_filter_without_projection():
    agg = GpuAggregateExec("Single", ["l_linestatus"], [AggregateExpr("max", "l_tax", "m")],
                           GpuFilterExec(col("l_quantity") > lit(0, pa.int64()), lineitem()))
    fused = fuse_pipelines(agg)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "dense" and fused.key_range == [(0, 1)]


def test_rule_leaves_alone_what_the_dense_sink_cannot_carry():
    same = lambda p: fuse_pipelines(p) is p
    # bounds unknown: a source without statistics
    class Stream(ExecutionPlan):
        def __init__(self, m): self.m, self.schema = m, m.schema
        def execute(self, ctx): return self.m.execute(ctx)
    assert same(q1(src=Stream(lineitem())))
    assert fuse_pipelines(q6()).sink == "dense" and not same(q6())
    # bounds unknown: the group column is not a source column with statistics (a projection below the filter, a computed key)
    below = GpuProjectionExec([(col("l_returnflag"), "l_returnflag"), (col("l_linestatus"), "l_linestatus")], lineitem())
    assert same(GpuAggregateExec("Single", ["l_returnflag", "l_linestatus"], [AggregateExpr("count", None, "n")],
                                 GpuFilterExec(col("l_returnflag") > lit(0, pa.int32()), below)))
    computed = GpuProjectionExec([(col("l_returnflag") + lit(1, pa.int32()), "k"), (col("l_quantity"), "q")],
                                 GpuFilterExec(col("l_quantity") > lit(0, pa.int64()), lineitem()))
    assert same(GpuAggregateExec("Single", ["k"], [AggregateExpr("sum", "q", "s")], computed))
    # a domain over 256 slots: 255 flag values + NULL = 256 slots fits, 256 values + NULL does not
    wide = GpuAggregateExec("Single", ["l_returnflag"], [AggregateExpr("count", None, "n")],
                            GpuFilterExec(col("l_quantity") > lit(0, pa.int64()), lineitem(n=400, flag_hi=255)))
    assert same(wide)
    fits = GpuAggregateExec("Single", ["l_returnflag"], [AggregateExpr("count", None, "n")],
                            GpuFilterExec(col("l_quantity") > lit(0, pa.int64()), lineitem(n=400, flag_hi=254)))
    assert fuse_pipelines(fits).sink == "dense"
    # FILTER clauses, Final mode, Partial with a decimal AVG
    assert same(q1(filter_clause="late"))
    assert same(q1(False, "Final"))
    assert same(q1(True, "Partial"))
    assert fuse_pipelines(q6(True, "Partial")).sink == "dense"                  # no AVG: Partial is fine
