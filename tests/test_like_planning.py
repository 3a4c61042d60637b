"""Planning decisions of plan_like_predicates (no GPU needed): which FilterExec predicates with LikeExpr it rewrites into a GpuLikeExec
mask and `mask = 1`, which it leaves alone, that the rewritten filter keeps its schema, and that the fusion rules fuse a LIKE-filtered
TPC-H Q13 / Q9 shape into the same stages and sink as the same plan with an integer predicate."""
import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, BinaryExpr, DictionaryEncodeExec, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuLikeExec,
                                  GpuPipelineExec, LikeExpr, Literal, MemoryExec, UnaryExpr, col, fuse_pipelines, lit, plan_string_dictionary,
                                  plan_like_predicates)


def orders(t=pa.string()):
    tab = pa.table({"o_orderkey": pa.array(np.arange(1, 9, dtype=np.int64)), "o_custkey": pa.array(np.arange(8, dtype=np.int64) % 3 + 1),
                    "o_comment": pa.array(["special requests", "x", None, "y", "special z requests", "", "a", "b"], t),
                    "o_x": pa.array(np.arange(8, dtype=np.int64)), "o_comment_int": pa.array(np.arange(8, dtype=np.int64))})
    return MemoryExec(tab.to_batches(), tab.schema)


NOT_LIKE = LikeExpr(col("o_comment"), "%special%requests%", negated=True)


def masks(plan):
    assert isinstance(plan, GpuFilterExec) and isinstance(plan.input, GpuLikeExec)
    return plan.input


def test_like_and_not_like_under_and_or_not_are_rewritten():
    for t in (pa.string(), pa.large_string(), pa.string_view()):
        src = orders(t)
        for pred in (NOT_LIKE, NOT_LIKE & (col("o_x") > lit(2)), (col("o_x") > lit(2)) | LikeExpr(col("o_comment"), "special%"), ~NOT_LIKE,
                     ~(LikeExpr(col("o_comment"), "%a%") & LikeExpr(col("o_comment"), "_", negated=True))):
            f = GpuFilterExec(pred, src, projection=[0, 1, 3])
            r = plan_like_predicates(f)
            lk = masks(r)
            assert r.schema == f.schema
            assert "o_comment" not in lk.schema.names                       # read by nothing but the LIKEs: dropped
            assert all(lk.schema.field(n).type == pa.uint8() for _, n in lk.likes)
            nodes: list = []
            r.predicate.rpn(lk.schema, nodes)                                # an ordinary expression program now
            assert sum(1 for k in nodes if k[0] == D.EXPR_COLUMN and lk.schema.field(k[1]).type == pa.uint8()) == len(lk.likes)


def test_mask_compares_equal_to_one():
    r = plan_like_predicates(GpuFilterExec(NOT_LIKE, orders(), projection=[0]))
    p = r.predicate
    assert isinstance(p, BinaryExpr) and p.op == D.OP_EQ and isinstance(p.right, Literal) and p.right.value == 1 and p.right.type == pa.uint8()
    (e, name), = masks(r).likes
    assert e is NOT_LIKE and p.left.name == name


def test_filters_left_alone():
    src = orders()
    same = lambda f: plan_like_predicates(f) is f  # noqa: E731
    assert same(GpuFilterExec(LikeExpr(col("o_comment"), "%special%", case_insensitive=True), src, projection=[0]))      # ILIKE
    assert same(GpuFilterExec(LikeExpr(col("o_comment"), col("o_comment")), src, projection=[0]))                      # column pattern
    assert same(GpuFilterExec(LikeExpr(col("o_comment"), "%50\\%%"), src, projection=[0]))                              # `\`
    assert same(GpuFilterExec(NOT_LIKE, src, projection=[0, 2]))                                                         # read above
    assert same(GpuFilterExec(NOT_LIKE, src))                                                                            # all columns above
    assert same(GpuFilterExec(NOT_LIKE & LikeExpr(col("o_comment"), "a%", case_insensitive=True), src, projection=[0]))  # one LIKE stays
    assert same(GpuFilterExec(col("o_x") > lit(2), src, projection=[0]))                                                 # no LIKE
    assert same(GpuFilterExec(LikeExpr(col("o_x"), "1%"), src, projection=[0]))                                        # not a string column


def test_column_read_by_the_rest_of_the_predicate_is_kept():
    f = GpuFilterExec(NOT_LIKE & col("o_comment").is_not_null(), orders(), projection=[0])
    r = plan_like_predicates(f)
    assert "o_comment" in masks(r).schema.names and r.schema == f.schema


def test_null_pattern_folds_to_null():
    f = GpuFilterExec(LikeExpr(col("o_comment"), None) | (col("o_x") > lit(2)), orders(), projection=[0])
    r = plan_like_predicates(f)
    assert isinstance(r, GpuFilterExec) and not isinstance(r.input, GpuLikeExec) and r.schema == f.schema
    assert isinstance(r.predicate.left, Literal) and r.predicate.left.value is None


def test_dictionary_coded_column():
    enc = DictionaryEncodeExec(orders(), plan_string_dictionary())
    f = GpuFilterExec(LikeExpr(col("o_comment"), "%special%"), enc)           # the INT32 codes may go above the filter
    r = plan_like_predicates(f)
    lk = masks(r)
    assert lk.dictionary_of is enc.dictionary_of and "o_comment" in lk.schema.names and r.schema == f.schema


def test_rewrite_reaches_filters_below_joins_and_aggregates():
    plan = q13(NOT_LIKE)
    r = plan_like_predicates(plan)
    assert r is not plan and r.schema == plan.schema
    assert isinstance(r.input.right.input, GpuLikeExec) and plan.input.right.input is orders_q13


# ---- Q13 / Q9 shapes: a LIKE predicate fuses exactly as an integer predicate ----
def customer():
    t = pa.Table.from_arrays([np.arange(1, 9, dtype=np.int64)], schema=pa.schema([pa.field("c_custkey", pa.int64(), False)]))
    return MemoryExec(t.to_batches(), t.schema)


orders_q13 = orders()


def q13(pred):
    f = GpuFilterExec(pred, orders_q13, projection=[0, 1])
    join = GpuHashJoinExec(customer(), f, [("c_custkey", "o_custkey")], "Left")
    return GpuAggregateExec("Single", ["c_custkey"], [AggregateExpr("count", "o_orderkey", "c_count")], join)


def shape(p):
    assert isinstance(p, GpuPipelineExec)
    return (p.sink, p.key, list(p.payload), list(p.group_by), [(k, pk, shape(b)) for k, pk, b in p.scan.stages], p.schema)


def test_q13_like_fuses_as_the_integer_predicate():
    a = fuse_pipelines(plan_like_predicates(q13(NOT_LIKE)))
    b = fuse_pipelines(q13(col("o_comment_int") < lit(6)))
    assert shape(a) == shape(b)
    assert a.scan.stages[-1][0] == D.STAGE_LEFT and a.sink == "aggregate"
    assert isinstance(a.scan.source, GpuLikeExec)


def part(t=pa.string()):
    tab = pa.table({"p_partkey": np.arange(1, 9, dtype=np.int64), "p_name": pa.array(["green x", "red", "dark green", "blue", None, "g", "green", "x"], t),
                    "p_int": np.arange(8, dtype=np.int64)})
    return MemoryExec(tab.to_batches(), tab.schema)


def q9(pred):
    lineitem = pa.table({"l_partkey": np.arange(20, dtype=np.int64) % 8 + 1, "l_qty": np.arange(20, dtype=np.int64)})
    build = GpuFilterExec(pred, part(), projection=[0])
    join = GpuHashJoinExec(build, MemoryExec(lineitem.to_batches(), lineitem.schema), [("p_partkey", "l_partkey")], "Inner")
    return GpuAggregateExec("Single", ["l_partkey"], [AggregateExpr("sum", "l_qty", "s")], join)


def test_q9_like_on_the_build_side_fuses_as_the_integer_predicate():
    a = fuse_pipelines(plan_like_predicates(q9(LikeExpr(col("p_name"), "%green%"))))
    b = fuse_pipelines(q9(col("p_int") < lit(3)))
    assert shape(a) == shape(b)
    kind, _, build = a.scan.stages[0]
    assert kind == D.STAGE_INNER and isinstance(build.scan.source, GpuLikeExec)
