"""Planning decisions of plan_string_predicates (no GPU needed): which string comparisons and IN lists it rewrites into a GpuLikeExec mask
and `mask = 1` (each operator, a literal on the left, IN / NOT IN, under AND / OR / NOT, beside LIKE, a NULL literal or list item), which
it leaves alone (a column against a column, a non-string IN list, a column read above the filter, an oversize list), that the filter keeps
its schema, and that the fusion rules fuse the Q3 / Q12 / Q19 shapes with the masks as pipeline sources."""
import numpy as np
import pyarrow as pa

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, BinaryExpr, Column, DictionaryEncodeExec, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec,
                                  GpuLikeExec, GpuPipelineExec, InListExpr, LikeExpr, Literal, MemoryExec, col, fuse_pipelines, lit,
                                  plan_like_predicates, plan_string_dictionary, plan_string_predicates)

OPS = {D.OP_EQ: D.OP_EQ, D.OP_NEQ: D.OP_NEQ, D.OP_LT: D.OP_GT, D.OP_LTEQ: D.OP_GTEQ, D.OP_GT: D.OP_LT, D.OP_GTEQ: D.OP_LTEQ}


def lineitem(t=pa.string()):
    tab = pa.table({"l_orderkey": pa.array(np.arange(1, 9, dtype=np.int64)), "l_shipmode": pa.array(["MAIL", "SHIP", None, "AIR", "", "RAIL", "FOB", "x"], t),
                    "l_other": pa.array(["a", "b", "c", "d", "e", "f", "g", "h"], t), "l_x": pa.array(np.arange(8, dtype=np.int64))})
    return MemoryExec(tab.to_batches(), tab.schema)


def masks(plan):
    assert isinstance(plan, GpuFilterExec) and isinstance(plan.input, GpuLikeExec)
    return plan.input


def is_mask_eq(e, name):
    return isinstance(e, BinaryExpr) and e.op == D.OP_EQ and isinstance(e.left, Column) and e.left.name == name and e.right.value == 1


def test_each_operator_and_a_literal_on_the_left():
    for t in (pa.string(), pa.large_string(), pa.string_view()):
        src = lineitem(t)
        for op, mirrored in OPS.items():
            for pred, want_op in ((BinaryExpr(col("l_shipmode"), op, lit("MAIL")), op), (BinaryExpr(lit("MAIL"), op, col("l_shipmode")), mirrored)):
                f = GpuFilterExec(pred, src, projection=[0, 3])
                r = plan_string_predicates(f)
                lk = masks(r)
                assert r.schema == f.schema and "l_shipmode" not in lk.schema.names
                (e, name), = lk.likes
                assert isinstance(e, BinaryExpr) and e.op == want_op and e.left.name == "l_shipmode" and e.right.value == "MAIL"
                assert is_mask_eq(r.predicate, name) and lk.schema.field(name).type == pa.uint8()


def test_in_and_not_in_under_and_or_not_and_beside_like():
    src = lineitem()
    ml = InListExpr(col("l_shipmode"), ["MAIL", "SHIP"])
    for pred, n_masks in ((ml, 1), (InListExpr(col("l_shipmode"), ["MAIL"], negated=True), 1), (ml & (col("l_x") > lit(2)), 1),
                          ((col("l_x") > lit(2)) | ~ml, 1), (~(ml & (col("l_other") < lit("c"))), 2),
                          (ml & LikeExpr(col("l_other"), "%a%") & (col("l_shipmode") != lit("AIR")), 3)):
        f = GpuFilterExec(pred, src, projection=[0])
        r = plan_string_predicates(f)
        lk = masks(r)
        assert r.schema == f.schema and len(lk.likes) == n_masks
        read = {(e.left if isinstance(e, BinaryExpr) else e.expr).name for e, _ in lk.likes}
        assert "l_shipmode" in read and not read & set(lk.schema.names)                   # read by nothing but the masks: dropped
        nodes: list = []
        r.predicate.rpn(lk.schema, nodes)                                    # an ordinary expression program now
        assert sum(1 for k in nodes if k[0] == D.EXPR_COLUMN and lk.schema.field(k[1]).type == pa.uint8()) == n_masks


def test_null_literal_and_null_list_item():
    src = lineitem()
    r = plan_string_predicates(GpuFilterExec((col("l_shipmode") == lit(None, pa.string())) | (col("l_x") > lit(2)), src, projection=[0]))
    assert not isinstance(r.input, GpuLikeExec) and isinstance(r.predicate.left, Literal) and r.predicate.left.value is None
    for neg, op in ((False, D.OP_OR), (True, D.OP_AND)):
        r = plan_string_predicates(GpuFilterExec(InListExpr(col("l_shipmode"), ["MAIL", None], negated=neg), src, projection=[0]))
        (e, name), = masks(r).likes
        assert [v.value for v in e.list] == ["MAIL"] and e.negated == neg
        p = r.predicate
        assert p.op == op and is_mask_eq(p.left, name) and isinstance(p.right, Literal) and p.right.value is None


def test_filters_left_alone():
    src = lineitem()
    same = lambda f: plan_string_predicates(f) is f  # noqa: E731
    assert same(GpuFilterExec(col("l_shipmode") == col("l_other"), src, projection=[0]))                            # column against column
    assert same(GpuFilterExec((col("l_shipmode") == col("l_other")) & (col("l_shipmode") == lit("MAIL")), src, projection=[0]))
    assert same(GpuFilterExec(InListExpr(col("l_x"), [lit(1), lit(2)]), src, projection=[0]))                      # not a string IN list
    assert same(GpuFilterExec(InListExpr(col("l_shipmode"), [lit("MAIL"), col("l_other")]), src, projection=[0]))   # a column in the list
    assert same(GpuFilterExec(col("l_shipmode") == lit("MAIL"), src, projection=[0, 1]))                            # read above the filter
    assert same(GpuFilterExec(InListExpr(col("l_shipmode"), ["MAIL"]), src))                                        # all columns above
    assert same(GpuFilterExec(InListExpr(col("l_shipmode"), [f"v{i}" for i in range(65)]), src, projection=[0]))   # 65 distinct values
    assert same(GpuFilterExec(InListExpr(col("l_shipmode"), ["x" * 600, "y" * 425]), src, projection=[0]))        # 1025 bytes
    assert same(GpuFilterExec(col("l_shipmode") < lit("x" * 257), src, projection=[0]))                            # literal over 256 bytes
    assert same(GpuFilterExec(col("l_x") > lit(2), src, projection=[0]))                                            # no string predicate
    at_caps = GpuFilterExec(InListExpr(col("l_shipmode"), [f"v{i}" for i in range(64)] * 2), src, projection=[0])
    assert isinstance(plan_string_predicates(at_caps).input, GpuLikeExec)


def test_raw_dictionary_type_is_left_alone_and_coded_columns_use_the_code_map():
    tab = pa.table({"k": np.arange(4, dtype=np.int64), "s": pa.array(["a", "b", "a", None]).dictionary_encode()})
    raw = GpuFilterExec(col("s") == lit("a"), MemoryExec(tab.to_batches(), tab.schema), projection=[0])
    assert plan_string_predicates(raw) is raw
    enc = DictionaryEncodeExec(lineitem(), plan_string_dictionary())
    f = GpuFilterExec(InListExpr(col("l_shipmode"), ["MAIL", "SHIP"]) & (col("l_other") >= lit("c")), enc)   # the codes may go above
    r = plan_string_predicates(f)
    lk = masks(r)
    assert lk.dictionary_of is enc.dictionary_of and "l_shipmode" in lk.schema.names and r.schema == f.schema
    hand = GpuFilterExec(col("l_shipmode") == lit(3, pa.int32()), enc)                                           # a hand-written code
    assert plan_string_predicates(hand) is hand


def test_plan_like_predicates_keeps_to_like():
    src = lineitem()
    f = GpuFilterExec(LikeExpr(col("l_other"), "%a%") & (col("l_shipmode") == lit("MAIL")), src, projection=[0])
    r = plan_like_predicates(f)
    (e, _), = masks(r).likes
    assert isinstance(e, LikeExpr) and "l_shipmode" in r.input.schema.names
    assert plan_like_predicates(GpuFilterExec(InListExpr(col("l_shipmode"), ["MAIL"]), src, projection=[0])).input is src


# ---- fused shapes: the masks are pipeline sources ----
def q19_arm():
    rng = np.random.default_rng(0)
    part = pa.table({"p_partkey": np.arange(1, 9, dtype=np.int64), "p_brand": pa.array([f"Brand#{i}" for i in range(11, 19)], pa.string_view()),
                     "p_container": pa.array(["SM CASE", "SM BOX", "LG BOX", "SM PKG", "JUMBO JAR", "SM PACK", "MED BAG", "SM CASE"], pa.large_string())})
    li = pa.table({"l_partkey": rng.integers(1, 9, 40).astype(np.int64), "l_price": np.arange(40, dtype=np.int64),
                   "l_shipinstruct": pa.array(["DELIVER IN PERSON", "NONE"] * 20)})
    pf = GpuFilterExec((col("p_brand") == lit("Brand#12")) & InListExpr(col("p_container"), ["SM CASE", "SM BOX", "SM PACK", "SM PKG"]),
                       MemoryExec(part.to_batches(), part.schema), projection=[0])
    lf = GpuFilterExec(lit("DELIVER IN PERSON") == col("l_shipinstruct"), MemoryExec(li.to_batches(), li.schema), projection=[0, 1])
    join = GpuHashJoinExec(pf, lf, [("p_partkey", "l_partkey")], "Inner")
    return GpuAggregateExec("Single", ["l_partkey"], [AggregateExpr("sum", "l_price", "revenue")], join)


def test_q19_arm_fuses_with_masks_on_both_sides():
    plan = q19_arm()
    r = plan_string_predicates(plan)
    assert r.schema == plan.schema
    fused = fuse_pipelines(r)
    assert isinstance(fused, GpuPipelineExec) and isinstance(fused.scan.source, GpuLikeExec)
    kind, _, build = fused.scan.stages[0]
    assert kind == D.STAGE_INNER and isinstance(build.scan.source, GpuLikeExec)


def test_q12_filter_fuses_into_an_aggregate():
    tab = pa.table({"l_price": np.arange(8, dtype=np.int64), "l_shipmode": pa.array(["MAIL", "SHIP", None, "AIR", "", "RAIL", "FOB", "x"]),
                    "l_late": np.arange(8, dtype=np.int32) % 2})
    f = GpuFilterExec(InListExpr(col("l_shipmode"), ["MAIL", "SHIP"]), MemoryExec(tab.to_batches(), tab.schema), projection=[0, 2])
    agg = GpuAggregateExec("Single", ["l_late"], [AggregateExpr("sum", "l_price", "s")], f)
    fused = fuse_pipelines(plan_string_predicates(agg))
    assert isinstance(fused, GpuPipelineExec) and isinstance(fused.scan.source, GpuLikeExec)
