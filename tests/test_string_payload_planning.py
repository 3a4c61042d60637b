"""plan_string_payloads on the CPU: what it rewrites (a carried Utf8 / LargeUtf8 / Utf8View column -> one row-id column per source, UINT32
on a join's build side, INT64 elsewhere; dropped outright when no output needs it; one gather at the root) and what it leaves alone
(read columns, dictionary-coded inputs, plans without strings, returned identical); the output schema, which is the plan's exactly; and
that the fusion rule then fuses the same shapes it fuses with an integer column in the string's place."""
import pyarrow as pa
import pytest

from datafusion_b200.exec import (AggregateExpr, DictionaryEncodeExec, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuLikeExec, GpuPipelineExec,
                                  GpuProjectionExec, GpuStringRowIdExec, GpuStringTakeExec, JoinFilter, LikeExpr, MemoryExec, col, fuse_full_joins,
                                  lit, plan_string_dictionary, plan_string_payloads, plan_string_predicates)

JOIN_TYPES = ["Inner", "Left", "Right", "Full", "LeftSemi", "RightSemi", "LeftAnti", "RightAnti", "LeftMark", "RightMark"]
STRING_TYPES = [pa.string(), pa.large_string(), pa.string_view()]


def src(**fields):
    schema = pa.schema([pa.field(n, t, nullable) for n, (t, nullable) in fields.items()])
    return MemoryExec([pa.RecordBatch.from_pylist([], schema=schema)], schema)


def customer(t=pa.string(), key_nullable=True):
    return src(c_custkey=(pa.int64(), key_nullable), c_name=(t, False), c_comment=(t, True), c_nation=(pa.int32(), True))


def orders(t=pa.string()):
    return src(o_custkey=(pa.int64(), True), o_orderkey=(pa.int64(), False), o_comment=(t, True))


def nodes(plan):
    out = [plan]
    for c in plan.children():
        out += nodes(c)
    return out


def shape(plan):
    """the plan's node types, depth first, with the row-id sources and the gather left out"""
    if isinstance(plan, GpuStringTakeExec):
        return shape(plan.input)
    return [type(plan).__name__] + [s for c in plan.children() if not isinstance(c, (MemoryExec, GpuStringRowIdExec)) for s in shape(c)]


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_join_output_schema_is_the_plans(jt, t):
    plan = GpuHashJoinExec(customer(t), orders(t), [("c_custkey", "o_custkey")], jt)
    out = plan_string_payloads(plan)
    assert out.schema.equals(plan.schema, check_metadata=True)
    assert [f.nullable for f in out.schema] == [f.nullable for f in plan.schema]
    assert not any(isinstance(n, DictionaryEncodeExec) for n in nodes(out))


def test_one_id_per_source_uint32_on_the_build_side_int64_on_the_probe_side():
    plan = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Inner")
    out = plan_string_payloads(plan)
    assert isinstance(out, GpuStringTakeExec)
    join = out.input
    build, probe = join.left, join.right
    assert isinstance(build, GpuStringRowIdExec) and build.build and build.keep == [1, 2]
    assert build.schema.names == ["c_custkey", "c_nation", "__string_row_id_0"] and build.schema.field(2).type == pa.uint32()
    assert isinstance(probe, GpuStringRowIdExec) and not probe.build and probe.schema.field(-1).type == pa.int64()
    assert [s[0] for s in out.spec] == ["col", "take", "take", "col", "col", "col", "take"]


@pytest.mark.parametrize("jt", ["Right", "Full", "Left"])
def test_outer_sides_ids_are_nullable(jt):
    join = plan_string_payloads(GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], jt)).input
    ids = {f.name: f.nullable for f in join.schema if f.name.startswith("__string_row_id_")}
    assert ids == {"__string_row_id_0": jt in ("Right", "Full"), "__string_row_id_1": jt in ("Left", "Full")}


def test_columns_no_output_needs_are_dropped_without_an_id():
    plan = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Inner", projection=[0, 5])
    out = plan_string_payloads(plan)
    assert not isinstance(out, GpuStringTakeExec) and out.schema.equals(plan.schema)
    build, probe = out.left, out.right
    assert isinstance(build, GpuStringRowIdExec) and build.keep == [] and build.schema.names == ["c_custkey", "c_nation"]
    assert isinstance(probe, GpuStringRowIdExec) and probe.keep == [] and probe.schema.names == ["o_custkey", "o_orderkey"]
    # a filter projection that keeps c_comment only: c_name leaves, c_comment is carried
    f = GpuFilterExec(col("c_nation") > lit(3, pa.int32()), customer(), projection=[2, 0])
    out = plan_string_payloads(f)
    assert out.schema.equals(f.schema) and out.input.input.keep == [2] and out.input.input.drop == [1, 2]


def test_join_projection_and_projection_node_are_remapped():
    plan = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Inner", projection=[5, 1, 0])
    out = plan_string_payloads(plan)
    assert out.schema.equals(plan.schema)
    proj = GpuProjectionExec([(col("o_comment"), "note"), (col("c_custkey"), "k")], GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Left"))
    out = plan_string_payloads(proj)
    assert out.schema.equals(proj.schema) and out.spec[0][0] == "take" and out.spec[1] == ("col", 0)


def test_read_columns_stay():
    # a string join key and a raw string predicate are read: nothing else is a string, so the plan comes back identical
    a = src(k=(pa.string(), True), v=(pa.int64(), True))
    b = src(k2=(pa.string(), True), w=(pa.int64(), True))
    plan = GpuHashJoinExec(a, b, [("k", "k2")], "Inner")
    assert plan_string_payloads(plan) is plan
    f = GpuFilterExec(col("k") == lit("x"), a)
    assert plan_string_payloads(f) is f
    # a JoinFilter operand is read; the other string is carried
    c = src(k=(pa.int64(), True), s=(pa.string(), True), t=(pa.string(), True))
    jf = JoinFilter(col("f0") == col("f1"), [("left", 1), ("right", 1)])
    plan = GpuHashJoinExec(c, src(k2=(pa.int64(), True), s2=(pa.string(), True)), [("k", "k2")], "Inner", filter=jf)
    out = plan_string_payloads(plan)
    assert out.input.left.drop == [2] and out.input.right is plan.right and out.schema.equals(plan.schema)
    assert out.input.filter.column_indices == [("left", 1), ("right", 1)]


def test_mask_inputs_stay_and_the_rest_is_carried():
    f = plan_string_predicates(GpuFilterExec(LikeExpr(col("c_comment"), "%special%") & (col("c_nation") > lit(2, pa.int32())), customer(),
                                             projection=[0, 1]))
    assert isinstance(f.input, GpuLikeExec)
    out = plan_string_payloads(f)
    assert out.schema.equals(f.schema)
    row_ids = [n for n in nodes(out) if isinstance(n, GpuStringRowIdExec)]
    assert len(row_ids) == 1 and row_ids[0].keep == [1] and row_ids[0].drop == [1]


def test_plans_without_carried_strings_come_back_identical():
    ints = src(a=(pa.int64(), True), b=(pa.int32(), True))
    ints2 = src(c=(pa.int64(), True))
    for plan in (GpuFilterExec(col("a") > lit(1), ints), GpuHashJoinExec(ints, ints2, [("a", "c")], "Full"),
                 GpuProjectionExec([(col("a"), "a")], ints), ints):
        assert plan_string_payloads(plan) is plan
    coded = src(k=(pa.int64(), True), s=(pa.dictionary(pa.int32(), pa.string()), True))
    plan = GpuHashJoinExec(coded, ints2, [("k", "c")], "Inner")
    assert plan_string_payloads(plan) is plan
    enc = GpuHashJoinExec(DictionaryEncodeExec(customer(), plan_string_dictionary()), ints2, [("c_custkey", "c")], "Inner")
    assert plan_string_payloads(enc) is enc


def test_strings_an_aggregate_does_not_read_leave_at_their_sources():
    """GpuAggregateExec(c_nation; COUNT(o_orderkey)) over a join carrying c_name, c_comment, o_comment: they are dropped at the sources,
    no gather runs under the aggregate, and the fusion rule fuses it as it does with an int32 in the strings' place"""
    def make(t):
        c = src(c_custkey=(pa.int64(), False), c_name=(t, True), c_nation=(pa.int32(), True))
        join = GpuHashJoinExec(c, orders(t), [("c_custkey", "o_custkey")], "Inner")
        return GpuAggregateExec("Single", ["c_nation"], [AggregateExpr("count", "o_orderkey")], join)
    plan = make(pa.string())
    out = plan_string_payloads(plan)
    assert isinstance(out, GpuAggregateExec) and out.schema.equals(plan.schema)
    assert not any(isinstance(n, GpuStringTakeExec) for n in nodes(out))
    row_ids = [n for n in nodes(out) if isinstance(n, GpuStringRowIdExec)]
    assert len(row_ids) == 2 and all(r.keep == [] for r in row_ids)
    with_strings, with_ints = fuse_full_joins(out), fuse_full_joins(make(pa.int32()))
    assert isinstance(with_ints, GpuPipelineExec) and isinstance(with_strings, GpuPipelineExec) and shape(with_strings) == shape(with_ints)
    # a string the aggregate groups on is read: it stays as it is, the other carried strings go
    join = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Inner")
    agg = GpuAggregateExec("Single", ["c_name"], [AggregateExpr("count", "o_orderkey")], join)
    out = plan_string_payloads(agg)
    build = out.input.left
    assert isinstance(build, GpuStringRowIdExec) and build.drop == [2] and build.keep == [] and "c_name" in build.schema.names


def test_the_rule_reaches_operators_under_a_node_it_does_not_pass_through():
    join = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Inner")
    agg = GpuAggregateExec("Single", ["c_nation"], [AggregateExpr("count", "o_orderkey")], join)
    top = GpuFilterExec(col("c_nation") > lit(1, pa.int32()), agg)
    out = plan_string_payloads(top)
    assert out.schema.equals(top.schema) and isinstance(out.input, GpuAggregateExec) and out.input is not agg
    assert [type(n) for n in nodes(out)].count(GpuStringRowIdExec) == 2


@pytest.mark.parametrize("jt", ["Inner", "Right", "Full", "Left", "RightSemi"])
def test_probe_sides_of_probe_order_joins_release_in_order(jt):
    out = plan_string_payloads(GpuHashJoinExec(customer(), GpuFilterExec(col("o_orderkey") > lit(3), orders()), [("c_custkey", "o_custkey")], jt))
    probe_keys = {k for k, build in out.sources.items() if not build}
    assert probe_keys and out.ordered == probe_keys
    assert not {k for k, build in out.sources.items() if build} & out.ordered
    # a probe side under the build side of an upper join is not in order
    inner = GpuHashJoinExec(customer(), orders(), [("c_custkey", "o_custkey")], "Inner")
    upper = GpuHashJoinExec(inner, src(k=(pa.int64(), True)), [("o_orderkey", "k")], "Inner")
    assert plan_string_payloads(upper).ordered == set()


def _fusion_pair(make, t):
    """the plan with string columns through plan_string_payloads and the fusion rule, and the same plan with int32 in their place"""
    return fuse_full_joins(plan_string_payloads(make(t))), fuse_full_joins(make(pa.int32()))


def _inner(t):
    c = src(c_custkey=(pa.int64(), False), c_name=(t, True))
    o = src(o_custkey=(pa.int64(), True), o_orderkey=(pa.int64(), False), o_comment=(t, True))
    return GpuHashJoinExec(c, GpuFilterExec(col("o_orderkey") > lit(5), o), [("c_custkey", "o_custkey")], "Inner")


def _outer(jt):
    def make(t):
        c = src(c_custkey=(pa.int64(), False), c_name=(t, True))
        o = src(o_custkey=(pa.int64(), True), o_orderkey=(pa.int64(), False), o_comment=(t, True))
        j = GpuHashJoinExec(c, o, [("c_custkey", "o_custkey")], jt)
        return GpuProjectionExec([(col("o_orderkey"), "o_orderkey"), (col("c_name"), "c_name"), (col("o_comment"), "o_comment")], j)
    return make


def _left_semi(t):
    c = src(c_custkey=(pa.int64(), False), c_name=(t, True))
    o = src(o_custkey=(pa.int64(), True), o_comment=(t, True))
    return GpuHashJoinExec(c, o, [("c_custkey", "o_custkey")], "LeftSemi")


def _too_wide(t):      # a Right join whose build carries the key (64 bits) and a string: 96 bits of payload, as with an int32
    c = src(c_custkey=(pa.int64(), False), c_name=(t, True))
    o = src(o_custkey=(pa.int64(), True), o_orderkey=(pa.int64(), False))
    return GpuHashJoinExec(c, o, [("c_custkey", "o_custkey")], "Right")


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
@pytest.mark.parametrize("make,fused", [(_inner, True), (_outer("Right"), True), (_outer("Full"), True), (_left_semi, True), (_too_wide, False)],
                         ids=["inner", "right", "full", "left_semi", "too_wide"])
def test_fusion_fuses_what_it_fuses_with_an_integer_in_the_strings_place(make, fused, t):
    with_strings, with_ints = _fusion_pair(make, t)
    assert isinstance(with_strings, GpuStringTakeExec)
    assert isinstance(with_strings.input, GpuPipelineExec) == fused == isinstance(with_ints, GpuPipelineExec)
    assert shape(with_strings) == shape(with_ints)
    assert with_strings.schema.equals(make(t).schema)
