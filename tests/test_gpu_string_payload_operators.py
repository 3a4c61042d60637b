"""Carried string columns through the GPU operators as row ids (plan_string_payloads) and gathered on the GPU (dfgpu_string_take),
against the same plan routed through DictionaryEncodeExec / DictionaryDecodeExec and against a pyarrow evaluation on the strings (each
source row carries its row number, so every gathered string must be its source's string at that row): the filter across batches its
coalescer merges, all ten join types with NULL keys under NullEqualsNothing and NullEqualsNull, and the fused output-sink plans (the
ordered Inner chain, RIGHT, FULL) and a LeftSemi onto the join-keyed sink.  The unfused operators keep their order, so those compare
row for row; a fused plan against the unfused dictionary route compares sorted (DESIGN §4).  The unordered output sink is not among
the fused cases: the twin's fusion rule only plans the ordered one, so no plan reaches it.  The store's held-bytes metric is checked
where its release rule lowers the peak: the filter and a join's probe side.  (The fused ordered sink emits after its finish, so its
probe batches are released as its output drains, not before.)"""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_b200.exec import (DictionaryDecodeExec, DictionaryEncodeExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec,
                                  GpuStringTakeExec, LikeExpr, MemoryExec, SessionConfig, TaskContext, col, collect, fuse_full_joins, lit,
                                  plan_string_dictionary, plan_string_payloads, plan_string_predicates)

pytestmark = pytest.mark.gpu

JOIN_TYPES = ["Inner", "Left", "Right", "Full", "LeftSemi", "RightSemi", "LeftAnti", "RightAnti", "LeftMark", "RightMark"]
TYPES = [pa.string(), pa.large_string(), pa.string_view()]
WORDS = ["furiously", "special", "requests", "ß", "deposits", "日本", "x", "packages", "quickly", "😀", "Customer#", "blithely"]
SOURCES = {"l_name": "lrow", "l_comment": "lrow", "r_comment": "rrow"}      # string column -> the row-number column of its source


def texts(rng, n, null_p=0.1, long_p=0.01):
    out = []
    for _ in range(n):
        r = rng.random()
        out.append(None if r < null_p else "".join(rng.choice(WORDS, int(rng.integers(40, 300)))) if r < null_p + long_p
                   else " ".join(rng.choice(WORDS, int(rng.integers(0, 8)))))
    return out


def mem(t, chunk):
    return MemoryExec(t.to_batches(max_chunksize=chunk), t.schema)


def left_table(rng, n, t, unique=False, key_nullable=True):
    k = rng.permutation(n * 2)[:n] if unique else rng.integers(0, n // 3, n)
    mask = rng.random(n) < 0.05 if key_nullable else None
    schema = pa.schema([pa.field("lk", pa.int64(), key_nullable), pa.field("lrow", pa.int64(), False), pa.field("l_name", t, True),
                        pa.field("l_comment", t, True)])
    return pa.table([pa.array(k, pa.int64(), mask=mask), pa.array(np.arange(n), pa.int64()), pa.array(texts(rng, n, 0.0)).cast(t),
                     pa.array(texts(rng, n)).cast(t)], schema=schema)


def right_table(rng, n, nl, t):
    return pa.table({"rk": pa.array(rng.integers(0, nl // 2, n), pa.int64(), mask=rng.random(n) < 0.05), "rrow": pa.array(np.arange(n), pa.int64()),
                     "r_comment": pa.array(texts(rng, n)).cast(t)})


def table(plan, tc):
    return pa.Table.from_batches(collect(plan, tc), plan.schema)


def dictionary_route(make, left, right, chunk):
    d = plan_string_dictionary()
    plan = make(DictionaryEncodeExec(mem(left, chunk), d), DictionaryEncodeExec(mem(right, chunk), d) if right is not None else None)
    names = [n for n in plan.schema.names if n in SOURCES]
    return DictionaryDecodeExec(plan, names, d, pa.string())


def rows(tab, ordered=True):
    cols = [c.combine_chunks() for c in tab.columns]
    cols = [c.cast(pa.large_string()) if pa.types.is_string(c.type) or pa.types.is_string_view(c.type) or pa.types.is_large_string(c.type) else c
            for c in cols]
    out = list(zip(*[c.to_pylist() for c in cols])) if cols else []
    return out if ordered else sorted(out, key=repr)


def check_strings(got, left, right):
    """every gathered string is its source's string at the row its row-number column names (NULL where that is NULL), where the output
    keeps that column"""
    srcs = {"lrow": left, "rrow": right}
    for name, rowcol in SOURCES.items():
        if name in got.schema.names and rowcol in got.schema.names:
            exp = pc.take(srcs[rowcol][name].combine_chunks().cast(pa.large_string()), got[rowcol].combine_chunks())
            assert got[name].combine_chunks().cast(pa.large_string()).equals(exp), name


def run_both(make, left, right, chunk, tc, fuse=False):
    plain = make(mem(left, chunk), mem(right, chunk) if right is not None else None)
    plan = plan_string_payloads(plain)
    assert isinstance(plan, GpuStringTakeExec) and not any(isinstance(n, DictionaryEncodeExec) for n in _nodes(plan))
    if fuse:
        plan = fuse_full_joins(plan)
        assert isinstance(plan.input, GpuPipelineExec)
    got = table(plan, tc)
    assert got.schema.equals(plain.schema)
    exp = table(dictionary_route(make, left, right, chunk), tc)
    assert rows(got, not fuse) == rows(exp, not fuse)
    check_strings(got, left, right)
    assert plan.metrics()["string_bytes_held"] == 0
    return plan, got


def _nodes(plan):
    out = [plan]
    for c in plan.children():
        out += _nodes(c)
    return out


@pytest.fixture(scope="module")
def tc(gpu_ctx):
    return TaskContext(SessionConfig(batch_size=8192), gpu_ctx)


@pytest.mark.parametrize("t", TYPES, ids=str)
def test_filter_across_coalesced_batches_releases_what_no_later_batch_reads(tc, t):
    rng = np.random.default_rng(1)
    left = left_table(rng, 60000, t)
    make = lambda l, r: GpuFilterExec(col("lk") > lit(3000), l, projection=[1, 3, 2])
    plan, got = run_both(make, left, None, 500, tc)
    assert got.num_rows > 10000 and got.num_rows == pc.sum(pc.greater(left["lk"], 3000)).as_py()
    check_release(plan, tc, left.select(["l_name", "l_comment"]).nbytes)


def check_release(plan, tc, table_string_bytes):
    """the ordered plan's peak against the same gather holding every batch to the end; and that one is about the strings' own size: each
    batch is uploaded compacted, not with the whole column its slice shares"""
    peak = plan.metrics()["peak_string_bytes_held"]
    plan.ordered = set()
    collect(plan, tc)
    held_all = plan.metrics()["peak_string_bytes_held"]
    assert 0 < peak < held_all / 2
    assert held_all < 2 * table_string_bytes


@pytest.mark.parametrize("t", TYPES, ids=str)
def test_join_probe_side_releases_in_probe_order(tc, t):
    rng = np.random.default_rng(7)
    left = left_table(rng, 1000, t)
    right = right_table(rng, 60000, 1000, t)
    make = lambda l, r: GpuHashJoinExec(l, r, [("lk", "rk")], "Inner")
    plan, _ = run_both(make, left, right, 500, tc)
    assert plan.ordered
    check_release(plan, tc, left.select(["l_name", "l_comment"]).nbytes + right["r_comment"].nbytes)


def test_filter_with_a_mask_and_a_carried_string(tc):
    rng = np.random.default_rng(2)
    left = left_table(rng, 30000, pa.string())
    make = lambda l, r: plan_string_predicates(GpuFilterExec(LikeExpr(col("l_name"), "%special%") & (col("lk") > lit(100)), l, projection=[1, 3]))
    run_both(make, left, None, 4000, tc)


@pytest.mark.parametrize("null_equality", ["NullEqualsNothing", "NullEqualsNull"])
@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_every_join_type(tc, jt, null_equality):
    t = TYPES[JOIN_TYPES.index(jt) % 3]
    rng = np.random.default_rng(JOIN_TYPES.index(jt))
    left = left_table(rng, 6000, t)
    right = right_table(rng, 20000, 6000, t)
    make = lambda l, r: GpuHashJoinExec(l, r, [("lk", "rk")], jt, null_equality=null_equality)
    _, got = run_both(make, left, right, 3000, tc)
    assert got.num_rows > 0


def _fused_tables(rng, t):
    left = left_table(rng, 5000, t, unique=True, key_nullable=False)
    right = right_table(rng, 40000, 10000, t)
    return left, right


@pytest.mark.parametrize("t", TYPES, ids=str)
def test_fused_ordered_inner_output_sink(tc, t):
    left, right = _fused_tables(np.random.default_rng(3), t)
    left = left.select(["lk", "l_name", "l_comment"])        # the build's payload is its one id: 32 bits
    make = lambda l, r: GpuHashJoinExec(l, GpuFilterExec(col("rrow") > lit(100), r), [("lk", "rk")], "Inner")
    _, got = run_both(make, left, right, 7000, tc, fuse=True)
    by_key = dict(zip(left["lk"].to_pylist(), left["l_name"].cast(pa.large_string()).to_pylist()))
    assert [by_key[k] for k in got["lk"].to_pylist()] == got["l_name"].cast(pa.large_string()).to_pylist()


@pytest.mark.parametrize("jt", ["Right", "Full"])
@pytest.mark.parametrize("t", TYPES, ids=str)
def test_fused_right_and_full_stages(tc, jt, t):
    left, right = _fused_tables(np.random.default_rng(4), t)
    make = lambda l, r: GpuProjectionExec([(col("rrow"), "rrow"), (col("l_comment"), "l_comment"), (col("r_comment"), "r_comment")],
                                          GpuHashJoinExec(l, r, [("lk", "rk")], jt))
    _, got = run_both(make, left, right, 7000, tc, fuse=True)
    # no row number of the build side is emitted: check its strings through the dictionary route's rows (above) and by key here
    by_key = dict(zip(left["lk"].to_pylist(), left["l_comment"].cast(pa.large_string()).to_pylist()))
    keys = dict(zip(right["rrow"].to_pylist(), right["rk"].to_pylist()))
    for rrow, lc in zip(got["rrow"].to_pylist(), got["l_comment"].cast(pa.large_string()).to_pylist()):
        if rrow is not None:
            assert lc == by_key.get(keys[rrow])


@pytest.mark.parametrize("t", TYPES, ids=str)
def test_fused_left_semi_emits_build_ids(tc, t):
    left, right = _fused_tables(np.random.default_rng(5), t)
    left = left.select(["lk", "l_name"])
    make = lambda l, r: GpuHashJoinExec(l, r, [("lk", "rk")], "LeftSemi")
    _, got = run_both(make, left, right, 7000, tc, fuse=True)
    by_key = dict(zip(left["lk"].to_pylist(), left["l_name"].cast(pa.large_string()).to_pylist()))
    assert [by_key[k] for k in got["lk"].to_pylist()] == got["l_name"].cast(pa.large_string()).to_pylist()


def test_customer_right_join_orders_without_a_dictionary(tc):
    """customer[c_custkey, c_name, c_comment] ⋈ orders[o_custkey, o_orderkey], Right, through plan_string_payloads and fuse_full_joins"""
    rng = np.random.default_rng(6)
    nc = 3000
    customer = pa.table({"c_custkey": pa.array(np.arange(1, nc + 1), pa.int64()), "c_name": pa.array([f"Customer#{i:09d}" for i in range(1, nc + 1)]),
                         "c_comment": pa.array(texts(rng, nc))})
    orders = pa.table({"o_custkey": pa.array(rng.integers(1, nc * 3 // 2, 30000), pa.int64()), "o_orderkey": pa.array(np.arange(30000) * 4, pa.int64())})
    make = lambda c, o: GpuHashJoinExec(c, o, [("c_custkey", "o_custkey")], "Right")
    plan = fuse_full_joins(plan_string_payloads(make(mem(customer, 1000), mem(orders, 5000))))
    assert not any(isinstance(n, DictionaryEncodeExec) for n in _nodes(plan))
    got = table(plan, tc)
    d = plan_string_dictionary()
    ref = DictionaryDecodeExec(make(DictionaryEncodeExec(mem(customer, 1000), d), mem(orders, 5000)), ["c_name", "c_comment"], d, pa.string())
    assert rows(got, False) == rows(table(ref, tc), False)
    names = dict(zip(customer["c_custkey"].to_pylist(), customer["c_name"].to_pylist()))
    assert [names.get(k) for k in got["o_custkey"].to_pylist()] == got["c_name"].to_pylist()
