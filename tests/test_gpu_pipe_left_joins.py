"""Left, LeftSemi and LeftAnti joins through the fused pipeline's join-keyed aggregate sink (DFGPU_STAGE_LEFT / DFGPU_STAGE_LEFT_ANTI, and
LeftSemi as an INNER stage with no aggregates), against a row-by-row Python restatement of the join, the oracle's hash join and the unfused
dfgpu_hashjoin of the same type.  Results are compared sorted: the sink emits in slot order."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(__file__))
from decimal_util import gpu_col_as_py  # noqa: E402
from harness import gpu_hash_join  # noqa: E402

pytestmark = pytest.mark.gpu

DEC = D.decimal128(15, 2)
N_ACC = 11   # enough for four aggregates with non-null counters; odd, so a key-only record has an even number of words
C = lambda i: (D.EXPR_COLUMN, i, 0, 0, 0, 0.0)                                 # noqa: E731
L = lambda v, t=D.INT64: (D.EXPR_LITERAL, 0, t, 0, v, 0.0)                     # noqa: E731
B = lambda op: (D.EXPR_BINARY, op, 0, 0, 0, 0.0)                               # noqa: E731
PRED = [C(4), L(80), B(D.OP_LT)]                                               # sel < 80


@pytest.fixture(scope="module")
def ctx():
    c = D.Context(0)
    yield c
    c.close()


def make_build(rng, n, null_key_rows=0):
    key = rng.permutation(np.arange(1, 4 * n + 1, dtype=np.int64))[:n]
    p1 = rng.integers(-1000, 1000, n).astype(np.int32)
    p2 = rng.integers(0, 50, n).astype(np.int32)
    valid = None
    if null_key_rows:
        valid = np.ones(n, bool)
        valid[rng.choice(n, null_key_rows, replace=False)] = False
    return key, valid, p1, p2


def make_probe(rng, n, build_key, null_frac=0.1):
    hit = rng.random(n) < 0.6
    pkey = np.where(hit, build_key[rng.integers(0, len(build_key), n)], rng.integers(1, 8 * len(build_key) + 2, n)).astype(np.int64)
    pvalid = rng.random(n) >= null_frac
    x = rng.integers(-10**6, 10**6, n).astype(np.int64)
    xvalid = rng.random(n) >= 0.2
    y = rng.integers(-4000, 4000, n).astype(np.float64) * 0.5                  # exact sums in any order
    d = rng.integers(-10**9, 10**9, n).astype(np.int64)
    dvalid = rng.random(n) >= 0.15
    sel = rng.integers(0, 100, n).astype(np.int64)
    return [(pkey, pvalid), (x, xvalid), (y, None), (d, dvalid), (sel, None)]


def probe_host(cols, s, e):
    out = []
    for i, (v, val) in enumerate(cols):
        vals = v[s:e]
        if i == 3:
            vals = D.decimal_to_words([int(z) for z in vals])
        out.append(D.HostColumn(vals, None if val is None else val[s:e], DEC if i == 3 else None))
    return out


PROBE_TYPES = [D.INT64, D.INT64, D.FLOAT64, DEC, D.INT64]


def build_lookup(ctx, build, n_pay, n_acc=N_ACC, **kw):
    key, kvalid, p1, p2 = build
    look = D.Lookup(ctx, D.INT64, [D.INT32] * n_pay, n_acc_words=n_acc, **kw)
    p = D.Pipeline(ctx, [D.INT64, D.INT32, D.INT32])
    p.sink_build(look, 0, list(range(1, n_pay + 1)))
    if len(key):
        p.push_host([D.HostColumn(key, kvalid), D.HostColumn(p1), D.HostColumn(p2)])
    p.finish()
    p.close()
    return look


def survivors(probe, semi_keys=None):
    pkey, pvalid = probe[0]
    keep = probe[4][0] < 80
    if semi_keys is not None:
        keep &= np.isin(probe[4][0], semi_keys)
    return keep & pvalid


def run(ctx, look, probe, kind, group, aggs=(), mode=D.AGG_SINGLE, pushes=3, semi=None):
    stages = ([(D.STAGE_SEMI, 4, semi)] if semi is not None else []) + [(kind, 0, look)]
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, stages)
    try:
        p.sink_aggregate(group, list(aggs), mode)
        n = len(probe[0][0])
        for k in range(pushes):
            s, e = n * k // pushes, n * (k + 1) // pushes
            if e > s:
                p.push_host(probe_host(probe, s, e))
        p.finish()
        outs = p.drain(host=True)
        ncols = outs[0].num_columns if outs else 0
        rows = []
        cols = [[] for _ in range(ncols)]
        for b in outs:
            for i in range(ncols):
                cols[i] += gpu_col_as_py(D, b, i)[0]
        rows = sorted(zip(*cols)) if cols else []
        return rows, {m: p.metric(m) for m in ("num_groups", "input_rows")}
    finally:
        p.close()


def semi_set(build, probe, n_pay, anti, semi_keys=None):
    key, _, p1, p2 = build
    keep = survivors(probe, semi_keys)
    reached = set(probe[0][0][keep].tolist())
    pay = [p1, p2][:n_pay]
    return sorted(tuple([int(key[i])] + [int(c[i]) for c in pay]) for i in range(len(key)) if (key[i] in reached) != anti)


@pytest.mark.parametrize("n_pay", [0, 1, 2])
@pytest.mark.parametrize("anti", [False, True])
@pytest.mark.parametrize("front_semi", [False, True])
def test_left_semi_and_anti(ctx, n_pay, anti, front_semi):
    rng = np.random.default_rng(10 * n_pay + 2 * anti + front_semi)
    build = make_build(rng, 3000)
    probe = make_probe(rng, 40000, build[0])
    semi_keys = np.arange(0, 100, 3, dtype=np.int64) if front_semi else None
    semi = None
    if front_semi:
        semi = D.Lookup(ctx, D.INT64, [])
        sp = D.Pipeline(ctx, [D.INT64]); sp.sink_build(semi, 0, []); sp.push_host([D.HostColumn(semi_keys)]); sp.finish(); sp.close()
    look = build_lookup(ctx, build, n_pay)
    group = [0] + [5 + i for i in range(n_pay)]
    got, m = run(ctx, look, probe, D.STAGE_LEFT_ANTI if anti else D.STAGE_INNER, group, semi=semi)
    exp = semi_set(build, probe, n_pay, anti, semi_keys)
    assert got == exp and m["num_groups"] == len(exp)
    # the oracle's and the unfused GPU join of the same type over the surviving probe rows
    keep = survivors(probe, semi_keys) | ~probe[0][1]
    bcols = [(build[0], None), (build[2], None), (build[3], None)]
    pcols = [(probe[0][0][keep], probe[0][1][keep])]
    jt = (O.J_LEFT_ANTI, D.JOIN_LEFT_ANTI) if anti else (O.J_LEFT_SEMI, D.JOIN_LEFT_SEMI)
    out_index = list(range(n_pay + 1))
    ref = O.hash_join(bcols, pcols, [0], [0], [0] * len(out_index), out_index, join_type=jt[0])
    uf = gpu_hash_join(ctx, bcols, pcols, [0], [0], [0] * len(out_index), out_index, join_type=jt[1])
    for cols in (ref, uf):
        assert sorted(zip(*[c[0].tolist() for c in cols])) == exp
    look.close()
    if semi is not None:
        semi.close()


@pytest.mark.parametrize("case", ["empty_probe", "all_filtered", "empty_build"])
def test_left_family_edge_inputs(ctx, case):
    rng = np.random.default_rng(7)
    build = make_build(rng, 0 if case == "empty_build" else 500)
    probe = make_probe(rng, 0 if case == "empty_probe" else 5000, build[0] if len(build[0]) else np.array([1], np.int64))
    if case == "all_filtered":
        probe[4] = (np.full(len(probe[4][0]), 99, np.int64), None)
    n_build = len(build[0])
    for kind, aggs in ((D.STAGE_INNER, []), (D.STAGE_LEFT_ANTI, []), (D.STAGE_LEFT, [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(1)])])):
        look = build_lookup(ctx, build, 1, expected_rows=16)   # an allocated table, also with no build row
        got, _ = run(ctx, look, probe, kind, [0, 5], aggs)
        look.close()
        if kind == D.STAGE_INNER:
            assert got == []
        elif kind == D.STAGE_LEFT_ANTI:
            assert got == sorted((int(build[0][i]), int(build[2][i])) for i in range(n_build))
        else:
            assert got == sorted((int(build[0][i]), int(build[2][i]), 1, None) for i in range(n_build))


def left_reference(build, probe, n_pay, funcs, partial=False):
    """per build row: its NULL-padded row when no surviving probe row matches, else the aggregates of its matches"""
    key, _, p1, p2 = build
    keep = survivors(probe)
    by_key = {}
    for r in np.nonzero(keep)[0]:
        by_key.setdefault(int(probe[0][0][r]), []).append(r)
    out = []
    for i in range(len(key)):
        rows = by_key.get(int(key[i]), [])
        row = [int(key[i])] + [int(c[i]) for c in [p1, p2][:n_pay]]
        for f, c in funcs:
            vals = [] if c is None else [probe[c][0][r] for r in rows if probe[c][1] is None or probe[c][1][r]]
            vals = [float(v) if c == 2 else int(v) for v in vals]
            if f == D.AGG_COUNT_STAR:
                row.append(max(len(rows), 1))
            elif f == D.AGG_COUNT:
                row.append(len(vals))
            elif f == D.AGG_SUM:
                row.append(sum(vals) if vals else None)
            elif f == D.AGG_MIN:
                row.append(min(vals) if vals else None)
            elif f == D.AGG_MAX:
                row.append(max(vals) if vals else None)
            elif partial:   # AVG state [count, sum]
                row += [len(vals), sum(vals) if vals else None]
            else:
                row.append(sum(vals) / len(vals) if vals else None)
        out.append(tuple(row))
    return sorted(out)


LEFT_CASES = {
    "counts": [(D.AGG_COUNT_STAR, None), (D.AGG_COUNT, 1)],
    "int64": [(D.AGG_SUM, 1), (D.AGG_MIN, 1), (D.AGG_MAX, 1), (D.AGG_COUNT_STAR, None)],
    "float64": [(D.AGG_SUM, 2), (D.AGG_MIN, 2), (D.AGG_MAX, 2), (D.AGG_AVG, 2)],
    "decimal": [(D.AGG_SUM, 3), (D.AGG_MIN, 3), (D.AGG_MAX, 3), (D.AGG_COUNT, 3)],
}
LEFT_SEEDS = {"counts": 11, "int64": 12, "float64": 13, "decimal": 14}


@pytest.mark.parametrize("n_pay", [0, 2])
@pytest.mark.parametrize("case", sorted(LEFT_CASES))
def test_left_aggregates(ctx, case, n_pay):
    rng = np.random.default_rng(LEFT_SEEDS[case] * 10 + n_pay)
    build = make_build(rng, 2500)
    probe = make_probe(rng, 30000, build[0])
    funcs = LEFT_CASES[case]
    look = build_lookup(ctx, build, n_pay)
    got, m = run(ctx, look, probe, D.STAGE_LEFT, [0] + [5 + i for i in range(n_pay)], [(f, None if c is None else [C(c)]) for f, c in funcs])
    look.close()
    exp = left_reference(build, probe, n_pay, funcs)
    assert m["num_groups"] == len(build[0])
    assert got == exp


def test_left_row_counter_stands_in_for_missing_non_null_counters(ctx):
    """n_acc_words = 3 holds the row counter, SUM and MAX of a non-nullable Int64, and no non-null counter: an unreached build row's SUM
    and MAX are NULL because its row counter is 0"""
    rng = np.random.default_rng(21)
    build = make_build(rng, 2000)
    probe = make_probe(rng, 20000, build[0])
    funcs = [(D.AGG_SUM, 4), (D.AGG_MAX, 4)]                                   # sel: no validity bitmap
    for n_pay in (0, 1):
        look = build_lookup(ctx, build, n_pay, n_acc=3)
        got, _ = run(ctx, look, probe, D.STAGE_LEFT, [0] + [5 + i for i in range(n_pay)], [(f, [C(c)]) for f, c in funcs])
        look.close()
        exp = left_reference(build, probe, n_pay, funcs)
        assert got == exp and any(r[-1] is None for r in exp) and any(r[-1] is not None for r in exp)


def test_left_counts_match_the_unfused_left_join(ctx):
    rng = np.random.default_rng(3)
    build = make_build(rng, 2000)
    probe = make_probe(rng, 20000, build[0])
    look = build_lookup(ctx, build, 0)
    got, _ = run(ctx, look, probe, D.STAGE_LEFT, [0], [(D.AGG_COUNT_STAR, None), (D.AGG_COUNT, [C(1)])])
    look.close()
    keep = survivors(probe) | ~probe[0][1]
    bcols = [(build[0], None)]
    pcols = [(probe[0][0][keep], probe[0][1][keep]), (probe[1][0][keep], probe[1][1][keep])]
    joined = gpu_hash_join(ctx, bcols, pcols, [0], [0], [0, 1], [0, 1], join_type=D.JOIN_LEFT)
    ref = O.hash_join(bcols, pcols, [0], [0], [0, 1], [0, 1], join_type=O.J_LEFT)
    for cols in (joined, ref):
        k, (x, xv) = cols[0][0], cols[1]
        xv = np.ones(len(x), bool) if xv is None else xv
        star = {int(a): int(b) for a, b in zip(*np.unique(k, return_counts=True))}
        cnt = {}
        for a, ok in zip(k.tolist(), xv.tolist()):
            cnt[a] = cnt.get(a, 0) + int(ok)
        assert got == sorted((a, star[a], cnt[a]) for a in star)


def test_left_partial_then_final_equals_single(ctx):
    rng = np.random.default_rng(4)
    build = make_build(rng, 2000)
    probe = make_probe(rng, 20000, build[0])
    funcs = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, 1), (D.AGG_MAX, 2), (D.AGG_AVG, 2)]
    aggs = [(f, None if c is None else [C(c)]) for f, c in funcs]
    look = build_lookup(ctx, build, 1)
    part, _ = run(ctx, look, probe, D.STAGE_LEFT, [0, 5], aggs, mode=D.AGG_PARTIAL)
    look.close()
    assert part == left_reference(build, probe, 1, funcs, partial=True)
    # the state columns through dfgpu_agg's Final
    cols = list(zip(*part))
    types = [D.INT64, D.INT32, D.INT64, D.INT64, D.FLOAT64, D.UINT64, D.FLOAT64]
    np_types = [np.int64, np.int32, np.int64, np.int64, np.float64, np.uint64, np.float64]
    host = [D.HostColumn(np.array([0 if v is None else v for v in c], dt), None if all(v is not None for v in c) else np.array([v is not None for v in c]), t)
            for c, dt, t in zip(cols, np_types, types)]
    a = D.AggHandle(ctx, types, [0, 1], [(D.AGG_COUNT_STAR, -1, -1), (D.AGG_SUM, -1, -1), (D.AGG_MAX, -1, -1), (D.AGG_AVG, -1, -1)], D.AGG_FINAL, 8192, 0)
    a.push_host(host)
    a.finish()
    outs = a.drain(host=True)
    final = []
    for b in outs:
        final += list(zip(*[gpu_col_as_py(D, b, i)[0] for i in range(b.num_columns)]))
    a.close()
    assert sorted(final) == left_reference(build, probe, 1, funcs)


def test_left_over_a_lookup_with_a_membership_filter(ctx):
    """a build of 2.5M keys sizes a table past 40 MB, which carries the Bloom filter in front of the probe"""
    rng = np.random.default_rng(5)
    build = make_build(rng, 2_500_000)
    probe = make_probe(rng, 4_000_000, build[0], null_frac=0.02)
    look = build_lookup(ctx, build, 0, n_acc=1, membership_filter=-1)
    assert look.metric("filter_bytes") > 0 and look.metric("table_bytes") > 40 << 20
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_LEFT, 0, look)])
    p.sink_aggregate([0], [(D.AGG_COUNT_STAR, None)])
    p.push_host(probe_host(probe, 0, len(probe[0][0])))
    p.finish()
    outs = p.drain(host=True)
    k = np.concatenate([b.column_numpy(0)[0] for b in outs]); c = np.concatenate([b.column_numpy(1)[0] for b in outs])
    p.close(); look.close()
    keep = survivors(probe)
    hits = dict(zip(*np.unique(probe[0][0][keep], return_counts=True)))
    exp = np.array([max(int(hits.get(int(x), 0)), 1) for x in k], np.int64)
    assert len(k) == len(build[0]) and np.array_equal(np.sort(k), np.sort(build[0])) and np.array_equal(c, exp)


def rejected(fn):
    with pytest.raises(D.DfgpuError) as e:
        fn()
    return e.value


def test_rejections(ctx):
    rng = np.random.default_rng(6)
    build = make_build(rng, 100)
    probe = make_probe(rng, 1000, build[0])
    look = build_lookup(ctx, build, 1)
    other = build_lookup(ctx, build, 0)
    try:
        # the new kinds only as the last stage, also when the last stage is one of them
        p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_LEFT, 0, look), (D.STAGE_INNER, 4, other)])
        rejected(lambda: p.sink_aggregate([0, 5], [(D.AGG_COUNT_STAR, None)])); p.close()
        for first in (D.STAGE_LEFT_ANTI, D.STAGE_LEFT):
            p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(first, 4, other), (D.STAGE_LEFT, 0, look)])
            rejected(lambda: p.sink_aggregate([0, 5], [(D.AGG_COUNT_STAR, None)])); p.close()
        # only with the join-keyed aggregate sink
        for sink in ("hash", "dense", "output", "build"):
            p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_LEFT_ANTI, 0, look)])
            if sink == "hash":
                rejected(lambda: p.sink_aggregate_hash([0], [(D.AGG_COUNT_STAR, None)]))
            elif sink == "dense":
                rejected(lambda: p.sink_aggregate_dense([4], [(0, 99)], [(D.AGG_COUNT_STAR, None)]))
            elif sink == "output":
                rejected(lambda: p.sink_output([0]))
            else:
                tgt = D.Lookup(ctx, D.INT64, [])
                rejected(lambda: p.sink_build(tgt, 0, [])); tgt.close()
            p.close()
        # LEFT_ANTI takes no aggregates
        p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_LEFT_ANTI, 0, look)])
        rejected(lambda: p.sink_aggregate([0], [(D.AGG_COUNT_STAR, None)])); p.close()
        # LEFT: an argument reading the LEFT stage's payload, an IS NULL argument, a build-only argument
        for arg in ([C(5)], [C(1), (D.EXPR_IS_NULL, 0, 0, 0, 0, 0.0)], [C(1), C(5), B(D.OP_PLUS)], [C(1), L(0), B(D.OP_GT), C(1), L(5), B(D.OP_LT), B(D.OP_AND)]):
            p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_LEFT, 0, look)])
            rejected(lambda: p.sink_aggregate([0], [(D.AGG_COUNT, arg)])); p.close()
        # a lookup without accumulator words
        bare = build_lookup(ctx, build, 0, n_acc=0)
        p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_LEFT, 0, bare)])
        rejected(lambda: p.sink_aggregate([0], [(D.AGG_COUNT_STAR, None)])); p.close(); bare.close()
    finally:
        look.close(); other.close()


def test_null_build_keys(ctx):
    rng = np.random.default_rng(8)
    probe = make_probe(rng, 2000, np.arange(1, 200, dtype=np.int64))
    # a bitmap without NULLs is accepted
    clean = make_build(rng, 200)
    clean = (clean[0], np.ones(200, bool), clean[2], clean[3])
    look = build_lookup(ctx, clean, 0)
    assert look.metric("null_keys") == 0
    got, _ = run(ctx, look, probe, D.STAGE_LEFT_ANTI, [0])
    assert got == semi_set(clean, probe, 0, True)
    look.close()
    # NULL keys: counted, and rejected by LEFT / LEFT_ANTI at the first push; INNER (LeftSemi) never emits them
    dirty = make_build(rng, 200, null_key_rows=7)
    for kind in (D.STAGE_LEFT, D.STAGE_LEFT_ANTI, D.STAGE_INNER):
        look = build_lookup(ctx, dirty, 0)
        assert look.metric("null_keys") == 7
        if kind == D.STAGE_INNER:
            got, _ = run(ctx, look, probe, kind, [0])
            valid = (dirty[0][dirty[1]], None, dirty[2][dirty[1]], dirty[3][dirty[1]])
            assert got == semi_set(valid, probe, 0, False)
        else:
            e = rejected(lambda: run(ctx, look, probe, kind, [0], [(D.AGG_COUNT_STAR, None)] if kind == D.STAGE_LEFT else []))
            assert e.code == -3   # DFGPU_ERR_UNSUPPORTED
        look.close()


def q13_tables(rng, n_cust=3000, n_ord=30000):
    ck = np.arange(1, n_cust + 1, dtype=np.int64)
    active = ck[ck % 3 != 0]                                  # one customer in three places no order, as dbgen's o_custkey
    ocust = active[rng.integers(0, len(active), n_ord)]
    okey = np.arange(1, n_ord + 1, dtype=np.int64)
    ocomment = rng.integers(0, 100, n_ord).astype(np.int64)  # an integer stand-in for o_comment NOT LIKE '%special%requests%'
    customer = pa.table({"c_custkey": pa.array(ck)}, schema=pa.schema([pa.field("c_custkey", pa.int64(), False)]))
    orders = pa.table({"o_orderkey": okey, "o_custkey": ocust, "o_comment": ocomment})
    return customer, orders


def test_q13_shape_through_the_twin(ctx):
    from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec, MemoryExec,
                                      TaskContext, col, collect, fuse_pipelines, lit)
    customer, orders = q13_tables(np.random.default_rng(9))
    mem = lambda t: MemoryExec(t.to_batches(max_chunksize=7000), t.schema)  # noqa: E731
    o = GpuFilterExec(col("o_comment") < lit(98, pa.int64()), mem(orders), projection=[0, 1])
    join = GpuHashJoinExec(mem(customer), o, [("c_custkey", "o_custkey")], "Left", projection=[0, 1])
    inner = GpuAggregateExec("Single", ["c_custkey"], [AggregateExpr("count", "o_orderkey", "c_count")], join)
    fused = fuse_pipelines(inner)
    assert isinstance(fused, GpuPipelineExec) and fused.scan.stages[-1][0] == D.STAGE_LEFT
    tc = TaskContext(ctx=ctx)
    outer = lambda below: GpuAggregateExec("Single", ["c_count"], [AggregateExpr("count_star", None, "custdist")],  # noqa: E731
                                           GpuProjectionExec([(col("c_count"), "c_count")], below))
    rows = lambda plan: sorted(tuple(r.values()) for b in collect(plan, tc) for r in b.to_pylist())  # noqa: E731
    assert rows(inner) == rows(fused)
    assert rows(outer(inner)) == rows(outer(fused))
    # LeftSemi / LeftAnti through the twin against the unfused join
    n = customer.num_rows
    with_bal = pa.table({"c_custkey": customer.column(0), "c_acctbal": pa.array((np.arange(n) * 7919 % 10007).astype(np.int64))},
                        schema=pa.schema([pa.field("c_custkey", pa.int64(), False), pa.field("c_acctbal", pa.int64(), False)]))
    for jt in ("LeftSemi", "LeftAnti"):
        for left, projection in ((customer, None), (with_bal, [1])):   # [1]: the join's projection drops the key it groups on
            plain = GpuHashJoinExec(mem(left), o, [("c_custkey", "o_custkey")], jt, projection=projection)
            f = fuse_pipelines(plain)
            assert isinstance(f, GpuPipelineExec) and f.project == projection
            assert rows(plain) == rows(f)
