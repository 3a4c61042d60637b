"""Full joins through the fused pipeline (a RIGHT stage turned into a Full join by dfgpu_pipeline_set_stage_full): every probe row reaching
the stage exactly as a RIGHT stage produces it, then, at finish, one row per build record no probe row matched, with every input column
NULL and the stage's payload fields holding the record's values.  The references are a numpy restatement of the join, the oracle's
hash_join(J_FULL) and the unfused dfgpu_hashjoin(JOIN_FULL), followed by dfgpu_agg where there is an aggregate.  The ordered sink is
compared row for row (validity bits included) over the probe rows and as a sorted multiset over the build rows it appends; the unordered
sink as a multiset.  Covered: probe key bitmaps at bit offsets 0, 3 and 37, payload fields 1, 2, 4 and 8 bytes wide, every / no build
row matched, empty probe and build sides, a predicate that drops every probe row, marks that persist across pushes, a composite key, the
dense sink grouped on a build field, on a probe column (its NULL slot) and without GROUP BY, the hash sink with growth and replayed rows,
Decimal128 probe columns, every refusal, a plain RIGHT stage over a lookup with an accumulator word, and the operator twin."""
import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from datafusion_b200.exec import (AggregateExpr, Column, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec,
                                  MemoryExec, col, collect, fuse_full_joins, lit)
from oracle import oracle as O
from harness import gpu_hash_join
from test_gpu_partition_bits import Src
from test_gpu_pipe_output_columns import assert_rows, drain
from test_gpu_pipe_right_joins import (BAL, C, CMP, DEC15, NODE, PAYS, agg_case, agg_rows, build_keys, key_set, match, pay_values,
                                       probe_push, probe_table, right_fields, sorted_rows, unfused_agg)

pytestmark = pytest.mark.gpu
UNSUPPORTED, INVALID, STATE = -3, -1, -5


def full_lookup(ctx, keys, pays, key_type=D.INT64, key_valid=None, n_acc_words=1):
    """a lookup with payload over unique keys and the accumulator word that holds the visited marks; pays = [(type, values)]"""
    look = D.Lookup(ctx, key_type, [t for t, _ in pays], n_acc_words=n_acc_words)
    b = D.Pipeline(ctx, [key_type] + [t for t, _ in pays])
    b.sink_build(look, 0, list(range(1, len(pays) + 1)))
    if len(keys):
        b.push_host([D.HostColumn(keys, key_valid, key_type)] + [D.HostColumn(v, None, t) for t, v in pays])
    b.finish()
    b.close()
    return look


def tail_rows(nb, idx, pv, n_probe_cols):
    """the build rows no probe row matched (idx: each probe row's partner, -1 for none): n_probe_cols NULL columns, then the payloads"""
    hit = np.zeros(nb, bool)
    hit[idx[idx >= 0]] = True
    un = np.flatnonzero(~hit)
    return [(np.zeros(len(un), np.int64), np.zeros(len(un), bool)) for _ in range(n_probe_cols)] + [(v[un], np.ones(len(un), bool)) for _, v in pv]


def concat(a, b):
    """[(values, valid)] + [(values, valid)] row-wise (the values of a NULL are compared through its validity bit only)"""
    out = []
    for (av, am), (bv, bm) in zip(a, b):
        am = np.ones(len(av), bool) if am is None else am
        out.append((np.concatenate([av, bv.astype(av.dtype)]), np.concatenate([am, bm])))
    return out


def tuples(cols, lo=0, hi=None):
    """rows [lo, hi) as a sorted list of tuples, None for NULL"""
    vals = []
    for v, m in cols:
        v = v[lo:hi]
        m = np.ones(len(v), bool) if m is None else m[lo:hi]
        vals.append([x if ok else None for x, ok in zip(v.tolist(), m.tolist())])
    return sorted(zip(*vals), key=repr)


def assert_full(got, part1, part2, ordered, what):
    """part1 row for row (ordered) and part2 appended in any order; the whole as a multiset (unordered)"""
    n1 = len(part1[0][0])
    exp = concat(part1, part2)
    assert got[0][0] is not None or len(exp[0][0]) == 0, what
    if len(exp[0][0]) == 0:
        return
    assert len(got[0][0]) == len(exp[0][0]), f"{what}: {len(got[0][0])} rows, expected {len(exp[0][0])}"
    if ordered:
        if n1:
            assert_rows([(v[:n1], None if m is None else m[:n1]) for v, m in got], part1, True, what + " (probe rows)")
        assert tuples(got, n1) == tuples(part2), what + " (unmatched build rows)"
    assert tuples(got) == tuples(exp), what


def run_output(ctx, specs, off, stages, out, ordered, pred=None, batch_size=0, stage_keys=None, full=True):
    srcs = [Src(ctx, t, v, vv, off) for t, v, vv in specs] if len(specs[0][1]) > off else []
    p = D.Pipeline(ctx, [t for t, _, _ in specs], pred, stages)
    try:
        for s, kc in (stage_keys or {}).items():
            p.set_stage_keys(s, kc)
        if full:
            p.set_stage_full(0)
        p.sink_output(out, batch_size=batch_size, ordered=ordered)
        if len(specs[0][1]) > off:
            p.push_device([s.col for s in srcs])
        p.finish()
        got, _, flags = drain(p, len(out))
        metrics = {k: p.metric(k) for k in ("input_rows", "unmatched_build_rows")}
    finally:
        p.close()
    return got, flags, metrics


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("off", [0, 3, 37])
@pytest.mark.parametrize("pays", sorted(PAYS))
def test_output_sinks_equal_the_unfused_full_join(gpu_ctx, ordered, off, pays):
    rng = np.random.default_rng(300 + 100 * off + 10 * ordered + len(pays))
    bk = build_keys(rng, 5000)
    pv = [(t, pay_values(rng, t, len(bk))) for t in PAYS[pays]]
    look = full_lookup(gpu_ctx, bk, pv)
    specs = probe_table(rng, 6000, off, bk)                                    # ~3600 partners: about half the build rows stay unmatched
    out = [1, 0] + [3 + j for j in range(len(pv))]
    try:
        got, _, met = run_output(gpu_ctx, specs, off, [(D.STAGE_RIGHT, 0, look)], out, ordered, CMP(2, D.OP_LT, D.INT32, 70))
    finally:
        look.close()
    key, kvalid, rid = specs[0][1][off:], specs[0][2][off:], specs[1][1][off:]
    keep = specs[2][1][off:] < 70
    idx = match(bk, key[keep], kvalid[keep])
    part1 = [(rid[keep], None), (key[keep], kvalid[keep])] + right_fields(idx, pv)
    part2 = tail_rows(len(bk), idx, pv, 2)
    assert met["input_rows"] == len(key) and met["unmatched_build_rows"] == len(part2[0][0]) > 1000, met
    assert_full(got, part1, part2, ordered, f"full {pays} off={off} ordered={ordered}")
    # the oracle's and the unfused GPU Full join over the rows the predicate keeps (probe = right side, build = left side)
    bcols = [(bk, None)] + [(v, None) for _, v in pv]
    pcols = [(key[keep], kvalid[keep]), (rid[keep], None)]
    sides, index = [1, 1] + [0] * len(pv), [1, 0] + [1 + j for j in range(len(pv))]
    ref = O.hash_join(bcols, pcols, [0], [0], sides, index, join_type=O.J_FULL)
    assert tuples(got) == tuples(ref), "oracle hash_join(J_FULL)"
    uf = gpu_hash_join(gpu_ctx, bcols, pcols, [0], [0], sides, index, join_type=D.JOIN_FULL, build_types=[D.INT64] + PAYS[pays],
                       probe_types=[D.INT64, D.INT64])
    assert tuples(got) == tuples(uf), "dfgpu_hashjoin(JOIN_FULL)"


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("case", ["all", "none", "empty_probe", "empty_build", "pred_drops_all"])
def test_edge_cases(gpu_ctx, ordered, case):
    """every build row matched (no tail), none matched, an empty probe side (every build row is emitted), an empty build side, and a
    predicate that drops every probe row (every build row is emitted, the probe rows still count as input)"""
    rng = np.random.default_rng(17 + ordered + 2 * ["all", "none", "empty_probe", "empty_build", "pred_drops_all"].index(case))
    bk = build_keys(rng, 0 if case == "empty_build" else 3000)
    pv = [(D.INT64, rng.integers(-10**12, 10**12, len(bk)).astype(np.int64))]
    look = full_lookup(gpu_ctx, bk, pv)
    n = 0 if case == "empty_probe" else 20000
    specs = probe_table(rng, n, 0, bk, hit={"all": 1.0, "none": 0.0}.get(case, 0.5))
    if case == "all":   # every build key once at least, no NULL key
        specs[0] = (D.INT64, np.concatenate([bk, specs[0][1][len(bk):]]), None)
    pred = CMP(2, D.OP_LT, D.INT32, 0) if case == "pred_drops_all" else None
    try:
        got, _, met = run_output(gpu_ctx, specs, 0, [(D.STAGE_RIGHT, 0, look)], [1, 3], ordered, pred)
    finally:
        look.close()
    keep = np.ones(n, bool) if pred is None else np.zeros(n, bool)
    idx = match(bk, specs[0][1][keep], None if specs[0][2] is None else specs[0][2][keep])
    part1 = [(specs[1][1][keep], None)] + right_fields(idx, pv)
    part2 = tail_rows(len(bk), idx, pv, 1)
    assert met["input_rows"] == n
    assert met["unmatched_build_rows"] == {"all": 0, "empty_build": 0}.get(case, len(part2[0][0])), met
    if case in ("none", "empty_probe", "pred_drops_all"):
        assert len(part2[0][0]) == len(bk)
    assert_full(got, part1, part2, ordered, case)


@pytest.mark.parametrize("ordered", [True, False])
def test_marks_persist_across_pushes(gpu_ctx, ordered):
    """build keys matched only by the first push stay matched: the tail holds the keys no push reached"""
    rng = np.random.default_rng(41 + ordered)
    bk = build_keys(rng, 4000)
    pv = [(D.INT32, rng.integers(-10**9, 10**9, len(bk)).astype(np.int32)), (D.UINT16, pay_values(rng, D.UINT16, len(bk)))]
    look = full_lookup(gpu_ctx, bk, pv)
    specs = probe_table(rng, 9000, 0, bk, hit=0.3)
    bounds = ((0, 100), (100, 4000), (4000, 4001), (4001, 9000))
    p = D.Pipeline(gpu_ctx, [t for t, _, _ in specs], CMP(2, D.OP_GTEQ, D.INT32, 20), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.set_stage_full(0)
        p.sink_output([1, 3, 4], batch_size=1000, ordered=ordered)
        for s, e in bounds:
            p.push_host([D.HostColumn(v[s:e], None if vv is None else vv[s:e], t) for t, v, vv in specs])
        p.finish()
        got, rows, _ = drain(p, 3)
    finally:
        p.close()
        look.close()
    keep = specs[2][1] >= 20
    idx = match(bk, specs[0][1][keep], specs[0][2][keep])
    first = match(bk, specs[0][1][:100][keep[:100]], specs[0][2][:100][keep[:100]])
    later = match(bk, specs[0][1][100:][keep[100:]], specs[0][2][100:][keep[100:]])
    assert len(np.setdiff1d(first[first >= 0], later[later >= 0])) > 0, "a key only the first push matches"
    part1, part2 = [(specs[1][1][keep], None)] + right_fields(idx, pv), tail_rows(len(bk), idx, pv, 1)
    # batches of batch_size: the probe rows', then the unmatched build rows' own (no copy into the probe rows' columns)
    n1, n2 = len(part1[0][0]), len(part2[0][0])
    assert rows == [1000] * (n1 // 1000) + ([n1 % 1000] if n1 % 1000 else []) + [1000] * (n2 // 1000) + ([n2 % 1000] if n2 % 1000 else [])
    assert_full(got, part1, part2, ordered, "pushes")


@pytest.mark.parametrize("ordered", [True, False])
def test_composite_key(gpu_ctx, ordered):
    """(x in [0, 49], y in [-5, 34]) tuples, the built ones with y <= 14; the probe draws x from [-3, 52] (outside the domain: the sentinel,
    a miss) with 5 % NULL x, and y from [15, 34] except on the few rows that copy a built tuple.  The tail rows' key is the record's packed
    tuple"""
    rng = np.random.default_rng(61 + ordered)
    n = 30000
    tup = rng.permutation(50 * 20)[:800]
    bx, by = (tup // 20).astype(np.int32), (tup % 20 - 5).astype(np.int32)
    bpv = [(D.INT64, rng.integers(-10**12, 10**12, len(tup)).astype(np.int64))]
    look = D.Lookup(gpu_ctx, payload_types=[D.INT64], key_types=[D.INT32, D.INT32], key_ranges=[(0, 49), (-5, 34)], n_acc_words=1)
    b = D.Pipeline(gpu_ctx, [D.INT32, D.INT32, D.INT64])
    b.sink_build(look, payload_cols=[2], key_cols=[0, 1])
    b.push_host([D.HostColumn(bx), D.HostColumn(by), D.HostColumn(bpv[0][1])])
    b.finish()
    b.close()
    pick = rng.integers(0, len(tup), n)
    hot = rng.random(n) < 0.02                                                  # few probe rows match: many build rows stay unmatched
    x = np.where(hot, bx[pick], rng.integers(-3, 53, n)).astype(np.int32)
    y = np.where(hot, by[pick], rng.integers(15, 35, n)).astype(np.int32)
    xv = rng.random(n) >= 0.05
    specs = [(D.INT64, np.arange(n, dtype=np.int64) * 3 + 1, None), (D.INT32, x, xv), (D.INT32, y, None)]
    try:
        got, _, met = run_output(gpu_ctx, specs, 0, [(D.STAGE_RIGHT, 1, look)], [0, 1, 2, 3], ordered, stage_keys={0: [1, 2]})
    finally:
        look.close()
    dom = (x >= 0) & (x <= 49) & xv
    idx = np.where(dom, match(bx.astype(np.int64) * 40 + by, x.astype(np.int64) * 40 + y, dom), -1)
    assert (~dom).sum() > 0 and (idx < 0).sum() > 0
    part1 = [(specs[0][1], None), (x, xv), (y, None)] + right_fields(idx, bpv)
    part2 = tail_rows(len(tup), idx, bpv, 3)
    assert met["unmatched_build_rows"] == len(part2[0][0]) > 0
    assert_full(got, part1, part2, ordered, "composite")


def full_joined(bk, pv, key, kvalid, money, sel, day, dec):
    """the unfused plan's rows: filter (sel < 80), Full join; columns day, nation, acct, CAST(acct AS Float64), money, money + acct,
    CAST(key IS NULL AS Int64)"""
    keep = sel < 80
    idx = match(bk, key[keep], kvalid[keep])
    (nat, natm), (acct, acctm) = right_fields(idx, pv)
    hit = np.zeros(len(bk), bool)
    hit[idx[idx >= 0]] = True
    un = np.flatnonzero(~hit)
    m = len(un)
    z, f = np.zeros(m, bool), np.ones(m, bool)
    day_c = (np.concatenate([day[keep], np.zeros(m, np.int32)]), np.concatenate([np.ones(keep.sum(), bool), z]))
    nat_c = (np.concatenate([nat, pv[0][1][un]]), np.concatenate([natm, f]))
    acct_c = (np.concatenate([acct, pv[1][1][un]]), np.concatenate([acctm, f]))
    bal_c = (acct_c[0].astype(np.float64), acct_c[1])
    mval = np.concatenate([money[keep], np.zeros(m, np.int64)])
    mvalid = np.concatenate([np.ones(keep.sum(), bool), z])
    money_c = (D.decimal_to_words([int(v) for v in mval]), mvalid) if dec else (mval, mvalid)
    mix = (mval + acct_c[0].astype(np.int64), mvalid & acct_c[1])
    knull = (np.concatenate([(~kvalid[keep]).astype(np.int64), np.ones(m, np.int64)]), None)
    cols = [day_c, nat_c, acct_c, bal_c, money_c, mix, knull]
    return cols, [D.INT32, D.INT8, D.INT32, D.FLOAT64, DEC15 if dec else D.INT64, D.INT64, D.INT64], m


# probe input columns 0 key, 1 money, 2 sel, 3 day; payload fields 4 nation, 5 acct.  (func, argument, column of full_joined())
MIX = [C(1), C(5), (D.EXPR_CAST, 0, D.INT64, 0, 0, 0.0), NODE(D.EXPR_BINARY, D.OP_PLUS)]
KNULL = [C(0), NODE(D.EXPR_IS_NULL), (D.EXPR_CAST, 0, D.INT64, 0, 0, 0.0)]
AGGS = [(D.AGG_COUNT_STAR, None, -1), (D.AGG_COUNT, [C(3)], 0), (D.AGG_SUM, MIX, 5), (D.AGG_MIN, [C(5)], 2), (D.AGG_MAX, [C(3)], 0),
        (D.AGG_AVG, BAL, 3), (D.AGG_SUM, KNULL, 6)]


@pytest.mark.parametrize("mode", [D.AGG_SINGLE, D.AGG_PARTIAL])
@pytest.mark.parametrize("group", ["build_field", "probe_column", "none"])
@pytest.mark.parametrize("dec", [False, True])
def test_dense_sink(gpu_ctx, mode, group, dec):
    """grouped on a build payload field (nation), on a probe column (day: the tail rows go to its NULL slot) or not at all; an argument
    that mixes a probe column and a build field, and one that reads IS NULL; Decimal128 money through the DEC instantiations"""
    rng = np.random.default_rng(500 + 4 * dec + 2 * (mode == D.AGG_PARTIAL) + ["build_field", "probe_column", "none"].index(group))
    bk, pv, key, kvalid, money, sel, day = agg_case(rng, 60000)
    key = np.where(rng.random(len(key)) < 0.05, key, key * 4 + 3)               # few partners: about half of the build rows stay unmatched
    case = (bk, pv, key, kvalid, money, sel, day)
    look = full_lookup(gpu_ctx, bk, pv)
    aggs = list(AGGS)
    if dec:   # the Decimal128 probe column: SUM, MIN, MAX (and AVG in Single mode)
        aggs = AGGS[:2] + [(D.AGG_SUM, [C(1)], 4), (D.AGG_MIN, [C(1)], 4), (D.AGG_MAX, [C(1)], 4), (D.AGG_MAX, [C(5)], 2), (D.AGG_SUM, KNULL, 6)]
        aggs += [(D.AGG_AVG, [C(1)], 4)] if mode == D.AGG_SINGLE else []
    gcol, gref, rng_ = {"build_field": ([4], [1], [(0, 24)]), "probe_column": ([3], [0], [(0, 199)]), "none": ([], [], [])}[group]
    p = D.Pipeline(gpu_ctx, [D.INT64, DEC15 if dec else D.INT64, D.INT32, D.INT32], CMP(2, D.OP_LT, D.INT32, 80), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.set_stage_full(0)
        p.sink_aggregate_dense(gcol, rng_, [(f, nd) for f, nd, _ in aggs], mode)
        for s, e in ((0, 25000), (25000, 60000)):
            p.push_host(probe_push(key, kvalid, money, sel, day, dec, s, e))
        p.finish()
        outs = p.drain(host=True)
        got = agg_rows(outs, outs[0].num_columns)
        tail = p.metric("unmatched_build_rows")
    finally:
        p.close()
        look.close()
    cols, types, m = full_joined(*case, dec)
    assert tail == m > 500
    exp = unfused_agg(gpu_ctx, cols, types, gref, [(f, c) for f, _, c in aggs], mode)
    if group == "probe_column":
        assert any(r[0] is None for r in got), "the NULL day slot holds the unmatched build rows"
    assert got == exp


@pytest.mark.parametrize("mode", [D.AGG_SINGLE, D.AGG_PARTIAL])
@pytest.mark.parametrize("dec", [False, True])
def test_hash_sink(gpu_ctx, mode, dec):
    """GROUP BY (day, nation): ~5000 groups from a first table of 1024 slots, so the table grows and deferred rows are replayed (the
    unmatched build rows too: their push is one more push); day is a probe column declared nullable"""
    rng = np.random.default_rng(700 + 2 * dec + (mode == D.AGG_PARTIAL))
    bk, pv, key, kvalid, money, sel, day = agg_case(rng, 150000)
    bk = np.concatenate([bk, build_keys(rng, 6000) + 10**8])                    # above every key agg_case draws: unmatched
    pv = [(t, np.concatenate([v, rng.integers(0, 25, 6000).astype(v.dtype)])) for t, v in pv]
    case = (bk, pv, key, kvalid, money, sel, day)
    look = full_lookup(gpu_ctx, bk, pv)
    aggs = [(D.AGG_SUM, MIX, 5), (D.AGG_COUNT, [C(5)], 2), (D.AGG_MIN, [C(5)], 2), (D.AGG_SUM, KNULL, 6)]
    if dec:
        aggs = [(D.AGG_SUM, [C(1)], 4), (D.AGG_MAX, [C(1)], 4), (D.AGG_COUNT, [C(5)], 2), (D.AGG_MIN, [C(5)], 2)]
    p = D.Pipeline(gpu_ctx, [D.INT64, DEC15 if dec else D.INT64, D.INT32, D.INT32], CMP(2, D.OP_LT, D.INT32, 80), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.set_stage_full(0)
        p.sink_aggregate_hash([3, 4], [(f, nd) for f, nd, _ in aggs], mode, nullable=[True, True])
        for s, e in ((0, 70000), (70000, 150000)):
            p.push_host(probe_push(key, kvalid, money, sel, day, dec, s, e))
        p.finish()
        outs = p.drain(host=True)
        got = agg_rows(outs, outs[0].num_columns)
        assert p.metric("group_rehashes") > 0 and p.metric("replayed_rows") > 0
        assert p.metric("unmatched_build_rows") >= 6000
    finally:
        p.close()
        look.close()
    cols, types, _ = full_joined(*case, dec)
    exp = unfused_agg(gpu_ctx, cols, types, [0, 1], [(f, c) for f, _, c in aggs], mode)
    assert any(r[0] is None for r in got), "NULL day groups: the unmatched build rows"
    assert got == exp


def test_refusals(gpu_ctx):
    rng = np.random.default_rng(3)
    bk = build_keys(rng, 100)
    pv = [(D.INT32, np.arange(100, dtype=np.int32))]
    marks = full_lookup(gpu_ctx, bk, pv)
    plain = full_lookup(gpu_ctx, bk, pv, n_acc_words=0)
    keys = key_set(gpu_ctx, bk)
    nulls = full_lookup(gpu_ctx, bk, pv, key_valid=np.arange(100) != 7)
    types = [D.INT64, D.INT64]
    probe = [D.HostColumn(np.array([bk[0], 2], np.int64)), D.HostColumn(np.zeros(2, np.int64))]

    def code(fn):
        with pytest.raises(D.DfgpuError) as e:
            fn()
        return e.value.code

    opened = []

    def pipe(stages):
        p = D.Pipeline(gpu_ctx, types, None, stages)
        opened.append(p)
        return p

    try:
        assert code(lambda: pipe([(D.STAGE_INNER, 0, marks)]).set_stage_full(0)) == INVALID          # not a RIGHT stage
        assert code(lambda: pipe([(D.STAGE_RIGHT, 0, marks)]).set_stage_full(1)) == INVALID          # no such stage
        assert code(lambda: pipe([(D.STAGE_SEMI, 1, keys), (D.STAGE_RIGHT, 0, marks)]).set_stage_full(1)) == UNSUPPORTED   # not the only stage
        assert code(lambda: pipe([(D.STAGE_RIGHT, 0, plain)]).set_stage_full(0)) == UNSUPPORTED      # no accumulator word
        p = pipe([(D.STAGE_RIGHT, 0, marks)])
        p.sink_output([1])
        assert code(lambda: p.set_stage_full(0)) == STATE                                            # after the sink
        # one FULL pipeline per lookup until dfgpu_lookup_clear
        first = pipe([(D.STAGE_RIGHT, 0, marks)])
        first.set_stage_full(0)
        assert code(lambda: first.set_stage_full(0)) == STATE
        assert code(lambda: pipe([(D.STAGE_RIGHT, 0, marks)]).set_stage_full(0)) == STATE
        marks.clear()
        pipe([(D.STAGE_RIGHT, 0, marks)]).set_stage_full(0)
        # the sinks and stage filters a RIGHT stage refuses
        target = D.Lookup(gpu_ctx, D.INT64, [D.INT32])
        opened.append(target)
        for sink in (lambda p: p.sink_build(target, 1, [2]), lambda p: p.sink_aggregate([0, 2], [(D.AGG_COUNT_STAR, None)]),
                     lambda p: p.set_stage_filter(0, CMP(0, D.OP_GT, D.INT64, 0))):
            marks.clear()
            p = pipe([(D.STAGE_RIGHT, 0, marks)])
            p.set_stage_full(0)
            assert code(lambda: sink(p)) == UNSUPPORTED
        # a build side with a NULL key: refused at the push, and at finish when nothing was pushed
        assert nulls.metric("null_keys") == 1
        p = pipe([(D.STAGE_RIGHT, 0, nulls)])
        p.set_stage_full(0)
        p.sink_output([1])
        assert code(lambda: p.push_host(probe)) == UNSUPPORTED
        nulls.clear()
        nulls2 = full_lookup(gpu_ctx, bk, pv, key_valid=np.arange(100) != 7)
        opened.append(nulls2)
        p = pipe([(D.STAGE_RIGHT, 0, nulls2)])
        p.set_stage_full(0)
        p.sink_output([1])
        assert code(lambda: p.finish()) == UNSUPPORTED
    finally:
        for o in reversed(opened):
            o.close()
        for lk in (marks, plain, keys, nulls):
            lk.close()


@pytest.mark.parametrize("ordered", [True, False])
def test_plain_right_stage_over_a_lookup_with_an_accumulator_word(gpu_ctx, ordered):
    """without dfgpu_pipeline_set_stage_full the stage stays a Right join: no tail, no marks (a later FULL pipeline sees every record
    unvisited)"""
    rng = np.random.default_rng(91 + ordered)
    bk = build_keys(rng, 3000)
    pv = [(D.INT32, rng.integers(-10**9, 10**9, len(bk)).astype(np.int32))]
    look = full_lookup(gpu_ctx, bk, pv)
    specs = probe_table(rng, 20000, 0, bk)
    try:
        got, _, met = run_output(gpu_ctx, specs, 0, [(D.STAGE_RIGHT, 0, look)], [1, 3], ordered, full=False)
        assert met["unmatched_build_rows"] == 0
        idx = match(bk, specs[0][1], specs[0][2])
        assert_rows(got, [(specs[1][1], None)] + right_fields(idx, pv), ordered, "right")
        # an empty probe side through a FULL pipeline on the same lookup: every build row
        got, _, met = run_output(gpu_ctx, [(t, v[:0], None if vv is None else vv[:0]) for t, v, vv in specs], 0, [(D.STAGE_RIGHT, 0, look)],
                                 [1, 3], ordered)
        assert met["unmatched_build_rows"] == len(bk)
        assert tuples(got) == tuples(tail_rows(len(bk), np.array([], np.int64), pv, 1))
    finally:
        look.close()


def twin_full_plans(cust, probe):
    join = GpuHashJoinExec(cust, probe, [("c_custkey", "o_custkey")], "Full")
    out = GpuProjectionExec([(Column(n), n) for n in ("o_orderkey", "o_totalprice", "c_nationkey", "c_acctbal")], join)
    aggs = [AggregateExpr("count_star", None, "n"), AggregateExpr("sum", "o_totalprice", "s"), AggregateExpr("max", "c_acctbal", "m")]
    return {"output": out, "dense": GpuAggregateExec("Single", ["c_nationkey"], aggs, join),
            "hash": GpuAggregateExec("Single", ["o_orderdate", "c_nationkey"], aggs, join)}


def twin_tables(rng, n, nc, dup=0):
    """customer (the build side; `dup` keys twice) and orders (o_custkey 5 % NULL, about half of the customers without an order)"""
    ck = rng.permutation(nc * 2)[:nc].astype(np.int64)
    ck = np.concatenate([ck, ck[:dup]])
    cust = pa.record_batch([pa.array(ck), pa.array(rng.integers(0, 25, len(ck)).astype(np.int32)), pa.array(rng.integers(-10**6, 10**6, len(ck)).astype(np.int32))],
                           schema=pa.schema([pa.field("c_custkey", pa.int64(), False), pa.field("c_nationkey", pa.int32(), False),
                                             pa.field("c_acctbal", pa.int32(), False)]))
    sch = pa.schema([pa.field("o_orderkey", pa.int64(), False), pa.field("o_custkey", pa.int64()), pa.field("o_orderdate", pa.date32(), False),
                     pa.field("o_totalprice", pa.int64(), False)])
    orders = pa.record_batch([pa.array(rng.permutation(n).astype(np.int64)), pa.array(rng.integers(0, nc * 2, n).astype(np.int64), mask=rng.random(n) < 0.05),
                              pa.array(rng.integers(0, 300, n).astype(np.int32)).cast(pa.date32()), pa.array(rng.integers(0, 10**9, n).astype(np.int64))], schema=sch)
    probe = GpuFilterExec(col("o_orderdate") < lit(200, pa.date32()), MemoryExec([orders.slice(s, 700) for s in range(0, n, 700)], sch))
    return MemoryExec([cust]), probe


@pytest.mark.parametrize("sink", ["output", "dense", "hash"])
def test_twin_fused_full_join_equals_the_unfused_plan(gpu_ctx, task_ctx, sink):
    rng = np.random.default_rng(["output", "dense", "hash"].index(sink))
    plan = twin_full_plans(*twin_tables(rng, 5000, 4000))[sink]
    fused = fuse_full_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == sink and fused.fallback is plan
    assert fused.schema == plan.schema
    got, exp = sorted_rows(collect(fused, task_ctx)), sorted_rows(collect(plan, task_ctx))
    assert got == exp and len(got[1]) > 0
    assert "fallback" not in fused.metrics()
    if sink == "output":   # the customers without an order: NULL order columns
        assert any(r[0] is None for r in got[1])


@pytest.mark.parametrize("sink", ["output", "dense", "hash"])
def test_twin_falls_back_on_duplicate_build_keys(gpu_ctx, task_ctx, sink):
    """duplicate customer keys: the lookup refuses them at the build, before any row leaves, and the unfused plan runs"""
    plan = twin_full_plans(*twin_tables(np.random.default_rng(9), 4000, 3000, dup=50))[sink]
    fused = fuse_full_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == sink
    got, exp = sorted_rows(collect(fused, task_ctx)), sorted_rows(collect(plan, task_ctx))
    assert "duplicate build keys" in fused.metrics()["fallback"]
    assert got == exp and len(got[1]) > 0


def py_rows(p, ncols):
    """the output batches as a sorted list of row tuples, Decimal128 words as signed ints, NULL as None"""
    cols = [[] for _ in range(ncols)]
    for b in p.drain(host=True):
        for i in range(ncols):
            v, m = b.column_numpy(i)
            if v.ndim == 2:
                v = [x - (1 << 128) if x >= 1 << 127 else x for x in (int(lo) | (int(hi) << 64) for lo, hi in v.tolist())]
            else:
                v = v.tolist()
            cols[i] += [x if m is None or m[j] else None for j, x in enumerate(v)]
    return sorted(zip(*cols), key=repr)


@pytest.mark.parametrize("ordered", [True, False])
def test_decimal128_columns_through_the_output_sinks(gpu_ctx, ordered):
    """a Decimal128(15, 2) probe column in the predicate (the DEC instantiations) and in the output: the unmatched build rows leave it
    NULL from the tail's zeroed 16-byte column"""
    rng = np.random.default_rng(131 + ordered)
    bk = build_keys(rng, 3000)
    pv = [(D.INT32, rng.integers(-10**9, 10**9, len(bk)).astype(np.int32))]
    look = full_lookup(gpu_ctx, bk, pv)
    n = 20000
    key = np.where(rng.random(n) < 0.1, bk[rng.integers(0, len(bk), n)], rng.integers(0, 10**7, n) * 4 + 3).astype(np.int64)
    money = rng.integers(-10**12, 10**12, n).astype(np.int64)
    specs = [(D.INT64, key, rng.random(n) >= 0.1), (D.INT64, np.arange(n, dtype=np.int64) + 1, None), (DEC15, D.decimal_to_words([int(z) for z in money]), None)]
    p = D.Pipeline(gpu_ctx, [t for t, _, _ in specs], CMP(2, D.OP_GT, DEC15, 0), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.set_stage_full(0)
        p.sink_output([1, 2, 3], ordered=ordered)
        p.push_host([D.HostColumn(v, vv, t) for t, v, vv in specs])
        p.finish()
        got = py_rows(p, 3)
        tail = p.metric("unmatched_build_rows")
    finally:
        p.close()
        look.close()
    keep = money > 0
    idx = match(bk, key[keep], specs[0][2][keep])
    (pay, pm), = right_fields(idx, pv)
    exp = list(zip(specs[1][1][keep].tolist(), money[keep].tolist(), [x if ok else None for x, ok in zip(pay.tolist(), pm.tolist())]))
    (_, _), (bv, _) = tail_rows(len(bk), idx, pv, 1)
    exp += [(None, None, x) for x in bv.tolist()]
    assert tail == len(bv) > 1000
    assert got == sorted(exp, key=repr)


@pytest.mark.parametrize("sink", ["output", "dense"])
@pytest.mark.parametrize("empty_probe", [True, False])
def test_tail_is_timed_as_its_own_family(sink, empty_probe):
    """with kernel timing on, the tail (selection and key emission, then its push) is the family "pipe_full_tail:<name>"; the probe
    pushes' family "pipe:<name>" counts the probe pushes only, and an empty probe side never creates it"""
    ctx = D.Context(0)
    try:
        ctx.set_kernel_timing(True)
        rng = np.random.default_rng(151 + empty_probe)
        bk = build_keys(rng, 2000)
        pv = [(D.INT8, rng.integers(0, 25, len(bk)).astype(np.int8))]
        look = full_lookup(ctx, bk, pv)
        specs = probe_table(rng, 0 if empty_probe else 10000, 0, bk, hit=0.2)
        p = D.Pipeline(ctx, [t for t, _, _ in specs], None, [(D.STAGE_RIGHT, 0, look)], name="ft")
        try:
            p.set_stage_full(0)
            if sink == "output":
                p.sink_output([1, 3], ordered=False)
            else:
                p.sink_aggregate_dense([3], [(0, 24)], [(D.AGG_COUNT_STAR, None)], D.AGG_SINGLE)
            if not empty_probe:
                p.push_host([D.HostColumn(v, vv, t) for t, v, vv in specs])
            p.finish()
            rows = sum(b.num_rows for b in p.drain(host=True))
            tail = p.metric("unmatched_build_rows")
        finally:
            p.close()
            look.close()
        assert tail > 0 and rows > 0
        assert ctx.kernel_time("pipe_full_tail:ft")[1] == 2            # the selection and emission, then the tail's pipeline kernel
        assert ctx.kernel_time("pipe:ft")[1] == (0 if empty_probe else 1)
    finally:
        ctx.close()


def test_more_refusals_and_a_failed_tail(gpu_ctx):
    """16 input columns leave no slot for the tail's keys; a tail push that fails leaves the pipeline finished, so a second finish is
    DFGPU_ERR_STATE and never pushes the unmatched rows twice"""
    rng = np.random.default_rng(171)
    bk = build_keys(rng, 200)
    look = full_lookup(gpu_ctx, bk, [(D.INT32, np.arange(200, dtype=np.int32))])
    try:
        p = D.Pipeline(gpu_ctx, [D.INT64] * 16, None, [(D.STAGE_RIGHT, 0, look)])
        with pytest.raises(D.DfgpuError) as e:
            p.set_stage_full(0)
        assert e.value.code == UNSUPPORTED
        p.close()
        # a probe group column declared non-nullable meets the tail's NULLs at finish
        p = D.Pipeline(gpu_ctx, [D.INT64, D.INT64], None, [(D.STAGE_RIGHT, 0, look)])
        try:
            p.set_stage_full(0)
            p.sink_aggregate_hash([1], [(D.AGG_COUNT_STAR, None)], nullable=[False])
            p.push_host([D.HostColumn(bk[:50].copy()), D.HostColumn(np.arange(50, dtype=np.int64))])
            with pytest.raises(D.DfgpuError) as e:
                p.finish()
            assert e.value.code == INVALID
            with pytest.raises(D.DfgpuError) as e:
                p.finish()
            assert e.value.code == STATE
        finally:
            p.close()
    finally:
        look.close()
