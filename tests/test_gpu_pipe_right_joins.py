"""Right joins through the fused pipeline (DFGPU_STAGE_RIGHT): every probe row reaching the stage continues, a matched one with its
build row's payload fields, an unmatched one (no partner, a NULL key, a composite key outside its domain) with them NULL.  The references
are a numpy restatement of the join, the oracle's hash_join(J_RIGHT) and the unfused dfgpu_hashjoin(JOIN_RIGHT), followed by dfgpu_agg
where there is an aggregate.  Covered: the ordered sink row for row (validity bits included) and the unordered one as a multiset, probe
key bitmaps at bit offsets 0, 3 and 37, payload fields 1, 2, 4 and 8 bytes wide (signed, unsigned, Date32, Float64), every row / no row
matching and an empty build side, multi-batch pushes, RIGHT after INNER / SEMI / ANTI stages, two RIGHT stages and a composite key, the
dense and hash sinks grouped on a RIGHT payload field (the NULL group; table growth and replayed rows), COUNT / SUM / MIN / MAX / AVG over
payload fields in Single and Partial modes, a Decimal128(15, 2) probe column next to a RIGHT group key, and every refusal."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
from decimal_util import gpu_col_as_py
from harness import gpu_hash_join
import pyarrow as pa
from datafusion_b200.exec import (AggregateExpr, Column, GpuAggregateExec, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec,
                                  MemoryExec, col, collect, fuse_right_joins, lit)
from test_gpu_partition_bits import Src
from test_gpu_pipe_output_columns import assert_rows, drain

pytestmark = pytest.mark.gpu
DEC15 = D.decimal128(15, 2)
NP = {D.INT8: np.int8, D.UINT16: np.uint16, D.DATE32: np.int32, D.INT32: np.int32, D.INT64: np.int64, D.FLOAT64: np.float64}
NODE = lambda k, a=0, t=0, v=0: (k, a, t, 0, v, 0.0)                       # noqa: E731
C = lambda i: NODE(D.EXPR_COLUMN, i)                                          # noqa: E731
CMP = lambda c, op, t, v: [C(c), NODE(D.EXPR_LITERAL, 0, t, v), NODE(D.EXPR_BINARY, op)]   # noqa: E731
PAYS = {"narrow": [D.INT8, D.UINT16, D.DATE32], "wide": [D.FLOAT64]}          # widths 1, 2, 4 and 8
UNSUPPORTED, INVALID = -3, -1


def pay_values(rng, t, m):
    if t == D.FLOAT64:
        return rng.integers(-4000, 4000, m).astype(np.float64) * 0.5        # exact sums in any order
    if t == D.DATE32:
        return rng.integers(0, 30000, m).astype(np.int32)
    info = np.iinfo(NP[t])
    return rng.integers(info.min, info.max, m, endpoint=True).astype(NP[t])


def build_lookup(ctx, keys, pays, key_type=D.INT64):
    """a lookup with payload over unique keys; pays = [(type, values)]"""
    look = D.Lookup(ctx, key_type, [t for t, _ in pays])
    b = D.Pipeline(ctx, [key_type] + [t for t, _ in pays])
    b.sink_build(look, 0, list(range(1, len(pays) + 1)))
    if len(keys):
        b.push_host([D.HostColumn(keys, None, key_type)] + [D.HostColumn(v, None, t) for t, v in pays])
    b.finish()
    b.close()
    return look


def match(bk, key, kvalid):
    """row -> index of its build partner, -1 for none (a NULL key matches nothing)"""
    if len(bk) == 0:
        return np.full(len(key), -1)
    order = np.argsort(bk, kind="stable")
    i = np.minimum(np.searchsorted(bk, key, sorter=order), len(bk) - 1)
    idx = order[i]
    ok = bk[idx] == key
    if kvalid is not None:
        ok &= kvalid
    return np.where(ok, idx, -1)


def right_fields(idx, pays):
    """the payload fields of a Right join's output: the partner's values, NULL (value 0) on unmatched rows"""
    m = idx >= 0
    return [(np.where(m, v[np.maximum(idx, 0)], np.zeros((), v.dtype)) if len(v) else np.zeros(len(idx), v.dtype), m.copy()) for _, v in pays]


def probe_table(rng, n, off, bk, hit=0.6):
    """[(type, values with `off` leading rows, valid)]: the probe key (10 % NULL), a unique row id, the predicate's Int32 column"""
    m = n + off
    miss = rng.integers(0, 10**7, m).astype(np.int64) * 4 + 3                 # build keys are 1 mod 4: never a partner
    part = bk[rng.integers(0, len(bk), m)] if len(bk) else miss
    key = np.where(rng.random(m) < hit, part, miss).astype(np.int64)
    return [(D.INT64, key, rng.random(m) >= 0.1), (D.INT64, np.arange(m, dtype=np.int64) * 7 + 5, None),
            (D.INT32, rng.integers(0, 100, m).astype(np.int32), None)]


def build_keys(rng, nb):
    return (rng.permutation(4 * max(nb, 1))[:nb].astype(np.int64) * 4 + 1)


def run_output(ctx, specs, off, stages, out, ordered, pred=None, batch_size=0, stage_keys=None):
    srcs = [Src(ctx, t, v, vv, off) for t, v, vv in specs]
    p = D.Pipeline(ctx, [t for t, _, _ in specs], pred, stages)
    try:
        for s, kc in (stage_keys or {}).items():
            p.set_stage_keys(s, kc)
        p.sink_output(out, batch_size=batch_size, ordered=ordered)
        p.push_device([s.col for s in srcs])
        p.finish()
        got, rows, flags = drain(p, len(out))
    finally:
        p.close()
    return got, flags


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("off", [0, 3, 37])
@pytest.mark.parametrize("pays", sorted(PAYS))
def test_output_sinks_equal_the_unfused_right_join(gpu_ctx, ordered, off, pays):
    rng = np.random.default_rng(100 * off + 10 * ordered + len(pays))
    bk = build_keys(rng, 5000)
    pv = [(t, pay_values(rng, t, len(bk))) for t in PAYS[pays]]
    look = build_lookup(gpu_ctx, bk, pv)
    specs = probe_table(rng, 60000, off, bk)
    out = [1, 0] + [3 + j for j in range(len(pv))]
    try:
        got, flags = run_output(gpu_ctx, specs, off, [(D.STAGE_RIGHT, 0, look)], out, ordered, CMP(2, D.OP_LT, D.INT32, 70))
    finally:
        look.close()
    key, kvalid = specs[0][1][off:], specs[0][2][off:]
    keep = specs[2][1][off:] < 70
    idx = match(bk, key[keep], kvalid[keep])
    exp = [(specs[1][1][off:][keep], None), (key[keep], kvalid[keep])] + right_fields(idx, pv)
    assert all(f == [False, True] + [True] * len(pv) for f in flags), flags   # every RIGHT payload column leaves with a bitmap
    assert_rows(got, exp, ordered, f"right {pays} off={off} ordered={ordered}")
    # the oracle's and the unfused GPU Right join over the rows the predicate keeps (probe = right side, build = left side)
    bcols = [(bk, None)] + [(v, None) for _, v in pv]
    pcols = [(key[keep], kvalid[keep]), (specs[1][1][off:][keep], None)]
    sides, index = [1, 1] + [0] * len(pv), [1, 0] + [1 + j for j in range(len(pv))]
    ref = O.hash_join(bcols, pcols, [0], [0], sides, index, join_type=O.J_RIGHT)
    assert_rows(got, ref, False, "oracle hash_join(J_RIGHT)")
    if ordered:
        uf = gpu_hash_join(gpu_ctx, bcols, pcols, [0], [0], sides, index, join_type=D.JOIN_RIGHT, build_types=[D.INT64] + PAYS[pays],
                           probe_types=[D.INT64, D.INT64])
        assert_rows(got, uf, True, "dfgpu_hashjoin(JOIN_RIGHT) row for row")


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("case", ["all", "none", "empty_build"])
def test_every_row_no_row_and_an_empty_build_side(gpu_ctx, ordered, case):
    rng = np.random.default_rng(7 + ordered)
    bk = build_keys(rng, 0 if case == "empty_build" else 3000)
    pv = [(D.INT64, rng.integers(-10**12, 10**12, len(bk)).astype(np.int64))]
    look = build_lookup(gpu_ctx, bk, pv)
    specs = probe_table(rng, 20000, 0, bk, hit={"all": 1.0, "none": 0.0, "empty_build": 0.5}[case])
    if case == "all":
        specs[0] = (D.INT64, specs[0][1], None)                                  # no NULL key either: every row matches
    try:
        got, _ = run_output(gpu_ctx, specs, 0, [(D.STAGE_RIGHT, 0, look)], [1, 3], ordered)
    finally:
        look.close()
    idx = match(bk, specs[0][1], specs[0][2])
    assert (idx >= 0).all() if case == "all" else (idx < 0).all()
    assert_rows(got, [(specs[1][1], None)] + right_fields(idx, pv), ordered, case)


@pytest.mark.parametrize("ordered", [True, False])
def test_multi_batch_pushes(gpu_ctx, ordered):
    rng = np.random.default_rng(31)
    bk = build_keys(rng, 4000)
    pv = [(D.INT32, rng.integers(-10**9, 10**9, len(bk)).astype(np.int32)), (D.UINT16, pay_values(rng, D.UINT16, len(bk)))]
    look = build_lookup(gpu_ctx, bk, pv)
    specs = probe_table(rng, 90000, 0, bk)
    p = D.Pipeline(gpu_ctx, [t for t, _, _ in specs], CMP(2, D.OP_GTEQ, D.INT32, 20), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.sink_output([1, 3, 4], batch_size=1000, ordered=ordered)
        for s, e in ((0, 100), (100, 40000), (40000, 40001), (40001, 90000)):
            p.push_host([D.HostColumn(v[s:e], None if vv is None else vv[s:e], t) for t, v, vv in specs])
        p.finish()
        got, rows, _ = drain(p, 3)
    finally:
        p.close()
        look.close()
    keep = specs[2][1] >= 20
    idx = match(bk, specs[0][1][keep], specs[0][2][keep])
    assert all(r == 1000 for r in rows[:-1])
    assert_rows(got, [(specs[1][1][keep], None)] + right_fields(idx, pv), ordered, "pushes")


def key_set(ctx, keys):
    look = D.Lookup(ctx, D.INT64, [])
    b = D.Pipeline(ctx, [D.INT64])
    b.sink_build(look, 0, [])
    b.push_host([D.HostColumn(keys)])
    b.finish()
    b.close()
    return look


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("combo", ["inner", "semi", "anti", "right", "composite"])
def test_stage_combinations(gpu_ctx, ordered, combo):
    """stage 0 (INNER / SEMI / ANTI / RIGHT on column 0), then a RIGHT stage on column 3 (on (3, 4) as a composite key); a probe
    component outside its declared domain packs to the sentinel and matches nothing"""
    rng = np.random.default_rng(["inner", "semi", "anti", "right", "composite"].index(combo) * 2 + ordered)
    n = 50000
    ak = build_keys(rng, 3000)
    apv = [(D.INT32, rng.integers(-10**9, 10**9, len(ak)).astype(np.int32))]
    specs = probe_table(rng, n, 0, ak)
    looks = []
    if combo in ("inner", "right"):
        looks.append(build_lookup(gpu_ctx, ak, apv))
    elif combo in ("semi", "anti"):
        looks.append(key_set(gpu_ctx, ak))
    bpv = [(D.INT64, rng.integers(-10**12, 10**12, 2000).astype(np.int64))]
    if combo == "composite":   # (x in [0, 49], y in [-5, 34]) tuples; the probe draws x from [-3, 52]
        tup = rng.permutation(50 * 40)[:2000]
        bx, by = (tup // 40).astype(np.int32), (tup % 40 - 5).astype(np.int32)
        look = D.Lookup(gpu_ctx, payload_types=[D.INT64], key_types=[D.INT32, D.INT32], key_ranges=[(0, 49), (-5, 34)])
        b = D.Pipeline(gpu_ctx, [D.INT32, D.INT32, D.INT64])
        b.sink_build(look, payload_cols=[2], key_cols=[0, 1])
        b.push_host([D.HostColumn(bx), D.HostColumn(by), D.HostColumn(bpv[0][1])])
        b.finish()
        b.close()
        looks.append(look)
        pick = rng.integers(0, 2000, n)
        x = np.where(rng.random(n) < 0.7, bx[pick], rng.integers(-3, 53, n)).astype(np.int32)
        y = np.where(rng.random(n) < 0.9, by[pick], rng.integers(-5, 35, n)).astype(np.int32)
        specs += [(D.INT32, x, rng.random(n) >= 0.05), (D.INT32, y, None)]
        stages, stage_keys = [(D.STAGE_RIGHT, 3, look)], {0: [3, 4]}
    else:
        bk = build_keys(rng, 2000)
        looks.append(build_lookup(gpu_ctx, bk, bpv))
        part = bk[rng.integers(0, len(bk), n)]
        specs.append((D.INT64, np.where(rng.random(n) < 0.5, part, part + 2), rng.random(n) >= 0.1))
        kind0 = {"inner": D.STAGE_INNER, "semi": D.STAGE_SEMI, "anti": D.STAGE_ANTI, "right": D.STAGE_RIGHT}[combo]
        stages, stage_keys = [(kind0, 0, looks[0]), (D.STAGE_RIGHT, 3, looks[1])], None
    nin = len(specs)
    a_fields = [nin] if combo in ("inner", "right") else []
    b_field = nin + len(a_fields)
    out = [1] + a_fields + [b_field]
    try:
        got, _ = run_output(gpu_ctx, specs, 0, stages, out, ordered, stage_keys=stage_keys)
    finally:
        for lk in looks:
            lk.close()
    keep = np.ones(n, bool)
    exp_a = []
    if combo != "composite":
        ia = match(ak, specs[0][1], specs[0][2])
        if combo == "inner":
            keep &= ia >= 0
        elif combo == "semi":
            keep &= ia >= 0
        elif combo == "anti":
            keep &= ia < 0
        if combo in ("inner", "right"):
            exp_a = [(c[keep], None if combo == "inner" else m[keep]) for c, m in right_fields(ia, apv)]
        ib = match(bk, specs[3][1][keep], specs[3][2][keep])
    else:
        dom = (x >= 0) & (x <= 49) & specs[3][2]
        ib = np.where(dom, match(bx.astype(np.int64) * 40 + by, x.astype(np.int64) * 40 + y, dom), -1)
    exp = [(specs[1][1][keep], None)] + exp_a + right_fields(ib, bpv)
    assert_rows(got, exp, ordered, combo)


def agg_rows(outs, ncols):
    cols = [[] for _ in range(ncols)]
    for b in outs:
        for i in range(ncols):
            cols[i] += gpu_col_as_py(D, b, i)[0]
    return sorted(zip(*cols), key=repr)


def unfused_agg(ctx, cols, types, group, aggs, mode):
    """dfgpu_agg over the joined columns: aggs [(func, column or -1)].  A Float64 AVG's Partial state [count, sum] of a group without
    values is [0, NULL] from the fused sinks, as AvgGroupsAccumulator::state emits it; dfgpu_agg emits [0, 0.0], compared as NULL here"""
    a = D.AggHandle(ctx, types, group, [(f, c, -1) for f, c in aggs], mode, 8192)
    try:
        a.push_host([D.HostColumn(v, m, t) for (v, m), t in zip(cols, types)])
        a.finish()
        outs = a.drain(host=True)
        rows = agg_rows(outs, outs[0].num_columns if outs else 0)
    finally:
        a.close()
    if mode == D.AGG_PARTIAL:
        rows = sorted((tuple(None if i and isinstance(v, float) and v == 0.0 and r[i - 1] == 0 else v for i, v in enumerate(r)) for r in rows), key=repr)
    return rows


def agg_case(rng, n, dec=False):
    """build: unique keys with (nation Int8 in [0, 24], acct Int32); probe: key (NULLs), money Int64 or Decimal128(15, 2), the
    predicate's column, a date-like Int32 in [0, 199]"""
    bk = build_keys(rng, 3000)
    pv = [(D.INT8, rng.integers(0, 25, len(bk)).astype(np.int8)), (D.INT32, rng.integers(-10**9, 10**9, len(bk)).astype(np.int32))]
    key = np.where(rng.random(n) < 0.6, bk[rng.integers(0, len(bk), n)], rng.integers(0, 10**7, n) * 4 + 3).astype(np.int64)
    kvalid = rng.random(n) >= 0.1
    money = rng.integers(-10**9, 10**9, n).astype(np.int64)
    sel = rng.integers(0, 100, n).astype(np.int32)
    day = rng.integers(0, 200, n).astype(np.int32)
    return bk, pv, key, kvalid, money, sel, day


def probe_push(key, kvalid, money, sel, day, dec, s, e):
    mcol = D.HostColumn(D.decimal_to_words([int(z) for z in money[s:e]]), None, DEC15) if dec else D.HostColumn(money[s:e])
    return [D.HostColumn(key[s:e], kvalid[s:e]), mcol, D.HostColumn(sel[s:e]), D.HostColumn(day[s:e])]


def joined(bk, pv, key, kvalid, money, sel, day, dec):
    """the unfused plan's rows: filter (sel < 80), Right join; columns day, nation, acct, CAST(acct AS Float64), money"""
    keep = sel < 80
    idx = match(bk, key[keep], kvalid[keep])
    (nat, natm), (acct, acctm) = right_fields(idx, pv)
    bal, balm = acct.astype(np.float64), acctm
    mval = money[keep]
    mcol = (D.decimal_to_words([int(z) for z in mval]), None) if dec else (mval, None)
    cols = [(day[keep], None), (nat, natm), (acct, acctm), (bal, balm), mcol]
    return cols, [D.INT32, D.INT8, D.INT32, D.FLOAT64, DEC15 if dec else D.INT64]


# probe input columns 0 key, 1 money, 2 sel, 3 day; payload fields 4 nation, 5 acct.  (func, argument, column of joined())
BAL = [C(5), (D.EXPR_CAST, 0, D.FLOAT64, 0, 0, 0.0)]
AGGS = [(D.AGG_COUNT_STAR, None, -1), (D.AGG_COUNT, [C(5)], 2), (D.AGG_SUM, [C(1)], 4), (D.AGG_MIN, [C(5)], 2), (D.AGG_MAX, [C(5)], 2),
        (D.AGG_AVG, BAL, 3), (D.AGG_SUM, [C(5)], 2)]


@pytest.mark.parametrize("mode", [D.AGG_SINGLE, D.AGG_PARTIAL])
@pytest.mark.parametrize("dec", [False, True])
def test_dense_sink_grouped_on_a_right_payload_field(gpu_ctx, mode, dec):
    rng = np.random.default_rng(50 + 2 * dec + (mode == D.AGG_PARTIAL))
    bk, pv, key, kvalid, money, sel, day = case = agg_case(rng, 120000)
    look = build_lookup(gpu_ctx, bk, pv)
    aggs = AGGS
    if dec:   # the Decimal128 probe column: SUM, MIN, MAX (and AVG in Single mode) next to the RIGHT group key
        aggs = AGGS[:3] + [(D.AGG_MIN, [C(1)], 4), (D.AGG_MAX, [C(1)], 4), (D.AGG_MAX, [C(5)], 2), (D.AGG_AVG, BAL, 3)]
        aggs += [(D.AGG_AVG, [C(1)], 4)] if mode == D.AGG_SINGLE else []
    p = D.Pipeline(gpu_ctx, [D.INT64, DEC15 if dec else D.INT64, D.INT32, D.INT32], CMP(2, D.OP_LT, D.INT32, 80), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.sink_aggregate_dense([4], [(0, 24)], [(f, nd) for f, nd, _ in aggs], mode)
        for s, e in ((0, 50000), (50000, 120000)):
            p.push_host(probe_push(key, kvalid, money, sel, day, dec, s, e))
        p.finish()
        outs = p.drain(host=True)
        got = agg_rows(outs, outs[0].num_columns)
    finally:
        p.close()
        look.close()
    cols, types = joined(*case, dec)
    exp = unfused_agg(gpu_ctx, cols, types, [1], [(f, c) for f, _, c in aggs], mode)
    assert any(r[0] is None for r in got), "the NULL group"
    assert got == exp


@pytest.mark.parametrize("mode", [D.AGG_SINGLE, D.AGG_PARTIAL])
@pytest.mark.parametrize("dec", [False, True])
def test_hash_sink_grouped_on_a_right_payload_field(gpu_ctx, mode, dec):
    """GROUP BY (day, nation): ~5000 groups from a first table of 1024 slots, so the table grows and deferred rows are replayed (and
    probed again)"""
    rng = np.random.default_rng(70 + 2 * dec + (mode == D.AGG_PARTIAL))
    bk, pv, key, kvalid, money, sel, day = case = agg_case(rng, 150000)
    look = build_lookup(gpu_ctx, bk, pv)
    aggs = AGGS[2:6]
    if dec:
        aggs = [(D.AGG_SUM, [C(1)], 4), (D.AGG_MAX, [C(1)], 4), (D.AGG_COUNT, [C(5)], 2), (D.AGG_MIN, [C(5)], 2)]
    p = D.Pipeline(gpu_ctx, [D.INT64, DEC15 if dec else D.INT64, D.INT32, D.INT32], CMP(2, D.OP_LT, D.INT32, 80), [(D.STAGE_RIGHT, 0, look)])
    try:
        p.sink_aggregate_hash([3, 4], [(f, nd) for f, nd, _ in aggs], mode, nullable=[False, True])
        for s, e in ((0, 70000), (70000, 150000)):
            p.push_host(probe_push(key, kvalid, money, sel, day, dec, s, e))
        p.finish()
        outs = p.drain(host=True)
        got = agg_rows(outs, outs[0].num_columns)
        assert p.metric("group_rehashes") > 0 and p.metric("replayed_rows") > 0
    finally:
        p.close()
        look.close()
    cols, types = joined(*case, dec)
    exp = unfused_agg(gpu_ctx, cols, types, [0, 1], [(f, c) for f, _, c in aggs], mode)
    assert any(r[1] is None for r in got), "NULL nation groups"
    assert got == exp


def test_refusals(gpu_ctx):
    rng = np.random.default_rng(3)
    bk = build_keys(rng, 100)
    pay = build_lookup(gpu_ctx, bk, [(D.INT32, np.arange(100, dtype=np.int32))])
    keys = key_set(gpu_ctx, bk)
    bitmap = D.Lookup(gpu_ctx, D.INT64, [], key_range=(0, 1000))
    fonly = D.Lookup(gpu_ctx, D.INT64, [], expected_rows=100, filter_only=True)
    types = [D.INT64, D.INT64]

    def code(fn):
        with pytest.raises(D.DfgpuError) as e:
            fn()
        return e.value.code

    try:
        for lk in (keys, bitmap, fonly):   # a RIGHT stage needs unique keys: a lookup with payload
            assert code(lambda: D.Pipeline(gpu_ctx, types, None, [(D.STAGE_RIGHT, 0, lk)])) == UNSUPPORTED
        target = D.Lookup(gpu_ctx, D.INT64, [D.INT32])
        comp = D.Lookup(gpu_ctx, payload_types=[D.INT32], key_types=[D.INT64, D.INT64], key_ranges=[(0, 9), (0, 9)])
        sinks = [lambda p: p.sink_build(target, 1, [2]), lambda p: p.sink_build(comp, payload_cols=[2], key_cols=[0, 1]),
                 lambda p: p.sink_aggregate([0, 2], [(D.AGG_COUNT_STAR, None)])]
        for sink in sinks:   # build / pack and join-keyed aggregate sinks, refused for the RIGHT stage itself
            p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_RIGHT, 0, pay)])
            with pytest.raises(D.DfgpuError) as e:
                sink(p)
            assert e.value.code == UNSUPPORTED and "RIGHT stage" in str(e.value), str(e.value)
            p.close()
        for stage in (0, 1):   # stage filters on any stage of a pipeline with a RIGHT stage
            p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_SEMI, 1, keys), (D.STAGE_RIGHT, 0, pay)])
            assert code(lambda: p.set_stage_filter(stage, CMP(0, D.OP_GT, D.INT64, 0))) == UNSUPPORTED
            p.close()
        # a RIGHT payload group column declared non-nullable meets its first unmatched row at the push
        p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_RIGHT, 0, pay)])
        p.sink_aggregate_hash([2], [(D.AGG_COUNT_STAR, None)], nullable=[False])
        assert code(lambda: p.push_host([D.HostColumn(np.array([bk[0], 2], np.int64)), D.HostColumn(np.zeros(2, np.int64))])) == INVALID
        p.close()
        target.close()
        comp.close()
    finally:
        for lk in (pay, keys, bitmap, fonly):
            lk.close()


def twin_tables(rng, n, nc, dup=0):
    """customer (the build side; `dup` keys twice) and orders (o_custkey 5 % NULL, half of them without a customer)"""
    ck = rng.permutation(nc * 2)[:nc].astype(np.int64)
    ck = np.concatenate([ck, ck[:dup]])
    cust = pa.record_batch([pa.array(ck), pa.array(rng.integers(0, 25, len(ck)).astype(np.int32)), pa.array(rng.integers(-10**6, 10**6, len(ck)).astype(np.int32))],
                           schema=pa.schema([pa.field("c_custkey", pa.int64(), False), pa.field("c_nationkey", pa.int32(), False),
                                             pa.field("c_acctbal", pa.int32(), False)]))
    sch = pa.schema([pa.field("o_orderkey", pa.int64(), False), pa.field("o_custkey", pa.int64()), pa.field("o_orderdate", pa.date32(), False),
                     pa.field("o_totalprice", pa.int64(), False)])
    orders = pa.record_batch([pa.array(rng.permutation(n).astype(np.int64)), pa.array(rng.integers(0, nc * 2, n).astype(np.int64), mask=rng.random(n) < 0.05),
                              pa.array(rng.integers(0, 300, n).astype(np.int32)).cast(pa.date32()), pa.array(rng.integers(0, 10**9, n).astype(np.int64))], schema=sch)
    probe = GpuFilterExec(col("o_orderdate") < lit(200, pa.date32()), MemoryExec([orders.slice(s, 7000) for s in range(0, n, 7000)], sch))
    return MemoryExec([cust]), probe


def twin_plans(cust, probe):
    join = GpuHashJoinExec(cust, probe, [("c_custkey", "o_custkey")], "Right")
    out = GpuProjectionExec([(Column(n), n) for n in ("o_orderkey", "o_totalprice", "c_nationkey", "c_acctbal")], join)
    aggs = [AggregateExpr("count_star", None, "n"), AggregateExpr("sum", "o_totalprice", "s"), AggregateExpr("max", "c_acctbal", "m")]
    return {"output": out, "dense": GpuAggregateExec("Single", ["c_nationkey"], aggs, join),
            "hash": GpuAggregateExec("Single", ["o_orderdate", "c_nationkey"], aggs, join)}


def sorted_rows(batches):
    t = pa.Table.from_batches(batches)
    return t.column_names, sorted(zip(*[t.column(c).to_pylist() for c in t.column_names]), key=repr)


@pytest.mark.parametrize("sink", ["output", "dense", "hash"])
def test_twin_fused_right_join_equals_the_unfused_plan(gpu_ctx, task_ctx, sink):
    rng = np.random.default_rng(["output", "dense", "hash"].index(sink))
    plan = twin_plans(*twin_tables(rng, 50_000, 4000))[sink]
    fused = fuse_right_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == sink and fused.fallback is plan
    got, exp = sorted_rows(collect(fused, task_ctx)), sorted_rows(collect(plan, task_ctx))
    assert got == exp and len(got[1]) > 0
    assert "fallback" not in fused.metrics()


@pytest.mark.parametrize("sink", ["output", "dense", "hash"])
def test_twin_falls_back_on_duplicate_build_keys(gpu_ctx, task_ctx, sink):
    """duplicate customer keys: the lookup refuses them at the build, before any row leaves, and the unfused plan runs"""
    plan = twin_plans(*twin_tables(np.random.default_rng(9), 20_000, 3000, dup=50))[sink]
    fused = fuse_right_joins(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == sink
    got, exp = sorted_rows(collect(fused, task_ctx)), sorted_rows(collect(plan, task_ctx))
    assert "duplicate build keys" in fused.metrics()["fallback"]
    assert got == exp and len(got[1]) > 0
