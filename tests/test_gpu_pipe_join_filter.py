"""JoinFilters inside the fused pipeline's probe stages (dfgpu_pipeline_set_stage_filter): every stage kind under every sink, against a
row-by-row Python restatement of the join with its filter, the oracle's hash join and the unfused dfgpu_hashjoin with the same filter.
Sinks that emit in slot order are compared sorted."""
import os
import sys

import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(__file__))
from decimal_util import gpu_col_as_py, gpu_nodes  # noqa: E402
from harness import gpu_group_by, gpu_hash_join  # noqa: E402

pytestmark = pytest.mark.gpu

DEC = D.decimal128(15, 2)
C = lambda i: (D.EXPR_COLUMN, i, 0, 0, 0, 0.0)                                 # noqa: E731
L = lambda v, t=D.INT64: (D.EXPR_LITERAL, 0, t, 0, v, 0.0)                     # noqa: E731
B = lambda op: (D.EXPR_BINARY, op, 0, 0, 0, 0.0)                               # noqa: E731
PRED = [C(5), L(80), B(D.OP_LT)]                                               # sel < 80
# probe: 0 key (nullable), 1 x Int64 (nullable), 2 q Int32, 3 d Decimal128(15, 2) (nullable), 4 rid, 5 sel, 6 zero
PROBE_TYPES = [D.INT64, D.INT64, D.INT32, DEC, D.INT64, D.INT64, D.INT64]
NIN = len(PROBE_TYPES)
ERR_INVALID, ERR_UNSUPPORTED, ERR_ARITH, ERR_STATE = -1, -3, -4, -5             # dfgpu_status (include/dfgpu.h)


@pytest.fixture(scope="module")
def ctx():
    c = D.Context(0)
    yield c
    c.close()


def make_build(rng, n):
    key = rng.permutation(np.arange(1, 4 * n + 1, dtype=np.int64))[:n]
    return key, rng.integers(-50, 50, n).astype(np.int32), rng.integers(0, 8, n).astype(np.int32)


def make_probe(rng, n, build_key, hit=0.6):
    h = rng.random(n) < hit
    key = np.where(h, build_key[rng.integers(0, len(build_key), n)], rng.integers(1, 8 * len(build_key) + 2, n)).astype(np.int64)
    return [(key, rng.random(n) >= 0.1), (rng.integers(-1000, 1000, n).astype(np.int64), rng.random(n) >= 0.2),
            (rng.integers(-50, 50, n).astype(np.int32), None), (rng.integers(-10**6, 10**6, n).astype(np.int64), rng.random(n) >= 0.15),
            (np.arange(n, dtype=np.int64), None), (rng.integers(0, 100, n).astype(np.int64), None), (np.zeros(n, np.int64), None)]


def host_cols(probe, s, e):
    out = []
    for i, (v, val) in enumerate(probe):
        vals = D.decimal_to_words([int(z) for z in v[s:e]]) if i == 3 else v[s:e]
        out.append(D.HostColumn(vals, None if val is None else val[s:e], DEC if i == 3 else None))
    return out


def push_all(p, probe, pushes=3):
    n = len(probe[0][0])
    for k in range(pushes):
        s, e = n * k // pushes, n * (k + 1) // pushes
        if e > s:
            p.push_host(host_cols(probe, s, e))
    p.finish()


def drain_rows(p):
    outs = p.drain(host=True)
    if not outs:
        return []
    cols = [[] for _ in range(outs[0].num_columns)]
    for b in outs:
        for i in range(len(cols)):
            cols[i] += gpu_col_as_py(D, b, i)[0]
    return list(zip(*cols))


def lookup(ctx, build, n_pay, n_acc=0, key_range=None, **kw):
    key, p1, p2 = build
    look = D.Lookup(ctx, D.INT64, [D.INT32] * n_pay, n_acc_words=n_acc, key_range=key_range, **kw)
    p = D.Pipeline(ctx, [D.INT64, D.INT32, D.INT32])
    p.sink_build(look, 0, list(range(1, n_pay + 1)))
    p.push_host([D.HostColumn(key), D.HostColumn(p1), D.HostColumn(p2)])
    p.finish()
    p.close()
    return look


# ---- filters: RPN over the stage's columns + the same predicate in Python (None = NULL) ----
def filt(name, pay0):
    """pay0: the virtual column of the stage's first payload field (p1; p2 follows)"""
    if name == "probe":      # x > 100: NULL where x is NULL
        return [C(1), L(100), B(D.OP_GT)], lambda r, b: None if r["x"] is None else r["x"] > 100
    if name == "payload":    # p1 < q
        return [C(pay0), C(2), B(D.OP_LT)], lambda r, b: b["p1"] < r["q"]
    if name == "kleene":     # x > 100 OR p2 = 3
        def f(r, b):
            a = None if r["x"] is None else r["x"] > 100
            return True if (a or b["p2"] == 3) else (None if a is None else False)
        return [C(1), L(100), B(D.OP_GT), C(pay0 + 1), L(3, D.INT32), B(D.OP_EQ), B(D.OP_OR)], f
    if name == "decimal":    # d > 0.00
        return [C(3), L(0, DEC), B(D.OP_GT)], lambda r, b: None if r["d"] is None else r["d"] > 0
    raise KeyError(name)


def candidates(build, probe, semi_keys=None):
    """per probe row surviving the predicate (and a SEMI stage on sel): its build row index, or -1"""
    key, p1, p2 = build
    pos = {int(k): i for i, k in enumerate(key)}
    keep = probe[5][0] < 80
    if semi_keys is not None:
        keep &= np.isin(probe[5][0], semi_keys)
    out = []
    for r in np.nonzero(keep)[0]:
        b = pos.get(int(probe[0][0][r]), -1) if probe[0][1][r] else -1
        out.append((int(r), b))
    return out


def row_view(probe, r):
    x = int(probe[1][0][r]) if probe[1][1][r] else None
    d = int(probe[3][0][r]) if probe[3][1][r] else None
    return {"x": x, "q": int(probe[2][0][r]), "d": d}


def build_view(build, b):
    return {"p1": int(build[1][b]), "p2": int(build[2][b])}


def passing(build, probe, f, semi_keys=None):
    """[(probe row, build row or -1, filter TRUE on the candidate pair)]"""
    return [(r, b, b >= 0 and f(row_view(probe, r), build_view(build, b)) is True) for r, b in candidates(build, probe, semi_keys)]


def output_run(ctx, look, probe, kind, filt_nodes, out_cols, ordered, semi=None):
    stages = ([(D.STAGE_SEMI, 5, semi)] if semi is not None else []) + [(kind, 0, look)]
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, stages)
    try:
        p.set_stage_filter(len(stages) - 1, filt_nodes)
        p.sink_output(out_cols, ordered=ordered)
        push_all(p, probe)
        rows = drain_rows(p)
        return rows if ordered else sorted(rows)
    finally:
        p.close()


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("fname", ["probe", "payload", "kleene", "decimal"])
@pytest.mark.parametrize("kind", [D.STAGE_INNER, D.STAGE_SEMI, D.STAGE_ANTI])
def test_output_sinks(ctx, kind, fname, ordered):
    rng = np.random.default_rng(100 * kind + 7 * len(fname) + ordered)
    build = make_build(rng, 3000)
    probe = make_probe(rng, 40000, build[0])
    look = lookup(ctx, build, 2)
    pay0 = NIN   # INNER: the stage's fields are virtual columns NIN, NIN + 1; SEMI / ANTI: the same indices, seen by the filter only
    nodes, f = filt(fname, pay0)
    out_cols = [4] + ([NIN, NIN + 1] if kind == D.STAGE_INNER else [])
    got = output_run(ctx, look, probe, kind, nodes, out_cols, ordered)
    look.close()
    res = passing(build, probe, f)
    if kind == D.STAGE_ANTI:
        exp = [(r,) for r, b, ok in res if not ok]
    elif kind == D.STAGE_SEMI:
        exp = [(r,) for r, b, ok in res if ok]
    else:
        exp = [(r, int(build[1][b]), int(build[2][b])) for r, b, ok in res if ok]
    assert got == (exp if ordered else sorted(exp))
    if fname == "probe" and kind == D.STAGE_ANTI:   # not the predicate pushed below the join: rows with x <= 100 or NULL stay when they match
        pushed = [(r,) for r, b, ok in res if b < 0 and f(row_view(probe, r), None) is True]
        assert exp != pushed and set(pushed) < set(exp)


@pytest.mark.parametrize("kind", ["inner", "right_semi", "right_anti"])
def test_against_oracle_and_unfused_join(ctx, kind):
    """the same filter through the oracle's hash join and dfgpu_hashjoin (build columns: key, p1, p2; probe columns: key, x, q, rid)"""
    rng = np.random.default_rng(5 + len(kind))
    build = make_build(rng, 2000)
    probe = make_probe(rng, 20000, build[0])
    look = lookup(ctx, build, 2)
    st = {"inner": D.STAGE_INNER, "right_semi": D.STAGE_SEMI, "right_anti": D.STAGE_ANTI}[kind]
    nodes, _ = filt("kleene", NIN)
    got = output_run(ctx, look, probe, st, nodes, [4], True)
    look.close()
    keep = probe[5][0] < 80
    bcols = [(build[0], None), (build[1], None), (build[2], None)]
    pcols = [(probe[0][0][keep], probe[0][1][keep]), (probe[1][0][keep], probe[1][1][keep]), (probe[2][0][keep], None), (probe[4][0][keep], None)]
    # the JoinFilter's intermediate batch: [probe x, build p2]
    onodes = [(O.E_COLUMN, 0, None, 0, 0), (O.E_LITERAL, 0, np.int64, 0, 100), (O.E_BINARY, O.OP_GT, None, 0, 0),
              (O.E_COLUMN, 1, None, 0, 0), (O.E_LITERAL, 0, np.int32, 0, 3), (O.E_BINARY, O.OP_EQ, None, 0, 0), (O.E_BINARY, O.OP_OR, None, 0, 0)]
    oj = {"inner": O.J_INNER, "right_semi": O.J_RIGHT_SEMI, "right_anti": O.J_RIGHT_ANTI}[kind]
    gj = {"inner": D.JOIN_INNER, "right_semi": D.JOIN_RIGHT_SEMI, "right_anti": D.JOIN_RIGHT_ANTI}[kind]
    ref = O.hash_join(bcols, pcols, [0], [0], [1], [3], join_type=oj, filter=([1, 0], [1, 2], onodes))
    uf = gpu_hash_join(ctx, bcols, pcols, [0], [0], [1], [3], join_type=gj, filter=([1, 0], [1, 2], gpu_nodes(D, onodes)))
    exp = sorted(int(v) for v in ref[0][0])
    assert sorted(int(v) for v in uf[0][0]) == exp
    assert sorted(r[0] for r in got) == exp


def agg_run(ctx, look, probe, kind, filt_nodes, group, aggs, semi=None):
    stages = ([(D.STAGE_SEMI, 5, semi)] if semi is not None else []) + [(kind, 0, look)]
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, stages)
    try:
        p.set_stage_filter(len(stages) - 1, filt_nodes)
        p.sink_aggregate(group, aggs)
        push_all(p, probe)
        return sorted(drain_rows(p), key=repr)
    finally:
        p.close()


# the same filters for dfgpu_hashjoin.set_filter: (sides, indices into [key, p1, p2] / [key, x, q, d], nodes over the intermediate batch)
UNFUSED_FILTERS = {
    "probe": ([1], [1], [C(0), L(100), B(D.OP_GT)]),
    "payload": ([0, 1], [1, 2], [C(0), C(1), B(D.OP_LT)]),
    "kleene": ([1, 0], [1, 2], [C(0), L(100), B(D.OP_GT), C(1), L(3, D.INT32), B(D.OP_EQ), B(D.OP_OR)]),
    "decimal": ([1], [3], [C(0), L(0, DEC), B(D.OP_GT)]),
}


def unfused_join_aggregate(ctx, build, probe, fname, join_type):
    """dfgpu_hashjoin with the filter -> dfgpu_agg: COUNT(*), SUM(x) GROUP BY build key, p2"""
    keep = probe[5][0] < 80
    bcols = [(build[0], None), (build[1], None), (build[2], None)]
    pcols = [(probe[0][0][keep], probe[0][1][keep]), (probe[1][0][keep], probe[1][1][keep]), (probe[2][0][keep], None),
             (O.Dec(probe[3][0][keep].tolist(), 15, 2), probe[3][1][keep])]
    from decimal_util import gpu_host_col
    j = D.HashJoinHandle(ctx, [D.INT64, D.INT32, D.INT32], [D.INT64, D.INT64, D.INT32, DEC], [0], [0], [0, 0, 1], [0, 2, 1], join_type, ordered_output=False)
    j.set_filter(*UNFUSED_FILTERS[fname])
    j.push_build_host([gpu_host_col(D, c) for c in bcols]); j.finish_build()
    j.push_probe_host([gpu_host_col(D, c) for c in pcols]); j.finish_probe()
    cols = [[] for _ in range(3)]
    for b in j.drain(host=True):
        for i in range(3):
            v, val = b.column_numpy(i)
            cols[i].append((v, val if val is not None else np.ones(len(v), bool)))
    j.close()
    joined = [(np.concatenate([c[0] for c in cs]), np.concatenate([c[1] for c in cs])) for cs in cols]
    out = gpu_group_by(ctx, joined, [0, 1], [(D.AGG_COUNT_STAR, -1, -1), (D.AGG_SUM, 2, -1)])
    rows = []
    for r in range(len(out[0][0])):
        rows.append(tuple(None if (val is not None and not val[r]) else int(v[r]) for v, val in out))
    return sorted(rows, key=repr)


@pytest.mark.parametrize("fname", ["probe", "payload", "kleene", "decimal"])
@pytest.mark.parametrize("kind", ["left", "left_anti", "left_semi", "inner"])
def test_join_keyed_sink(ctx, kind, fname):
    rng = np.random.default_rng(31 + len(kind) + 3 * len(fname))
    build = make_build(rng, 2500)
    probe = make_probe(rng, 30000, build[0])
    look = lookup(ctx, build, 2, n_acc=5)
    nodes, f = filt(fname, NIN)
    res = passing(build, probe, f)
    per = {}
    for r, b, ok in res:
        if ok:
            per.setdefault(b, []).append(r)
    key = build[0]
    st = {"left": D.STAGE_LEFT, "left_anti": D.STAGE_LEFT_ANTI, "left_semi": D.STAGE_INNER, "inner": D.STAGE_INNER}[kind]
    aggs = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(1)])] if kind in ("left", "inner") else []
    got = agg_run(ctx, look, probe, st, nodes, [0, NIN + 1], aggs)
    look.close()

    def sums(rows):
        v = [int(probe[1][0][r]) for r in rows if probe[1][1][r]]
        return sum(v) if v else None
    if kind == "left":
        exp = [(int(key[b]), int(build[2][b]), max(len(per.get(b, [])), 1), sums(per.get(b, []))) for b in range(len(key))]
    elif kind == "left_anti":
        exp = [(int(key[b]), int(build[2][b])) for b in range(len(key)) if b not in per]
    elif kind == "left_semi":
        exp = [(int(key[b]), int(build[2][b])) for b in per]
    else:
        exp = [(int(key[b]), int(build[2][b]), len(rows), sums(rows)) for b, rows in per.items()]
    assert got == sorted(exp, key=repr)
    if kind in ("left", "inner"):
        assert unfused_join_aggregate(ctx, build, probe, fname, D.JOIN_LEFT if kind == "left" else D.JOIN_INNER) == got


def test_stage_filters_on_two_stages_read_earlier_payload(ctx):
    """stage 0 INNER over lookup A (payload a1, a2), stage 1 SEMI over lookup B with its own payload: B's filter reads A's field and
    its own; sink = dense aggregate without GROUP BY"""
    rng = np.random.default_rng(77)
    ba = make_build(rng, 2000)
    bb = (ba[0].copy(), rng.integers(-50, 50, 2000).astype(np.int32), rng.integers(0, 8, 2000).astype(np.int32))
    probe = make_probe(rng, 30000, ba[0])
    la, lb = lookup(ctx, ba, 2), lookup(ctx, bb, 1)
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_INNER, 0, la), (D.STAGE_SEMI, 0, lb)])
    p.set_stage_filter(0, [C(1), L(-500), B(D.OP_GT)])                                   # x > -500
    p.set_stage_filter(1, [C(NIN), C(NIN + 2), B(D.OP_LT)])                             # a1 < b1 (B's own payload)
    p.sink_aggregate_dense([], [], [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(4)])])
    push_all(p, probe)
    got = drain_rows(p)
    p.close(); la.close(); lb.close()
    rows = [r for r, b, ok in passing(ba, probe, lambda rv, bv: None if rv["x"] is None else rv["x"] > -500) if ok and ba[1][b] < bb[1][b]]
    assert got == [(len(rows), sum(rows) if rows else None)]


@pytest.mark.parametrize("fname", ["payload", "decimal"])
def test_dense_sink_grouped_on_payload(ctx, fname):
    rng = np.random.default_rng(41 + len(fname))
    build = make_build(rng, 2000)
    probe = make_probe(rng, 30000, build[0])
    look = lookup(ctx, build, 2)
    nodes, f = filt(fname, NIN)
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_INNER, 0, look)])
    p.set_stage_filter(0, nodes)
    p.sink_aggregate_dense([NIN + 1], [(0, 7)], [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(4)])])
    push_all(p, probe)
    got = drain_rows(p)
    p.close(); look.close()
    groups = {}
    for r, b, ok in passing(build, probe, f):
        if ok:
            groups.setdefault(int(build[2][b]), []).append(r)
    assert got == [(g, len(v), sum(v)) for g, v in sorted(groups.items())]


@pytest.mark.parametrize("fname", ["kleene", "decimal"])
def test_hash_sink_grows_and_replays(ctx, fname):
    rng = np.random.default_rng(43 + len(fname))
    build = make_build(rng, 3000)
    probe = make_probe(rng, 200000, build[0], hit=0.9)
    look = lookup(ctx, build, 2)
    nodes, f = filt(fname, NIN)
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_INNER, 0, look)])
    p.set_stage_filter(0, nodes)
    p.sink_aggregate_hash([2, NIN], [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(4)])], capacity_hint=1)
    push_all(p, probe, pushes=1)
    got = sorted(drain_rows(p))
    replayed = p.metric("replayed_rows")
    p.close(); look.close()
    groups = {}
    for r, b, ok in passing(build, probe, f):
        if ok:
            groups.setdefault((int(probe[2][0][r]), int(build[1][b])), []).append(r)
    assert replayed > 0
    assert got == sorted((k[0], k[1], len(v), sum(v)) for k, v in groups.items())


@pytest.mark.parametrize("fname", ["payload", "decimal"])
@pytest.mark.parametrize("pack", [False, True])
def test_build_sink(ctx, pack, fname):
    """filtered INNER stage -> build sink (direct when the table is sized up front, pack otherwise), read back through an INNER stage"""
    rng = np.random.default_rng(51 + pack + len(fname))
    build = make_build(rng, 2000)
    probe = make_probe(rng, 30000, build[0])
    look = lookup(ctx, build, 2)
    nodes, f = filt(fname, NIN)
    target = D.Lookup(ctx, D.INT64, [D.INT32], expected_rows=0 if pack else 40000)
    p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_INNER, 0, look)])
    p.set_stage_filter(0, nodes)
    p.sink_build(target, 4, [NIN + 1])
    push_all(p, probe)
    p.close()
    exp = sorted((r, int(build[2][b])) for r, b, ok in passing(build, probe, f) if ok)
    rid = np.arange(len(probe[0][0]), dtype=np.int64)
    q = D.Pipeline(ctx, [D.INT64], None, [(D.STAGE_INNER, 0, target)])
    q.sink_output([0, 1], ordered=True)
    q.push_host([D.HostColumn(rid)])
    q.finish()
    got = drain_rows(q)
    q.close(); look.close(); target.close()
    assert got == exp


@pytest.mark.parametrize("kind", [D.STAGE_INNER, D.STAGE_SEMI, D.STAGE_ANTI])
@pytest.mark.parametrize("structure", ["bitmap", "bloom"])
def test_bitmap_and_bloom_lookups(ctx, kind, structure):
    rng = np.random.default_rng(61 + kind + 5 * len(structure))
    build = make_build(rng, 3000)
    probe = make_probe(rng, 40000, build[0])
    if structure == "bitmap":   # key set over a dense range: a bitmap, decided in phase A unless its ANTI stage has a filter
        look = lookup(ctx, build, 0, key_range=(1, 12000))
        assert look.metric("mode") == 1
    else:
        look = lookup(ctx, build, 2, membership_filter=1)
        assert look.metric("filter_bytes") > 0
    nodes, f = filt("probe", NIN)
    out_cols = [4]
    for ordered in (True, False):
        got = output_run(ctx, look, probe, kind, nodes, out_cols, ordered)
        res = passing(build, probe, f)
        exp = [(r,) for r, b, ok in res if ok != (kind == D.STAGE_ANTI)]
        assert got == (exp if ordered else sorted(exp))
    look.close()


def test_division_by_zero_raises_only_on_candidate_pairs(ctx):
    rng = np.random.default_rng(71)
    build = make_build(rng, 1000)
    probe = make_probe(rng, 20000, build[0], hit=0.0)
    probe[0] = (probe[0][0] + 10**9, probe[0][1])               # no key matches
    look = lookup(ctx, build, 2)
    nodes = [C(4), C(6), B(D.OP_DIVIDE), L(0), B(D.OP_GT)]       # rid / zero > 0
    for kind in (D.STAGE_INNER, D.STAGE_ANTI):
        got = output_run(ctx, look, probe, kind, nodes, [4], True)
        assert len(got) == (0 if kind == D.STAGE_INNER else int((probe[5][0] < 80).sum()))
    probe2 = make_probe(rng, 20000, build[0], hit=0.9)
    with pytest.raises(D.DfgpuError) as e:
        output_run(ctx, look, probe2, D.STAGE_INNER, nodes, [4], True)
    assert e.value.code == ERR_ARITH
    look.close()


def test_rejections(ctx):
    rng = np.random.default_rng(81)
    build = make_build(rng, 500)
    look = lookup(ctx, build, 2)
    maybe = D.Lookup(ctx, D.INT64, [], expected_rows=1000, filter_only=True)
    ok = [C(1), L(0), B(D.OP_GT)]

    def code(stages, stage, nodes, before=None):
        p = D.Pipeline(ctx, PROBE_TYPES, None, stages)
        try:
            if before:
                before(p)
            p.set_stage_filter(stage, nodes)
            return D.OK
        except D.DfgpuError as err:
            return err.code
        finally:
            p.close()
    inner = [(D.STAGE_INNER, 0, look)]
    assert code([(D.STAGE_MAYBE, 0, maybe)], 0, ok) == ERR_UNSUPPORTED
    assert code(inner, 0, [C(1), L(0), B(D.OP_PLUS)]) == ERR_INVALID                  # not Boolean
    assert code(inner, 0, [C(NIN + 2), L(0), B(D.OP_GT)]) == ERR_INVALID              # out of range
    assert code(inner + [(D.STAGE_INNER, 0, look)], 0, [C(NIN + 2), L(0, D.INT32), B(D.OP_GT)]) == ERR_INVALID   # a later stage's field
    assert code(inner, 1, ok) == ERR_INVALID                                         # no such stage
    fallible = [C(1), L(0), B(D.OP_GT), C(4), C(6), B(D.OP_DIVIDE), L(0), B(D.OP_GT), B(D.OP_AND)]
    assert code(inner, 0, fallible) == ERR_UNSUPPORTED
    big = [C(1), L(0), B(D.OP_GT)] + [C(1), L(0), B(D.OP_GT), B(D.OP_OR)] * 32          # 131 nodes
    assert code(inner, 0, big) == ERR_UNSUPPORTED
    assert code(inner, 0, ok, before=lambda p: p.set_stage_filter(0, ok)) == ERR_STATE

    def pushed(p):
        p.sink_output([4])
        p.push_host(host_cols(make_probe(rng, 10, build[0]), 0, 10))
    assert code(inner, 0, ok, before=pushed) == ERR_STATE
    look.close(); maybe.close()


def test_filtered_pipeline_takes_neither_ring_nor_partitioned_path(ctx, monkeypatch):
    monkeypatch.setenv("DFGPU_PIPE_RADIX_PARTS", "2")   # admits the partitioned aggregate on a small table
    rng = np.random.default_rng(91)
    build = make_build(rng, 5000)
    n = 1 << 20
    probe = make_probe(rng, n, build[0])
    probe[0] = (probe[0][0], None)                        # keys without a validity bitmap: ring-eligible
    look = lookup(ctx, build, 0, n_acc=2, membership_filter=1)
    res = {}
    for filtered in (False, True):
        p = D.Pipeline(ctx, PROBE_TYPES, None, [(D.STAGE_INNER, 0, look)])
        if filtered:
            p.set_stage_filter(0, [C(2), L(0, D.INT32), B(D.OP_GT)])    # q > 0
        p.sink_aggregate([0], [(D.AGG_SUM, [C(4)])])
        push_all(p, probe, pushes=1)
        res[filtered] = (sorted(drain_rows(p)), p.metric("ring_launches"), p.metric("partitioned_launches"))
        p.close()
        look.close()
        look = lookup(ctx, build, 0, n_acc=2, membership_filter=1)
    look.close()
    assert res[False][1] > 0 and res[False][2] > 0
    assert res[True][1] == 0 and res[True][2] == 0
    pos = {int(k): i for i, k in enumerate(build[0])}
    per = {}
    for r in np.nonzero(probe[2][0] > 0)[0]:
        b = pos.get(int(probe[0][0][r]))
        if b is not None:
            per[int(build[0][b])] = per.get(int(build[0][b]), 0) + int(r)
    assert res[True][0] == sorted(per.items())


def test_q19_and_q17_shapes(ctx):
    """small-SF Q19 (INNER stage on part with the three-way OR filter) and Q17 (SEMI on a part key set, INNER on {partkey -> avg quantity}
    with CAST(quantity AS Float64) < 0.2 * avg), no GROUP BY, against numpy"""
    rng = np.random.default_rng(19)
    n_part, n_li = 20000, 600000
    pkey = np.arange(1, n_part + 1, dtype=np.int64)
    brand = rng.integers(0, 25, n_part).astype(np.int8); cont = rng.integers(0, 40, n_part).astype(np.int8); size = rng.integers(1, 51, n_part).astype(np.int16)
    lpk = rng.integers(1, n_part + 1, n_li).astype(np.int64); qty = rng.integers(1, 51, n_li).astype(np.int64)
    price = rng.integers(90_000, 10_500_000, n_li).astype(np.int64); disc = rng.integers(0, 11, n_li).astype(np.int64)
    mode = rng.integers(0, 7, n_li).astype(np.int8); instr = rng.integers(0, 4, n_li).astype(np.int8)
    part = D.Lookup(ctx, D.INT64, [D.INT8, D.INT8, D.INT16])
    bp = D.Pipeline(ctx, [D.INT64, D.INT8, D.INT8, D.INT16]); bp.sink_build(part, 0, [1, 2, 3])
    bp.push_host([D.HostColumn(pkey), D.HostColumn(brand), D.HostColumn(cont), D.HostColumn(size)]); bp.finish(); bp.close()
    # lineitem: 0 partkey, 1 qty, 2 price, 3 disc, 4 shipmode, 5 shipinstruct; part fields 6 brand, 7 container, 8 size
    I8 = lambda v: L(v, D.INT8)                                                   # noqa: E731

    def eq_any(col, vals):
        out = [C(col), I8(vals[0]), B(D.OP_EQ)]
        for v in vals[1:]:
            out += [C(col), I8(v), B(D.OP_EQ), B(D.OP_OR)]
        return out

    def conj(b, conts, qlo, qhi, smax):
        return ([C(6), I8(b), B(D.OP_EQ)] + eq_any(7, conts) + [B(D.OP_AND), C(1), L(qlo), B(D.OP_GTEQ), B(D.OP_AND), C(1), L(qhi), B(D.OP_LTEQ),
                B(D.OP_AND), C(8), L(1, D.INT16), B(D.OP_GTEQ), B(D.OP_AND), C(8), L(smax, D.INT16), B(D.OP_LTEQ), B(D.OP_AND)])
    arms = [(12, [0, 1, 2, 3], 1, 11, 5), (23, [10, 11, 12, 13], 10, 20, 10), (34 % 25, [20, 21, 22, 23], 20, 30, 15)]
    f19 = conj(*arms[0]) + conj(*arms[1]) + [B(D.OP_OR)] + conj(*arms[2]) + [B(D.OP_OR)]
    assert len(f19) <= 128
    pred = [C(4), I8(1), B(D.OP_EQ), C(4), I8(3), B(D.OP_EQ), B(D.OP_OR), C(5), I8(0), B(D.OP_EQ), B(D.OP_AND)]
    rev = [C(2), L(100), C(3), B(D.OP_MINUS), B(D.OP_MULTIPLY)]
    li_types = [D.INT64, D.INT64, D.INT64, D.INT64, D.INT8, D.INT8]
    li_cols = lambda: [D.HostColumn(lpk), D.HostColumn(qty), D.HostColumn(price), D.HostColumn(disc), D.HostColumn(mode), D.HostColumn(instr)]  # noqa: E731
    p = D.Pipeline(ctx, li_types, pred, [(D.STAGE_INNER, 0, part)])
    p.set_stage_filter(0, f19)
    p.sink_aggregate_dense([], [], [(D.AGG_SUM, rev)])
    p.push_host(li_cols()); p.finish()
    got19 = drain_rows(p)[0][0]
    p.close()
    b, c, s = brand[lpk - 1], cont[lpk - 1], size[lpk - 1]
    m = ((mode == 1) | (mode == 3)) & (instr == 0)
    arm = np.zeros(n_li, bool)
    for br, cs, qlo, qhi, smax in arms:
        arm |= (b == br) & np.isin(c, cs) & (qty >= qlo) & (qty <= qhi) & (s >= 1) & (s <= smax)
    assert got19 == int((price * (100 - disc))[m & arm].sum()) and (m & arm).sum() > 0
    # Q17: the AVG build is {partkey -> avg quantity (Float64)} from numpy here; the fused pass is the one under test
    sel_parts = pkey[(brand == 3) & (cont < 8)]
    keyset = D.Lookup(ctx, D.INT64, [])
    kp = D.Pipeline(ctx, [D.INT64]); kp.sink_build(keyset, 0, []); kp.push_host([D.HostColumn(sel_parts)]); kp.finish(); kp.close()
    cnt = np.bincount(lpk, minlength=n_part + 1); tot = np.bincount(lpk, weights=qty.astype(np.float64), minlength=n_part + 1)
    has = cnt[1:] > 0
    avg = (tot[1:][has] / cnt[1:][has])
    avgl = D.Lookup(ctx, D.INT64, [D.FLOAT64])
    ap = D.Pipeline(ctx, [D.INT64, D.FLOAT64]); ap.sink_build(avgl, 0, [1]); ap.push_host([D.HostColumn(pkey[has]), D.HostColumn(avg)]); ap.finish(); ap.close()
    f17 = [C(1), (D.EXPR_CAST, 0, D.FLOAT64, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.FLOAT64, 0, 0, 0.2), C(6), B(D.OP_MULTIPLY), B(D.OP_LT)]
    p = D.Pipeline(ctx, li_types, None, [(D.STAGE_SEMI, 0, keyset), (D.STAGE_INNER, 0, avgl)])
    p.set_stage_filter(1, f17)
    p.sink_aggregate_dense([], [], [(D.AGG_SUM, [C(2)]), (D.AGG_COUNT_STAR, None)])
    p.push_host(li_cols()); p.finish()
    got17 = drain_rows(p)[0]
    p.close(); part.close(); keyset.close(); avgl.close()
    avg_of = np.zeros(n_part + 1); avg_of[1:][has] = avg
    m17 = np.isin(lpk, sel_parts) & (qty.astype(np.float64) < 0.2 * avg_of[lpk])
    assert got17 == (int(price[m17].sum()) if m17.any() else None, int(m17.sum()))


def test_device_push_matches_host_push(ctx):
    """the same filtered pipeline fed by device columns (no validity bitmaps) and by host columns"""
    rng = np.random.default_rng(97)
    build = make_build(rng, 2000)
    probe = [(v, None) for v, _ in make_probe(rng, 30000, build[0])]
    look = lookup(ctx, build, 2)
    nodes, f = filt("kleene", NIN)
    res = {}
    for device in (False, True):
        p = D.Pipeline(ctx, PROBE_TYPES, PRED, [(D.STAGE_INNER, 0, look)])
        p.set_stage_filter(0, nodes)
        p.sink_output([4, NIN], ordered=True)
        if device:
            bufs, cols = [], []
            for i, (v, _) in enumerate(probe):
                arr = np.asarray(D.decimal_to_words([int(z) for z in v])) if i == 3 else v
                bufs.append(ctx.to_device(arr))
                c = D.Column()
                c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = PROBE_TYPES[i], 0, len(v), 0, 0, bufs[-1].ptr, None
                cols.append(c)
            p.push_device(cols)
            p.finish()
        else:
            push_all(p, probe, pushes=1)
        res[device] = drain_rows(p)
        p.close()
    look.close()
    pos = {int(k): i for i, k in enumerate(build[0])}
    exp = []
    for r in np.nonzero(probe[5][0] < 80)[0]:
        b = pos.get(int(probe[0][0][r]), -1)
        if b >= 0 and (int(probe[1][0][r]) > 100 or int(build[2][b]) == 3):
            exp.append((int(r), int(build[1][b])))
    assert res[True] == res[False] == exp
