"""Fused joins on composite keys (dfgpu_lookup_create_composite, dfgpu_pipeline_set_stage_keys, dfgpu_pipeline_sink_build_composite):
2 to 4 integer-like key columns packed exactly into one 64-bit key.  Checked against a row-by-row Python restatement of the join
(NullEqualsNothing: a NULL component never matches), the oracle's multi-column hash join and the unfused dfgpu_hashjoin on the same
keys.  The packed key of a probe row with a NULL or out-of-domain component is the sentinel D = prod r_g, which no lookup holds."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(__file__))
from harness import assert_cols_equal, batches_to_cols, gpu_group_by, gpu_hash_join  # noqa: E402

pytestmark = pytest.mark.gpu

C = lambda i: (D.EXPR_COLUMN, i, 0, 0, 0, 0.0)                                 # noqa: E731
L = lambda v, t=D.INT64: (D.EXPR_LITERAL, 0, t, 0, v, 0.0)                     # noqa: E731
B = lambda op: (D.EXPR_BINARY, op, 0, 0, 0, 0.0)                               # noqa: E731
ERR_INVALID, ERR_UNSUPPORTED, ERR_STATE = -1, -3, -5                           # include/dfgpu.h
NP = {D.INT32: np.int32, D.INT64: np.int64, D.UINT16: np.uint16, D.DATE32: np.int32, D.INT8: np.int8, D.UINT64: np.uint64}
# (type, min, max) per component; D.INT32 with a small domain stands for dictionary codes
SPECS = {
    2: [(D.INT32, -50, 49), (D.INT64, -10**12, -10**12 + 999)],
    3: [(D.UINT16, 0, 300), (D.DATE32, -20, 40), (D.INT64, -7, 1000)],
    4: [(D.INT32, 0, 24), (D.INT32, -1000, -900), (D.UINT16, 5, 17), (D.INT64, -3, 3)],
}


@pytest.fixture(scope="module")
def ctx():
    c = D.Context(0)
    yield c
    c.close()


def domain(spec):
    d = 1
    for _, lo, hi in spec:
        d *= hi - lo + 1
    return d


def decode(spec, idx):
    """the component tuples of packed indices idx (component 0 varies fastest)"""
    out = []
    for t, lo, hi in spec:
        r = hi - lo + 1
        out.append((idx % r + lo).astype(NP[t]))
        idx = idx // r
    return out


def make_build(rng, spec, n, null_rows=0):
    idx = rng.choice(domain(spec), n, replace=False).astype(np.int64)
    comps = decode(spec, idx)
    valid = None
    if null_rows:
        valid = np.ones(n, bool)
        valid[rng.choice(n, null_rows, replace=False)] = False
    keys = [(c, valid if g == 1 else None) for g, c in enumerate(comps)]
    return keys, rng.integers(-10**6, 10**6, n).astype(np.int64)


def make_probe(rng, spec, n, build_keys, null_frac=0.1):
    """60 % build tuples, the rest random in-domain tuples; some components one past either end of their domain; NULLs"""
    nb = len(build_keys[0][0])
    pick = rng.integers(0, nb, n)
    hit = rng.random(n) < 0.6
    rand = decode(spec, rng.integers(0, domain(spec), n).astype(np.int64))
    cols = []
    for g, (t, lo, hi) in enumerate(spec):
        v = np.where(hit, build_keys[g][0][pick], rand[g]).astype(np.int64)
        out = rng.random(n) < 0.03
        edge = np.where(rng.random(n) < 0.5, lo - 1, hi + 1)
        if t in (D.UINT16,) and lo == 0:
            edge = np.full(n, hi + 1)
        v = np.where(out, edge, v).astype(NP[t])
        valid = rng.random(n) >= null_frac if g != 1 else None
        cols.append((v, valid))
    return cols


def ref_index(build_keys):
    m = {}
    nb = len(build_keys[0][0])
    for i in range(nb):
        if any(val is not None and not val[i] for _, val in build_keys):
            continue
        m[tuple(int(v[i]) for v, _ in build_keys)] = i
    return m


def probe_tuple(cols, j):
    if any(val is not None and not val[j] for _, val in cols):
        return None
    return tuple(int(v[j]) for v, _ in cols)


def dcol(ctx, keep, t, vals, valid, off=0):
    """a device column whose values and bitmap start `off` rows into their buffers (Arrow offset)"""
    n = len(vals)
    buf = ctx.to_device(np.concatenate([np.zeros(off, vals.dtype), vals]))
    keep.append(buf)
    c = D.Column()
    c.type, c.flags, c.length, c.offset = t, 0, n, off
    c.values = buf.ptr
    if valid is not None:
        vb = ctx.to_device(D.pack_bits(np.concatenate([np.zeros(off, bool), valid])))
        keep.append(vb)
        c.validity, c.null_count = vb.ptr, -1
    else:
        c.validity, c.null_count = None, 0
    return c


def build_lookup(ctx, spec, keys, pay=None, off=0, n_acc=0, pushes=1, **kw):
    """a composite-key lookup built by a pipeline's composite build sink: input = the key columns (+ payload)"""
    types = [t for t, _, _ in spec]
    look = D.Lookup(ctx, key_types=types, key_ranges=[(lo, hi) for _, lo, hi in spec],
                    payload_types=[D.INT64] if pay is not None else [], n_acc_words=n_acc, **kw)
    p = D.Pipeline(ctx, types + ([D.INT64] if pay is not None else []))
    try:
        k = len(spec)
        p.sink_build(look, key_cols=list(range(k)), payload_cols=[k] if pay is not None else [])
        n = len(keys[0][0])
        keep = []
        for q in range(pushes):
            s, e = n * q // pushes, n * (q + 1) // pushes
            cols = [dcol(ctx, keep, t, v[s:e], None if val is None else val[s:e], off) for (t, _, _), (v, val) in zip(spec, keys)]
            if pay is not None:
                cols.append(dcol(ctx, keep, D.INT64, pay[s:e], None))
            p.push_device(cols)
        p.finish()
    finally:
        p.close()
    return look


# ---------------------------------------------------------------------------------------------------------------------------------
# INNER with payload, through the ordered output sink, against the restatement, the oracle and dfgpu_hashjoin
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("off", [0, 3, 37])
def test_inner_with_payload_matches_every_reference(ctx, k, off):
    rng = np.random.default_rng(100 * k + off)
    spec = SPECS[k]
    nb, n = 5000, 40_000
    bkeys, pay = make_build(rng, spec, nb, null_rows=50)
    probe = make_probe(rng, spec, n, bkeys)
    x = np.arange(n, dtype=np.int64)
    look = build_lookup(ctx, spec, bkeys, pay, off=off, n_acc=1)
    assert look.metric("key_domain") == domain(spec) and look.metric("rows") == nb - 50 and look.metric("null_keys") == 50
    types = [t for t, _, _ in spec] + [D.INT64]
    p = D.Pipeline(ctx, types, stages=[(D.STAGE_INNER, list(range(k)), look)])
    keep = []
    try:
        p.sink_output([k, k + 1])       # the probe row number, the build payload
        p.push_device([dcol(ctx, keep, t, v, val, off) for (t, _, _), (v, val) in zip(spec, probe)] + [dcol(ctx, keep, D.INT64, x, None, off)])
        p.finish()
        got = batches_to_cols(p.drain(host=True), 2)
    finally:
        p.close(); look.close()
    m = ref_index(bkeys)
    rows = [(j, m[t]) for j in range(n) for t in [probe_tuple(probe, j)] if t is not None and t in m]
    exp = [(np.array([j for j, _ in rows], np.int64), None), (pay[np.array([i for _, i in rows], np.int64)], None)]
    assert_cols_equal(got, exp, ordered=True, what="restatement")
    # the oracle and the unfused join: build (keys, payload), probe (keys, row number); output probe row number, build payload
    build_t = bkeys + [(pay, None)]
    probe_t = probe + [(x, None)]
    on = list(range(k))
    ora = O.hash_join(build_t, probe_t, on, on, [1, 0], [k, k], phj_threshold=0, phj_density=float("inf"))
    assert_cols_equal(got, ora, ordered=False, what="oracle")
    bt = [t for t, _, _ in spec] + [D.INT64]
    unf = gpu_hash_join(ctx, build_t, probe_t, on, on, [1, 0], [k, k], build_types=bt, probe_types=bt)
    assert_cols_equal(got, unf, ordered=False, what="dfgpu_hashjoin")


def test_aliasing_tuples_do_not_match(ctx):
    """domains [0, 9] x [0, 9]: (0, 10) and (-1, 5) are out of domain, so they must not alias (1, 0) or (0, 5)"""
    spec = [(D.INT64, 0, 9), (D.INT64, 0, 9)]
    bk = [(np.array([1, 0], np.int64), None), (np.array([0, 5], np.int64), None)]
    for payload in (False, True):
        look = build_lookup(ctx, spec, bk, np.array([11, 22], np.int64) if payload else None)
        assert look.metric("mode") == (0 if payload else 1)       # a key set over D = 100 is a bitmap
        pk = [np.array([0, -1, 1, 0, 10, 0], np.int64), np.array([10, 5, 0, 5, 0, -10], np.int64)]
        for kind, exp in ((D.STAGE_SEMI, [2, 3]), (D.STAGE_ANTI, [0, 1, 4, 5])):
            p = D.Pipeline(ctx, [D.INT64, D.INT64, D.INT64], stages=[(kind, [0, 1], look)])
            try:
                p.sink_output([2])
                p.push_host([D.HostColumn(pk[0]), D.HostColumn(pk[1]), D.HostColumn(np.arange(6, dtype=np.int64))])
                p.finish()
                got = batches_to_cols(p.drain(host=True), 1)
            finally:
                p.close()
            assert got[0][0].tolist() == exp, (payload, kind)
        look.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# stage kinds: SEMI / ANTI over bitmap and hash key sets, MAYBE, LEFT, LEFT_ANTI; a stage filter; NULL keys on both sides
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("kind", [D.STAGE_SEMI, D.STAGE_ANTI, D.STAGE_MAYBE])
def test_semi_anti_maybe_stages(ctx, k, kind):
    rng = np.random.default_rng(7 * k + kind)
    spec = SPECS[k]
    bkeys, _ = make_build(rng, spec, 3000, null_rows=40)
    probe = make_probe(rng, spec, 30_000, bkeys)
    n = len(probe[0][0])
    extra = {"filter_only": True, "expected_rows": 3000} if kind == D.STAGE_MAYBE else {}
    look = build_lookup(ctx, spec, bkeys, off=3, **extra)
    assert look.metric("null_keys") == 40
    if kind != D.STAGE_MAYBE:
        assert look.metric("mode") == (1 if domain(spec) < (1 << 32) else 0)
    types = [t for t, _, _ in spec] + [D.INT64]
    p = D.Pipeline(ctx, types, stages=[(kind, list(range(k)), look)])
    try:
        p.sink_output([k], ordered=False)
        p.push_host([D.HostColumn(v, val, t) for (t, _, _), (v, val) in zip(spec, probe)] + [D.HostColumn(np.arange(n, dtype=np.int64))])
        p.finish()
        got = np.sort(batches_to_cols(p.drain(host=True), 1)[0][0])
    finally:
        p.close(); look.close()
    m = ref_index(bkeys)
    hit = np.array([probe_tuple(probe, j) in m for j in range(n)])
    if kind == D.STAGE_MAYBE:      # a membership pre-filter: every match survives, false positives may
        assert set(np.nonzero(hit)[0]) <= set(got.tolist()) and len(got) < n
    else:
        assert got.tolist() == np.nonzero(hit if kind == D.STAGE_SEMI else ~hit)[0].tolist()


@pytest.mark.parametrize("kind", [D.STAGE_SEMI, D.STAGE_ANTI])
def test_semi_and_anti_over_a_hash_key_set(ctx, kind):
    """a key set whose domain does not fit a bitmap (D >= 2^32) is a hash table without payload"""
    rng = np.random.default_rng(3)
    spec = [(D.INT64, -(1 << 40), (1 << 40)), (D.INT32, -5, 5)]
    b0 = rng.integers(-(1 << 40), 1 << 40, 4000).astype(np.int64)
    b1 = rng.integers(-5, 6, 4000).astype(np.int32)
    bkeys = [(b0, None), (b1, None)]
    look = build_lookup(ctx, spec, bkeys)
    assert look.metric("mode") == 0
    n = 20_000
    pick = rng.integers(0, 4000, n)
    p0 = np.where(rng.random(n) < 0.5, b0[pick], rng.integers(-(1 << 40), 1 << 40, n)).astype(np.int64)
    p1 = np.where(rng.random(n) < 0.8, b1[pick], rng.integers(-7, 8, n)).astype(np.int32)
    p = D.Pipeline(ctx, [D.INT64, D.INT32, D.INT64], stages=[(kind, [0, 1], look)])
    try:
        p.sink_output([2])
        p.push_host([D.HostColumn(p0), D.HostColumn(p1), D.HostColumn(np.arange(n, dtype=np.int64))])
        p.finish()
        got = batches_to_cols(p.drain(host=True), 1)[0][0]
    finally:
        p.close(); look.close()
    s = set(zip(b0.tolist(), b1.tolist()))
    assert got.tolist() == [j for j in range(n) if ((int(p0[j]), int(p1[j])) in s) == (kind == D.STAGE_SEMI)]


@pytest.mark.parametrize("mode", ["single", "partial"])
@pytest.mark.parametrize("k", [2, 4])
def test_join_keyed_sink_grouped_on_the_components(ctx, k, mode):
    """INNER stage + join-keyed sink grouped on every component and the payload: SUM(x), COUNT(x); Partial states merged by dfgpu_agg Final"""
    rng = np.random.default_rng(11 * k + len(mode))
    spec = SPECS[k]
    bkeys, pay = make_build(rng, spec, 4000)
    probe = make_probe(rng, spec, 50_000, bkeys)
    n = len(probe[0][0])
    xv = rng.integers(-10**6, 10**6, n).astype(np.int64)
    xval = rng.random(n) >= 0.2
    look = build_lookup(ctx, spec, bkeys, pay, n_acc=5)
    types = [t for t, _, _ in spec] + [D.INT64]
    p = D.Pipeline(ctx, types, stages=[(D.STAGE_INNER, list(range(k)), look)])
    amode = D.AGG_SINGLE if mode == "single" else D.AGG_PARTIAL
    try:
        p.sink_aggregate(list(range(k)) + [k + 1], [(D.AGG_SUM, [C(k)]), (D.AGG_COUNT, [C(k)])], amode)
        for s, e in ((0, n // 3), (n // 3, n)):
            p.push_host([D.HostColumn(v[s:e], None if val is None else val[s:e], t) for (t, _, _), (v, val) in zip(spec, probe)]
                        + [D.HostColumn(xv[s:e], xval[s:e])])
        p.finish()
        got = batches_to_cols(p.drain(host=True), k + 3)
    finally:
        p.close(); look.close()
    if mode == "partial":
        got = gpu_group_by(ctx, got, list(range(k + 1)), [(D.AGG_SUM, -1, -1), (D.AGG_COUNT, -1, -1)], mode=D.AGG_FINAL,
                           types=[t for t, _, _ in spec] + [D.INT64, D.INT64, D.INT64])
    m = ref_index(bkeys)
    acc = {}
    for j in range(n):
        t = probe_tuple(probe, j)
        if t is None or t not in m:
            continue
        s, c = acc.get(m[t], (None, 0))
        if xval[j]:
            s, c = (s or 0) + int(xv[j]), c + 1
        acc[m[t]] = (s, c)
    rows = sorted(acc)
    idx = np.array(rows, np.int64)
    sums = np.array([acc[i][0] or 0 for i in rows], np.int64)
    exp = [(bkeys[g][0][idx], None) for g in range(k)] + [(pay[idx], None), (sums, np.array([acc[i][0] is not None for i in rows])),
                                                         (np.array([acc[i][1] for i in rows], np.int64), None)]
    assert_cols_equal(got, exp, ordered=False, what=f"join-keyed {mode}")


@pytest.mark.parametrize("kind", [D.STAGE_LEFT, D.STAGE_LEFT_ANTI])
def test_left_and_left_anti_emit_the_build_components(ctx, kind):
    rng = np.random.default_rng(kind)
    spec = SPECS[3]
    bkeys, _ = make_build(rng, spec, 3000)
    probe = make_probe(rng, spec, 20_000, bkeys)
    n = len(probe[0][0])
    xv = rng.integers(0, 100, n).astype(np.int64)
    look = build_lookup(ctx, spec, bkeys, n_acc=3 if kind == D.STAGE_LEFT else 1)
    types = [t for t, _, _ in spec] + [D.INT64]
    p = D.Pipeline(ctx, types, stages=[(kind, [0, 1, 2], look)])
    try:
        p.sink_aggregate([0, 1, 2], [(D.AGG_SUM, [C(3)])] if kind == D.STAGE_LEFT else [])
        p.push_host([D.HostColumn(v, val, t) for (t, _, _), (v, val) in zip(spec, probe)] + [D.HostColumn(xv)])
        p.finish()
        got = batches_to_cols(p.drain(host=True), 4 if kind == D.STAGE_LEFT else 3)
    finally:
        p.close(); look.close()
    m = ref_index(bkeys)
    sums = {}
    for j in range(n):
        t = probe_tuple(probe, j)
        if t is not None and t in m:
            sums[m[t]] = sums.get(m[t], 0) + int(xv[j])
    rows = list(range(3000)) if kind == D.STAGE_LEFT else [i for i in range(3000) if i not in sums]
    idx = np.array(rows, np.int64)
    exp = [(bkeys[g][0][idx], None) for g in range(3)]
    if kind == D.STAGE_LEFT:
        exp.append((np.array([sums.get(i, 0) for i in rows], np.int64), np.array([i in sums for i in rows])))
    assert_cols_equal(got, exp, ordered=False, what="left")


def test_stage_filter_on_a_composite_stage(ctx):
    """INNER stage with a JoinFilter payload < x: a key match counts only when the filter is TRUE"""
    rng = np.random.default_rng(21)
    spec = SPECS[2]
    bkeys, pay = make_build(rng, spec, 2000)
    probe = make_probe(rng, spec, 20_000, bkeys)
    n = len(probe[0][0])
    xv = rng.integers(-10**6, 10**6, n).astype(np.int64)
    look = build_lookup(ctx, spec, bkeys, pay, n_acc=1)
    p = D.Pipeline(ctx, [D.INT32, D.INT64, D.INT64, D.INT64], stages=[(D.STAGE_INNER, [0, 1], look)])
    try:
        p.set_stage_filter(0, [C(4), C(2), B(D.OP_LT)])
        p.sink_output([3, 4])
        p.push_host([D.HostColumn(v, val, t) for (t, _, _), (v, val) in zip(spec, probe)] + [D.HostColumn(xv), D.HostColumn(np.arange(n, dtype=np.int64))])
        p.finish()
        got = batches_to_cols(p.drain(host=True), 2)
    finally:
        p.close(); look.close()
    m = ref_index(bkeys)
    rows = [(j, m[t]) for j in range(n) for t in [probe_tuple(probe, j)] if t is not None and t in m and pay[m[t]] < xv[j]]
    assert_cols_equal(got, [(np.array([j for j, _ in rows], np.int64), None), (pay[np.array([i for _, i in rows], np.int64)], None)], what="filter")


# ---------------------------------------------------------------------------------------------------------------------------------
# sinks: a build chain into a second composite stage, dense, hash, unordered output; multi-push host chunks
# ---------------------------------------------------------------------------------------------------------------------------------
def test_build_chain_into_a_second_composite_stage(ctx):
    """pipeline 1: probe a composite SEMI stage, build the survivors into a second composite lookup (other key columns);
    pipeline 2 probes that lookup with INNER and emits its payload"""
    rng = np.random.default_rng(31)
    spec_a = SPECS[2]
    spec_b = [(D.INT64, 0, 9999), (D.UINT16, 0, 99)]
    akeys, _ = make_build(rng, spec_a, 1500)
    la = build_lookup(ctx, spec_a, akeys)
    n1 = 6000
    mid = make_probe(rng, spec_a, n1, akeys, null_frac=0.0)
    bidx = rng.choice(domain(spec_b), n1, replace=False)
    bk = decode(spec_b, bidx)
    bpay = rng.integers(0, 10**9, n1).astype(np.int64)
    lb = D.Lookup(ctx, key_types=[t for t, _, _ in spec_b], key_ranges=[(lo, hi) for _, lo, hi in spec_b], payload_types=[D.INT64])
    p = D.Pipeline(ctx, [D.INT32, D.INT64, D.INT64, D.UINT16, D.INT64], stages=[(D.STAGE_SEMI, [0, 1], la)])
    try:
        p.sink_build(lb, key_cols=[2, 3], payload_cols=[4])
        p.push_host([D.HostColumn(mid[0][0]), D.HostColumn(mid[1][0]), D.HostColumn(bk[0]), D.HostColumn(bk[1], None, D.UINT16), D.HostColumn(bpay)])
        p.finish()
    finally:
        p.close()
    ma = ref_index(akeys)
    kept = [j for j in range(n1) if probe_tuple(mid, j) in ma]
    assert lb.metric("rows") == len(kept)
    n2 = 30_000
    q = rng.integers(0, n1, n2)
    q0, q1 = bk[0][q], bk[1][q]
    p = D.Pipeline(ctx, [D.INT64, D.UINT16], stages=[(D.STAGE_INNER, [0, 1], lb)])
    try:
        p.sink_output([2])
        p.push_host([D.HostColumn(q0), D.HostColumn(q1, None, D.UINT16)])
        p.finish()
        got = batches_to_cols(p.drain(host=True), 1)[0][0]
    finally:
        p.close(); la.close(); lb.close()
    ks = set(kept)
    assert got.tolist() == [int(bpay[q[j]]) for j in range(n2) if int(q[j]) in ks]


@pytest.mark.parametrize("sink", ["dense", "hash", "unordered"])
def test_other_sinks_over_a_composite_stage(ctx, sink):
    rng = np.random.default_rng(41 + len(sink))
    spec = SPECS[3]
    bkeys, pay = make_build(rng, spec, 3000)
    probe = make_probe(rng, spec, 40_000, bkeys)
    n = len(probe[0][0])
    g = rng.integers(0, 5, n).astype(np.int32)
    look = build_lookup(ctx, spec, bkeys, pay, n_acc=1)
    types = [t for t, _, _ in spec] + [D.INT32]
    p = D.Pipeline(ctx, types, stages=[(D.STAGE_INNER, [0, 1, 2], look)])
    try:
        if sink == "dense":
            p.sink_aggregate_dense([3], [(0, 4)], [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(4)])])
        elif sink == "hash":
            p.sink_aggregate_hash([1, 3], [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(4)])])
        else:
            p.sink_output([0, 1, 2, 4], ordered=False)
        for s, e in ((0, 1000), (1000, n)):
            p.push_host([D.HostColumn(v[s:e], None if val is None else val[s:e], t) for (t, _, _), (v, val) in zip(spec, probe)] + [D.HostColumn(g[s:e])])
        p.finish()
        got = batches_to_cols(p.drain(host=True), {"dense": 3, "hash": 4, "unordered": 4}[sink])
    finally:
        p.close(); look.close()
    m = ref_index(bkeys)
    rows = [(j, m[t]) for j in range(n) for t in [probe_tuple(probe, j)] if t is not None and t in m]
    js = np.array([j for j, _ in rows], np.int64)
    bi = np.array([i for _, i in rows], np.int64)
    if sink == "unordered":
        exp = [(probe[c][0][js], None) for c in range(3)] + [(pay[bi], None)]
    else:
        keys = [g[js]] if sink == "dense" else [probe[1][0][js], g[js]]
        acc = {}
        for r, kk in enumerate(zip(*[k.tolist() for k in keys])):
            c, s = acc.get(kk, (0, 0))
            acc[kk] = (c + 1, s + int(pay[bi[r]]))
        ks = sorted(acc)
        exp = [(np.array([kk[q] for kk in ks], keys[q].dtype), None) for q in range(len(keys))]
        exp += [(np.array([acc[kk][0] for kk in ks], np.int64), None), (np.array([acc[kk][1] for kk in ks], np.int64), None)]
    assert_cols_equal(got, exp, ordered=False, what=sink)


# ---------------------------------------------------------------------------------------------------------------------------------
# errors
# ---------------------------------------------------------------------------------------------------------------------------------
def test_errors(ctx):
    spec = [(D.INT32, 0, 9), (D.INT64, -5, 5)]
    types, rng_ = [D.INT32, D.INT64], [(0, 9), (-5, 5)]
    # an out-of-domain build value: the build pipeline's finish refuses it
    look = D.Lookup(ctx, key_types=types, key_ranges=rng_)
    p = D.Pipeline(ctx, types)
    p.sink_build(look, key_cols=[0, 1])
    p.push_host([D.HostColumn(np.array([1, 2, 10], np.int32)), D.HostColumn(np.array([0, 0, 0], np.int64))])
    with pytest.raises(D.DfgpuError) as e:
        p.finish()
    assert e.value.code == ERR_INVALID
    p.close(); look.close()
    look = build_lookup(ctx, spec, [(np.array([1, 2], np.int32), None), (np.array([0, 1], np.int64), None)])
    # set_stage_keys after a push
    p = D.Pipeline(ctx, types + [D.INT64], stages=[(D.STAGE_SEMI, 0, look)])
    p.sink_output([2])
    with pytest.raises(D.DfgpuError) as e:      # a composite stage without its keys
        p.push_host([D.HostColumn(np.array([1], np.int32)), D.HostColumn(np.array([0], np.int64)), D.HostColumn(np.array([0], np.int64))])
    assert e.value.code == ERR_STATE
    p.close()
    p = D.Pipeline(ctx, types + [D.INT64], stages=[(D.STAGE_SEMI, [0, 1], look)])
    p.sink_output([2])
    p.push_host([D.HostColumn(np.array([1], np.int32)), D.HostColumn(np.array([0], np.int64)), D.HostColumn(np.array([0], np.int64))])
    with pytest.raises(D.DfgpuError) as e:
        p.set_stage_keys(0, [0, 1])
    assert e.value.code == ERR_STATE
    p.close()
    # a type mismatch
    p = D.Pipeline(ctx, [D.INT32, D.INT32], stages=[(D.STAGE_SEMI, 0, look)])
    with pytest.raises(D.DfgpuError) as e:
        p.set_stage_keys(0, [0, 1])
    assert e.value.code == ERR_INVALID
    p.close()
    # 15 inputs + two packed keys exceed 16 columns
    look2 = build_lookup(ctx, spec, [(np.array([1], np.int32), None), (np.array([0], np.int64), None)])
    p = D.Pipeline(ctx, types + [D.INT64] * 13, stages=[(D.STAGE_SEMI, 0, look), (D.STAGE_SEMI, 0, look2)])
    p.set_stage_keys(0, [0, 1])
    with pytest.raises(D.DfgpuError) as e:
        p.set_stage_keys(1, [0, 1])
    assert e.value.code == ERR_UNSUPPORTED
    p.close(); look.close(); look2.close()
    # domains: D = 2^63 refused, 2^62 accepted; min > max; has_key_range
    with pytest.raises(D.DfgpuError) as e:
        D.Lookup(ctx, key_types=[D.INT64, D.INT64], key_ranges=[(0, (1 << 62) - 1), (0, 1)])
    assert e.value.code == ERR_UNSUPPORTED
    ok = D.Lookup(ctx, key_types=[D.INT64, D.INT64], key_ranges=[(0, (1 << 61) - 1), (0, 1)])
    assert ok.metric("key_domain") == 1 << 62
    ok.close()
    with pytest.raises(D.DfgpuError) as e:
        D.Lookup(ctx, key_types=[D.INT64, D.INT64], key_ranges=[(5, 4), (0, 1)])
    assert e.value.code == ERR_INVALID
    with pytest.raises(D.DfgpuError) as e:
        D.Lookup(ctx, key_types=[D.INT64, D.INT64], key_ranges=[(0, 4), (0, 1)], key_range=(0, 9))
    assert e.value.code == ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------------------------
# the paths only large inputs select: ring-fed phase A + partitioned aggregate, partitioned build insert
# ---------------------------------------------------------------------------------------------------------------------------------
def test_large_composite_aggregate_and_build_take_the_partitioned_paths(ctx):
    rng = np.random.default_rng(51)
    spec = [(D.INT64, 1, 2_000_000), (D.INT32, 1, 50)]
    nb, n = 2_000_000, 8_000_000
    idx = rng.choice(domain(spec), nb, replace=False).astype(np.int64)
    bk = decode(spec, idx)
    bpay = rng.integers(0, 1000, nb).astype(np.int64)
    # the build: 2 M records with payload, table size unknown -> > 40 MB, inserted one slot range at a time
    big = D.Lookup(ctx, key_types=[D.INT64, D.INT32], key_ranges=[(1, 2_000_000), (1, 50)], payload_types=[D.INT64])
    p = D.Pipeline(ctx, [D.INT64, D.INT32, D.INT64])
    try:
        p.sink_build(big, key_cols=[0, 1], payload_cols=[2])
        p.push_host([D.HostColumn(bk[0]), D.HostColumn(bk[1]), D.HostColumn(bpay)])
        p.finish()
        assert p.metric("partitioned_inserts") > 0 and big.metric("rows") == nb
    finally:
        p.close()
    # the aggregate: a 3-word record table of 2 M keys (> 40 MB) with a Bloom filter, SUM over an Int64 column without NULLs
    agg = D.Lookup(ctx, key_types=[D.INT64, D.INT32], key_ranges=[(1, 2_000_000), (1, 50)], n_acc_words=2, expected_rows=nb)
    p = D.Pipeline(ctx, [D.INT64, D.INT32])
    try:
        p.sink_build(agg, key_cols=[0, 1])
        p.push_host([D.HostColumn(bk[0]), D.HostColumn(bk[1])])
        p.finish()
    finally:
        p.close()
    assert agg.metric("table_bytes") > 40 << 20
    pick = rng.integers(0, nb, n)
    hit = rng.random(n) < 0.3
    q0 = np.where(hit, bk[0][pick], rng.integers(1, 2_000_001, n)).astype(np.int64)
    q1 = np.where(hit, bk[1][pick], rng.integers(1, 51, n)).astype(np.int32)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    sel = rng.integers(0, 10, n).astype(np.int32)   # 4 bytes: two 8-byte ring columns would not fit the aggregate sink's ring
    p = D.Pipeline(ctx, [D.INT64, D.INT32, D.INT64, D.INT32], [C(3), L(7, D.INT32), B(D.OP_LT)], [(D.STAGE_INNER, [0, 1], agg)])
    try:
        p.sink_aggregate([0, 1], [(D.AGG_SUM, [C(2)])])
        p.push_host([D.HostColumn(q0), D.HostColumn(q1), D.HostColumn(v), D.HostColumn(sel)])
        p.finish()
        assert p.metric("ring_launches") > 0 and p.metric("partitioned_launches") > 0
        got = batches_to_cols(p.drain(host=True), 3)
    finally:
        p.close(); agg.close()
    # exact reference: group by the packed tuple with numpy
    key = (q0 - 1) + (q1.astype(np.int64) - 1) * 2_000_000
    bset = np.zeros(domain(spec), bool)
    bset[idx] = True
    m = bset[key] & (sel < 7)
    u, inv = np.unique(key[m], return_inverse=True)
    s = np.bincount(inv, weights=None, minlength=len(u))
    sums = np.zeros(len(u), np.int64)
    np.add.at(sums, inv, v[m])
    exp = [((u % 2_000_000) + 1, None), ((u // 2_000_000 + 1).astype(np.int32), None), (sums, None)]
    assert len(s) == len(u)
    assert_cols_equal(got, exp, ordered=False, what="partitioned composite aggregate")
    # the build's payload, probed back through the partitioned-insert table
    p = D.Pipeline(ctx, [D.INT64, D.INT32], stages=[(D.STAGE_INNER, [0, 1], big)])
    try:
        p.sink_output([2])
        p.push_host([D.HostColumn(bk[0][:100_000]), D.HostColumn(bk[1][:100_000])])
        p.finish()
        got = batches_to_cols(p.drain(host=True), 1)[0][0]
    finally:
        p.close(); big.close()
    assert np.array_equal(got, bpay[:100_000])


# ---------------------------------------------------------------------------------------------------------------------------------
# the operator twin: a Q9-shaped plan fused and unfused
# ---------------------------------------------------------------------------------------------------------------------------------
def test_q9_shaped_plan_fused_equals_unfused():
    """lineitem x partsupp on (partkey, suppkey), profit SUM grouped by l_suppkey: the twin keeps this shape unfused (it measured slower,
    README), so the fused node its rules would build is built here by hand, over the same composite stage, and must give the same groups"""
    from datafusion_b200 import exec as X
    rng = np.random.default_rng(61)
    nps, nl = 8000, 60_000
    pk = np.repeat(np.arange(1, 2001, dtype=np.int64), 4)
    sk = ((pk * 7 + np.tile(np.arange(4), 2000) * 131) % 500 + 1).astype(np.int64)
    cost = rng.integers(100, 100_000, nps).astype(np.int64)
    partsupp = pa.record_batch([pa.array(pk), pa.array(sk), pa.array(cost)], names=["ps_partkey", "ps_suppkey", "ps_supplycost"])
    pick = rng.integers(0, nps, nl)
    lpk = np.where(rng.random(nl) < 0.9, pk[pick], rng.integers(1, 2001, nl)).astype(np.int64)
    lsk = np.where(rng.random(nl) < 0.9, sk[pick], rng.integers(1, 501, nl)).astype(np.int64)
    qty = rng.integers(1, 50, nl).astype(np.int64)
    price = rng.integers(1000, 10**6, nl).astype(np.int64)
    lineitem = pa.record_batch([pa.array(lpk), pa.array(lsk), pa.array(qty), pa.array(price)], names=["l_partkey", "l_suppkey", "l_quantity", "l_extendedprice"])
    join = X.GpuHashJoinExec(X.MemoryExec([partsupp]), X.MemoryExec([lineitem]), [("ps_partkey", "l_partkey"), ("ps_suppkey", "l_suppkey")], "Inner")
    amount = X.Column("l_extendedprice") - X.Column("ps_supplycost") * X.Column("l_quantity")
    proj = X.GpuProjectionExec([(X.Column("l_suppkey"), "l_suppkey"), (amount, "amount")], join)
    plan = X.GpuAggregateExec("Single", ["l_suppkey"], [X.AggregateExpr("sum", "amount", "profit")], proj)
    assert X.fuse_output_pipelines(plan) is plan
    sc = X._as_scan(join)
    assert sc.stages[0][1] == ["l_partkey", "l_suppkey"] and sc.stages[0][2].key == ["ps_partkey", "ps_suppkey"]
    fused = X.GpuPipelineExec(sc, sink="hash", group_by=["l_suppkey"], aggs=[("sum", amount, "profit")], out_schema=plan.schema, nullable=[False])

    def rows(p):
        t = pa.Table.from_batches(X.collect(p))
        return sorted(zip(t.column(0).to_pylist(), t.column(1).to_pylist()))
    got, exp = rows(fused), rows(plan)
    assert got == exp and len(got) > 0
