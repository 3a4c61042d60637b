"""The fused pipeline (dfgpu_lookup / dfgpu_pipeline) over every integer-like column type, at every position that reads or writes
one: probe keys of bitmap, hash and filtered-hash lookups under every stage kind, the build sink's key and packed payload fields, payload
fields read back as aggregate arguments, stage filters and group keys, the join-keyed aggregate sink, phase A's loads of 1-, 2-, 4- and
8-byte columns at 32-byte, 16-byte and element alignment (with and without the ring), the radix-partitioned aggregate and build, and
composite keys of narrow, unsigned and temporal components.  Values come from each type's edge pool (min, max, 0, 1, all ones, and
UInt64 values >= 2^63) and 200-value windows at both ends of its domain.

The references are plain Python / numpy and share no code with the kernels: joins match on the key's value as a Python int, payload
and output columns are gathered with numpy from the typed input arrays, integer SUMs are Python ints wrapped to the result width,
float SUM / AVG are checked within the math.fsum error bound and float MIN / MAX bit for bit (test_gpu_operator_types' group-by
reference)."""
import ctypes

import numpy as np
import pytest

from datafusion_b200 import capi as D
from test_gpu_operator_types import NAME, agg_reference, check_agg, drain, filler, npt, pool, splits, window

pytestmark = pytest.mark.gpu

KEY_TYPES = [D.INT8, D.INT16, D.INT32, D.INT64, D.UINT8, D.UINT16, D.UINT32, D.UINT64, D.DATE32, D.DATE64, D.TIMESTAMP]
KIDS = [NAME[t] for t in KEY_TYPES]
INTS = [D.INT8, D.INT16, D.INT32, D.INT64, D.UINT8, D.UINT16, D.UINT32, D.UINT64]
UNSIGNED = (D.UINT8, D.UINT16, D.UINT32, D.UINT64)
INVALID, UNSUPPORTED = -1, -3
NODE = lambda k, a=0, t=0, v=0: (k, a, t, 0, v, 0.0)                        # noqa: E731
COL = lambda i: NODE(D.EXPR_COLUMN, i)                                        # noqa: E731
CAST64 = NODE(D.EXPR_CAST, 0, D.INT64)


def i64(x):
    """a Python int as the int64 whose bits it has (UInt64 values >= 2^63 are negative)"""
    x = int(x) % (1 << 64)
    return x - (1 << 64) if x >= 1 << 63 else x


def lit(t, v):
    return NODE(D.EXPR_LITERAL, 0, t, i64(v))


def cmp(c, op, t, v):
    return [COL(c), lit(t, v), NODE(D.EXPR_BINARY, op)]


def conj(*terms):
    out = list(terms[0])
    for t in terms[1:]:
        out += t + [NODE(D.EXPR_BINARY, D.OP_AND)]
    return out


def dom(t):
    info = np.iinfo(npt(t))
    return int(info.min), int(info.max)


def all_ones(t):
    """the key whose 64-bit form is the hash table's empty slot: -1 of a signed type (sign-extended), UInt64::MAX"""
    return -1 if t not in UNSIGNED else (dom(t)[1] if t == D.UINT64 else None)


def key_values(t, reserved=False):
    """the distinct build keys of type t: its pool and both windows, without the reserved all-ones key unless asked"""
    vals = set(pool(t)) | set(window(t, False)) | set(window(t, True))
    if not reserved:
        vals.discard(all_ones(t))
    return sorted(vals)


def arr(vals, t):
    return np.array([int(v) for v in vals], dtype=npt(t)) if len(vals) else np.zeros(0, npt(t))


# ---- references (plain Python) ------------------------------------------------------------------------------------------------
def partners(bkeys, pkeys, pvalid=None):
    """probe row -> index of the build row with the same key value (unique build keys), -1 for none or a NULL probe key"""
    where = {int(k): i for i, k in enumerate(bkeys)}
    idx = np.array([where.get(int(k), -1) for k in pkeys], np.int64)
    if pvalid is not None:
        idx[~np.asarray(pvalid, bool)] = -1
    return idx


def kept_rows(kind, idx):
    """the probe rows a stage of `kind` passes on (a NULL key never matches: ANTI keeps it, RIGHT NULL-pads it)"""
    if kind in (D.STAGE_INNER, D.STAGE_SEMI):
        return np.nonzero(idx >= 0)[0]
    if kind == D.STAGE_ANTI:
        return np.nonzero(idx < 0)[0]
    return np.arange(len(idx))


def gather(vals, idx):
    """vals[idx] with validity idx >= 0 (the NULL-padded side of an outer join holds 0)"""
    vals = np.asarray(vals)
    ok = idx >= 0
    out = vals[np.where(ok, idx, 0)] if len(vals) else np.zeros(len(idx), vals.dtype)
    return np.where(ok, out, np.zeros((), out.dtype)), ok


def left_groups(bkeys, idx, probe_vals, anti=False):
    """LEFT: {build key: (COUNT(*), SUM(v) or None)} with the NULL-padded row of an unmatched build row; LEFT_ANTI: the build keys
    no probe row matched"""
    cnt = np.bincount(idx[idx >= 0], minlength=len(bkeys))
    if anti:
        return sorted(int(k) for k, c in zip(bkeys, cnt) if c == 0)
    sums = [0] * len(bkeys)
    for i, v in zip(idx, probe_vals):
        if i >= 0:
            sums[i] += int(v)
    return sorted((int(k), int(c) if c else 1, i64(s) if c else None) for k, c, s in zip(bkeys, cnt, sums))


# ---- device columns --------------------------------------------------------------------------------------------------------------
def aligned_col(ctx, v, t, shift, keep):
    """column values placed `shift` bytes past a 32-byte boundary of a device allocation (vec = 2 / 1 / 0 in pipeline.cu's ColRef)"""
    v = np.ascontiguousarray(v)
    buf = D.DeviceBuffer(ctx, v.nbytes + 64)
    base = (buf.ptr + 31) & ~31
    assert base % 32 == 0
    if v.nbytes:
        ctx.check(ctx.lib.dfgpu_memcpy_h2d(ctx.h, ctypes.c_void_p(base + shift), v.ctypes.data_as(ctypes.c_void_p), v.nbytes))
    ctx.sync()
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count = t, 0, len(v), 0, 0
    c.values, c.validity = base + shift, None
    keep.append(buf)
    return c


def host(v, t, ok=None):
    return D.HostColumn(np.asarray(v, npt(t)), None if ok is None or ok.all() else ok, t)


def build_lookup(ctx, t, keys, pays=(), parts_pushes=2, **kw):
    """a lookup of key type t built by a pipeline's build sink; pays = [(type, values)]"""
    look = D.Lookup(ctx, t, [pt for pt, _ in pays], **kw)
    b = D.Pipeline(ctx, [t] + [pt for pt, _ in pays])
    try:
        b.sink_build(look, 0, list(range(1, len(pays) + 1)))
        for s, e in splits(len(keys), parts_pushes):
            b.push_host([host(keys[s:e], t)] + [host(v[s:e], pt) for pt, v in pays])
        b.finish()
        metrics = {m: b.metric(m) for m in ("sink_rows", "partitioned_inserts")}
    finally:
        b.close()
    return look, metrics


def output_rows(ctx, types, cols, stages, out, pred=None, ordered=True, stage_filter=None):
    """runs an output-sink pipeline over host pushes; -> [(values, valid)] per output column"""
    p = D.Pipeline(ctx, types, pred, stages)
    try:
        if stage_filter is not None:
            p.set_stage_filter(*stage_filter)
        p.sink_output(out, ordered=ordered)
        n = len(cols[0][0])
        for s, e in splits(n, 3):
            p.push_host([host(v[s:e], t, None if ok is None else ok[s:e]) for (v, ok), t in zip(cols, types)])
        p.finish()
        got, _ = drain(p)
    finally:
        p.close()
    return got


def assert_cols(got, exp, ordered, what):
    """exp: [(values, valid or None)]; unordered results are sorted by their first column (a unique row id)"""
    n = len(exp[0][0])
    if got is None:
        assert n == 0, f"{what}: no output, expected {n} rows"
        return
    assert len(got[0][0]) == n, f"{what}: {len(got[0][0])} rows, expected {n}"
    go = np.arange(n) if ordered else np.argsort(got[0][0], kind="stable")
    eo = np.arange(n) if ordered else np.argsort(exp[0][0], kind="stable")
    for c, ((gv, gm), (ev, em)) in enumerate(zip(got, exp)):
        gv, gm, ev = np.asarray(gv)[go], np.asarray(gm)[go], np.asarray(ev)[eo]
        em = np.ones(n, bool) if em is None else np.asarray(em, bool)[eo]
        assert np.array_equal(gm, em), f"{what}: column {c} validity differs at {np.nonzero(gm != em)[0][:5]}"
        bad = np.nonzero([int(a) != int(b) for a, b in zip(gv[em], ev[em])])[0]
        assert not len(bad), f"{what}: column {c} differs at {len(bad)} rows, first {int(gv[em][bad[0]])} != {int(ev[em][bad[0]])}"


def probe_keys(rng, t, n, extra=()):
    """n probe keys of type t drawn from the pool, both windows and `extra`, 8 % NULL"""
    cand = sorted(set(pool(t)) | set(window(t, False)) | set(window(t, True)) | {int(x) for x in extra})
    v = arr(cand, t)[rng.integers(0, len(cand), n)]
    v[:len(cand)] = arr(cand, t)
    return v, rng.random(n) >= 0.08


# ---- 1. probe keys under every lookup mode and stage kind --------------------------------------------------------------------------
def bitmap_ranges(t):
    lo, hi = dom(t)
    return [(lo, min(hi, lo + 1000)), (max(lo, hi - 1000), hi)]


@pytest.mark.parametrize("t", KEY_TYPES, ids=KIDS)
def test_probe_key_of_a_bitmap_lookup_at_both_ends_of_the_domain(gpu_ctx, t):
    """SEMI / ANTI / INNER stages over a bitmap lookup whose range sits at the bottom and at the top of the key's domain; probes with
    keys inside, just outside and far outside the range (kmin + 2^32 + j), and NULLs"""
    rng = np.random.default_rng(10 + t)
    lo, hi = dom(t)
    for rlo, rhi in bitmap_ranges(t):
        span = np.arange(rhi - rlo + 1, dtype=object) + rlo
        bk = sorted({rlo, rhi} | {int(x) for x in span[rng.random(len(span)) < 0.5]})
        extra = [x for x in (rlo - 1, rhi + 1, rlo + (1 << 32), rlo + (1 << 32) + 1, rhi - (1 << 32)) if lo <= x <= hi]
        extra += [x for x in bk[:4]]
        look, _ = build_lookup(gpu_ctx, t, arr(bk, t), key_range=(i64(rlo), i64(rhi)))
        try:
            assert look.metric("mode") == 1 and look.metric("rows") == len(bk)
            n = 20_011
            pk, pv = probe_keys(rng, t, n, extra)
            rid = np.arange(n, dtype=np.int64) * 3 + 1
            idx = partners(bk, pk, pv)
            assert (idx >= 0).sum() > 100 and (idx < 0).sum() > 100
            for kind in (D.STAGE_SEMI, D.STAGE_ANTI, D.STAGE_INNER):
                for ordered in (True, False):   # the ordered sink's output kernel, the unordered sink's pipeline kernel (phase A)
                    got = output_rows(gpu_ctx, [t, D.INT64], [(pk, pv), (rid, None)], [(kind, 0, look)], [1, 0], ordered=ordered)
                    keep = kept_rows(kind, idx)
                    assert_cols(got, [(rid[keep], None), (pk[keep], pv[keep])], ordered,
                                f"{NAME[t]} bitmap [{rlo}, {rhi}] stage {kind} ordered={ordered}")
        finally:
            look.close()


def hash_case(rng, t, n=24_007):
    """unique build keys of type t (no all-ones key) with an Int32 payload; probe keys with misses and NULLs"""
    bk = [k for k in key_values(t) if rng.random() < 0.75]
    pay = rng.integers(-2**31, 2**31, len(bk)).astype(np.int32)
    pk, pv = probe_keys(rng, t, n, [x for x in (all_ones(t),) if x is not None])
    return arr(bk, t), pay, pk, pv, np.arange(n, dtype=np.int64) * 5 - 7


@pytest.mark.parametrize("filt", [0, 1], ids=["table", "membership_filter"])
@pytest.mark.parametrize("t", KEY_TYPES, ids=KIDS)
def test_probe_key_of_a_hash_lookup_under_every_stage_kind(gpu_ctx, t, filt):
    """INNER, SEMI, ANTI and RIGHT stages through the output sink, LEFT and LEFT_ANTI through the join-keyed aggregate sink, over a
    hash lookup with and without its membership filter"""
    rng = np.random.default_rng(100 + 2 * t + filt)
    bk, pay, pk, pv, rid = hash_case(rng, t)
    look, _ = build_lookup(gpu_ctx, t, bk, [(D.INT32, pay)], membership_filter=filt)
    try:
        assert look.metric("mode") == 0 and look.metric("rows") == len(bk)
        assert (look.metric("filter_bytes") > 0) == bool(filt)
        idx = partners(bk, pk, pv)
        assert (idx >= 0).sum() > 1000 and (idx < 0).sum() > 1000
        for kind in (D.STAGE_INNER, D.STAGE_SEMI, D.STAGE_ANTI, D.STAGE_RIGHT):
            out = [1, 0, 2] if kind in (D.STAGE_INNER, D.STAGE_RIGHT) else [1, 0]
            for ordered in (True, False):
                got = output_rows(gpu_ctx, [t, D.INT64], [(pk, pv), (rid, None)], [(kind, 0, look)], out, ordered=ordered)
                keep = kept_rows(kind, idx)
                exp = [(rid[keep], None), (pk[keep], pv[keep])]
                if len(out) == 3:
                    pv_, pok = gather(pay, idx[keep])
                    exp.append((pv_, pok if kind == D.STAGE_RIGHT else None))
                assert_cols(got, exp, ordered, f"{NAME[t]} hash filt={filt} stage {kind} ordered={ordered}")
    finally:
        look.close()
    # LEFT / LEFT_ANTI: the lookup holds an accumulator record per build row
    for kind in (D.STAGE_LEFT, D.STAGE_LEFT_ANTI):
        look, _ = build_lookup(gpu_ctx, t, bk, [(D.INT32, pay)], membership_filter=filt, n_acc_words=2)
        try:
            p = D.Pipeline(gpu_ctx, [t, D.INT64], None, [(kind, 0, look)])
            try:
                aggs = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [COL(1)])] if kind == D.STAGE_LEFT else []
                p.sink_aggregate([0], aggs)
                for s, e in splits(len(pk), 3):
                    p.push_host([host(pk[s:e], t, pv[s:e]), host(rid[s:e], D.INT64)])
                p.finish()
                got, _ = drain(p)
            finally:
                p.close()
        finally:
            look.close()
        exp = left_groups(bk, idx, rid, anti=kind == D.STAGE_LEFT_ANTI)
        if kind == D.STAGE_LEFT_ANTI:
            rows = sorted(int(x) for x in got[0][0]) if got else []
        else:
            rows = sorted((int(k), int(c), int(s) if ok else None) for k, (c, s, ok) in
                          zip(got[0][0], zip(got[1][0], got[2][0], got[2][1])))
        assert rows == exp, f"{NAME[t]} filt={filt} stage {kind}"


# ---- 2 / 6. the build sink: key and packed payload fields of mixed widths -------------------------------------------------------
PAYLOADS = {
    "i8-i16-i32-i8": [D.INT8, D.INT16, D.INT32, D.INT8],                 # shifts 0 / 8 / 24 / 56: 64 bits
    "u8x8": [D.UINT8] * 8,
    "u16-date32-i16": [D.UINT16, D.DATE32, D.INT16],                     # 16 / 32 / 16
    "u32-i8-u16-u8": [D.UINT32, D.INT8, D.UINT16, D.UINT8],
}


def build_and_probe(ctx, rng, t, pname, n_probe=30_011):
    """a build sink of key type t with payload PAYLOADS[pname] (values over each field's whole domain), read back through an INNER
    stage whose output sink emits every payload field; -> build metrics"""
    ptypes = PAYLOADS[pname]
    bk = arr([k for k in key_values(t) if rng.random() < 0.8], t)
    pays = [(pt, filler(rng, pt, len(bk))[0]) for pt in ptypes]
    look, metrics = build_lookup(ctx, t, bk, pays)
    try:
        assert look.metric("rows") == len(bk)
        pk, pv = probe_keys(rng, t, n_probe)
        rid = np.arange(n_probe, dtype=np.int64)
        nin = 2
        out = [1, 0] + [nin + j for j in range(len(ptypes))]
        got = output_rows(ctx, [t, D.INT64], [(pk, pv), (rid, None)], [(D.STAGE_INNER, 0, look)], out)
    finally:
        look.close()
    idx = partners(bk, pk, pv)
    keep = kept_rows(D.STAGE_INNER, idx)
    exp = [(rid[keep], None), (pk[keep], None)] + [(gather(v, idx[keep])[0], None) for _, v in pays]
    assert len(keep) > 1000
    assert_cols(got, exp, True, f"{NAME[t]} payload {pname}")
    return metrics


@pytest.mark.parametrize("pname", sorted(PAYLOADS))
@pytest.mark.parametrize("t", KEY_TYPES, ids=KIDS)
def test_build_sink_key_and_packed_payload_fields(gpu_ctx, t, pname):
    rng = np.random.default_rng(300 + 7 * t + len(pname))
    build_and_probe(gpu_ctx, rng, t, pname)


@pytest.fixture
def parts_hook(monkeypatch):
    """sets DFGPU_PIPE_RADIX_PARTS for the test (None: unset); the hook is removed again when the test ends"""
    def set_parts(parts):
        if parts:
            monkeypatch.setenv("DFGPU_PIPE_RADIX_PARTS", str(parts))
        else:
            monkeypatch.delenv("DFGPU_PIPE_RADIX_PARTS", raising=False)
    set_parts(None)
    yield set_parts
    set_parts(None)


PART_TYPES = [D.INT8, D.UINT8, D.INT16, D.UINT16, D.UINT32, D.UINT64, D.DATE32, D.DATE64, D.TIMESTAMP]


@pytest.mark.parametrize("t", PART_TYPES, ids=[NAME[t] for t in PART_TYPES])
def test_partitioned_build_of_narrow_unsigned_and_temporal_keys(gpu_ctx, parts_hook, t):
    """the build sink's radix-partitioned insert, forced on a small table: its records carry sign-extended keys"""
    parts_hook(8)
    metrics = build_and_probe(gpu_ctx, np.random.default_rng(400 + t), t, "i8-i16-i32-i8")
    assert metrics["partitioned_inserts"] > 0


@pytest.mark.parametrize("t", PART_TYPES, ids=[NAME[t] for t in PART_TYPES])
def test_partitioned_aggregate_on_narrow_unsigned_and_temporal_keys(gpu_ctx, parts_hook, t):
    """the join-keyed sink's radix-partitioned probe (ring-fed pass 1 through the folded membership filter, then records by slot
    range), forced on a small table: SUM(v) grouped on the key and two payload fields"""
    parts_hook(4)
    rng = np.random.default_rng(500 + t)
    bk = arr([k for k in key_values(t) if rng.random() < 0.8], t)
    p8, p16 = filler(rng, D.INT8, len(bk))[0], filler(rng, D.UINT16, len(bk))[0]
    n = 60_013
    cand = sorted(set(key_values(t, reserved=True)))
    pk = arr(cand, t)[rng.integers(0, len(cand), n)]
    v = rng.integers(-2**62, 2**62, n).astype(np.int64)
    look, _ = build_lookup(gpu_ctx, t, bk, [(D.INT8, p8), (D.UINT16, p16)], membership_filter=1, n_acc_words=2)
    try:
        p = D.Pipeline(gpu_ctx, [t, D.INT64], None, [(D.STAGE_INNER, 0, look)])
        try:
            p.sink_aggregate([0, 2, 3], [(D.AGG_SUM, [COL(1)])])
            for s, e in splits(n, 2):
                p.push_host([host(pk[s:e], t), host(v[s:e], D.INT64)])
            p.finish()
            assert p.metric("partitioned_launches") > 0
            got, _ = drain(p)
        finally:
            p.close()
    finally:
        look.close()
    idx = partners(bk, pk)
    sums = {}
    for i, x in zip(idx, v):
        if i >= 0:
            sums[i] = sums.get(i, 0) + int(x)
    exp = sorted((int(bk[i]), int(p8[i]), int(p16[i]), i64(s)) for i, s in sums.items())
    rows = sorted(zip(*[[int(x) for x in c[0]] for c in got]))
    assert rows == exp and len(exp) > 50


# ---- 3. payload fields as aggregate arguments, stage filters and group keys ----------------------------------------------------
PAY3 = [D.UINT8, D.INT8, D.INT16, D.UINT16, D.INT8]   # shifts 0, 8, 16, 32, 48: virtual columns 3..7 behind (key, x Int16, rowid)


@pytest.mark.parametrize("sink", ["dense", "hash"])
@pytest.mark.parametrize("filtered", [False, True], ids=["all", "stage_filter"])
def test_payload_fields_as_arguments_filters_and_group_keys(gpu_ctx, sink, filtered):
    """SUM(CAST(p_i8) * CAST(x_i16)), MIN(p_i16), MAX(p_u16), COUNT(*) grouped on narrow payload fields (dense: p_i8 at shift 48 in
    [-100, 100]; hash: (p_i8, p_u8)); with a stage filter p_i8 < -1 on the INNER stage"""
    rng = np.random.default_rng(600 + 2 * filtered + (sink == "hash"))
    nb, n = 5000, 80_021
    bk = rng.permutation(1 << 20)[:nb].astype(np.int64) * 977 - (1 << 40)
    pays = [filler(rng, pt, nb)[0] for pt in PAY3]
    pays[4] = rng.integers(-100, 101, nb).astype(np.int8)
    pk = np.where(rng.random(n) < 0.7, bk[rng.integers(0, nb, n)], rng.integers(0, 1 << 40, n) * 2 + 1).astype(np.int64)
    x = filler(rng, D.INT16, n)[0]
    rid = np.arange(n, dtype=np.int64)
    look, _ = build_lookup(gpu_ctx, D.INT64, bk, list(zip(PAY3, pays)))
    aggs = [(D.AGG_SUM, [COL(4), CAST64, COL(1), CAST64, NODE(D.EXPR_BINARY, D.OP_MULTIPLY)]), (D.AGG_MIN, [COL(5)]), (D.AGG_MAX, [COL(6)]),
            (D.AGG_COUNT_STAR, None)]
    group = [7] if sink == "dense" else [4, 3]
    try:
        p = D.Pipeline(gpu_ctx, [D.INT64, D.INT16, D.INT64], None, [(D.STAGE_INNER, 0, look)])
        try:
            if filtered:
                p.set_stage_filter(0, cmp(4, D.OP_LT, D.INT8, -1))
            if sink == "dense":
                p.sink_aggregate_dense(group, [(-100, 100)], aggs)
            else:
                p.sink_aggregate_hash(group, aggs)
            for s, e in splits(n, 3):
                p.push_host([host(pk[s:e], D.INT64), host(x[s:e], D.INT16), host(rid[s:e], D.INT64)])
            p.finish()
            out, otypes = drain(p)
        finally:
            p.close()
    finally:
        look.close()
    idx = partners(bk, pk)
    keep = idx >= 0
    if filtered:
        keep &= pays[1][np.maximum(idx, 0)] < -1
    j = idx[keep]
    prod = (pays[1][j].astype(np.int64) * x[keep].astype(np.int64)).astype(np.int64)
    cols = [(pays[4][j], None), (pays[1][j], None), (pays[0][j], None), (prod, None), (pays[2][j], None), (pays[3][j], None)]
    types = [D.INT8, D.INT8, D.UINT8, D.INT64, D.INT16, D.UINT16]
    gcols = [0] if sink == "dense" else [1, 2]
    ref_aggs = [(D.AGG_SUM, 3, -1), (D.AGG_MIN, 4, -1), (D.AGG_MAX, 5, -1), (D.AGG_COUNT_STAR, -1, -1)]
    ref = agg_reference(cols, types, gcols, ref_aggs)
    assert len(ref) > 20 and keep.sum() > 1000
    check_agg(out, otypes, ref, types, gcols, ref_aggs, f"{sink} filtered={filtered}")


# ---- 4. the join-keyed aggregate sink -------------------------------------------------------------------------------------------
def arg_col(rng, t, n):
    if t == D.FLOAT32:
        return rng.integers(-2**20, 2**20, n).astype(np.float32) * np.float32(0.25)
    if t == D.FLOAT64:
        return rng.standard_normal(n) * 1e6
    return filler(rng, t, n)[0]


# the sink takes at most four aggregates: each set runs on a lookup of its own (the accumulators are words of its records);
# (func, input column) with input columns 1, 2 = the integer arguments, 3 = Float32, 4 = Float64
AGG_SETS = [[(D.AGG_COUNT_STAR, -1), (D.AGG_SUM, 1), (D.AGG_MIN, 1), (D.AGG_MAX, 1)],
            [(D.AGG_SUM, 2), (D.AGG_MIN, 2), (D.AGG_MAX, 2), (D.AGG_SUM, 3)],
            [(D.AGG_AVG, 4), (D.AGG_COUNT_STAR, -1)]]


@pytest.mark.parametrize("mode", [D.AGG_SINGLE, D.AGG_PARTIAL], ids=["Single", "Partial+Final"])
@pytest.mark.parametrize("t", KEY_TYPES, ids=KIDS)
def test_join_keyed_sink_over_every_key_and_argument_type(gpu_ctx, t, mode):
    """GROUP BY (probe key of type t, Int8 payload field with negatives): COUNT(*), SUM / MIN / MAX over two integer arguments (each
    integer type appears across the key types, UInt64 values above 2^63 and Int8 negatives among them), SUM over Float32, AVG over
    Float64; Partial states finished by dfgpu_agg's Final"""
    i = KEY_TYPES.index(t)
    a1, a2 = INTS[i % 8], INTS[(i + 4) % 8]
    rng = np.random.default_rng(700 + 2 * t + (mode == D.AGG_PARTIAL))
    bk = arr([k for k in key_values(t) if rng.random() < 0.8], t)
    pay = filler(rng, D.INT8, len(bk))[0]
    n = 40_009
    pk, pv = probe_keys(rng, t, n)
    args = [arg_col(rng, a, n) for a in (a1, a2, D.FLOAT32, D.FLOAT64)]
    in_types = [t, a1, a2, D.FLOAT32, D.FLOAT64]
    idx = partners(bk, pk, pv)
    keep = idx >= 0
    # reference columns: 0 key, 1 payload, then input column c at c + 1
    cols = [(pk[keep], None), (pay[idx[keep]], None)] + [(v[keep], None) for v in args]
    types = [t, D.INT8] + in_types[1:]
    for k, aset in enumerate(AGG_SETS):
        aggs = [(f, None if c < 0 else [COL(c)]) for f, c in aset]
        ref_aggs = [(f, -1 if c < 0 else c + 1, -1) for f, c in aset]
        look, _ = build_lookup(gpu_ctx, t, bk, [(D.INT8, pay)], n_acc_words=5)
        try:
            p = D.Pipeline(gpu_ctx, in_types, None, [(D.STAGE_INNER, 0, look)])
            try:
                p.sink_aggregate([0, 5], aggs, mode)
                for s, e in splits(n, 3):
                    p.push_host([host(pk[s:e], t, pv[s:e])] + [host(v[s:e], at) for v, at in zip(args, in_types[1:])])
                p.finish()
                out, otypes = drain(p)
            finally:
                p.close()
        finally:
            look.close()
        ref = agg_reference(cols, types, [0, 1], ref_aggs)
        assert len(ref) > 100
        what = f"{NAME[t]} set {k} args {NAME[a1]} / {NAME[a2]}"
        if mode == D.AGG_SINGLE:
            check_agg(out, otypes, ref, types, [0, 1], ref_aggs, what)
            continue
        h = D.AggHandle(gpu_ctx, otypes, [0, 1], [(f, -1, -1) for f, _, _ in ref_aggs], D.AGG_FINAL, 8192)
        try:
            for s, e in splits(len(out[0][0]), 2):
                h.push_host([host(v[s:e], ot, ok[s:e]) for (v, ok), ot in zip(out, otypes)])
            h.finish()
            fout, ftypes = drain(h)
        finally:
            h.close()
        check_agg(fout, ftypes, ref, types, [0, 1], ref_aggs, what + " partial+final")


# ---- 5. phase A's loads at every alignment ----------------------------------------------------------------------------------------
def phase_a_pred(t):
    """c > min AND c < max AND c >= m AND c != 1: the type's ends and both sides of 0 (of 2^63 for UInt64, of half the domain for the
    other unsigned types)"""
    lo, hi = dom(t)
    m = -1 if t not in UNSIGNED else (hi + 1) // 2
    return conj(cmp(0, D.OP_GT, t, lo), cmp(0, D.OP_LT, t, hi), cmp(0, D.OP_GTEQ, t, m), cmp(0, D.OP_NEQ, t, 1)), \
        lambda v: [(lo < int(x) < hi) and int(x) >= m and int(x) != 1 for x in v]


@pytest.mark.parametrize("shift", ["aligned32", "aligned16", "one_element"])
@pytest.mark.parametrize("t", KEY_TYPES, ids=KIDS)
def test_phase_a_loads_of_every_width_and_alignment(gpu_ctx, t, shift):
    """device columns starting 0, 16 bytes and one element past a 32-byte boundary; a conjunction over the column of type t and a
    bitmap SEMI stage: through the join-keyed sink (the ring-fed kernel when aligned; ring_load8) and the output sink (load8's
    whole-sector, 16-byte and scalar paths); full 256-row tiles and a ragged tail"""
    w = D.WIDTH[t]
    rng = np.random.default_rng(800 + 3 * t + len(shift))
    n = 250_007 if shift == "aligned32" else 37_131
    cand = sorted(set(pool(t)) | set(window(t, False)) | set(window(t, True)))
    c = arr(cand, t)[rng.integers(0, len(cand), n)]
    c[:len(cand)] = arr(cand, t)
    key = rng.integers(0, 8192, n).astype(np.int32)      # 4 bytes: an 8-byte column and this key still fit two ring tiles per warp
    bits = rng.permutation(4096)[:2500].astype(np.int32)
    rid = np.arange(n, dtype=np.int64)
    bitmap, _ = build_lookup(gpu_ctx, D.INT32, bits, key_range=(0, 4095))
    rows, _ = build_lookup(gpu_ctx, D.INT64, rid, n_acc_words=2, expected_rows=n)
    pred, ref_pred = phase_a_pred(t)
    keep_mask = np.array(ref_pred(c)) & np.isin(key, bits)
    keep = np.nonzero(keep_mask)[0]
    assert 0 < len(keep) < n
    keepers = []

    def cols(byte_shift):
        return [aligned_col(gpu_ctx, c, t, byte_shift(w), keepers), aligned_col(gpu_ctx, key, D.INT32, byte_shift(4), keepers),
                aligned_col(gpu_ctx, rid, D.INT64, byte_shift(8), keepers)]
    byte_shift = {"aligned32": lambda width: 0, "aligned16": lambda width: 16, "one_element": lambda width: width}[shift]
    types = [t, D.INT32, D.INT64]
    try:
        # join-keyed sink grouped on the row id (INNER over a lookup of every row id): exactly the surviving rows
        p = D.Pipeline(gpu_ctx, types, pred, [(D.STAGE_SEMI, 1, bitmap), (D.STAGE_INNER, 2, rows)])
        try:
            p.sink_aggregate([2], [(D.AGG_COUNT_STAR, None)])
            p.push_device(cols(byte_shift))
            p.finish()
            ring = p.metric("ring_launches")
            got, _ = drain(p)
        finally:
            p.close()
        assert (ring > 0) == (shift != "one_element"), (shift, ring)
        order = np.argsort(got[0][0], kind="stable")
        assert np.array_equal(got[0][0][order], rid[keep]) and (got[1][0] == 1).all(), f"{NAME[t]} {shift}: surviving rows"
        # output sink: load8 without the ring
        p = D.Pipeline(gpu_ctx, types, pred, [(D.STAGE_SEMI, 1, bitmap)])
        try:
            p.sink_output([2, 0])
            p.push_device(cols(byte_shift))
            p.finish()
            got, _ = drain(p)
        finally:
            p.close()
        assert_cols(got, [(rid[keep], None), (c[keep], None)], True, f"{NAME[t]} {shift} output sink")
    finally:
        bitmap.close()
        rows.close()


# ---- 7. composite keys ------------------------------------------------------------------------------------------------------------
COMPOSITES = {
    "i8-u32": ([D.INT8, D.UINT32], [(-128, -80), ((1 << 32) - 60, (1 << 32) - 1)]),
    "date64-ts": ([D.DATE64, D.TIMESTAMP], [(-10**12 - 40, -10**12 + 9), (-(1 << 63), -(1 << 63) + 45)]),
    "ts-i8-u32": ([D.TIMESTAMP, D.INT8, D.UINT32], [((1 << 63) - 20, (1 << 63) - 1), (-5, 4), (0, 30)]),
}


@pytest.mark.parametrize("name", sorted(COMPOSITES))
def test_composite_keys_of_narrow_unsigned_and_temporal_components(gpu_ctx, name):
    """build sink and INNER / ANTI probe stages on 2..3 key columns with negative and edge domains; probe components just outside
    their domains and NULL match nothing"""
    types, ranges = COMPOSITES[name]
    rng = np.random.default_rng(900 + len(name))
    spans = [hi - lo + 1 for lo, hi in ranges]
    total = int(np.prod(spans))
    tup = rng.permutation(total)[: total // 2]
    comps, rest = [], tup
    for (lo, _), r in zip(ranges, spans):
        comps.append(rest % r + lo)
        rest = rest // r
    bcols = [arr(list(v), t) for v, t in zip(comps, types)]
    pay = rng.integers(-2**62, 2**62, len(tup)).astype(np.int64)
    look = D.Lookup(gpu_ctx, payload_types=[D.INT64], key_types=types, key_ranges=[(i64(lo), i64(hi)) for lo, hi in ranges])
    nk = len(types)
    try:
        b = D.Pipeline(gpu_ctx, types + [D.INT64])
        try:
            b.sink_build(look, payload_cols=[nk], key_cols=list(range(nk)))
            b.push_host([host(v, t) for v, t in zip(bcols, types)] + [host(pay, D.INT64)])
            b.finish()
        finally:
            b.close()
        n = 30_007
        pick = rng.integers(0, len(tup), n)
        pcols, pvalid = [], []
        for (lo, hi), t, v in zip(ranges, types, bcols):
            dlo, dhi = dom(t)
            near = [x for x in (lo - 1, lo, hi, hi + 1) if dlo <= x <= dhi]
            alt = arr(near, t)[rng.integers(0, len(near), n)]
            pcols.append(np.where(rng.random(n) < 0.85, v[pick], alt).astype(npt(t)))
            pvalid.append(rng.random(n) >= 0.04)
        rid = np.arange(n, dtype=np.int64)
        where = {tuple(int(v[i]) for v in bcols): i for i in range(len(tup))}
        idx = np.array([where.get(tuple(int(v[r]) for v in pcols), -1) if all(ok[r] for ok in pvalid) else -1 for r in range(n)], np.int64)
        assert (idx >= 0).sum() > 1000 and (idx < 0).sum() > 1000
        for kind in (D.STAGE_INNER, D.STAGE_ANTI):
            out = [nk] + list(range(nk)) + ([nk + 1] if kind == D.STAGE_INNER else [])
            got = output_rows(gpu_ctx, types + [D.INT64], [(v, ok) for v, ok in zip(pcols, pvalid)] + [(rid, None)],
                              [(kind, list(range(nk)), look)], out)
            keep = kept_rows(kind, idx)
            exp = [(rid[keep], None)] + [(v[keep], ok[keep]) for v, ok in zip(pcols, pvalid)]
            if kind == D.STAGE_INNER:
                exp.append((pay[idx[keep]], None))
            assert_cols(got, exp, True, f"{name} stage {kind}")
    finally:
        look.close()


# ---- 8. contract pins: the reserved all-ones key, refused types ----------------------------------------------------------------
def err_code(fn):
    with pytest.raises(D.DfgpuError) as e:
        fn()
    return e.value.code


@pytest.mark.parametrize("t", KEY_TYPES, ids=KIDS)
def test_all_ones_key_in_hash_and_bitmap_lookups(gpu_ctx, t):
    """a hash lookup refuses the key whose 64-bit form is all ones (-1 of a signed width, sign-extended; UInt64::MAX) with
    DFGPU_ERR_INVALID and takes the narrower unsigned all-ones values; a bitmap lookup holds every one of them.  Probing a hash lookup
    with the reserved key matches nothing: INNER / SEMI drop it, ANTI keeps it, RIGHT NULL-pads it"""
    lo, hi = dom(t)
    ones = -1 if t not in UNSIGNED else hi
    reserved = all_ones(t) is not None
    keys = arr(sorted({0, 1, ones, lo, hi - 1}), t)
    for pays in ([], [(D.INT32, np.arange(len(keys), dtype=np.int32))]):
        if reserved:
            assert err_code(lambda: build_lookup(gpu_ctx, t, keys, pays, parts_pushes=1)) == INVALID, (NAME[t], len(pays))
        else:
            look, _ = build_lookup(gpu_ctx, t, keys, pays, parts_pushes=1)
            assert look.metric("rows") == len(set(int(k) for k in keys))
            look.close()
    # a bitmap around the all-ones value holds and matches it
    rlo, rhi = (ones - 10, ones + 10) if t not in UNSIGNED else (hi - 20, hi)
    rlo, rhi = max(rlo, lo), min(rhi, hi)
    bk = arr(sorted({ones, rlo, rhi}), t)
    look, _ = build_lookup(gpu_ctx, t, bk, key_range=(i64(rlo), i64(rhi)))
    try:
        assert look.metric("mode") == 1 and look.metric("rows") == len(bk)
        pk = arr([ones, ones + 1 if ones < hi else ones - 1, ones, rlo, rhi], t)
        rid = np.arange(len(pk), dtype=np.int64)
        got = output_rows(gpu_ctx, [t, D.INT64], [(pk, None), (rid, None)], [(D.STAGE_SEMI, 0, look)], [1])
        keep = np.nonzero(np.isin(pk, bk))[0]
        assert_cols(got, [(rid[keep], None)], True, f"{NAME[t]} bitmap with all ones")
    finally:
        look.close()
    # probing a hash lookup (no reserved key inside) with the reserved key
    if not reserved:
        return
    top = hi - 1 if t == D.UINT64 else hi
    bk = arr(sorted({0, 1, lo, top}), t)
    bpay = np.arange(len(bk), dtype=np.int32) + 5
    look, _ = build_lookup(gpu_ctx, t, bk, [(D.INT32, bpay)])
    try:
        pk = arr([ones, 0, ones, top, ones], t)
        rid = np.arange(len(pk), dtype=np.int64)
        idx = partners(bk, pk)
        assert list(idx < 0) == [True, False, True, False, True]
        for kind in (D.STAGE_INNER, D.STAGE_SEMI, D.STAGE_ANTI, D.STAGE_RIGHT):
            out = [1, 2] if kind in (D.STAGE_INNER, D.STAGE_RIGHT) else [1]
            got = output_rows(gpu_ctx, [t, D.INT64], [(pk, None), (rid, None)], [(kind, 0, look)], out)
            keep = kept_rows(kind, idx)
            exp = [(rid[keep], None)]
            if len(out) == 2:
                v, ok = gather(bpay, idx[keep])
                exp.append((v, ok if kind == D.STAGE_RIGHT else None))
            assert_cols(got, exp, True, f"{NAME[t]} probe with all ones, stage {kind}")
    finally:
        look.close()


def test_refused_key_and_payload_types(gpu_ctx):
    """keys: one integer-like column of <= 8 bytes (Boolean, floats and Decimal128 are DFGPU_ERR_UNSUPPORTED, as composite components
    too); payload: fixed-width columns of <= 8 bytes, <= 64 bits together; a probe column whose width or signedness differs from the
    lookup's key is DFGPU_ERR_INVALID"""
    dec = D.decimal128(38, 0)
    for kt in (D.BOOL, D.FLOAT32, D.FLOAT64, dec):
        assert err_code(lambda: D.Lookup(gpu_ctx, kt, [])) == UNSUPPORTED, kt
        assert err_code(lambda: D.Lookup(gpu_ctx, kt, [D.INT32])) == UNSUPPORTED, kt
        assert err_code(lambda: D.Lookup(gpu_ctx, payload_types=[D.INT32], key_types=[D.INT32, kt], key_ranges=[(0, 9), (0, 9)])) == UNSUPPORTED
    for pays in ([D.BOOL], [dec], [D.INT64, D.INT8], [D.UINT32, D.UINT32, D.INT8]):
        assert err_code(lambda: D.Lookup(gpu_ctx, D.INT64, pays)) == UNSUPPORTED, pays
    look = D.Lookup(gpu_ctx, D.INT32, [D.INT64])
    try:
        for pt in (D.BOOL, D.UINT32, D.INT16, D.INT64, D.FLOAT32):
            assert err_code(lambda: D.Pipeline(gpu_ctx, [pt, D.INT64], None, [(D.STAGE_INNER, 0, look)])) == INVALID, NAME[pt]
        p = D.Pipeline(gpu_ctx, [D.DATE32, D.INT64], None, [(D.STAGE_INNER, 0, look)])   # same width and signedness: accepted
        p.close()
    finally:
        look.close()
