"""One dfgpu_lookup over its whole life: built once and read by several pipelines in a row, cleared and refilled, built by two pipelines,
and the column statistics that size it.  Some consumers write into the lookup's records: the join-keyed aggregate sink (LEFT and LEFT_ANTI
stages and the partitioned pass included) accumulates into their accumulator words, and a FULL stage marks each matched record visited in
the first one.  A consumer that claims words an earlier one wrote starts from zero: the words are reset (kernel-timing family
"lookup_acc_reset"; a fresh or cleared lookup launches nothing), not refused, so a build side serves any number of aggregates without a
rebuild.  Every result is compared with a plain reference over that consumer's own probe rows and the lookup's current build rows only, so
the order in which consumers run never matters.  Each consumer reaches build keys it alone probes, keys another consumer also probes, and
some build keys no probe reaches: stale state from an earlier consumer shows up as extra groups, inflated counts or missing tail rows."""
import ctypes as CT

import numpy as np
import pytest

from datafusion_b200 import capi as D
from decimal_util import gpu_col_as_py
from test_gpu_partition_bits import Src

pytestmark = pytest.mark.gpu
UNSUPPORTED, INVALID, STATE = -3, -1, -5
N_ACC = 8            # row counter + COUNT(x) + SUM / MIN / MAX(x) each with its non-null counter, four aggregates at most per sink
PAY_MAX = 199        # payloads lie in [0, PAY_MAX]: the dense sink groups on them
C = lambda i: (D.EXPR_COLUMN, i, 0, 0, 0, 0.0)                                 # noqa: E731
COUNT_STAR = (D.AGG_COUNT_STAR, None)

# which probe stage each consumer runs
KIND = {"inner": D.STAGE_INNER, "semi": D.STAGE_SEMI, "anti": D.STAGE_ANTI, "maybe": D.STAGE_MAYBE, "right": D.STAGE_RIGHT, "full": D.STAGE_RIGHT,
        "dense": D.STAGE_INNER, "hash": D.STAGE_INNER, "agg": D.STAGE_INNER, "agg_partial": D.STAGE_INNER, "agg_sum": D.STAGE_INNER,
        "left": D.STAGE_LEFT, "left_anti": D.STAGE_LEFT_ANTI}


class Shape:
    """the key of a lookup and the probe schema around it.  Build keys are codes in [0, universe): a one-column Int64 key 2 * code, or
    the composite key (a, b) = (code // 50, code % 50 - 50) of Int32 components over the domains a in [0, 199], b in [-50, 49].  Probe
    rows that must miss take keys no build holds: odd Int64 keys, or b in [0, 49] (a few with a out of its domain).  Probe columns: the
    key column(s), x (Int64, nullable), rid (Int64, unique); the stage's payload field follows them."""

    def __init__(self, composite=False):
        self.composite = composite
        self.nk = 2 if composite else 1
        self.types = ([D.INT32, D.INT32] if composite else [D.INT64]) + [D.INT64, D.INT64]
        self.x, self.rid, self.pay = self.nk, self.nk + 1, self.nk + 2
        self.key = [0, 1] if composite else 0
        self.group = list(range(self.nk)) + [self.pay]
        self.universe = 200 * 50 if composite else 1 << 40

    def lookup(self, ctx, payload=True, n_acc_words=N_ACC, **kw):
        if self.composite:
            return D.Lookup(ctx, payload_types=[D.INT32] if payload else [], key_types=[D.INT32, D.INT32], key_ranges=[(0, 199), (-50, 49)],
                            n_acc_words=n_acc_words, **kw)
        return D.Lookup(ctx, D.INT64, [D.INT32] if payload else [], n_acc_words=n_acc_words, **kw)

    def key_cols(self, codes, miss=None, valid=None):
        """the key column(s) of `codes` as [(values, valid, type)]; rows flagged in `miss` take a key no build holds"""
        codes = np.asarray(codes, np.int64)
        if not self.composite:
            k = 2 * codes if miss is None else np.where(miss, 2 * codes + 1, 2 * codes)
            return [(k, valid, D.INT64)]
        a, b = codes // 50, codes % 50 - 50
        if miss is not None:
            a = np.where(miss, codes % 210, a)          # a few a > 199: outside the domain, the packed sentinel
            b = np.where(miss, codes % 50, b)
        return [(a.astype(np.int32), valid, D.INT32), (b.astype(np.int32), None, D.INT32)]

    def out_key(self, code):
        """the group key columns the join-keyed sink emits for the record of `code`"""
        return (code // 50, code % 50 - 50) if self.composite else (2 * code,)


SINGLE, COMPOSITE = Shape(), Shape(composite=True)


def fill(ctx, shape, look, codes, pays=None, null_key_row=False):
    """one build pipeline into `look`: the keys of `codes` with payload `pays` (None: a key set), plus one row with a NULL key"""
    cols = shape.key_cols(codes)
    if null_key_row:
        cols = [(np.append(v, v[:1]), np.append(np.ones(len(codes), bool), False) if g == 0 else None, t) for g, (v, _, t) in enumerate(cols)]
    if pays is not None:
        cols.append((np.append(pays, pays[:1]) if null_key_row else pays, None, D.INT32))
    types = [t for _, _, t in cols]
    b = D.Pipeline(ctx, types)
    try:
        pay_cols = [shape.nk] if pays is not None else []
        if shape.composite:
            b.sink_build(look, payload_cols=pay_cols, key_cols=[0, 1])
        else:
            b.sink_build(look, 0, pay_cols)
        if len(codes):
            b.push_host([D.HostColumn(v, m, t) for v, m, t in cols])
        b.finish()
    finally:
        b.close()


class Probe:
    """n probe rows: ~70 % reach a code of `reach` (every code of it once more in front when `every`), the others miss, 5 % have a NULL
    key and 20 % a NULL x (`nulls`).  codes[i] is the build code row i can match, None for a miss or a NULL key."""

    def __init__(self, rng, shape, reach, n, every=False, nulls=True):
        reach = np.asarray(reach, np.int64)
        hit = rng.random(n) < 0.7
        code = np.where(hit, reach[rng.integers(0, len(reach), n)], rng.integers(0, 1 << 20, n))
        if every:
            code, hit = np.concatenate([reach, code]), np.concatenate([np.ones(len(reach), bool), hit])
        m = len(code)
        kvalid = rng.random(m) >= 0.05 if nulls else None
        if every and nulls:
            kvalid[:len(reach)] = True
        self.x = rng.integers(-10**6, 10**6, m).astype(np.int64)
        self.xvalid = rng.random(m) >= 0.2 if nulls else None
        self.rid = np.arange(m, dtype=np.int64) * 3 + 1
        self.cols = shape.key_cols(code, ~hit, kvalid) + [(self.x, self.xvalid, D.INT64), (self.rid, None, D.INT64)]
        ok = hit if kvalid is None else hit & kvalid
        self.codes = [int(c) if k else None for c, k in zip(code.tolist(), ok.tolist())]
        xv = np.ones(m, bool) if self.xvalid is None else self.xvalid
        self.xs = [v if k else None for v, k in zip(self.x.tolist(), xv.tolist())]

    def host(self, s=0, e=None):
        return [D.HostColumn(v[s:e], None if m is None else m[s:e], t) for v, m, t in self.cols]


def rows_of(outs):
    """the batches as a sorted list of row tuples, None for NULL"""
    if not outs:
        return []
    cols = [[] for _ in range(outs[0].num_columns)]
    for b in outs:
        for i in range(len(cols)):
            cols[i] += gpu_col_as_py(D, b, i)[0]
    return sorted(zip(*cols), key=repr)


def final(ctx, outs, n_group, funcs):
    """the Partial state batches through dfgpu_agg's Final"""
    rows = rows_of(outs)
    if not rows:
        return []
    types = [outs[0].column(i).type for i in range(outs[0].num_columns)]
    cols = list(zip(*rows))
    host = [D.HostColumn(np.array([0 if v is None else v for v in c], D.NP_OF_TYPE[t]),
                         None if all(v is not None for v in c) else np.array([v is not None for v in c]), t) for c, t in zip(cols, types)]
    a = D.AggHandle(ctx, types, list(range(n_group)), [(f, -1, -1) for f in funcs], D.AGG_FINAL, 8192)
    try:
        a.push_host(host)
        a.finish()
        return rows_of(a.drain(host=True))
    finally:
        a.close()


def set_sink(p, shape, name):
    X = [C(shape.x)]
    if name in ("inner", "right", "full"):
        p.sink_output([shape.rid, shape.pay], ordered=False)
    elif name in ("semi", "anti", "maybe"):
        p.sink_output([shape.rid], ordered=False)
    elif name == "dense":
        p.sink_aggregate_dense([shape.pay], [(0, PAY_MAX)], [COUNT_STAR, (D.AGG_COUNT, X), (D.AGG_SUM, X), (D.AGG_MIN, X), (D.AGG_MAX, X)])
    elif name == "hash":
        p.sink_aggregate_hash([shape.pay], [COUNT_STAR, (D.AGG_SUM, X), (D.AGG_MIN, X), (D.AGG_MAX, X)])
    elif name == "agg":
        p.sink_aggregate(shape.group, [COUNT_STAR, (D.AGG_COUNT, X), (D.AGG_SUM, X), (D.AGG_MIN, X)])
    elif name == "agg_partial":
        p.sink_aggregate(shape.group, [COUNT_STAR, (D.AGG_SUM, X), (D.AGG_MAX, X), (D.AGG_COUNT, X)], D.AGG_PARTIAL)
    elif name == "agg_sum":   # one SUM over a non-null input column: the shape the partitioned pass takes
        p.sink_aggregate(shape.group, [(D.AGG_SUM, [C(shape.rid)])])
    elif name == "left":
        p.sink_aggregate(shape.group, [COUNT_STAR, (D.AGG_COUNT, X), (D.AGG_SUM, X), (D.AGG_MAX, X)])
    elif name == "left_anti":
        p.sink_aggregate(shape.group, [])


def run(ctx, shape, look, name, pr):
    """consumer `name` over probe `pr` (two pushes of device columns), closed before it returns: (sorted rows, metrics)"""
    p = D.Pipeline(ctx, shape.types, None, [(KIND[name], shape.key, look)])
    try:
        if name == "full":
            p.set_stage_full(0)
        set_sink(p, shape, name)
        n, keep = len(pr.rid), []
        for s, e in ((0, n // 3), (n // 3, n)):
            keep.append([D.DeviceColumn.from_host(ctx, c) for c in pr.host(s, e)])
            p.push_device(keep[-1])
        p.finish()
        outs = p.drain(host=True)
        got = final(ctx, outs, len(shape.group), [D.AGG_COUNT_STAR, D.AGG_SUM, D.AGG_MAX, D.AGG_COUNT]) if name == "agg_partial" else rows_of(outs)
        met = {m: p.metric(m) for m in ("partitioned_launches", "unmatched_build_rows", "input_rows")}
    finally:
        p.close()
    return got, met


def stats(xs):
    """COUNT(*), COUNT(x), SUM(x), MIN(x), MAX(x) of a group's x values (None = NULL)"""
    v = [x for x in xs if x is not None]
    return len(xs), len(v), (sum(v) if v else None), (min(v) if v else None), (max(v) if v else None)


def reference(shape, name, bd, pr):
    """consumer `name`'s rows from the build rows bd (code -> payload; None for a key set) and its own probe rows only"""
    hits = [(i, c) for i, c in enumerate(pr.codes) if c is not None and c in bd]
    hit_rows = {i for i, _ in hits}
    reached = {c for _, c in hits}
    rid = pr.rid.tolist()
    rows = []
    if name == "inner":
        rows = [(rid[i], bd[c]) for i, c in hits]
    elif name in ("semi", "maybe"):
        rows = [(rid[i],) for i, _ in hits]
    elif name == "anti":
        rows = [(rid[i],) for i in range(len(rid)) if i not in hit_rows]
    elif name in ("right", "full"):
        pay = dict(hits)
        rows = [(rid[i], bd[pay[i]] if i in pay else None) for i in range(len(rid))]
        if name == "full":
            rows += [(None, v) for c, v in bd.items() if c not in reached]
    elif name in ("dense", "hash"):
        g = {}
        for i, c in hits:
            g.setdefault(bd[c], []).append(pr.xs[i])
        s = {k: stats(v) for k, v in g.items()}
        rows = [(k,) + (s[k] if name == "dense" else (s[k][0],) + s[k][2:]) for k in g]
    elif name in ("agg", "agg_partial", "agg_sum", "left"):
        g = {}
        for i, c in hits:
            g.setdefault(c, []).append(i)
        keys = bd if name == "left" else g
        for c in keys:
            idx = g.get(c, [])
            n, cnt, sm, mn, mx = stats([pr.xs[i] for i in idx])
            head = shape.out_key(c) + (bd[c],)
            if name == "agg":
                rows.append(head + (n, cnt, sm, mn))
            elif name == "agg_partial":
                rows.append(head + (n, sm, mx, cnt))
            elif name == "agg_sum":
                rows.append(head + (sum(rid[i] for i in idx),))
            else:   # a build row no probe row reached: the NULL-padded row, COUNT(*) 1
                rows.append(head + (max(n, 1), cnt, sm, mx))
    elif name == "left_anti":
        rows = [shape.out_key(c) + (v,) for c, v in bd.items() if c not in reached]
    return sorted(rows, key=repr)


def check(ctx, shape, look, name, bd, pr, what=""):
    got, met = run(ctx, shape, look, name, pr)
    exp = reference(shape, name, bd, pr)
    assert len(got) == len(exp), f"{what}{name}: {len(got)} rows, expected {len(exp)}"
    assert got == exp, f"{what}{name}"
    return got, met


def key_plan(rng, shape, n_consumers, shared=400, own=250, untouched=300):
    """the build codes, split into the codes every consumer reaches, those each one alone reaches, and those none reaches"""
    n = shared + own * n_consumers + untouched
    codes = rng.choice(shape.universe, n, replace=False).astype(np.int64)
    own_sets = [codes[shared + own * j: shared + own * (j + 1)] for j in range(n_consumers)]
    return codes, codes[:shared], own_sets


# (a) one lookup, several consumers in a row, no clear; FULL last (it keeps its marks until a clear)
SEQUENCES = {
    "agg_agg": ["agg", "agg_partial"],
    "agg_left": ["agg_partial", "left"],
    "agg_left_anti": ["agg", "left_anti"],
    "agg_full": ["agg", "full"],
    "left_agg": ["left", "agg"],
    "left_anti_left": ["left_anti", "left", "full"],
    "every_consumer": ["agg", "inner", "semi", "anti", "right", "dense", "hash", "left_anti", "agg_sum", "left", "agg_partial", "full"],
}


@pytest.mark.parametrize("shape", [SINGLE, COMPOSITE], ids=["int64_key", "composite_key"])
@pytest.mark.parametrize("seq", sorted(SEQUENCES))
def test_consumers_in_a_row(gpu_ctx, seq, shape):
    names = SEQUENCES[seq]
    rng = np.random.default_rng(sorted(SEQUENCES).index(seq) + 100 * shape.composite)
    codes, shared, own = key_plan(rng, shape, len(names))
    pays = rng.integers(0, PAY_MAX + 1, len(codes)).astype(np.int32)
    bd = dict(zip(codes.tolist(), pays.tolist()))
    look = shape.lookup(gpu_ctx)
    try:
        fill(gpu_ctx, shape, look, codes, pays)
        for j, name in enumerate(names):
            pr = Probe(rng, shape, np.concatenate([shared, own[j]]), 5000)
            _, met = check(gpu_ctx, shape, look, name, bd, pr, f"{seq} step {j}: ")
            if name == "full":
                assert met["unmatched_build_rows"] == len(codes) - len({c for c in pr.codes if c is not None})
    finally:
        look.close()


def test_consumers_in_a_row_through_the_partitioned_pass(gpu_ctx, monkeypatch):
    """DFGPU_PIPE_RADIX_PARTS sends the join-keyed aggregate through the partitioned pass (records partitioned by slot range, then
    probed and accumulated one range at a time).  It admits a lookup of two accumulator words with a membership filter (the ring-fed
    phase A tests it) and probes without NULLs"""
    monkeypatch.setenv("DFGPU_PIPE_RADIX_PARTS", "4")
    names = ["agg_sum", "agg_sum", "left_anti", "agg_sum", "full"]
    rng = np.random.default_rng(7)
    codes, shared, own = key_plan(rng, SINGLE, len(names))
    pays = rng.integers(0, PAY_MAX + 1, len(codes)).astype(np.int32)
    bd = dict(zip(codes.tolist(), pays.tolist()))
    look = SINGLE.lookup(gpu_ctx, n_acc_words=2, membership_filter=1)
    try:
        fill(gpu_ctx, SINGLE, look, codes, pays)
        for j, name in enumerate(names):
            pr = Probe(rng, SINGLE, np.concatenate([shared, own[j]]), 20000, nulls=False)
            _, met = check(gpu_ctx, SINGLE, look, name, bd, pr, f"partitioned step {j}: ")
            if name == "agg_sum":
                assert met["partitioned_launches"] >= 1
    finally:
        look.close()


def test_acc_reset_runs_only_on_a_reused_lookup():
    """kernel-timing family "lookup_acc_reset": no launch for the first writer of a fresh lookup, one per later writer (a read-only
    consumer in between adds none), and none again after dfgpu_lookup_clear"""
    ctx = D.Context(0)
    try:
        ctx.set_kernel_timing(True)
        rng = np.random.default_rng(11)
        codes, shared, own = key_plan(rng, SINGLE, 6)
        pays = rng.integers(0, PAY_MAX + 1, len(codes)).astype(np.int32)
        bd = dict(zip(codes.tolist(), pays.tolist()))
        look = SINGLE.lookup(ctx)
        resets = lambda: ctx.kernel_time("lookup_acc_reset")[1]               # noqa: E731
        try:
            fill(ctx, SINGLE, look, codes, pays)
            for j, (name, n) in enumerate((("agg", 0), ("left", 1), ("inner", 1), ("left_anti", 2), ("full", 3))):
                check(ctx, SINGLE, look, name, bd, Probe(rng, SINGLE, np.concatenate([shared, own[j]]), 3000))
                assert resets() == n, f"after {name}"
            look.clear()
            fill(ctx, SINGLE, look, codes, pays)
            check(ctx, SINGLE, look, "agg", bd, Probe(rng, SINGLE, np.concatenate([shared, own[5]]), 3000))
            assert resets() == 3, "a cleared lookup's words are already 0"
        finally:
            look.close()
    finally:
        ctx.close()


def code_of(fn):
    with pytest.raises(D.DfgpuError) as e:
        fn()
    return e.value.code


def test_claim_rules(gpu_ctx):
    """the rules that stay: a live aggregate pipeline blocks a second aggregate, a FULL stage and dfgpu_lookup_clear; after a FULL stage
    an aggregate sink or a second FULL stage is DFGPU_ERR_STATE until dfgpu_lookup_clear, even once that pipeline is closed"""
    rng = np.random.default_rng(13)
    codes, shared, own = key_plan(rng, SINGLE, 2)
    pays = rng.integers(0, PAY_MAX + 1, len(codes)).astype(np.int32)
    bd = dict(zip(codes.tolist(), pays.tolist()))
    look = SINGLE.lookup(gpu_ctx)
    opened = []

    def pipe(kind):
        p = D.Pipeline(gpu_ctx, SINGLE.types, None, [(kind, 0, look)])
        opened.append(p)
        return p

    def agg(p):
        p.sink_aggregate(SINGLE.group, [COUNT_STAR])

    try:
        fill(gpu_ctx, SINGLE, look, codes, pays)
        live = pipe(D.STAGE_INNER)
        agg(live)
        live.push_host(Probe(rng, SINGLE, shared, 1000).host())
        assert code_of(lambda: agg(pipe(D.STAGE_INNER))) == STATE
        assert code_of(lambda: agg(pipe(D.STAGE_LEFT))) == STATE
        assert code_of(lambda: pipe(D.STAGE_RIGHT).set_stage_full(0)) == STATE
        assert code_of(look.clear) == STATE
        live.close()
        look.clear()
        fill(gpu_ctx, SINGLE, look, codes, pays)
        full = pipe(D.STAGE_RIGHT)
        full.set_stage_full(0)
        full.sink_output([SINGLE.rid])
        full.push_host(Probe(rng, SINGLE, shared, 1000).host())
        full.finish()
        full.close()
        assert code_of(lambda: agg(pipe(D.STAGE_INNER))) == STATE
        assert code_of(lambda: pipe(D.STAGE_RIGHT).set_stage_full(0)) == STATE
        check(gpu_ctx, SINGLE, look, "inner", bd, Probe(rng, SINGLE, own[0], 2000))   # reading is still allowed
        look.clear()
        fill(gpu_ctx, SINGLE, look, codes, pays)
        check(gpu_ctx, SINGLE, look, "agg", bd, Probe(rng, SINGLE, own[1], 2000))
        check(gpu_ctx, SINGLE, look, "full", bd, Probe(rng, SINGLE, own[0], 2000))
    finally:
        for p in opened:
            p.close()
        look.close()


# (b) clear and refill
def refill_sets(rng, universe, case, n1):
    """K1 and K2 codes: K2 disjoint from K1, overlapping half of it, or four times its size (so the refill needs a larger table)"""
    n2 = 4 * n1 if case == "larger" else n1
    pool = rng.choice(universe, n1 + n2, replace=False).astype(np.int64)
    k1 = pool[:n1]
    k2 = np.concatenate([k1[: n1 // 2], pool[n1: n1 + n2 - n1 // 2]]) if case == "overlap" else pool[n1:]
    return k1, k2


def filter_words(ctx, look):
    ptr, nbytes = look.filter_buffer()
    assert ptr and nbytes > 0
    return ctx.to_host(ptr, nbytes)


@pytest.mark.parametrize("case", ["disjoint", "overlap", "larger"])
@pytest.mark.parametrize("shape", [SINGLE, COMPOSITE], ids=["int64_key", "composite_key"])
def test_clear_and_refill(gpu_ctx, shape, case):
    """a hash lookup with payload and a membership filter (one-column or composite key): K1 with a NULL-key row, consumers, clear, K2
    (whose payloads are not K1's: [100, 199] against [0, 99]), consumers again over probes that also reach K1-only keys"""
    rng = np.random.default_rng(["disjoint", "overlap", "larger"].index(case) + 10 * shape.composite)
    k1, k2 = refill_sets(rng, shape.universe, case, 1200 if shape.composite else 3000)
    p1, p2 = rng.integers(0, 100, len(k1)).astype(np.int32), rng.integers(100, 200, len(k2)).astype(np.int32)
    bd1, bd2 = dict(zip(k1.tolist(), p1.tolist())), dict(zip(k2.tolist(), p2.tolist()))
    look = shape.lookup(gpu_ctx, membership_filter=1)
    try:
        fill(gpu_ctx, shape, look, k1, p1, null_key_row=True)
        assert look.metric("rows") == len(k1) and look.metric("null_keys") == 1
        cap1 = look.metric("capacity")
        for name in ("agg", "inner", "semi", "agg_partial"):
            check(gpu_ctx, shape, look, name, bd1, Probe(rng, shape, k1, 4000), "K1 ")
        assert filter_words(gpu_ctx, look).any()
        look.clear()
        assert look.metric("rows") == 0 and look.metric("null_keys") == 0
        assert not filter_words(gpu_ctx, look).any(), "the membership filter is all zero after a clear"
        check(gpu_ctx, shape, look, "semi", {}, Probe(rng, shape, k1, 2000), "cleared ")
        fill(gpu_ctx, shape, look, k2, p2)
        assert look.metric("rows") == len(k2) and look.metric("null_keys") == 0
        if case == "larger":
            assert look.metric("capacity") > cap1
        k1_only = np.setdiff1d(k1, k2)
        assert len(k1_only) > 0
        for name in ("inner", "semi", "anti", "agg", "left", "left_anti", "agg_partial", "full"):
            reach = np.concatenate([k2[: len(k2) // 2], k1_only])
            pr = Probe(rng, shape, reach, 6000, every=name == "anti")       # every K2 key half: ANTI keeps none of their rows
            got, _ = check(gpu_ctx, shape, look, name, bd2, pr, f"K2 {case} ")
            assert any(c in set(k1_only.tolist()) for c in pr.codes if c is not None), "the probe reaches K1-only keys"
    finally:
        look.close()


@pytest.mark.parametrize("case", ["disjoint", "overlap", "larger"])
def test_clear_and_refill_bitmap(gpu_ctx, case):
    """a key set over a key range from dfgpu_column_minmax_device (a bitmap): after the clear no key matches, after the refill exactly K2"""
    rng = np.random.default_rng(30 + ["disjoint", "overlap", "larger"].index(case))
    lo, hi = 5000, 5000 + 60000
    k1, k2 = refill_sets(rng, (hi - lo) // 2 - 2, case, 3000)
    k1, k2 = k1 + lo // 2 + 1, k2 + lo // 2 + 1                                  # keys 2 * code inside (lo, hi - 2)
    k1 = np.concatenate([k1, [lo // 2, (hi - 2) // 2]])                          # and K1 at the range's ends
    dev = D.DeviceColumn.from_host(gpu_ctx, D.HostColumn(2 * k1))
    kr = D.column_minmax_device(gpu_ctx, dev)
    assert kr == (lo, hi - 2, len(k1))
    look = D.Lookup(gpu_ctx, D.INT64, [], key_range=kr[:2])
    try:
        assert look.metric("mode") == 1
        fill(gpu_ctx, SINGLE, look, k1)
        s1 = dict.fromkeys(k1.tolist())
        for name in ("semi", "anti"):
            check(gpu_ctx, SINGLE, look, name, s1, Probe(rng, SINGLE, k1, 4000), "K1 ")
        look.clear()
        assert look.metric("rows") == 0
        check(gpu_ctx, SINGLE, look, "semi", {}, Probe(rng, SINGLE, k1, 2000), "cleared ")
        fill(gpu_ctx, SINGLE, look, k2)
        s2 = dict.fromkeys(k2.tolist())
        reach = np.concatenate([k2, np.setdiff1d(k1, k2)])
        for name in ("semi", "anti"):
            check(gpu_ctx, SINGLE, look, name, s2, Probe(rng, SINGLE, reach, 8000, every=name == "anti"), f"K2 {case} ")
    finally:
        look.close()


def test_clear_and_refill_filter_only(gpu_ctx):
    """a filter-only lookup sized for 12M keys carries the coarse level behind its exact blocks: both are zero after a clear, and after
    the refill a MAYBE stage passes every K2 row (no false negatives) and almost no row of a K1-only key"""
    rng = np.random.default_rng(41)
    expected = 12_000_000
    blocks = expected // 4
    coarse = (max(4096, expected // 8) + 1) & ~1
    look = D.Lookup(gpu_ctx, D.INT64, [], expected_rows=expected, filter_only=True)
    try:
        assert look.filter_buffer()[1] == blocks * 8 + coarse * 4
        k1, k2 = refill_sets(rng, SINGLE.universe, "overlap", 20000)
        fill(gpu_ctx, SINGLE, look, k1)
        w = filter_words(gpu_ctx, look)
        assert w[: blocks * 8].any() and w[blocks * 8:].any(), "both levels hold K1's bits"
        look.clear()
        assert not filter_words(gpu_ctx, look).any(), "exact blocks and coarse level are all zero after a clear"
        check(gpu_ctx, SINGLE, look, "maybe", {}, Probe(rng, SINGLE, k1, 3000), "cleared ")
        fill(gpu_ctx, SINGLE, look, k2)
        k1_only = np.setdiff1d(k1, k2)
        pr = Probe(rng, SINGLE, np.concatenate([k2, k1_only]), 30000, every=True)
        got, _ = run(gpu_ctx, SINGLE, look, "maybe", pr)
        got = {r[0] for r in got}
        s2, s1 = set(k2.tolist()), set(k1_only.tolist())
        rid = pr.rid.tolist()
        must = {rid[i] for i, c in enumerate(pr.codes) if c in s2}
        stale = [rid[i] for i, c in enumerate(pr.codes) if c in s1]
        assert must <= got, "a MAYBE stage passes every K2 row"
        assert len(stale) > 10000 and sum(r in got for r in stale) <= len(stale) // 100
    finally:
        look.close()


def test_clear_recovers_from_refused_builds(gpu_ctx):
    """a build push refused for a duplicate key (in one push, or split across two build pipelines into one target) or for a key outside
    a bitmap's range leaves records behind; a clear and a correct build then give exact results"""
    rng = np.random.default_rng(51)
    codes, shared, own = key_plan(rng, SINGLE, 3)
    pays = rng.integers(0, PAY_MAX + 1, len(codes)).astype(np.int32)
    bd = dict(zip(codes.tolist(), pays.tolist()))
    look = SINGLE.lookup(gpu_ctx)
    bits = D.Lookup(gpu_ctx, D.INT64, [], key_range=(0, 2 * 99999))
    try:
        dup = np.append(codes, codes[17])
        assert code_of(lambda: fill(gpu_ctx, SINGLE, look, dup, np.append(pays, 5))) == UNSUPPORTED
        look.clear()
        fill(gpu_ctx, SINGLE, look, codes, pays)
        for j, name in enumerate(("agg", "left_anti", "inner")):
            check(gpu_ctx, SINGLE, look, name, bd, Probe(rng, SINGLE, np.concatenate([shared, own[j]]), 4000), "after a duplicate ")
        look.clear()
        half = len(codes) // 2
        fill(gpu_ctx, SINGLE, look, codes[:half], pays[:half])
        assert code_of(lambda: fill(gpu_ctx, SINGLE, look, codes[half - 3:], pays[half - 3:])) == UNSUPPORTED
        look.clear()
        fill(gpu_ctx, SINGLE, look, codes[:half], pays[:half])
        fill(gpu_ctx, SINGLE, look, codes[half:], pays[half:])
        assert look.metric("rows") == len(codes)
        for j, name in enumerate(("left", "agg_partial", "full")):
            check(gpu_ctx, SINGLE, look, name, bd, Probe(rng, SINGLE, np.concatenate([shared, own[j]]), 4000), "after a split duplicate ")
        # the bitmap: keys 2 * code, code < 100000 in range; one push with a key past the range
        k = rng.choice(100000, 5000, replace=False).astype(np.int64)
        assert code_of(lambda: fill(gpu_ctx, SINGLE, bits, np.append(k, 100000))) == INVALID
        bits.clear()
        fill(gpu_ctx, SINGLE, bits, k)
        s = dict.fromkeys(k.tolist())
        for name in ("semi", "anti"):
            check(gpu_ctx, SINGLE, bits, name, s, Probe(rng, SINGLE, np.arange(100000), 8000), "bitmap after an out-of-range key ")
    finally:
        bits.close()
        look.close()


# (c) two build pipelines into one target
def test_two_build_pipelines_into_one_target(gpu_ctx):
    """a UNION ALL build side: 400 keys, then 5000 disjoint ones that outgrow expected_rows, so the table is rehashed with its membership
    filter; every key is found with its own payload, ANTI drops all of them, and the aggregates that follow start from zero"""
    rng = np.random.default_rng(61)
    codes = rng.choice(1 << 40, 5400, replace=False).astype(np.int64)
    pays = rng.integers(0, PAY_MAX + 1, len(codes)).astype(np.int32)
    bd = dict(zip(codes.tolist(), pays.tolist()))
    look = SINGLE.lookup(gpu_ctx, expected_rows=500, membership_filter=1)
    try:
        fill(gpu_ctx, SINGLE, look, codes[:400], pays[:400])
        assert look.metric("rehashes") == 0
        fill(gpu_ctx, SINGLE, look, codes[400:], pays[400:])
        assert look.metric("rehashes") >= 1 and look.metric("rows") == len(codes)
        every = Probe(rng, SINGLE, codes, 3000, every=True)
        got, _ = check(gpu_ctx, SINGLE, look, "inner", bd, every)
        assert {r[0] for r in got} >= set(every.rid[: len(codes)].tolist())
        got, _ = check(gpu_ctx, SINGLE, look, "anti", bd, every)
        assert not set(every.rid[: len(codes)].tolist()) & {r[0] for r in got}
        shared, mine, theirs = codes[:300], codes[300:2000], codes[2000:4000]
        for name, own in (("agg", mine), ("agg_partial", theirs), ("left", mine), ("full", theirs)):
            check(gpu_ctx, SINGLE, look, name, bd, Probe(rng, SINGLE, np.concatenate([shared, own]), 5000))
    finally:
        look.close()


# (d) column statistics: dfgpu_column_minmax_device and dfgpu_column_sum_device
STAT_TYPES = [D.INT8, D.INT16, D.INT32, D.INT64, D.UINT8, D.UINT16, D.UINT32, D.UINT64, D.DATE32, D.DATE64, D.TIMESTAMP]
DEC = D.decimal128(38, 4)


def stat_values(rng, t, m):
    """m values over the type's whole range, its extremes at rows 5 and 9 of the column (after any offset)"""
    if t == DEC:
        return rng.integers(0, 1 << 64, (m, 2), dtype=np.uint64, endpoint=False)
    dt = np.dtype(D.NP_OF_TYPE[t])
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, m, dtype=dt, endpoint=True)


def col_sum(ctx, col):
    s, cnt = CT.c_uint64(), CT.c_int64()
    ctx.check(ctx.lib.dfgpu_column_sum_device(ctx.h, CT.byref(col), CT.byref(s), CT.byref(cnt)))
    return s.value, cnt.value


def ref_stats(t, vals, valid):
    """(min, max, valid count) as dfgpu_column_minmax_device returns them (an unsigned value as its bit pattern in an int64; min 0,
    max -1 without a valid value) and the wrapping sum (Decimal128: low word + 3 x high word per value)"""
    keep = np.ones(len(vals), bool) if valid is None else valid
    v = vals[keep]
    if t == DEC:
        return None, (sum(int(lo) + 3 * int(hi) for lo, hi in v.tolist()) % (1 << 64), len(v))
    ints = [int(x) for x in v.tolist()]
    sm = sum(ints) % (1 << 64)
    if not ints:
        return (0, -1, 0), (sm, 0)
    as_i64 = lambda x: x - (1 << 64) if x >= 1 << 63 else x                    # noqa: E731
    return (as_i64(min(ints)), as_i64(max(ints)), len(ints)), (sm, len(ints))


def check_stats(ctx, t, vals, valid, off, what):
    src = Src(ctx, t, vals, valid, off)
    mm, sm = ref_stats(t, vals[off:], None if valid is None else valid[off:])
    if mm is not None:
        assert D.column_minmax_device(ctx, src.col) == mm, f"minmax {what}"
    assert col_sum(ctx, src.col) == sm, f"sum {what}"


@pytest.mark.parametrize("off", [0, 3, 37])
@pytest.mark.parametrize("t", STAT_TYPES + [DEC], ids=lambda t: {D.INT8: "i8", D.INT16: "i16", D.INT32: "i32", D.INT64: "i64", D.UINT8: "u8",
                                                                  D.UINT16: "u16", D.UINT32: "u32", D.UINT64: "u64", D.DATE32: "date32",
                                                                  D.DATE64: "date64", D.TIMESTAMP: "ts", DEC: "dec128"}[t])
def test_column_statistics(gpu_ctx, t, off):
    rng = np.random.default_rng(t * 100 + off)
    m = off + 3000
    vals = stat_values(rng, t, m)
    if t != DEC:
        info = np.iinfo(vals.dtype)
        vals[off + 5], vals[off + 9] = info.min, info.max
    valid = rng.random(m) >= 0.3
    valid[off + 5] = valid[off + 9] = True
    check_stats(gpu_ctx, t, vals, None, off, "no bitmap")
    check_stats(gpu_ctx, t, vals, valid, off, "bitmap")
    # the extremes NULL: the statistics skip them
    hidden = valid.copy()
    hidden[off + 5] = hidden[off + 9] = False
    check_stats(gpu_ctx, t, vals, hidden, off, "extremes NULL")
    check_stats(gpu_ctx, t, vals, np.zeros(m, bool), off, "all NULL")
    check_stats(gpu_ctx, t, vals[: off + 1], None, off + 1, "empty")


def test_column_statistics_past_one_grid_pass(gpu_ctx):
    """~1.1M rows: more than the kNumSMs * 8 blocks of 256 threads cover in one pass"""
    rng = np.random.default_rng(71)
    m = 1_100_003
    for t in STAT_TYPES + [DEC]:
        vals = stat_values(rng, t, m)
        valid = rng.random(m) >= 0.1
        check_stats(gpu_ctx, t, vals, valid, 3, f"type {t}")
        check_stats(gpu_ctx, t, vals, None, 0, f"type {t}")


def test_column_minmax_pinned_results(gpu_ctx):
    """UInt64 values at and above 2^63 come back as their bit patterns in an int64; a column without a valid value is (0, -1, 0)"""
    v = np.array([1 << 63, (1 << 64) - 1, 5, (1 << 63) + 7], np.uint64)
    src = Src(gpu_ctx, D.UINT64, v, None, 0)
    assert D.column_minmax_device(gpu_ctx, src.col) == (5, -1, 4)
    src = Src(gpu_ctx, D.UINT64, v, np.array([True, False, False, True]), 0)
    assert D.column_minmax_device(gpu_ctx, src.col) == (-(1 << 63), -(1 << 63) + 7, 2)
    src = Src(gpu_ctx, D.INT64, np.array([3, 4], np.int64), np.zeros(2, bool), 0)
    assert D.column_minmax_device(gpu_ctx, src.col) == (0, -1, 0)
