"""Float MIN / MAX on every aggregate path against the bit-exact totalOrder reference of tests/float_order.py: dfgpu_agg (Single from host
and device, Partial -> [PartialReduce ->] Final, skip-partial state rows, no GROUP BY, Float64 and Float32), the fused pipeline's
join-keyed sink (with and without non-null counters, beside a Decimal128 SUM, Partial -> dfgpu_agg Final, a LEFT stage), its dense sink
(the per-warp and the per-block accumulators, a one-slot domain, no GROUP BY, Partial) and its hash sink (Single, growth with replay,
beside a Decimal128 SUM, Partial -> Final), and the operator twin's fused plans against GpuAggregateExec.  The edge data puts +-NaN with
and without payloads, +-0.0, +-inf and the extreme finite values into groups that isolate each case, in row order and reversed, with
different batch sizes; one case races a million rows of +0.0 and -0.0 on 16 groups.  SUM / AVG / COUNT run beside MIN / MAX: a SUM or
AVG is compared by its class (NaN, +inf, -inf, finite) and a finite one within the math.fsum bound."""
import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import float_order as FO
from decimal_util import gpu_nodes
from harness import split_points

pytestmark = pytest.mark.gpu

COL = lambda i: [(O.E_COLUMN, i, None, 0, 0)]                       # noqa: E731
FUNCS = [D.AGG_MIN, D.AGG_MAX, D.AGG_SUM, D.AGG_AVG, D.AGG_COUNT]
F4 = [D.AGG_MIN, D.AGG_MAX, D.AGG_AVG, D.AGG_COUNT]                  # the join-keyed and hash sinks take four aggregates
NG = 48
ORDERS = [(False, 3000), (True, 7777)]                               # (reversed, rows per push)
NP_T = {np.float64: D.FLOAT64, np.float32: D.FLOAT32}


@pytest.fixture(scope="module")
def edge64():
    return FO.edge_case(np.random.default_rng(64), np.float64, NG)


def in_order(cols, rev):
    return [(v[::-1].copy(), None if ok is None else ok[::-1].copy()) for v, ok in cols] if rev else cols


def drain(h):
    """-> ([(values, valid or None)] per output column, [type codes])"""
    outs = h.drain(host=True)
    if not outs:
        return [], []
    types = [outs[0].column(i).type for i in range(outs[0].num_columns)]
    cols = []
    for c in range(len(types)):
        parts = [b.column_numpy(c) for b in outs]
        v = np.concatenate([p[0] for p in parts])
        ok = np.concatenate([np.ones(len(p[0]), bool) if p[1] is None else p[1] for p in parts])
        cols.append((v, ok))
    return cols, types


def push(ctx, h, cols, types, batch_rows, device=False):
    keep = []
    for s, e in split_points(len(cols[0][0]), batch_rows):
        hc = []
        for (v, ok), t in zip(cols, types):
            if D.type_base(t) == D.DECIMAL128:
                hc.append(D.HostColumn(D.decimal_to_words([int(x) for x in v[s:e]]), None if ok is None else ok[s:e], t))
            else:
                hc.append(D.HostColumn(v[s:e], None if ok is None else ok[s:e], t))
        if device:
            dc = [D.DeviceColumn.from_host(ctx, x) for x in hc]
            keep.append(dc)
            h.push_device(dc)
        else:
            h.push_host(hc)
    return keep


def check(out, ref, funcs, dtype, what, nk=1, first=None):
    """out: output columns, group key in column 0 (None when nk == 0), the aggregates `funcs` from column `first` (default nk) on;
    ref: {group: FO.reference tuple}"""
    first = nk if first is None else first
    if nk:
        keys = out[0][0].tolist()
        assert sorted(keys) == sorted(ref), f"{what}: groups {sorted(set(keys) ^ set(ref))[:8]} differ"
        rows = {k: i for i, k in enumerate(keys)}
    else:
        assert len(out[0][0]) == 1 and list(ref) == [0], what
        rows = {0: 0}
    gs = sorted(ref)
    idx = np.array([rows[g] for g in gs], np.int64)
    for j, f in enumerate(funcs):
        v, ok = out[first + j]
        v, ok = v[idx], ok[idx]
        w = what + f" agg {j}"
        if f in (D.AGG_MIN, D.AGG_MAX):
            cell = [ref[g][0 if f == D.AGG_MIN else 1] for g in gs]
            want = np.zeros(len(gs), dtype)
            for i, x in enumerate(cell):
                if x is not None:
                    want[i] = x
            FO.assert_same_bits(v, ok, want, np.array([x is not None for x in cell]), w)
        elif f in (D.AGG_SUM, D.AGG_AVG):
            for i, g in enumerate(gs):
                exp = ref[g][2 if f == D.AGG_SUM else 3]
                got = float(v[i]) if ok[i] else None
                if exp is None:
                    assert got is None, f"{w} group {g}: {got!r}, expected NULL"
                else:
                    FO.check_sum(got, exp, f"{w} group {g}")
        elif f == D.AGG_COUNT:
            assert v.tolist() == [ref[g][4] for g in gs] and ok.all(), w


def agg_specs(funcs, arg=1):
    return [(f, arg, -1) for f in funcs]


def final_of(ctx, part, ptypes, funcs, nk=1):
    """dfgpu_agg Final over Partial state columns"""
    h = D.AggHandle(ctx, ptypes, list(range(nk)), [(f, -1, -1) for f in funcs], D.AGG_FINAL, 8192)
    push(ctx, h, part, ptypes, 5000)
    h.finish()
    out, _ = drain(h)
    h.close()
    return out


# ---------------------------------------------------------------- dfgpu_agg
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_dfgpu_agg_single_partial_final_and_reduce(gpu_ctx, dtype):
    keys, vals, valid = FO.edge_case(np.random.default_rng(7), dtype, NG)
    ref = FO.reference(keys, vals, valid, NG)
    types = [D.INT64, NP_T[dtype]]
    for rev, br in ORDERS:
        cols = in_order([(keys, None), (vals, valid)], rev)
        for device in (False, True):
            h = D.AggHandle(gpu_ctx, types, [0], agg_specs(FUNCS), D.AGG_SINGLE, 8192)
            push(gpu_ctx, h, cols, types, br, device)
            h.finish()
            out, ot = drain(h)
            h.close()
            check(out, ref, FUNCS, dtype, f"single rev={rev} device={device}")
            assert ot[1] == ot[2] == NP_T[dtype]
        h = D.AggHandle(gpu_ctx, types, [0], agg_specs(FUNCS), D.AGG_PARTIAL, 8192)
        push(gpu_ctx, h, cols, types, br)
        h.finish()
        part, pt = drain(h)
        h.close()
        check(final_of(gpu_ctx, part, pt, FUNCS), ref, FUNCS, dtype, f"partial->final rev={rev}")
        h = D.AggHandle(gpu_ctx, pt, [0], [(f, -1, -1) for f in FUNCS], D.AGG_PARTIAL_REDUCE, 8192)
        push(gpu_ctx, h, part, pt, 17)
        h.finish()
        red, rt = drain(h)
        h.close()
        assert rt == pt
        check(final_of(gpu_ctx, red, rt, FUNCS), ref, FUNCS, dtype, f"partial->reduce->final rev={rev}")


def test_dfgpu_agg_skip_partial_state_rows(gpu_ctx, edge64):
    keys, vals, valid = edge64
    ref = FO.reference(keys, vals, valid, NG)
    types = [D.INT64, D.FLOAT64]
    h = D.AggHandle(gpu_ctx, types, [0], agg_specs(FUNCS), D.AGG_PARTIAL, 8192)
    h.set_skip_partial(1, 0.0)         # every batch after the first passes through as state rows
    push(gpu_ctx, h, [(keys, None), (vals, valid)], types, 2000, device=True)
    h.finish()
    part, pt = drain(h)
    assert h.metric("skipped_aggregation_rows") > 0
    h.close()
    check(final_of(gpu_ctx, part, pt, FUNCS), ref, FUNCS, np.float64, "skip-partial")


def test_dfgpu_agg_without_group_by(gpu_ctx, edge64):
    keys, vals, valid = edge64
    for sel in (None, 2, 3, 9):   # everything, then the signed zeros, -NaN / +NaN, -NaN / 1.0 alone
        m = np.ones(len(keys), bool) if sel is None else keys == sel
        k, v, ok = np.zeros(int(m.sum()), np.int64), vals[m], valid[m]
        ref = FO.reference(k, v, ok, 1)
        for rev, br in ORDERS:
            cols = in_order([(v, ok)], rev)
            h = D.AggHandle(gpu_ctx, [D.FLOAT64], [], agg_specs(FUNCS, 0), D.AGG_SINGLE, 8192)
            push(gpu_ctx, h, cols, [D.FLOAT64], br)
            h.finish()
            out, _ = drain(h)
            h.close()
            check(out, ref, FUNCS, np.float64, f"no group by, group {sel}", nk=0)


# ---------------------------------------------------------------- the join-keyed sink
def key_lookup(ctx, keys, n_acc):
    look = D.Lookup(ctx, D.INT64, [], n_acc_words=n_acc, expected_rows=len(keys))
    p = D.Pipeline(ctx, [D.INT64])
    p.sink_build(look, 0, [])
    p.push_host([D.HostColumn(np.asarray(keys, np.int64))])
    p.finish()
    p.close()
    return look


def run_pipe(ctx, p, cols, types, br, setup):
    try:
        setup(p)
        push(ctx, p, cols, types, br)
        p.finish()
        out, ot = drain(p)
        return out, ot, {m: p.metric(m) for m in ("num_groups", "sink_rows", "dense_block_launches", "group_rehashes", "replayed_rows")}
    finally:
        p.close()


def pipe_aggs(funcs, arg=1):
    return [(f, None if f == D.AGG_COUNT_STAR else gpu_nodes(D, COL(arg))) for f in funcs]


@pytest.mark.parametrize("case", ["nullable", "non_null", "decimal_sum", "partial", "left"])
def test_join_keyed_sink(gpu_ctx, edge64, case):
    keys, vals, valid = edge64
    if case == "non_null":
        valid = np.ones(len(keys), bool)
    ref = FO.reference(keys, vals, valid, NG)
    funcs = [D.AGG_MIN, D.AGG_MAX, D.AGG_COUNT] if case == "decimal_sum" else F4
    # words: the row counter, MIN, MAX, AVG {sum, count}, COUNT = 6, then one non-null counter each for MIN and MAX; with the Decimal128
    # SUM instead of AVG: 6 and three counters
    n_acc = {"non_null": 6, "decimal_sum": 9}.get(case, 8)
    build = np.arange(NG + (12 if case == "left" else 0), dtype=np.int64)
    stage = D.STAGE_LEFT if case == "left" else D.STAGE_INNER
    mode = D.AGG_PARTIAL if case == "partial" else D.AGG_SINGLE
    types = [D.INT64, D.FLOAT64]
    dec = None
    if case == "decimal_sum":
        dec = np.random.default_rng(9).integers(-10 ** 12, 10 ** 12, len(keys))
        types.append(D.decimal128(15, 2))
    if case == "left":
        for g in range(NG, NG + 12):
            ref[g] = (None, None, None, None, 0)
    for rev, br in ORDERS:
        look = key_lookup(gpu_ctx, build, n_acc)
        cols = [(keys, None), (vals, None if case == "non_null" else valid)] + ([(dec, None)] if dec is not None else [])
        aggs = pipe_aggs(funcs) + ([(D.AGG_SUM, gpu_nodes(D, COL(2)))] if dec is not None else [])
        out, ot, _ = run_pipe(gpu_ctx, D.Pipeline(gpu_ctx, types, None, [(stage, 0, look)]), in_order(cols, rev), types, br,
                              lambda p: p.sink_aggregate([0], aggs, mode))
        look.close()
        what = f"{case} rev={rev}"
        if mode == D.AGG_PARTIAL:
            out = final_of(gpu_ctx, out, ot, funcs)
        check(out, ref, funcs, np.float64, what)
        if dec is not None:   # the Decimal128 SUM beside the float path, exactly
            got = dict(zip(out[0][0].tolist(), D.words_to_decimal(out[1 + len(funcs)][0])))
            want = {}
            for k, x in zip(keys.tolist(), dec.tolist()):
                want[k] = want.get(k, 0) + x
            assert got == want, what


# ---------------------------------------------------------------- the dense sink
@pytest.mark.parametrize("case", ["per_warp", "per_block", "one_slot", "no_group_by", "partial"])
def test_dense_sink(gpu_ctx, edge64, case):
    keys, vals, valid = edge64
    zero = np.zeros(len(keys), np.int64)
    types = [D.INT64, D.FLOAT64, D.INT64]
    if case in ("one_slot", "no_group_by"):
        ref = FO.reference(zero, vals, valid, 1)
    else:
        ref = FO.reference(keys, vals, valid, NG)
    group, rng_, nk, first = {"per_warp": ([0], [(0, NG - 1)], 1, 1), "per_block": ([0, 2], [(0, NG - 1), (0, 3)], 1, 2),
                              "one_slot": ([2], [(0, 0)], 1, 1), "no_group_by": ([], [], 0, 0),
                              "partial": ([0], [(0, NG - 1)], 1, 1)}[case]
    mode = D.AGG_PARTIAL if case == "partial" else D.AGG_SINGLE
    for rev, br in ORDERS:
        cols = in_order([(keys, None), (vals, valid), (zero, None)], rev)
        out, ot, m = run_pipe(gpu_ctx, D.Pipeline(gpu_ctx, types), cols, types, br,
                              lambda p: p.sink_aggregate_dense(group, rng_, pipe_aggs(FUNCS), mode))
        what = f"{case} rev={rev}"
        assert (m["dense_block_launches"] > 0) == (case == "per_block"), what
        if mode == D.AGG_PARTIAL:
            out = final_of(gpu_ctx, out, ot, FUNCS)
        check(out, ref, FUNCS, np.float64, what, nk=nk, first=first)


# ---------------------------------------------------------------- the hash sink
@pytest.mark.parametrize("case", ["single", "growth", "decimal_sum", "partial"])
def test_hash_sink(gpu_ctx, edge64, case):
    ids, vals, valid = edge64
    n_ids = NG
    if case == "growth":   # 300 000 more groups of ordinary values after the edge rows: the table grows past its one-group hint
        rng = np.random.default_rng(12)
        fid = NG + rng.integers(0, 300_000, 600_000)
        fv = rng.standard_normal(len(fid))
        fv[::97] = -0.0
        ids, vals, valid, n_ids = np.concatenate([ids, fid]), np.concatenate([vals, fv]), np.concatenate([valid, np.ones(len(fid), bool)]), NG + 300_000
    keys = ids * 1_000_003 - 7          # not a dense domain
    ref = {g * 1_000_003 - 7: r for g, r in FO.reference(ids, vals, valid, n_ids).items()}
    types = [D.INT64, D.FLOAT64]
    dec = None
    if case == "decimal_sum":
        dec = np.random.default_rng(11).integers(-10 ** 12, 10 ** 12, len(keys))
        types.append(D.decimal128(15, 2))
    mode = D.AGG_PARTIAL if case == "partial" else D.AGG_SINGLE
    hint = 1 if case == "growth" else 0
    funcs = {"single": [D.AGG_MIN, D.AGG_MAX, D.AGG_SUM, D.AGG_COUNT], "growth": F4, "decimal_sum": F4[:3],
             "partial": [D.AGG_MIN, D.AGG_MAX, D.AGG_SUM, D.AGG_AVG]}[case]
    for rev, br in ORDERS:
        cols = [(keys, None), (vals, valid)] + ([(dec, None)] if dec is not None else [])
        aggs = pipe_aggs(funcs) + ([(D.AGG_SUM, gpu_nodes(D, COL(2)))] if dec is not None else [])
        out, ot, m = run_pipe(gpu_ctx, D.Pipeline(gpu_ctx, types), in_order(cols, rev), types, br if case != "growth" else None,
                              lambda p: p.sink_aggregate_hash([0], aggs, mode, 0, hint))
        what = f"{case} rev={rev}"
        assert m["sink_rows"] == len(keys) and m["num_groups"] == len(ref), (what, m)   # every row reached a record, every group one
        if case == "growth":
            assert m["group_rehashes"] > 0 and m["replayed_rows"] > 0, (what, m)
        if mode == D.AGG_PARTIAL:
            out = final_of(gpu_ctx, out, ot, funcs)
        check(out, ref, funcs, np.float64, what)
        if dec is not None:
            got = dict(zip(out[0][0].tolist(), D.words_to_decimal(out[1 + len(funcs)][0])))
            want = {}
            for k, x in zip(keys.tolist(), dec.tolist()):
                want[k] = want.get(k, 0) + x
            assert got == want, what


# ---------------------------------------------------------------- a million rows of signed zeros racing on 16 groups
def test_signed_zero_race_on_every_path(gpu_ctx):
    keys, vals = FO.race_case(np.random.default_rng(16))
    ref = FO.reference(keys, vals, None, 16)
    assert FO.bits(ref[10][0]) == FO.bits(-0.0) and FO.bits(ref[10][1]) == FO.bits(0.0)
    types = [D.INT64, D.FLOAT64, D.INT64]
    funcs = [D.AGG_MIN, D.AGG_MAX, D.AGG_COUNT]
    for rev, br in ((False, None), (True, 300_000)):
        cols = in_order([(keys, None), (vals, None), (np.zeros(len(keys), np.int64), None)], rev)
        h = D.AggHandle(gpu_ctx, types, [0], agg_specs(funcs), D.AGG_SINGLE, 8192)
        push(gpu_ctx, h, cols, types, br, device=True)
        h.finish()
        out, _ = drain(h)
        h.close()
        check(out, ref, funcs, np.float64, f"dfgpu_agg rev={rev}")
        look = key_lookup(gpu_ctx, np.arange(16), 4)
        out, _, _ = run_pipe(gpu_ctx, D.Pipeline(gpu_ctx, types, None, [(D.STAGE_INNER, 0, look)]), cols, types, br,
                             lambda p: p.sink_aggregate([0], pipe_aggs(funcs), D.AGG_SINGLE))
        look.close()
        check(out, ref, funcs, np.float64, f"join-keyed rev={rev}")
        for group, rr, first in (([0], [(0, 15)], 1), ([0, 2], [(0, 15), (0, 12)], 2)):   # per-warp; 17 x 14 slots per block
            out, _, m = run_pipe(gpu_ctx, D.Pipeline(gpu_ctx, types), cols, types, br,
                                 lambda p: p.sink_aggregate_dense(group, rr, pipe_aggs(funcs), D.AGG_SINGLE))
            assert (m["dense_block_launches"] > 0) == (len(group) == 2)
            check(out, ref, funcs, np.float64, f"dense {len(group)} keys rev={rev}", first=first)
        out, _, _ = run_pipe(gpu_ctx, D.Pipeline(gpu_ctx, types), cols, types, br,
                             lambda p: p.sink_aggregate_hash([0], pipe_aggs(funcs), D.AGG_SINGLE))
        check(out, ref, funcs, np.float64, f"hash rev={rev}")


# ---------------------------------------------------------------- Float32 MIN / MAX stays on dfgpu_agg
def test_float32_min_max_is_rejected_by_every_pipeline_sink(gpu_ctx):
    types = [D.INT64, D.FLOAT32]
    for f in (D.AGG_MIN, D.AGG_MAX):
        aggs = pipe_aggs([f])
        look = key_lookup(gpu_ctx, np.arange(4), 4)
        for stages, sink in (([(D.STAGE_INNER, 0, look)], lambda p: p.sink_aggregate([0], aggs)),
                             ([], lambda p: p.sink_aggregate_dense([0], [(0, 3)], aggs)), ([], lambda p: p.sink_aggregate_hash([0], aggs))):
            p = D.Pipeline(gpu_ctx, types, None, stages)
            with pytest.raises(D.DfgpuError, match="Float32") as ei:
                sink(p)
            assert ei.value.code == -3
            p.close()
        look.close()


# ---------------------------------------------------------------- the operator twin
def test_twin_fused_plans_equal_the_unfused_aggregate(gpu_ctx, edge64):
    from datafusion_b200.exec import (AggregateExpr, GpuAggregateExec, GpuFilterExec, GpuPipelineExec, MemoryExec, TaskContext, col, collect,
                                      fuse_hash_aggregates, fuse_pipelines, lit)
    keys, vals, valid = edge64
    t = pa.table({"g": keys, "h": keys * 1_000_003 - 7, "x": pa.array(vals, mask=~valid), "keep": np.ones(len(keys), np.int64)})
    src = MemoryExec(t.to_batches(max_chunksize=5000), t.schema)
    tctx = TaskContext(ctx=gpu_ctx)
    names = {D.AGG_MIN: "min", D.AGG_MAX: "max", D.AGG_SUM: "sum", D.AGG_AVG: "avg", D.AGG_COUNT: "count"}
    for key, sink, fuse, funcs in (("g", "dense", fuse_pipelines, FUNCS), ("h", "hash", lambda p: fuse_hash_aggregates(fuse_pipelines(p)), F4)):
        aggr = [AggregateExpr(names[f], "x", names[f] + "_x") for f in funcs]
        plan = GpuAggregateExec("Single", [key], aggr, GpuFilterExec(col("keep") > lit(0, pa.int64()), src))
        fused = fuse(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == sink
        got = pa.Table.from_batches(collect(fused, tctx), schema=plan.schema).sort_by(key)
        want = pa.Table.from_batches(collect(plan, tctx), schema=plan.schema).sort_by(key)
        assert got.num_rows == want.num_rows == NG
        for name in ("min_x", "max_x"):
            g, w = got.column(name).combine_chunks(), want.column(name).combine_chunks()
            gv, wv = g.is_valid().to_numpy(zero_copy_only=False), w.is_valid().to_numpy(zero_copy_only=False)
            FO.assert_same_bits(g.to_numpy(zero_copy_only=False), gv, w.to_numpy(zero_copy_only=False), wv, f"{sink} {name}")
        assert got.column("count_x").to_pylist() == want.column("count_x").to_pylist()
        ref = FO.reference(keys, vals, valid, NG)
        out = [(got.column(c).combine_chunks().to_numpy(zero_copy_only=False), got.column(c).combine_chunks().is_valid().to_numpy(zero_copy_only=False))
               for c in [key] + [names[f] + "_x" for f in funcs]]
        if key == "h":
            ref = {g * 1_000_003 - 7: r for g, r in ref.items()}
        check(out, ref, funcs, np.float64, f"twin {sink}")
