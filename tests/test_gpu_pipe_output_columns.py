"""Nullable and Decimal128 columns out of the fused pipeline's output sinks (dfgpu_pipeline_sink_output and _unordered).  Every result is
compared with a numpy restatement of the pipeline: in exact order for the ordered sink, as a multiset (sorted by the unique key column)
for the unordered one, NULLs as NULLs (the validity bits exactly, the values at the valid rows).  An output column has a bitmap exactly
when its input column had one in that push.  The cases cover every column width with and without bitmaps at Arrow bit offsets 0, 3 and
37 (an all-NULL column, a bitmap without NULLs), predicate-only / SEMI / ANTI / INNER (payload fields) / MAYBE / stage-filter / Decimal128
predicate pipelines, 0 % to 100 % survivors from below one tile to millions of rows, pushes mixing batches with and without bitmaps under
batch_size slicing, the multi-GPU plan's Decimal128 lineitem scan through the local hash exchange into per-partition Q3 aggregates, and
the operator twin's fuse_output_pipelines against the unfused joins."""
from decimal import Decimal

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from datafusion_b200.exec import (Column, GpuFilterExec, GpuHashJoinExec, GpuPipelineExec, GpuProjectionExec, MemoryExec, collect, col,
                                  fuse_output_pipelines, lit)
from test_gpu_partition_bits import Src

pytestmark = pytest.mark.gpu
DEC15, DEC38 = D.decimal128(15, 2), D.decimal128(38, 4)
KINDS = [D.INT8, D.INT16, D.INT32, D.INT64, D.FLOAT32, D.FLOAT64, D.DATE32, DEC15, DEC38]
NP = {D.INT8: np.int8, D.INT16: np.int16, D.INT32: np.int32, D.INT64: np.int64, D.FLOAT32: np.float32, D.FLOAT64: np.float64,
      D.DATE32: np.int32}
NODE = lambda k, a=0, t=0, v=0: (k, a, t, 0, v, 0.0)
CMP = lambda c, op, t, v: [NODE(D.EXPR_COLUMN, c), NODE(D.EXPR_LITERAL, 0, t, v), NODE(D.EXPR_BINARY, op)]
SEL, DCOL = 1, 2 + KINDS.index(DEC15)   # the predicate's Int32 column, the Decimal128(15, 2) column


def dec15_words(v):
    return np.stack([v.view(np.uint64), np.where(v < 0, np.uint64(2**64 - 1), np.uint64(0))], axis=1)


def values(rng, t, m):
    if t == DEC15:
        return dec15_words(rng.integers(-10**15 + 1, 10**15, m).astype(np.int64))
    if t == DEC38:
        return rng.integers(0, 2**63, (m, 2)).astype(np.uint64)
    if t in (D.FLOAT32, D.FLOAT64):
        return rng.standard_normal(m).astype(NP[t])
    info = np.iinfo(NP[t])
    return rng.integers(info.min, info.max, m, endpoint=True).astype(NP[t])


def table(rng, n, off, nulls):
    """[(type, values with `off` leading rows, valid or None)]: a unique Int64 key, the predicate's Int32 column, every kind (with
    bitmaps when `nulls`), and with bitmaps an all-NULL Int32 column and an Int64 column whose bitmap holds no NULL"""
    m = n + off
    specs = [(D.INT64, rng.permutation(m).astype(np.int64) * 3 + 1, None), (D.INT32, rng.integers(0, 1000, m).astype(np.int32), None)]
    specs += [(t, values(rng, t, m), (rng.random(m) > 0.3) if nulls else None) for t in KINDS]
    if nulls:
        specs += [(D.INT32, values(rng, D.INT32, m), np.zeros(m, bool)), (D.INT64, values(rng, D.INT64, m), np.ones(m, bool))]
    return specs


def sources(ctx, specs, off):
    return [Src(ctx, t, v, vv, off) for t, v, vv in specs]


def lookup(ctx, keys, kind):
    """the build side over unique Int64 keys: payload (Int32 key % 1000, Date32 key % 20000) for INNER, a filter for MAYBE"""
    if kind == D.STAGE_MAYBE:
        look = D.Lookup(ctx, D.INT64, [], expected_rows=len(keys), filter_only=True)
    elif kind == D.STAGE_INNER:
        look = D.Lookup(ctx, D.INT64, [D.INT32, D.DATE32])
    else:
        look = D.Lookup(ctx, D.INT64, [])
    inner = kind == D.STAGE_INNER
    b = D.Pipeline(ctx, [D.INT64, D.INT32, D.DATE32] if inner else [D.INT64])
    b.sink_build(look, 0, [1, 2] if inner else [])
    cols = [D.HostColumn(keys)] + ([D.HostColumn((keys % 1000).astype(np.int32)), D.HostColumn((keys % 20000).astype(np.int32), None, D.DATE32)]
                                   if inner else [])
    b.push_host(cols)
    b.finish()
    b.close()
    return look


def drain(p, ncols):
    """the output batches as [(values, valid or None)] per column, and the per-batch row counts and bitmap flags"""
    parts, rows, flags = [[] for _ in range(ncols)], [], []
    for b in p.drain(host=True):
        rows.append(b.num_rows)
        cs = [b.column_numpy(i) for i in range(ncols)]
        flags.append([v is not None for _, v in cs])
        for i, c in enumerate(cs):
            parts[i].append(c)
    out = []
    for i in range(ncols):
        if not parts[i]:
            out.append((None, None))
            continue
        v = np.concatenate([x for x, _ in parts[i]])
        anyv = any(m is not None for _, m in parts[i])
        out.append((v, np.concatenate([np.ones(len(x), bool) if m is None else m for x, m in parts[i]]) if anyv else None))
    return out, rows, flags


def assert_rows(got, exp, ordered, what):
    """exp: [(values, valid or None)]; column 0 is the unique key (the multiset order of the unordered sink)"""
    n = len(exp[0][0])
    if n == 0:
        assert all(v is None or len(v) == 0 for v, _ in got), f"{what}: rows out of nothing"
        return
    assert got[0][0] is not None and len(got[0][0]) == n, f"{what}: {0 if got[0][0] is None else len(got[0][0])} rows, expected {n}"
    go, eo = (np.arange(n), np.arange(n)) if ordered else (np.argsort(got[0][0], kind="stable"), np.argsort(exp[0][0], kind="stable"))
    for c, ((gv, gm), (ev, em)) in enumerate(zip(got, exp)):
        gv, ev = np.ascontiguousarray(gv[go]), np.ascontiguousarray(ev[eo])
        if em is None:
            assert gm is None or gm.all(), f"{what}: column {c} has NULLs"
            assert np.array_equal(gv.view(np.uint8), ev.view(np.uint8)), f"{what}: column {c} values"
        else:
            gm, em = (np.ones(n, bool) if gm is None else gm[go]), em[eo]
            assert np.array_equal(gm, em), f"{what}: column {c} validity"
            assert np.array_equal(gv[em].view(np.uint8), ev[em].view(np.uint8)), f"{what}: column {c} values at valid rows"


def case(ctx, rng, n, off, nulls, shape, frac, ordered, batch_size=0):
    specs = table(rng, n, off, nulls)
    srcs = sources(ctx, specs, off)
    nin = len(specs)
    key = specs[0][1][off:]
    bk = np.unique(np.concatenate([key[rng.random(n) < 0.6], rng.integers(0, 10**6, 1000) * 3 + 2]))   # partners and keys nobody has
    kind = {"pred": None, "semi": D.STAGE_SEMI, "anti": D.STAGE_ANTI, "inner": D.STAGE_INNER, "maybe": D.STAGE_MAYBE, "filter": D.STAGE_INNER,
            "decpred": None}[shape]
    thr = int(round(frac * 1000))
    pred = CMP(DCOL, D.OP_GT, DEC15, 0) if shape == "decpred" else CMP(SEL, D.OP_LT, D.INT32, thr)
    look = lookup(ctx, bk, kind) if kind is not None else None
    p = D.Pipeline(ctx, [t for t, _, _ in specs], pred, [(kind, 0, look)] if look is not None else [])
    try:
        if shape == "filter":
            p.set_stage_filter(0, CMP(nin, D.OP_GT, D.INT32, 500))
        out = list(range(nin)) + ([nin, nin + 1] if kind == D.STAGE_INNER else [])
        p.sink_output(out, batch_size=batch_size, ordered=ordered)
        p.push_device([s.col for s in srcs])
        p.finish()
        got, rows, flags = drain(p, len(out))
    finally:
        p.close()
        if look is not None:
            look.close()
    # the restatement
    if shape == "decpred":
        d = specs[DCOL][1][off:, 0].view(np.int64)
        keep = d > 0 if specs[DCOL][2] is None else (d > 0) & specs[DCOL][2][off:]
    else:
        keep = specs[SEL][1][off:] < thr
    member = np.isin(key, bk)
    if kind in (D.STAGE_SEMI, D.STAGE_INNER):
        keep &= member
    elif kind == D.STAGE_ANTI:
        keep &= ~member
    if shape == "filter":
        keep &= (key % 1000) > 500
    exp = [(v[off:][keep], None if vv is None else vv[off:][keep]) for _, v, vv in specs]
    if kind == D.STAGE_INNER:
        exp += [((key[keep] % 1000).astype(np.int32), None), ((key[keep] % 20000).astype(np.int32), None)]
    what = f"{shape} n={n} off={off} nulls={nulls} frac={frac} ordered={ordered}"
    for f in flags:
        assert f[:nin] == [vv is not None for _, _, vv in specs] and not any(f[nin:]), f"{what}: bitmap flags {f}"
    if batch_size:
        assert all(r == batch_size for r in rows[:-1]) and (not rows or rows[-1] <= batch_size), f"{what}: batch sizes {rows}"
    if kind == D.STAGE_MAYBE:   # the filter has no false negatives: every partner survives, and what survives passed the predicate
        gk = got[0][0] if got[0][0] is not None else np.zeros(0, np.int64)
        assert set(key[keep & member].tolist()) <= set(gk.tolist()) and len(set(gk.tolist())) == len(gk), what
        sub = np.isin(key, gk)
        assert not (sub & ~keep).any(), f"{what}: a row that failed the predicate"
        exp = [(v[off:][sub], None if vv is None else vv[off:][sub]) for _, v, vv in specs]
    assert_rows(got, exp, ordered, what)


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("off", [0, 3, 37])
@pytest.mark.parametrize("shape", ["pred", "semi", "anti", "inner", "filter", "decpred", "maybe"])
def test_every_column_kind_leaves_both_sinks(gpu_ctx, shape, off, ordered):
    if shape == "maybe" and ordered:
        pytest.skip("MAYBE stages feed an exchange: the unordered sink")
    case(gpu_ctx, np.random.default_rng(100 * off + len(shape) + ordered), 5000, off, True, shape, 0.5, ordered)


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("shape", ["pred", "semi", "inner", "filter", "decpred"])
def test_columns_without_bitmaps_next_to_16_byte_ones(gpu_ctx, shape, ordered):
    case(gpu_ctx, np.random.default_rng(7 + len(shape) + ordered), 20_000, 0, False, shape, 0.5, ordered)


@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("frac", [0.0, 0.01, 0.5, 1.0])
@pytest.mark.parametrize("n", [700, 100_003, 3_000_000])
def test_survivor_fractions_and_sizes(gpu_ctx, n, frac, ordered):
    case(gpu_ctx, np.random.default_rng(n + int(frac * 100) + ordered), n, 3, True, "inner", frac, ordered)


@pytest.mark.parametrize("ordered", [True, False])
def test_pushes_mixing_bitmaps_and_batch_size_slicing(gpu_ctx, ordered):
    """three pushes (bitmaps at offset 37, none, bitmaps at offset 3): the output columns merge them, sliced into 1000-row batches"""
    rng = np.random.default_rng(41 + ordered)
    batches = [(table(rng, 30_011, 37, True), 37), (table(rng, 20_000, 0, False), 0), (table(rng, 9_999, 3, True), 3)]
    for i, (specs, _) in enumerate(batches):   # keys unique over all pushes
        specs[0] = (D.INT64, specs[0][1] + np.int64(10**8 * i), None)
    types = [t for t, _, _ in batches[0][0]][:2 + len(KINDS)]
    p = D.Pipeline(gpu_ctx, types, CMP(SEL, D.OP_LT, D.INT32, 700))
    keep_alive, exp = [], []
    try:
        p.sink_output(list(range(len(types))), batch_size=1000, ordered=ordered)
        for specs, off in batches:
            specs = specs[:len(types)]
            srcs = sources(gpu_ctx, specs, off)
            keep_alive.append(srcs)
            p.push_device([s.col for s in srcs])
            keep = specs[SEL][1][off:] < 700
            exp.append([(v[off:][keep], (np.ones(keep.sum(), bool) if vv is None else vv[off:][keep])) for _, v, vv in specs])
        p.finish()
        got, rows, flags = drain(p, len(types))
    finally:
        p.close()
    merged = [(np.concatenate([e[c][0] for e in exp]), np.concatenate([e[c][1] for e in exp])) for c in range(len(types))]
    merged = [(v, None if c < 2 else m) for c, (v, m) in enumerate(merged)]
    assert all(r == 1000 for r in rows[:-1]) and 0 < rows[-1] <= 1000, rows
    assert all(f == [False, False] + [True] * len(KINDS) for f in flags), "every batch carries the merged bitmaps"
    assert_rows(got, merged, ordered, f"mixed pushes ordered={ordered}")


def test_decimal_lineitem_scan_through_the_local_exchange_is_q3(gpu_ctx):
    """the multi-GPU plan's data path on one GPU: the lineitem scan (l_shipdate > cut, MAYBE on the orders filter) -> unordered output of
    l_orderkey and Decimal128 l_extendedprice / l_discount (nullable) -> dfgpu_hash_partition_device -> per partition an INNER stage on
    the partition's orders + the join-keyed aggregate SUM(l_extendedprice * (1 - l_discount)) == pandas' Q3 over the same data"""
    from decimal_util import gpu_nodes
    from test_gpu_pipe_decimal_aggs import REV
    ctx, rng = gpu_ctx, np.random.default_rng(3)
    no, nl, cut, P = 60_000, 400_000, 9200, 5
    okey = rng.permutation(no * 4)[:no].astype(np.int64) + 1
    odate = rng.integers(8000, 10500, no).astype(np.int32); oprio = rng.integers(0, 3, no).astype(np.int32)
    osel = odate < cut                                                    # the orders side's own filter
    lkey = np.where(rng.random(nl) < 0.8, okey[rng.integers(0, no, nl)], rng.integers(1, no * 4, nl)).astype(np.int64)
    price = rng.integers(90_000, 10_500_000, nl).astype(np.int64); disc = rng.integers(0, 11, nl).astype(np.int64)
    pvalid = rng.random(nl) > 0.02
    ship = rng.integers(8000, 10600, nl).astype(np.int32)
    filt = D.Lookup(ctx, D.INT64, [], expected_rows=int(osel.sum()), filter_only=True)
    b = D.Pipeline(ctx, [D.INT64]); b.sink_build(filt, 0, []); b.push_host([D.HostColumn(okey[osel])]); b.finish(); b.close()
    p = D.Pipeline(ctx, [D.INT64, DEC15, DEC15, D.DATE32], CMP(3, D.OP_GT, D.DATE32, cut), [(D.STAGE_MAYBE, 0, filt)])
    p.sink_output([0, 1, 2], ordered=False)
    p.push_host([D.HostColumn(lkey), D.HostColumn(dec15_words(price), pvalid, DEC15), D.HostColumn(dec15_words(disc), None, DEC15),
                 D.HostColumn(ship, None, D.DATE32)])
    p.finish()
    outs = p.drain(host=False)
    assert len(outs) == 1 and outs[0].column(1).validity and not outs[0].column(0).validity
    lparts, loffs = D.hash_partition_device(ctx, [outs[0].column(i) for i in range(3)], [0], P)
    for o in outs:
        o.release()
    p.close(); filt.close()
    oc = [D.DeviceColumn.from_host(ctx, h) for h in (D.HostColumn(okey[osel]), D.HostColumn(odate[osel], None, D.DATE32), D.HostColumn(oprio[osel]))]
    oparts, ooffs = D.hash_partition_device(ctx, [c.c() for c in oc], [0], P)

    def part(batch, offs, q, i):
        c = batch.column(i)
        s = D.Column()
        s.type, s.flags, s.length, s.offset, s.null_count = c.type, 0, offs[q + 1] - offs[q], c.offset + offs[q], (-1 if c.validity else 0)
        s.values, s.validity = c.values, c.validity
        return s

    rows = []
    for q in range(P):
        look = D.Lookup(ctx, D.INT64, [D.DATE32, D.INT32], n_acc_words=4)
        b = D.Pipeline(ctx, [D.INT64, D.DATE32, D.INT32]); b.sink_build(look, 0, [1, 2])
        b.push_device([part(oparts, ooffs, q, i) for i in range(3)]); b.finish(); b.close()
        a = D.Pipeline(ctx, [D.INT64, DEC15, DEC15], None, [(D.STAGE_INNER, 0, look)])
        a.sink_aggregate([0, 3, 4], [(D.AGG_SUM, gpu_nodes(D, REV))])
        if loffs[q + 1] > loffs[q]:
            a.push_device([part(lparts, loffs, q, i) for i in range(3)])
        a.finish()
        for ob in a.drain(host=True):
            k, dt, pr = (ob.column_numpy(i)[0] for i in range(3))
            sv, sm = ob.column_numpy(3)
            rev = D.words_to_decimal(sv)
            rows += [(int(k[i]), int(dt[i]), int(pr[i]), rev[i]) for i in range(len(k)) if sm is None or sm[i]]
        a.close(); look.close()
    lparts.release(); oparts.release()
    li = pd.DataFrame({"k": lkey, "price": price, "disc": disc, "pv": pvalid, "ship": ship})
    od = pd.DataFrame({"k": okey[osel], "date": odate[osel], "prio": oprio[osel]})
    j = li[(li.ship > cut) & li.pv].merge(od, on="k")
    j["rev"] = [int(x) * (100 - int(y)) for x, y in zip(j.price, j.disc)]     # Decimal128(15,2) * (1 - Decimal128(15,2)) at scale 4
    want = {(int(k), int(d), int(pr)): int(r) for (k, d, pr), r in j.groupby(["k", "date", "prio"])["rev"].sum().items()}
    assert len(rows) == len(want) and dict(((k, d, pr), r) for k, d, pr, r in rows) == want


def _twin_tables(rng, n, nc):
    ck = rng.permutation(nc * 2)[:nc].astype(np.int64)
    cust = pa.record_batch([pa.array(ck), pa.array(rng.integers(0, 25, nc).astype(np.int32))],
                           schema=pa.schema([pa.field("c_custkey", pa.int64(), False), pa.field("c_nation", pa.int32(), False)]))
    price = [None if rng.random() < 0.1 else Decimal(int(x)).scaleb(-2) for x in rng.integers(-10**9, 10**9, n)]
    okey = rng.permutation(n).astype(np.int64)
    ocust = pa.array(rng.integers(0, nc * 2, n).astype(np.int64), mask=rng.random(n) < 0.05)
    odate = pa.array(rng.integers(8000, 10500, n).astype(np.int32), mask=rng.random(n) < 0.1).cast(pa.date32())
    big = [Decimal(int(x)).scaleb(-4) for x in rng.integers(-2**62, 2**62, n)]
    sch = pa.schema([pa.field("o_orderkey", pa.int64(), False), pa.field("o_custkey", pa.int64()), pa.field("o_totalprice", pa.decimal128(15, 2)),
                     pa.field("o_orderdate", pa.date32()), pa.field("o_big", pa.decimal128(38, 4))])
    orders = pa.record_batch([pa.array(okey), ocust, pa.array(price, pa.decimal128(15, 2)), odate, pa.array(big, pa.decimal128(38, 4))], schema=sch)
    step = 7000
    return MemoryExec([cust]), MemoryExec([orders.slice(s, step) for s in range(0, n, step)], sch)


@pytest.mark.parametrize("join_type", ["Inner", "RightSemi", "RightAnti"])
def test_twin_fused_output_equals_the_unfused_joins(gpu_ctx, task_ctx, join_type):
    rng = np.random.default_rng(len(join_type))
    cust, orders = _twin_tables(rng, 50_000, 4000)
    probe = GpuFilterExec(col("o_orderdate") < lit(9500, pa.date32()), orders)
    join = GpuHashJoinExec(cust, probe, [("c_custkey", "o_custkey")], join_type)
    names = ["o_orderkey", "o_totalprice", "o_orderdate", "o_big"] + (["c_nation", "c_custkey"] if join_type == "Inner" else [])
    plans = [join, GpuProjectionExec([(Column(n), n) for n in names], join)]
    for plan in plans:
        fused = fuse_output_pipelines(plan)
        assert isinstance(fused, GpuPipelineExec) and fused.sink == "output"
        got, exp = pa.Table.from_batches(collect(fused, task_ctx)), pa.Table.from_batches(collect(plan, task_ctx))
        assert got.num_rows == exp.num_rows > 0
        assert got.column_names == exp.column_names
        for c in got.column_names:
            assert got.column(c).to_pylist() == exp.column(c).to_pylist(), (join_type, c)
        assert "fallback" not in fused.metrics() and fused.metrics()["output_rows"] == got.num_rows


def test_twin_falls_back_to_the_unfused_join_on_duplicate_build_keys(gpu_ctx, task_ctx):
    """duplicate customer keys: the fused lookup refuses them at the build, before any row is emitted, and the unfused join runs"""
    rng = np.random.default_rng(17)
    cust, orders = _twin_tables(rng, 20_000, 3000)
    cb = cust.batches[0]
    dup = pa.record_batch([pa.concat_arrays([cb.column(0), cb.column(0).slice(0, 100)]), pa.concat_arrays([cb.column(1), cb.column(1).slice(0, 100)])],
                          schema=cb.schema)
    plan = GpuHashJoinExec(MemoryExec([dup]), orders, [("c_custkey", "o_custkey")], "Inner")
    fused = fuse_output_pipelines(plan)
    assert isinstance(fused, GpuPipelineExec) and fused.sink == "output"
    got, exp = pa.Table.from_batches(collect(fused, task_ctx)), pa.Table.from_batches(collect(plan, task_ctx))
    assert "duplicate build keys" in fused.metrics()["fallback"]
    assert got.num_rows == exp.num_rows > 0 and got.column_names == exp.column_names
    for c in got.column_names:
        assert got.column(c).to_pylist() == exp.column(c).to_pylist(), c


@pytest.mark.parametrize("ordered", [True, False])
def test_decimal128_columns_from_8_byte_aligned_buffers(gpu_ctx, ordered):
    """Arrow promises 8-byte alignment only: Decimal128 inputs whose buffers start 8 bytes past a 16-byte boundary (one with a bitmap
    at bit offset 5) leave both sinks through the two-load path"""
    rng = np.random.default_rng(5 + ordered)
    n, off = 50_001, 5
    key = rng.permutation(n).astype(np.int64)
    sel = rng.integers(0, 1000, n).astype(np.int32)
    d15, d38 = values(rng, DEC15, n + off), values(rng, DEC38, n)
    valid = rng.random(n + off) > 0.3
    keep = []

    def shifted(t, vals, valid, off):
        buf = gpu_ctx.to_device(np.concatenate([np.zeros(8, np.uint8), np.ascontiguousarray(vals).view(np.uint8).ravel()]))
        keep.append(buf)
        c = D.Column()
        c.type, c.flags, c.length, c.offset, c.null_count = t, 0, len(vals) - off, off, (-1 if valid is not None else 0)
        c.values = buf.ptr + 8
        if valid is not None:
            vb = gpu_ctx.to_device(D.pack_bits(valid))
            keep.append(vb)
            c.validity = vb.ptr
        assert (c.values + 16 * off) % 16 == 8
        return c

    plain = [Src(gpu_ctx, D.INT64, key, None, 0), Src(gpu_ctx, D.INT32, sel, None, 0)]
    cols = [plain[0].col, plain[1].col, shifted(DEC15, d15, valid, off), shifted(DEC38, d38, None, 0)]
    p = D.Pipeline(gpu_ctx, [D.INT64, D.INT32, DEC15, DEC38], CMP(1, D.OP_LT, D.INT32, 500))
    try:
        p.sink_output([0, 2, 3], ordered=ordered)
        p.push_device(cols)
        p.finish()
        got, _, flags = drain(p, 3)
    finally:
        p.close()
    m = sel < 500
    assert all(f == [False, True, False] for f in flags)
    assert_rows(got, [(key[m], None), (d15[off:][m], valid[off:][m]), (d38[m], None)], ordered, f"8-byte aligned ordered={ordered}")
