"""TPC-H Q9's lineitem x partsupp step on its two-column key, fused (composite key packed into the fused lookup's 64-bit key) against the
unfused operators it replaces, device resident.

    lineitem (SF x 6,000,000 rows: l_partkey, l_suppkey, l_quantity, l_extendedprice, l_discount, Int64 money)
      JOIN partsupp (SF x 800,000 rows: ps_partkey, ps_suppkey, ps_supplycost) ON (l_partkey, l_suppkey) = (ps_partkey, ps_suppkey)
      WHERE l_quantity < 50
      GROUP BY l_suppkey: SUM(l_extendedprice * (100 - l_discount) - ps_supplycost * l_quantity)
    fused   : partsupp -> dfgpu_pipeline_sink_build_composite (key domain [1, SF x 200,000] x [1, SF x 10,000]);
              lineitem -> INNER stage on the packed (l_partkey, l_suppkey) -> hash-keyed aggregate sink.  Each push first runs the
              packing pass ("pipe_keys:<name>"), then the pipeline kernel.
    unfused : dfgpu_filter -> dfgpu_hashjoin on the two Int64 keys (its wide-key path: a hidden hash column, equality as a JoinFilter
              conjunct, every joined row materialised) -> the profit expression (dfgpu_expr_evaluate_device) -> dfgpu_agg, in 2^26-row
              lineitem slices.
Q9 filters part, not lineitem; the predicate (98 % of the rows pass it) keeps the unfused chain's dfgpu_filter in the shape.

Keys follow the TPC-H generator: ps_suppkey = (ps_partkey + j (S / 4 + (ps_partkey - 1) / S)) % S + 1 for j = 0..3, and l_suppkey is one
of its part's four suppliers, so every lineitem row has exactly one partsupp partner.  Data come from the counter-based generators.
Both arms build their side inside the timer.  The arms alternate after a warm-up; each time is a host clock around work that ends in a
device synchronise.  Every run checks that the two arms return the same groups, group by group.  A last, separate run with kernel
timing on reports the packing pass (and its achieved bandwidth: 16 B read and 8 B written per row, against 3.35 TB/s) and the
pipeline kernel.

usage: python scripts/pipe_composite_key_timing.py [SF=100] [rounds=5]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from datafusion_b200 import capi as D

C = lambda i: (D.EXPR_COLUMN, i, 0, 0, 0, 0.0)                                # noqa: E731
L = lambda v, t=D.INT64: (D.EXPR_LITERAL, 0, t, 0, v, 0.0)                   # noqa: E731
B = lambda op: (D.EXPR_BINARY, op, 0, 0, 0, 0.0)                              # noqa: E731
I64 = D.INT64
PRED = [C(2), L(50), B(D.OP_LT)]
PROFIT_FUSED = [C(3), L(100), C(4), B(D.OP_MINUS), B(D.OP_MULTIPLY), C(5), C(2), B(D.OP_MULTIPLY), B(D.OP_MINUS)]   # payload field 5
# the join's output: l_suppkey, l_quantity, l_extendedprice, l_discount, ps_supplycost
PROFIT_UNFUSED = [C(2), L(100), C(3), B(D.OP_MINUS), B(D.OP_MULTIPLY), C(4), C(1), B(D.OP_MULTIPLY), B(D.OP_MINUS)]
SLICE = 1 << 26
HBM = 3.35e12


def dcol(buf, n, off=0):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count = I64, 0, n, 0, 0
    c.values, c.validity = buf.ptr + 8 * off, None
    return c


def suppkey(ctx, keep, pk, j, n, s):
    """(pk + j (S / 4 + (pk - 1) / S)) % S + 1"""
    nodes = [C(0), C(1), L(s // 4), C(0), L(1), B(D.OP_MINUS), L(s), B(D.OP_DIVIDE), B(D.OP_PLUS), B(D.OP_MULTIPLY), B(D.OP_PLUS),
             L(s), B(D.OP_MODULO), L(1), B(D.OP_PLUS)]
    b = D.evaluate_device(ctx, [dcol(pk, n), dcol(j, n)], n, nodes)
    keep.append(b)
    return b.column(0)


def gen(ctx, sf, seed=9):
    nparts, nsupp = int(200_000 * sf), int(10_000 * sf)
    nps, nl = 4 * nparts, int(6_000_000 * sf)
    keep = []
    g = lambda k, lo, hi, n: ctx.generate_i64(D.GEN_UNIFORM, seed + k, lo, hi - lo + 1, 0, n)   # noqa: E731  values in [lo, hi]
    i = ctx.generate_i64(D.GEN_SEQ, 0, 0, 0, 0, nps)
    pk = D.evaluate_device(ctx, [dcol(i, nps)], nps, [C(0), L(4), B(D.OP_DIVIDE), L(1), B(D.OP_PLUS)])
    j = D.evaluate_device(ctx, [dcol(i, nps)], nps, [C(0), L(4), B(D.OP_MODULO)])
    keep += [pk]
    pkc = pk.column(0)
    jc = j.column(0)
    sk = D.evaluate_device(ctx, [pkc, jc], nps, [C(0), C(1), L(nsupp // 4), C(0), L(1), B(D.OP_MINUS), L(nsupp), B(D.OP_DIVIDE), B(D.OP_PLUS),
                                                 B(D.OP_MULTIPLY), B(D.OP_PLUS), L(nsupp), B(D.OP_MODULO), L(1), B(D.OP_PLUS)])
    cost = g(1, 100, 100_000, nps)
    keep += [sk, cost]
    del i, j
    partsupp = [pkc, sk.column(0), dcol(cost, nps)]
    lpk, lj = g(2, 1, nparts, nl), g(3, 0, 3, nl)
    lsk = suppkey(ctx, keep, lpk, lj, nl, nsupp)
    del lj
    qty, price, disc = g(4, 1, 50, nl), g(5, 90_000, 10_500_000, nl), g(6, 0, 10, nl)
    keep += [lpk, qty, price, disc]
    lineitem_bufs = [lpk, lsk, qty, price, disc]
    ctx.sync()
    return partsupp, lineitem_bufs, nl, nparts, nsupp, keep


def lineitem_cols(bufs, n, off=0):
    """device columns of rows [off, off + n); the l_suppkey column is a batch column (already a Column)"""
    out = []
    for b in bufs:
        if isinstance(b, D.Column):
            c = D.Column()
            c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = b.type, 0, n, 0, 0, b.values + 8 * off, None
            out.append(c)
        else:
            out.append(dcol(b, n, off))
    return out


def fused(ctx, partsupp, li, nl, nparts, nsupp, times):
    t0 = time.perf_counter()
    look = D.Lookup(ctx, key_types=[I64, I64], key_ranges=[(1, nparts), (1, nsupp)], payload_types=[I64], expected_rows=4 * nparts)
    b = D.Pipeline(ctx, [I64] * 3, name="partsupp")
    b.sink_build(look, key_cols=[0, 1], payload_cols=[2])
    b.push_device(partsupp)
    b.finish()
    b.close()
    ctx.sync()
    times.append((time.perf_counter() - t0) * 1e3)
    p = D.Pipeline(ctx, [I64] * 5, PRED, [(D.STAGE_INNER, [0, 1], look)], name="lineitem")
    p.sink_aggregate_hash([1], [(D.AGG_SUM, PROFIT_FUSED)], capacity_hint=nsupp)
    p.push_device(lineitem_cols(li, nl))
    p.finish()
    out = p.drain(host=False)
    p.close()
    look.close()
    return out


def unfused(ctx, partsupp, li, nl, nsupp):
    j = D.HashJoinHandle(ctx, [I64] * 3, [I64] * 5, [0, 1], [0, 1], [1, 1, 1, 1, 0], [1, 2, 3, 4, 2], D.JOIN_INNER, batch_size=1 << 30,
                         ordered_output=False)
    f = D.FilterHandle(ctx, [I64] * 5, PRED, batch_size=SLICE)
    a = D.AggHandle(ctx, [I64, I64], [0], [(D.AGG_SUM, 1, -1)], D.AGG_SINGLE, batch_size=1 << 30, capacity_hint=nsupp)

    def aggregate():   # the joined rows so far -> profit -> the group-by
        for jb in j.drain(host=False):
            cols = [jb.column(i) for i in range(5)]
            amt = D.evaluate_device(ctx, cols, jb.num_rows, PROFIT_UNFUSED)
            a.push_device([cols[0], amt.column(0)])
            amt.release()
            jb.release()

    def probe():       # the filtered rows so far -> the join
        for fb in f.drain(host=False):
            j.push_probe_device([fb.column(i) for i in range(5)])
            aggregate()
            fb.release()

    try:
        j.push_build_device(partsupp)
        j.finish_build()
        for off in range(0, nl, SLICE):
            f.push_device(lineitem_cols(li, min(SLICE, nl - off), off))
            probe()
        f.finish()
        probe()
        j.finish_probe()
        aggregate()
        a.finish()
        return a.drain(host=False)
    finally:
        a.close(); f.close(); j.close()


def groups(out):
    ks, vs = [], []
    for b in out:
        k, _ = b.column_numpy(0)
        v, _ = b.column_numpy(1)
        ks.append(k); vs.append(v)
        b.release()
    k, v = np.concatenate(ks), np.concatenate(vs)
    o = np.argsort(k, kind="stable")
    return k[o], v[o]


def timed(ctx, fn):
    ctx.sync()
    t0 = time.perf_counter()
    r = fn()
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    ctx = D.Context(0)
    partsupp, li, nl, nparts, nsupp, keep = gen(ctx, sf)
    build_ms = []
    arms = {"fused": lambda: fused(ctx, partsupp, li, nl, nparts, nsupp, build_ms), "unfused": lambda: unfused(ctx, partsupp, li, nl, nsupp)}
    for fn in arms.values():   # warm-up
        groups(fn())
    build_ms.clear()
    times = {k: [] for k in arms}
    n_groups = 0
    for _ in range(rounds):
        res = {}
        for name, fn in arms.items():
            ms, out = timed(ctx, fn)
            times[name].append(ms)
            res[name] = groups(out)
        (fk, fv), (uk, uv) = res["fused"], res["unfused"]
        assert np.array_equal(fk, uk) and np.array_equal(fv, uv), "fused and unfused groups differ"
        n_groups = len(fk)
    # kernel families, in a run of their own
    ctx.set_kernel_timing(True)
    ctx.kernel_time_reset()
    kb = []
    groups(fused(ctx, partsupp, li, nl, nparts, nsupp, kb))
    kern = {name: ctx.kernel_time(name) for name in ("pipe_keys:lineitem", "pipe:lineitem", "pipe_keys:partsupp", "pipe:partsupp",
                                                      "lookup_partition", "lookup_insert")}
    ctx.set_kernel_timing(False)
    keys_ms = kern["pipe_keys:lineitem"][0]
    summary = {
        "sf": sf, "rounds": rounds, "card": card, "lineitem_rows": nl, "partsupp_rows": 4 * nparts, "groups": n_groups, "equal": True,
        "median_ms": {k: float(np.median(v)) for k, v in times.items()},
        "range_ms": {k: [float(min(v)), float(max(v))] for k, v in times.items()},
        "all_ms": times,
        "fused_partsupp_build_ms": {"median": float(np.median(build_ms)), "range": [float(min(build_ms)), float(max(build_ms))]},
        "kernel_ms": {k: v[0] for k, v in kern.items()},
        "pipe_keys_lineitem_bytes_per_s": nl * 24 / (keys_ms * 1e-3) if keys_ms > 0 else None,
        "pipe_keys_lineitem_share_of_3_35_TBps": nl * 24 / (keys_ms * 1e-3) / HBM if keys_ms > 0 else None,
    }
    print(json.dumps(summary), flush=True)
    del keep


if __name__ == "__main__":
    main()
