"""Joins with a JoinFilter through the fused pipeline's stage filters against the unfused GPU chain, device resident.

    Q19: lineitem JOIN part ON p_partkey = l_partkey AND (three-way OR of conjunctions over p_brand, p_container, p_size, l_quantity),
         (l_shipmode = 1 OR l_shipmode = 3) AND l_shipinstruct = 0 on lineitem, SUM(l_extendedprice * (100 - l_discount)), no GROUP BY.
         SF x 6,000,000 lineitem rows, SF x 200,000 parts; brand, container, ship mode and ship instruct are Int8 codes, size Int16
         (IN lists written as ORs of equalities).
        fused   : part build pipeline -> lookup {p_partkey -> brand, container, size}; lineitem pipeline with the predicate, an INNER stage
                  carrying the OR filter, the dense sink without GROUP BY
        unfused : dfgpu_filter -> dfgpu_hashjoin(Inner, set_filter) -> revenue expression -> dfgpu_agg grouped on a zero column.  The
                  hash join's filter takes at most 48 nodes and the OR has 107, so the unfused chain runs the three arms, which are disjoint
                  (each names its own brand), as three filtered joins over the same filtered lineitem, each built from the parts of its brand
                  (dfgpu_filter), into one aggregate
    Q17: lineitem JOIN (part WHERE p_brand = 3 AND p_container = 5) JOIN (AVG(l_quantity) per partkey) ON partkey
         AND CAST(l_quantity AS Float64) < 0.2 * avg, SUM(l_extendedprice).  The AVG build (dfgpu_agg over lineitem) is common to both arms
         and timed on its own.
        fused   : a SEMI stage on the filtered part key set, an INNER stage on {partkey -> avg} with the filter, the dense sink
        unfused : dfgpu_filter(part) -> dfgpu_hashjoin(Inner) -> dfgpu_hashjoin(Inner, set_filter) -> dfgpu_agg grouped on a zero column

Data come from the counter-based generators (dfgpu_generate_i64); the narrow codes are cast on the device.  Fused and unfused runs
alternate in one process after a warm-up; each time is a host clock around work that ends in a device synchronise.  Checks, on every run:
SUM and the number of joined rows of the fused plan equal the unfused plan's exactly.

usage: python scripts/pipe_join_filter_timing.py [SF=100] [steps=3]"""
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
CAST = lambda t: (D.EXPR_CAST, 0, t, 0, 0, 0.0)                               # noqa: E731
I8 = lambda v: L(v, D.INT8)                                                   # noqa: E731
# Q19's three arms: (brand, containers, quantity lo, quantity hi, max size)
ARMS = [(12, [0, 1, 2, 3], 1, 11, 5), (23, [10, 11, 12, 13], 10, 20, 10), (9, [20, 21, 22, 23], 20, 30, 15)]
Q17_BRAND, Q17_CONTAINER = 3, 5


# ---- the exact check (host side; tests/test_pipe_join_filter_timing_checks.py runs it on tiny data) ----
def check_sum(name, fused, unfused) -> dict:
    """fused / unfused: (SUM, joined rows).  Raises on any difference."""
    assert fused == unfused, f"{name}: fused {fused} != unfused {unfused}"
    return {"sum": fused[0], "rows": fused[1]}


# ---- filters as RPN over a stage's columns: cols maps the names to column indices ----
def eq_any(c, vals):
    out = [C(c), I8(vals[0]), B(D.OP_EQ)]
    for v in vals[1:]:
        out += [C(c), I8(v), B(D.OP_EQ), B(D.OP_OR)]
    return out


def q19_arm(qty, brand, cont, size, b, conts, qlo, qhi, smax):
    return ([C(brand), I8(b), B(D.OP_EQ)] + eq_any(cont, conts) + [B(D.OP_AND), C(qty), L(qlo), B(D.OP_GTEQ), B(D.OP_AND),
            C(qty), L(qhi), B(D.OP_LTEQ), B(D.OP_AND), C(size), L(1, D.INT16), B(D.OP_GTEQ), B(D.OP_AND), C(size), L(smax, D.INT16),
            B(D.OP_LTEQ), B(D.OP_AND)])


def q19_filter(qty, brand, cont, size):
    arm = lambda *a: q19_arm(qty, brand, cont, size, *a)  # noqa: E731
    return arm(*ARMS[0]) + arm(*ARMS[1]) + [B(D.OP_OR)] + arm(*ARMS[2]) + [B(D.OP_OR)]


def q17_filter(qty, avg):
    return [C(qty), CAST(D.FLOAT64), (D.EXPR_LITERAL, 0, D.FLOAT64, 0, 0, 0.2), C(avg), B(D.OP_MULTIPLY), B(D.OP_LT)]


# ---- device side ----
def dcol(buf, n, t=D.INT64):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = t, 0, n, 0, 0, buf.ptr, None
    return c


def narrow(ctx, keep, buf, n, t):
    """an Int64 device column cast to t on the device (the batch stays alive in keep)"""
    b = D.evaluate_device(ctx, [dcol(buf, n)], n, [C(0), CAST(t)])
    keep.append(b)
    return b.column(0)


def gen(ctx, sf, seed=19):
    n_li, n_part = int(6_000_000 * sf), int(200_000 * sf)
    keep = []
    g = lambda k, lo, hi, n: ctx.generate_i64(D.GEN_UNIFORM, seed + k, lo, hi, 0, n)  # noqa: E731
    lpk, qty, price, disc = g(1, 1, n_part, n_li), g(2, 1, 50, n_li), g(3, 90_000, 10_500_000, n_li), g(4, 0, 10, n_li)
    keep += [lpk, qty, price, disc]
    mode, instr = g(5, 0, 6, n_li), g(6, 0, 3, n_li)
    lineitem = [dcol(lpk, n_li), dcol(qty, n_li), dcol(price, n_li), dcol(disc, n_li), narrow(ctx, keep, mode, n_li, D.INT8),
                narrow(ctx, keep, instr, n_li, D.INT8)]
    del mode, instr
    pkey = ctx.to_device(np.arange(1, n_part + 1, dtype=np.int64))
    keep.append(pkey)
    brand, cont, size = g(7, 0, 24, n_part), g(8, 0, 39, n_part), g(9, 1, 50, n_part)
    part = [dcol(pkey, n_part), narrow(ctx, keep, brand, n_part, D.INT8), narrow(ctx, keep, cont, n_part, D.INT8), narrow(ctx, keep, size, n_part, D.INT16)]
    del brand, cont, size
    ctx.sync()
    return lineitem, part, keep


LI_TYPES = [D.INT64, D.INT64, D.INT64, D.INT64, D.INT8, D.INT8]   # partkey, quantity, extendedprice, discount, shipmode, shipinstruct
PART_TYPES = [D.INT64, D.INT8, D.INT8, D.INT16]                   # partkey, brand, container, size
LI_PRED = [C(4), I8(1), B(D.OP_EQ), C(4), I8(3), B(D.OP_EQ), B(D.OP_OR), C(5), I8(0), B(D.OP_EQ), B(D.OP_AND)]
REVENUE = [C(2), L(100), C(3), B(D.OP_MINUS), B(D.OP_MULTIPLY)]


def dense_result(p):
    """(SUM, COUNT(*)) of a dense sink without GROUP BY; SUM NULL (no row) as 0"""
    out = p.drain(host=True)
    s, v = out[0].column_numpy(0)
    n = int(out[0].column_numpy(1)[0][0])
    return (0 if (v is not None and not v[0]) else int(s[0])), n


def q19_fused(ctx, lineitem, part):
    look = D.Lookup(ctx, D.INT64, [D.INT8, D.INT8, D.INT16], expected_rows=part[0].length)
    bp = D.Pipeline(ctx, PART_TYPES)
    bp.sink_build(look, 0, [1, 2, 3]); bp.push_device(part); bp.finish(); bp.close()
    p = D.Pipeline(ctx, LI_TYPES, LI_PRED, [(D.STAGE_INNER, 0, look)], name="q19")
    p.set_stage_filter(0, q19_filter(1, 6, 7, 8))                # virtual columns: lineitem 0..5, then brand 6, container 7, size 8
    p.sink_aggregate_dense([], [], [(D.AGG_SUM, REVENUE), (D.AGG_COUNT_STAR, None)])
    p.push_device(lineitem); p.finish()
    r = dense_result(p)
    p.close(); look.close()
    return r


def zero_sum_agg(ctx, value_type=D.INT64):
    return D.AggHandle(ctx, [D.INT64, value_type], [0], [(D.AGG_SUM, 1, -1), (D.AGG_COUNT_STAR, -1, -1)], D.AGG_SINGLE, 1 << 30, 4)


def agg_result(agg):
    agg.finish()
    out = agg.drain(host=True)
    agg.close()
    if not out or out[0].num_rows == 0:
        return 0, 0
    return int(out[0].column_numpy(1)[0][0]), int(out[0].column_numpy(2)[0][0])


def push_zero_grouped(ctx, agg, col, value):
    """agg.push([0, value]): the zero column is col * 0, evaluated on the device"""
    z = D.evaluate_device(ctx, [col], col.length, [C(0), L(0), B(D.OP_MULTIPLY)])
    agg.push_device([z.column(0), value])
    z.release()


def q19_unfused(ctx, lineitem, part):
    f = D.FilterHandle(ctx, LI_TYPES, LI_PRED, [0, 1, 2, 3], batch_size=0)     # partkey, quantity, price, discount
    f.push_device(lineitem); f.finish()
    fl = f.drain(host=False)
    f.close()
    agg = zero_sum_agg(ctx)
    for arm in ARMS:
        pf = D.FilterHandle(ctx, PART_TYPES, [C(1), I8(arm[0]), B(D.OP_EQ)], None, batch_size=0)   # the parts of this arm's brand
        pf.push_device(part); pf.finish()
        fp = pf.drain(host=False)
        pf.close()
        j = D.HashJoinHandle(ctx, PART_TYPES, [D.INT64] * 4, [0], [0], [1, 1, 1], [0, 2, 3], D.JOIN_INNER, batch_size=1 << 28, ordered_output=False)
        # the JoinFilter's columns: probe quantity, build brand, container, size
        j.set_filter([1, 0, 0, 0], [1, 1, 2, 3], q19_arm(0, 1, 2, 3, *arm))
        for b in fp:
            j.push_build_device([b.column(i) for i in range(4)])
        j.finish_build()

        def consume(batches):
            for jb in batches:
                n = jb.num_rows
                rev = D.evaluate_device(ctx, [jb.column(0), jb.column(0), jb.column(1), jb.column(2)], n, REVENUE)
                push_zero_grouped(ctx, agg, jb.column(0), rev.column(0))
                rev.release(); jb.release()
        for b in fl:
            j.push_probe_device([b.column(i) for i in range(4)])
            consume(j.drain(host=False))
        j.finish_probe()
        consume(j.drain(host=False))
        j.close()
        for b in fp:
            b.release()
    for b in fl:
        b.release()
    return agg_result(agg)


def avg_build(ctx, lineitem):
    """AVG(l_quantity) per partkey (common to both Q17 arms): device batches [partkey, avg]"""
    n_part = int(lineitem[0].length // 30)
    agg = D.AggHandle(ctx, [D.INT64, D.INT64], [0], [(D.AGG_AVG, 1, -1)], D.AGG_SINGLE, 1 << 30, n_part)
    agg.push_device([lineitem[0], lineitem[1]]); agg.finish()
    out = agg.drain(host=False)
    agg.close()
    return out


def q17_fused(ctx, lineitem, part, avg):
    keys = D.Lookup(ctx, D.INT64, [])
    kp = D.Pipeline(ctx, PART_TYPES, [C(1), I8(Q17_BRAND), B(D.OP_EQ), C(2), I8(Q17_CONTAINER), B(D.OP_EQ), B(D.OP_AND)])
    kp.sink_build(keys, 0, []); kp.push_device(part); kp.finish(); kp.close()
    al = D.Lookup(ctx, D.INT64, [D.FLOAT64], expected_rows=sum(b.num_rows for b in avg))
    ap = D.Pipeline(ctx, [D.INT64, D.FLOAT64])
    ap.sink_build(al, 0, [1])
    for b in avg:
        a = b.column(1)
        a.validity, a.null_count = None, 0                        # every group has a quantity: no AVG is NULL
        ap.push_device([b.column(0), a])
    ap.finish(); ap.close()
    p = D.Pipeline(ctx, LI_TYPES[:3], None, [(D.STAGE_SEMI, 0, keys), (D.STAGE_INNER, 0, al)], name="q17")
    p.set_stage_filter(1, q17_filter(1, 3))                       # virtual columns: partkey, quantity, price, then avg 3
    p.sink_aggregate_dense([], [], [(D.AGG_SUM, [C(2)]), (D.AGG_COUNT_STAR, None)])
    p.push_device(lineitem[:3]); p.finish()
    r = dense_result(p)
    p.close(); keys.close(); al.close()
    return r


def q17_unfused(ctx, lineitem, part, avg):
    f = D.FilterHandle(ctx, PART_TYPES, [C(1), I8(Q17_BRAND), B(D.OP_EQ), C(2), I8(Q17_CONTAINER), B(D.OP_EQ), B(D.OP_AND)], [0], batch_size=0)
    f.push_device(part); f.finish()
    fp = f.drain(host=False)
    f.close()
    j1 = D.HashJoinHandle(ctx, [D.INT64], [D.INT64] * 3, [0], [0], [1, 1, 1], [0, 1, 2], D.JOIN_INNER, batch_size=1 << 28, ordered_output=False)
    for b in fp:
        j1.push_build_device([b.column(0)])
    j1.finish_build()
    j2 = D.HashJoinHandle(ctx, [D.INT64, D.FLOAT64], [D.INT64] * 3, [0], [0], [1], [2], D.JOIN_INNER, batch_size=1 << 28, ordered_output=False)
    j2.set_filter([1, 0], [1, 1], q17_filter(0, 1))               # the JoinFilter's columns: probe quantity, build avg
    for b in avg:
        j2.push_build_device([b.column(0), b.column(1)])
    j2.finish_build()
    agg = zero_sum_agg(ctx)

    def consume(batches):
        for jb in batches:
            push_zero_grouped(ctx, agg, jb.column(0), jb.column(0))
            jb.release()

    def probe2(batches):
        for b in batches:
            j2.push_probe_device([b.column(0), b.column(1), b.column(2)])
            consume(j2.drain(host=False))
            b.release()
    j1.push_probe_device(lineitem[:3])
    probe2(j1.drain(host=False))
    j1.finish_probe()
    probe2(j1.drain(host=False))
    j2.finish_probe()
    consume(j2.drain(host=False))
    j1.close(); j2.close()
    for b in fp:
        b.release()
    return agg_result(agg)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed(ctx, fn):
    ctx.sync()
    t0 = time.perf_counter()
    r = fn()
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100.0
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    ctx = D.Context(0)
    out = {"sf": sf, "card": card(), "steps": steps}
    lineitem, part, _keep = gen(ctx, sf)
    ta, avg = timed(ctx, lambda: avg_build(ctx, lineitem))
    out["q17_avg_build_ms"] = round(ta, 2)
    plans = {"q19": (lambda: q19_fused(ctx, lineitem, part), lambda: q19_unfused(ctx, lineitem, part)),
             "q17": (lambda: q17_fused(ctx, lineitem, part, avg), lambda: q17_unfused(ctx, lineitem, part, avg))}
    for name, (fused, unfused) in plans.items():
        for fn in (fused, unfused):   # warm-up
            fn()
        tf, tu = [], []
        for _ in range(steps):
            a, rf = timed(ctx, fused)
            b, ru = timed(ctx, unfused)
            summary = check_sum(name, rf, ru)
            tf.append(a); tu.append(b)
        out[name] = {"fused_ms": [round(x, 2) for x in tf], "unfused_ms": [round(x, 2) for x in tu], "check": summary}
        print(json.dumps({name: out[name]}), flush=True)
    out["card_after"] = card()
    out["checks"] = "SUM and joined-row count of the fused plan equal the unfused plan's on every run"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
