"""TPC-H Q1 and Q6 through the fused pipeline's dense-group aggregate sink, against the unfused GPU operator chain, device resident.

    Q1: FilterExec(l_shipdate <= 1998-09-02) -> AggregateExec GROUP BY l_returnflag, l_linestatus:
        SUM(l_quantity), SUM(l_extendedprice), SUM(price * (1 - disc)), SUM(price * (1 - disc) * (1 + tax)),
        AVG(l_quantity), AVG(l_extendedprice), AVG(l_discount), COUNT(*)
    Q6: FilterExec(1994-01-01 <= l_shipdate < 1995-01-01 AND 0.05 <= l_discount <= 0.07 AND l_quantity < 24) -> SUM(price * disc)

lineitem-shaped columns are generated in HBM with dfgpu_generate_i64 (seeded): l_returnflag, l_linestatus as Int32 codes (3 and 2
values), l_shipdate Date32, and the money columns l_quantity, l_extendedprice, l_discount, l_tax in hundredths, as Int64 or as
Decimal128(15,2) (the same unscaled integers).  The fused results are checked exactly against a host evaluation of the same columns
at the timed size, in chunks (Float64 AVG within 1e-9 relative); kernels are timed with dfgpu_kernel_time over warmed steps.  The
unfused chain (dfgpu_filter -> dfgpu_expr_evaluate_device -> dfgpu_agg) runs Q1 and Q6 in both money types, checked exactly the same
way.  It streams the table in slices, as the operators would see batches.

usage: python scripts/q1_q6_fused_timing.py [SF=100] [steps=5]"""
import datetime
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_b200 import capi as D

EPOCH = datetime.date(1970, 1, 1)
day = lambda y, m, d: (datetime.date(y, m, d) - EPOCH).days
D0, D1 = day(1992, 1, 2), day(1998, 12, 1)
Q1_CUT = day(1998, 9, 2)
Q6_LO, Q6_HI = day(1994, 1, 1), day(1995, 1, 1)
PEAK_BPS = 3.35e12                       # H100 SXM HBM3, data sheet
DEC = D.decimal128(15, 2)
SLICE = 50_000_000                       # rows per batch of the unfused chain and per host-check chunk


def C(i): return [(D.EXPR_COLUMN, i, 0, 0, 0, 0.0)]
def L(v, t=D.INT64): return [(D.EXPR_LITERAL, 0, t, 0, int(v), 0.0)]
def B(op, l, r): return l + r + [(D.EXPR_BINARY, op, 0, 0, 0, 0.0)]
def CAST(e, t): return e + [(D.EXPR_CAST, 0, t, 0, 0, 0.0)]
def AND(*xs):
    out = xs[0]
    for x in xs[1:]:
        out = B(D.OP_AND, out, x)
    return out


def col(ptr, n, t, offset=0):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = t, 0, n, 0, 0, ptr + offset * D.WIDTH[t], None
    return c


# columns: 0 l_returnflag, 1 l_linestatus, 2 l_shipdate, 3 l_quantity, 4 l_extendedprice, 5 l_discount, 6 l_tax
def generate(ctx, n, seed=7):
    keep = []

    def ev(c, buf, nodes, t):
        b = D.evaluate_device(ctx, [c], n, nodes); keep.append(b)
        out = b.column(0); out.type = t; out.validity = None; out.null_count = 0
        ctx.sync()
        buf.free()                                       # the generator's int64 values are not needed any more
        return out

    def gen(s, a, span):
        buf = ctx.generate_i64(D.GEN_UNIFORM, seed + s, a, span, 0, n)
        return col(buf.ptr, n, D.INT64), buf

    def kept(s, a, span):
        c, buf = gen(s, a, span); keep.append(buf)
        return c

    i32 = lambda t, s, a, span: ev(*gen(s, a, span), CAST(C(0), D.INT32), t)
    cols = [i32(D.INT32, 1, 0, 3), i32(D.INT32, 2, 0, 2), i32(D.DATE32, 3, D0, D1 - D0 + 1),
            ev(*gen(4, 1, 50), B(D.OP_MULTIPLY, C(0), L(100)), D.INT64), kept(5, 90_000, 10_405_001), kept(6, 0, 11), kept(7, 0, 9)]
    ctx.sync()
    return cols, keep


def as_decimal(ctx, cols, n, keep):
    """the money columns as Decimal128(15,2): CAST(int64 AS Decimal128(15,0)) relabelled at scale 2 (the same unscaled integers)"""
    out = list(cols)
    for i in (3, 4, 5, 6):
        b = D.evaluate_device(ctx, [cols[i]], n, CAST(C(0), D.decimal128(15, 0))); keep.append(b)
        c = b.column(0); c.type = DEC; c.validity = None; c.null_count = 0
        out[i] = c
    ctx.sync()
    return out


def q1_exprs(dec):
    """Q1's two computed money expressions and its AVG argument programs"""
    if dec:
        one = [(D.EXPR_LITERAL, 0, D.decimal128(20, 0), 0, 1, 0.0)]
        dp = B(D.OP_MULTIPLY, C(4), B(D.OP_MINUS, one, C(5)))
        ch = B(D.OP_MULTIPLY, dp, B(D.OP_PLUS, one, C(6)))
        avg = lambda i: C(i)
    else:
        dp = B(D.OP_MULTIPLY, C(4), B(D.OP_MINUS, L(100), C(5)))
        ch = B(D.OP_MULTIPLY, dp, B(D.OP_PLUS, L(100), C(6)))
        avg = lambda i: CAST(C(i), D.FLOAT64)
    return dp, ch, avg


def q1_program(dec):
    dp, ch, avg = q1_exprs(dec)
    pred = B(D.OP_LTEQ, C(2), L(Q1_CUT, D.DATE32))
    aggs = [(D.AGG_SUM, C(3)), (D.AGG_SUM, C(4)), (D.AGG_SUM, dp), (D.AGG_SUM, ch), (D.AGG_AVG, avg(3)), (D.AGG_AVG, avg(4)), (D.AGG_AVG, avg(5)),
            (D.AGG_COUNT_STAR, None)]
    return pred, aggs


def q6_program(dec):
    lit = (lambda v: [(D.EXPR_LITERAL, 0, DEC, 0, v, 0.0)]) if dec else (lambda v: L(v))
    pred = AND(B(D.OP_GTEQ, C(2), L(Q6_LO, D.DATE32)), B(D.OP_LT, C(2), L(Q6_HI, D.DATE32)), B(D.OP_GTEQ, C(5), lit(5)),
               B(D.OP_LTEQ, C(5), lit(7)), B(D.OP_LT, C(3), lit(2400)))
    return pred, [(D.AGG_SUM, B(D.OP_MULTIPLY, C(4), C(5))), (D.AGG_COUNT_STAR, None)]


def rows_of(batches):
    rows = []
    for b in batches:
        cs = []
        for i in range(b.num_columns):
            v, val = b.column_numpy(i)
            vals = D.words_to_decimal(v) if D.type_base(b.column(i).type) == D.DECIMAL128 else [x.item() for x in v]
            cs.append([None if val is not None and not val[k] else vals[k] for k in range(len(vals))])
        rows += list(zip(*cs))
    return rows


def run_fused(ctx, cols, types, n, pred, aggs, groups, ranges, name):
    p = D.Pipeline(ctx, types, pred, name=name)
    p.sink_aggregate_dense(groups, ranges, aggs)
    p.push_device(cols)
    p.finish()
    out = rows_of(p.drain(host=True))
    p.close()
    return out


def run_unfused(ctx, cols, types, n, pred, exprs, groups, aggs):
    """dfgpu_filter -> dfgpu_expr_evaluate_device -> dfgpu_agg, over slices of SLICE rows pushed into one aggregate.
    exprs: argument programs over the filtered columns (appended as new columns); aggs: [(func, column)] over [filtered..., exprs...]"""
    nin = len(types)
    a = None
    for s in range(0, n, SLICE):
        m = min(SLICE, n - s)
        f = D.FilterHandle(ctx, types, pred, None, batch_size=0)
        f.push_device([col(c.values, m, t, s) for c, t in zip(cols, types)]); f.finish()
        fo = f.drain(host=False); f.close()
        for b in fo:
            fc = [b.column(i) for i in range(nin)]
            ev = [D.evaluate_device(ctx, fc, b.num_rows, e) for e in exprs]
            ec = [x.column(0) for x in ev]
            if a is None:
                a = D.AggHandle(ctx, [c.type for c in fc + ec], groups, [(fn, c, -1) for fn, c in aggs], D.AGG_SINGLE, 8192, 16)
            a.push_device(fc + ec)
            for x in ev:
                x.release()
            b.release()
    a.finish()
    out = rows_of(a.drain(host=True))
    a.close()
    return out


def timed(ctx, fn, steps, families):
    fn()                                                 # warm-up: module loads, allocator
    ctx.set_kernel_timing(True); ctx.kernel_time_reset()
    e0, e1 = ctx.event(), ctx.event()
    ctx.record(e0)
    for _ in range(steps):
        out = fn()
    ctx.record(e1)
    ms = ctx.elapsed_ms(e0, e1) / steps
    kt = {k: ctx.kernel_time(k) for k in families}
    ctx.set_kernel_timing(False)
    return out, {"step_ms": ms, "kernel_ms": {k: v[0] / steps for k, v in kt.items() if v[1]}}


# ---- host evaluation of the same columns, in chunks ----
def host_cols(ctx, cols, types, s, m):
    out = []
    for c, t in zip(cols, types):
        raw = ctx.to_host(c.values + s * D.WIDTH[t], m * D.WIDTH[t])
        out.append(raw.view(np.int32 if D.WIDTH[t] == 4 else np.int64).astype(np.int64))
    return out


def host_reference(ctx, cols, types, n):
    """exact per-group Python-int sums and counts for Q1, and Q6's sum and count"""
    q1 = {}
    q6 = [0, 0]
    for s in range(0, n, SLICE // 5):
        m = min(SLICE // 5, n - s)
        rf, ls, ship, qty, price, disc, tax = host_cols(ctx, cols, types, s, m)
        dp = price * (100 - disc)                        # < 2^40 per row: int64 sums of 10M rows stay exact
        ch = dp * (100 + tax)                            # < 2^47
        sel = ship <= Q1_CUT
        g = (rf * 2 + ls)[sel]
        for k in np.unique(g):
            mk = g == k
            acc = q1.setdefault(int(k), [0] * 6)
            for j, v in enumerate((qty[sel][mk], price[sel][mk], dp[sel][mk], ch[sel][mk], disc[sel][mk])):
                acc[j] += int(v.sum())
            acc[5] += int(mk.sum())
        s6 = (ship >= Q6_LO) & (ship < Q6_HI) & (disc >= 5) & (disc <= 7) & (qty < 2400)
        q6[0] += int((price[s6] * disc[s6]).sum()); q6[1] += int(s6.sum())
    return q1, q6


def wrap64(x):
    x %= 1 << 64
    return x - (1 << 64) if x >= 1 << 63 else x


def tdiv(a, b):
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def check_q1(rows, ref, dec):
    assert len(rows) == len(ref), (len(rows), len(ref))
    for r, k in zip(rows, sorted(ref)):
        sq, sp, sdp, sch, sd, cnt = ref[k]
        assert (r[0], r[1]) == (k // 2, k % 2), (r[:2], k)
        assert r[9] == cnt, (r[9], cnt)
        if dec:
            assert list(r[2:6]) == [sq, sp, sdp, sch], (r[2:6], (sq, sp, sdp, sch))
            assert list(r[6:9]) == [tdiv(x * 10 ** 4, cnt) for x in (sq, sp, sd)], r[6:9]
        else:
            assert list(r[2:6]) == [wrap64(x) for x in (sq, sp, sdp, sch)], (r[2:6], (sq, sp, sdp, sch))
            for got, x in zip(r[6:9], (sq, sp, sd)):
                assert abs(got - x / cnt) <= 1e-9 * abs(x / cnt), (got, x / cnt)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    n = int(6_000_000 * sf)
    ctx = D.Context(0)
    out = {"sf": sf, "rows": n, "gpu": gpu_info()}
    cols, keep = generate(ctx, n)
    itypes = [D.INT32, D.INT32, D.DATE32, D.INT64, D.INT64, D.INT64, D.INT64]
    ref_q1, ref_q6 = host_reference(ctx, cols, itypes, n)
    fam = ["pipe:q1", "pipe:q6", "filter_fused", "expr_eval", "agg_update"]
    res = {}
    for money in ("int64", "decimal128"):
        dec = money == "decimal128"
        if dec:
            ctx.trim_device_cache()                      # the unfused chain's batches: room for the four Decimal128 columns
        dcols, types = (as_decimal(ctx, cols, n, keep), [D.INT32, D.INT32, D.DATE32] + [DEC] * 4) if dec else (cols, itypes)
        pred, aggs = q1_program(dec)
        rows, t = timed(ctx, lambda: run_fused(ctx, dcols, types, n, pred, aggs, [0, 1], [(0, 2), (0, 1)], "q1"), steps, fam)
        check_q1(rows, ref_q1, dec)
        res[f"q1_{money}_fused"] = t
        pred6, aggs6 = q6_program(dec)
        rows, t = timed(ctx, lambda: run_fused(ctx, dcols, types, n, pred6, aggs6, [], [], "q6"), steps, fam)
        assert rows == [(ref_q6[0] if dec else wrap64(ref_q6[0]), ref_q6[1])], (rows, ref_q6)
        res[f"q6_{money}_fused"] = t
        # the unfused chain; Q6 is SUM alone: dfgpu_agg without GROUP BY
        ex6 = [B(D.OP_MULTIPLY, C(4), C(5))]
        rows, t = timed(ctx, lambda: run_unfused(ctx, dcols, types, n, pred6, ex6, [], [(D.AGG_SUM, 7)]), 1, fam)
        assert rows == [(ref_q6[0] if dec else wrap64(ref_q6[0]),)], (rows, ref_q6)
        res[f"q6_{money}_unfused"] = t
        dp, ch, avg = q1_exprs(dec)
        if dec:   # AVG over the Decimal128 columns themselves
            ex1, avg_cols = [dp, ch], (3, 4, 5)
        else:
            ex1, avg_cols = [dp, ch] + [avg(i) for i in (3, 4, 5)], (9, 10, 11)
        a1 = [(D.AGG_SUM, 3), (D.AGG_SUM, 4), (D.AGG_SUM, 7), (D.AGG_SUM, 8)] + [(D.AGG_AVG, i) for i in avg_cols] + [(D.AGG_COUNT_STAR, -1)]
        rows, t = timed(ctx, lambda: run_unfused(ctx, dcols, types, n, pred, ex1, [0, 1], a1), 1, fam)
        check_q1(sorted(rows, key=lambda r: (r[0], r[1])), ref_q1, dec)
        res[f"q1_{money}_unfused"] = t
    # DRAM floors from the shapes (not measured): every streamed byte once; Q6 touches l_extendedprice only for its survivors
    q6_sel = ref_q6[1] / n
    floors = {"q1_int64": 44 * n, "q1_decimal128": 76 * n, "q6_int64": (4 + 8 + 8 + 8 * q6_sel) * n, "q6_decimal128": (4 + 16 + 16 + 16 * q6_sel) * n}
    for k, b in floors.items():
        f = res[f"{k}_fused"]
        f["floor_ms"] = b / PEAK_BPS * 1e3
        f["share_of_floor"] = f["floor_ms"] / f["step_ms"]
    out["results"] = res
    out["q6_selectivity"] = q6_sel
    out["checks"] = "passed"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
