"""The C3 group-by shape (1B rows -> 1M groups, as scripts/agg_timing.py) with SUM, MIN, MAX, AVG and COUNT of one value column, once
over Int64 and once over the same unscaled integers as Decimal128(15,2), through dfgpu_agg (the general hash group-by).

Keys and values are generated in HBM with dfgpu_generate_i64 (seeded); the Decimal128 column is CAST(v AS Decimal128(15,0)) relabelled
at scale 2.  Each run is timed with CUDA events around push + finish, over warmed iterations.  At the timed size the Decimal128 result
is checked exactly against the Int64 result, group by group: SUM, MIN, MAX and COUNT equal, and AVG = tdiv(SUM * 10^4, COUNT)
(DecimalAverager::avg into Decimal128(19,6): the scale grows by 4, truncated toward zero).  The card name and power limit are printed
with the times.

usage: python scripts/agg_decimal_timing.py [rows=1e9] [groups=1e6] [iters=3]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_b200 import capi as D

DEC = D.decimal128(15, 2)
AGGS = [(D.AGG_SUM, 1, -1), (D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_AVG, 1, -1), (D.AGG_COUNT, 1, -1)]
V_LO, V_SPAN = -2**31, 2**32               # values as in scripts/agg_timing.py: no Int64 sum of a group can wrap


def tdiv(a: int, b: int) -> int:
    """Rust's integer `/`: truncation toward zero"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def check_exact(int_rows, dec_rows):
    """int_rows: (key, sum, min, max, avg: float, count) of the Int64 run; dec_rows: (key, sum, min, max, avg, count) of the
    Decimal128(15,2) run with the decimals as unscaled Python ints.  Raises AssertionError on the first difference."""
    assert len(int_rows) == len(dec_rows), (len(int_rows), len(dec_rows))
    ref = {r[0]: r for r in int_rows}
    assert len(ref) == len(int_rows), "duplicate group keys in the Int64 result"
    for k, s, mn, mx, avg, cnt in dec_rows:
        assert k in ref, f"group {k} missing from the Int64 result"
        _, si, mni, mxi, _, ci = ref[k]
        assert (s, mn, mx, cnt) == (si, mni, mxi, ci), (k, (s, mn, mx, cnt), (si, mni, mxi, ci))
        assert avg == tdiv(s * 10 ** 4, cnt), (k, avg, s, cnt)


def col(ptr, n, t):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = t, 0, n, 0, 0, ptr, None
    return c


def rows_of(batches):
    rows = []
    for b in batches:
        cs = []
        for i in range(b.num_columns):
            v, val = b.column_numpy(i)
            assert val is None or val.all(), "no group of this input is all NULL"
            cs.append(D.words_to_decimal(v) if D.type_base(b.column(i).type) == D.DECIMAL128 else v.tolist())
        rows += list(zip(*cs))
    return rows


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return q.stdout.strip()


def run(ctx, n, groups, keys, vals, vtype, iters):
    times, out = [], None
    for it in range(iters + 1):                           # iteration 0 warms up
        e0, e1 = ctx.event(), ctx.event()
        a = D.AggHandle(ctx, [D.INT64, vtype], [0], AGGS, D.AGG_SINGLE, 8192, groups)
        ctx.record(e0)
        a.push_device([col(keys, n, D.INT64), col(vals, n, vtype)])
        a.finish()
        ctx.record(e1)
        ms = ctx.elapsed_ms(e0, e1)
        if it:
            times.append(round(ms, 3))
        if it == iters:
            out = rows_of(a.drain(host=True))
        else:
            for b in a.drain(host=False):
                b.release()
        a.close()
    return times, out


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 1_000_000_000
    groups = int(float(sys.argv[2])) if len(sys.argv) > 2 else 1_000_000
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    ctx = D.Context(0)
    info = gpu_info()
    k = ctx.generate_i64(D.GEN_UNIFORM, 5, 0, groups, 0, n)
    v = ctx.generate_i64(D.GEN_UNIFORM, 6, V_LO, V_SPAN, 0, n)
    t_int, rows_int = run(ctx, n, groups, k.ptr, v.ptr, D.INT64, iters)
    cast = [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0), (D.EXPR_CAST, 0, D.decimal128(15, 0), 0, 0, 0.0)]
    vd = D.evaluate_device(ctx, [col(v.ptr, n, D.INT64)], n, cast)
    ctx.sync()
    v.free()
    t_dec, rows_dec = run(ctx, n, groups, k.ptr, vd.column(0).values, DEC, iters)
    check_exact(rows_int, rows_dec)
    print(json.dumps({"gpu": info, "rows": n, "groups": len(rows_int), "aggregates": "SUM, MIN, MAX, AVG, COUNT",
                      "int64_ms": t_int, "decimal128_15_2_ms": t_dec, "check": "decimal == int64 exactly (AVG = tdiv(sum * 10^4, count))"}, indent=1))


if __name__ == "__main__":
    main()
