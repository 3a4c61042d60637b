"""The fused TPC-H Q3 plan (scripts/q3_device_pipeline.py, run_q3_fused) with SUM, MIN, MAX and AVG of the revenue expression in the
lineitem pipeline's join-keyed aggregate sink, next to the SUM-only Decimal128 Q3 step.

Tables are generated in HBM (gen_tables, seeded); decimal_money turns l_extendedprice and l_discount into Decimal128(15,2) with the same
unscaled integers.  Three runs of the whole plan, each timed with CUDA events over warmed iterations:
  - decimal_sum:      SUM(l_extendedprice * (1 - l_discount)) over Decimal128(15,2) money -> Decimal128(38,4) (the existing step);
  - decimal_aggs:     SUM, MIN, MAX and AVG of the same expression (AVG -> Decimal128(38,8)); L2 reserves 11 accumulator words;
  - int64_aggs:       SUM, MIN, MAX and COUNT(*) of price_cents * (100 - discount_percent) over Int64 money (AVG takes only Float64
                      there); 4 words.
The revenue integers are the same in both runs, so the Decimal128 result is checked exactly against the Int64 one, group by group:
SUM, MIN and MAX equal, and AVG = tdiv(SUM * 10^4, COUNT) (agg_decimal_timing.check_exact's rule).  The card name and power limit are
printed with the times.

usage: python scripts/q3_decimal_aggs_timing.py [sf=100] [iters=5]"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from datafusion_b200 import capi as D
import q3_device_pipeline as Q
from agg_decimal_timing import gpu_info

DEC_AGGS = (D.AGG_SUM, D.AGG_MIN, D.AGG_MAX, D.AGG_AVG)
INT_AGGS = (D.AGG_SUM, D.AGG_MIN, D.AGG_MAX, D.AGG_COUNT_STAR)
DEC_WORDS, INT_WORDS = 11, 4   # row counter + padding + 2 pairs + SUM {lo, hi} + AVG {lo, hi, count}; row counter + 3 (no NULLs)


def pipeline_aggs(funcs, l_types):
    rev = Q.revenue_expr(l_types)
    return [(f, None if f == D.AGG_COUNT_STAR else rev) for f in funcs]


def host_cols(batches):
    """result batches -> int64 numpy columns [l_orderkey, o_orderdate, o_shippriority, agg0 .. agg3].  A Decimal128 column becomes its
    unscaled value after a check that every high word only extends the sign of its low word: Q3's revenue sums (at most seven
    lineitems of at most 1.05e9 each per group) and their AVG (* 10^4) stay far inside 64 bits.  SF100 has ~13M groups: vectorised."""
    parts = []
    for b in batches:
        cs = []
        for i in range(b.num_columns):
            v, val = b.column_numpy(i)
            assert val is None or val.all(), "every group of Q3 has a revenue"
            if D.type_base(b.column(i).type) == D.DECIMAL128:
                w = np.ascontiguousarray(v).view(np.int64).reshape(-1, 2)
                assert np.array_equal(w[:, 1], w[:, 0] >> 63), "a Decimal128 result beyond 64 bits"
                cs.append(w[:, 0].copy())
            else:
                cs.append(np.asarray(v).astype(np.int64))
        parts.append(cs)
    return [np.concatenate([p[i] for p in parts]) for i in range(len(parts[0]))] if parts else []


def check_rows(ints, decs):
    """ints: columns [l_orderkey, o_orderdate, o_shippriority, SUM, MIN, MAX, COUNT(*)] of the Int64 run; decs: [the group columns,
    SUM, MIN, MAX, AVG] of the Decimal128 run (unscaled).  Group by group: SUM, MIN and MAX equal, and AVG = tdiv(SUM * 10^4, COUNT),
    the rule of agg_decimal_timing.check_exact (DecimalAverager::avg into Decimal128(38,8): truncation toward zero).  The Decimal128
    run's COUNT is the Int64 run's: the same rows join the same groups.  Raises AssertionError on the first difference."""
    assert len(ints[0]) == len(decs[0]), (len(ints[0]), len(decs[0]))
    i = [c[np.lexsort(ints[2::-1])] for c in ints]
    d = [c[np.lexsort(decs[2::-1])] for c in decs]
    same = lambda a, b: np.nonzero(a != b)[0]
    assert not ((i[0][1:] == i[0][:-1]) & (i[1][1:] == i[1][:-1]) & (i[2][1:] == i[2][:-1])).any(), "duplicate groups in the Int64 result"
    for j, what in enumerate(("l_orderkey", "o_orderdate", "o_shippriority", "SUM", "MIN", "MAX")):
        bad = same(i[j], d[j])
        assert not len(bad), f"{what} differs in {len(bad)} groups, e.g. {[int(c[bad[0]]) for c in d]} against {[int(c[bad[0]]) for c in i]}"
    s, cnt = i[3], i[6]
    assert np.all(np.abs(s) < 2 ** 63 // 10 ** 4) and np.all(cnt > 0)
    q = np.abs(s * 10 ** 4) // cnt
    q = np.where(s < 0, -q, q)                   # tdiv: truncation toward zero
    bad = same(d[6], q)
    assert not len(bad), f"AVG differs in {len(bad)} groups, e.g. sum {int(s[bad[0]])}, count {int(cnt[bad[0]])}: {int(d[6][bad[0]])} != {int(q[bad[0]])}"


def timed(ctx, iters, fn, what):
    """(ms per iteration after one warm-up, the last iteration's result batches on the host)"""
    times, out = [], None
    for it in range(iters + 1):
        e0, e1 = ctx.event(), ctx.event()
        ctx.record(e0)
        res, stages = fn()
        ctx.record(e1)
        ms = ctx.elapsed_ms(e0, e1)
        print(f"{what} iteration {it}: {ms:.3f} ms", file=sys.stderr, flush=True)
        if it:
            times.append(round(ms, 3))
        if it == iters:
            out = host_cols(res)
        for b in res:
            b.release()
    return times, out, stages


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100.0
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    ctx = D.Context(0)
    info = gpu_info()
    customer, orders, lineitem = Q.gen_tables(ctx, sf)
    dline = Q.decimal_money(ctx, lineitem)
    ctx.sync()
    print(f"{info}; SF{sf:g} tables generated", file=sys.stderr, flush=True)
    t_sum, _, st = timed(ctx, iters, lambda: Q.run_q3_fused(ctx, customer, orders, dline), "decimal_sum")
    t_dec, rows_dec, _ = timed(ctx, iters, lambda: Q.run_q3_fused(ctx, customer, orders, dline, pipeline_aggs(DEC_AGGS, dline.types), DEC_WORDS), "decimal_aggs")
    t_int, rows_int, _ = timed(ctx, iters, lambda: Q.run_q3_fused(ctx, customer, orders, lineitem, pipeline_aggs(INT_AGGS, lineitem.types), INT_WORDS), "int64_aggs")
    print(f"{len(rows_dec[0])} groups on the host; checking", file=sys.stderr, flush=True)
    check_rows(rows_int, rows_dec)
    print(json.dumps({"gpu": info, "sf": sf, "joined_rows": st["joined_rows"], "groups": len(rows_dec[0]), "iters": iters,
                      "decimal_sum_ms": t_sum, "decimal_sum_min_max_avg_ms": t_dec, "int64_sum_min_max_count_ms": t_int,
                      "check": "decimal == int64 exactly per group (SUM, MIN, MAX; AVG = tdiv(sum * 10^4, count))"}, indent=1))


if __name__ == "__main__":
    main()
