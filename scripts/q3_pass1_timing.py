"""Where the partitioned Q3 lineitem pass (pass 1 of the fused pipeline's partitioned aggregate) spends its time, set against the
bytes it must move.  At SF100 (device resident, seed 1) it times, with the library's kernel timers:

  stream   the date predicate alone, nothing survives: the l_shipdate stream, the floor of any pass over lineitem;
  filter   the predicate + the orders table's exact (16 bits per key) Bloom filter (a MAYBE stage) -> l_orderkey out: phase A plus a
           compaction (the A0 / A2 variants of pipe_breakdown.py); its sink rows are the survivors incl. the exact filter's false positives;
  full     the fused lineitem pipeline as bench.py runs it: `pipe_filter_fold` (the filter folded to 8 bits per key), pass 1
           (`pipe:lineitem`, which tests the folded filter and writes "partitioned_records"), `pipe_partition` and `pipe_probe_agg`.

The bytes are estimated from the measured counts (lineitem rows, records R, sink rows), not from the generators:
  pass 1: 12 B per row streamed (l_shipdate 4 + l_orderkey 8), the 32-byte sectors of l_extendedprice and l_discount that hold at
          least one record's row (rows uniform: 1 - (1 - R/n)^4 of them), 16 B per record written;
  filter: 12 B per row + 8 B per record written;  fold: the exact filter read, half of it written;
  partition: 16 B per record read twice (histogram, scatter) and written once;
  probe-aggregate: 16 B per record read (the table's slot ranges are L2-resident by construction).
usage: python scripts/q3_pass1_timing.py [--sf 100] [--reps 5] [--json FILE]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from datafusion_b200 import capi as D  # noqa: E402
import q3_device_pipeline as Q  # noqa: E402

B, C, L = Q.B, Q.C, Q.L


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, max_sm, sm = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": max_sm, "clocks_sm": sm}
    except Exception as exc:   # the timings stand without it; say so instead of guessing
        return {"error": f"{type(exc).__name__}: {exc}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=100)
    ap.add_argument("--reps", type=int, default=5, help="timed runs per variant (after one warm-up run); the median is reported")
    ap.add_argument("--json", help="also write the result to this file")
    args = ap.parse_args()
    ctx = D.Context(0)
    cu, orr, li = Q.gen_tables(ctx, args.sf)
    n = li.rows
    kmin, kmax, _ = D.column_minmax_device(ctx, cu.cols[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p = D.Pipeline(ctx, cu.types, B(D.OP_EQ, C(1), L(1))); p.sink_build(l1, 0, []); p.push_device(cu.cols); p.finish(); p.close()

    def orders_table():
        l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=-1)
        p = D.Pipeline(ctx, orr.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)], name="orders")
        p.sink_build(l2, 0, [2, 3]); p.push_device(orr.cols); p.finish(); p.close()
        return l2

    l2 = orders_table()
    rev = Q.revenue_expr(li.types)
    variants = {
        "stream": (lambda: D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(2**30, D.INT32)), name="v"), lambda p: p.sink_output([0], ordered=False), "pipe:v"),
        "filter": (lambda: D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_MAYBE, 0, l2)], name="v"),
                   lambda p: p.sink_output([0], ordered=False), "pipe:v"),
    }
    ctx.set_kernel_timing(True)
    res = {"gpu": gpu_info(), "sf": args.sf, "lineitem_rows": n}
    med = lambda xs: sorted(xs)[len(xs) // 2]
    for name, (mk, sink, timer) in variants.items():
        ms = []
        for it in range(args.reps + 1):
            p = mk(); sink(p)
            ctx.kernel_time_reset()
            p.push_device(li.cols); p.finish()
            for b in p.drain(host=False):
                b.release()
            t, k = ctx.kernel_time(timer)
            rows = p.metric("sink_rows")
            p.close()
            if it:
                ms.append(t / max(k, 1))
        res[name] = {"kernel_ms": med(ms), "runs_ms": ms, "sink_rows": rows}
    recs = res["filter"]["sink_rows"]
    # the full lineitem pipeline, as bench.py runs it (the orders table is rebuilt for every run: the sums accumulate in its records)
    full = []
    for it in range(args.reps + 1):
        l2.close()
        l2 = orders_table()
        p = D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
        p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, rev)], D.AGG_SINGLE_PARTITIONED)
        ctx.kernel_time_reset()
        p.push_device(li.cols); p.finish()
        for b in p.drain(host=False):
            b.release()
        t = {k: ctx.kernel_time(k)[0] for k in ("pipe:lineitem", "pipe_filter_fold", "pipe_partition", "pipe_probe_agg")}
        metrics = {m: p.metric(m) for m in ("sink_rows", "partitioned_launches", "partitioned_records", "ring_launches")}
        p.close()
        if it:
            full.append(t)
    res["full"] = {k: med([f[k] for f in full]) for k in full[0]}
    res["full"]["runs_ms"] = full
    res["full"].update(metrics)
    fbytes = l2.metric("filter_bytes")
    l2.close(); l1.close()

    # pass 1 tests the filter folded to half size, so it writes more records than the exact filter lets through
    precs = res["full"]["partitioned_records"] if res["full"]["partitioned_records"] >= 0 else recs
    sectors = 1.0 - (1.0 - precs / n) ** 4 if n else 0.0
    gather = 2 * 8 * n * sectors
    bytes_ = {"stream": 4 * n, "filter": 12 * n + 8 * recs, "pipe:lineitem": 12 * n + gather + 16 * precs,
              "pipe_filter_fold": 1.5 * fbytes, "pipe_partition": 48 * precs, "pipe_probe_agg": 16 * precs}
    res["records"] = recs
    res["partitioned_records"] = precs
    res["pass1_gather_bytes"] = gather
    res["estimated_bytes"] = bytes_
    times = {"stream": res["stream"]["kernel_ms"], "filter": res["filter"]["kernel_ms"], **{k: res["full"][k] for k in ("pipe:lineitem", "pipe_filter_fold", "pipe_partition", "pipe_probe_agg")}}
    res["achieved_gbs"] = {k: bytes_[k] / (times[k] / 1e3) / 1e9 if times[k] > 0 else None for k in bytes_}
    g = res["gpu"]
    print(f"{g.get('name')}  power limit {g.get('power_limit')}  max SM clock {g.get('clocks_max_sm')}  SF{args.sf:g}: {n} lineitem rows, "
          f"{recs} exact-filter records, {precs} partitioned records, {res['full']['sink_rows']} sink rows")
    for k in bytes_:
        print(f"  {k:16s} {times[k]:8.3f} ms  {bytes_[k] / 1e9:7.2f} GB  {res['achieved_gbs'][k] or 0:7.0f} GB/s")
    print(f"  full pass: ring launches {res['full']['ring_launches']}, partitioned launches {res['full']['partitioned_launches']}")
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
