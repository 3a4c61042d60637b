"""where the lineitem pass of Q3 spends its time: the same scan with progressively more of the pipeline switched on (SF100, device resident)"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from datafusion_b200 import capi as D
import q3_device_pipeline as Q
B, C, L = Q.B, Q.C, Q.L
sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100
ctx = D.Context(0)
cu, orr, li = Q.gen_tables(ctx, sf)
# build the orders-side structures once: L2 (table + Bloom) and a filter-only copy of its keys
kmin, kmax, _ = D.column_minmax_device(ctx, cu.cols[0])
l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
p = D.Pipeline(ctx, cu.types, B(D.OP_EQ, C(1), L(1))); p.sink_build(l1, 0, []); p.push_device(cu.cols); p.finish(); p.close()
l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=1)
p = D.Pipeline(ctx, orr.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2, 0, [2, 3]); p.push_device(orr.cols); p.finish()
nq = p.metric("sink_rows"); p.close()
q = D.Pipeline(ctx, orr.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); q.sink_output([0], ordered=False); q.push_device(orr.cols); q.finish()
qk = q.drain(host=False); q.close()
F = D.Lookup(ctx, D.INT64, [], expected_rows=nq, filter_only=True)
p = D.Pipeline(ctx, [D.INT64]); p.sink_build(F, 0, []); p.push_device([qk[0].column(0)]); p.finish(); p.close()
F8 = D.Lookup(ctx, D.INT64, [], expected_rows=8 * nq, filter_only=True)      # the geometry of an 8-GPU run's merged filter (8x the keys' bits; only this rank's keys set)
p = D.Pipeline(ctx, [D.INT64]); p.sink_build(F8, 0, []); p.push_device([qk[0].column(0)]); p.finish(); p.close()
print("filter bytes: 1-GPU geometry", F.filter_buffer()[1], " 8-GPU geometry", F8.filter_buffer()[1], flush=True)
l2n = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=0)        # the same table without a Bloom filter
p = D.Pipeline(ctx, orr.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2n, 0, [2, 3]); p.push_device(orr.cols); p.finish(); p.close()

rev = B(D.OP_MULTIPLY, C(1), B(D.OP_MINUS, L(100), C(2)))
variants = {
    "A0 predicate only, nothing survives (streams l_shipdate)": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(2**30, D.INT32)), name="v"), lambda p: p.sink_output([0], ordered=False)),
    "A1 predicate, 54% survive -> output l_orderkey": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), name="v"), lambda p: p.sink_output([0], ordered=False)),
    "A2 predicate + membership filter (MAYBE) -> output l_orderkey": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_MAYBE, 0, F)], name="v"), lambda p: p.sink_output([0], ordered=False)),
    "A2x8 predicate + membership filter of 8-GPU geometry -> output l_orderkey": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_MAYBE, 0, F8)], name="v"), lambda p: p.sink_output([0], ordered=False)),
    "A3 predicate + membership filter -> output key, price, discount": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_MAYBE, 0, F)], name="v"), lambda p: p.sink_output([0, 1, 2], ordered=False)),
    "B1 predicate + Bloom + probe (SEMI) -> output l_orderkey": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 0, l2)], name="v"), lambda p: p.sink_output([0], ordered=False)),
    "B2 full: predicate + Bloom + probe + SUM(price * (100 - disc))": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="v"), lambda p: p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, rev)])),
    "B3 full without the Bloom filter": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2n)], name="v"), lambda p: p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, rev)])),
    "B4 full, COUNT(*) only (no argument columns)": lambda: (D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="v"), lambda p: p.sink_aggregate([0, 4, 5], [(D.AGG_COUNT_STAR, None)])),
}
out = {}
ctx.set_kernel_timing(True)
for name, mk in variants.items():
    ms = []
    for it in range(4):
        p, sink = mk()
        sink(p)
        ctx.kernel_time_reset()
        p.push_device(li.cols); p.finish()
        for b in p.drain(host=False):
            b.release()
        t, n_ = ctx.kernel_time("pipe:v")
        # the partitioned aggregate (a table larger than L2: B2, B3): pass 1 is "pipe:v", then the partition and the probe-aggregate kernels
        tp, _ = ctx.kernel_time("pipe_partition"); ta, _ = ctx.kernel_time("pipe_probe_agg")
        rows, part = p.metric("sink_rows"), p.metric("partitioned_launches")
        p.close()
        if it:
            ms.append((t / max(n_, 1), tp, ta))
    best = min(ms, key=lambda m: sum(m))
    out[name] = {"kernel_ms": round(best[0], 3), "partition_ms": round(best[1], 3), "probe_agg_ms": round(best[2], 3), "partitioned": part, "sink_rows": rows}
    print(f"{name:75s} {best[0]:7.3f} ms" + (f" + partition {best[1]:.3f} + probe-aggregate {best[2]:.3f} ms" if part else "") + f"   sink rows {rows}", flush=True)
json.dump(out, open("gpurun_out/r2_pipe_breakdown.json", "w"), indent=1)
