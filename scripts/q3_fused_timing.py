"""timing of the fused Q3 pipelines vs the operator-by-operator path at a given scale factor (device resident)"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from datafusion_b200 import capi as D
import q3_device_pipeline as Q

sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100
ctx = D.Context(0)
cu, orr, li = Q.gen_tables(ctx, sf)
out = {"sf": sf}
for name, fn in (("fused", Q.run_q3_fused), ("unfused", Q.run_q3)):
    for _ in range(2):
        res, st = fn(ctx, cu, orr, li)
        fp = Q.result_fingerprint(ctx, res)
        for b in res: b.release()
    ctx.set_kernel_timing(True); ctx.kernel_time_reset()
    e0, e1 = ctx.event(), ctx.event()
    ctx.record(e0)
    for _ in range(5):
        res, st = fn(ctx, cu, orr, li)
        for b in res: b.release()
    ctx.record(e1)
    ms = ctx.elapsed_ms(e0, e1) / 5
    kt = {k: ctx.kernel_time(k) for k in ("pipe:lineitem", "pipe:orders", "pipeline_count", "pipeline_build", "lookup_partition", "lookup_insert", "pipeline_agg", "pipeline_output", "join_probe", "join_build", "filter_fused", "agg_update")}
    ctx.set_kernel_timing(False)
    out[name] = {"ms": ms, "stages": st, "fingerprint": fp, "kernel_ms": {k: v[0] / max(v[1], 1) for k, v in kt.items() if v[1]}, "kernel_n": {k: v[1] for k, v in kt.items() if v[1]}}
print(json.dumps(out, indent=1))
assert out["fused"]["fingerprint"] == out["unfused"]["fingerprint"], "fused and unfused results differ"
