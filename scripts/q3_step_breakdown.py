"""Where one Q3 step (bench.py's headline, Q.run_q3_fused at SF100, device resident, seed 1) spends its time.

  timed     the step's wall time between device events, as bench.py takes it, over --steps steps after --warmup;
  families  the library's kernel timers of the step (dfgpu_kernel_time), per step;
  rest      step - families: host synchronises, memsets, untimed kernels (key bounds, table init, group emission), launch gaps;
  profile   one more step under torch.profiler (a separate run: tracing slows the host) with every kernel, memset and copy on the
            device by name, and the device-idle remainder of that step.

It also reports the partitioned aggregate's "partitioned_records" (the {key, value} records pass 1 wrote) and sink rows of the
lineitem pipeline, and the card's name, power limit and clocks.
usage: python scripts/q3_step_breakdown.py [--sf 100] [--steps 10] [--warmup 3] [--no-profile] [--json FILE]"""
import argparse
import json
import os
import re
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from datafusion_b200 import capi as D  # noqa: E402
import q3_device_pipeline as Q  # noqa: E402
from q3_pass1_timing import gpu_info  # noqa: E402

# the kernel timer families one fused Q3 step can record, in plan order
FAMILIES = ("pipeline_build",                                   # P1 customer -> key bitmap
            "pipe:orders", "lookup_partition", "lookup_insert",  # P2 orders -> packed records -> (partitioned) insert + filter
            "pipe:lineitem",                                    # P3 pass 1 (partitioned) or the direct probe
            "pipe_filter_fold", "pipe_partition", "pipe_probe_agg")
LINEITEM_METRICS = ("sink_rows", "partitioned_launches", "partitioned_records", "ring_launches")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--json", help="also write the result to this file")
    args = ap.parse_args()
    ctx = D.Context(0)
    cu, orr, li = Q.gen_tables(ctx, args.sf)

    # the step is Q.run_q3_fused itself; the lineitem pipeline's metrics are read as it closes
    seen = {}
    close = D.Pipeline.close

    def close_and_record(p):
        if p.h and getattr(p, "_name", None) == "lineitem":
            seen.update({m: p.metric(m) for m in LINEITEM_METRICS})
        close(p)
    D.Pipeline.close = close_and_record

    def step():
        res, _ = Q.run_q3_fused(ctx, cu, orr, li)
        for b in res:
            b.release()

    for _ in range(args.warmup):
        step()
    ctx.sync()
    ctx.set_kernel_timing(True)
    ctx.kernel_time_reset()
    e0, e1 = ctx.event(), ctx.event()
    launches0 = ctx.launches
    ctx.record(e0)
    for _ in range(args.steps):
        step()
    ctx.record(e1)
    ctx.sync()
    step_ms = ctx.elapsed_ms(e0, e1) / args.steps
    launches = (ctx.launches - launches0) / args.steps
    fam = {}
    for k in FAMILIES:
        ms, n = ctx.kernel_time(k)
        fam[k] = {"ms_per_step": ms / args.steps, "launches_per_step": n / args.steps}
    ctx.set_kernel_timing(False)
    timed = sum(v["ms_per_step"] for v in fam.values())
    res = {"gpu": gpu_info(), "sf": args.sf, "steps": args.steps, "step_ms": step_ms, "library_launches_per_step": launches,
           "families": fam, "families_ms": timed, "rest_ms": step_ms - timed, "lineitem": dict(seen)}

    if not args.no_profile:
        try:
            res["profile"] = profile_step(step, ctx)
        except Exception as exc:   # the event timings above stand without it; say so instead of guessing
            res["profile"] = {"error": f"{type(exc).__name__}: {exc}"[:300]}

    g = res["gpu"]
    print(f"{g.get('name')}  power limit {g.get('power_limit')}  max SM clock {g.get('clocks_max_sm')}  SM clock {g.get('clocks_sm')}  SF{args.sf:g}")
    print(f"  step {step_ms:8.3f} ms  ({launches:.0f} library launches)")
    for k, v in fam.items():
        print(f"  {k:20s} {v['ms_per_step']:8.3f} ms  x{v['launches_per_step']:g}")
    print(f"  {'rest':20s} {step_ms - timed:8.3f} ms")
    print(f"  lineitem: {seen}")
    prof = res.get("profile", {})
    for k, v in prof.get("device_ms", {}).items():
        print(f"  profile {k:60.60s} {v:8.3f} ms")
    if "idle_ms" in prof:
        print(f"  profile step {prof['step_ms']:.3f} ms, device busy {prof['busy_ms']:.3f} ms, idle {prof['idle_ms']:.3f} ms")
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


def profile_step(step, ctx):
    """one step under torch.profiler: device time per kernel (template arguments dropped), memset and copy"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    ctx.sync()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        step()
        ctx.sync()
        wall = (time.perf_counter() - t0) * 1e3
    dev = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = re.sub(r"<.*", "", e.name).replace("void ", "").strip()
        dev[name] = dev.get(name, 0.0) + e.time_range.elapsed_us() / 1e3
    busy = sum(dev.values())
    return {"step_ms": wall, "busy_ms": busy, "idle_ms": wall - busy, "device_ms": dict(sorted(dev.items(), key=lambda kv: -kv[1]))}


if __name__ == "__main__":
    main()
