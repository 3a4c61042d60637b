"""Push time of a fused join-keyed aggregate with Float64 MIN / MAX (pipe_kernel<SINK_AGG>): device-resident probe rows stream through
an INNER stage into MIN(x), MAX(x), COUNT(*) per build row.  Two shapes: many groups (the words spread over the table) and 64 groups
(every row contends for a few words).  Prints one JSON line per shape: the median push time over --reps pushes, each timed from a
device synchronise to a device synchronise, and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from datafusion_b200 import capi as D  # noqa: E402

X = [(D.EXPR_COLUMN, 1, 0, 0, 0, 0.0)]


def lookup(ctx, groups):
    look = D.Lookup(ctx, D.INT64, [], n_acc_words=3, expected_rows=groups)   # row counter, MIN, MAX
    p = D.Pipeline(ctx, [D.INT64])
    p.sink_build(look, 0, [])
    p.push_host([D.HostColumn(np.arange(groups, dtype=np.int64))])
    p.finish()
    p.close()
    return look


def run(ctx, rows, groups, reps, warmup):
    rng = np.random.default_rng(1)
    cols = [D.DeviceColumn.from_host(ctx, D.HostColumn(rng.integers(0, groups, rows).astype(np.int64))),
            D.DeviceColumn.from_host(ctx, D.HostColumn(rng.standard_normal(rows)))]
    look = lookup(ctx, groups)
    times = []
    for i in range(warmup + reps):
        p = D.Pipeline(ctx, [D.INT64, D.FLOAT64], None, [(D.STAGE_INNER, 0, look)])
        p.sink_aggregate([0], [(D.AGG_MIN, X), (D.AGG_MAX, X), (D.AGG_COUNT_STAR, None)])
        ctx.sync()
        t0 = time.perf_counter()
        p.push_device(cols)
        ctx.sync()
        if i >= warmup:
            times.append(time.perf_counter() - t0)
        p.finish()
        p.drain(host=False)
        p.close()
    look.close()
    return float(np.median(times)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    ctx = D.Context(0)
    for groups in (4_000_000, 64):
        ms = run(ctx, a.rows, groups, a.reps, a.warmup)
        print(json.dumps({"rows": a.rows, "groups": groups, "push_ms_median": round(ms, 3), "rows_per_s": round(a.rows / ms * 1e3), "card": card}))
    ctx.close()


if __name__ == "__main__":
    main()
