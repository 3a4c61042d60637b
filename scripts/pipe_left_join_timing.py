"""Left-family joins through the fused pipeline's join-keyed aggregate sink against the unfused GPU chain, device resident.

    Q13: customer LEFT JOIN orders ON c_custkey = o_custkey AND <predicate on orders>, count(o_orderkey) GROUP BY c_custkey, then
         count(*) GROUP BY c_count.  SF x 150,000 customers, SF x 1,500,000 orders; o_custkey skips every third customer, so one customer
         in three has no order, as in dbgen.  An integer column o_comment uniform over [0, 100) with `o_comment < 98` stands in for
         `o_comment NOT LIKE '%special%requests%'` (it keeps 98 % of the orders; strings are not carried here).
        fused   : customer build pipeline -> lookup with accumulator words; orders pipeline over a LEFT stage into the join-keyed sink;
                  dfgpu_agg for the histogram
        unfused : dfgpu_filter -> dfgpu_hashjoin(Left) -> dfgpu_agg -> dfgpu_agg
    Semi / anti: customer LEFT SEMI / LEFT ANTI JOIN the orders of one quarter of the date range (o_orderdate uniform over 2406 days)
        fused   : an INNER stage (LeftSemi) or a LEFT_ANTI stage into the join-keyed sink without aggregates
        unfused : dfgpu_filter -> dfgpu_hashjoin(LeftSemi / LeftAnti)

Fused and unfused runs alternate in one process after a warm-up; each time is a host clock around work that ends in a device synchronise.
Q13's times end at the per-customer counts on the device: the histogram aggregate over them is the same dfgpu_agg call on both sides and
runs with the check, untimed.
Checks, on every run: Q13's c_count histogram exactly, plus a per-customer fingerprint (wrapping sum over customers of a mix of the key and
its count); semi / anti: the row count and the wrapping sum of the emitted keys (dfgpu_column_sum_device).

usage: python scripts/pipe_left_join_timing.py [SF=100] [steps=3]"""
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
L = lambda v: (D.EXPR_LITERAL, 0, D.INT64, 0, v, 0.0)                        # noqa: E731
B = lambda op: (D.EXPR_BINARY, op, 0, 0, 0, 0.0)                              # noqa: E731
COMMENT_KEEP = 98
DATE_DAYS, DATE_LO, DATE_HI = 2406, 600, 1200                                 # the semi / anti join's orders: o_orderdate in [600, 1200)
MIX = np.uint64(0x9E3779B97F4A7C15)


# ---- the exact checks (host side; tests/test_pipe_left_join_timing_checks.py runs them on tiny data) ----
def customer_fingerprint(keys, counts) -> int:
    """wrapping sum over customers of key * MIX xor count: independent of the row order, changed by any key or count"""
    k = np.asarray(keys, np.int64).view(np.uint64)
    c = np.asarray(counts, np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        return int(np.bitwise_xor(k * MIX, c).sum(dtype=np.uint64))


def histogram(c_count, custdist) -> dict:
    """the second aggregate's rows {c_count: custdist}"""
    h = {}
    for a, b in zip(np.asarray(c_count).tolist(), np.asarray(custdist).tolist()):
        assert a not in h, f"c_count {a} appears twice"
        h[a] = b
    return h


def check_q13(fused, unfused) -> dict:
    """fused / unfused: (customer keys, their counts, histogram dict).  Raises on any difference."""
    fk, fc, fh = fused
    uk, uc, uh = unfused
    assert len(fk) == len(uk), f"Q13: {len(fk)} customers fused, {len(uk)} unfused"
    ff, uf = customer_fingerprint(fk, fc), customer_fingerprint(uk, uc)
    assert ff == uf, f"Q13: per-customer fingerprint {ff:#x} != {uf:#x}"
    assert fh == uh, "Q13: the c_count histograms differ"
    assert sum(fh.values()) == len(fk), "Q13: the histogram does not count every customer"
    return {"customers": len(fk), "fingerprint": f"{ff:#x}", "zero_order_customers": fh.get(0, 0)}


def check_keys(name, fused, unfused) -> dict:
    """fused / unfused: (rows, wrapping key sum)"""
    assert fused == unfused, f"{name}: fused {fused} != unfused {unfused}"
    return {"rows": fused[0], "key_sum": f"{fused[1]:#x}"}


# ---- device side ----
def dcol(buf, n, t=D.INT64):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = t, 0, n, 0, 0, buf.ptr, None
    return c


def gen(ctx, sf, seed=13):
    n_cust, n_ord = int(150_000 * sf), int(1_500_000 * sf)
    rng = np.random.default_rng(seed)
    u = rng.integers(0, n_cust - n_cust // 3, n_ord)
    ocust = (u // 2) * 3 + (u % 2) + 1                                       # skips c_custkey = 3, 6, 9, ...
    keep = [ctx.to_device(np.arange(1, n_cust + 1, dtype=np.int64)), ctx.to_device(np.arange(1, n_ord + 1, dtype=np.int64)),
            ctx.to_device(ocust.astype(np.int64)), ctx.generate_i64(D.GEN_UNIFORM, seed + 1, 0, 99, 0, n_ord),
            ctx.generate_i64(D.GEN_UNIFORM, seed + 2, 0, DATE_DAYS - 1, 0, n_ord)]
    customer = [dcol(keep[0], n_cust)]
    orders = [dcol(b, n_ord) for b in keep[1:]]                              # o_orderkey, o_custkey, o_comment, o_orderdate
    return customer, orders, keep


ORDER_TYPES = [D.INT64] * 4
Q13_PRED = [C(2), L(COMMENT_KEEP), B(D.OP_LT)]
DATE_PRED = [C(3), L(DATE_LO), B(D.OP_GTEQ), C(3), L(DATE_HI), B(D.OP_LT), B(D.OP_AND)]


def customer_lookup(ctx, customer, n_acc):
    look = D.Lookup(ctx, D.INT64, [], expected_rows=customer[0].length, n_acc_words=n_acc)
    p = D.Pipeline(ctx, [D.INT64])
    p.sink_build(look, 0, []); p.push_device(customer); p.finish(); p.close()
    return look


def histogram_of(ctx, batches):
    """dfgpu_agg count(*) GROUP BY c_count over column 1 of the per-customer batches -> (keys, counts, histogram)"""
    agg = D.AggHandle(ctx, [D.INT64], [0], [(D.AGG_COUNT_STAR, -1, -1)], D.AGG_SINGLE, 1 << 30, 64)
    keys, counts = [], []
    for b in batches:
        agg.push_device([b.column(1)])
    agg.finish()
    h = {}
    for r in agg.drain(host=True):
        h.update(histogram(r.column_numpy(0)[0], r.column_numpy(1)[0]))
    agg.close()
    for b in batches:
        keys.append(np.asarray(b.column_numpy(0)[0], np.int64)); counts.append(np.asarray(b.column_numpy(1)[0], np.int64))
        b.release()
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)  # noqa: E731
    return cat(keys), cat(counts), h


def q13_fused(ctx, customer, orders):
    look = customer_lookup(ctx, customer, 2)                                 # row counter, COUNT(o_orderkey)
    p = D.Pipeline(ctx, ORDER_TYPES, Q13_PRED, [(D.STAGE_LEFT, 1, look)], name="q13_left")
    p.sink_aggregate([1], [(D.AGG_COUNT, [C(0)])], D.AGG_SINGLE_PARTITIONED)
    p.push_device(orders); p.finish()
    res = p.drain(host=False)
    p.close(); look.close()
    return res


def filtered_orders(ctx, orders, pred):
    f = D.FilterHandle(ctx, ORDER_TYPES, pred, [0, 1], batch_size=0)        # [o_orderkey, o_custkey]
    f.push_device(orders); f.finish()
    fo = f.drain(host=False)
    f.close()
    return fo


def q13_unfused(ctx, customer, orders):
    fo = filtered_orders(ctx, orders, Q13_PRED)
    j = D.HashJoinHandle(ctx, [D.INT64], [D.INT64, D.INT64], [0], [1], [0, 1], [0, 0], D.JOIN_LEFT, batch_size=1 << 28, ordered_output=False)
    j.push_build_device(customer); j.finish_build()
    agg = D.AggHandle(ctx, [D.INT64, D.INT64], [0], [(D.AGG_COUNT, 1, -1)], D.AGG_SINGLE_PARTITIONED, 1 << 30, customer[0].length)
    for b in fo:
        j.push_probe_device([b.column(0), b.column(1)])
        for jb in j.drain(host=False):
            agg.push_device([jb.column(0), jb.column(1)]); jb.release()
    j.finish_probe()
    for jb in j.drain(host=False):
        agg.push_device([jb.column(0), jb.column(1)]); jb.release()
    agg.finish()
    res = agg.drain(host=False)
    agg.close(); j.close()
    for b in fo:
        b.release()
    return res


def key_fingerprint(ctx, batches):
    rows, s = 0, 0
    for b in batches:
        rows += b.num_rows
        s = (s + D.column_sum_device(ctx, b.column(0))) % (1 << 64)
        b.release()
    return rows, s


def filter_join_fused(ctx, customer, orders, anti):
    look = customer_lookup(ctx, customer, 1)                                 # row counter only
    p = D.Pipeline(ctx, ORDER_TYPES, DATE_PRED, [(D.STAGE_LEFT_ANTI if anti else D.STAGE_INNER, 1, look)], name="left_anti" if anti else "left_semi")
    p.sink_aggregate([1], [], D.AGG_SINGLE)
    p.push_device(orders); p.finish()
    res = p.drain(host=False)
    p.close(); look.close()
    return res


def filter_join_unfused(ctx, customer, orders, anti):
    fo = filtered_orders(ctx, orders, DATE_PRED)
    j = D.HashJoinHandle(ctx, [D.INT64], [D.INT64, D.INT64], [0], [1], [0], [0], D.JOIN_LEFT_ANTI if anti else D.JOIN_LEFT_SEMI, batch_size=1 << 28,
                         ordered_output=False)
    j.push_build_device(customer); j.finish_build()
    out = []
    for b in fo:
        j.push_probe_device([b.column(0), b.column(1)])
        out += j.drain(host=False)
    j.finish_probe()
    out += j.drain(host=False)
    j.close()
    for b in fo:
        b.release()
    return out


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
    customer, orders, _keep = gen(ctx, sf)
    plans = {"q13": (lambda: q13_fused(ctx, customer, orders), lambda: q13_unfused(ctx, customer, orders), lambda r: histogram_of(ctx, r), check_q13)}
    for anti in (False, True):
        name = "left_anti" if anti else "left_semi"
        plans[name] = (lambda anti=anti: filter_join_fused(ctx, customer, orders, anti), lambda anti=anti: filter_join_unfused(ctx, customer, orders, anti),
                       lambda r: key_fingerprint(ctx, r), lambda f, u, name=name: check_keys(name, f, u))
    for name, (fused, unfused, reduce, check) in plans.items():
        for fn in (fused, unfused):   # warm-up
            reduce(fn())
        tf, tu = [], []
        for _ in range(steps):
            a, rf = timed(ctx, fused)
            rf = reduce(rf)
            b, ru = timed(ctx, unfused)
            ru = reduce(ru)
            summary = check(rf, ru)
            tf.append(a); tu.append(b)
        out[name] = {"fused_ms": [round(x, 2) for x in tf], "unfused_ms": [round(x, 2) for x in tu], "check": summary}
        print(json.dumps({name: out[name]}), flush=True)
    out["checks"] = "Q13: c_count histogram equal, per-customer fingerprint equal; semi / anti: row count and key sum equal"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
