"""Full joins through the fused pipeline (a RIGHT stage turned into a Full join, dfgpu_pipeline_set_stage_full) against the unfused GPU
chain, device resident.

    Build: the customers with c_mktsegment = BUILDING (one segment in five: about 3M of SF x 150,000) carrying c_nationkey (Int32, 0..24)
           and an Int32 c_acctbal.  Probe: SF x 1,500,000 orders filtered on o_orderdate < 1200 (uniform over 2406 days: about half),
           joined o_custkey = c_custkey as a Full join.  As in TPC-H, a customer key divisible by 3 has no order, so about 1M BUILDING
           customers are matched by no order and come out with NULL order columns; the orders whose customer is not BUILDING come out
           with NULL customer columns.
    (a) GROUP BY c_nationkey: count(*), sum(o_totalprice), max(c_acctbal) -- the dense sink, 25 nations plus the NULL group; once with
        Int64 money and once with Decimal128(15, 2) money
    (b) the same join GROUP BY (o_orderdate, c_nationkey) -- the hash sink (o_orderdate is NULL on the unmatched customers)
    (c) o_orderkey, o_totalprice, c_nationkey through the unordered output sink
        fused   : customer build pipeline -> lookup with payload and one accumulator word (the visited marks); orders pipeline with a FULL
                  stage into the sink, the unmatched customers pushed through the same sink at finish
        unfused : dfgpu_filter (customers) -> dfgpu_hashjoin build; dfgpu_filter (orders) -> dfgpu_hashjoin(Full) probe -> dfgpu_agg for
                  (a) and (b), the join output for (c)

Fused and unfused runs alternate in one process after a warm-up; each time is a host clock around work that ends in a device synchronise,
the customer build included on both sides.
Checks, on every run: (a) and (b) every group exactly; (c) the row count, the wrapping sum and the NULL count of o_orderkey, the NULL count
of c_nationkey and the sum of its valid values.

usage: python scripts/pipe_full_join_timing.py [SF=100] [steps=3]"""
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
BUILDING, DATE_DAYS, DATE_CUT = 1, 2406, 1200
DEC15 = D.decimal128(15, 2)


# ---- the exact checks (host side; tests/test_pipe_full_join_timing_checks.py runs them on tiny data) ----
def group_rows(columns, n_keys) -> dict:
    """[(values, valid or None)] per column (a Decimal128 column as [n, 2] words) -> {group key tuple: aggregate tuple}, NULL as None"""
    def py(c):
        v, m = c
        v = np.asarray(v)
        if v.ndim == 2:   # Decimal128 words -> signed Python ints
            vals = [int(lo) | (int(hi) << 64) for lo, hi in v.tolist()]
            vals = [x - (1 << 128) if x >= 1 << 127 else x for x in vals]
        else:
            vals = v.tolist()
        return [None if (m is not None and not m[i]) else vals[i] for i in range(len(vals))]
    cols = [py(c) for c in columns]
    out = {}
    for r in zip(*cols):
        k = tuple(r[:n_keys])
        assert k not in out, f"group {k} appears twice"
        out[k] = tuple(r[n_keys:])
    return out


def check_groups(name, fused: dict, unfused: dict) -> dict:
    assert fused.keys() == unfused.keys(), f"{name}: {len(fused)} groups fused, {len(unfused)} unfused, or different keys"
    bad = [k for k in fused if fused[k] != unfused[k]]
    assert not bad, f"{name}: groups differ, e.g. {bad[0]}: {fused[bad[0]]} != {unfused[bad[0]]}"
    null_rows = sum(v[0] for k, v in fused.items() if k[-1] is None)
    return {"groups": len(fused), "rows": sum(v[0] for v in fused.values()), "null_nation_rows": null_rows}


def output_summary(rows, key_sum, key_nulls, nation_nulls, nation_sum) -> tuple:
    return int(rows), int(key_sum) % (1 << 64), int(key_nulls), int(nation_nulls), int(nation_sum) % (1 << 64)


def check_output(fused: tuple, unfused: tuple) -> dict:
    """(rows, wrapping sum of the valid o_orderkey values, o_orderkey NULLs, c_nationkey NULLs, wrapping sum of the valid c_nationkey
    values)"""
    assert fused == unfused, f"output: fused {fused} != unfused {unfused}"
    return {"rows": fused[0], "key_sum": f"{fused[1]:#x}", "key_nulls": fused[2], "nation_nulls": fused[3], "nation_sum": fused[4]}


# ---- device side ----
def dcol(buf, n, t=D.INT64):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = t, 0, n, 0, 0, buf.ptr, None
    return c


def gen(ctx, sf, seed=17):
    n_cust, n_ord = int(150_000 * sf), int(1_500_000 * sf)
    rng = np.random.default_rng(seed)
    keep = [ctx.to_device(np.arange(1, n_cust + 1, dtype=np.int64)), ctx.to_device(rng.integers(0, 5, n_cust).astype(np.int32)),
            ctx.to_device(rng.integers(0, 25, n_cust).astype(np.int32)), ctx.to_device(rng.integers(-99_999, 999_999, n_cust).astype(np.int32))]
    customer = [dcol(keep[0], n_cust), dcol(keep[1], n_cust, D.INT32), dcol(keep[2], n_cust, D.INT32), dcol(keep[3], n_cust, D.INT32)]
    price = rng.integers(90_000, 50_000_000, n_ord).astype(np.int64)
    words = np.zeros((n_ord, 2), np.uint64)
    words[:, 0] = price.view(np.uint64)
    u = rng.integers(0, 2 * (n_cust // 3), n_ord)
    custkey = (u // 2) * 3 + 1 + u % 2                                          # 1, 2, 4, 5, ...: no key divisible by 3 (TPC-H)
    del u
    keep += [ctx.to_device(np.arange(1, n_ord + 1, dtype=np.int64)), ctx.to_device(custkey.astype(np.int64)),
             ctx.to_device(rng.integers(0, DATE_DAYS, n_ord).astype(np.int32)), ctx.to_device(price), ctx.to_device(words)]
    del price, words, custkey
    orders = {False: [dcol(keep[4], n_ord), dcol(keep[5], n_ord), dcol(keep[6], n_ord, D.DATE32), dcol(keep[7], n_ord)],
              True: [dcol(keep[4], n_ord), dcol(keep[5], n_ord), dcol(keep[6], n_ord, D.DATE32), dcol(keep[8], n_ord, DEC15)]}
    return customer, orders, keep


CUST_TYPES = [D.INT64, D.INT32, D.INT32, D.INT32]          # c_custkey, c_mktsegment, c_nationkey, c_acctbal
CUST_PRED = [C(1), L(BUILDING, D.INT32), B(D.OP_EQ)]
ORD_PRED = [C(2), L(DATE_CUT, D.DATE32), B(D.OP_LT)]


def ord_types(dec):
    return [D.INT64, D.INT64, D.DATE32, DEC15 if dec else D.INT64]   # o_orderkey, o_custkey, o_orderdate, o_totalprice


# aggregates over the orders pipeline's virtual columns: 4 c_nationkey, 5 c_acctbal
AGGS = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, [C(3)]), (D.AGG_MAX, [C(5)])]


def customer_lookup(ctx, customer):
    look = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], expected_rows=customer[0].length // 4, n_acc_words=1)
    p = D.Pipeline(ctx, CUST_TYPES, CUST_PRED)
    p.sink_build(look, 0, [2, 3]); p.push_device(customer); p.finish(); p.close()
    return look


def fused(ctx, customer, orders, plan, dec):
    look = customer_lookup(ctx, customer)
    p = D.Pipeline(ctx, ord_types(dec), ORD_PRED, [(D.STAGE_RIGHT, 1, look)], name="full_" + plan)
    p.set_stage_full(0)
    if plan == "dense":
        p.sink_aggregate_dense([4], [(0, 24)], AGGS, D.AGG_SINGLE)
    elif plan == "hash":
        p.sink_aggregate_hash([2, 4], AGGS, D.AGG_SINGLE, nullable=[True, True], capacity_hint=(DATE_CUT + 1) * 26)
    else:
        p.sink_output([0, 3, 4], ordered=False)
    p.push_device(orders); p.finish()
    res = p.drain(host=False)
    p.close(); look.close()
    return res


def unfused(ctx, customer, orders, plan, dec):
    fc = D.FilterHandle(ctx, CUST_TYPES, CUST_PRED, [0, 2, 3], batch_size=0)
    fc.push_device(customer); fc.finish()
    cb = fc.drain(host=False)
    fc.close()
    fo = D.FilterHandle(ctx, ord_types(dec), ORD_PRED, [0, 1, 2, 3], batch_size=0)
    fo.push_device(orders); fo.finish()
    ob = fo.drain(host=False)
    fo.close()
    # join output: o_orderkey, o_orderdate, o_totalprice, c_nationkey, c_acctbal
    j = D.HashJoinHandle(ctx, [D.INT64, D.INT32, D.INT32], ord_types(dec), [0], [1], [1, 1, 1, 0, 0], [0, 2, 3, 1, 2], D.JOIN_FULL, batch_size=1 << 28,
                         ordered_output=False)
    for b in cb:
        j.push_build_device([b.column(0), b.column(1), b.column(2)])
    j.finish_build()
    out, agg = [], None
    if plan != "output":
        gcols = [3] if plan == "dense" else [1, 3]
        agg = D.AggHandle(ctx, [D.INT64, D.DATE32, DEC15 if dec else D.INT64, D.INT32, D.INT32], gcols,
                          [(D.AGG_COUNT_STAR, -1, -1), (D.AGG_SUM, 2, -1), (D.AGG_MAX, 4, -1)], D.AGG_SINGLE, 1 << 30, 64 if plan == "dense" else (DATE_CUT + 1) * 26)

    def take(batches):
        for jb in batches:
            if agg is None:
                out.append(jb)
            else:
                agg.push_device([jb.column(i) for i in range(5)]); jb.release()
    for b in ob:
        j.push_probe_device([b.column(i) for i in range(4)])
        take(j.drain(host=False))
    j.finish_probe()
    take(j.drain(host=False))
    j.close()
    for b in cb + ob:
        b.release()
    if agg is None:
        return out
    agg.finish()
    res = agg.drain(host=False)
    agg.close()
    return res


def reduce_groups(batches, n_keys):
    """the aggregate batches -> {group: (count, sum, max)}"""
    cols = None
    for b in batches:
        cs = [b.column_numpy(i) for i in range(b.num_columns)]
        if cols is None:
            cols = [([], []) for _ in cs]
        for i, (v, m) in enumerate(cs):
            cols[i][0].append(v); cols[i][1].append(np.ones(len(v), bool) if m is None else m)
        b.release()
    if cols is None:
        return {}
    return group_rows([(np.concatenate(v), np.concatenate(m)) for v, m in cols], n_keys)


def reduce_output(ctx, batches, key_col, nation_col):
    rows, ks, kn, nn, ns = 0, 0, 0, 0, 0
    for b in batches:
        rows += b.num_rows
        ks += D.column_sum_device(ctx, b.column(key_col))
        ns += D.column_sum_device(ctx, b.column(nation_col))
        _, m = b.column_numpy(key_col)
        kn += 0 if m is None else int((~m).sum())
        _, m = b.column_numpy(nation_col)
        nn += 0 if m is None else int((~m).sum())
        b.release()
    return output_summary(rows, ks, kn, nn, ns)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
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
    plans = {}
    for name, plan, dec in (("a_dense_int64", "dense", False), ("a_dense_decimal", "dense", True), ("b_hash", "hash", False), ("c_output", "output", False)):
        if plan == "output":
            red_f, red_u = (lambda r: reduce_output(ctx, r, 0, 2)), (lambda r: reduce_output(ctx, r, 0, 3))
            check = check_output
        else:
            nk = 1 if plan == "dense" else 2
            red_f = red_u = (lambda r, nk=nk: reduce_groups(r, nk))
            check = (lambda f, u, name=name: check_groups(name, f, u))
        plans[name] = (lambda plan=plan, dec=dec: fused(ctx, customer, orders[dec], plan, dec),
                       lambda plan=plan, dec=dec: unfused(ctx, customer, orders[dec], plan, dec), red_f, red_u, check)
    for name, (f, u, red_f, red_u, check) in plans.items():
        red_f(f()); red_u(u())   # warm-up
        tf, tu = [], []
        for _ in range(steps):
            a, rf = timed(ctx, f)
            rf = red_f(rf)
            b, ru = timed(ctx, u)
            ru = red_u(ru)
            summary = check(rf, ru)
            tf.append(a); tu.append(b)
        out[name] = {"fused_ms": [round(x, 2) for x in tf], "unfused_ms": [round(x, 2) for x in tu], "fused_median_ms": round(float(np.median(tf)), 2),
                     "unfused_median_ms": round(float(np.median(tu)), 2), "check": summary}
        print(json.dumps({name: out[name]}), flush=True)
    out["checks"] = "(a), (b): every group equal; (c): row count, o_orderkey valid sum and NULL count, c_nationkey NULL count and valid sum equal"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
