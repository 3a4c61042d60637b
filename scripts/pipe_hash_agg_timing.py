"""The fused pipeline's hash-keyed aggregate sink (dfgpu_pipeline_sink_aggregate_hash) against the best unfused GPU chain, device resident.

    Q15 revenue0: FilterExec(1996-01-01 <= l_shipdate < 1996-04-01) -> AggregateExec GROUP BY l_suppkey
                  SUM(l_extendedprice * (1 - l_discount)),  l_suppkey uniform over SF x 10,000
        fused   : one pipeline, the hash sink
        unfused : dfgpu_filter -> dfgpu_expr_evaluate_device -> dfgpu_agg
    Q3 by customer: the Q3 join (scripts/q3_device_pipeline.py) grouped by o_custkey, SUM(l_extendedprice * (1 - l_discount))
        fused   : customer and orders build pipelines (orders carries o_custkey as payload), the lineitem pipeline into the hash sink
        unfused : the same build pipelines, the lineitem pipeline into the unordered output sink -> dfgpu_expr_evaluate_device ->
                  dfgpu_agg.  The output sink carries no 16-byte column, so with Decimal128 money it emits the Int64 money columns and
                  the chain casts them to Decimal128(15,2) on the device (the same unscaled integers) before the expression.

Tables come from dfgpu_generate_i64 (q3_device_pipeline.gen_tables, seeded), with Int64 money and with Decimal128(15,2) money.  Fused
and unfused runs alternate in one process after a warm-up; each time is a host clock around work that ends in a device synchronise, and
the kernel split of one more run of each comes from dfgpu_kernel_time.  Every run is checked group by group, exactly: fused against
unfused, and the Decimal128 result against the Int64 one.

usage: python scripts/pipe_hash_agg_timing.py [SF=100] [steps=3]"""
import datetime
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from datafusion_b200 import capi as D
from q3_device_pipeline import B, C, CAST, CUT, L, Table, decimal_money, gen_tables, revenue_expr

EPOCH = datetime.date(1970, 1, 1)
day = lambda y, m, d: (datetime.date(y, m, d) - EPOCH).days
Q15_LO, Q15_HI = day(1996, 1, 1), day(1996, 4, 1)
WINDOW = B(D.OP_AND, B(D.OP_GTEQ, C(3), L(Q15_LO, D.INT32)), B(D.OP_LT, C(3), L(Q15_HI, D.INT32)))


def with_suppkey(ctx, lineitem, nsupp, seed=11):
    """lineitem + column 4 l_suppkey, uniform over [1, nsupp]"""
    buf = ctx.generate_i64(D.GEN_UNIFORM, seed, 1, nsupp, 0, lineitem.rows)
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = D.INT64, 0, lineitem.rows, 0, 0, buf.ptr, None
    return Table(lineitem.names + ["l_suppkey"], lineitem.types + [D.INT64], list(lineitem.cols) + [c], lineitem.rows, list(lineitem._keep) + [buf])


def drain_cols(batches):
    """device result batches [key, sum] -> (keys int64, sums as Python-comparable int64 or 128-bit word pairs)"""
    ks, vs = [], []
    for b in batches:
        k, _ = b.column_numpy(0)
        v, _ = b.column_numpy(1)
        ks.append(np.asarray(k, np.int64)); vs.append(np.asarray(v).reshape(len(k), -1))
        b.release()
    k = np.concatenate(ks) if ks else np.zeros(0, np.int64)
    v = np.concatenate(vs) if vs else np.zeros((0, 1), np.uint64)
    o = np.argsort(k, kind="stable")
    return k[o], v[o]


def as_i64(v):
    """Decimal128 sums [n, 2] words that fit int64 (checked) -> int64; Int64 sums [n, 1] -> int64"""
    if v.shape[1] == 1:
        return v[:, 0].view(np.int64) if v.dtype == np.uint64 else v[:, 0].astype(np.int64)
    lo = v[:, 0].view(np.int64)
    assert (v[:, 1].view(np.int64) == (lo >> 63)).all(), "a Decimal128 sum outside int64"
    return lo


def q15_fused(ctx, t, nsupp):
    p = D.Pipeline(ctx, t.types, WINDOW, name="q15_hash")
    p.sink_aggregate_hash([4], [(D.AGG_SUM, revenue_expr(t.types))], D.AGG_SINGLE_PARTITIONED, 0, nsupp)
    p.push_device(t.cols); p.finish()
    res = p.drain(host=False)
    m = {k: p.metric(k) for k in ("sink_rows", "num_groups", "group_rehashes", "replayed_rows")}
    p.close()
    return res, m


def q15_unfused(ctx, t, nsupp):
    f = D.FilterHandle(ctx, t.types, WINDOW, [4, 1, 2], batch_size=0)   # [l_suppkey, price, discount]: revenue_expr's columns 1 and 2
    f.push_device(t.cols); f.finish()
    fo = f.drain(host=False)
    f.close()
    res = []
    if fo:
        n = fo[0].num_rows
        cols = [fo[0].column(i) for i in range(3)]
        rev = D.evaluate_device(ctx, cols, n, revenue_expr([D.INT64, t.types[1], t.types[2]]))
        rc = rev.column(0)
        agg = D.AggHandle(ctx, [D.INT64, rc.type], [0], [(D.AGG_SUM, 1, -1)], D.AGG_SINGLE_PARTITIONED, 8192, nsupp)
        agg.push_device([cols[0], rc]); agg.finish()
        res = agg.drain(host=False)
        agg.close(); rev.release()
    for b in fo:
        b.release()
    return res


def q3_builds(ctx, customer, orders):
    kmin, kmax, _ = D.column_minmax_device(ctx, customer.cols[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p1 = D.Pipeline(ctx, customer.types, B(D.OP_EQ, C(1), L(1)))
    p1.sink_build(l1, 0, []); p1.push_device(customer.cols); p1.finish(); p1.close()
    l2 = D.Lookup(ctx, D.INT64, [D.INT64], membership_filter=-1)                     # o_orderkey -> o_custkey
    p2 = D.Pipeline(ctx, orders.types, B(D.OP_LT, C(2), L(CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)], name="orders")
    p2.sink_build(l2, 0, [1]); p2.push_device(orders.cols); p2.finish(); p2.close()
    return l1, l2


def q3_fused(ctx, customer, orders, lineitem, ncust):
    l1, l2 = q3_builds(ctx, customer, orders)
    p = D.Pipeline(ctx, lineitem.types, B(D.OP_GT, C(3), L(CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="q3_cust_hash")
    p.sink_aggregate_hash([len(lineitem.types)], [(D.AGG_SUM, revenue_expr(lineitem.types))], D.AGG_SINGLE_PARTITIONED, 0, ncust)   # o_custkey
    p.push_device(lineitem.cols); p.finish()
    res = p.drain(host=False)
    m = {k: p.metric(k) for k in ("sink_rows", "num_groups", "group_rehashes", "replayed_rows")}
    p.close(); l2.close(); l1.close()
    return res, m


def q3_unfused(ctx, customer, orders, lineitem_i64, dec, ncust):
    l1, l2 = q3_builds(ctx, customer, orders)
    p = D.Pipeline(ctx, lineitem_i64.types, B(D.OP_GT, C(3), L(CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="q3_cust_output")
    p.sink_output([len(lineitem_i64.types), 1, 2], ordered=False)                     # [o_custkey, price, discount]
    p.push_device(lineitem_i64.cols); p.finish()
    jo = p.drain(host=False)
    p.close(); l2.close(); l1.close()
    res, keep = [], []
    if jo:
        assert len(jo) == 1
        n = jo[0].num_rows
        cols = [jo[0].column(i) for i in range(3)]
        if dec:
            for i in (1, 2):
                b = D.evaluate_device(ctx, [cols[i]], n, CAST(C(0), D.decimal128(15, 0))); keep.append(b)
                cols[i] = b.column(0); cols[i].type = D.decimal128(15, 2)
        rev = D.evaluate_device(ctx, cols, n, revenue_expr([D.INT64, cols[1].type, cols[2].type])); keep.append(rev)
        rc = rev.column(0)
        agg = D.AggHandle(ctx, [D.INT64, rc.type], [0], [(D.AGG_SUM, 1, -1)], D.AGG_SINGLE_PARTITIONED, 8192, ncust)
        agg.push_device([cols[0], rc]); agg.finish()
        res = agg.drain(host=False)
        agg.close()
    for b in keep + jo:
        b.release()
    return res


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


def kernel_split(ctx, fn, families):
    ctx.set_kernel_timing(True); ctx.kernel_time_reset()
    r = fn()
    ctx.sync()
    kt = {k: round(ctx.kernel_time(k)[0], 3) for k in families}
    ctx.set_kernel_timing(False)
    return kt, r


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100.0
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    ctx = D.Context(0)
    out = {"sf": sf, "card": card(), "steps": steps}
    customer, orders, li = gen_tables(ctx, sf)
    nsupp, ncust = int(sf * 10_000), int(150_000 * sf)
    li = with_suppkey(ctx, li, nsupp)
    ld = decimal_money(ctx, li)
    ref = {}
    families = ["pipe:q15_hash", "filter", "expr", "agg_update", "pipe:orders", "pipe:q3_cust_hash", "pipe:q3_cust_output", "pipeline_build"]
    for money, t in (("int64", li), ("decimal", ld)):
        dec = money == "decimal"
        plans = {"q15": (lambda t=t: q15_fused(ctx, t, nsupp)[0], lambda t=t: q15_unfused(ctx, t, nsupp)),
                 "q3_by_custkey": (lambda t=t: q3_fused(ctx, customer, orders, t, ncust)[0], lambda dec=dec: q3_unfused(ctx, customer, orders, li, dec, ncust))}
        for name, (fused, unfused) in plans.items():
            for fn in (fused, unfused):   # warm-up
                for b in fn():
                    b.release()
            tf, tu = [], []
            for _ in range(steps):
                a, rf = timed(ctx, fused)
                b, ru = timed(ctx, unfused)
                kf, vf = drain_cols(rf)
                ku, vu = drain_cols(ru)
                assert np.array_equal(kf, ku) and np.array_equal(vf, vu), f"{name} {money}: fused != unfused"
                tf.append(a); tu.append(b)
            sums = as_i64(vf)
            if name in ref:
                assert np.array_equal(ref[name][0], kf) and np.array_equal(ref[name][1], sums), f"{name}: Decimal128 != Int64"
            ref[name] = (kf, sums)
            m = (q15_fused(ctx, t, nsupp) if name == "q15" else q3_fused(ctx, customer, orders, t, ncust))
            for b in m[0]:
                b.release()
            kfu, r1 = kernel_split(ctx, fused, families)
            for b in r1:
                b.release()
            kun, r2 = kernel_split(ctx, unfused, families)
            for b in r2:
                b.release()
            out[f"{name}_{money}"] = {"fused_ms": [round(x, 2) for x in tf], "unfused_ms": [round(x, 2) for x in tu], "groups": int(len(kf)),
                                      "metrics": m[1], "fused_kernels_ms": {k: v for k, v in kfu.items() if v},
                                      "unfused_kernels_ms": {k: v for k, v in kun.items() if v}}
            print(json.dumps({f"{name}_{money}": out[f"{name}_{money}"]}), flush=True)
    out["checks"] = "fused == unfused group by group; Decimal128 == Int64"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
