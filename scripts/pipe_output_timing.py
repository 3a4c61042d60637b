"""The fused pipeline's output sinks with nullable and Decimal128 columns, device resident, against what they replace.

    (a) Q3's orders chain: o_orderdate < CUT, SEMI on the customer bitmap (c_mktsegment = 1) -> ordered output of o_orderkey,
        o_orderdate, o_shippriority and a nullable Decimal128(15,2) o_totalprice.  SF x 1,500,000 orders, SF x 150,000 customers.
          fused        : one pipeline, dfgpu_pipeline_sink_output (pipe_output_cols_kernel)
          unfused      : dfgpu_filter -> dfgpu_hashjoin(RightSemi), the customer keys as the build side
          fused, Int64 : the same pipeline with an Int64 o_totalprice without bitmap (the instantiation that ran before)
        Every arm builds its customer side (the fused pipelines' bitmap lookup, the join's table) inside the timer, from the same
        device-resident key column.
    (b) the multi-GPU plan's lineitem scan: l_shipdate > CUT, MAYBE on the orders filter -> unordered output of l_orderkey and Decimal128
        l_extendedprice / l_discount.  SF x 6,000,000 lineitem rows.
          fused        : dfgpu_pipeline_sink_output_unordered (pipe_kernel VAR bit 512)
          fused, Int64 : the same pipeline with Int64 money (the instantiation that ran before)

Data come from the counter-based generators (dfgpu_generate_i64); the validity bitmap of o_totalprice is random words (half the rows
NULL).  The arms alternate in one process after a warm-up; each time is a host clock around work that ends in a device synchronise.
Checks, on every run: (a) the fused and unfused outputs are equal row for row, values and validity, and the Int64 run has the same rows;
(b) the Decimal128 and Int64 runs keep the same number of rows and the same wrapping sum of l_orderkey.

usage: python scripts/pipe_output_timing.py [SF=100] [steps=3]"""
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
CAST = lambda t: (D.EXPR_CAST, 0, t, 0, 0, 0.0)                               # noqa: E731
CUT = 9204                                                                    # 1995-03-15 as Date32
DEC = D.decimal128(15, 2)


def dcol(buf, n, t=D.INT64, valid=None):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count = t, 0, n, 0, (-1 if valid is not None else 0)
    c.values, c.validity = buf.ptr, (valid.ptr if valid is not None else None)
    return c


def narrow(ctx, keep, buf, n, t):
    b = D.evaluate_device(ctx, [dcol(buf, n)], n, [C(0), CAST(t)])
    keep.append(b)
    return b.column(0)


def gen(ctx, sf, seed=3):
    no, nl, nc = int(1_500_000 * sf), int(6_000_000 * sf), int(150_000 * sf)
    keep = []
    g = lambda k, lo, hi, n: ctx.generate_i64(D.GEN_UNIFORM, seed + k, lo, hi - lo + 1, 0, n)   # noqa: E731  values in [lo, hi]
    okey = ctx.generate_i64(D.GEN_SEQ, 0, 1, 0, 0, no)
    ocust, price_i, price_d = g(1, 1, nc, no), g(4, 90_000, 50_000_000, no), g(5, 0, 10**9, 2 * no)
    mask = ctx.generate_i64(D.GEN_SPLITMIX, seed + 6, 0, 0, 0, (no + 63) // 64)
    keep += [okey, ocust, price_i, price_d, mask]
    d32, p32 = narrow(ctx, keep, g(2, 8035, 10592, no), no, D.DATE32), narrow(ctx, keep, g(3, 0, 0, no), no, D.INT32)   # the Int64 draws are freed
    orders_dec = [dcol(okey, no), dcol(ocust, no), d32, p32, dcol(price_d, no, DEC, mask)]
    orders_i64 = [dcol(okey, no), dcol(ocust, no), d32, p32, dcol(price_i, no)]
    lkey = g(7, 1, no, nl)                                                                      # l_orderkey: an existing o_orderkey
    lp_i, ld_i, lp_d, ld_d = g(9, 90_000, 10_500_000, nl), g(10, 0, 10, nl), g(11, 0, 10**9, 2 * nl), g(12, 0, 10, 2 * nl)
    keep += [lkey, lp_i, ld_i, lp_d, ld_d]
    s32 = narrow(ctx, keep, g(8, 8035, 10592, nl), nl, D.DATE32)
    li_dec = [dcol(lkey, nl), dcol(lp_d, nl, DEC), dcol(ld_d, nl, DEC), s32]
    li_i64 = [dcol(lkey, nl), dcol(lp_i, nl), dcol(ld_i, nl), s32]
    rng = np.random.default_rng(seed)
    cust_keys = np.nonzero(rng.integers(0, 5, nc) == 1)[0].astype(np.int64) + 1
    ctx.sync()
    return orders_dec, orders_i64, li_dec, li_i64, cust_keys, nc, keep


ORD_DEC = [D.INT64, D.INT64, D.DATE32, D.INT32, DEC]
ORD_I64 = [D.INT64, D.INT64, D.DATE32, D.INT32, D.INT64]
LI_DEC = [D.INT64, DEC, DEC, D.DATE32]
LI_I64 = [D.INT64, D.INT64, D.INT64, D.DATE32]
OPRED = [C(2), L(CUT, D.DATE32), B(D.OP_LT)]
LPRED = [C(3), L(CUT, D.DATE32), B(D.OP_GT)]
OUT_A = [0, 2, 3, 4]                       # o_orderkey, o_orderdate, o_shippriority, o_totalprice


def to_host(batches, ncols):
    out = []
    for c in range(ncols):
        parts = [b.column_numpy(c) for b in batches]
        v = np.concatenate([x for x, _ in parts]) if parts else np.zeros(0)
        anyv = any(m is not None for _, m in parts)
        out.append((v, np.concatenate([np.ones(len(x), bool) if m is None else m for x, m in parts]) if anyv else None))
    return out


def same(a, b, what):
    assert len(a) == len(b), what
    for c, ((av, am), (bv, bm)) in enumerate(zip(a, b)):
        assert (am is None) == (bm is None), f"{what}: column {c} bitmap"
        assert len(av) == len(bv), f"{what}: column {c} rows"
        if am is not None:
            assert np.array_equal(am, bm), f"{what}: column {c} validity"
            av, bv = av[am], bv[bm]
        assert np.array_equal(np.ascontiguousarray(av).view(np.uint8), np.ascontiguousarray(bv).view(np.uint8)), f"{what}: column {c} values"


def timed(ctx, fn):
    ctx.sync()
    t0 = time.perf_counter()
    r = fn()
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3, r


def fused_a(ctx, ckeys, nc, cols, types):
    """the customer bitmap built from the device-resident keys, then the orders pipeline"""
    lcust = D.Lookup(ctx, D.INT64, [], key_range=(1, nc))
    b = D.Pipeline(ctx, [D.INT64]); b.sink_build(lcust, 0, []); b.push_device([ckeys]); b.finish(); b.close()
    p = D.Pipeline(ctx, types, OPRED, [(D.STAGE_SEMI, 1, lcust)])
    p.sink_output(OUT_A)
    p.push_device(cols); p.finish()
    out = p.drain(host=False)
    p.close(); lcust.close()
    return out


def unfused_a(ctx, ckeys, cols):
    """the join's table built from the same device-resident keys, the filter's output probing it"""
    f = D.FilterHandle(ctx, ORD_DEC, OPRED, batch_size=1 << 30)
    f.push_device(cols); f.finish()
    fb = f.drain(host=False)
    j = D.HashJoinHandle(ctx, [D.INT64], ORD_DEC, [0], [1], [1] * 4, OUT_A, D.JOIN_RIGHT_SEMI, batch_size=1 << 30)
    j.push_build_device([ckeys]); j.finish_build()
    for b in fb:
        j.push_probe_device([b.column(i) for i in range(len(ORD_DEC))])
    j.finish_probe()
    out = j.drain(host=False)
    j.close(); f.close()
    return out


def fused_b(ctx, filt, cols, types):
    p = D.Pipeline(ctx, types, LPRED, [(D.STAGE_MAYBE, 0, filt)])
    p.sink_output([0, 1, 2], ordered=False)
    p.push_device(cols); p.finish()
    out = p.drain(host=False)
    p.close()
    return out


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    ctx = D.Context(0)
    orders_dec, orders_i64, li_dec, li_i64, cust_keys, nc, keep = gen(ctx, sf)
    ckeys_buf = ctx.to_device(cust_keys)                 # both arms of shape (a) build their customer side from these, inside the timer
    ckeys = dcol(ckeys_buf, len(cust_keys))
    filt = D.Lookup(ctx, D.INT64, [], expected_rows=int(750_000 * sf), filter_only=True)
    b = D.Pipeline(ctx, ORD_I64, OPRED); b.sink_build(filt, 0, []); b.push_device(orders_i64); b.finish(); b.close()
    arms = {
        "a_fused": lambda: fused_a(ctx, ckeys, nc, orders_dec, ORD_DEC),
        "a_unfused": lambda: unfused_a(ctx, ckeys, orders_dec),
        "a_fused_int64": lambda: fused_a(ctx, ckeys, nc, orders_i64, ORD_I64),
        "b_fused": lambda: fused_b(ctx, filt, li_dec, LI_DEC),
        "b_fused_int64": lambda: fused_b(ctx, filt, li_i64, LI_I64),
    }
    for fn in arms.values():   # warm-up
        for o in fn():
            o.release()
    times = {k: [] for k in arms}
    checks = {}
    for _ in range(steps):
        res, rows_b = {}, []
        for name, fn in arms.items():
            ms, out = timed(ctx, fn)
            times[name].append(ms)
            if name.startswith("b_"):   # shape (b)'s outputs are summarised and freed at once: two of them do not fit beside the inputs
                n = sum(o.num_rows for o in out)
                ks = sum(D.column_sum_device(ctx, o.column(0)) for o in out) % (1 << 64)
                rows_b.append((n, ks))
                for o in out:
                    o.release()
            else:
                res[name] = out
        fa, ua, ia = (to_host(res[k], 4) for k in ("a_fused", "a_unfused", "a_fused_int64"))
        same(fa, ua, "shape (a): fused vs dfgpu_filter -> dfgpu_hashjoin(RightSemi)")
        same(fa[:3], ia[:3], "shape (a): Decimal128 vs Int64 money, the other columns")
        assert rows_b[0] == rows_b[1], f"shape (b): Decimal128 {rows_b[0]} != Int64 {rows_b[1]}"
        checks = {"a_rows": len(fa[0][0]), "a_null_prices": int((~fa[3][1]).sum()), "b_rows": rows_b[0][0]}
        for outs in res.values():
            for o in outs:
                o.release()
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"sf": sf, "steps": steps, "card": card, "median_ms": med, "all_ms": times, "checks": checks, "equal": True}), flush=True)
    filt.close()
    del keep, ckeys_buf


if __name__ == "__main__":
    main()
