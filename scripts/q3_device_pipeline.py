"""BASELINE config C4, device resident: the TPC-H Q3-shaped operator pipeline of the reference's physical plan
(sqllogictest/test_files/tpch/plans/q3.slt.part:60-76), every operator through the C ABI with HBM-resident columns:

    FilterExec(c_mktsegment = 1)                                   customer   (1 = 'BUILDING')
    FilterExec(o_orderdate < 1995-03-15)                           orders
    HashJoinExec RightSemi (c_custkey = o_custkey)                 -> orders of BUILDING customers
    FilterExec(l_shipdate > 1995-03-15)                            lineitem
    HashJoinExec Inner (o_orderkey = l_orderkey)
    ProjectionExec rev = l_extendedprice * (100 - l_discount)      (int64 fixed point: cents x hundredths, exact)
    AggregateExec gby [l_orderkey, o_orderdate, o_shippriority] SUM(rev)

Tables are synthetic with TPC-H cardinalities (SF x 150k customers, 1.5M orders, 6M lineitems), generated in HBM with the
counter-based generators + the expression kernels: sparse order keys (8 of every 32, as dbgen), a third of the customers
without orders, dates uniform over 1992-01-01..1998-08-02 (+ up to 121 days for ship dates).  Dates are int32 days."""
import datetime

import numpy as np

from datafusion_b200 import capi as D

EPOCH = datetime.date(1970, 1, 1)
D0, D1 = (datetime.date(1992, 1, 1) - EPOCH).days, (datetime.date(1998, 8, 2) - EPOCH).days
CUT = (datetime.date(1995, 3, 15) - EPOCH).days


def C(i): return [(D.EXPR_COLUMN, i, 0, 0, 0, 0.0)]
def L(v, t=None): return [(D.EXPR_LITERAL, 0, t if t is not None else D.INT64, 0, int(v), 0.0)]
def B(op, l, r): return l + r + [(D.EXPR_BINARY, op, 0, 0, 0, 0.0)]
def CAST(e, t): return e + [(D.EXPR_CAST, 0, t, 0, 0, 0.0)]


class Table:
    def __init__(self, names, types, cols, rows, keep):
        self.names, self.types, self.cols, self.rows, self._keep = names, types, cols, rows, keep

    def host(self, ctx):
        return {n: ctx.to_host(c.values, self.rows * D.WIDTH[t]).view(D.NP_OF_TYPE[t]).copy() for n, t, c in zip(self.names, self.types, self.cols)}


def _col(buf, n, t=None):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = (t if t is not None else D.INT64), 0, n, 0, 0, buf.ptr, None
    return c


def gen_tables(ctx, sf, seed=1, rank=0, world=1):
    """rank's shard (rows [rank*n, (rank+1)*n) of every table) of the SF(sf*world) database; world == 1 is the whole SF(sf) database"""
    nc, no, nl = int(150_000 * sf), int(1_500_000 * sf), int(6_000_000 * sf)
    NC, NO = nc * world, no * world
    keep = []

    def gen(kind, s, a, b, n, start=0):
        buf = ctx.generate_i64(kind, s, a, b, start, n); keep.append(buf)
        return _col(buf, n)

    def ev(cols, n, nodes):
        b = D.evaluate_device(ctx, cols, n, nodes); keep.append(b)
        c = b.column(0)
        c.validity = None; c.null_count = 0          # inputs have no NULLs
        return c

    sparse = lambda e: B(D.OP_PLUS, B(D.OP_PLUS, B(D.OP_MULTIPLY, B(D.OP_DIVIDE, e, L(8)), L(32)), B(D.OP_MODULO, e, L(8))), L(1))   # 8 of every 32 keys
    customer = Table(["c_custkey", "c_mktsegment"], [D.INT64, D.INT64], [gen(D.GEN_SEQ, 0, 1 + rank * nc, 0, nc), gen(D.GEN_UNIFORM, seed + 1, 0, 5, nc, rank * nc)], nc, keep)
    oidx = gen(D.GEN_SEQ, 0, rank * no, 0, no)
    orders = Table(["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"], [D.INT64, D.INT64, D.INT32, D.INT32],
                   [ev([oidx], no, sparse(C(0))), gen(D.GEN_UNIFORM, seed + 2, 1, max(NC * 2 // 3, 1), no, rank * no),
                    ev([gen(D.GEN_UNIFORM, seed + 3, D0, D1 - D0 + 1, no, rank * no)], no, CAST(C(0), D.INT32)),
                    ev([oidx], no, CAST(B(D.OP_MULTIPLY, C(0), L(0)), D.INT32))], no, keep)
    lidx = gen(D.GEN_UNIFORM, seed + 4, 0, NO, nl, rank * nl)
    lineitem = Table(["l_orderkey", "l_extendedprice", "l_discount", "l_shipdate"], [D.INT64, D.INT64, D.INT64, D.INT32],
                     [ev([lidx], nl, sparse(C(0))), gen(D.GEN_UNIFORM, seed + 5, 90_000, 10_410_000, nl, rank * nl), gen(D.GEN_UNIFORM, seed + 6, 0, 11, nl, rank * nl),
                      ev([gen(D.GEN_UNIFORM, seed + 7, D0 + 1, D1 - D0 + 121, nl, rank * nl)], nl, CAST(C(0), D.INT32))], nl, keep)
    ctx.sync()
    return customer, orders, lineitem


def _filter(ctx, t, nodes, projection):
    f = D.FilterHandle(ctx, t.types, nodes, projection, batch_size=0)
    f.push_device(t.cols); f.finish()
    outs = f.drain(host=False)
    f.close()
    return outs


def _bcols(batches):
    assert len(batches) == 1, "the pipeline runs on whole-table batches"
    return [batches[0].column(i) for i in range(batches[0].num_columns)]


def run_q3(ctx, customer, orders, lineitem):
    """returns (result batches [l_orderkey, o_orderdate, o_shippriority, revenue], stage row counts)"""
    stages = {}
    c = _filter(ctx, customer, B(D.OP_EQ, C(1), L(1)), [0])
    o = _filter(ctx, orders, B(D.OP_LT, C(2), L(CUT, D.INT32)), None)
    stages["customer_building"], stages["orders_before_cut"] = c[0].num_rows if c else 0, o[0].num_rows if o else 0
    semi = D.HashJoinHandle(ctx, [D.INT64], orders.types, [0], [1], [1, 1, 1], [0, 2, 3], D.JOIN_RIGHT_SEMI)
    semi.push_build_device(_bcols(c)); semi.finish_build()
    semi.push_probe_device(_bcols(o)); semi.finish_probe()
    so = semi.drain(host=False)
    semi.close()
    stages["orders_of_building_customers"] = sum(b.num_rows for b in so)
    l = _filter(ctx, lineitem, B(D.OP_GT, C(3), L(CUT, D.INT32)), [0, 1, 2])
    stages["lineitem_after_cut"] = l[0].num_rows if l else 0
    inner = D.HashJoinHandle(ctx, [D.INT64, D.INT32, D.INT32], [D.INT64, D.INT64, D.INT64], [0], [0], [1, 0, 0, 1, 1], [0, 1, 2, 1, 2])
    inner.push_build_device(_bcols(so)); inner.finish_build()
    inner.push_probe_device(_bcols(l)); inner.finish_probe()
    jo = inner.drain(host=False)
    inner.close()
    jc = _bcols(jo) if jo else None
    stages["joined_rows"] = jo[0].num_rows if jo else 0
    res = []
    if jc is not None:
        n = jo[0].num_rows
        rev = D.evaluate_device(ctx, jc, n, B(D.OP_MULTIPLY, C(3), B(D.OP_MINUS, L(100), C(4))))
        rc = rev.column(0)
        agg = D.AggHandle(ctx, [D.INT64, D.INT32, D.INT32, D.INT64], [0, 1, 2], [(D.AGG_SUM, 3, -1)], D.AGG_SINGLE_PARTITIONED, 8192, max(stages["orders_of_building_customers"], 1024))
        agg.push_device([jc[0], jc[1], jc[2], rc]); agg.finish()
        res = agg.drain(host=False)
        agg.close()
        rev.release()
    stages["groups"] = sum(b.num_rows for b in res)
    for b in c + o + so + l + jo:
        b.release()
    return res, stages


DEC_MONEY = D.decimal128(15, 2)     # l_extendedprice, l_discount in the TPC-H schema (benchmarks/src/tpch/mod.rs:52-122)


def decimal_money(ctx, lineitem):
    """the lineitem table with its money columns as Decimal128(15,2) — the reference's TPC-H schema — instead of int64 cents /
    percent: CAST(int64 AS Decimal128(15,0)) on the device, relabelled at scale 2 (same unscaled integers)"""
    cols, types, keep = list(lineitem.cols), list(lineitem.types), list(lineitem._keep)
    for i in (1, 2):
        b = D.evaluate_device(ctx, [lineitem.cols[i]], lineitem.rows, CAST(C(0), D.decimal128(15, 0)))
        c = b.column(0)
        c.type = DEC_MONEY
        cols[i], types[i] = c, DEC_MONEY
        keep.append(b)
    return Table(lineitem.names, types, cols, lineitem.rows, keep)


def revenue_expr(l_types):
    """sum argument of q3.slt.part:62: l_extendedprice * (1 - l_discount); int64 money: price_cents * (100 - discount_percent)"""
    if D.type_base(l_types[1]) == D.DECIMAL128:
        one = [(D.EXPR_LITERAL, 0, D.decimal128(20, 0), 0, 1, 0.0)]          # Int64 literal coerced to Decimal128(20,0)
        return B(D.OP_MULTIPLY, C(1), B(D.OP_MINUS, one, C(2)))             # -> Decimal128(38,4)
    return B(D.OP_MULTIPLY, C(1), B(D.OP_MINUS, L(100), C(2)))


def run_q3_fused(ctx, customer, orders, lineitem, aggs=None, n_acc_words=None):
    """the same plan as three fused pipelines (dfgpu_pipeline): every table is read once, no intermediate batch touches HBM

        P1  customer : FilterExec(c_mktsegment = 1)                      -> build L1 = key set {c_custkey}   (dense range -> bitmap)
        P2  orders   : FilterExec(o_orderdate < CUT) -> RightSemi vs L1  -> build L2 = {o_orderkey -> (o_orderdate, o_shippriority)}
        P3  lineitem : FilterExec(l_shipdate > CUT)  -> Inner vs L2      -> AggregateExec gby [l_orderkey, o_orderdate, o_shippriority]
                                                                            SUM(l_extendedprice * (100 - l_discount))
    The group keys are the join key plus build-side columns, so the group id is the build row and the sums live in L2's records.
    aggs / n_acc_words: other aggregates of P3 ([(func, nodes)]) and the accumulator words of L2 they need (default: the SUM)."""
    stages = {}
    kmin, kmax, _ = D.column_minmax_device(ctx, customer.cols[0])       # the bounds collect_left_input tracks (exec.rs:2585-2619)
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p1 = D.Pipeline(ctx, customer.types, B(D.OP_EQ, C(1), L(1)))
    p1.sink_build(l1, 0, [])
    p1.push_device(customer.cols); p1.finish()
    stages["customer_building"] = p1.metric("sink_rows")
    p1.close()
    dec = D.type_base(lineitem.types[1]) == D.DECIMAL128                 # a Decimal128 SUM takes two accumulator words
    l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=n_acc_words or (3 if dec else 2), membership_filter=-1)
    p2 = D.Pipeline(ctx, orders.types, B(D.OP_LT, C(2), L(CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)], name="orders")
    p2.sink_build(l2, 0, [2, 3])
    p2.push_device(orders.cols); p2.finish()
    stages["orders_of_building_customers"] = p2.metric("sink_rows")
    p2.close()
    p3 = D.Pipeline(ctx, lineitem.types, B(D.OP_GT, C(3), L(CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
    p3.sink_aggregate([0, 4, 5], aggs or [(D.AGG_SUM, revenue_expr(lineitem.types))], D.AGG_SINGLE_PARTITIONED)
    p3.push_device(lineitem.cols); p3.finish()
    res = p3.drain(host=False)
    stages["joined_rows"] = p3.metric("sink_rows")
    stages["groups"] = p3.metric("num_groups")
    stages["lookup_bytes"] = l2.metric("table_bytes"); stages["filter_bytes"] = l2.metric("filter_bytes")
    p3.close(); l2.close(); l1.close()
    return res, stages


def run_q3_fused_host(ctx, c_host, o_host, l_host, c_types, o_types, l_types):
    """the fused plan fed with HOST columns through the C ABI (`*_push_host`: H2D copies inside), result rows drained to host memory.
    The customer table (the small build side) is uploaded once and read twice: key bounds (what collect_left_input tracks), then the build.
    returns (host result batches, stage rows, D2H bytes)"""
    stages = {}
    c_dev = [D.DeviceColumn.from_host(ctx, h) for h in c_host]
    kmin, kmax, _ = D.column_minmax_device(ctx, c_dev[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p1 = D.Pipeline(ctx, c_types, B(D.OP_EQ, C(1), L(1)))
    p1.sink_build(l1, 0, [])
    p1.push_device(c_dev); p1.finish(); p1.close()
    l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=-1)
    p2 = D.Pipeline(ctx, o_types, B(D.OP_LT, C(2), L(CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)], name="orders")
    p2.sink_build(l2, 0, [2, 3])
    p2.push_host(o_host); p2.finish()
    stages["orders_of_building_customers"] = p2.metric("sink_rows")
    p2.close()
    p3 = D.Pipeline(ctx, l_types, B(D.OP_GT, C(3), L(CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
    p3.sink_aggregate([0, 4, 5], [(D.AGG_SUM, B(D.OP_MULTIPLY, C(1), B(D.OP_MINUS, L(100), C(2))))], D.AGG_SINGLE_PARTITIONED)
    p3.push_host(l_host); p3.finish()
    res = p3.drain(host=True)
    stages["joined_rows"], stages["groups"] = p3.metric("sink_rows"), p3.metric("num_groups")
    d2h = sum(b.num_rows for b in res) * (8 + 4 + 4 + 8)
    p3.close(); l2.close(); l1.close()
    for c in c_dev:
        c.values.free()
    return res, stages, d2h


def result_fingerprint(ctx, res):
    """order-independent fingerprint of the result rows (row count, wrapping sums of every column, computed on the device) —
    the same formula the CPU arm's oracle_bench_q3 returns"""
    n, sums = 0, [0, 0, 0, 0]
    for b in res:
        n += b.num_rows
        for i in range(4):
            sums[i] = (sums[i] + D.column_sum_device(ctx, b.column(i))) & (2**64 - 1)
    return [n] + sums


def q3_expected(c, o, l):
    """independent numpy / pandas evaluation on the downloaded tables"""
    import pandas as pd
    ck = set(c["c_custkey"][c["c_mktsegment"] == 1].tolist())
    od = pd.DataFrame(o); od = od[(od.o_orderdate < CUT) & od.o_custkey.isin(ck)]
    ld = pd.DataFrame(l); ld = ld[ld.l_shipdate > CUT]
    j = ld.merge(od, left_on="l_orderkey", right_on="o_orderkey")
    j["rev"] = j.l_extendedprice * (100 - j.l_discount)
    g = j.groupby(["l_orderkey", "o_orderdate", "o_shippriority"], as_index=False)["rev"].sum()
    return sorted(zip(g.l_orderkey.tolist(), g.o_orderdate.tolist(), g.o_shippriority.tolist(), g.rev.tolist()))


def result_rows(ctx, res):
    out = []
    for b in res:
        cols = [b.column(i) for i in range(4)]
        arrs = [ctx.to_host(cc.values, b.num_rows * D.WIDTH[cc.type]).view(D.NP_OF_TYPE[cc.type]) for cc in cols]
        out += list(zip(*[a.tolist() for a in arrs]))
    return sorted(out)
