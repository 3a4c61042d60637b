"""The fused pipeline's partitioned aggregate: when the aggregate stage's table exceeds L2, the lineitem pass of TPC-H Q3 writes
{key, SUM argument} records instead of probing, radix_partition groups them by slot range, and pipe_probe_agg_kernel probes and
accumulates one L2-sized range of the table at a time.  DFGPU_PIPE_RADIX_PARTS forces the path (and P) on tables far smaller than
the L2, DFGPU_PIPE_RADIX_CAP a record buffer so small that most rows take the in-kernel fallback.  Every result must equal pandas'
and the direct probe's, with the same sink rows."""
import os
import sys

import numpy as np
import pytest

from datafusion_b200 import capi as D

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import q3_device_pipeline as Q  # noqa: E402
from q3_device_pipeline import B, C, L  # noqa: E402

pytestmark = pytest.mark.gpu
SF = 0.05


def build_orders(ctx, customer, orders, n_acc_words=2):
    kmin, kmax, _ = D.column_minmax_device(ctx, customer.cols[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p = D.Pipeline(ctx, customer.types, B(D.OP_EQ, C(1), L(1))); p.sink_build(l1, 0, []); p.push_device(customer.cols); p.finish(); p.close()
    l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=n_acc_words, membership_filter=1)
    p = D.Pipeline(ctx, orders.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2, 0, [2, 3])
    p.push_device(orders.cols); p.finish(); p.close()
    return l1, l2


def lineitem_pass(ctx, lineitem, l2, aggs, pushes=1):
    """Q3's lineitem pipeline into l2's records; returns (result batches, sink rows, partitioned launches)"""
    p = D.Pipeline(ctx, lineitem.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
    p.sink_aggregate([0, 4, 5], aggs, D.AGG_SINGLE_PARTITIONED)
    for _ in range(pushes):
        p.push_device(lineitem.cols)
    p.finish()
    res = p.drain(host=False)
    out = res, p.metric("sink_rows"), p.metric("partitioned_launches")
    p.close()
    return out


def q3(ctx, monkeypatch, tables, parts=None, cap=None, pushes=1, aggs=None, n_acc_words=2, lineitem=None):
    customer, orders, li = tables
    monkeypatch.delenv("DFGPU_PIPE_RADIX_PARTS", raising=False); monkeypatch.delenv("DFGPU_PIPE_RADIX_CAP", raising=False)
    if parts:
        monkeypatch.setenv("DFGPU_PIPE_RADIX_PARTS", str(parts))
    if cap:
        monkeypatch.setenv("DFGPU_PIPE_RADIX_CAP", str(cap))
    l1, l2 = build_orders(ctx, customer, orders, n_acc_words)
    try:
        return lineitem_pass(ctx, lineitem or li, l2, aggs or [(D.AGG_SUM, Q.revenue_expr(li.types))], pushes)
    finally:
        monkeypatch.delenv("DFGPU_PIPE_RADIX_PARTS", raising=False); monkeypatch.delenv("DFGPU_PIPE_RADIX_CAP", raising=False)
        l2.close(); l1.close()


def release(res):
    for b in res:
        b.release()


@pytest.fixture(scope="module")
def tables(gpu_ctx):
    return Q.gen_tables(gpu_ctx, SF)


@pytest.fixture(scope="module")
def direct(gpu_ctx, tables):
    """the direct probe's rows and sink rows (no hook: the SF0.05 table is far below the L2 threshold)"""
    customer, orders, li = tables
    l1, l2 = build_orders(gpu_ctx, customer, orders)
    res, rows, parts = lineitem_pass(gpu_ctx, li, l2, [(D.AGG_SUM, Q.revenue_expr(li.types))])
    assert parts == 0
    got = Q.result_rows(gpu_ctx, res)
    release(res); l2.close(); l1.close()
    exp = Q.q3_expected(customer.host(gpu_ctx), orders.host(gpu_ctx), li.host(gpu_ctx))
    assert got == exp and len(exp) > 1000
    return got, rows


@pytest.mark.parametrize("parts", [2, 8, 64])
def test_partitioned_q3_equals_pandas_and_the_direct_probe(gpu_ctx, monkeypatch, tables, direct, parts):
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=parts)
    assert launches == 1
    assert Q.result_rows(gpu_ctx, res) == direct[0] and rows == direct[1]
    release(res)


@pytest.mark.parametrize("cap", [1, 1000])
def test_rows_past_the_record_buffer_take_the_in_kernel_probe(gpu_ctx, monkeypatch, tables, direct, cap):
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=8, cap=cap)
    assert launches == 1 and direct[1] > 10 * cap
    assert Q.result_rows(gpu_ctx, res) == direct[0] and rows == direct[1]
    release(res)


def test_several_pushes_accumulate_into_the_same_records(gpu_ctx, monkeypatch, tables, direct):
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=8, pushes=3)
    assert launches == 3 and rows == 3 * direct[1]
    assert Q.result_rows(gpu_ctx, res) == [(k, d, p, 3 * s) for k, d, p, s in direct[0]]
    release(res)


def test_keys_without_a_partner_add_nothing(gpu_ctx, monkeypatch, tables):
    """every l_orderkey moved off the order keys (8 of every 32): only the Bloom filter's false positives become records, and they
    find no record in the table"""
    customer, orders, li = tables
    moved = D.evaluate_device(gpu_ctx, [li.cols[0]], li.rows, B(D.OP_PLUS, C(0), L(8)))
    kc = moved.column(0); kc.validity = None; kc.null_count = 0
    miss = Q.Table(li.names, li.types, [kc] + li.cols[1:], li.rows, [moved])
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=8, lineitem=miss)
    assert launches == 1 and rows == 0 and sum(b.num_rows for b in res) == 0
    release(res)
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, lineitem=miss)
    assert launches == 0 and rows == 0 and sum(b.num_rows for b in res) == 0
    release(res)


def test_shapes_outside_the_partitioned_path_keep_the_direct_probe(gpu_ctx, monkeypatch, tables, direct):
    customer, orders, li = tables
    price = C(1)
    # MIN, a program that reads a build payload field (o_shippriority, virtual column 5), two aggregates
    for aggs in ([(D.AGG_MIN, price)], [(D.AGG_SUM, C(5))], [(D.AGG_SUM, Q.revenue_expr(li.types)), (D.AGG_COUNT_STAR, None)]):
        res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=8, aggs=aggs)
        assert launches == 0 and rows == direct[1], aggs
        release(res)
    # Decimal128 money
    dl = Q.decimal_money(gpu_ctx, li)
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=8, aggs=[(D.AGG_SUM, Q.revenue_expr(dl.types))], n_acc_words=3, lineitem=dl)
    assert launches == 0 and rows == direct[1]
    release(res)
    # a nullable argument (its non-null counter is a third accumulator word)
    valid = gpu_ctx.to_device(np.full((li.rows + 7) // 8, 0xEF, np.uint8))
    pc = D.Column()
    pc.type, pc.flags, pc.length, pc.offset, pc.values, pc.validity = D.INT64, 0, li.rows, 0, li.cols[1].values, valid.ptr
    pc.null_count = li.rows - int(np.unpackbits(np.full((li.rows + 7) // 8, 0xEF, np.uint8), bitorder="little")[:li.rows].sum())
    nl = Q.Table(li.names, li.types, [li.cols[0], pc] + li.cols[2:], li.rows, [valid])
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables, parts=8, n_acc_words=3, lineitem=nl)
    assert launches == 0 and rows == direct[1]
    release(res)
    # the same Q3 shape with a table under the L2 threshold and no hook
    res, rows, launches = q3(gpu_ctx, monkeypatch, tables)
    assert launches == 0 and Q.result_rows(gpu_ctx, res) == direct[0]
    release(res)
