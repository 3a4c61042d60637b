"""The fused pipeline kernel's ring-fed phase A (TMA bulk copies of the streamed columns into per-warp shared-memory rings) and its
gathered aggregate arguments: the Q3-shaped plans must give exactly what the oracle's unfused operator chain gives, for row counts
that are not whole ring tiles, for several pushes into one pipeline, for the pack (build) sink, and for input columns whose base is
not 16-byte aligned (those run the kernel without the ring)."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
from harness import assert_cols_equal, batches_to_cols, host_cols, split_points
from test_gpu_filter import B, C, L, to_nodes
import test_gpu_pipeline as TP

pytestmark = pytest.mark.gpu
CUT = 9200
CT, OT, LT = [D.INT64, D.INT64], [D.INT64, D.INT64, D.DATE32, D.INT32], [D.INT64, D.INT64, D.INT64, D.DATE32]
CPRED, OPRED, LPRED = B(D.OP_EQ, C(1), L(1, np.int64)), B(D.OP_LT, C(2), L(CUT, np.int32)), B(D.OP_GT, C(3), L(CUT, np.int32))
REV = B(D.OP_MULTIPLY, C(1), B(D.OP_MINUS, L(100, np.int64), C(2)))


def device_cols(ctx, cols, types, s, e, shift, keep):
    """columns [s, e) in HBM; shift > 0 places every column's values `shift` elements past a 16-byte-aligned allocation"""
    out = []
    for hc, (v, _) in zip(host_cols(cols, s, e, types), cols):
        if not shift:
            out.append(D.DeviceColumn.from_host(ctx, hc))
            continue
        part = v[s:e]
        buf = ctx.to_device(np.concatenate([np.zeros(shift, part.dtype), part]))
        c = D.Column()
        c.type, c.flags, c.length, c.offset, c.null_count = hc.type, 0, e - s, 0, 0
        c.values, c.validity = buf.ptr + shift * part.dtype.itemsize, None
        keep.append(buf)
        out.append(c)
    keep.append(out)
    return out


def run_q3(ctx, nl, batch_rows, shift, no=30_000):
    """the Q3 plan through the fused pipelines, checked against the oracle's unfused chain; returns the ring-fed launches of the
    orders (pack sink) and lineitem (aggregate sink) passes"""
    rng = np.random.default_rng(nl)
    cust, orders, line = TP.q3_like_tables(rng, 3000, no, nl, False)
    keep = []
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(1, 3000))
    p = D.Pipeline(ctx, CT, to_nodes(CPRED, True)); p.sink_build(l1, 0, [])
    p.push_device(device_cols(ctx, cust, CT, 0, len(cust[0][0]), 0, keep)); p.finish(); p.close()
    # the orders table grows by packed passes (pack sink): the table is sized only after each batch
    l2 = D.Lookup(ctx, D.INT64, [D.DATE32, D.INT32], n_acc_words=2, membership_filter=1)
    p = D.Pipeline(ctx, OT, to_nodes(OPRED, True), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2, 0, [2, 3])
    for s, e in split_points(len(orders[0][0]), batch_rows):
        p.push_device(device_cols(ctx, orders, OT, s, e, shift, keep))
    p.finish()
    n2, ring_o = p.metric("sink_rows"), p.metric("ring_launches"); p.close()
    p = D.Pipeline(ctx, LT, to_nodes(LPRED, True), [(D.STAGE_INNER, 0, l2)])
    p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, to_nodes(REV, True)), (D.AGG_COUNT_STAR, None)], D.AGG_SINGLE)
    for s, e in split_points(nl, batch_rows):
        p.push_device(device_cols(ctx, line, LT, s, e, shift, keep))
    p.finish()
    got = batches_to_cols(p.drain(host=False), 5)
    ring_l = p.metric("ring_launches")
    p.close(); l2.close(); l1.close()
    fc, fo, fl = TP.oracle_filter(cust, CPRED), TP.oracle_filter(orders, OPRED), TP.oracle_filter(line, LPRED)
    so = O.hash_join(fc, fo, [0], [1], [1, 1, 1], [0, 2, 3], join_type=O.J_RIGHT_SEMI)
    assert len(so[0][0]) == n2
    j = O.hash_join(so, fl, [0], [0], [1, 0, 0, 1, 1], [0, 1, 2, 1, 2])
    arg = O.eval_expr([j[0], j[3], j[4]], to_nodes(REV, False))
    keys, res = O.group_by([j[0], j[1], j[2]], [(O.A_SUM, arg, None), (O.A_COUNT_STAR, None, None)])
    exp = list(keys) + O.agg_output_columns(O.A_SUM, res[0], np.int64, False) + O.agg_output_columns(O.A_COUNT_STAR, res[1], np.int64, False)
    assert_cols_equal(got, exp, ordered=False, what=f"q3, {nl} lineitem rows in pushes of {batch_rows}, shift {shift}")
    assert len(keys[0][0]) > 1000
    return ring_o, ring_l


def test_ring_q3_ragged_row_count(gpu_ctx):
    """a row count that is not a multiple of the 256-row warp tile or of a ring: the last tile is read without the ring"""
    assert run_q3(gpu_ctx, 256 * 4 * 97 + 131, None, 0) == (1, 1)


def test_ring_q3_several_pushes(gpu_ctx):
    ring_o, ring_l = run_q3(gpu_ctx, 200_001, 37_777, 0)
    assert ring_o >= 1 and ring_l == 6


def test_ring_q3_rings_wrap_several_times(gpu_ctx):
    """one push of 6.5M rows per table: with every SM's blocks resident, each warp takes 8 (lineitem: 3 blocks per SM, 2-tile rings)
    or 12 (orders: 2 blocks per SM, 4-tile rings) tiles, so every stage is refilled and waited on with both mbarrier parities, and
    the ragged last tile comes after the rings have wrapped"""
    assert run_q3(gpu_ctx, 6_500_077, None, 0, no=6_500_011) == (1, 1)


def test_ring_q3_unaligned_column_bases(gpu_ctx):
    """values 8 (int64) / 4 (int32) bytes past a 16-byte boundary: no bulk copies, the kernel without the ring, the same answer"""
    assert run_q3(gpu_ctx, 150_007, 50_000, 1) == (0, 0)


def test_ring_pack_sink_builds_the_same_table(gpu_ctx, monkeypatch):
    """orders -> filter + semi bitmap probe -> packed {key, payload} records -> table: read back through an output probe"""
    rng = np.random.default_rng(5)
    cust, orders, _ = TP.q3_like_tables(rng, 3000, 100_003, 10, False)
    probe_keys = orders[0][0][rng.integers(0, len(orders[0][0]), 50_000)]

    def build_and_probe():
        l1, _ = TP.build_lookup(gpu_ctx, cust, CT, 0, [], pred=CPRED, key_range=(1, 3000), device=True)
        l2, rows = TP.build_lookup(gpu_ctx, orders, OT, 0, [2, 3], pred=OPRED, stages=[(D.STAGE_SEMI, 1, l1)], payload_types=[D.DATE32, D.INT32],
                                   device=True, batch_rows=40_000)
        p = D.Pipeline(gpu_ctx, [D.INT64], None, [(D.STAGE_INNER, 0, l2)])
        p.sink_output([0, 1, 2])
        keep = []
        TP.push_all(p, [(probe_keys, None)], [D.INT64], None, True, gpu_ctx, keep)
        p.finish()
        got = batches_to_cols(p.drain(host=True), 3)
        p.close(); l2.close(); l1.close()
        return rows, got

    rows, got = build_and_probe()
    monkeypatch.setenv("DFGPU_PIPE_VAR", "11")
    rows_ref, ref = build_and_probe()
    assert rows == rows_ref > 1000
    assert_cols_equal(got, ref, ordered=True, what="pack sink via the ring vs without")


@pytest.mark.parametrize("nl", [1, 255, 123_457])
def test_ring_matches_the_kernel_without_it(gpu_ctx, monkeypatch, nl):
    """the default (ring) and DFGPU_PIPE_VAR=11 (the kernel without the ring) give identical groups and sums, also when no tile is full"""
    def q3():
        rng = np.random.default_rng(3)
        cust, orders, line = TP.q3_like_tables(rng, 3000, 30_000, nl, False)
        keep = []
        l1, _ = TP.build_lookup(gpu_ctx, cust, CT, 0, [], pred=CPRED, key_range=(1, 3000), device=True)
        l2, _ = TP.build_lookup(gpu_ctx, orders, OT, 0, [2, 3], pred=OPRED, stages=[(D.STAGE_SEMI, 1, l1)], payload_types=[D.DATE32, D.INT32],
                                n_acc_words=2, membership_filter=1, device=True)
        p = D.Pipeline(gpu_ctx, LT, to_nodes(LPRED, True), [(D.STAGE_INNER, 0, l2)])
        p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, to_nodes(REV, True))], D.AGG_SINGLE)
        p.push_device(device_cols(gpu_ctx, line, LT, 0, nl, 0, keep)); p.finish()
        rows = p.metric("sink_rows")
        got = batches_to_cols(p.drain(host=False), 4)
        p.close(); l2.close(); l1.close()
        order = np.argsort(got[0][0], kind="stable")
        return rows, [v[order] for v, _ in got]

    monkeypatch.delenv("DFGPU_PIPE_VAR", raising=False)
    rows, ring = q3()
    monkeypatch.setenv("DFGPU_PIPE_VAR", "11")
    rows_plain, plain = q3()
    assert rows == rows_plain and (rows > 1000 or nl < 1000)
    assert all(np.array_equal(a, b) for a, b in zip(ring, plain))
