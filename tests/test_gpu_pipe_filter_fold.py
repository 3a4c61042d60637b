"""The partitioned aggregate's folded membership filter.  Pass 1 of the fused pipeline's partitioned aggregate tests the aggregate
stage's Bloom filter folded once (out[i] = in[2i] | in[2i+1], 8 bits per key) and probed with half the blocks; the lookup keeps the
exact filter (16 bits per key) for the direct probe.  A numpy restatement of bloom_pos / bloom_mask rebuilds the exact filter from the
build keys, folds it, and counts the date-qualified lineitem rows that pass it: that count is exactly "partitioned_records".  Every
result must equal the direct probe's and pandas'."""
import os
import sys

import numpy as np
import pytest

from datafusion_b200 import capi as D

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import q3_device_pipeline as Q  # noqa: E402
from q3_device_pipeline import B, C, L  # noqa: E402

HOOKS = ("DFGPU_PIPE_RADIX_PARTS", "DFGPU_PIPE_RADIX_CAP", "DFGPU_PIPE_VAR")


# ---- numpy restatement of bloom.cuh ----
def bloom_pos(keys, blocks):
    """(block, t) of every uint64 key for a filter of `blocks` 64-bit blocks"""
    keys = np.asarray(keys, np.uint64)
    lo, hi = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32), (keys >> np.uint64(32)).astype(np.uint32)
    h1 = (lo ^ (hi * np.uint32(0x85EBCA6B))) * np.uint32(0x9E3779B1)
    h1 ^= h1 >> np.uint32(15)
    block = (h1.astype(np.uint64) * np.uint64(blocks)) >> np.uint64(32)
    t = (h1 * np.uint32(0xC2B2AE35)) >> np.uint32(12)
    return block.astype(np.int64), t


def bloom_mask(t):
    one = np.uint32(1)
    bit = lambda s: one << ((t >> np.uint32(s)) & np.uint32(31))
    m0, m1 = bit(0) | bit(5), bit(10) | bit(15)
    return (m1.astype(np.uint64) << np.uint64(32)) | m0.astype(np.uint64)


def bloom_build(keys, blocks):
    f = np.zeros(blocks, np.uint64)
    block, t = bloom_pos(keys, blocks)
    np.bitwise_or.at(f, block, bloom_mask(t))
    return f


def bloom_passes(f, keys):
    block, t = bloom_pos(keys, len(f))
    m = bloom_mask(t)
    return (f[block] & m) == m


def test_fastrange_halves_exactly_at_the_edges():
    """umulhi(h, 2b) >> 1 == umulhi(h, b): the reason a key of exact block k is in folded block k >> 1"""
    rng = np.random.default_rng(7)
    hs = [0, 1, 2**31 - 1, 2**31, 2**32 - 2, 2**32 - 1] + [int(x) for x in rng.integers(0, 2**32, 200)]
    bs = [2, 4, 1024, 1826, 2**31, 2**32 - 4, 2**32 - 2] + [2 * int(x) for x in rng.integers(1, 2**31, 200)]
    for h in hs:
        for b in bs:
            assert ((h * b) >> 32) >> 1 == (h * (b // 2)) >> 32, (h, b)


# ---- GPU ----
@pytest.fixture(scope="module")
def small(gpu_ctx):
    tables = Q.gen_tables(gpu_ctx, 0.05)
    return tables, [t.host(gpu_ctx) for t in tables]


@pytest.fixture(scope="module")
def natural(gpu_ctx):
    tables = Q.gen_tables(gpu_ctx, 5)
    return tables, [t.host(gpu_ctx) for t in tables]


def q3(ctx, monkeypatch, tables, membership_filter, parts=None, direct=False):
    """Q3 as fused pipelines; returns result rows, sink rows, partitioned launches and records, the orders lookup's exact filter
    (None without one) and capacity.  direct=True sets DFGPU_PIPE_VAR, which the partitioned aggregate refuses."""
    customer, orders, li = tables
    for v in HOOKS:
        monkeypatch.delenv(v, raising=False)
    if parts:
        monkeypatch.setenv("DFGPU_PIPE_RADIX_PARTS", str(parts))
    if direct:
        monkeypatch.setenv("DFGPU_PIPE_VAR", "11")
    kmin, kmax, _ = D.column_minmax_device(ctx, customer.cols[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=membership_filter)
    try:
        p = D.Pipeline(ctx, customer.types, B(D.OP_EQ, C(1), L(1))); p.sink_build(l1, 0, []); p.push_device(customer.cols); p.finish(); p.close()
        p = D.Pipeline(ctx, orders.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2, 0, [2, 3])
        p.push_device(orders.cols); p.finish(); p.close()
        ptr, nbytes = l2.filter_buffer()
        filt = ctx.to_host(ptr, nbytes).view(np.uint64).copy() if ptr else None
        p = D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
        p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, Q.revenue_expr(li.types))], D.AGG_SINGLE_PARTITIONED)
        p.push_device(li.cols); p.finish()
        res = p.drain(host=False)
        out = {"rows": Q.result_rows(ctx, res), "sink": p.metric("sink_rows"), "launches": p.metric("partitioned_launches"),
               "records": p.metric("partitioned_records"), "filter": filt, "capacity": l2.metric("capacity"), "table_bytes": l2.metric("table_bytes")}
        for b in res:
            b.release()
        p.close()
        return out
    finally:
        for v in HOOKS:
            monkeypatch.delenv(v, raising=False)
        l2.close(); l1.close()


def build_keys(host):
    c, o, _ = host
    building = np.isin(o["o_custkey"], c["c_custkey"][c["c_mktsegment"] == 1])
    return o["o_orderkey"][(o["o_orderdate"] < Q.CUT) & building].view(np.uint64)


def probe_keys(host):
    li = host[2]
    return li["l_orderkey"][li["l_shipdate"] > Q.CUT].view(np.uint64)


def check_folded_records(got, host):
    """the exact filter equals the restatement's; the folded one lets through exactly the records pass 1 wrote"""
    f = got["filter"]
    assert len(f) % 2 == 0 and len(f) == (max(1024, got["capacity"] // 8) + 1) & ~1
    assert np.array_equal(f, bloom_build(build_keys(host), len(f)))
    folded = f[0::2] | f[1::2]
    probe = probe_keys(host)
    passed = int(bloom_passes(folded, probe).sum())
    assert got["records"] == passed
    exact = int(bloom_passes(f, probe).sum())
    assert passed > exact, "the folded filter lets more keys through than the exact one"
    return passed, exact


@pytest.mark.gpu
def test_small_table_with_a_filter_folds_it(gpu_ctx, monkeypatch, small):
    tables, host = small
    direct = q3(gpu_ctx, monkeypatch, tables, membership_filter=1)
    assert direct["launches"] == 0 and direct["records"] == 0
    assert direct["rows"] == Q.q3_expected(*host) and len(direct["rows"]) > 1000
    for parts in (2, 8):
        got = q3(gpu_ctx, monkeypatch, tables, membership_filter=1, parts=parts)
        assert got["launches"] == 1
        assert got["rows"] == direct["rows"] and got["sink"] == direct["sink"]
        assert np.array_equal(got["filter"], direct["filter"]), "the lookup keeps its exact filter"
        check_folded_records(got, host)


@pytest.mark.gpu
def test_partitioned_push_without_a_filter_writes_every_qualified_row(gpu_ctx, monkeypatch, small):
    tables, host = small
    got = q3(gpu_ctx, monkeypatch, tables, membership_filter=0, parts=8)
    assert got["filter"] is None and got["launches"] == 1
    assert got["records"] == len(probe_keys(host))
    assert got["rows"] == Q.q3_expected(*host)


@pytest.mark.gpu
def test_natural_size_folds_the_filter_of_a_table_larger_than_l2(gpu_ctx, monkeypatch, natural):
    tables, host = natural
    got = q3(gpu_ctx, monkeypatch, tables, membership_filter=-1)
    assert got["table_bytes"] > 40 << 20 and got["launches"] == 1
    passed, exact = check_folded_records(got, host)
    assert passed < len(host[2]["l_orderkey"]) // 8, "the records fit the buffer of one in eight input rows"
    direct = q3(gpu_ctx, monkeypatch, tables, membership_filter=-1, direct=True)
    assert direct["launches"] == 0 and direct["records"] == 0
    assert got["rows"] == direct["rows"] and got["sink"] == direct["sink"]
    assert got["rows"] == Q.q3_expected(*host) and len(got["rows"]) > 100_000
