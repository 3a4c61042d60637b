"""The fused pipeline's partitioned build: when the packed {key, payload} records of a build sink go into a table larger than L2,
radix_partition_records groups them by slot range and lookup_insert_part_kernel inserts them one L2-sized range at a time.
DFGPU_PIPE_RADIX_PARTS forces the path (and P) on tables far smaller than the L2.  Every result must equal pandas' or numpy's and the
unpartitioned insert's, and the build keeps its errors: duplicate keys, the reserved all-ones key, NULL keys skipped."""
import os
import sys

import numpy as np
import pytest

from datafusion_b200 import capi as D

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import q3_device_pipeline as Q  # noqa: E402
from q3_device_pipeline import B, C, L  # noqa: E402
from harness import batches_to_cols  # noqa: E402

pytestmark = pytest.mark.gpu
SF, SF_LARGE = 0.05, 5
L2_RULE = 40 << 20              # table bytes above which the build sink partitions its records (pipeline.cu kL2TableBytes)


@pytest.fixture
def parts_hook(monkeypatch):
    """sets DFGPU_PIPE_RADIX_PARTS for the test (None: unset); the hook is removed again when the test ends"""
    def set_parts(parts):
        if parts:
            monkeypatch.setenv("DFGPU_PIPE_RADIX_PARTS", str(parts))
        else:
            monkeypatch.delenv("DFGPU_PIPE_RADIX_PARTS", raising=False)
    set_parts(None)
    yield set_parts
    set_parts(None)


def q3(ctx, tables):
    """TPC-H Q3 as fused pipelines; returns (result rows, partitioned inserts of the orders build, orders table bytes)"""
    customer, orders, li = tables
    kmin, kmax, _ = D.column_minmax_device(ctx, customer.cols[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p = D.Pipeline(ctx, customer.types, B(D.OP_EQ, C(1), L(1))); p.sink_build(l1, 0, []); p.push_device(customer.cols); p.finish(); p.close()
    l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=1)
    p = D.Pipeline(ctx, orders.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2, 0, [2, 3])
    p.push_device(orders.cols); p.finish()
    inserts = p.metric("partitioned_inserts")
    p.close()
    p = D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
    p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, Q.revenue_expr(li.types))], D.AGG_SINGLE_PARTITIONED)
    p.push_device(li.cols); p.finish()
    res = p.drain(host=False)
    out = Q.result_rows(ctx, res), inserts, l2.metric("table_bytes")
    for b in res:
        b.release()
    p.close(); l2.close(); l1.close()
    return out


@pytest.fixture(scope="module")
def small(gpu_ctx):
    """SF0.05 tables and their Q3 result from pandas"""
    tables = Q.gen_tables(gpu_ctx, SF)
    exp = Q.q3_expected(*(t.host(gpu_ctx) for t in tables))
    assert len(exp) > 1000
    return tables, exp


def test_unforced_small_build_keeps_the_direct_insert(gpu_ctx, parts_hook, small):
    tables, exp = small
    rows, inserts, tbytes = q3(gpu_ctx, tables)
    assert tbytes < L2_RULE and inserts == 0
    assert rows == exp


@pytest.mark.parametrize("parts", [2, 8, 64])
def test_partitioned_build_q3_equals_pandas(gpu_ctx, parts_hook, small, parts):
    tables, exp = small
    parts_hook(parts)
    rows, inserts, _ = q3(gpu_ctx, tables)
    assert inserts == 1
    assert rows == exp


def test_partitioned_build_at_its_natural_size(gpu_ctx, parts_hook):
    """no hook: the SF5 orders table exceeds the 40 MB rule, so its build takes the path by size alone"""
    tables = Q.gen_tables(gpu_ctx, SF_LARGE, seed=3)
    rows, inserts, tbytes = q3(gpu_ctx, tables)
    assert tbytes > L2_RULE, f"SF{SF_LARGE}: the orders table ({tbytes} B) no longer exceeds the partitioning threshold"
    assert inserts == 1
    exp = Q.q3_expected(*(t.host(gpu_ctx) for t in tables))
    assert rows == exp and len(exp) > 100_000


# ---------------------------------------------------------------------------------------------------------------------------------
# build errors and NULL keys on the forced path
# ---------------------------------------------------------------------------------------------------------------------------------
def build(ctx, pushes, membership_filter=1):
    """a lookup {int64 key -> int32 payload} built by one host push per (keys, valid, payload); returns (lookup, partitioned inserts)"""
    look = D.Lookup(ctx, D.INT64, [D.INT32], membership_filter=membership_filter)
    p = D.Pipeline(ctx, [D.INT64, D.INT32])
    p.sink_build(look, 0, [1])
    try:
        for k, valid, v in pushes:
            p.push_host([D.HostColumn(k, valid), D.HostColumn(v)])
        p.finish()
        return look, p.metric("partitioned_inserts")
    except Exception:
        look.close()
        raise
    finally:
        p.close()


def probe(ctx, look, keys):
    """inner probe of `keys`: sorted (key, payload) rows"""
    p = D.Pipeline(ctx, [D.INT64], None, [(D.STAGE_INNER, 0, look)])
    p.sink_output([0, 1], ordered=False)
    p.push_host([D.HostColumn(keys)])
    p.finish()
    (k, kv), (v, vv) = batches_to_cols(p.drain(host=True), 2)
    p.close()
    assert kv is None and vv is None
    o = np.lexsort((v, k))
    return k[o], v[o]


def reference(bkeys, bvals, pkeys):
    """inner join of pkeys on unique build keys: sorted (key, payload) rows"""
    order = np.argsort(bkeys)
    sk, sv = bkeys[order], bvals[order]
    pos = np.minimum(np.searchsorted(sk, pkeys), len(sk) - 1)
    hit = sk[pos] == pkeys
    k, v = pkeys[hit], sv[pos[hit]]
    o = np.lexsort((v, k))
    return k[o], v[o]


def test_duplicate_build_keys_are_still_rejected(gpu_ctx, parts_hook):
    parts_hook(8)
    rng = np.random.default_rng(1)
    k = rng.permutation(50_000).astype(np.int64) * 7 - 1000
    k[40_000] = k[123]
    with pytest.raises(D.DfgpuError) as ei:
        build(gpu_ctx, [(k, None, np.arange(len(k), dtype=np.int32))])
    assert ei.value.code == -3 and "duplicate" in str(ei.value)


def test_the_reserved_all_ones_key_is_still_rejected(gpu_ctx, parts_hook):
    parts_hook(8)
    k = np.arange(50_000, dtype=np.int64)
    k[777] = -1                     # 0xFFFF'FFFF'FFFF'FFFF, the empty-slot marker
    with pytest.raises(D.DfgpuError) as ei:
        build(gpu_ctx, [(k, None, np.arange(len(k), dtype=np.int32))])
    assert ei.value.code == -1 and "reserved" in str(ei.value)


def test_null_build_keys_are_skipped(gpu_ctx, parts_hook):
    """NULL keys never become records: the ones that repeat a valid key or hold the all-ones value raise nothing, and no probe finds them"""
    parts_hook(8)
    rng = np.random.default_rng(2)
    n = 60_000
    k = rng.permutation(4 * n)[:n].astype(np.int64) * 11 + 5
    v = rng.integers(-2**31, 2**31, n).astype(np.int32)
    valid = rng.random(n) > 0.1
    nulls = np.flatnonzero(~valid)
    k[nulls[: len(nulls) // 2]] = k[np.flatnonzero(valid)[: len(nulls) // 2]]   # duplicates of valid keys, but NULL
    k[nulls[-1]] = -1
    look, inserts = build(gpu_ctx, [(k, valid, v)])
    try:
        assert inserts == 1 and look.metric("rows") == int(valid.sum())
        pk = np.concatenate([k[valid], k[~valid][len(nulls) // 2:-1], rng.integers(0, 44 * n, n).astype(np.int64)])
        got = probe(gpu_ctx, look, pk)
    finally:
        look.close()
    exp = reference(k[valid], v[valid], pk)
    assert len(exp[0]) >= valid.sum()
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])


def test_second_push_grows_the_table_then_inserts_partitioned(gpu_ctx, parts_hook):
    """the second push does not fit the table sized for the first: it grows by rehash (old records and their Bloom bits move over),
    then its own records are partitioned and inserted.  A key the Bloom filter lost would be a missing row."""
    parts_hook(8)
    rng = np.random.default_rng(3)
    n1, n2 = 150_000, 400_000
    ids = rng.permutation(3 * (n1 + n2))
    keys = ids[: n1 + n2].astype(np.int64) * 1_000_003 - 77
    vals = rng.integers(-2**31, 2**31, n1 + n2).astype(np.int32)
    look, inserts = build(gpu_ctx, [(keys[:n1], None, vals[:n1]), (keys[n1:], None, vals[n1:])])
    try:
        assert inserts == 2 and look.metric("rehashes") >= 1 and look.metric("rows") == n1 + n2
        assert look.metric("filter_bytes") > 0
        misses = ids[n1 + n2:].astype(np.int64) * 1_000_003 - 77
        pk = np.concatenate([keys, misses])[rng.permutation(len(ids))]
        got = probe(gpu_ctx, look, pk)
    finally:
        look.close()
    exp = reference(keys, vals, pk)
    assert len(exp[0]) == n1 + n2
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
