"""Kernel paths that only large inputs select, run at the sizes that select them, against exact references:

  * the pipelined host probe of the hash join (push_probe_host_pipelined + join_probe_inline_staged_kernel): host pushes of at least
    2 x 8 Mi rows, no NULLs, inline table;
  * the coarse first level of a filter-only lookup (coarse_pos / filter_set): an exact Bloom level larger than 20 MiB;
  * the partitioned aggregate of the fused pipeline (radix_partition + pipe_probe_agg_kernel): an aggregate table larger than 40 MiB;
  * the radix-partitioned join probe (radix_probe.cuh): an inline table larger than 40 MiB and at least 4 Mi probe rows.

No environment hook forces a path (except DFGPU_PIPE_VAR, which turns the partitioned aggregate off for its comparison run).  Every
test asserts the metric that proves its path ran, or did not, so that a moved threshold fails here instead of quietly testing the
small-input path."""
import os
import sys

import numpy as np
import pytest

from datafusion_b200 import capi as D

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import q3_device_pipeline as Q  # noqa: E402
from q3_device_pipeline import B, C, L  # noqa: E402

pytestmark = pytest.mark.gpu

CHUNK = 8 << 20                 # rows per chunk of the pipelined host probe (push_probe_host_pipelined's kChunk)
L2_RULE = 40 << 20              # table bytes above which the join and the pipeline partition their probes
DEC = D.decimal128(38, 2)


# ---------------------------------------------------------------------------------------------------------------------------------
# references and helpers
# ---------------------------------------------------------------------------------------------------------------------------------
def composite(keys):
    """one int64 per row for a key of one or two columns (two Int32 columns pack into 64 bits)"""
    if len(keys) == 1:
        return keys[0].astype(np.int64)
    a, b = keys
    return (a.astype(np.int64) << 32) | (b.astype(np.int64) & 0xFFFFFFFF)


def unique_join_rows(bkey, pkey, pvalid=None):
    """inner join on unique build keys: (probe rows with a partner, in probe order; their build rows)"""
    order = np.argsort(bkey, kind="stable")
    sk = bkey[order]
    assert len(np.unique(sk)) == len(sk), "the reference needs unique build keys"
    pos = np.searchsorted(sk, pkey)
    pos[pos == len(sk)] = 0
    hit = sk[pos] == pkey
    if pvalid is not None:
        hit &= pvalid
    prow = np.flatnonzero(hit)
    return prow, order[pos[prow]]


def expected_columns(build, probe, out, prow, brow):
    return [build[ix][0][brow] if side == 0 else probe[ix][0][prow] for side, ix in out]


def batches_arrays(batches, n_out):
    """output batches -> one numpy array per column; every value must be non-NULL"""
    cols = []
    for c in range(n_out):
        parts = []
        for b in batches:
            v, valid = b.column_numpy(c)
            assert valid is None or valid.all()
            parts.append(v)
        cols.append(np.concatenate(parts))
    for b in batches:
        b.release()
    return cols


def assert_arrays_equal(got, exp, what):
    assert len(got) == len(exp), what
    for c, (g, e) in enumerate(zip(got, exp)):
        assert g.dtype == e.dtype and g.shape == e.shape, f"{what}: column {c} {g.dtype}{g.shape} != {e.dtype}{e.shape}"
        bad = np.flatnonzero(np.any((g != e).reshape(len(g), -1), axis=1)) if len(g) else []
        assert len(bad) == 0, f"{what}: column {c} differs in {len(bad)} rows, first at {bad[0]}: {g[bad[0]]} != {e[bad[0]]}"


def assert_same_multiset(got, exp, what):
    """row multisets equal: both sides sorted by all their columns"""
    assert len(got[0]) == len(exp[0]), f"{what}: {len(got[0])} rows != {len(exp[0])}"
    og, oe = np.lexsort(got[::-1]), np.lexsort(exp[::-1])
    assert_arrays_equal([g[og] for g in got], [e[oe] for e in exp], what)


def host_col(vals, valid, t):
    return D.HostColumn(vals, valid, t)


def dec_words(rng, n):
    """Decimal128 words of signed 64-bit values: [n, 2] uint64 (low, sign-extended high)"""
    v = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    return np.stack([v.view(np.uint64), (v >> 63).view(np.uint64)], axis=1)


def new_join(ctx, build, btypes, ptypes, on_b, on_p, out, phj, ordered_output=True):
    j = D.HashJoinHandle(ctx, btypes, ptypes, on_b, on_p, [s for s, _ in out], [i for _, i in out], phj_threshold=phj[0],
                         phj_density=phj[1], ordered_output=ordered_output)
    j.push_build_host([host_col(v, val, t) for (v, val), t in zip(build, btypes)])
    j.finish_build()
    return j


def probe_metrics(j):
    return {m: j.metric(m) for m in ("input_rows", "probe_hits", "output_rows", "pipelined_host_probes", "radix_partitioned_probes",
                                     "array_map_created_count")}


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. pipelined host probe
# ---------------------------------------------------------------------------------------------------------------------------------
N_BIG = 4 * CHUNK + 4097        # five chunks: both staging buffers reused twice, a ragged last tile
PAD = 3                         # rows in front of the probe data: one column is passed with offset PAD, the Arrow batch is sliced there
NB = 1_500_000
BIG_PTYPES = [D.INT64, D.INT8, D.INT16, D.INT32, D.INT64, DEC]
BIG_BTYPES = [D.INT64, D.INT32, D.INT16, D.INT8]
# the build key (read from the probe key), three packed build payload fields (W = 2) and six probe columns: five of <= 8 bytes, more
# than the kStageCols = 4 the kernel stages through shared memory, and a Decimal128 (width 16)
BIG_OUT = [(0, 0), (1, 1), (0, 1), (1, 2), (1, 3), (0, 2), (1, 4), (1, 5), (0, 3), (1, 0)]


def sparse_keys(ids):
    return ids.astype(np.int64) * 1_000_003 - 5


@pytest.fixture(scope="module")
def big():
    """unique build keys; probe keys hit ~60 % of the time, except chunk 1 (rows [8 Mi, 16 Mi)), which has no hit at all"""
    rng = np.random.default_rng(2024)
    ids = rng.permutation(2 * NB)
    bk, miss = sparse_keys(ids[:NB]), sparse_keys(ids[NB:])
    build = [(bk, None), (rng.integers(-2**31, 2**31, NB).astype(np.int32), None), (rng.integers(-2**15, 2**15, NB).astype(np.int16), None),
             (rng.integers(-128, 128, NB).astype(np.int8), None)]
    n = N_BIG + PAD
    pk = np.where(rng.random(n) < 0.6, bk[rng.integers(0, NB, n)], miss[rng.integers(0, NB, n)])
    pk[PAD + CHUNK:PAD + 2 * CHUNK] = miss[rng.integers(0, NB, CHUNK)]
    base = [pk, rng.integers(-128, 128, n).astype(np.int8), rng.integers(-2**15, 2**15, n).astype(np.int16),
            rng.integers(-2**31, 2**31, n).astype(np.int32), rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64), dec_words(rng, n)]
    probe = [(c[PAD:], None) for c in base]
    prow, brow = unique_join_rows(bk, probe[0][0])
    assert 0.45 * N_BIG < len(prow) < 0.5 * N_BIG and not ((prow >= CHUNK) & (prow < 2 * CHUNK)).any()
    return dict(build=build, base=base, probe=probe, exp=expected_columns(build, probe, BIG_OUT, prow, brow), hits=len(prow))


def offset_column(vals, t):
    """the column's rows start PAD values into `vals` (host or device address in `ptr`)"""
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.validity = t, 0, len(vals) - PAD, PAD, 0, None
    return c


def check_host_batches(j, n_out, what):
    """the pipelined probe yields one host batch: next(host=False) refuses it (DFGPU_ERR_STATE) and leaves it queued"""
    with pytest.raises(D.DfgpuError) as ei:
        j.next(host=False)
    assert ei.value.code == -5, what
    got = batches_arrays(j.drain(host=True), n_out)
    j.finish_probe()
    assert j.drain(host=True) == []
    return got


def assert_probe_metrics(j, n, hits, pipelined, what):
    m = probe_metrics(j)
    assert (m["input_rows"], m["probe_hits"], m["output_rows"], m["pipelined_host_probes"]) == (n, hits, hits, pipelined), f"{what}: {m}"


def test_pipelined_host_probe_wide_output_with_offset_column(gpu_ctx, big):
    """five chunks, ten output columns (packed payload, six probe-side columns, Decimal128), one column with a nonzero offset"""
    j = new_join(gpu_ctx, big["build"], BIG_BTYPES, BIG_PTYPES, [0], [0], BIG_OUT, (0, float("inf")))
    cols = [host_col(v, None, t) for (v, _), t in zip(big["probe"], BIG_PTYPES)]
    oc = offset_column(big["base"][3], D.INT32)
    oc.values = big["base"][3].ctypes.data
    cols[3] = oc
    j.push_probe_host(cols)
    got = check_host_batches(j, len(BIG_OUT), "host push")
    assert_probe_metrics(j, N_BIG, big["hits"], 1, "host push")
    assert j.metric("array_map_created_count") == 0 and j.metric("output_batches") == 1
    j.close()
    assert_arrays_equal(got, big["exp"], "pipelined host probe")


def test_pipelined_host_probe_equals_the_device_probe(gpu_ctx, big):
    j = new_join(gpu_ctx, big["build"], BIG_BTYPES, BIG_PTYPES, [0], [0], BIG_OUT, (0, float("inf")))
    bufs = [gpu_ctx.to_device(c) for c in big["base"]]
    cols = []
    for b, t in zip(bufs, BIG_PTYPES):
        c = offset_column(big["base"][0], t)     # every column a view PAD rows into its device buffer
        c.values = b.ptr
        cols.append(c)
    j.push_probe_device(cols)
    j.finish_probe()
    got = batches_arrays(j.drain(host=True), len(BIG_OUT))
    assert_probe_metrics(j, N_BIG, big["hits"], 0, "device push")
    j.close()
    for b in bufs:
        b.free()
    assert_arrays_equal(got, big["exp"], "device probe")


def test_pipelined_host_probe_from_a_sliced_arrow_batch(gpu_ctx, big):
    """the way exec.py reaches the path: push_probe_arrow of a RecordBatch slice (every child carries offset PAD)"""
    pa = pytest.importorskip("pyarrow")
    n = N_BIG + PAD
    arrays = [pa.array(c) for c in big["base"][:5]] + [pa.Array.from_buffers(pa.decimal128(38, 2), n, [None, pa.py_buffer(big["base"][5])])]
    rb = pa.record_batch(arrays, names=[f"p{i}" for i in range(6)]).slice(PAD, N_BIG)
    j = new_join(gpu_ctx, big["build"], BIG_BTYPES, BIG_PTYPES, [0], [0], BIG_OUT, (0, float("inf")))
    j.push_probe_arrow(rb)
    got = check_host_batches(j, len(BIG_OUT), "arrow push")
    assert_probe_metrics(j, N_BIG, big["hits"], 1, "arrow push")
    j.close()
    assert_arrays_equal(got, big["exp"], "pipelined host probe (Arrow)")


def variant_case(name):
    """(build, build types, probe, probe types, on_build, on_probe, out, phj, probe rows, pipelined?, array map?)"""
    rng = np.random.default_rng(sum(map(ord, name)))
    nb = 1_000_000
    hashed = (0, float("inf"))
    n = {"no_payload_at_threshold": 2 * CHUNK, "no_payload_one_row_short": 2 * CHUNK - 1, "dense_array_map": 2 * CHUNK + 1,
         "int32_key": 2 * CHUNK + 3, "two_column_key": 2 * CHUNK + 5, "validity_without_nulls": 2 * CHUNK,
         "one_null_key": 2 * CHUNK}[name]
    ids = rng.permutation(2 * nb)
    pick = rng.random(n) < 0.6
    pid = np.where(pick, ids[:nb][rng.integers(0, nb, n)], ids[nb:][rng.integers(0, nb, n)])
    pv = rng.integers(-2**31, 2**31, n).astype(np.int32)
    if name == "dense_array_map":
        # build keys: a dense range (the reference's ArrayMap); probe keys also below and above it
        bk = rng.permutation(nb).astype(np.int64) + 10_000
        pk = rng.integers(10_000 - nb // 2, 10_000 + nb + nb // 2, n).astype(np.int64)
        build = [(bk, None), (rng.integers(-2**31, 2**31, nb).astype(np.int32), None)]
        return build, [D.INT64, D.INT32], [(pk, None), (pv, None)], [D.INT64, D.INT32], [0], [0], [(1, 0), (0, 1), (1, 1)], (1024, 0.15), n, True, True
    if name == "int32_key":
        build = [((ids[:nb] * 613 - 7).astype(np.int32), None), (rng.integers(-2**15, 2**15, nb).astype(np.int16), None)]
        probe = [((pid * 613 - 7).astype(np.int32), None), (pv, None)]
        return build, [D.INT32, D.INT16], probe, [D.INT32, D.INT32], [0], [0], [(0, 0), (0, 1), (1, 1)], hashed, n, True, False
    if name == "two_column_key":
        split = lambda x: [((x // 1000) * 3 + 1).astype(np.int32), ((x % 1000) * 7 - 3).astype(np.int32)]
        bkey, pkey = split(ids[:nb]), split(pid)
        build = [(bkey[0], None), (bkey[1], None), (rng.integers(-2**63, 2**63 - 1, nb, dtype=np.int64), None)]
        probe = [(pv, None), (pkey[1], None), (pkey[0], None)]
        return (build, [D.INT32, D.INT32, D.INT64], probe, [D.INT32, D.INT32, D.INT32], [0, 1], [2, 1],
                [(0, 2), (1, 0), (0, 0), (1, 1)], hashed, n, True, False)
    bk, pk = sparse_keys(ids[:nb]), sparse_keys(pid)
    build = [(bk, None)]
    out = [(1, 0), (0, 0), (1, 1)]        # no build payload: one word per slot (W = 1)
    kvalid = None
    if name == "validity_without_nulls":
        kvalid = np.ones(n, bool)
    if name == "one_null_key":
        kvalid = np.ones(n, bool)
        kvalid[np.flatnonzero(pick)[12345]] = False
    pipelined = name in ("no_payload_at_threshold", "validity_without_nulls")
    return build, [D.INT64], [(pk, kvalid), (pv, kvalid)], [D.INT64, D.INT32], [0], [0], out, hashed, n, pipelined, False


@pytest.mark.parametrize("name", ["no_payload_at_threshold", "no_payload_one_row_short", "dense_array_map", "int32_key", "two_column_key",
                                  "validity_without_nulls", "one_null_key"])
def test_pipelined_host_probe_shapes_and_boundaries(gpu_ctx, name):
    build, btypes, probe, ptypes, on_b, on_p, out, phj, n, pipelined, amap = variant_case(name)
    kvalid = probe[on_p[0]][1]
    prow, brow = unique_join_rows(composite([build[c][0] for c in on_b]), composite([probe[c][0] for c in on_p]), kvalid)
    exp = expected_columns(build, probe, out, prow, brow)
    assert 0.5 * n < len(prow) < 0.7 * n or (name == "dense_array_map" and 0.4 * n < len(prow))
    runs = []
    for device in (False, True):
        j = new_join(gpu_ctx, build, btypes, ptypes, on_b, on_p, out, phj)
        hc = [host_col(v, val, t) for (v, val), t in zip(probe, ptypes)]
        if device:
            dc = [D.DeviceColumn.from_host(gpu_ctx, h) for h in hc]
            j.push_probe_device(dc)
        else:
            j.push_probe_host(hc)
        j.finish_probe()
        runs.append(batches_arrays(j.drain(host=True), len(out)))
        assert_probe_metrics(j, n, len(prow), 1 if pipelined and not device else 0, f"{name} device={device}")
        assert j.metric("array_map_created_count") == (1 if amap else 0)
        j.close()
        assert_arrays_equal(runs[-1], exp, f"{name} device={device}")


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. coarse first level of a filter-only lookup
# ---------------------------------------------------------------------------------------------------------------------------------
NF_BUILD, NF_PROBE = 12_000_000, 30_000_000


@pytest.fixture(scope="module")
def filter_data():
    rng = np.random.default_rng(77)
    ids = rng.permutation(3 * NF_BUILD)
    bk = sparse_keys(ids[:NF_BUILD])
    pid = np.where(rng.random(NF_PROBE) < 0.4, ids[:NF_BUILD][rng.integers(0, NF_BUILD, NF_PROBE)],
                   ids[NF_BUILD:][rng.integers(0, 2 * NF_BUILD, NF_PROBE)])
    pk = sparse_keys(pid)
    return bk, pk, np.isin(pid, ids[:NF_BUILD])


def filter_pass(ctx, filt, pk):
    """MAYBE stage + unordered output of (key, row id): returns a bool mask of the probe rows that passed"""
    p = D.Pipeline(ctx, [D.INT64, D.INT64], None, [(D.STAGE_MAYBE, 0, filt)])
    p.sink_output([0, 1], ordered=False)
    p.push_host([D.HostColumn(pk), D.HostColumn(np.arange(len(pk), dtype=np.int64))])
    p.finish()
    bs = p.drain(host=True)
    sink_rows = p.metric("sink_rows")
    p.close()
    passed = np.zeros(len(pk), bool)
    if not bs:
        return passed, sink_rows
    key, rid = batches_arrays(bs, 2)
    assert len(rid) == sink_rows and len(np.unique(rid)) == len(rid)     # every survivor once
    assert np.array_equal(pk[rid], key)                                   # carried with its own key
    passed[rid] = True
    return passed, sink_rows


def built_filter(ctx, expected_rows, bk):
    filt = D.Lookup(ctx, D.INT64, [], expected_rows=expected_rows, filter_only=True)
    b = D.Pipeline(ctx, [D.INT64])
    b.sink_build(filt, 0, [])
    b.push_host([D.HostColumn(bk)])
    b.finish()
    assert b.metric("sink_rows") == len(bk)
    b.close()
    return filt


def test_coarse_filter_level_has_no_false_negatives(gpu_ctx, filter_data, capsys):
    bk, pk, partner = filter_data
    rates = {}
    # 12 M expected rows: 3 M exact blocks of 8 B (24 MB > 20 MiB) plus 1.5 M coarse words of 4 B; 10 M: 20 MB, no coarse level
    for expected, nbytes in ((12_000_000, 30_000_000), (10_000_000, 20_000_000)):
        filt = built_filter(gpu_ctx, expected, bk)
        try:   # released before the session's context even when an assertion fails
            assert filt.filter_buffer()[1] == nbytes and filt.metric("filter_bytes") >= nbytes
            passed, _ = filter_pass(gpu_ctx, filt, pk)
            assert passed[partner].all(), f"{expected}: {(~passed[partner]).sum()} false negatives"
            rates[expected] = (passed & ~partner).sum() / (~partner).sum()
            if expected == 12_000_000:
                # clear() zeroes both levels: nothing passes
                filt.clear()
                assert filt.filter_buffer()[1] == nbytes
                passed, rows = filter_pass(gpu_ctx, filt, pk)
                assert rows == 0 and not passed.any()
        finally:
            filt.close()
    with capsys.disabled():
        print(f"\nfilter false-positive rate: coarse + exact {rates[12_000_000]:.5f}, exact only (10 M geometry) {rates[10_000_000]:.5f}")
    # 16 bits per expected key, 4 more for the coarse level: well under 1 %; the coarse level only removes candidates
    assert rates[12_000_000] < 0.01 and rates[10_000_000] < 0.03 and rates[12_000_000] <= rates[10_000_000]


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. partitioned aggregate of the fused pipeline at its natural size
# ---------------------------------------------------------------------------------------------------------------------------------
SF_PART, SF_SMALL = 5, 1


def q3_fused(ctx, monkeypatch, tables, pushes=1, direct=False):
    """TPC-H Q3 as fused pipelines (no hook); direct=True sets DFGPU_PIPE_VAR, which partitioned_table_bytes refuses.
    returns (result rows, sink rows, partitioned launches, orders lookup table bytes)"""
    customer, orders, li = tables
    for v in ("DFGPU_PIPE_RADIX_PARTS", "DFGPU_PIPE_RADIX_CAP", "DFGPU_PIPE_VAR"):
        monkeypatch.delenv(v, raising=False)
    if direct:
        monkeypatch.setenv("DFGPU_PIPE_VAR", "11")
    kmin, kmax, _ = D.column_minmax_device(ctx, customer.cols[0])
    l1 = D.Lookup(ctx, D.INT64, [], key_range=(kmin, kmax))
    p = D.Pipeline(ctx, customer.types, B(D.OP_EQ, C(1), L(1))); p.sink_build(l1, 0, []); p.push_device(customer.cols); p.finish(); p.close()
    l2 = D.Lookup(ctx, D.INT64, [D.INT32, D.INT32], n_acc_words=2, membership_filter=1)
    p = D.Pipeline(ctx, orders.types, B(D.OP_LT, C(2), L(Q.CUT, D.INT32)), [(D.STAGE_SEMI, 1, l1)]); p.sink_build(l2, 0, [2, 3])
    p.push_device(orders.cols); p.finish(); p.close()
    p = D.Pipeline(ctx, li.types, B(D.OP_GT, C(3), L(Q.CUT, D.INT32)), [(D.STAGE_INNER, 0, l2)], name="lineitem")
    p.sink_aggregate([0, 4, 5], [(D.AGG_SUM, Q.revenue_expr(li.types))], D.AGG_SINGLE_PARTITIONED)
    for _ in range(pushes):
        p.push_device(li.cols)
    p.finish()
    res = p.drain(host=False)
    out = Q.result_rows(ctx, res), p.metric("sink_rows"), p.metric("partitioned_launches"), l2.metric("table_bytes")
    for b in res:
        b.release()
    p.close(); l2.close(); l1.close()
    monkeypatch.delenv("DFGPU_PIPE_VAR", raising=False)
    return out


@pytest.fixture(scope="module")
def q3_large(gpu_ctx):
    tables = Q.gen_tables(gpu_ctx, SF_PART)
    exp = Q.q3_expected(*(t.host(gpu_ctx) for t in tables))
    return tables, exp


@pytest.mark.parametrize("pushes", [1, 2])
def test_partitioned_q3_aggregate_at_its_natural_size(gpu_ctx, monkeypatch, q3_large, pushes):
    tables, exp = q3_large
    rows, sink, launches, tbytes = q3_fused(gpu_ctx, monkeypatch, tables, pushes)
    assert tbytes > L2_RULE, f"SF{SF_PART}: the orders table ({tbytes} B) no longer exceeds the partitioning threshold"
    assert launches == pushes
    assert rows == [(k, d, p, pushes * s) for k, d, p, s in exp] and len(exp) > 100_000
    drows, dsink, dlaunches, _ = q3_fused(gpu_ctx, monkeypatch, tables, pushes, direct=True)
    assert dlaunches == 0 and drows == rows and dsink == sink


def test_q3_aggregate_under_the_threshold_keeps_the_direct_probe(gpu_ctx, monkeypatch):
    tables = Q.gen_tables(gpu_ctx, SF_SMALL, seed=5)
    rows, _, launches, tbytes = q3_fused(gpu_ctx, monkeypatch, tables)
    assert tbytes < L2_RULE and launches == 0
    assert rows == Q.q3_expected(*(t.host(gpu_ctx) for t in tables))


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. radix-partitioned join probe at its natural size
# ---------------------------------------------------------------------------------------------------------------------------------
RADIX_MIN_ROWS = 1 << 22


def inline_table_bytes(build_rows, words):
    """hashed inline table: 2.5 slots per build row, rounded up to 4 slots; 8 B per word"""
    return ((max(1024, build_rows * 250 // 100) + 3) & ~3) * 8 * words


def radix_data(seed, nb, npr, nullable=False):
    rng = np.random.default_rng(seed)
    ids = rng.permutation(2 * nb)
    bk = sparse_keys(ids[:nb])
    pk = sparse_keys(np.where(rng.random(npr) < 0.6, ids[:nb][rng.integers(0, nb, npr)], ids[nb:][rng.integers(0, nb, npr)]))
    kvalid = None
    if nullable:
        kvalid = rng.random(npr) > 0.01
    build = [(bk, None), (rng.integers(-2**63, 2**63 - 1, nb, dtype=np.int64), None)]
    probe = [(pk, kvalid), (rng.integers(-2**63, 2**63 - 1, npr, dtype=np.int64), None), (rng.integers(-2**63, 2**63 - 1, npr, dtype=np.int64), None)]
    return build, probe


def radix_join(ctx, build, probe, out, key_offset=0):
    """unordered inner join, probe pushed from device memory; key_offset > 0 shifts the key column's start by that many rows"""
    j = new_join(ctx, build, [D.INT64, D.INT64], [D.INT64] * 3, [0], [0], out, (0, float("inf")), ordered_output=False)
    hc = [host_col(v, val, D.INT64) for v, val in probe]
    dc = [D.DeviceColumn.from_host(ctx, h) for h in hc]
    cols = [c.c() for c in dc]
    keep = None
    if key_offset:
        keep = ctx.to_device(np.concatenate([np.zeros(key_offset, np.int64), probe[0][0]]))
        cols[0].values, cols[0].offset = keep.ptr, key_offset
    j.push_probe_device(cols)
    j.finish_probe()
    got = batches_arrays(j.drain(host=True), len(out))
    m = probe_metrics(j)
    j.close()
    return got, m


def radix_expected(build, probe, out):
    prow, brow = unique_join_rows(build[0][0], probe[0][0], probe[0][1])
    return expected_columns(build, probe, out, prow, brow)


OUT_PAYLOAD = [(0, 0), (0, 1), (1, 0), (1, 1)]          # build key + payload (W = 2), probe key + one carried column
OUT_NO_PAYLOAD = [(0, 0), (1, 0), (1, 1)]               # no payload (W = 1)


@pytest.mark.parametrize("nb,out,words", [(1_200_000, OUT_PAYLOAD, 2), (2_200_000, OUT_NO_PAYLOAD, 1)], ids=["payload", "no_payload"])
def test_radix_probe_at_its_natural_size(gpu_ctx, nb, out, words):
    assert inline_table_bytes(nb, words) > L2_RULE
    npr = RADIX_MIN_ROWS + 1234
    build, probe = radix_data(11 + words, nb, npr)
    got, m = radix_join(gpu_ctx, build, probe, out)
    exp = radix_expected(build, probe, out)
    assert m["radix_partitioned_probes"] == 1 and m["array_map_created_count"] == 0, m
    assert m["probe_hits"] == len(exp[0]) == m["output_rows"] and m["input_rows"] == npr, m
    assert_same_multiset(got, exp, f"radix probe W={words}")


@pytest.mark.parametrize("case", ["misaligned_key", "nullable_key", "two_carried_columns", "one_row_short"])
def test_radix_probe_refusals_keep_the_rows(gpu_ctx, case):
    nb = 1_200_000
    assert inline_table_bytes(nb, 2) > L2_RULE
    npr = RADIX_MIN_ROWS - 1 if case == "one_row_short" else RADIX_MIN_ROWS + 1234
    build, probe = radix_data(31, nb, npr, nullable=case == "nullable_key")
    out = OUT_PAYLOAD + [(1, 2)] if case == "two_carried_columns" else OUT_PAYLOAD
    got, m = radix_join(gpu_ctx, build, probe, out, key_offset=1 if case == "misaligned_key" else 0)   # 8 B past a 16 B boundary
    exp = radix_expected(build, probe, out)
    assert m["radix_partitioned_probes"] == 0 and m["probe_hits"] == len(exp[0]) == m["output_rows"], m
    assert_same_multiset(got, exp, f"radix refusal {case}")
