"""The dense aggregate sink's accumulators (pipe_kernel<SINK_DENSE>): both accumulator paths (one copy of the slots per warp with plain
stores, one per block with shared atomics; dfgpu_pipeline_metric "dense_block_launches" says which ran), every operator over Int64,
UInt64, Float64 and Decimal128, the MIN / MAX identities and NULL rules, 128-bit carries and wrapping, the Decimal128 AVG rule at capped
precisions and scales, the peer-combining shuffle tree, key domains at the ends of the integer types, predicate terms beyond
kMaxTerms and the 48 KB per-warp threshold.  Every result is compared with a plain reference (tests/dense_cases.py: Python ints,
math.fsum for Float64 sums) and, where the oracle covers the case, with the oracle's unfused chain."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import decimal_agg as DA
import dense_cases as C
from decimal_util import gpu_col_as_py, gpu_host_col, gpu_nodes
from test_gpu_pipe_dense import assert_rows, bop, col, lit, oracle_dense, run_dense

pytestmark = pytest.mark.gpu


def nodes_of(aggs):
    return [(f, None if c is None else [col(c)]) for f, c in aggs]


def dense(ctx, cols, types, group_cols, key_range, aggs, pred=None, keep=None, mode=D.AGG_SINGLE, what="", **kw):
    """run the fused sink on cols and compare it with the reference; aggs: [(func, argument column or None)] -> metrics"""
    got, _, m = run_dense(ctx, cols, types, pred, group_cols, key_range, nodes_of(aggs), mode=mode, **kw)
    want = C.reference(cols, types, keep, group_cols, key_range, aggs, partial=mode == D.AGG_PARTIAL)
    C.check_rows(got, want, what)
    m["rows"] = got
    return m


def dense_both(ctx, cols, types, small, big, aggs, what="", **kw):
    """the same data on both accumulator paths: small = (group_cols, key_range) of a per-warp domain, big = one of >= 200 slots"""
    ms = dense(ctx, cols, types, *small, aggs, what=what + " per-warp", **kw)
    mb = dense(ctx, cols, types, *big, aggs, what=what + " per-block", **kw)
    assert ms["dense_block_launches"] == 0 and mb["dense_block_launches"] > 0, what
    assert mb["num_groups"] >= 200, what
    return ms, mb


def dec_col(vals, p, s, valid=None):
    return (O.Dec(vals, p, s), valid)


# ---- a. every operator, both paths ----------------------------------------------------------------------
def matrix_data(rng, n):
    """0 key Int32 in [0, 3] (NULL ~3%), 1 key Int16 in [0, 49], 2 Int64, 3 UInt64, 4 Float64 whose group sums cancel, 5 Decimal128(38, 6).
    The second half of the rows repeats the keys of the first half with the negated Float64 values plus a small term."""
    h = n // 2
    k1 = rng.integers(0, 4, h).astype(np.int32); k1v = rng.random(h) > 0.03
    k2 = rng.integers(0, 50, h).astype(np.int16)
    f = np.round(rng.standard_normal(h) * 1e9, 3)
    small = rng.standard_normal(h)
    cols = [(np.concatenate([k1, k1]), np.concatenate([k1v, k1v])), (np.concatenate([k2, k2]), None),
            (rng.integers(C.I64_MIN, C.I64_MAX, 2 * h, endpoint=True), rng.random(2 * h) > 0.1),
            (rng.integers(0, C.U64_MAX, 2 * h, dtype=np.uint64, endpoint=True), rng.random(2 * h) > 0.1),
            (np.concatenate([f, -f + small]), rng.random(2 * h) > 0.05),
            dec_col([int(a) * 10 ** 10 + int(b) for a, b in zip(rng.integers(-10 ** 17, 10 ** 17, 2 * h), rng.integers(0, 10 ** 10, 2 * h))],
                    38, 6, rng.random(2 * h) > 0.1)]
    perm = rng.permutation(2 * h)
    cols = [(c[0][perm], None if c[1] is None else c[1][perm]) for c in cols]
    return cols, [D.INT32, D.INT16, D.INT64, D.UINT64, D.FLOAT64, D.decimal128(38, 6)]


MATRIX_AGGS = {
    "int": [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, 2), (D.AGG_MIN, 2), (D.AGG_MAX, 2), (D.AGG_SUM, 3), (D.AGG_MIN, 3), (D.AGG_MAX, 3),
            (D.AGG_COUNT, 3)],
    "float": [(D.AGG_SUM, 4), (D.AGG_MIN, 4), (D.AGG_MAX, 4), (D.AGG_AVG, 4), (D.AGG_COUNT, 4), (D.AGG_COUNT_STAR, None)],
    # Decimal128 fields at padded (MIN, SUM, AVG) and unpadded (MAX) offsets
    "decimal": [(D.AGG_MIN, 5), (D.AGG_COUNT, 5), (D.AGG_MAX, 5), (D.AGG_SUM, 5), (D.AGG_AVG, 5), (D.AGG_COUNT_STAR, None), (D.AGG_SUM, 2)],
}
SMALL, BIG = ([0], [(0, 3)]), ([0, 1], [(0, 3), (0, 49)])   # 5 slots; 5 x 51 = 255 slots


@pytest.mark.parametrize("which", list(MATRIX_AGGS))
def test_operator_matrix_on_both_paths(gpu_ctx, which):
    cols, types = matrix_data(np.random.default_rng(101), 60_000)
    aggs = MATRIX_AGGS[which]
    ms, mb = dense_both(gpu_ctx, cols, types, SMALL, BIG, aggs, what=which, batch_rows=17_000, device=which == "float")
    if which != "float":   # the oracle's unfused chain agrees (Float64 sums are compared against math.fsum only)
        for (g, r), m in ((SMALL, ms), (BIG, mb)):
            assert_rows(m["rows"], oracle_dense(cols, None, g, nodes_of(aggs)), which + " oracle")
    if which == "float":   # Partial: AVG's state columns [count, sum] on the per-block path
        m = dense(gpu_ctx, cols, types, *BIG, aggs, mode=D.AGG_PARTIAL, what="partial", batch_rows=25_000)
        assert m["dense_block_launches"] > 0 and len(m["rows"][0]) == 2 + len(aggs) + 1


# ---- b. values equal to the MIN / MAX identities, and the NULL rules ---------------------------------------
def identity_data(rng, n):
    """0 key Int32 in [0, 9] and NULL, 1 key Int32 in [0, 19], 2 Int64, 3 UInt64, 4 Float64 with +-inf, 5 Decimal128(38, 0),
    6 finite Float64.  Key 0 holds only the largest values, key 1 only the smallest, key 2 only NULL arguments."""
    g = rng.integers(0, 11, n)
    nul = (g == 2) | (rng.random(n) < 0.1) & (g > 2)
    ext = rng.random(n)
    def pick(lo, hi, rand):
        v = rand.copy() if not isinstance(rand, list) else list(rand)
        for i in range(n):
            if g[i] == 0 or (g[i] > 2 and ext[i] < 0.1):
                v[i] = hi
            elif g[i] == 1 or (g[i] > 2 and ext[i] > 0.9):
                v[i] = lo
        return v
    i64 = pick(C.I64_MIN, C.I64_MAX, rng.integers(-10 ** 12, 10 ** 12, n))
    u64 = pick(0, C.U64_MAX, rng.integers(1, 1 << 63, n, dtype=np.uint64))
    f64 = pick(-np.inf, np.inf, rng.standard_normal(n) * 1e6)
    dec = pick(-C.DEC38_MAX, C.DEC38_MAX, [int(x) * 10 ** 20 for x in rng.integers(-10 ** 17, 10 ** 17, n)])
    fin = np.round(rng.standard_normal(n) * 1e3, 2)
    v = ~nul
    cols = [(np.minimum(g, 9).astype(np.int32), g < 10), (rng.integers(0, 20, n).astype(np.int32), None), (i64, v), (u64, v), (f64, v),
            dec_col(dec, 38, 0, v), (fin, v)]
    return cols, [D.INT32, D.INT32, D.INT64, D.UINT64, D.FLOAT64, D.decimal128(38, 0), D.FLOAT64]


IDENTITY_AGGS = [
    [(D.AGG_MIN, 2), (D.AGG_MAX, 2), (D.AGG_MIN, 3), (D.AGG_MAX, 3), (D.AGG_SUM, 2), (D.AGG_SUM, 3), (D.AGG_COUNT, 2), (D.AGG_COUNT_STAR, None)],
    [(D.AGG_MIN, 4), (D.AGG_MAX, 4), (D.AGG_MIN, 5), (D.AGG_MAX, 5), (D.AGG_SUM, 5), (D.AGG_AVG, 6), (D.AGG_COUNT, 5), (D.AGG_COUNT_STAR, None)],
]


@pytest.mark.parametrize("which", [0, 1], ids=["integers", "float_decimal"])
def test_identity_values_and_null_rules_on_both_paths(gpu_ctx, which):
    cols, types = identity_data(np.random.default_rng(202), 24_000)
    aggs = IDENTITY_AGGS[which]
    ms, mb = dense_both(gpu_ctx, cols, types, ([0], [(0, 9)]), ([0, 1], [(0, 9), (0, 19)]), aggs, what="identities", batch_rows=9000)
    top, bottom, nulls = ms["rows"][0], ms["rows"][1], ms["rows"][2]
    assert top[0] == 0 and bottom[0] == 1 and nulls[0] == 2
    if which == 0:
        assert top[1:5] == (C.I64_MAX, C.I64_MAX, C.U64_MAX, C.U64_MAX) and bottom[1:5] == (C.I64_MIN, C.I64_MIN, 0, 0)
    else:
        assert top[1:5] == (np.inf, np.inf, C.DEC38_MAX, C.DEC38_MAX) and bottom[1:5] == (-np.inf, -np.inf, -C.DEC38_MAX, -C.DEC38_MAX)
    # arguments all NULL, rows present: MIN / MAX / SUM / AVG NULL, COUNT(x) 0, COUNT(*) > 0
    assert nulls[1:7] == (None,) * 6 and nulls[7] == 0 and nulls[8] > 0


# ---- c. 128-bit carries and wrapping ----------------------------------------------------------------------
CARRY_AGGS = [(D.AGG_SUM, 2), (D.AGG_MIN, 2), (D.AGG_MAX, 2), (D.AGG_COUNT_STAR, None)]


@pytest.mark.parametrize("n", [60_000, 1000], ids=["blocks", "one_block"])
def test_decimal_carries_and_wrapping_on_both_paths(gpu_ctx, n):
    cols, types = C.carry_case(np.random.default_rng(31), n)
    ms, mb = dense_both(gpu_ctx, cols, types, ([0], [(0, 7)]), ([0, 1], [(0, 7), (0, 24)]), CARRY_AGGS, what="carries",
                        batch_rows=None if n <= 1024 else 25_000)
    rows = {r[0]: r for r in ms["rows"]}
    assert rows[1][1] < 0 and rows[6][2:4] == ((1 << 63) - 1, 1 << 63) and rows[7][2:4] == (-(1 << 64), -1)
    assert_rows(ms["rows"], oracle_dense(cols, None, [0], nodes_of(CARRY_AGGS)), "carries oracle")


# ---- d. AVG over Decimal128 ----------------------------------------------------------------------------
@pytest.mark.parametrize("p,s", C.AVG_TYPES)
def test_decimal_avg_rule(gpu_ctx, p, s):
    cols, types = C.avg_case(np.random.default_rng(41 + p), p, s)
    aggs = [(D.AGG_AVG, 1), (D.AGG_SUM, 1), (D.AGG_COUNT, 1), (D.AGG_COUNT_STAR, None)]
    got, ot, m = run_dense(gpu_ctx, cols, types, None, [0], [(0, 3)], nodes_of(aggs), batch_rows=1500)
    C.check_rows(got, C.reference(cols, types, None, [0], [(0, 3)], aggs), "avg")
    assert_rows(got, oracle_dense(cols, None, [0], nodes_of(aggs)), "avg oracle")
    assert ot[1] == D.decimal128(min(38, p + 4), min(38, s + 4)) and m["dense_block_launches"] == 0
    assert any(r[1] < 0 for r in got)


@pytest.mark.parametrize("p,s,inside,outside", [(36, 35, 10 ** 35 - 1, 10 ** 35), (36, 35, -(10 ** 35 - 1), -(10 ** 35)),
                                                (38, 0, 10 ** 34 - 1, 10 ** 34)], ids=["36_35", "36_35_negative", "38_0"])
def test_decimal_avg_just_inside_and_outside_the_target_precision(gpu_ctx, p, s, inside, outside):
    """Decimal128(36, 35) -> (38, 38): sum * 10^3 / count; Decimal128(38, 0) -> (38, 4): sum * 10^4 / count.  The value just inside
    the 38 digits is exact, the one just outside is DFGPU_ERR_ARITH like DecimalAverager::avg's error"""
    aggs = [(D.AGG_AVG, 1), (D.AGG_COUNT_STAR, None)]
    for v, ok in ((inside, True), (outside, False)):
        cols, types = [(np.zeros(3, np.int32), None), dec_col([v, 0, 7], p, s, np.array([True, False, False]))], [D.INT32, D.decimal128(p, s)]
        if ok:
            got, _, _ = run_dense(gpu_ctx, cols, types, None, [0], [(0, 0)], nodes_of(aggs))
            assert got == [(0, v * 10 ** C.avg_mul(p, s), 3)] == C.reference(cols, types, None, [0], [(0, 0)], aggs)
            assert abs(got[0][1]) == 10 ** 38 - 10 ** C.avg_mul(p, s)
        else:
            with pytest.raises(O.ArrowArithmeticOverflow):
                DA.decimal_avg(v, 1, p, s)
            with pytest.raises(D.DfgpuError) as ei:
                run_dense(gpu_ctx, cols, types, None, [0], [(0, 0)], nodes_of(aggs))
            assert ei.value.code == -4


# ---- e. peer-combining patterns ---------------------------------------------------------------------------
PEER_AGGS = [(D.AGG_SUM, 2), (D.AGG_MIN, 2), (D.AGG_SUM, 3), (D.AGG_MAX, 3), (D.AGG_COUNT, 3), (D.AGG_COUNT_STAR, None)]
PEER_SIZES = [1, 31, 257, 1025, 300_007]


def peer_data(rng, n, pattern):
    """0 key Int32, 1 filter column Int32 (the sparse pattern keeps the rows where it is 0), 2 Decimal128(38, 0) values +-(2^63 + r)
    whose low words carry whenever two of one sign meet, 3 Int64 (~5% NULL)"""
    r = np.arange(n)
    key, kv = {"one": (np.full(n, 5), None), "null": (np.full(n, 5), np.zeros(n, bool)), "lanes": (r % 32, None), "mod3": (r % 3, None),
               "sparse": (r % 32, None)}[pattern]
    filt = rng.integers(0, 97, n).astype(np.int32) if pattern == "sparse" else np.zeros(n, np.int32)
    mag = rng.integers(0, 1 << 62, n)
    sign = rng.random(n) < 0.3
    dec = [-((1 << 63) + int(m)) if s else (1 << 63) + int(m) for m, s in zip(mag.tolist(), sign.tolist())]
    return ([(key.astype(np.int32), kv), (filt, None), dec_col(dec, 38, 0), (rng.integers(-10 ** 15, 10 ** 15, n), rng.random(n) > 0.05)],
            [D.INT32, D.INT32, D.decimal128(38, 0), D.INT64])


@pytest.mark.parametrize("pattern", ["one", "null", "lanes", "mod3", "sparse"])
def test_peer_combining_patterns(gpu_ctx, pattern):
    rng = np.random.default_rng(303)
    pred = [col(1), lit(0, np.int32), bop(O.OP_EQ)]
    for n in PEER_SIZES:
        cols, types = peer_data(rng, n, pattern)
        keep = cols[1][0] == 0
        what = f"{pattern} n={n}"
        # [0, 31]: 33 slots x 14 words, per-warp; [0, 200]: 202 slots, per-block
        ms = dense(gpu_ctx, cols, types, [0], [(0, 31)], PEER_AGGS, pred=pred, keep=keep, what=what + " per-warp", device=n > 1000)
        mb = dense(gpu_ctx, cols, types, [0], [(0, 200)], PEER_AGGS, pred=pred, keep=keep, what=what + " per-block")
        assert ms["dense_block_launches"] == 0 and mb["dense_block_launches"] == 1, what
        assert ms["sink_rows"] == mb["sink_rows"] == int(keep.sum())
    assert pattern != "sparse" or 2_500 < int(keep.sum()) < 3_700


def test_many_small_pushes_host_and_device_with_an_empty_batch(gpu_ctx):
    rng = np.random.default_rng(304)
    cols, types = peer_data(rng, 6000, "mod3")
    cols[0] = (rng.integers(0, 40, 6000).astype(np.int32), rng.random(6000) > 0.1)
    sizes = [1, 31, 0, 257, 1, 1025, 0, 500, 2185]
    assert sum(sizes) == 4000
    for key_range, block in (((0, 39), 0), ((0, 200), 1)):
        p = D.Pipeline(gpu_ctx, types)
        p.sink_aggregate_dense([0], [key_range], [(f, gpu_nodes(D, nd) if nd else None) for f, nd in nodes_of(PEER_AGGS)])
        keep, s = [], 0
        for i, k in enumerate(sizes):
            hc = [gpu_host_col(D, (c[0][s:s + k], None if c[1] is None else c[1][s:s + k]), t) for c, t in zip(cols, types)]
            if i % 2 and k:
                dc = [D.DeviceColumn.from_host(gpu_ctx, h) for h in hc]
                keep.append(dc)
                p.push_device(dc)
            else:
                p.push_host(hc)
            s += k
        p.finish()
        got = []
        for b in p.drain(host=True):
            got += list(zip(*[gpu_col_as_py(D, b, i)[0] for i in range(b.num_columns)]))
        launches, rows_in = p.metric("dense_block_launches"), p.metric("input_rows")
        p.close()
        part = [(c[0][:4000], None if c[1] is None else c[1][:4000]) for c in cols]
        C.check_rows(got, C.reference(part, types, None, [0], [key_range], PEER_AGGS), "pushes")
        assert launches == block * (len(sizes) - 2) and rows_in == 4000


# ---- f. key domains and key sources -----------------------------------------------------------------------
KEY_AGGS = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, 1), (D.AGG_MIN, 1)]


def key_cases():
    u = 1 << 64
    return {   # name: (key type, declared (min, max), values drawn from, NULL share)
        "int8_full": (D.INT8, (-128, 126), (-128, 127), 0.05),
        "uint8_full": (D.UINT8, (0, 254), (0, 255), 0.05),
        "uint64_top": (D.UINT64, (u - 200, u - 1), (u - 200, u), 0.05),
        "int64_bottom": (D.INT64, (C.I64_MIN, C.I64_MIN + 200), (C.I64_MIN, C.I64_MIN + 201), 0.05),
        "int64_top": (D.INT64, (C.I64_MAX - 200, C.I64_MAX), (C.I64_MAX - 200, C.I64_MAX + 1), 0.05),
        "date32": (D.DATE32, (19_000, 19_100), (19_000, 19_101), 0.05),
    }


def key_column(rng, t, lo, hi, n, null_share):
    dt = D.NP_OF_TYPE[t]
    v = np.array([lo + int(x) for x in rng.integers(0, hi - lo, n)], dtype=object).astype(dt)
    return (v, rng.random(n) > null_share)


@pytest.mark.parametrize("name", list(key_cases()))
def test_key_domains_at_the_ends_of_their_types(gpu_ctx, name):
    t, rng_decl, rng_draw, nulls = key_cases()[name]
    rng = np.random.default_rng(404)
    n = 40_000
    cols = [key_column(rng, t, *rng_draw, n, nulls), (rng.integers(-10 ** 12, 10 ** 12, n), rng.random(n) > 0.05)]
    types = [t, D.INT64]
    m = dense(gpu_ctx, cols, types, [0], [rng_decl], KEY_AGGS, what=name, batch_rows=15_000)
    span = (rng_decl[1] - rng_decl[0]) % (1 << 64)
    assert m["num_groups"] == span + 2 and m["rows"][-1][0] is None
    assert m["rows"][0][0] == rng_decl[0] and m["rows"][-2][0] == rng_decl[1]


def test_eight_one_value_keys_decode_every_stride(gpu_ctx):
    rng = np.random.default_rng(405)
    n = 30_000
    kt = [D.INT8, D.INT16, D.INT32, D.INT64, D.UINT8, D.UINT16, D.UINT32, D.DATE32]
    kv = [-5, 300, -70_000, 1 << 40, 200, 60_000, 4_000_000_000, 19_000]
    cols = [(np.full(n, v, D.NP_OF_TYPE[t]), rng.random(n) > 0.5) for t, v in zip(kt, kv)] + [(rng.integers(-1000, 1000, n), None)]
    types = kt + [D.INT64]
    aggs = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, 8), (D.AGG_MAX, 8)]
    m = dense(gpu_ctx, cols, types, list(range(8)), [(v, v) for v in kv], aggs, what="eight keys", batch_size=100)
    assert m["num_groups"] == 256 and m["batches"] == 3 and m["dense_block_launches"] > 0
    for i, r in enumerate(m["rows"]):     # slot i: bit 7 - g says whether key g is NULL
        assert [x is None for x in r[:8]] == [bool((i >> (7 - g)) & 1) for g in range(8)]


def test_three_keys_of_mixed_types(gpu_ctx):
    rng = np.random.default_rng(406)
    n = 40_000
    cols = [key_column(rng, D.INT8, -3, 2, n, 0.05), key_column(rng, D.UINT32, 4_000_000_000, 4_000_000_006, n, 0.05),
            key_column(rng, D.DATE32, 18_000, 18_004, n, 0.05), (rng.integers(-10 ** 12, 10 ** 12, n), None)]
    types = [D.INT8, D.UINT32, D.DATE32, D.INT64]
    aggs = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, 3), (D.AGG_MIN, 3), (D.AGG_MAX, 3)]
    m = dense(gpu_ctx, cols, types, [0, 1, 2], [(-3, 1), (4_000_000_000, 4_000_000_005), (18_000, 18_003)], aggs, what="three keys",
              device=True, batch_rows=12_000)
    assert m["num_groups"] == 6 * 7 * 5
    assert_rows(m["rows"], oracle_dense(cols, None, [0, 1, 2], nodes_of(aggs)), "three keys oracle")


def test_stage_payload_keys_and_arguments(gpu_ctx):
    """an INNER stage's negative Int8 payload as the group key, its Int16 payload inside aggregates"""
    rng = np.random.default_rng(407)
    nb, n = 1000, 50_000
    p8 = rng.integers(-5, 5, nb).astype(np.int8)
    p16 = rng.integers(-30_000, 30_000, nb).astype(np.int16)
    lk = D.Lookup(gpu_ctx, D.INT64, [D.INT8, D.INT16], expected_rows=nb)
    bp = D.Pipeline(gpu_ctx, [D.INT64, D.INT8, D.INT16])
    bp.sink_build(lk, 0, [1, 2])
    bp.push_host([D.HostColumn(np.arange(1, nb + 1, dtype=np.int64), None, D.INT64), D.HostColumn(p8, None, D.INT8),
                  D.HostColumn(p16, None, D.INT16)])
    bp.finish(); bp.close()
    cust = rng.integers(1, nb + 201, n)
    tag = rng.integers(0, 3, n).astype(np.int32)
    price = rng.integers(-10 ** 9, 10 ** 9, n)
    cols, types = [(cust, None), (price, None), (tag, None)], [D.INT64, D.INT64, D.INT32]
    hit = cust <= nb
    idx = np.where(hit, cust - 1, 0)
    vcols, vtypes = cols + [(p8[idx], None), (p16[idx], None)], types + [D.INT8, D.INT16]
    aggs = [(D.AGG_SUM, 4), (D.AGG_MIN, 4), (D.AGG_MAX, 4), (D.AGG_SUM, 1), (D.AGG_COUNT_STAR, None)]
    for g, r in (([3], [(-5, 4)]), ([3, 2], [(-5, 4), (0, 2)])):
        got, ot, m = run_dense(gpu_ctx, cols, types, None, g, r, nodes_of(aggs), stages=[(D.STAGE_INNER, 0, lk)], batch_rows=20_000)
        C.check_rows(got, C.reference(vcols, vtypes, hit, g, r, aggs), "payload")
        assert ot[0] == D.INT8 and got[0][0] == -5 and m["sink_rows"] == int(hit.sum())
    lk.close()


def test_keys_outside_the_range_on_rejected_rows_do_not_raise(gpu_ctx):
    rng = np.random.default_rng(408)
    n = 30_000
    k = rng.integers(0, 20, n).astype(np.int32)
    cols, types = [(k, None), (rng.integers(-1000, 1000, n), None), (np.arange(n, dtype=np.int64), None)], [D.INT32, D.INT64, D.INT64]
    pred = [col(0), lit(9, np.int32), bop(O.OP_LTEQ)]
    dense(gpu_ctx, cols, types, [0], [(0, 9)], KEY_AGGS, pred=pred, keep=k <= 9, what="predicate")
    inside = np.nonzero(k <= 9)[0].astype(np.int64)
    lk = D.Lookup(gpu_ctx, D.INT64, [], expected_rows=len(inside))
    bp = D.Pipeline(gpu_ctx, [D.INT64])
    bp.sink_build(lk, 0, [])
    bp.push_host([D.HostColumn(inside, None, D.INT64)]); bp.finish(); bp.close()
    dense(gpu_ctx, cols, types, [0], [(0, 9)], KEY_AGGS, keep=k <= 9, what="semi", stages=[(D.STAGE_SEMI, 2, lk)])
    lk.close()


U = 1 << 64


@pytest.mark.parametrize("t,lo,hi,bad", [
    (D.INT32, 0, 9, -1), (D.INT32, 0, 9, 10), (D.UINT8, 1, 254, 0), (D.UINT8, 0, 254, 255),
    (D.UINT64, U - 200, U - 1, U - 201), (D.UINT64, U - 200, U - 2, U - 1), (D.UINT64, 0, 10, U - 1), (D.UINT64, 5, 10, 11),
    (D.INT64, C.I64_MIN + 1, C.I64_MIN + 9, C.I64_MIN), (D.INT64, C.I64_MAX - 9, C.I64_MAX - 1, C.I64_MAX),
    (D.DATE32, 19_000, 19_010, 19_011)],
    ids=["int32_min-1", "int32_max+1", "uint8_min-1", "uint8_max+1", "uint64_min-1", "uint64_max+1", "uint64_0_min-1_wraps",
         "uint64_max+1_small", "int64_min-1", "int64_max+1", "date32_max+1"])
def test_a_kept_key_just_outside_its_range_raises(gpu_ctx, t, lo, hi, bad):
    n = 5000
    vals = np.array([lo + (i % (hi - lo + 1)) for i in range(n)], dtype=object)
    vals[3777] = bad
    cols, types = [(vals.astype(D.NP_OF_TYPE[t]), None), (np.ones(n, np.int64), None)], [t, D.INT64]
    with pytest.raises(D.DfgpuError) as ei:
        run_dense(gpu_ctx, cols, types, None, [0], [(lo, hi)], nodes_of(KEY_AGGS))
    assert ei.value.code == -1
    ok = [(c[0][:3777], None) for c in cols]        # the rows before it are fine
    dense(gpu_ctx, ok, types, [0], [(lo, hi)], KEY_AGGS, what="inside")


# ---- g. conjunctions longer than kMaxTerms --------------------------------------------------------------------
def term_data(rng, n):
    """0 key Int32 in [0, 4], 1 value Int64, then the term columns: 2 a Int64, 3 b Int64 (10% NULL), 4 c UInt64 around 2^63, 5 d Int8,
    6 e Date32, 7 f Int32 (mostly 0), 8 g, 9 h, 10 i Int64"""
    cols = [(rng.integers(0, 5, n).astype(np.int32), None), (rng.integers(-10 ** 9, 10 ** 9, n), None),
            (rng.integers(-1000, 1000, n), None), (rng.integers(0, 50, n), rng.random(n) > 0.1),
            (rng.integers((1 << 63) - (1 << 60), C.U64_MAX, n, dtype=np.uint64, endpoint=True), None),
            (rng.integers(-128, 128, n).astype(np.int8), None), (rng.integers(18_000, 20_000, n).astype(np.int32), None),
            ((rng.random(n) < 0.1).astype(np.int32), None), (rng.integers(0, 100, n), None), (rng.integers(-10, 100, n), None),
            (rng.integers(0, 1100, n), None)]
    return cols, [D.INT32, D.INT64, D.INT64, D.INT64, D.UINT64, D.INT8, D.DATE32, D.INT32, D.INT64, D.INT64, D.INT64]


TERMS = {   # name: (column, literal, literal type, op)
    "a": (2, -900, np.int64, O.OP_GT), "b": (3, 7, np.int64, O.OP_NEQ), "c": (4, (1 << 63) + 1000, np.uint64, O.OP_GTEQ),
    "d": (5, 100, np.int8, O.OP_LT), "e": (6, 19_500, np.int32, O.OP_LTEQ), "f": (7, 0, np.int32, O.OP_EQ),
    "g": (8, 5, np.int64, O.OP_GT), "h": (9, -3, np.int64, O.OP_GTEQ), "i": (10, 1000, np.int64, O.OP_LTEQ),
}


def conjunction(names):
    nodes = []
    for k, nm in enumerate(names):
        c, v, dt, op = TERMS[nm]
        nodes += [col(c), lit(v, dt), bop(op)] + ([bop(O.OP_AND)] if k else [])
    return nodes


@pytest.mark.parametrize("order", ["aghibcde", "cegh" + "fabd"])
def test_conjunctions_past_kmaxterms(gpu_ctx, order):
    """the first four terms sit in PipeParams, terms five to eight in DenseParams; nine terms run the interpreter.  Over the two
    orders the extra terms carry all six comparison ops, a nullable column, UInt64 against 2^63 + 1000, Int8 and Date32"""
    cols, types = term_data(np.random.default_rng(505), 60_000)
    aggs = [(D.AGG_COUNT_STAR, None), (D.AGG_SUM, 1), (D.AGG_MIN, 1)]
    names = list(order) + [x for x in "abcdefghi" if x not in order]
    for k in range(5, 10):
        pred = conjunction(names[:k])
        f, fv = O.eval_expr(cols, pred)     # the oracle's filter
        keep = np.asarray(f, bool) & (True if fv is None else np.asarray(fv, bool))
        m = dense(gpu_ctx, cols, types, [0], [(0, 4)], aggs, pred=pred, keep=keep, what=f"{k} terms", batch_rows=25_000)
        assert m["sink_rows"] == int(keep.sum()) > 1000


# ---- h. the per-warp threshold, and the largest layout ---------------------------------------------------------
def test_per_warp_threshold_at_48k(gpu_ctx):
    rng = np.random.default_rng(606)
    n = 60_000
    cols = [(rng.integers(0, 191, n).astype(np.int32), rng.random(n) > 0.02), (rng.integers(-10 ** 15, 10 ** 15, n), rng.random(n) > 0.1)]
    types = [D.INT32, D.INT64]
    aggs = [(D.AGG_SUM, 1)]
    assert C.per_warp(192, [(D.AGG_SUM, False)]) and not C.per_warp(193, [(D.AGG_SUM, False)])
    m192 = dense(gpu_ctx, cols, types, [0], [(0, 190)], aggs, what="192 slots", batch_rows=20_000)
    m193 = dense(gpu_ctx, cols, types, [0], [(0, 191)], aggs, what="193 slots", batch_rows=20_000)
    assert m192["dense_block_launches"] == 0 and m193["dense_block_launches"] == 3
    assert m192["rows"] == m193["rows"] and len(m192["rows"]) == 192


def test_largest_layout_256_slots_of_eight_decimal_aggregates(gpu_ctx):
    rng = np.random.default_rng(607)
    n = 50_000
    d1 = [int(x) * (1 << 40) + int(y) for x, y in zip(rng.integers(-(1 << 50), 1 << 50, n), rng.integers(0, 1 << 40, n))]
    d2 = [int(x) for x in rng.integers(-10 ** 17, 10 ** 17, n)]
    cols = [(rng.integers(0, 255, n).astype(np.uint8), rng.random(n) > 0.01), dec_col(d1, 38, 2, rng.random(n) > 0.05), dec_col(d2, 20, 4)]
    types = [D.UINT8, D.decimal128(38, 2), D.decimal128(20, 4)]
    aggs = [(f, c) for c in (1, 2) for f in (D.AGG_SUM, D.AGG_MIN, D.AGG_MAX, D.AGG_AVG)]
    assert C.slot_words([(f, True) for f, _ in aggs]) == 34
    m = dense(gpu_ctx, cols, types, [0], [(0, 254)], aggs, what="256 x 34 words", batch_rows=20_000, device=True)
    assert m["num_groups"] == 256 and m["dense_block_launches"] == 3
    assert_rows(m["rows"], oracle_dense(cols, None, [0], nodes_of(aggs)), "256 x 34 words oracle")
