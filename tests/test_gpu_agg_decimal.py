"""MIN, MAX and AVG over Decimal128 in the hash group-by (dfgpu_agg), and Decimal128 SUM / MIN / MAX / AVG without GROUP BY.

Every result is compared exactly with tests/decimal_agg.py (MIN / MAX / AVG over decimals, DataFusion's DecimalAverager::avg) on top of
the oracle (groups, SUM, COUNT), keyed by the group tuple since the table's output order is unspecified.  The cases cover the
Decimal128 shapes (15,2) .. (38,38) with NULLs, FILTER clauses and all-NULL groups; i128::MIN / MAX, low words across bit 63, carries
and wrapping sums; AVG at its precision edge and past it (DFGPU_ERR_ARITH); growth by rehash, 128-bit keys and wide keys; Partial ->
PartialReduce -> Final / FinalPartitioned and skip-partial for MIN / MAX / SUM; the AVG Partial rejection; AggregateStream; the TPC-H
Q1 shape against the dense pipeline sink; and GpuAggregateExec in Single mode."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import decimal_agg as DA
import dense_cases as C
from decimal_util import col_as_py, gpu_col_as_py, gpu_host_col, gpu_nodes
from harness import split_points

pytestmark = pytest.mark.gpu
F = {D.AGG_SUM: O.A_SUM, D.AGG_COUNT: O.A_COUNT, D.AGG_MIN: O.A_MIN, D.AGG_MAX: O.A_MAX, D.AGG_AVG: O.A_AVG, D.AGG_COUNT_STAR: O.A_COUNT_STAR}
I128_MIN, I128_MAX = -(1 << 127), (1 << 127) - 1
TYPES = [(15, 2), (20, 0), (34, 10), (38, 4), (38, 38)]


def _slice(c, s, e):
    return (c[0][s:e], None if c[1] is None else np.asarray(c[1])[s:e])


def push(ctx, h, cols, types, batch_rows=None, device=False):
    keep = []
    if not len(cols[0][0]):
        return keep
    for s, e in split_points(len(cols[0][0]), batch_rows):
        hc = [gpu_host_col(D, _slice(c, s, e), t) for c, t in zip(cols, types)]
        if device:
            dc = [D.DeviceColumn.from_host(ctx, x) for x in hc]
            keep.append(dc)
            h.push_device(dc)
        else:
            h.push_host(hc)
    return keep


def drain_rows(h):
    rows, otypes = [], []
    for b in h.drain(host=True):
        cs = [gpu_col_as_py(D, b, i) for i in range(b.num_columns)]
        otypes = [t for _, t in cs]
        rows += list(zip(*[v for v, _ in cs]))
    return rows, otypes


def run_agg(ctx, cols, types, group_cols, aggs, mode=D.AGG_SINGLE, batch_rows=None, device=False, capacity_hint=0, skip=None):
    """dfgpu_agg -> (rows as tuples of Python values, output type codes, metrics)"""
    h = D.AggHandle(ctx, types, group_cols, aggs, mode, 8192, capacity_hint)
    if skip is not None:
        h.set_skip_partial(*skip)
    push(ctx, h, cols, types, batch_rows, device)
    h.finish()
    rows, otypes = drain_rows(h)
    m = {k: h.metric(k) for k in ("num_groups", "rehashes", "key_words", "skipped_aggregation_rows", "output_rows")}
    h.close()
    return rows, otypes, m


def reference(cols, group_cols, aggs):
    """{group tuple: aggregate values} from decimal_agg / the oracle; aggs as for dfgpu_agg: (func, arg_col, filter_col)"""
    ref = [(F[f], None if a < 0 else cols[a], None if fc < 0 else cols[fc]) for f, a, fc in aggs]
    if not group_cols:
        n = len(cols[0][0])
        res = DA.scalar_aggregate([(f, a, filt, n) for f, a, filt in ref])
        return {(): tuple(col_as_py(c)[0] for c in res)}
    keys, res = DA.group_by([cols[g] for g in group_cols], ref)
    out = list(keys)
    for (f, a, _), r in zip(ref, res):
        out += DA.agg_output_columns(f, r, None if a is None else (object if isinstance(a[0], O.Dec) else np.asarray(a[0]).dtype), False)
    rows = list(zip(*[col_as_py(c) for c in out])) if len(out[0][0]) else []
    nk = len(group_cols)
    return {r[:nk]: r[nk:] for r in rows}


def as_map(rows, nk):
    m = {r[:nk]: r[nk:] for r in rows}
    assert len(m) == len(rows), "a group was emitted twice"
    return m


def assert_same(got_rows, want, nk, what=""):
    got = as_map(got_rows, nk)
    assert len(got) == len(want), f"{what}: {len(got)} groups, expected {len(want)}"
    bad = [k for k in want if got.get(k) != want[k]]
    assert not bad, f"{what}: {len(bad)} groups differ, e.g. {bad[0]}: {got.get(bad[0])} != {want[bad[0]]}"


def dec_values(rng, n, p, s):
    """values of Decimal128(p, s) whose group sums * 10^(ts - s) stay inside i128 (dense_cases.avg_case's bound)"""
    m = min(10 ** p - 1, 10 ** (33 - C.avg_mul(p, s)))
    big = rng.integers(-10 ** 6, 10 ** 6, n)
    return [max(-m, min(m, int(b) * (m // 10 ** 6) + int(x))) for b, x in zip(big, rng.integers(-999, 1000, n))]


def general_case(rng, n, p, s, nkeys=40):
    """cols: 0 key Int64 in [0, nkeys] (NULL ~3 %; key nkeys has only NULL values), 1 Decimal128(p, s) with ~10 % NULL, 2 Boolean
    FILTER with NULLs"""
    key = rng.integers(0, nkeys + 1, n).astype(np.int64)
    kvalid = rng.random(n) > 0.03
    vvalid = (rng.random(n) > 0.1) & (key != nkeys)
    filt = (rng.random(n) > 0.4, rng.random(n) > 0.05)
    return [(key, kvalid), (O.Dec(dec_values(rng, n, p, s), p, s), vvalid), filt], [D.INT64, D.decimal128(p, s), D.BOOL]


GENERAL_AGGS = [(D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_AVG, 1, -1), (D.AGG_SUM, 1, -1), (D.AGG_COUNT, 1, -1),
                (D.AGG_MAX, 1, 2), (D.AGG_AVG, 1, 2), (D.AGG_COUNT_STAR, -1, -1)]


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("p,s", TYPES)
def test_min_max_avg_sum_over_decimal_types(gpu_ctx, p, s, device):
    rng = np.random.default_rng(100 + p + s)
    cols, types = general_case(rng, 20_000, p, s)
    got, ot, m = run_agg(gpu_ctx, cols, types, [0], GENERAL_AGGS, batch_rows=7000, device=device)
    want = reference(cols, [0], GENERAL_AGGS)
    assert_same(got, want, 1, f"decimal({p},{s})")
    tp, ts = min(38, p + 4), min(38, s + 4)
    assert ot == [D.INT64, D.decimal128(p, s), D.decimal128(p, s), D.decimal128(tp, ts), D.decimal128(min(38, p + 10), s), D.INT64,
                  D.decimal128(p, s), D.decimal128(tp, ts), D.INT64]
    allnull = as_map(got, 1)[(40,)]
    assert allnull[:4] == (None, None, None, None) and allnull[4] == 0 and allnull[7] > 0
    assert any(r[3] is not None and r[3] < 0 for r in got) and (None,) in want


def test_identity_values_and_bit63_pairs(gpu_ctx):
    """values equal to the MIN / MAX identities (i128::MAX / i128::MIN) are results, not NULLs, with and without NULLs in the input;
    pairs that differ only across bit 63 of the low word"""
    groups = {0: [I128_MAX], 1: [I128_MIN], 2: [I128_MAX, I128_MIN], 3: [(1 << 63) - 1, 1 << 63], 4: [-(1 << 64), -1],
              5: [(1 << 64) + (1 << 63), (1 << 64) + (1 << 63) - 1], 6: [-(1 << 63), -(1 << 63) - 1], 7: [0]}
    keys, vals = [], []
    for _ in range(50):
        for g, vs in groups.items():
            keys += [g] * len(vs); vals += vs
    aggs = [(D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_COUNT_STAR, -1, -1)]
    types = [D.INT32, D.decimal128(38, 0)]
    for nulls in (False, True):
        k = np.array(keys + ([8] * 3 if nulls else []), np.int32)
        v = vals + ([5] * 3 if nulls else [])
        valid = np.array([True] * len(vals) + [False] * 3) if nulls else None
        cols = [(k, None), (O.Dec(v, 38, 0), valid)]
        got, _, _ = run_agg(gpu_ctx, cols, types, [0], aggs, batch_rows=97)
        want = reference(cols, [0], aggs)
        assert_same(got, want, 1, f"identities nulls={nulls}")
        g = as_map(got, 1)
        assert g[(0,)][:2] == (I128_MAX, I128_MAX) and g[(1,)][:2] == (I128_MIN, I128_MIN) and g[(2,)][:2] == (I128_MIN, I128_MAX)
        assert g[(3,)][:2] == ((1 << 63) - 1, 1 << 63) and g[(4,)][:2] == (-(1 << 64), -1) and g[(6,)][:2] == (-(1 << 63) - 1, -(1 << 63))
        if nulls:
            assert g[(8,)] == (None, None, 3)


@pytest.mark.parametrize("n", [60_000, 1000])
def test_carries_and_wrapping_sums(gpu_ctx, n):
    """dense_cases.carry_case: sums that carry out of the low word in every group, and that wrap past +-2^127"""
    cols, types = C.carry_case(np.random.default_rng(31), n)
    aggs = [(D.AGG_SUM, 2, -1), (D.AGG_MIN, 2, -1), (D.AGG_MAX, 2, -1), (D.AGG_COUNT_STAR, -1, -1)]
    for gc in ([0], [0, 1]):
        got, _, m = run_agg(gpu_ctx, cols, types, gc, aggs, batch_rows=25_000)
        assert_same(got, reference(cols, gc, aggs), len(gc), f"carries {gc}")
        assert m["key_words"] == len(gc)          # two Int32 keys + two NULL flags: 66 bits


@pytest.mark.parametrize("p,s", [(15, 2), (20, 0), (34, 10), (36, 35), (38, 38)])
def test_avg_rule_of_dense_cases(gpu_ctx, p, s):
    cols, types = C.avg_case(np.random.default_rng(41 + p), p, s)
    aggs = [(D.AGG_AVG, 1, -1), (D.AGG_SUM, 1, -1), (D.AGG_COUNT, 1, -1), (D.AGG_COUNT_STAR, -1, -1)]
    got, ot, _ = run_agg(gpu_ctx, cols, types, [0], aggs, batch_rows=1500)
    assert_same(got, reference(cols, [0], aggs), 1, "avg")
    assert ot[1] == D.decimal128(min(38, p + 4), min(38, s + 4)) and any(r[1] is not None and r[1] < 0 for r in got)


@pytest.mark.parametrize("p,s,inside,outside", [(36, 35, 10 ** 35 - 1, 10 ** 35), (36, 35, -(10 ** 35 - 1), -(10 ** 35)),
                                                (38, 0, 10 ** 34 - 1, 10 ** 34), (38, 0, 10 ** 34 - 1, 10 ** 37)],
                         ids=["36_35", "36_35_negative", "38_0", "38_0_multiply_overflow"])
def test_avg_at_and_past_the_target_precision(gpu_ctx, p, s, inside, outside):
    """the value just inside the 38 digits is exact; just outside, or a sum whose * 10^(ts - s) overflows i128, is DFGPU_ERR_ARITH
    "Arithmetic Overflow in AvgAccumulator", grouped and without GROUP BY"""
    aggs = [(D.AGG_AVG, 1, -1), (D.AGG_COUNT_STAR, -1, -1)]
    types = [D.INT32, D.decimal128(p, s)]
    for v, ok in ((inside, True), (outside, False)):
        vals = [v, 0, 7] if v != 10 ** 37 else [v, v, 7]
        valid = np.array([True, False, False]) if v != 10 ** 37 else np.array([True, True, False])
        cols = [(np.zeros(3, np.int32), None), (O.Dec(vals, p, s), valid)]
        for gc in ([0], []):
            a = aggs if gc else [(f, ac - 1 if ac > 0 else ac, fc) for f, ac, fc in aggs]
            cc, tt = (cols, types) if gc else (cols[1:], types[1:])
            if ok:
                got, _, _ = run_agg(gpu_ctx, cc, tt, gc, a)
                assert got == [tuple([0] * len(gc)) + (v * 10 ** C.avg_mul(p, s), 3)]
            else:
                with pytest.raises(O.ArrowArithmeticOverflow):
                    reference(cc, gc, a)
                with pytest.raises(D.DfgpuError, match="Arithmetic Overflow in AvgAccumulator") as ei:
                    run_agg(gpu_ctx, cc, tt, gc, a)
                assert ei.value.code == -4


def test_growth_and_128_bit_keys(gpu_ctx):
    """more groups than the first table holds (rehashes > 0), one key column and two packed above 64 bits (key_words == 2)"""
    rng = np.random.default_rng(7)
    n = 400_000
    k1 = (rng.integers(0, 150_000, n) * 7919 - 10 ** 9).astype(np.int64)
    k2 = (rng.integers(0, 3, n).astype(np.int32), rng.random(n) > 0.01)
    v = (O.Dec(dec_values(rng, n, 15, 2), 15, 2), rng.random(n) > 0.05)
    cols, types = [(k1, None), k2, v], [D.INT64, D.INT32, D.decimal128(15, 2)]
    aggs = [(D.AGG_MIN, 2, -1), (D.AGG_MAX, 2, -1), (D.AGG_AVG, 2, -1), (D.AGG_SUM, 2, -1)]
    for gc, kw in (([0], 1), ([0, 1], 2)):
        got, _, m = run_agg(gpu_ctx, cols, types, gc, aggs, batch_rows=150_000)
        assert m["rehashes"] > 0 and m["key_words"] == kw and m["num_groups"] > 256
        assert_same(got, reference(cols, gc, aggs), len(gc), f"growth {gc}")


SPREAD = 10 ** 20 + 3   # Decimal128 keys of 90 bits


def test_wide_key_with_eight_pair_accumulators(gpu_ctx):
    """GROUP BY Decimal128 + Int32 (the wide-key path: hash tag + stored tuples), 4 MIN / MAX and 4 AVG over Decimal128 with NULLs
    (seen[] tracked), through growth: the rehash moves every 16-byte accumulator, the count and seen arrays and the stored key words"""
    rng = np.random.default_rng(8)
    n = 300_000
    x = rng.integers(-60_000, 60_000, n).astype(np.int64)
    dk = (O.Dec([int(v) * SPREAD for v in x], 38, 0), rng.random(n) > 0.01)
    ik = (rng.integers(0, 2, n).astype(np.int32), None)
    a = (O.Dec(dec_values(rng, n, 20, 0), 20, 0), rng.random(n) > 0.1)
    b = (O.Dec(dec_values(rng, n, 34, 10), 34, 10), rng.random(n) > 0.1)
    cols, types = [dk, ik, a, b], [D.decimal128(38, 0), D.INT32, D.decimal128(20, 0), D.decimal128(34, 10)]
    aggs = [(D.AGG_MIN, 2, -1), (D.AGG_MAX, 2, -1), (D.AGG_MIN, 3, -1), (D.AGG_MAX, 3, -1),
            (D.AGG_AVG, 2, -1), (D.AGG_AVG, 3, -1), (D.AGG_AVG, 2, -1), (D.AGG_AVG, 3, -1)]
    got, _, m = run_agg(gpu_ctx, cols, types, [0, 1], aggs, batch_rows=100_000)
    assert m["rehashes"] > 0 and m["num_groups"] > 100_000
    # the oracle groups by integers only: group by x, which the Decimal128 key is a bijection of, and map the keys back
    want = reference([(x, dk[1])] + cols[1:], [0, 1], aggs)
    assert_same(got, {(None if k0 is None else k0 * SPREAD, k1): v for (k0, k1), v in want.items()}, 2, "wide key")


def _state_cols(batches_rows, types):
    """state rows -> oracle-style columns of the given types"""
    cols = []
    for j, t in enumerate(types):
        vals = [r[j] for r in batches_rows]
        valid = np.array([x is not None for x in vals], bool)
        if D.type_base(t) == D.DECIMAL128:
            p, s = D.decimal_precision_scale(t)
            cols.append((O.Dec([0 if x is None else x for x in vals], p, s), None if valid.all() else valid))
        else:
            cols.append((np.array([0 if x is None else x for x in vals], np.int64), None if valid.all() else valid))
    return cols


MMS_AGGS = [(D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_SUM, 1, -1), (D.AGG_COUNT, 1, -1)]


@pytest.mark.parametrize("final_mode", [D.AGG_FINAL, D.AGG_FINAL_PARTITIONED])
def test_partial_reduce_final_for_min_max_sum(gpu_ctx, final_mode):
    """Partial states of MIN / MAX are the argument's type, SUM's Decimal128(p + 10, s); PartialReduce keeps them; Final merges"""
    rng = np.random.default_rng(9)
    cols, types = general_case(rng, 30_000, 20, 3, nkeys=3000)
    st_types = [D.INT64, D.decimal128(20, 3), D.decimal128(20, 3), D.decimal128(30, 3), D.INT64]
    parts = []
    for s, e in ((0, 12_000), (12_000, 30_000)):
        rows, ot, _ = run_agg(gpu_ctx, [_slice(c, s, e) for c in cols], types, [0], MMS_AGGS, mode=D.AGG_PARTIAL, batch_rows=5000)
        assert ot == st_types
        parts.append(rows)
    sagg = [(f, -1, -1) for f, _, _ in MMS_AGGS]
    reduced, ot, _ = run_agg(gpu_ctx, _state_cols(parts[0], st_types), st_types, [0], sagg, mode=D.AGG_PARTIAL_REDUCE)
    assert ot == st_types
    got, ot, _ = run_agg(gpu_ctx, _state_cols(reduced + parts[1], st_types), st_types, [0], sagg, mode=final_mode, batch_rows=4000)
    assert ot == st_types
    assert_same(got, reference(cols, [0], MMS_AGGS), 1, "partial -> final")


def test_skip_partial_passes_decimal_min_max_states_through(gpu_ctx):
    rng = np.random.default_rng(10)
    cols, types = general_case(rng, 40_000, 38, 4, nkeys=30_000)
    rows, ot, m = run_agg(gpu_ctx, cols, types, [0], MMS_AGGS, mode=D.AGG_PARTIAL, batch_rows=4000, skip=(5000, 0.1))
    assert m["skipped_aggregation_rows"] > 0
    st_types = [D.INT64, D.decimal128(38, 4), D.decimal128(38, 4), D.decimal128(38, 4), D.INT64]
    assert ot == st_types
    got, _, _ = run_agg(gpu_ctx, _state_cols(rows, st_types), st_types, [0], [(f, -1, -1) for f, _, _ in MMS_AGGS], mode=D.AGG_FINAL, batch_rows=20_000)
    assert_same(got, reference(cols, [0], MMS_AGGS), 1, "skip partial")


def test_avg_partial_and_final_are_rejected(gpu_ctx):
    """AVG(Decimal128) has no pinned Partial state: Partial, PartialReduce, Final and FinalPartitioned are DFGPU_ERR_UNSUPPORTED,
    grouped and without GROUP BY"""
    dec = D.decimal128(15, 2)
    for gc in ([0], []):
        with pytest.raises(D.DfgpuError) as ei:
            D.AggHandle(gpu_ctx, [D.INT64, dec], gc, [(D.AGG_AVG, 1, -1)], D.AGG_PARTIAL)
        assert ei.value.code == -3 and "Single modes only" in str(ei.value)
        for mode in (D.AGG_FINAL, D.AGG_FINAL_PARTITIONED, D.AGG_PARTIAL_REDUCE):
            st = [D.INT64, D.UINT64, dec] if gc else [D.UINT64, dec]
            with pytest.raises(D.DfgpuError) as ei:
                D.AggHandle(gpu_ctx, st, gc, [(D.AGG_AVG, -1, -1)], mode)
            assert ei.value.code == -3


@pytest.mark.parametrize("p,s", [(15, 2), (38, 4), (38, 38)])
def test_no_group_by(gpu_ctx, p, s):
    """AggregateStream: exactly one row, over data (several batches, NULLs, a FILTER) and over empty input (NULLs and COUNT 0)"""
    rng = np.random.default_rng(11 + p)
    cols, types = general_case(rng, 50_000, p, s)
    cols, types = cols[1:], types[1:]
    aggs = [(D.AGG_SUM, 0, -1), (D.AGG_MIN, 0, -1), (D.AGG_MAX, 0, -1), (D.AGG_AVG, 0, -1), (D.AGG_AVG, 0, 1), (D.AGG_COUNT, 0, -1)]
    for n in (50_000, 0):
        cc = [_slice(c, 0, n) for c in cols]
        got, ot, _ = run_agg(gpu_ctx, cc, types, [], aggs, batch_rows=12_000, device=n > 0)
        assert len(got) == 1 and got[0] == reference(cc, [], aggs)[()]
        assert ot[:4] == [D.decimal128(min(38, p + 10), s), D.decimal128(p, s), D.decimal128(p, s), D.decimal128(min(38, p + 4), min(38, s + 4))]
        if n == 0:
            assert got[0] == (None,) * 5 + (0,)
    # Partial -> Final without GROUP BY for SUM / MIN / MAX: the states carry the decimal types
    mms = [(D.AGG_SUM, 0, -1), (D.AGG_MIN, 0, -1), (D.AGG_MAX, 0, -1), (D.AGG_COUNT, 0, -1)]
    st_types = [D.decimal128(min(38, p + 10), s), D.decimal128(p, s), D.decimal128(p, s), D.INT64]
    states = []
    for s0, e0 in ((0, 20_000), (20_000, 50_000), (0, 0)):
        rows, ot, _ = run_agg(gpu_ctx, [_slice(c, s0, e0) for c in cols], types, [], mms, mode=D.AGG_PARTIAL)
        assert ot == st_types and len(rows) == 1
        states += rows
    got, _, _ = run_agg(gpu_ctx, _state_cols(states, st_types), st_types, [], [(f, -1, -1) for f, _, _ in mms], mode=D.AGG_FINAL)
    assert got == [reference(cols, [], mms)[()]]


def test_q1_shape_equals_the_dense_sink(gpu_ctx):
    """one seeded Q1-shaped input with Decimal128(15,2) money, 4 SUMs, 3 AVGs and COUNT(*): the fused dense sink and
    dfgpu_filter -> dfgpu_expr_evaluate_device -> dfgpu_agg give identical columns"""
    from test_gpu_pipe_dense import Q1_PRED, lineitem, q1_aggs, run_dense
    rng = np.random.default_rng(12)
    cols, types = lineitem(rng, 150_011, True, nulls=True)
    aggs = q1_aggs(True)
    dense, dtypes, _ = run_dense(gpu_ctx, cols, types, Q1_PRED, [0, 1], [(0, 2), (0, 1)], aggs, batch_rows=60_000)
    f = D.FilterHandle(gpu_ctx, types, gpu_nodes(D, Q1_PRED), None, 0, -1)
    push(gpu_ctx, f, cols, types, 60_000)
    f.finish()
    fo = f.drain(host=False)
    f.close()
    exprs = [nodes for _, nodes in aggs[2:4]]
    agg_cols = [3, 4, 7, 8, 3, 4, 5, -1]
    h = None
    for b in fo:
        fc = [b.column(i) for i in range(len(types))]
        ev = [D.evaluate_device(gpu_ctx, fc, b.num_rows, gpu_nodes(D, e)) for e in exprs]
        ec = [x.column(0) for x in ev]
        if h is None:
            h = D.AggHandle(gpu_ctx, [c.type for c in fc + ec], [0, 1], [(fn, c, -1) for (fn, _), c in zip(aggs, agg_cols)], D.AGG_SINGLE)
        h.push_device(fc + ec)
        for x in ev:
            x.release()
        b.release()
    h.finish()
    unfused, utypes = drain_rows(h)
    h.close()
    order = lambda r: tuple((1, 0) if v is None else (0, v) for v in r[:2])
    assert utypes == dtypes
    assert sorted(unfused, key=order) == dense and len(dense) >= 6


def test_exec_single_mode_decimal_aggregate_is_left_unfused_and_exact(gpu_ctx):
    """GpuAggregateExec(Single) over a Decimal128(15,2) column grouped by a high-cardinality key: no dense fusion (unknown bounds), and
    MIN / MAX / AVG / SUM equal the restatement"""
    import decimal
    import pyarrow as pa
    from datafusion_b200.exec import AggregateExpr, GpuAggregateExec, GpuPipelineExec, MemoryExec, TaskContext, collect, fuse_pipelines
    rng = np.random.default_rng(13)
    n = 60_000
    k = rng.integers(0, 20_000, n).astype(np.int64)
    vals = dec_values(rng, n, 15, 2)
    valid = rng.random(n) > 0.1
    arr = pa.array([decimal.Decimal(v).scaleb(-2) if ok else None for v, ok in zip(vals, valid)], pa.decimal128(15, 2))
    t = pa.table({"k": pa.array(k), "m": arr})
    exprs = [AggregateExpr("min", "m", "mn"), AggregateExpr("max", "m", "mx"), AggregateExpr("avg", "m", "av"), AggregateExpr("sum", "m", "sm")]
    plan = GpuAggregateExec("Single", ["k"], exprs, MemoryExec(t.to_batches(max_chunksize=16_384), t.schema))
    assert not isinstance(fuse_pipelines(plan), GpuPipelineExec)
    assert [f.type for f in plan.schema][1:] == [pa.decimal128(15, 2), pa.decimal128(15, 2), pa.decimal128(19, 6), pa.decimal128(25, 2)]
    out = pa.Table.from_batches(collect(plan, TaskContext(ctx=gpu_ctx)), schema=plan.schema)
    scales = [2, 2, 6, 2]
    got = {}
    for row in zip(*[out.column(i).to_pylist() for i in range(5)]):
        got[(row[0],)] = tuple(None if x is None else int(x.scaleb(sc)) for x, sc in zip(row[1:], scales))
    cols = [(k, None), (O.Dec(vals, 15, 2), valid)]
    want = reference(cols, [0], [(D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_AVG, 1, -1), (D.AGG_SUM, 1, -1)])
    assert got == want and len(got) > 10_000
