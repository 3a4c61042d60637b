"""The stand-alone hash join (dfgpu_hashjoin) and hash group-by (dfgpu_agg) over every column type the C ABI accepts, fed as sliced
Arrow batches whose buffers start at bit offsets 0, 3 and 37.  The references are plain Python / numpy and share no code with the kernels:

- join: each key tuple is encoded by its components' value bytes (floats by their bits, Decimal128 by its 16 bytes, NULL stays NULL);
  the oracle joins those codes, so it supplies only the join-type semantics, and every output column is gathered with numpy from the
  original typed arrays;
- group-by: a dict keyed by the group tuple (-0.0 folded into +0.0, NaN kept by its bits, NULL its own group), integer SUMs as Python
  ints wrapped to the result width, float SUM / AVG within the math.fsum error bound, float MIN / MAX bit for bit in totalOrder."""
import math

import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import dense_cases as DC
import float_order as FO
from test_oracle_golden import JT, out_mapping

pytestmark = pytest.mark.gpu

DEC = D.decimal128(38, 0)
PADS = (0, 3, 37)
PA_TYPE = {D.BOOL: pa.bool_(), D.INT8: pa.int8(), D.INT16: pa.int16(), D.INT32: pa.int32(), D.INT64: pa.int64(), D.UINT8: pa.uint8(),
           D.UINT16: pa.uint16(), D.UINT32: pa.uint32(), D.UINT64: pa.uint64(), D.FLOAT32: pa.float32(), D.FLOAT64: pa.float64(),
           D.DATE32: pa.date32(), D.DATE64: pa.date64(), D.TIMESTAMP: pa.timestamp("us"), DEC: pa.decimal128(38, 0)}
NAME = {D.BOOL: "Boolean", D.INT8: "Int8", D.INT16: "Int16", D.INT32: "Int32", D.INT64: "Int64", D.UINT8: "UInt8", D.UINT16: "UInt16",
        D.UINT32: "UInt32", D.UINT64: "UInt64", D.FLOAT32: "Float32", D.FLOAT64: "Float64", D.DATE32: "Date32", D.DATE64: "Date64",
        D.TIMESTAMP: "Timestamp", DEC: "Decimal128"}
INTS = [D.INT8, D.INT16, D.INT32, D.INT64, D.UINT8, D.UINT16, D.UINT32, D.UINT64]
ALL = INTS + [D.FLOAT32, D.FLOAT64, D.DATE32, D.DATE64, D.TIMESTAMP, D.BOOL, DEC]
GJT = {"Inner": D.JOIN_INNER, "Left": D.JOIN_LEFT, "Right": D.JOIN_RIGHT, "Full": D.JOIN_FULL, "LeftSemi": D.JOIN_LEFT_SEMI,
       "RightSemi": D.JOIN_RIGHT_SEMI, "LeftAnti": D.JOIN_LEFT_ANTI, "RightAnti": D.JOIN_RIGHT_ANTI, "LeftMark": D.JOIN_LEFT_MARK,
       "RightMark": D.JOIN_RIGHT_MARK}
ORDERED = {"Inner", "RightSemi", "RightAnti", "RightMark"}
PHJ_ON, PHJ_OFF = (819200, 0.0), (0, float("inf"))


def npt(t):
    return object if t == DEC else (np.bool_ if t == D.BOOL else D.NP_OF_TYPE[t])


def f64(*bits):
    return list(np.array(bits, np.uint64).view(np.float64))


def f32(*bits):
    return list(np.array(bits, np.uint32).view(np.float32))


def pool(t):
    """the distinct values of a key column of type t: the type's extremes, 0, -1 / all ones, and for floats +-0, +-inf and NaNs of
    several payloads and both signs"""
    if t == D.BOOL:
        return [True, False]
    if t == DEC:
        m = 10 ** 38 - 1
        return [0, 1, -1, m, -m, 1 << 64, -(1 << 64), (1 << 63), -(1 << 63) - 1, 12345678901234567890123]
    if t == D.FLOAT64:
        return [0.0, -0.0, math.inf, -math.inf, 1.5, -2.25, 5e-324, 1.7976931348623157e308] + \
            f64(0x7FF8000000000000, 0x7FF8000000000123, 0xFFF8000000000000, 0xFFFC000000000001)
    if t == D.FLOAT32:
        return [0.0, -0.0, math.inf, -math.inf, 1.5, -2.25] + f32(0x00000001, 0x7F7FFFFF, 0x7FC00000, 0x7FC00123, 0xFFC00000, 0xFFE00001)
    info = np.iinfo(npt(t))
    lo, hi = int(info.min), int(info.max)
    vals = {lo, hi, 0, 1, lo + 1, hi - 1, (lo + hi) // 2, hi // 3}
    vals.add(-1 if lo < 0 else hi)              # all ones
    if t == D.UINT64:
        vals |= {1 << 63, (1 << 63) + 12345, (1 << 64) - 2}
    return sorted(vals)


def window(t, high):
    """about 200 consecutive values at the top or bottom of an integer domain: the ArrayMap's range arithmetic at the domain's edges"""
    info = np.iinfo(npt(t))
    return list(range(int(info.max) - 199, int(info.max) + 1)) if high else list(range(int(info.min), int(info.min) + 200))


def arr(vals, t):
    return np.array(vals, dtype=npt(t))


def draw(rng, vals, t, n, null_frac):
    v = arr(vals, t)[rng.integers(0, len(vals), n)]
    ok = None if null_frac == 0 else rng.random(n) >= null_frac
    return v, ok


def filler(rng, t, n, null_frac=0.0):
    """a payload column: random values of the full domain plus the pool's edges"""
    if t in (D.BOOL, DEC, D.FLOAT32, D.FLOAT64):
        return draw(rng, pool(t), t, n, null_frac)
    info = np.iinfo(npt(t))
    v = rng.integers(int(info.min), int(info.max), n, dtype=np.int64 if t != D.UINT64 else np.uint64, endpoint=True).astype(npt(t))
    p = arr(pool(t), t)
    v[:len(p)] = p
    return v, (None if null_frac == 0 else rng.random(n) >= null_frac)


# ---- Arrow input -----------------------------------------------------------------------------------------------------------------
def arrow_col(v, ok, t, pad):
    """an Arrow array of type t whose values and validity start `pad` elements (bits) into their buffers"""
    n = len(v)
    if t == D.BOOL:
        vals = D.pack_bits(np.concatenate([np.zeros(pad, bool), np.asarray(v, bool)]))
    elif t == DEC:
        w = v if (v.dtype == np.uint64 and v.ndim == 2) else D.decimal_to_words([int(x) for x in v])   # words: a drained output
        vals = np.concatenate([np.zeros((pad, 2), np.uint64), w]).reshape(-1)
    else:
        vals = np.concatenate([np.zeros(pad, npt(t)), np.asarray(v, npt(t))])
    validity = None if ok is None else pa.py_buffer(D.pack_bits(np.concatenate([np.ones(pad, bool), np.asarray(ok, bool)])))
    nulls = 0 if ok is None else int(n - np.count_nonzero(ok))
    a = pa.Array.from_buffers(PA_TYPE[t], n + pad, [validity, pa.py_buffer(np.ascontiguousarray(vals))], null_count=nulls)
    return a.slice(pad, n)


def push_arrow(push, cols, types, bounds, pad_start=0):
    for i, (s, e) in enumerate(bounds):
        pad = PADS[(i + pad_start) % len(PADS)]
        arrays = [arrow_col(v[s:e], None if ok is None else ok[s:e], t, pad) for (v, ok), t in zip(cols, types)]
        push(pa.RecordBatch.from_arrays(arrays, names=[f"c{i}" for i in range(len(arrays))]))


def splits(n, k):
    cut = sorted(set([0, n] + [n * i // k + (i % 3) for i in range(1, k)]))
    return list(zip(cut[:-1], cut[1:]))


def drain(h):
    """-> (output columns [(values, valid bool array)], output type codes); Decimal128 values as [n, 2] uint64 words"""
    outs = h.drain(host=True)
    if not outs:
        return None, None
    types = [outs[0].column(i).type for i in range(outs[0].num_columns)]
    cols = []
    for c in range(len(types)):
        parts = [b.column_numpy(c) for b in outs]
        v = np.concatenate([p[0] for p in parts])
        ok = np.concatenate([np.ones(len(p[0]), bool) if p[1] is None else p[1] for p in parts])
        cols.append((v, ok))
    return cols, types


# ---- comparison ------------------------------------------------------------------------------------------------------------------
def words(v, ok, t):
    """one column -> [n, k] uint64: validity, then the value's bits (floats by their bits, zero where NULL)"""
    n = len(v)
    ok = np.ones(n, bool) if ok is None else np.asarray(ok, bool)
    if t == DEC:
        w = np.asarray(v, np.uint64).reshape(n, 2) if (isinstance(v, np.ndarray) and v.dtype == np.uint64) else \
            D.decimal_to_words([int(x) for x in v]).reshape(n, 2)
    elif t == D.BOOL:
        w = np.asarray(v, bool).astype(np.uint64)[:, None]
    else:
        a = np.ascontiguousarray(np.asarray(v, npt(t)))
        w = a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]).astype(np.uint64)[:, None]
    w = np.where(ok[:, None], w, np.uint64(0))
    return np.concatenate([ok.astype(np.uint64)[:, None], w], axis=1)


def assert_rows_equal(got, gtypes, exp, etypes, ordered, what):
    assert gtypes == etypes, f"{what}: output types {[NAME.get(t, t) for t in gtypes]} != {[NAME.get(t, t) for t in etypes]}"
    g = np.concatenate([words(v, ok, t) for (v, ok), t in zip(got, gtypes)], axis=1)
    e = np.concatenate([words(v, ok, t) for (v, ok), t in zip(exp, etypes)], axis=1)
    assert g.shape == e.shape, f"{what}: {g.shape[0]} rows, expected {e.shape[0]}"
    if not ordered and len(g):
        g, e = g[np.lexsort(g.T[::-1])], e[np.lexsort(e.T[::-1])]
    bad = np.nonzero((g != e).any(axis=1))[0]
    assert not len(bad), f"{what}: {len(bad)} rows differ, first at {bad[0]}: got {g[bad[0]].tolist()} expected {e[bad[0]].tolist()}"


# ---- join --------------------------------------------------------------------------------------------------------------------------
def value_bytes(v, t):
    if t == DEC:
        return [bytes(r) for r in D.decimal_to_words([int(x) for x in v]).view(np.uint8).reshape(len(v), 16)]
    a = np.ascontiguousarray(np.asarray(v, npt(t)))
    if t == D.BOOL:
        a = a.astype(np.uint8)
    return [bytes(r) for r in a.view(np.uint8).reshape(len(v), a.dtype.itemsize)]


def key_codes(build, probe, on_b, on_p, bt, pt):
    """one int64 code per distinct key tuple (its components' value bytes), NULL when any component is NULL"""
    codes = {}
    out = []
    for cols, on, types in ((build, on_b, bt), (probe, on_p, pt)):
        n = len(cols[0][0])
        comps = [value_bytes(cols[c][0], types[c]) for c in on]
        ok = np.ones(n, bool)
        for c in on:
            if cols[c][1] is not None:
                ok &= np.asarray(cols[c][1], bool)
        code = np.array([codes.setdefault(tuple(x[i] for x in comps), len(codes)) for i in range(n)], np.int64)
        out.append((code, None if ok.all() else ok))
    return out


def take(col, t, idx):
    v, ok = col
    safe = np.where(idx >= 0, idx, 0)
    out = np.asarray(v)[safe] if len(v) else np.zeros(len(idx), npt(t))
    valid = idx >= 0
    if ok is not None and len(v):
        valid &= np.asarray(ok, bool)[safe]
    return out, valid


def join_reference(build, probe, on_b, on_p, bt, pt, side, index, jt, nen=False, probe_batch_rows=None):
    bc, pc = key_codes(build, probe, on_b, on_p, bt, pt)
    b, p, m, _ = O.hash_join_indices([bc], [pc], join_type=JT[jt], null_equals_null=nen, phj_threshold=0, phj_density=float("inf"),
                                     probe_batch_rows=probe_batch_rows)
    cols, types = [], []
    for s, ix in zip(side, index):
        if s == 2:
            cols.append((m, None)); types.append(D.BOOL)
        elif s == 0:
            cols.append(take(build[ix], bt[ix], b)); types.append(bt[ix])
        else:
            cols.append(take(probe[ix], pt[ix], p)); types.append(pt[ix])
    return cols, types


def run_join(ctx, build, probe, on_b, on_p, bt, pt, side, index, jt="Inner", nen=False, phj=PHJ_OFF, build_parts=2, probe_parts=3):
    """-> (columns, types, handle metrics) with the build pushed in `build_parts` and the probe in `probe_parts` Arrow batches"""
    h = D.HashJoinHandle(ctx, bt, pt, on_b, on_p, side, index, GJT[jt], D.NULL_EQUALS_NULL if nen else D.NULL_EQUALS_NOTHING, 8192,
                         phj[0], phj[1])
    try:
        push_arrow(h.push_build_arrow, build, bt, splits(len(build[0][0]), build_parts))
        h.finish_build()
        outs_types, chunks = None, []
        pb = splits(len(probe[0][0]), probe_parts)
        for i, b in enumerate(pb):
            push_arrow(h.push_probe_arrow, probe, pt, [b], pad_start=i + 1)
            c, ty = drain(h)
            if c is not None:
                chunks.append(c); outs_types = ty
        h.finish_probe()
        c, ty = drain(h)
        if c is not None:
            chunks.append(c); outs_types = ty
        metrics = {k: h.metric(k) for k in ("array_map_created_count", "inline_payload_words", "build_distinct_keys")}
    finally:
        h.close()
    if not chunks:
        return None, None, metrics, [e - s for s, e in pb]
    cols = [(np.concatenate([ch[c][0] for ch in chunks]), np.concatenate([ch[c][1] for ch in chunks])) for c in range(len(outs_types))]
    return cols, outs_types, metrics, [e - s for s, e in pb]


def check_join(ctx, build, probe, on_b, on_p, bt, pt, side, index, jt="Inner", nen=False, phj=PHJ_OFF, what=""):
    got, gtypes, metrics, pbr = run_join(ctx, build, probe, on_b, on_p, bt, pt, side, index, jt, nen, phj)
    exp, etypes = join_reference(build, probe, on_b, on_p, bt, pt, side, index, jt, nen, pbr)
    if got is None:
        assert len(exp[0][0]) == 0, f"{what}: no output, expected {len(exp[0][0])} rows"
    else:
        assert_rows_equal(got, gtypes, exp, etypes, jt in ORDERED, f"{what} {jt}")
    return metrics, exp


def array_map_expected(keys, t, phj):
    """the ArrayMap rule (try_create_array_map): an integer (not date / time) single key whose non-NULL build values span at most 2^31
    values; with density 0 every such span qualifies"""
    if phj != PHJ_ON or t not in INTS:
        return 0
    v, ok = keys
    v = np.asarray(v)[np.ones(len(v), bool) if ok is None else np.asarray(ok, bool)]
    if not len(v):
        return 0
    lo, hi = int(v.min()), int(v.max())
    return 1 if hi - lo + 1 <= (1 << 31) else 0


def key_tables(rng, types, nb, npr, pools=None, null_frac=0.1):
    """build / probe tables: the key columns `types` drawn from their pools (duplicates, misses), a build row id and a probe row id"""
    pools = pools or [pool(t) for t in types]
    build, probe = [], []
    for t, p in zip(types, pools):
        hit = p[: max(1, (3 * len(p)) // 4)]   # the probe side also sees values the build side never has
        build.append(draw(rng, hit, t, nb, null_frac))
        probe.append(draw(rng, p, t, npr, null_frac))
    build.append((np.arange(nb, dtype=np.int32), None)); probe.append((np.arange(npr, dtype=np.int64), None))
    return build, probe, list(types) + [D.INT32], list(types) + [D.INT64]


@pytest.mark.parametrize("t", ALL, ids=[NAME[t] for t in ALL])
def test_join_single_key_of_every_type(gpu_ctx, t):
    rng = np.random.default_rng(100 + t)
    datasets = [("edges", None)]
    if t in INTS:
        datasets += [("low", [window(t, False)]), ("high", [window(t, True)])]
    for name, pools in datasets:
        build, probe, bt, pt = key_tables(rng, [t], 1001, 3001, pools)
        side, index = [0, 0, 1, 1], [0, 1, 0, 1]
        for phj in ((PHJ_ON, PHJ_OFF) if t in INTS else (PHJ_OFF,)):
            metrics, exp = check_join(gpu_ctx, build, probe, [0], [0], bt, pt, side, index, phj=phj, what=f"{NAME[t]} {name} phj={phj}")
            assert metrics["array_map_created_count"] == array_map_expected(build[0], t, phj), f"{NAME[t]} {name} phj={phj}"
            assert len(exp[0][0]) > 1000
    if t in (D.INT8, D.UINT8, D.INT16, D.UINT16):   # a narrow domain always takes the ArrayMap when the settings allow it
        assert array_map_expected(build[0], t, PHJ_ON) == 1


def test_join_unique_all_ones_and_extreme_keys_in_the_array_map(gpu_ctx):
    """unique build keys (the inline table, or the ArrayMap) holding -1 / all ones and the domain's extremes"""
    for t in INTS:
        p = pool(t)
        build = [(arr(p, t), None), (np.arange(len(p), dtype=np.int32), None)]
        pv = arr(p * 3, t)
        probe = [(pv, np.arange(len(pv)) % 7 != 3), (np.arange(len(pv), dtype=np.int64), None)]
        for phj in (PHJ_ON, PHJ_OFF):
            metrics, exp = check_join(gpu_ctx, build, probe, [0], [0], [t, D.INT32], [t, D.INT64], [0, 0, 1, 1], [0, 1, 0, 1], phj=phj,
                                      what=f"{NAME[t]} unique phj={phj}")
            assert metrics["array_map_created_count"] == array_map_expected(build[0], t, phj)


MULTI = [(D.FLOAT32, D.FLOAT32), (D.FLOAT64, D.INT8), (D.FLOAT64, D.FLOAT64), (D.FLOAT64, D.INT64), (D.UINT32, D.INT16), (D.BOOL, D.INT32),
         (D.FLOAT32, D.INT16, D.UINT8), (D.FLOAT64, D.FLOAT32, D.INT8), (DEC, D.FLOAT64), (D.UINT64, D.FLOAT32)]


@pytest.mark.parametrize("types", MULTI, ids=["-".join(NAME[t] for t in m) for m in MULTI])
def test_join_multi_column_keys_on_both_key_paths(gpu_ctx, types):
    """the same float and integer data through the exact 64-bit tag (<= 64 key bits) and the wide-key path (more bits, Boolean or
    Decimal128): both must equal the bitwise reference, so -0.0 never joins +0.0 and a NaN joins only a NaN with the same bits"""
    rng = np.random.default_rng(sum(types) * 7)
    pools = [pool(t)[:6] if t in INTS else pool(t) for t in types]   # small pools: every tuple repeats
    build, probe, bt, pt = key_tables(rng, types, 1500, 2901, pools, null_frac=0.05)
    nk = len(types)
    side, index = [0] * (nk + 1) + [1] * (nk + 1), list(range(nk + 1)) * 2
    _, exp = check_join(gpu_ctx, build, probe, list(range(nk)), list(range(nk)), bt, pt, side, index, what="-".join(NAME[t] for t in types))
    assert len(exp[0][0]) > 0


def test_join_signed_zero_and_nan_payloads_on_a_wide_key(gpu_ctx):
    """(Float64, Int64) keys take the wide-key path; the single Float64 key the exact tag.  Both keep -0.0 and +0.0 apart, and NaNs
    match by their bits, as create_hashes does by hashing a float's bits"""
    keys = [0.0, -0.0] + f64(0x7FF8000000000000, 0x7FF8000000000123, 0xFFF8000000000000)
    bk = np.array(keys, np.float64); pk = np.array(keys[::-1] * 2, np.float64)
    build = [(bk, None), (np.full(len(bk), 7, np.int64), None), (np.arange(len(bk), dtype=np.int32), None)]
    probe = [(pk, None), (np.full(len(pk), 7, np.int64), None), (np.arange(len(pk), dtype=np.int64), None)]
    bt, pt = [D.FLOAT64, D.INT64, D.INT32], [D.FLOAT64, D.INT64, D.INT64]
    for on in ([0], [0, 1]):
        _, exp = check_join(gpu_ctx, build, probe, on, on, bt, pt, [0, 0, 1, 1], [0, 2, 0, 2], what=f"keys {on}")
        assert len(exp[0][0]) == len(pk)     # every probe row meets exactly its own bit pattern


PAYLOADS = {
    "inline64": [D.INT32, D.INT16, D.UINT8, D.INT8],                      # 64 bits: packed beside the key
    "gather72": [D.INT64, D.INT8],                                         # 72 bits: gathered after the probe
    "narrow": [D.UINT16, D.UINT32, D.FLOAT32, D.DATE32],                   # 96 bits
    "wide": [D.UINT64, D.FLOAT64, D.DATE64, D.TIMESTAMP],
    "bool_dec": [D.BOOL, DEC, D.INT8],
}


@pytest.mark.parametrize("nulls", [False, True], ids=["valid", "nullable"])
@pytest.mark.parametrize("name", list(PAYLOADS))
def test_join_payload_columns_of_every_type(gpu_ctx, name, nulls):
    """unique Int64 build keys with payloads of every width on both sides; the inline table carries the build payload only when its
    widths sum to at most 64 bits and no column is Boolean, nullable or 16 bytes wide"""
    rng = np.random.default_rng(len(name) * 31 + nulls)
    nb, npr = 2001, 5003
    bk = (rng.permutation(10_000)[:nb].astype(np.int64) * 1_000_003) - 5_000_000_000
    pk = bk[rng.integers(0, nb, npr)]
    pk[::5] += 1                                                               # misses
    pt_types = PAYLOADS[name]
    build = [(bk, None)] + [filler(rng, t, nb, 0.1 if nulls else 0.0) for t in pt_types]
    probe = [(pk, None)] + [filler(rng, t, npr, 0.1 if nulls else 0.0) for t in pt_types[::-1]]
    bt, pt = [D.INT64] + pt_types, [D.INT64] + pt_types[::-1]
    k = len(pt_types)
    side, index = [0] * (k + 1) + [1] * (k + 1), list(range(k + 1)) * 2
    metrics, exp = check_join(gpu_ctx, build, probe, [0], [0], bt, pt, side, index, what=f"payload {name} nulls={nulls}")
    bits = sum(8 * D.WIDTH[t] for t in pt_types)
    inline = not nulls and bits <= 64 and D.BOOL not in pt_types and DEC not in pt_types
    assert metrics["inline_payload_words"] == (2 if inline else 0), (name, nulls, metrics)
    assert (name == "inline64" and not nulls) == inline
    assert len(exp[0][0]) > npr // 2


def test_join_date32_build_key_emitted_from_an_int32_probe_key(gpu_ctx):
    """a build key column is read from the probe key of the same width; its output keeps the build side's type"""
    rng = np.random.default_rng(3)
    bk = rng.permutation(50_000)[:3001].astype(np.int32) - 20_000
    pk = bk[rng.integers(0, len(bk), 7001)]
    pk[::9] = 2**31 - 1
    build = [(bk, None), filler(rng, D.INT16, len(bk))]
    probe = [(pk, None), filler(rng, D.UINT8, len(pk))]
    for bt, pt in (([D.DATE32, D.INT16], [D.INT32, D.UINT8]), ([D.INT32, D.INT16], [D.DATE32, D.UINT8])):
        metrics, _ = check_join(gpu_ctx, build, probe, [0], [0], bt, pt, [0, 0, 1, 1], [0, 1, 0, 1], what=f"{NAME[bt[0]]} / {NAME[pt[0]]}")
        assert metrics["inline_payload_words"] == 2 and metrics["array_map_created_count"] == 0


@pytest.mark.parametrize("jt", list(GJT))
@pytest.mark.parametrize("kt", [D.INT8, D.FLOAT64], ids=["Int8", "Float64"])
def test_join_every_type_with_boolean_and_decimal_payloads(gpu_ctx, kt, jt):
    """Left / Right / Full padding and the Mark column over bit-packed and 16-byte output columns"""
    rng = np.random.default_rng(kt * 100 + GJT[jt])
    build, probe, bt, pt = key_tables(rng, [kt], 777, 2345, null_frac=0.08)
    for cols, types, n in ((build, bt, 777), (probe, pt, 2345)):
        cols += [filler(rng, D.BOOL, n, 0.2), filler(rng, DEC, n, 0.2), filler(rng, D.BOOL, n)]
        types += [D.BOOL, DEC, D.BOOL]
    side, index = out_mapping(jt, len(bt), len(pt))
    for phj in ((PHJ_ON, PHJ_OFF) if kt == D.INT8 else (PHJ_OFF,)):
        check_join(gpu_ctx, build, probe, [0], [0], bt, pt, side, index, jt, phj=phj, what=f"{NAME[kt]} phj={phj}")


@pytest.mark.parametrize("kt", [D.FLOAT64, D.BOOL], ids=["Float64", "Boolean"])
def test_join_null_equals_null_on_float_and_boolean_keys(gpu_ctx, kt):
    rng = np.random.default_rng(kt)
    build, probe, bt, pt = key_tables(rng, [kt], 301, 1203, null_frac=0.2)
    build.append(filler(rng, D.BOOL, 301, 0.3)); bt.append(D.BOOL)
    for jt in ("Inner", "Left", "Full", "RightSemi", "RightAnti", "LeftMark"):
        side, index = out_mapping(jt, len(bt), len(pt))
        check_join(gpu_ctx, build, probe, [0], [0], bt, pt, side, index, jt, nen=True, what=f"{NAME[kt]} NullEqualsNull")


def test_join_refuses_key_types_that_differ_between_sides(gpu_ctx):
    for b, p in ((D.INT32, D.UINT32), (D.INT32, D.FLOAT32), (D.UINT64, D.FLOAT64), (D.INT64, D.UINT64), (D.decimal128(38, 0), D.decimal128(38, 2)),
                 (D.decimal128(20, 0), D.decimal128(38, 0))):
        with pytest.raises(D.DfgpuError) as e:
            D.HashJoinHandle(gpu_ctx, [b, D.INT64], [p, D.INT64], [0], [0], [0, 1], [1, 1])
        assert e.value.code == -1, (b, p)     # DFGPU_ERR_INVALID


# ---- group-by ----------------------------------------------------------------------------------------------------------------------
SIGNED_RESULT = {t: D.INT64 for t in (D.INT8, D.INT16, D.INT32, D.INT64)}
UNSIGNED = (D.UINT8, D.UINT16, D.UINT32, D.UINT64)


def group_value(v, t):
    """a group key component as the reference's group values compare it: -0.0 folded into +0.0, NaN by its bits"""
    if t == D.FLOAT64:
        b = int(np.float64(v).view(np.uint64))
        return 0 if b == 1 << 63 else b
    if t == D.FLOAT32:
        b = int(np.float32(v).view(np.uint32))
        return 0 if b == 1 << 31 else b
    if t == D.BOOL:
        return bool(v)
    return int(v)


def out_group_values(col, t):
    v, ok = col
    if t == DEC:
        v = D.words_to_decimal(v)
    return [group_value(v[i], t) if ok[i] else None for i in range(len(ok))]


def agg_result_type(func, t):
    if func in (D.AGG_COUNT, D.AGG_COUNT_STAR):
        return D.INT64
    if func == D.AGG_AVG:
        return D.FLOAT64
    if func == D.AGG_SUM:
        return D.FLOAT64 if t in (D.FLOAT32, D.FLOAT64) else (D.UINT64 if t in UNSIGNED else D.INT64)
    return t


def agg_reference(cols, types, group_cols, aggs):
    """{group tuple: [cell per aggregate]}: exact ints, Approx for float SUM / AVG, the chosen input value for MIN / MAX"""
    n = len(cols[0][0])
    gvals = [[group_value(cols[g][0][i], types[g]) if (cols[g][1] is None or cols[g][1][i]) else None for i in range(n)] for g in group_cols]
    rows = {}
    for i in range(n):
        rows.setdefault(tuple(gv[i] for gv in gvals), []).append(i)
    ref = {}
    for key, idx in rows.items():
        cells = []
        for func, a, f in aggs:
            sel = [i for i in idx if f < 0 or ((cols[f][1] is None or cols[f][1][i]) and cols[f][0][i])]
            if func == D.AGG_COUNT_STAR:
                cells.append(len(sel)); continue
            v, ok = cols[a]
            xs = [v[i] for i in sel if ok is None or ok[i]]
            t = types[a]
            if func == D.AGG_COUNT:
                cells.append(len(xs))
            elif not xs:
                cells.append(None)
            elif func == D.AGG_SUM and t in (D.FLOAT32, D.FLOAT64):
                cells.append(DC._fsum_cells([float(x) for x in xs], False))
            elif func == D.AGG_SUM:
                s = sum(int(x) for x in xs) % (1 << 64)
                cells.append(s if t in UNSIGNED else (s - (1 << 64) if s >= 1 << 63 else s))
            elif func == D.AGG_AVG:
                cells.append(DC._fsum_cells([float(x) for x in xs], True))
            elif t in (D.FLOAT32, D.FLOAT64):
                k = FO.order_key(np.array(xs, npt(t)))
                cells.append(xs[int(np.argmin(k) if func == D.AGG_MIN else np.argmax(k))])
            else:
                cells.append(min(int(x) for x in xs) if func == D.AGG_MIN else max(int(x) for x in xs))
        ref[key] = cells
    return ref


def check_agg(out, otypes, ref, types, group_cols, aggs, what):
    ng = len(group_cols)
    want_types = [types[g] for g in group_cols] + [agg_result_type(f, types[a] if a >= 0 else D.INT64) for f, a, _ in aggs]
    assert otypes == want_types, f"{what}: output types {[NAME.get(t, t) for t in otypes]} != {[NAME.get(t, t) for t in want_types]}"
    keys = list(zip(*[out_group_values(out[c], types[g]) for c, g in enumerate(group_cols)]))
    assert len(keys) == len(set(keys)), f"{what}: a group is emitted twice"
    assert set(keys) == set(ref), f"{what}: groups differ: {sorted(set(keys) ^ set(ref), key=repr)[:6]}"
    for r, key in enumerate(keys):
        for j, (func, a, _) in enumerate(aggs):
            v, ok = out[ng + j]
            exp, w = ref[key][j], f"{what} group {key} agg {j} ({func})"
            if exp is None:
                assert not ok[r], f"{w}: {v[r]!r}, expected NULL"
                continue
            assert ok[r], f"{w}: NULL, expected {exp!r}"
            if isinstance(exp, DC.Approx):
                assert abs(float(v[r]) - exp.exact) <= exp.tol, f"{w}: {v[r]!r} != {exp!r}"
            elif otypes[ng + j] in (D.FLOAT32, D.FLOAT64):
                dt = npt(otypes[ng + j])
                assert FO.bits(v[r], dt) == FO.bits(exp, dt), f"{w}: {v[r]!r} ({hex(FO.bits(v[r], dt))}), expected {exp!r} ({hex(FO.bits(exp, dt))})"
            else:
                assert int(v[r]) == int(exp), f"{w}: {int(v[r])}, expected {int(exp)}"


def run_agg(ctx, cols, types, group_cols, aggs, mode, parts=3):
    h = D.AggHandle(ctx, types, group_cols, aggs, mode, 8192)
    try:
        push_arrow(h.push_arrow, cols, types, splits(len(cols[0][0]), parts))
        h.finish()
        out, otypes = drain(h)
        kw = h.metric("key_words")
    finally:
        h.close()
    return out, otypes, kw


def run_agg_modes(ctx, cols, types, group_cols, aggs, what):
    """Single, SinglePartitioned, and Partial followed by Final: every result must equal the reference; returns the key_words metric"""
    ref = agg_reference(cols, types, group_cols, aggs)
    ng = len(group_cols)
    for mode in (D.AGG_SINGLE, D.AGG_SINGLE_PARTITIONED):
        out, otypes, kw = run_agg(ctx, cols, types, group_cols, aggs, mode)
        check_agg(out, otypes, ref, types, group_cols, aggs, f"{what} mode {mode}")
    part, ptypes, _ = run_agg(ctx, cols, types, group_cols, aggs, D.AGG_PARTIAL)
    h = D.AggHandle(ctx, ptypes, list(range(ng)), [(f, -1, -1) for f, _, _ in aggs], D.AGG_FINAL, 8192)
    try:
        pv = [(v, None if ok.all() else ok) for v, ok in part]
        push_arrow(h.push_arrow, pv, ptypes, splits(len(pv[0][0]), 2), pad_start=1)
        h.finish()
        out, otypes = drain(h)
    finally:
        h.close()
    check_agg(out, otypes, ref, [ptypes[c] for c in range(ng)] + types[ng:], list(range(ng)), [(f, a, -1) for f, a, _ in aggs], f"{what} partial+final")
    return kw


GROUP_KEY_TYPES = ALL


@pytest.mark.parametrize("t", GROUP_KEY_TYPES, ids=[NAME[t] for t in GROUP_KEY_TYPES])
def test_group_by_single_key_of_every_type(gpu_ctx, t):
    rng = np.random.default_rng(200 + t)
    n = 5003
    p = pool(t)
    if t in (D.DATE64, D.TIMESTAMP):
        p = p + [-(1 << 63) + 2, (1 << 63) - 3]
    key = draw(rng, p, t, n, 0.07)
    vals = (rng.integers(-1000, 1000, n).astype(np.int64), rng.random(n) > 0.1)
    cols, types = [key, vals], [t, D.INT64]
    aggs = [(D.AGG_SUM, 1, -1), (D.AGG_COUNT, 1, -1), (D.AGG_MIN, 1, -1), (D.AGG_COUNT_STAR, -1, -1)]
    run_agg_modes(gpu_ctx, cols, types, [0], aggs, NAME[t])
    groups = len(agg_reference(cols, types, [0], aggs))
    if t == D.BOOL:
        assert groups == 3            # true, false, NULL
    if t == D.FLOAT32:                # +-0 fold into one group, the four NaNs stay four groups
        assert groups == len(p) - 1 + 1


MULTI_GROUP = {
    "bool-i8-u16-f32": ([D.BOOL, D.INT8, D.UINT16, D.FLOAT32], 1),   # 57 value bits + 4 NULL flags: one exact tag word
    "i64-u64": ([D.INT64, D.UINT64], 2),                              # 128 value bits: the tag without NULL flags
    "i64-f64-f32-date32-i8": ([D.INT64, D.FLOAT64, D.FLOAT32, D.DATE32, D.INT8], 1),   # 200 bits: the wide path (hash tag + stored tuples)
    "dec-bool": ([DEC, D.BOOL], 1),                                   # a Decimal128 beside another column: wide
}


@pytest.mark.parametrize("name", list(MULTI_GROUP))
def test_group_by_multi_column_keys(gpu_ctx, name):
    types, key_words = MULTI_GROUP[name]
    rng = np.random.default_rng(len(name))
    n = 4099
    nullable = name != "i64-u64"
    cols = [draw(rng, pool(t)[:7] if t in INTS else pool(t), t, n, 0.06 if nullable else 0.0) for t in types]
    cols.append((rng.integers(-2**40, 2**40, n).astype(np.int64), None))
    k = len(types)
    aggs = [(D.AGG_SUM, k, -1), (D.AGG_MAX, k, -1), (D.AGG_COUNT_STAR, -1, -1)]
    kw = run_agg_modes(gpu_ctx, cols, types + [D.INT64], list(range(k)), aggs, name)
    assert kw == key_words, (name, kw)
    if name == "i64-u64":
        # without NULL flags a NULL key cannot be represented: it is refused, never folded into another group
        h = D.AggHandle(gpu_ctx, types + [D.INT64], [0, 1], aggs, D.AGG_SINGLE, 8192)
        bad = [(cols[0][0][:100], np.arange(100) != 41), (cols[1][0][:100], None), (cols[2][0][:100], None)]
        with pytest.raises(D.DfgpuError):
            push_arrow(h.push_arrow, bad, types + [D.INT64], [(0, 100)], pad_start=2)
        h.close()


ARG_TYPES = [D.INT8, D.INT16, D.INT32, D.INT64, D.UINT8, D.UINT16, D.UINT32, D.UINT64, D.FLOAT32, D.FLOAT64, D.DATE32, D.DATE64, D.TIMESTAMP]


def arg_values(rng, t, n):
    """values at the type's edges: SUMs that wrap (UInt64) and SUMs of Int8 / Int16 extremes that must not wrap (they accumulate in
    Int64), MIN / MAX across 2^63 for UInt64 and of Int8 -128; floats are finite here, with +-0 and subnormals (NaN and +-inf MIN / MAX:
    test_group_by_float_min_max_bit_for_bit)"""
    if t in (D.FLOAT32, D.FLOAT64):
        return draw(rng, [x for x in pool(t) if abs(float(x)) < 1e300] + [3.25, -1e10, 1e-3], t, n, 0.15)   # sums stay finite
    if t == D.INT64:
        return draw(rng, [-(1 << 63), (1 << 63) - 1, -(1 << 63) + 7, (1 << 63) - 100, 0, -1, 5], t, n, 0.15)
    if t in (D.DATE64, D.TIMESTAMP):
        return draw(rng, [-(1 << 62), (1 << 62) + 3, 0, -1, 1_700_000_000_000], t, n, 0.15)
    return draw(rng, pool(t), t, n, 0.15)


@pytest.mark.parametrize("t", ARG_TYPES, ids=[NAME[t] for t in ARG_TYPES])
def test_group_by_aggregates_over_every_argument_type(gpu_ctx, t):
    rng = np.random.default_rng(300 + t)
    n = 6007
    g = (rng.integers(0, 23, n).astype(np.int32), rng.random(n) > 0.03)
    v = arg_values(rng, t, n)
    filt = (rng.random(n) > 0.3, rng.random(n) > 0.1)
    cols, types = [g, v, filt], [D.INT32, t, D.BOOL]
    aggs = [(D.AGG_SUM, 1, -1), (D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_AVG, 1, -1), (D.AGG_COUNT, 1, -1),
            (D.AGG_SUM, 1, 2), (D.AGG_MAX, 1, 2), (D.AGG_COUNT, 2, -1)]
    if t in (D.DATE32, D.DATE64, D.TIMESTAMP):
        aggs = [a for a in aggs if a[0] in (D.AGG_MIN, D.AGG_MAX, D.AGG_COUNT)]
    run_agg_modes(gpu_ctx, cols, types, [0], aggs, NAME[t])
    if t in (D.INT8, D.INT16, D.UINT64):        # the data reaches the edge each case names
        ref = agg_reference(cols, types, [0], aggs)
        sums = [c[0] for c in ref.values() if c[0] is not None]
        info = np.iinfo(npt(t))
        if t == D.UINT64:
            raw = [sum(int(x) for x, ok, gg, gv in zip(v[0], v[1], g[0], g[1]) if ok and gv and gg == k) for k in range(23)]
            assert any(s >= 1 << 64 for s in raw)
        else:
            assert any(s > info.max or s < info.min for s in sums)


def test_group_by_float_min_max_bit_for_bit(gpu_ctx):
    """Float32 and Float64 MIN / MAX over +-0, +-inf and NaNs of both signs and several payloads: the result is one of the inputs bit for
    bit in totalOrder, with the argument's type"""
    rng = np.random.default_rng(11)
    n = 3001
    for t in (D.FLOAT32, D.FLOAT64):
        g = (rng.integers(0, 40, n).astype(np.int16), None)
        v = draw(rng, pool(t), t, n, 0.2)
        aggs = [(D.AGG_MIN, 1, -1), (D.AGG_MAX, 1, -1), (D.AGG_MIN, 1, 2)]
        run_agg_modes(gpu_ctx, [g, v, (rng.random(n) > 0.5, None)], [D.INT16, t, D.BOOL], [0], aggs, NAME[t])


def test_group_by_avg_of_int64_near_the_extremes(gpu_ctx):
    n = 2049
    rng = np.random.default_rng(5)
    g = (rng.integers(0, 3, n).astype(np.uint8), None)
    v = (np.where(rng.random(n) < 0.5, np.int64(-(1 << 63)), np.int64((1 << 63) - 1)), None)
    run_agg_modes(gpu_ctx, [g, v], [D.UINT8, D.INT64], [0], [(D.AGG_AVG, 1, -1), (D.AGG_SUM, 1, -1)], "avg extremes")


def test_group_by_refuses_arithmetic_on_boolean(gpu_ctx):
    for func in (D.AGG_SUM, D.AGG_MIN, D.AGG_MAX, D.AGG_AVG):
        with pytest.raises(D.DfgpuError) as e:
            D.AggHandle(gpu_ctx, [D.INT32, D.BOOL], [0], [(func, 1, -1)], D.AGG_SINGLE, 8192)
        assert e.value.code == -3, func       # DFGPU_ERR_UNSUPPORTED
