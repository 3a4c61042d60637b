"""The float MIN / MAX rule restated on the CPU: IEEE-754 totalOrder on the value's bits (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf <
+NaN, payloads ordered by their bits), the result one of the inputs bit for bit, NULL for a group without a non-NULL value.  Also the
class rule of a float SUM / AVG over data with NaN and +-inf, and the edge data the GPU tests feed every aggregate path.  Needs no GPU."""
import math
import struct

import numpy as np

_U = {np.dtype(np.float64): (np.uint64, 64), np.dtype(np.float32): (np.uint32, 32)}


def order_key(a):
    """float64 / float32 array -> unsigned keys of the same width that sort in totalOrder: all bits flipped when the sign is set,
    else the sign bit set"""
    a = np.ascontiguousarray(a)
    ut, bits = _U[a.dtype]
    u = a.view(ut)
    top = ut(1 << (bits - 1))
    return np.where(u & top, ~u, u | top).astype(ut)


def from_key(k, dtype):
    """the inverse of order_key"""
    ut, bits = _U[np.dtype(dtype)]
    k = np.asarray(k, ut)
    top = ut(1 << (bits - 1))
    return np.ascontiguousarray(np.where(k & top, k & ~top, ~k).astype(ut)).view(dtype)


def group_min_max(values, valid, groups, n_groups, is_min):
    """per-group MIN or MAX in totalOrder -> (values of the input dtype, valid: the group has a non-NULL value)"""
    values = np.ascontiguousarray(values)
    ut, _ = _U[values.dtype]
    sel = np.ones(len(values), bool) if valid is None else np.asarray(valid, bool)
    g = np.asarray(groups, np.int64)[sel]
    k = order_key(values)[sel]
    acc = np.full(n_groups, np.iinfo(ut).max if is_min else 0, ut)
    (np.minimum if is_min else np.maximum).at(acc, g, k)
    has = np.bincount(g, minlength=n_groups) > 0
    return np.where(has, from_key(acc, values.dtype), values.dtype.type(0)), has


def bits(x, dtype=np.float64):
    return int(np.asarray([x], dtype).view(_U[np.dtype(dtype)][0])[0])


def assert_same_bits(got, got_valid, want, want_valid, what=""):
    """values compared by their bits where valid; the validity exactly"""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.dtype == want.dtype and len(got) == len(want), f"{what}: {got.dtype}[{len(got)}] vs {want.dtype}[{len(want)}]"
    gv = np.ones(len(got), bool) if got_valid is None else np.asarray(got_valid, bool)
    wv = np.ones(len(want), bool) if want_valid is None else np.asarray(want_valid, bool)
    bad = np.nonzero(gv != wv)[0]
    assert not len(bad), f"{what}: row {bad[0]} valid {gv[bad[0]]}, expected {wv[bad[0]]}"
    ut = _U[got.dtype][0]
    gb, wb = got.view(ut), want.view(ut)
    bad = np.nonzero(wv & (gb != wb))[0]
    assert not len(bad), (f"{what}: {len(bad)} rows differ, e.g. row {bad[0]}: {hex(int(gb[bad[0]]))} ({got[bad[0]]!r}), "
                          f"expected {hex(int(wb[bad[0]]))} ({want[bad[0]]!r})")


# ---- SUM / AVG over NaN and +-inf --------------------------------------------------------------------------------
ANY = "any"   # the finite terms can overflow in some order: no class is promised


def fclass(x):
    if math.isnan(x):
        return "nan"
    if math.isinf(x):
        return "+inf" if x > 0 else "-inf"
    return "finite"


def sum_expect(xs, avg=False):
    """the class a float SUM (AVG) of xs has in every order, with the Approx bound of a finite one; ANY where the finite terms can
    overflow"""
    xs = [float(x) for x in xs]
    if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
        return "nan"
    if math.inf in xs:
        return "+inf"
    if -math.inf in xs:
        return "-inf"
    try:
        if math.fsum(abs(x) for x in xs) * (1 + (len(xs) + 64) * 2.0 ** -52) >= np.finfo(np.float64).max:
            return ANY
    except OverflowError:
        return ANY
    import dense_cases   # not at the top: dense_cases imports this module
    return dense_cases._fsum_cells(xs, avg)


def check_sum(got, want, what=""):
    """got: a Python float or None; want: from sum_expect.  A NaN is compared by its class, never its bits"""
    if want == ANY:
        return
    assert got is not None, f"{what}: NULL"
    if isinstance(want, str):
        assert fclass(got) == want, f"{what}: {got!r} is not {want}"
    else:
        assert fclass(got) == "finite" and abs(got - want.exact) <= want.tol, f"{what}: {got!r} != {want!r}"


# ---- edge data -------------------------------------------------------------------------------------------------
def _f64(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def _f32(b):
    return np.array([b], np.uint32).view(np.float32)[0]


DBL_MAX, DBL_MIN, DBL_TRUE_MIN = np.finfo(np.float64).max, np.finfo(np.float64).tiny, np.float64(5e-324)
# quiet NaNs only (bit 51 / bit 22 set): a conversion may quiet a signalling NaN
NANS64 = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF800000000BEEF, 0xFFFC00000000CAFE, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF]
NANS32 = [0x7FC00000, 0xFFC00000, 0x7FC0BEEF, 0xFFE0CAFE, 0x7FFFFFFF, 0xFFFFFFFF]


def edge_values(dtype):
    """every edge value of the type, as an array of that dtype"""
    if dtype == np.float64:
        nans = [_f64(b) for b in NANS64]
        fin = np.finfo(np.float64)
        special = [0.0, -0.0, np.inf, -np.inf, fin.max, -fin.max, fin.tiny, -fin.tiny, DBL_TRUE_MIN, -DBL_TRUE_MIN, 1.0, -1.5, 1e300, -3e-300]
        return np.array(nans + special, np.float64)
    fin = np.finfo(np.float32)
    nans = [_f32(b) for b in NANS32]
    special = [np.float32(x) for x in (0.0, -0.0, np.inf, -np.inf, fin.max, -fin.max, fin.tiny, -fin.tiny, 1e-45, -1e-45, 1.0, -1.5)]
    return np.array(nans + special, np.float32)


def nan(i, dtype=np.float64):
    """the i-th quiet NaN of NANS64 / NANS32: 0 +NaN, 1 -NaN, 2 +NaN with a payload, 3 -NaN with a payload"""
    return _f64(NANS64[i]) if dtype == np.float64 else _f32(NANS32[i])


def edge_groups(dtype):
    """{group: [values, None = NULL]}: the groups that isolate each case"""
    N = lambda i: nan(i, dtype)
    t = np.dtype(dtype).type
    big, tiny = np.finfo(dtype).max, np.finfo(dtype).tiny
    return {
        0: [N(0)],                              # NaN only
        1: [N(0), N(2)],                        # NaN only, with a payload
        2: [t(0.0), t(-0.0)],                   # the signed zeros
        3: [N(1), N(0)],                        # -NaN, +NaN
        4: [N(0), t(np.inf)],                   # NaN, +inf
        5: [t(-np.inf), N(1)],                  # -inf, -NaN
        6: [None, None],                        # all NULL
        7: [None, N(0)],                        # NULL plus NaN
        8: [t(1.0), N(0)],                      # MAX -> NaN
        9: [N(1), t(1.0)],                      # MIN -> -NaN
        10: [t(-0.0)],                          # -0.0 only
        11: [N(2), N(3)],                       # payloads of both signs
        12: [big, -big, tiny, -tiny],           # the largest and smallest normals
        13: [t(0.0), t(-0.0), tiny, -tiny, t(np.inf), t(-np.inf)],
    }


N_EDGE_GROUPS = 14


def edge_case(rng, dtype, n_groups=48, copies=24, n_random=6000):
    """-> (group Int64 keys, values, valid) in a shuffled row order.  Every value of an isolating group appears `copies` times; groups
    N_EDGE_GROUPS .. n_groups - 1 draw from the edge values, ordinary values and NULL at random"""
    eg = edge_groups(dtype)
    keys, vals, valid = [], [], []
    for g, vs in eg.items():
        for _ in range(copies):
            for v in vs:
                keys.append(g)
                vals.append(0.0 if v is None else v)
                valid.append(v is not None)
    pool = edge_values(dtype)
    ordinary = (rng.standard_normal(n_random) * 1e3).astype(dtype)
    pick = rng.integers(0, len(pool), n_random)
    use_edge = rng.random(n_random) < 0.3
    keys += rng.integers(N_EDGE_GROUPS, n_groups, n_random).tolist()
    vals += list(np.where(use_edge, pool[pick], ordinary))
    valid += (rng.random(n_random) > 0.1).tolist()
    k = np.array(keys, np.int64)
    v = np.empty(len(vals), dtype)
    for i, x in enumerate(vals):   # element by element: a NaN's bits survive only without arithmetic
        v[i] = x
    ok = np.array(valid, bool)
    perm = rng.permutation(len(k))
    return k[perm], v[perm], ok[perm]


def race_case(rng, n=1 << 20, n_groups=16):
    """>= 1M rows on 16 groups: half +0.0 and half -0.0, a few +-NaN in groups 0..3 and +-inf in group 4 -> (keys, values)"""
    keys = rng.integers(0, n_groups, n).astype(np.int64)
    v = np.where(rng.random(n) < 0.5, 0.0, -0.0)
    for g, b in ((0, NANS64[0]), (1, NANS64[1]), (2, NANS64[2]), (3, NANS64[3])):
        idx = rng.choice(np.nonzero(keys == g)[0], 7, replace=False)
        v.view(np.uint64)[idx] = b
    idx4 = np.nonzero(keys == 4)[0][:2]
    v[idx4] = [np.inf, -np.inf]
    return keys, v


def reference(keys, values, valid, n_groups):
    """{group: (MIN, MAX, SUM expectation, AVG expectation, COUNT)} over the groups with at least one row; MIN / MAX are numpy scalars
    of the input dtype or None"""
    mn, has = group_min_max(values, valid, keys, n_groups, True)
    mx, _ = group_min_max(values, valid, keys, n_groups, False)
    ok = np.ones(len(values), bool) if valid is None else np.asarray(valid, bool)
    out = {}
    order = np.argsort(keys, kind="stable")
    bounds = np.flatnonzero(np.diff(keys[order])) + 1
    for rows in np.split(order, bounds) if len(order) else []:
        g = int(keys[rows[0]])
        xs = values[rows[ok[rows]]].astype(np.float64)
        out[g] = (mn[g] if has[g] else None, mx[g] if has[g] else None, sum_expect(xs) if len(xs) else None,
                  sum_expect(xs, True) if len(xs) else None, len(xs))
    return out
