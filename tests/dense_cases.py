"""Test support for the dense aggregate sink's accumulator tests: a plain Python reference of the sink (integers and decimals as
Python ints, Float64 sums with math.fsum and an error bound), the data of the edge cases, and a restatement of the sink's
accumulator word layout.  Needs no GPU."""
import math

import numpy as np

from datafusion_b200 import capi as D
from oracle import oracle as O
import decimal_agg as DA
import float_order as FO

I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
DEC38_MAX = 10 ** 38 - 1
WARP_BYTES, WARPS = 48 * 1024, 8          # per-warp accumulator copies when all eight fit in 48 KB


def kind_of(t):
    if D.type_base(t) == D.DECIMAL128:
        return "dec"
    if t == D.FLOAT64:
        return "f64"
    return "u64" if t in (D.UINT8, D.UINT16, D.UINT32, D.UINT64) else "i64"


class Approx:
    """a Float64 SUM or AVG: the exactly rounded value and how far a float sum of the same values may be from it"""

    def __init__(self, exact, tol):
        self.exact, self.tol = exact, tol

    def __repr__(self):
        return f"Approx({self.exact!r} +- {self.tol!r})"


def _fsum_cells(xs, avg):
    n = len(xs)
    exact, mag = math.fsum(xs), math.fsum(abs(x) for x in xs)
    tol = (n + 64) * 2.0 ** -52 * mag    # |sum in any order - exact sum| for n doubles
    if not avg:
        return Approx(exact, tol)
    return Approx(exact / n, tol / n + 2.0 ** -52 * abs(exact / n))


def key_slots(cols, group_cols, key_range):
    """slot of every row (row-major over radix max - min + 2, NULL = max - min + 1); keys are compared modulo 2^64 like Int64 / UInt64
    bounds passed through the C ABI"""
    n = len(cols[0][0])
    slot, stride, inside = np.zeros(n, np.int64), 1, np.ones(n, bool)
    for g, (lo, hi) in reversed(list(zip(group_cols, key_range))):
        v, valid = cols[g]
        span = (int(hi) - int(lo)) % (1 << 64)
        with np.errstate(over="ignore"):
            idx = np.asarray(v).astype(np.uint64) - np.uint64(int(lo) % (1 << 64))
        inside &= idx <= np.uint64(span)
        idx = np.where(idx <= np.uint64(span), idx, 0).astype(np.int64)
        if valid is not None:
            idx = np.where(np.asarray(valid, bool), idx, span + 1)
            inside |= ~np.asarray(valid, bool)
        slot += idx * stride
        stride *= span + 2
    return slot, inside


def _py(col, i):
    v, valid = col
    if valid is not None and not valid[i]:
        return None
    x = v[i]
    return int(x) if isinstance(v, O.Dec) else np.asarray(v)[i].item()


def reference(cols, types, keep, group_cols, key_range, aggs, partial=False):
    """the dense sink restated -> rows in output order.  cols: oracle columns (virtual columns of probe stages appended); keep: the
    rows that reach the sink (None = all); aggs: [(func, argument column or None)]"""
    n = len(cols[0][0])
    keep = np.ones(n, bool) if keep is None else np.asarray(keep, bool)
    if group_cols:
        slot, inside = key_slots(cols, group_cols, key_range)
        assert inside[keep].all(), "reference: a kept row's key lies outside its declared range"
    else:
        slot = np.zeros(n, np.int64)
    rows_all = np.nonzero(keep)[0]
    order = rows_all[np.argsort(slot[rows_all], kind="stable")]
    bounds = np.flatnonzero(np.diff(slot[order])) + 1
    groups = np.split(order, bounds) if len(order) else ([] if group_cols else [order])
    out = []
    for rows in groups:
        key = tuple(_py(cols[g], rows[0]) for g in group_cols)
        cells = []
        for func, c in aggs:
            if func == D.AGG_COUNT_STAR:
                cells.append(len(rows))
                continue
            v, valid = cols[c]
            sel = rows if valid is None else rows[np.asarray(valid, bool)[rows]]
            if func == D.AGG_COUNT:
                cells.append(len(sel))
                continue
            k = kind_of(types[c])
            if k == "dec":
                xs = [int(x) for x in v[sel]]
            elif k == "f64":
                xs = np.asarray(v, np.float64)[sel].tolist()
            else:
                xs = np.asarray(v)[sel].tolist()
            if func == D.AGG_AVG and partial:    # state: [count UInt64, sum Float64 (NULL without a value)]
                cells += [len(xs), _fsum_cells(xs, False) if xs else None]
                continue
            if not xs:
                cells.append(None)
            elif func in (D.AGG_MIN, D.AGG_MAX) and k == "f64":   # IEEE totalOrder on the bits
                ordk = FO.order_key(np.asarray(xs, np.float64))
                cells.append(xs[int(np.argmin(ordk) if func == D.AGG_MIN else np.argmax(ordk))])
            elif func == D.AGG_MIN:
                cells.append(min(xs))
            elif func == D.AGG_MAX:
                cells.append(max(xs))
            elif k == "dec":
                p, s = D.decimal_precision_scale(types[c])
                cells.append(DA._wrap128(sum(xs)) if func == D.AGG_SUM else DA.decimal_avg(sum(xs), len(xs), p, s)[0])
            elif k == "f64":
                cells.append(_fsum_cells(xs, func == D.AGG_AVG))
            else:
                assert func == D.AGG_SUM
                t = sum(xs) % (1 << 64)
                cells.append(t if k == "u64" else (t - (1 << 64) if t > I64_MAX else t))
        out.append(key + tuple(cells))
    return sorted(out, key=lambda r: tuple((1, 0) if x is None else (0, x) for x in r[:len(group_cols)]))


def check_rows(got, want, what=""):
    """integers, decimals, MIN / MAX exactly; Float64 SUM / AVG within the bound of an n-term float sum"""
    assert len(got) == len(want), f"{what}: {len(got)} rows, expected {len(want)}"
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w), f"{what}: row {i} has {len(g)} columns, expected {len(w)}"
        for j, (a, b) in enumerate(zip(g, w)):
            if isinstance(b, Approx):
                assert a is not None and abs(a - b.exact) <= b.tol, f"{what}: row {i} col {j}: {a!r} != {b!r}"
            else:
                assert a == b and (a is None) == (b is None), f"{what}: row {i} col {j}: {a!r} != {b!r}"


# ---- the sink's accumulator layout, restated -------------------------------------------------------
def slot_words(aggs):
    """words of one slot for aggs = [(func, is_decimal)]: word 0 counts the rows; COUNT(x) takes one word; SUM / MIN / MAX / AVG take
    one value word (two for Decimal128, at an even word) and a non-null counter; the total is even"""
    w = 1
    for func, dec in aggs:
        if func == D.AGG_COUNT_STAR:
            continue
        if func == D.AGG_COUNT:
            w += 1
            continue
        if dec:
            w += (w & 1) + 2
        else:
            w += 1
        w += 1
    return w + (w & 1)


def per_warp(slots, aggs):
    return WARPS * slots * slot_words(aggs) * 8 <= WARP_BYTES


# ---- case c: 128-bit carries and wrapping, Decimal128(38, 0) ----------------------------------------
CARRY_GROUPS = 8          # key 0..7 and NULL


def _carry_value(rng, g):
    k = int(rng.integers(1, 1000))
    if g == 0:
        return (1 << 64) - k                                  # lo near 2^64, hi = 0
    if g == 1:
        return -k                                             # lo near 2^64, hi all ones: a negative sum
    if g == 2:
        return ((1 << 64) - k) * (1 if rng.random() < 0.5 else -1)   # mixed signs
    if g == 3:
        return int(rng.integers(-(1 << 62), 1 << 62)) << 38
    if g == 4:
        return DEC38_MAX - k                                  # the sum passes 2^127 and wraps
    if g == 5:
        return -(DEC38_MAX - k)                               # ... and -2^127
    if g == 6:
        return (1 << 63) - 1 if rng.random() < 0.5 else 1 << 63      # low words across bit 63, hi = 0
    if g == 7:
        return -1 if rng.random() < 0.5 else -(1 << 64)       # lo all ones or 0, hi all ones
    return (1 << 63) + k                                      # the NULL key's rows


def carry_case(rng, n):
    """cols: 0 key Int32 in [0, 7] (NULL ~1/9), 1 second key Int32 in [0, 24], 2 Decimal128(38, 0)"""
    g = rng.integers(0, CARRY_GROUPS + 1, n)
    vals = [_carry_value(rng, int(x)) for x in g]
    k1 = (np.minimum(g, CARRY_GROUPS - 1).astype(np.int32), g < CARRY_GROUPS)
    k2 = (rng.integers(0, 25, n).astype(np.int32), None)
    return [k1, k2, (O.Dec(vals, 38, 0), None)], [D.INT32, D.INT32, D.decimal128(38, 0)]


def group_values(cols, key_col, arg_col):
    """{key (None for NULL): [Python ints of the non-NULL arguments]}"""
    out = {}
    for i in range(len(cols[key_col][0])):
        a = _py(cols[arg_col], i)
        if a is not None:
            out.setdefault(_py(cols[key_col], i), []).append(a)
    return out


# ---- case d: AVG over Decimal128(p, s) ----------------------------------------------------------------
AVG_TYPES = [(15, 2), (20, 0), (34, 10), (36, 35), (38, 38)]


def avg_mul(p, s):
    return min(38, s + 4) - s


def avg_case(rng, p, s, n=4000):
    """cols: 0 key Int32 in [0, 3] and NULL, 1 Decimal128(p, s) with ~10% NULL.  Group 0 is all negative, 1 mixed with a negative
    lean, 2 mixed with a positive lean, 3 has seven rows, all negative; magnitudes keep sum * 10^(ts - s) inside i128"""
    m = min(10 ** p - 1, 10 ** (33 - avg_mul(p, s)))
    g = rng.integers(0, 5, n)
    g[:7], g[7:][g[7:] == 3] = 3, 2
    def big(lo, hi):   # uniform-ish over [lo * m, hi * m] with all digits random
        return int(lo * m + (hi - lo) * m * rng.random()) + int(rng.integers(-999, 1000))
    vals = []
    for x in g:
        v = {0: big(-1.0, -0.01), 1: big(-1.0, 0.6), 2: big(-0.6, 1.0), 3: big(-1.0, -0.01)}.get(int(x), big(-1.0, 1.0))
        vals.append(max(-m, min(m, v)))
    if sum(vals[:7]) * 10 ** avg_mul(p, s) % 7 == 0:   # group 3: seven values whose average has a remainder
        vals[0] += 1
    valid = rng.random(n) > 0.1
    valid[:7] = True
    key = (np.minimum(g, 3).astype(np.int32), g < 4)
    return [key, (O.Dec(vals, p, s), valid)], [D.INT32, D.decimal128(p, s)]
