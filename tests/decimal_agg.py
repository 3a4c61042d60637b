"""MIN / MAX / AVG (and SUM) over Decimal128 for the tests of the dense aggregate sink: a restatement on top of the oracle, whose
group_by / scalar_aggregate cover SUM and COUNT over `Dec` only.  Python ints throughout.

AVG over Decimal128(p, s) as DataFusion 55 evaluates it: Avg::return_type (functions-aggregate average.rs) is
Decimal128(min(38, p + 4), min(38, s + 4)) = (tp, ts); DecimalAverager::avg (functions-aggregate-common utils.rs) takes the i128
add_wrapping sum, computes sum.mul_checked(10^(ts - s)).div_wrapping(count) (truncation toward zero) and validates the value
against precision tp.  An overflow of the multiply or of the precision raises "Arithmetic Overflow in AvgAccumulator"
(ArrowArithmeticOverflow here).  MIN / MAX keep the argument's type; no value -> NULL."""
from typing import List, Sequence

import numpy as np

from oracle import oracle as O

_I128_MIN, _I128_MAX = -(1 << 127), (1 << 127) - 1
_PY = (O.A_MIN, O.A_MAX, O.A_AVG)


def _is_dec(arg) -> bool:
    return arg is not None and isinstance(arg[0], O.Dec)


def _wrap128(x: int) -> int:
    x %= 1 << 128
    return x - (1 << 128) if x >= (1 << 127) else x


def _tdiv(a: int, b: int) -> int:      # Rust's `/` on integers truncates toward zero
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def decimal_avg(total: int, count: int, p: int, s: int):
    """DecimalAverager::avg for AVG(Decimal128(p, s)) over `count` values summing to `total` -> (value, tp, ts)"""
    tp, ts = min(38, p + 4), min(38, s + 4)
    m = _wrap128(total) * 10 ** (ts - s)
    if not (_I128_MIN <= m <= _I128_MAX):
        raise O.ArrowArithmeticOverflow("Arithmetic Overflow in AvgAccumulator")
    q = _tdiv(m, count)
    if not abs(q) < 10 ** tp:
        raise O.ArrowArithmeticOverflow("Arithmetic Overflow in AvgAccumulator")
    return q, tp, ts


def _dec_agg(func: int, vals: list, p: int, s: int):
    """one aggregate over the non-NULL values `vals` -> (value, precision, scale, valid)"""
    if func == O.A_SUM:   # i128 add_wrapping into Decimal128(min(38, p + 10), s) (Sum::return_type)
        return _wrap128(sum(vals)), min(38, p + 10), s, bool(vals)
    if func == O.A_AVG:
        if not vals:
            return (0,) + (min(38, p + 4), min(38, s + 4)) + (False,)
        return decimal_avg(sum(vals), len(vals), p, s) + (True,)
    if not vals:
        return 0, p, s, False
    return (min(vals) if func == O.A_MIN else max(vals)), p, s, True


def _active(n: int, arg, filt) -> np.ndarray:
    act = np.ones(n, bool) if arg[1] is None else np.asarray(arg[1], bool).copy()
    if filt is not None:
        act &= np.asarray(filt[0], bool) & (np.ones(n, bool) if filt[1] is None else np.asarray(filt[1], bool))
    return act


def _key_rows(keys: Sequence[O.Col], n: int) -> list:
    cols = [(np.asarray(k[0]).tolist(), None if k[1] is None else np.asarray(k[1], bool).tolist()) for k in keys]
    return [tuple(None if (v is not None and not v[i]) else c[i] for c, v in cols) for i in range(n)]


def group_by(keys: Sequence[O.Col], aggs: Sequence[tuple]):
    """O.group_by (groups in first-seen order, one result dict per aggregate) where MIN / MAX / AVG over a `Dec` argument are computed
    here; their dicts carry dec=Dec(...) and valid.  The oracle takes each other aggregate in a call of its own."""
    n = len(keys[0][0])
    out_keys, _ = O.group_by(keys, [(O.A_COUNT_STAR, None, None)])
    ng = len(out_keys[0][0]) if out_keys else 0
    rows = _key_rows(keys, n)
    ids = {}
    gid = np.array([ids.setdefault(r, len(ids)) for r in rows], np.int64)
    assert list(ids) == _key_rows(out_keys, ng), "group_by's groups are not in first-seen order"
    res: List[dict] = []
    for ag in aggs:
        func, arg, filt = ag[0], ag[1], ag[2] if len(ag) > 2 else None
        if func in _PY and _is_dec(arg):
            per = [[] for _ in range(ng)]
            for i in np.nonzero(_active(n, arg, filt))[0].tolist():
                per[gid[i]].append(int(arg[0][i]))
            r = [_dec_agg(func, v, arg[0].p, arg[0].s) for v in per]
            pp, ss = (r[0][1], r[0][2]) if r else _dec_agg(func, [], arg[0].p, arg[0].s)[1:3]
            res.append(dict(dec=O.Dec([x[0] for x in r], pp, ss), valid=np.array([x[3] for x in r], bool), i=None, f=None, c=None))
        else:
            k, r1 = O.group_by(keys, [ag])
            assert _key_rows(k, ng) == list(ids)
            res.append(r1[0])
    return out_keys, res


def agg_output_columns(func: int, r: dict, arg_dtype, state: bool) -> List[O.Col]:
    """O.agg_output_columns, with the Decimal128 results of group_by above"""
    if r.get("dec") is not None:
        return [(r["dec"], None if r["valid"].all() else r["valid"])]
    return O.agg_output_columns(func, r, arg_dtype, state)


def scalar_aggregate(aggs: Sequence[tuple], state: bool = False) -> List[O.Col]:
    """O.scalar_aggregate (AggregateStream: one row, also for empty input) where SUM / MIN / MAX / AVG over `Dec` are computed here"""
    out: List[O.Col] = []
    for ag in aggs:
        func, arg, filt = ag[0], ag[1], ag[2] if len(ag) > 2 else None
        if func in (O.A_SUM,) + _PY and _is_dec(arg):
            if state and func == O.A_AVG:
                raise NotImplementedError("AVG over Decimal128 has no state restated here")
            vals = [int(arg[0][i]) for i in np.nonzero(_active(len(arg[0]), arg, filt))[0].tolist()]
            v, pp, ss, ok = _dec_agg(func, vals, arg[0].p, arg[0].s)
            out.append((O.Dec([v if ok else 0], pp, ss), None if ok else np.array([False])))
        else:
            out += O.scalar_aggregate([ag], state=state)
    return out
