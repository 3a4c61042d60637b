"""Host side of MIN / MAX / AVG over Decimal128 in the hash group-by, no GPU needed: the operator twin's Single-mode schema, the AVG
Partial state it refuses to invent, and the exact Int64 <-> Decimal128 check of scripts/agg_decimal_timing.py on tiny host data."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

from datafusion_b200.exec import AggregateExpr, GpuAggregateExec, MemoryExec
import decimal_agg as DA

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import agg_decimal_timing as T  # noqa: E402


def _src():
    from decimal import Decimal
    t = pa.table({"k": pa.array([1, 2], pa.int64()), "m": pa.array([Decimal("1.25"), None], pa.decimal128(15, 2)),
                  "w": pa.array([Decimal("0.5"), Decimal("1.5")], pa.decimal128(38, 36))})
    return MemoryExec(t.to_batches(), t.schema)


@pytest.mark.parametrize("mode", ["Single", "SinglePartitioned"])
def test_single_mode_schema_of_decimal_min_max_avg(mode):
    exprs = [AggregateExpr("min", "m", "mn"), AggregateExpr("max", "m", "mx"), AggregateExpr("avg", "m", "av"), AggregateExpr("avg", "w", "aw"),
             AggregateExpr("sum", "m", "sm")]
    plan = GpuAggregateExec(mode, ["k"], exprs, _src())
    assert [(f.name, f.type) for f in plan.schema] == [("k", pa.int64()), ("mn", pa.decimal128(15, 2)), ("mx", pa.decimal128(15, 2)),
                                                       ("av", pa.decimal128(19, 6)), ("aw", pa.decimal128(38, 38)), ("sm", pa.decimal128(25, 2))]


def test_avg_decimal_state_fields_raise_and_partial_fails_at_planning():
    with pytest.raises(NotImplementedError, match="Single modes only"):
        AggregateExpr("avg", "m").state_fields(pa.decimal128(15, 2))
    part = GpuAggregateExec("Partial", ["k"], [AggregateExpr("avg", "m", "av")], _src())   # constructible: the fusion rules inspect it
    with pytest.raises(NotImplementedError, match="av: AVG over decimal128"):
        part.schema
    with pytest.raises(NotImplementedError):
        next(part.execute(None))
    # MIN / MAX / SUM keep their Partial states; AVG over Float64 keeps [count, sum: Float64]
    assert [f.type for f in AggregateExpr("min", "m").state_fields(pa.decimal128(15, 2))] == [pa.decimal128(15, 2)]
    assert [f.type for f in AggregateExpr("sum", "m").state_fields(pa.decimal128(15, 2))] == [pa.decimal128(25, 2)]
    assert [f.type for f in AggregateExpr("avg", "m").state_fields(pa.float64())] == [pa.uint64(), pa.float64()]


def _runs(keys, vals):
    """what the script's two runs return, computed here: Int64 rows (AVG as Float64) and Decimal128(15,2) rows (unscaled ints, AVG by
    the DecimalAverager restatement of tests/decimal_agg.py)"""
    ints, decs = [], []
    for k in np.unique(keys):
        v = [int(x) for x in vals[keys == k]]
        s, c = sum(v), len(v)
        ints.append((int(k), s, min(v), max(v), s / c, c))
        decs.append((int(k), s, min(v), max(v), DA.decimal_avg(s, c, 15, 2)[0], c))
    return ints, decs


def test_timing_script_exact_check_on_host_data():
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 50, 2000)
    vals = rng.integers(T.V_LO, T.V_LO + T.V_SPAN, 2000)
    ints, decs = _runs(keys, vals)
    assert any(d[1] < 0 and d[1] * 10 ** 4 % d[5] for d in decs), "no negative group sum with a remainder: truncation is untested"
    T.check_exact(ints, decs[::-1])                      # output order does not matter
    for j in (1, 2, 3, 4, 5):                            # every compared column is compared
        bad = list(decs)
        bad[7] = bad[7][:j] + (bad[7][j] + 1,) + bad[7][j + 1:]
        with pytest.raises(AssertionError):
            T.check_exact(ints, bad)
    with pytest.raises(AssertionError):
        T.check_exact(ints, decs[:-1])
    with pytest.raises(AssertionError):                  # floor division instead of truncation toward zero
        T.check_exact(ints, [d[:4] + ((d[1] * 10 ** 4) // d[5],) + d[5:] for d in decs])
