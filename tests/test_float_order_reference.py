"""The float MIN / MAX reference (tests/float_order.py) on the CPU: its totalOrder key against a brute-force sort of the struct-packed
bits, the edge data's bits, and the oracle's grouped and ungrouped float MIN / MAX against the reference over the edge data in both row
orders.  Needs no GPU."""
import math
import struct

import numpy as np
import pytest

from oracle import oracle as O
import dense_cases as C
import float_order as FO

from datafusion_b200 import capi as D


def brute_total_order(bits, width):
    """sort of raw bit patterns by IEEE totalOrder from first principles: sign, then (negatives reversed) magnitude bits"""
    sign = 1 << (width - 1)
    return sorted(bits, key=lambda b: (1, b) if not b & sign else (0, -(b & (sign - 1))))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_order_key_matches_a_brute_force_sort(dtype):
    rng = np.random.default_rng(1)
    width = 64 if dtype == np.float64 else 32
    ut = np.uint64 if width == 64 else np.uint32
    edge = FO.edge_values(dtype).view(ut).tolist()
    rand = rng.integers(0, 1 << width, 3000, dtype=ut, endpoint=False).tolist()
    bits = sorted(set(edge + rand))
    a = np.array(bits, ut).view(dtype)
    got = a.view(ut)[np.argsort(FO.order_key(a), kind="stable")].tolist()
    assert got == brute_total_order(bits, width)
    assert FO.from_key(FO.order_key(a), dtype).view(ut).tolist() == bits
    # the named landmarks in order
    inf, z = np.array([np.inf], dtype)[0], dtype(0.0)
    marks = np.array([FO.nan(1, dtype), -inf, -np.finfo(dtype).max, dtype(-1.0), -z, z, np.finfo(dtype).tiny, inf, FO.nan(0, dtype)], dtype)
    k = FO.order_key(marks)
    assert all(int(x) < int(y) for x, y in zip(k, k[1:]))


def test_edge_data_keeps_its_bits():
    for dtype, nans in ((np.float64, FO.NANS64), (np.float32, FO.NANS32)):
        ut = np.uint64 if dtype == np.float64 else np.uint32
        v = FO.edge_values(dtype).view(ut)
        assert set(nans) <= set(v.tolist())
        keys, vals, valid = FO.edge_case(np.random.default_rng(2), dtype)
        vb = set(vals.view(ut)[valid].tolist())
        assert set(nans[:4]) <= vb and FO.bits(-0.0, dtype) in vb and FO.bits(0.0, dtype) in vb
    _, v = FO.race_case(np.random.default_rng(3), n=1 << 16)
    assert {FO.bits(0.0), FO.bits(-0.0)} <= set(v.view(np.uint64).tolist()) and set(FO.NANS64[:4]) <= set(v.view(np.uint64).tolist())


def test_reference_on_the_isolating_groups():
    keys, vals, valid = FO.edge_case(np.random.default_rng(4), np.float64)
    ref = FO.reference(keys, vals, valid, 48)
    b = lambda x: None if x is None else FO.bits(x)
    want = {0: (FO.NANS64[0], FO.NANS64[0]), 1: (FO.NANS64[0], FO.NANS64[2]), 2: (FO.bits(-0.0), FO.bits(0.0)),
            3: (FO.NANS64[1], FO.NANS64[0]), 4: (FO.bits(np.inf), FO.NANS64[0]), 5: (FO.NANS64[1], FO.bits(-np.inf)),
            6: (None, None), 7: (FO.NANS64[0], FO.NANS64[0]), 8: (FO.bits(1.0), FO.NANS64[0]), 9: (FO.NANS64[1], FO.bits(1.0)),
            10: (FO.bits(-0.0), FO.bits(-0.0)), 11: (FO.NANS64[3], FO.NANS64[2]),
            12: (FO.bits(-FO.DBL_MAX), FO.bits(FO.DBL_MAX)), 13: (FO.bits(-np.inf), FO.bits(np.inf))}
    for g, (mn, mx) in want.items():
        assert (b(ref[g][0]), b(ref[g][1])) == (mn, mx), g
    assert ref[6][2:] == (None, None, 0) and ref[7][2] == "nan" and ref[7][4] == 24
    assert ref[4][2] == "nan" and ref[13][2] == "nan" and ref[10][2].exact == 0.0 and ref[12][2] == FO.ANY


def test_sum_class_rule():
    assert FO.sum_expect([1.0, math.inf]) == "+inf" and FO.sum_expect([-math.inf, 2.0]) == "-inf"
    assert FO.sum_expect([math.inf, -math.inf]) == "nan" and FO.sum_expect([FO.nan(1), 1.0]) == "nan"
    assert FO.sum_expect([FO.DBL_MAX, FO.DBL_MAX]) == FO.ANY
    FO.check_sum(FO.nan(3), "nan")                    # any NaN's bits pass as the class
    with pytest.raises(AssertionError):
        FO.check_sum(math.inf, "nan")
    with pytest.raises(AssertionError):
        FO.check_sum(1.0 + 1e-9, FO.sum_expect([0.5, 0.5]))


def _oracle_rows(keys, vals, valid, dtype):
    """the oracle's group_by -> {key: (MIN, MAX)} as numpy scalars of dtype (None for NULL)"""
    ok, res = O.group_by([(keys, None)], [(O.A_MIN, (vals, valid), None), (O.A_MAX, (vals, valid), None)])
    mn = O.agg_output_columns(O.A_MIN, res[0], dtype, False)[0]
    mx = O.agg_output_columns(O.A_MAX, res[1], dtype, False)[0]
    out = {}
    for i, k in enumerate(ok[0][0].tolist()):
        v = lambda c: None if (c[1] is not None and not c[1][i]) else c[0][i]
        out[k] = (v(mn), v(mx))
    return out


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_oracle_group_by_min_max_equals_the_reference_in_both_orders(dtype):
    keys, vals, valid = FO.edge_case(np.random.default_rng(5), dtype)
    ref = FO.reference(keys, vals, valid, 48)
    ut = np.uint64 if dtype == np.float64 else np.uint32
    bits = lambda x: None if x is None else int(np.array([x], dtype).view(ut)[0])
    for order in (slice(None), slice(None, None, -1)):
        got = _oracle_rows(keys[order], vals[order], valid[order], dtype)
        assert set(got) == set(ref)
        for g in ref:
            assert (bits(got[g][0]), bits(got[g][1])) == (bits(ref[g][0]), bits(ref[g][1])), (g, got[g], ref[g][:2])


def test_oracle_scalar_min_max_equals_the_reference():
    keys, vals, valid = FO.edge_case(np.random.default_rng(6), np.float64)
    for g in (2, 3, 8, 9, 11, 13):
        m = (keys == g) & valid
        for order in (slice(None), slice(None, None, -1)):
            x = vals[m][order]
            mn, mx = O.scalar_aggregate([(O.A_MIN, (x, None), None), (O.A_MAX, (x, None), None)])
            want = FO.reference(np.zeros(len(x), np.int64), x, None, 1)[0]
            assert (FO.bits(mn[0][0]), FO.bits(mx[0][0])) == (FO.bits(want[0]), FO.bits(want[1])), g


def test_dense_reference_min_max_is_total_order():
    keys, vals, valid = FO.edge_case(np.random.default_rng(7), np.float64)
    cols = [(keys.astype(np.int32), None), (vals, valid)]
    rows = C.reference(cols, [D.INT32, D.FLOAT64], None, [0], [(0, 47)], [(D.AGG_MIN, 1), (D.AGG_MAX, 1)])
    ref = FO.reference(keys, vals, valid, 48)
    b = lambda x: None if x is None else struct.unpack("<Q", struct.pack("<d", x))[0]
    for r in rows:
        assert (b(r[1]), b(r[2])) == (b(None if ref[r[0]][0] is None else float(ref[r[0]][0])),
                                      b(None if ref[r[0]][1] is None else float(ref[r[0]][1]))), r[0]
