"""The CPU restatement of string comparisons and IN lists (tests/string_predicate_oracle.py) on hand-picked cases, and cross-checked
against Arrow C++ (pyarrow.compute) on generated data.  No GPU."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from string_predicate_oracle import LITERALS, OPS, compare, gen_strings, in_list

ARROW = {"=": pc.equal, "<>": pc.not_equal, "<": pc.less, "<=": pc.less_equal, ">": pc.greater, ">=": pc.greater_equal}


def test_order_is_bytewise_with_prefixes_first():
    vals = ["", "a", "ab", "abc", "b", "B", None, "é", "z", "a\x00"]
    assert compare(vals, "<", "ab") == [True, True, False, False, False, True, None, False, False, True]
    assert compare(vals, "=", "ab") == [False, False, True, False, False, False, None, False, False, False]
    assert compare(vals, ">=", "") == [True] * 6 + [None] + [True] * 3
    assert compare(["é"], ">", "z") == [True]                  # 0xC3 > 0x7A: UTF-8 bytes, which is code-point order
    assert compare(["中😀", "中"], "<", "中😀") == [False, True]


def test_three_valued_in():
    vals = ["MAIL", "SHIP", "AIR", None, ""]
    assert in_list(vals, ["MAIL", "SHIP"]) == [True, True, False, None, False]
    assert in_list(vals, ["MAIL", "SHIP"], negated=True) == [False, False, True, None, True]
    assert in_list(vals, ["MAIL", None]) == [True, None, None, None, None]
    assert in_list(vals, ["MAIL", None], negated=True) == [False, None, None, None, None]
    assert in_list(vals, [None]) == [None] * 5
    assert in_list(vals, [""]) == [False, False, False, None, True]
    assert in_list(["é", "e"], ["é"]) == [True, False]


def test_compare_matches_arrow():
    rng = np.random.default_rng(1)
    vals = gen_strings(rng, 4000, null_p=0.1)
    for t in (pa.string(), pa.large_string()):               # Arrow C++ has no comparison kernel for string_view
        arr = pa.array(vals, t)
        for lit in LITERALS:
            for op in OPS:
                exp = ARROW[op](arr, pa.scalar(lit, t)).to_pylist()
                assert compare(vals, op, lit) == exp, (t, op, lit)


def test_in_list_matches_arrow():
    rng = np.random.default_rng(2)
    vals = gen_strings(rng, 4000, null_p=0.1)
    arr = pa.array(vals)
    for k in range(40):
        items = list(rng.choice(LITERALS, int(rng.integers(1, 8))))
        exp = pc.is_in(arr, value_set=pa.array(items)).to_pylist()
        got = in_list(vals, items)
        # pyarrow's is_in gives False for a NULL input (skip_nulls); SQL's IN gives NULL
        assert [g for g, v in zip(got, vals) if v is not None] == [e for e, v in zip(exp, vals) if v is not None], items
        assert all(g is None for g, v in zip(got, vals) if v is None)
        assert in_list(vals, items, negated=True) == [None if g is None else not g for g in got]
