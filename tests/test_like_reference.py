"""The CPU restatement of LikeExpr (tests/like_oracle.py) against Arrow C++'s `match_like`, an independent implementation of the same
definition on patterns without `\\`: text of 1- to 4-byte characters with newline, NUL and empty strings; exact, empty, `%`, `%%`,
prefix, suffix, contains and multi-segment patterns; `_` at the start, middle and end, all-`_` patterns and patterns longer than any
string."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from like_oracle import FIXED_PATTERNS, gen_pattern, gen_strings, like


def arrow_like(values, pattern, negated=False):
    got = pc.match_like(pa.array(values, pa.string()), pattern).to_pylist()
    return [None if g is None else g != negated for g in got]


def test_text_covers_every_width_newline_nul_and_empty():
    vals = gen_strings(np.random.default_rng(0), 2000, null_p=0.05)
    widths = {len(c.encode()) for v in vals if v for c in v}
    assert widths == {1, 2, 3, 4}
    assert any(v == "" for v in vals) and any(v and "\n" in v for v in vals) and any(v and "\x00" in v for v in vals)
    assert any(v is None for v in vals)


@pytest.mark.parametrize("negated", [False, True])
def test_fixed_patterns_agree_with_arrow(negated):
    vals = gen_strings(np.random.default_rng(1), 1500, null_p=0.05) + ["", "a", "ab", "special requests", "PROMO BRUSHED", "é€中😀𝄞", "\n\x00"]
    for p in FIXED_PATTERNS:
        assert like(vals, p, negated) == arrow_like(vals, p, negated), repr(p)


def test_generated_patterns_agree_with_arrow():
    rng = np.random.default_rng(2)
    vals = gen_strings(rng, 800, null_p=0.05)
    pats = [gen_pattern(rng) for _ in range(300)]
    assert any(p.startswith("_") for p in pats) and any(p.endswith("_") for p in pats) and any("%" in p[1:-1] for p in pats)
    for p in pats:
        assert like(vals, p) == arrow_like(vals, p), repr(p)


def test_patterns_longer_than_any_string():
    vals = gen_strings(np.random.default_rng(3), 300, max_len=10)
    for p in ("_" * 40, "a" * 40, "%" + "b" * 40 + "%", "_" * 30 + "%"):
        exp = like(vals, p)
        assert exp == arrow_like(vals, p) and not any(exp), repr(p)


def test_code_points_not_bytes():
    assert like(["é", "€", "😀", "ab", "a"], "_") == [True, True, True, False, True]
    assert like(["aéb", "a€b", "a😀b", "axyb"], "a_b") == [True, True, True, False]
    assert like(["x\ny", "x\x00y", None], "x_y", negated=True) == [False, False, None]
