"""The CPU restatement of `LikeExpr` (physical-expr/src/expressions/like.rs -> arrow-string `like` / `nlike`) that the GPU LIKE is
checked against, plus seeded generators of strings and patterns.

    s LIKE p is an anchored whole-string match over Unicode code points: `%` matches any run of zero or more code points, `_` exactly
    one, every other character itself; case-sensitive, newline and NUL are ordinary characters.  A NULL string gives NULL for LIKE
    and NOT LIKE; on a non-NULL string NOT LIKE is the negation of LIKE.  Patterns with `\\` are refused by the GPU library and not
    restated here.

The restatement translates the pattern to Python `re` (DOTALL, fullmatch over str, i.e. code points).  tests/test_like_reference.py
cross-checks it against Arrow C++ (`pyarrow.compute.match_like`), an independent implementation of the same definition."""
import re
from typing import List, Optional, Sequence

import numpy as np


def like_regex(pattern: str) -> "re.Pattern":
    assert "\\" not in pattern, "escapes are not restated"
    return re.compile("".join(".*" if c == "%" else "." if c == "_" else re.escape(c) for c in pattern), re.DOTALL)


def like(values: Sequence[Optional[str]], pattern: str, negated: bool = False) -> List[Optional[bool]]:
    rx = like_regex(pattern)
    return [None if v is None else (rx.fullmatch(v) is not None) != negated for v in values]


# ---- generators ----
ALPHABET = ["a", "b", "c", "x", " ", "é", "ß", "€", "中", "😀", "𝄞", "\n", "\x00", "%", "_"]
WORDS = ["special", "requests", "green", "forest", "PROMO", "BRASS", "MEDIUM POLISHED", "Customer", "Complaints", "ing", "é€", "中😀"]


def gen_strings(rng: np.random.Generator, n: int, max_len: int = 24, null_p: float = 0.0) -> List[Optional[str]]:
    """text over 1- to 4-byte characters, newline and NUL, empty strings, and words the patterns look for"""
    out = []
    for _ in range(n):
        if rng.random() < null_p:
            out.append(None)
            continue
        parts, ln = [], int(rng.integers(0, max_len + 1))
        while sum(len(p) for p in parts) < ln:
            parts.append(WORDS[rng.integers(len(WORDS))] if rng.random() < 0.3 else ALPHABET[rng.integers(len(ALPHABET) - 2)])
        out.append("".join(parts))
    return out


FIXED_PATTERNS = ["", "%", "%%", "_", "__", "___", "%_", "_%", "%_%", "a", "ab", "a%", "%a", "%a%", "a%b", "a_b", "_a", "a_", "%special%requests%",
                  "%green%", "PROMO%", "%BRASS", "MEDIUM POLISHED%", "%Customer%Complaints%", "forest%", "é%", "%€", "%中_", "_😀%", "%𝄞",
                  "\n%", "%\x00%", "%a%b%c%", "%x_x%", "_" * 30, "a" * 40 + "%", "%" + "é" * 3 + "%ß%", "%%special%%"]


def gen_pattern(rng: np.random.Generator) -> str:
    """prefix / suffix / contains / multi-segment patterns with `_` at the start, middle and end"""
    k = int(rng.integers(0, 6))
    toks = []
    for _ in range(k):
        r = rng.random()
        if r < 0.25:
            toks.append("%")
        elif r < 0.45:
            toks.append("_")
        elif r < 0.7:
            w = WORDS[rng.integers(len(WORDS))]
            a = int(rng.integers(0, len(w)))
            toks.append(w[a:a + int(rng.integers(1, 4))])
        else:
            toks.append(ALPHABET[rng.integers(len(ALPHABET) - 2)])
    return "".join(toks)
