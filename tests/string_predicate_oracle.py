"""The plain row-by-row restatement of a string column compared with a Utf8 literal (BinaryExpr -> arrow-ord `eq` / `neq` / `lt` /
`lt_eq` / `gt` / `gt_eq`) and of InListExpr with a static list of Utf8 literals, that the GPU string predicates are checked against,
plus a seeded generator of strings near the literals.

    Order is Arrow's for strings: byte-wise lexicographic over the UTF-8 bytes, a proper prefix first; equal means equal length and
    equal bytes.  A NULL string gives NULL.
    IN is SQL's three-valued IN: a NULL string gives NULL; a string found in the list gives True (False for NOT IN); a string found
    nowhere gives NULL when the list holds a NULL, else False (True for NOT IN).

tests/test_string_predicate_reference.py cross-checks this against Arrow C++ (`pyarrow.compute`)."""
from typing import List, Optional, Sequence

import numpy as np

OPS = ["=", "<>", "<", "<=", ">", ">="]


def compare(values: Sequence[Optional[str]], op: str, literal: str) -> List[Optional[bool]]:
    b = literal.encode("utf-8")
    out = []
    for v in values:
        if v is None:
            out.append(None)
            continue
        s = v.encode("utf-8")
        out.append({"=": s == b, "<>": s != b, "<": s < b, "<=": s <= b, ">": s > b, ">=": s >= b}[op])
    return out


def in_list(values: Sequence[Optional[str]], items: Sequence[Optional[str]], negated: bool = False) -> List[Optional[bool]]:
    found_set = {x.encode("utf-8") for x in items if x is not None}
    has_null = any(x is None for x in items)
    out = []
    for v in values:
        if v is None:
            out.append(None)
        elif v.encode("utf-8") in found_set:
            out.append(not negated)
        elif has_null:
            out.append(None)
        else:
            out.append(negated)
    return out


# ---- generator ----
LITERALS = ["", "a", "ab", "abc", "MAIL", "SHIP", "BUILDING", "Brand#12", "SM CASE", "DELIVER IN PERSON", "é", "éa", "中😀", "abcdefghijkl",
            "abcdefghijklm", "special requests and more", "\x00", "a\x00", "zz"]


def gen_strings(rng: np.random.Generator, n: int, null_p: float = 0.0) -> List[Optional[str]]:
    """strings at and around the literals: the literals, their proper prefixes, one byte more or less at the end, a changed byte, long
    strings, multi-byte UTF-8, empty strings and NULLs"""
    out = []
    for _ in range(n):
        if rng.random() < null_p:
            out.append(None)
            continue
        w = LITERALS[rng.integers(len(LITERALS))]
        r = rng.random()
        if r < 0.3:
            out.append(w)
        elif r < 0.45:
            out.append(w[:int(rng.integers(0, len(w) + 1))])
        elif r < 0.6:
            out.append(w + "abcé\x00z"[rng.integers(6)])
        elif r < 0.75 and w:
            i = int(rng.integers(len(w)))
            out.append(w[:i] + chr(max(1, ord(w[i]) + int(rng.integers(-1, 2)))) + w[i + 1:])
        elif r < 0.85:
            out.append(w * int(rng.integers(2, 6)))
        else:
            out.append("".join("aé€😀 Z"[k] for k in rng.integers(0, 6, int(rng.integers(0, 20)))))
    return out
