"""The exact checks and the text generator of scripts/string_predicate_timing.py on tiny host data (no GPU): the chunked summary equals
the summary of the whole mask and rejects a changed count and a moved match, the generated rows are the column's values, pyarrow's
evaluation agrees with the row-by-row restatement, and the computed DRAM floors."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import string_predicate_timing as T  # noqa: E402
from string_predicate_oracle import compare, in_list  # noqa: E402


def test_chunked_summary_equals_the_whole_mask():
    m = np.random.default_rng(0).random(1000) < 0.2
    for step in (1000, 300, 7):
        assert T.chunked_summary((s, m[s:s + step]) for s in range(0, len(m), step)) == T.L.mask_summary(m)
    ref = T.L.mask_summary(m)
    moved = m.copy(); moved[np.flatnonzero(m)[0]] = False; moved[np.flatnonzero(~m)[0]] = True
    extra = m.copy(); extra[np.flatnonzero(~m)[-1]] = True
    for bad in (moved, extra):
        with pytest.raises(AssertionError):
            T.L.check_mask("x", T.chunked_summary([(0, bad)]), ref)


def test_generated_rows_and_the_arrow_masks():
    codes, offs, data = T.value_text(np.random.default_rng(1), 5000, T.MODES)
    arr = T.L.utf8_array(offs, data, large=True)
    vals = arr.to_pylist()
    assert vals == [T.MODES[c] for c in codes] and offs[-1] == len(data)
    assert T.arrow_mask(arr, ("in", ["MAIL", "SHIP"])).tolist() == in_list(vals, ["MAIL", "SHIP"])
    for op in ("=", "<>", "<", "<=", ">", ">="):
        assert T.arrow_mask(arr, (op, "RAIL")).tolist() == compare(vals, op, "RAIL")
    share = T.arrow_mask(arr, ("in", ["MAIL", "SHIP"])).mean()
    assert 0.25 < share < 0.32
    assert len(T.CONTAINERS) == 40 and len(T.BRANDS) == 25 and "Brand#12" in T.BRANDS


def test_floors():
    n = 600_000_000
    assert T.floor_bytes("utf8_view", n, 0) == 17 * n
    assert T.floor_bytes("dictionary_codes", n, 0) == 5 * n
    assert T.floor_bytes("utf8_blocks", n, 2_570_000_000, 150) == 4 * (n + 150) + 2_570_000_000 + n
