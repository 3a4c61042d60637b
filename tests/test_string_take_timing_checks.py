"""The checks, generators and floor arithmetic of scripts/string_take_timing.py on tiny host data (no GPU): the per-row byte sums equal
a row-by-row restatement and the sum check refuses a changed sum, the sector counts of random and nondecreasing ranges, the Utf8View layout of a
block against pyarrow's, the c_name text, and the floors."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import string_take_timing as T  # noqa: E402


def test_row_sums_equal_the_restatement():
    offs, data = T.L.word_text(np.random.default_rng(0), 3000, T.L.WORDS, T.L.comment_weights(), 0, 40)
    vals = T.L.utf8_array(offs, data, large=True).to_pylist()
    exp = np.array([sum(v.encode()) for v in vals], np.uint64)
    assert np.array_equal(T.row_sums(offs, data), exp)
    assert np.array_equal(T.row_sums(offs[100:201], data), exp[100:200])
    T.check_sum("x", int(exp.sum()), int(T.row_sums(offs, data).sum()))
    with pytest.raises(AssertionError):
        T.check_sum("x", int(exp.sum()) + 1, int(exp.sum()))


def test_sector_bytes():
    assert T.sector_bytes([0], [32]) == 32 and T.sector_bytes([31], [2]) == 64 and T.sector_bytes([5], [0]) == 0
    assert T.sector_bytes([0, 0, 40], [8, 8, 8]) == 96                     # per range: a random gather reads each one
    assert T.sector_bytes([0, 8, 40, 70], [8, 8, 8, 40], distinct=True) == 4 * 32   # sectors 0, 1, 2, 3 once
    rng = np.random.default_rng(1)
    starts = np.sort(rng.integers(0, 5000, 400)); lens = rng.integers(0, 60, 400)
    touched = set()
    for s, n in zip(starts, lens):
        touched |= set(range(s // 32, (s + n - 1) // 32 + 1)) if n else set()
    assert T.sector_bytes(starts, lens, distinct=True) == 32 * len(touched)


def test_block_views_match_pyarrow():
    vals = ["", "short", "exactly12byt", "thirteen byte", "a much longer string than twelve", "ß日本"]
    offs = np.concatenate([[0], np.cumsum([len(v.encode()) for v in vals])]).astype(np.int64)
    data = np.frombuffer("".join(vals).encode(), np.uint8)
    v = T.block_views(offs, data)
    ref = np.frombuffer(pa.array(vals, pa.string_view()).buffers()[1], np.uint32).reshape(-1, 4)
    inline = v[:, 0] <= 12
    assert np.array_equal(v[inline], ref[inline])
    assert np.array_equal(v[~inline, :2], ref[~inline, :2]) and np.array_equal(v[~inline, 3], offs[:-1][~inline].astype(np.uint32))


def test_name_text():
    offs, data = T.name_text(3)
    assert T.L.utf8_array(offs, data).to_pylist() == ["Customer#000000001", "Customer#000000002", "Customer#000000003"]


def test_floors():
    n = 150_000_000
    assert T.floor_bytes("utf8_view", n, 4, 32 * n, 0, 0) == 4 * n + 32 * n + 16 * n + n // 8
    assert T.floor_bytes("large_utf8", n, 4, 32 * n, 7_000, 5_000) == 4 * n + 32 * n + 7_000 + 8 * (n + 1) + 5_000 + n // 8
    assert T.floor_bytes("large_utf8", 9, 8, 0, 0, 0) == 72 + 80 + 2
