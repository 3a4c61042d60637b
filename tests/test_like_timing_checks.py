"""The exact checks and the text generator of scripts/like_timing.py on tiny host data (no GPU): the summary of a repeated block equals
the summary of the materialised mask, the mask check rejects a changed count and a moved match, and the generated comments have the
TPC-H lengths and a '%special%requests%' match share of about 1-2 %."""
import os
import sys

import numpy as np
import pyarrow.compute as pc
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import like_timing as T  # noqa: E402


def test_tiled_summary_equals_the_materialised_mask():
    m = np.random.default_rng(0).random(1000) < 0.05
    for n in (1000, 2500, 3000, 999):
        assert T.tiled_summary(m, n) == T.mask_summary(np.resize(m, n))


def test_mask_check_rejects_differences():
    m = np.zeros(100, bool); m[[3, 50, 97]] = True
    ref = T.mask_summary(m)
    assert T.check_mask("x", T.mask_summary(m.copy()), ref) == ref
    moved = m.copy(); moved[50], moved[51] = False, True
    extra = m.copy(); extra[0] = True
    for bad in (moved, extra):
        with pytest.raises(AssertionError):
            T.check_mask("x", T.mask_summary(bad), ref)


def test_generated_comments():
    offs, data = T.word_text(np.random.default_rng(1), 200_000, T.WORDS, T.comment_weights(), 19, 78)
    lens = np.diff(offs)
    assert lens.min() >= 19 and lens.max() <= 78 and 47 < lens.mean() < 51 and offs[-1] == len(data)
    share = np.asarray(pc.match_like(T.utf8_array(offs, data), "%special%requests%")).mean()
    assert 0.01 <= share <= 0.02, share
    assert len(T.TYPES) == 150 and sum(t.startswith("PROMO") for t in T.TYPES) == 25
