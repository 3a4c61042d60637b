"""The plain reference of tests/test_gpu_pipe_column_types.py (partners, kept_rows, gather, left_groups) against the oracle's hash_join
and group_by, on small tables of every key type and every join kind a probe stage runs: Inner, RightSemi, RightAnti, Right, and the
Left / LeftAnti joins of the join-keyed sink.  No GPU: both sides are CPU code."""
import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
import test_gpu_pipe_column_types as PT

STAGE_JOIN = {D.STAGE_INNER: O.J_INNER, D.STAGE_SEMI: O.J_RIGHT_SEMI, D.STAGE_ANTI: O.J_RIGHT_ANTI, D.STAGE_RIGHT: O.J_RIGHT}


def small_case(t, seed):
    rng = np.random.default_rng(seed)
    keys = PT.key_values(t)
    bk = PT.arr(sorted(set(keys[i] for i in rng.integers(0, len(keys), 60))), t)
    pk = PT.arr([keys[i] for i in rng.integers(0, len(keys), 400)], t)
    pv = rng.random(400) >= 0.1
    pay = rng.integers(-1000, 1000, len(bk)).astype(np.int32)
    rid = np.arange(400, dtype=np.int64) * 3 + 2
    return bk, pay, pk, pv, rid


def rows(cols):
    """[(values, valid or None)] -> sorted tuples, None for NULL"""
    n = len(cols[0][0])
    out = []
    for r in range(n):
        out.append(tuple(None if (ok is not None and not ok[r]) else int(v[r]) for v, ok in cols))
    return sorted(out, key=repr)


@pytest.mark.parametrize("kind", sorted(STAGE_JOIN))
@pytest.mark.parametrize("t", PT.KEY_TYPES, ids=PT.KIDS)
def test_probe_stage_reference_equals_the_oracle_join(t, kind):
    bk, pay, pk, pv, rid = small_case(t, 10 * t + kind)
    idx = PT.partners(bk, pk, pv)
    keep = PT.kept_rows(kind, idx)
    mine = [(rid[keep], None), (pk[keep], pv[keep])]
    side, index = [1, 1], [1, 0]
    if kind in (D.STAGE_INNER, D.STAGE_RIGHT):
        v, ok = PT.gather(pay, idx[keep])
        mine.append((v, ok))
        side, index = side + [0], index + [1]
    ref = O.hash_join([(bk, None), (pay, None)], [(pk, pv), (rid, None)], [0], [0], side, index, join_type=STAGE_JOIN[kind])
    assert rows(mine) == rows(ref)
    assert 0 < len(keep) < len(pk) or kind == D.STAGE_RIGHT


@pytest.mark.parametrize("anti", [False, True], ids=["Left", "LeftAnti"])
@pytest.mark.parametrize("t", PT.KEY_TYPES, ids=PT.KIDS)
def test_left_reference_equals_the_oracle_join_and_group_by(t, anti):
    bk, _, pk, pv, rid = small_case(t, 20 * t + anti)
    idx = PT.partners(bk, pk, pv)
    mine = PT.left_groups(bk, idx, rid, anti=anti)
    if anti:
        ref = O.hash_join([(bk, None)], [(pk, pv), (rid, None)], [0], [0], [0], [0], join_type=O.J_LEFT_ANTI)
        assert mine == sorted(int(k) for k in ref[0][0])
        assert 0 < len(mine) < len(bk)
        return
    j = O.hash_join([(bk, None)], [(pk, pv), (rid, None)], [0], [0], [0, 1], [0, 1], join_type=O.J_LEFT)
    keys, res = O.group_by([j[0]], [(O.A_COUNT_STAR, None, None), (O.A_SUM, j[1], None)])
    cnt = O.agg_output_columns(O.A_COUNT_STAR, res[0], np.int64, False)
    total = O.agg_output_columns(O.A_SUM, res[1], np.int64, False)
    assert sorted(mine, key=repr) == rows([keys[0]] + cnt + total)
    assert any(s is None for _, _, s in mine) and any(s is not None for _, _, s in mine)


def test_key_values_hold_each_domain_s_edges_and_no_reserved_key():
    for t in PT.KEY_TYPES:
        lo, hi = PT.dom(t)
        ks = PT.key_values(t)
        assert lo in ks and lo + 199 in ks and hi - 199 in ks
        assert (hi in ks) == (t != D.UINT64)
        assert PT.all_ones(t) not in ks and (PT.all_ones(t) is None or PT.all_ones(t) in PT.key_values(t, reserved=True))
    assert PT.i64((1 << 64) - 1) == -1 and PT.i64(1 << 63) == -(1 << 63) and PT.i64(5) == 5
