"""oracle.py — Python face of the CPU restatement oracle (TEST INFRASTRUCTURE ONLY).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product path (datafusion_b200/) never does.

* join / group-by / repartition: ctypes over oracle/liboracle.so (oracle.c — each function cites the
  reference file:line it restates).
* expressions / FilterExec: numpy restatement of PhysicalExpr::evaluate
  (physical-expr/src/expressions/binary.rs:536-676, physical-expr-common/src/datum.rs:36-105) and
  filter_record_batch semantics (physical-plan/src/filter.rs:1339-1445).

Columns are (values: np.ndarray, valid: np.ndarray[bool] | None) pairs.
PARITY UNPINNED for hash VALUES only (foldhash 0.2 is not restated; outputs do not depend on it).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "liboracle.so")
Col = Tuple[np.ndarray, Optional[np.ndarray]]

J_INNER, J_LEFT, J_RIGHT, J_FULL, J_LEFT_SEMI, J_RIGHT_SEMI, J_LEFT_ANTI, J_RIGHT_ANTI, J_LEFT_MARK, J_RIGHT_MARK = range(10)
A_SUM, A_COUNT, A_MIN, A_MAX, A_AVG, A_COUNT_STAR = range(1, 7)


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "-s"])


_lib = None


class _JoinResult(C.Structure):
    _fields_ = [("build_idx", C.POINTER(C.c_int64)), ("probe_idx", C.POINTER(C.c_int64)), ("mark", C.POINTER(C.c_int8)),
                ("n", C.c_int64), ("used_array_map", C.c_int)]


class _AggIn(C.Structure):
    _fields_ = [("func", C.c_int), ("is_float", C.c_int), ("arg", C.c_void_p), ("arg_valid", C.c_void_p), ("arg2", C.c_void_p),
                ("arg2_valid", C.c_void_p), ("filter", C.c_void_p), ("filter_valid", C.c_void_p)]


class _GroupResult(C.Structure):
    _fields_ = [("nkeys", C.c_int), ("naggs", C.c_int), ("ngroups", C.c_int64), ("key_vals", C.POINTER(C.POINTER(C.c_int64))),
                ("key_valid", C.POINTER(C.POINTER(C.c_uint8))), ("out_i", C.POINTER(C.c_int64) * 8), ("out_f", C.POINTER(C.c_double) * 8),
                ("out_c", C.POINTER(C.c_uint64) * 8), ("out_valid", C.POINTER(C.c_uint8) * 8)]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        _lib = C.CDLL(LIB)
        _lib.oracle_bench_join.restype = C.c_double
        _lib.oracle_bench_groupby.restype = C.c_double
        _lib.oracle_version.restype = C.c_char_p
    return _lib


_PAIR_FILTER = C.CFUNCTYPE(C.c_int, C.c_int64, C.c_int64)


def _i64(a) -> np.ndarray:
    a = np.asarray(a)
    if a.dtype == np.bool_:
        return a.astype(np.int64)
    if a.dtype.kind == "f":
        return np.ascontiguousarray(a.astype(np.float64)).view(np.int64)
    if a.dtype == np.uint64:
        return np.ascontiguousarray(a).view(np.int64)
    return np.ascontiguousarray(a.astype(np.int64))


def _u8(v: Optional[np.ndarray]):
    return None if v is None else np.ascontiguousarray(np.asarray(v, dtype=bool).astype(np.uint8))


def _ptr_array(arrs, ctype):
    PT = C.POINTER(ctype)
    out = (PT * max(len(arrs), 1))()
    for i, a in enumerate(arrs):
        out[i] = a.ctypes.data_as(PT) if a is not None else PT()
    return out


# ---------------------------------------------------------------------------------------------
# hash join
# ---------------------------------------------------------------------------------------------
def hash_join_indices(build_keys: Sequence[Col], probe_keys: Sequence[Col], join_type: int = J_INNER, null_equals_null: bool = False,
                      batch_size: int = 8192, phj_threshold: int = 1024, phj_density: float = 0.15, force_collisions: bool = False,
                      build_batch_rows: Optional[Sequence[int]] = None, probe_batch_rows: Optional[Sequence[int]] = None,
                      key_is_integer: bool = True, pair_filter=None, null_aware: bool = False):
    """(build_idx, probe_idx, mark, used_array_map): -1 = NULL index.  Order = the reference's emission order."""
    L = lib()
    nk = len(build_keys)
    nb = len(build_keys[0][0])
    npr = len(probe_keys[0][0])
    bk = [_i64(k[0]) for k in build_keys]
    pk = [_i64(k[0]) for k in probe_keys]
    bv = [_u8(k[1]) for k in build_keys]
    pv = [_u8(k[1]) for k in probe_keys]
    bbr = np.array(build_batch_rows if build_batch_rows is not None else [nb], np.int64)
    pbr = np.array(probe_batch_rows if probe_batch_rows is not None else [npr], np.int64)
    assert bbr.sum() == nb and pbr.sum() == npr
    res = _JoinResult()
    L.oracle_hash_join(C.c_int(nk), _ptr_array(bk, C.c_int64), _ptr_array(bv, C.c_uint8) if any(v is not None for v in bv) else None,
                       C.c_int64(nb), bbr.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(bbr)),
                       _ptr_array(pk, C.c_int64), _ptr_array(pv, C.c_uint8) if any(v is not None for v in pv) else None, C.c_int64(npr),
                       pbr.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(len(pbr)), C.c_int(join_type), C.c_int(1 if null_equals_null else 0),
                       C.c_int64(batch_size), C.c_int64(phj_threshold), C.c_double(phj_density), C.c_int(1 if force_collisions else 0),
                       C.c_int(1 if key_is_integer else 0), C.byref(res), None,
                       _PAIR_FILTER(lambda b, p: 1 if pair_filter(int(b), int(p)) else 0) if pair_filter is not None else None,
                       C.c_int(1 if null_aware else 0))
    n = res.n
    if n == 0:
        b, p, m = np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, bool)
    else:
        b = np.ctypeslib.as_array(res.build_idx, (n,)).copy()
        p = np.ctypeslib.as_array(res.probe_idx, (n,)).copy()
        m = np.ctypeslib.as_array(res.mark, (n,)).copy().astype(bool)
    used = bool(res.used_array_map)
    L.oracle_free_join_result(C.byref(res))
    return b, p, m, used


def _step(fn, head_args, probe_n, limit, offset):
    cap = max(int(limit), 1) + 8
    pi = np.zeros(cap * 4 + probe_n + 8, np.int64); bi = np.zeros_like(pi)
    n = C.c_int64(0)
    off = np.array([offset[0], 0 if offset[1] is None else 1, 0 if offset[1] is None else offset[1]], np.int64)
    nxt = np.zeros(3, np.int64)
    has = fn(*head_args, C.c_int64(limit), off.ctypes.data_as(C.POINTER(C.c_int64)), pi.ctypes.data_as(C.POINTER(C.c_int64)),
             bi.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(n), nxt.ctypes.data_as(C.POINTER(C.c_int64)))
    nx = None if not has else (int(nxt[0]), int(nxt[2]) if nxt[1] else None)
    return pi[:n.value].tolist(), bi[:n.value].tolist(), nx


def array_map_step(build: Col, min_val: int, max_val: int, probe: Col, limit: int, offset=(0, None)):
    """one ArrayMap::get_matched_indices_with_limit_offset call -> (probe_indices, build_indices, next MapOffset or None)"""
    L = lib()
    b, p = _i64(build[0]), _i64(probe[0])
    bv, pv = _u8(build[1]), _u8(probe[1])
    args = (b.ctypes.data_as(C.POINTER(C.c_int64)), bv.ctypes.data_as(C.POINTER(C.c_uint8)) if bv is not None else None, C.c_int64(len(b)),
            C.c_uint64(min_val & (2**64 - 1)), C.c_uint64(max_val & (2**64 - 1)), p.ctypes.data_as(C.POINTER(C.c_int64)),
            pv.ctypes.data_as(C.POINTER(C.c_uint8)) if pv is not None else None, C.c_int64(len(p)))
    return _step(L.oracle_array_map_step, args, len(p), limit, offset)


def join_hash_map_step(build_hashes, probe_hashes, valid_keys, limit: int, offset=(0, None)):
    """one JoinHashMap::get_matched_indices_with_limit_offset call on raw hash values (build rows inserted in forward order)"""
    L = lib()
    b = np.ascontiguousarray(np.asarray(build_hashes, np.uint64)); p = np.ascontiguousarray(np.asarray(probe_hashes, np.uint64))
    v = _u8(valid_keys)
    args = (b.ctypes.data_as(C.POINTER(C.c_uint64)), C.c_int64(len(b)), p.ctypes.data_as(C.POINTER(C.c_uint64)),
            v.ctypes.data_as(C.POINTER(C.c_uint8)) if v is not None else None, C.c_int64(len(p)))
    return _step(L.oracle_join_hash_map_step, args, len(p), limit, offset)


def equal_rows(left_idx, right_idx, left_keys: Sequence[Col], right_keys: Sequence[Col], null_equals_null: bool = False):
    """equal_rows_arr (joins/utils.rs:2191-2257): filter candidate (build, probe) index pairs by key equality"""
    L = lib()
    L.oracle_equal_rows.restype = C.c_int64
    li = np.ascontiguousarray(np.asarray(left_idx, np.int64)).copy(); ri = np.ascontiguousarray(np.asarray(right_idx, np.int64)).copy()
    lk = [_i64(k[0]) for k in left_keys]; rk = [_i64(k[0]) for k in right_keys]
    lv = [_u8(k[1]) for k in left_keys]; rv = [_u8(k[1]) for k in right_keys]
    n = L.oracle_equal_rows(C.c_int(len(lk)), _ptr_array(lk, C.c_int64) if lk else None, _ptr_array(lv, C.c_uint8) if lk else None,
                            _ptr_array(rk, C.c_int64) if rk else None, _ptr_array(rv, C.c_uint8) if rk else None, C.c_int(1 if null_equals_null else 0),
                            li.ctypes.data_as(C.POINTER(C.c_int64)), ri.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(len(li)))
    return li[:n].tolist(), ri[:n].tolist()


def take(col: Col, idx: np.ndarray) -> Col:
    """arrow `take` with nullable indices (-1 -> NULL)"""
    vals, valid = col
    vals = np.asarray(vals)
    safe = np.where(idx >= 0, idx, 0)
    out = vals[safe] if len(vals) else np.zeros(len(idx), vals.dtype)
    ov = idx >= 0
    if valid is not None and len(vals):
        ov = ov & np.asarray(valid, bool)[safe]
    out = np.where(ov, out, np.zeros((), vals.dtype)) if len(idx) else out
    return out, (None if ov.all() else ov)


def hash_join(build: Sequence[Col], probe: Sequence[Col], on_build: Sequence[int], on_probe: Sequence[int], out_side: Sequence[int],
              out_index: Sequence[int], **kw) -> List[Col]:
    """Materialised join output (build_batch_from_indices, joins/utils.rs:1332-1387)."""
    if "filter" in kw:   # (col_side, col_index, nodes): evaluated per candidate pair with the numpy expression oracle
        fs, fi, nodes = kw.pop("filter")

        def pf(brow, prow):
            cols = []
            for sd, ix in zip(fs, fi):
                v, val = (build if sd == 0 else probe)[ix]
                r = brow if sd == 0 else prow
                cols.append((np.asarray(v)[r:r + 1], None if val is None else np.asarray(val, bool)[r:r + 1]))
            rv, rvalid = eval_expr(cols, nodes)
            return bool(rv[0]) and (rvalid is None or bool(rvalid[0]))
        kw["pair_filter"] = pf
    b, p, m, _ = hash_join_indices([build[i] for i in on_build], [probe[i] for i in on_probe], **kw)
    jt = kw.get("join_type", J_INNER)
    out = []
    for side, ix in zip(out_side, out_index):
        if side == 2:
            out.append((m.copy(), None))
        elif side == 0:
            out.append(take(build[ix], b))
        else:
            out.append(take(probe[ix], p))
    return out


# ---------------------------------------------------------------------------------------------
# group by
# ---------------------------------------------------------------------------------------------
def group_by(keys: Sequence[Col], aggs: Sequence[tuple], merge: bool = False, batch_size: int = 8192, force_collisions: bool = False):
    """aggs: [(func, arg: Col | None, filter: Col | None)]   (merge: [(func, state_col(s)...)] with arg = count/sum state;
    AVG merge passes arg=(count col) and a 4th element (sum col)).
    Returns (group key columns in FIRST-SEEN order, [per aggregate dict(i=, f=, c=, valid=)]).
    A SUM over a Decimal128 column (`Dec`) is i128 add_wrapping (sum.rs:316 with Decimal128Type): restated as three 64-bit wrapping sums over
    the limbs lo & 0xffffffff, lo >> 32 and hi, recombined mod 2^128; its result dict carries dec=Dec(..., min(38, p + 10), s)
    (Sum::return_type, sum.rs:247-249; merge keeps the state's own type)."""
    if any(len(ag) > 1 and ag[1] is not None and isinstance(ag[1][0], Dec) for ag in aggs):
        flat, where = [], []
        for ag in aggs:
            arg = ag[1] if len(ag) > 1 else None
            if arg is not None and isinstance(arg[0], Dec):
                d, val = arg
                filt = ag[2] if len(ag) > 2 else None
                if ag[0] == A_SUM:
                    u = [int(x) % (1 << 128) for x in d]
                    limbs = [np.array([x & 0xffffffff for x in u], np.int64), np.array([(x >> 32) & 0xffffffff for x in u], np.int64),
                             np.array([x >> 64 for x in u], np.uint64).view(np.int64)]
                    where.append(("dec", len(flat), d.p if merge else min(38, d.p + 10), d.s))
                    flat += [(A_SUM, (l, val), filt) for l in limbs]
                elif ag[0] in (A_COUNT, A_COUNT_STAR):
                    where.append(("one", len(flat)))
                    flat.append((ag[0], (np.zeros(len(d), np.int64), val), filt))
                else:
                    raise NotImplementedError("oracle: only SUM / COUNT over Decimal128")
            else:
                where.append(("one", len(flat)))
                flat.append(ag)
        out_keys, res = group_by(keys, flat, merge=merge, batch_size=batch_size, force_collisions=force_collisions)
        out = []
        for w in where:
            if w[0] == "one":
                out.append(res[w[1]])
            else:
                _, at, pp, ss = w
                l0, l1, hi = res[at]["i"], res[at + 1]["i"], res[at + 2]["i"].view(np.uint64)
                tot = [(int(a) + (int(b) << 32) + (int(c) << 64)) % (1 << 128) for a, b, c in zip(l0, l1, hi)]
                tot = [x - (1 << 128) if x >= (1 << 127) else x for x in tot]
                out.append(dict(dec=Dec(tot, pp, ss), valid=res[at]["valid"], i=None, f=None, c=None))
        return out_keys, out
    L = lib()
    nk = len(keys)
    n = len(keys[0][0]) if nk else 0
    kv = [_i64(k[0]) for k in keys]
    kval = [_u8(k[1]) for k in keys]
    kfloat = np.array([1 if np.asarray(k[0]).dtype.kind == "f" else 0 for k in keys], np.int32)
    keep = []
    ains = (_AggIn * max(len(aggs), 1))()
    for i, ag in enumerate(aggs):
        func, arg, filt = ag[0], ag[1], ag[2] if len(ag) > 2 else None
        a = ains[i]
        a.func = func
        if arg is not None:
            vals = np.asarray(arg[0])
            if vals.dtype.kind == "f":
                av = np.ascontiguousarray(vals.astype(np.float64)); a.is_float = 1
            elif vals.dtype == np.uint64:
                av = np.ascontiguousarray(vals); a.is_float = 2
            else:
                av = np.ascontiguousarray(vals.astype(np.int64)); a.is_float = 0
            vv = _u8(arg[1])
            keep += [av, vv]
            a.arg = av.ctypes.data
            a.arg_valid = vv.ctypes.data if vv is not None else None
        if len(ag) > 3 and ag[3] is not None:  # AVG merge: sum column
            sv = np.ascontiguousarray(np.asarray(ag[3][0]).astype(np.float64)); svv = _u8(ag[3][1])
            keep += [sv, svv]
            a.arg2 = sv.ctypes.data
            a.arg2_valid = svv.ctypes.data if svv is not None else None
            a.is_float = 1
        if filt is not None:
            fv = _u8(filt[0]); fvv = _u8(filt[1])
            keep += [fv, fvv]
            a.filter = fv.ctypes.data
            a.filter_valid = fvv.ctypes.data if fvv is not None else None
    res = _GroupResult()
    L.oracle_group_by(C.c_int(nk), _ptr_array(kv, C.c_int64), _ptr_array(kval, C.c_uint8) if any(v is not None for v in kval) else None,
                      kfloat.ctypes.data_as(C.POINTER(C.c_int)), C.c_int64(n), C.c_int(len(aggs)), ains, C.c_int(1 if merge else 0),
                      C.c_int64(batch_size), C.c_int(1 if force_collisions else 0), C.byref(res))
    ng = res.ngroups
    out_keys = []
    for c in range(nk):
        vals = np.ctypeslib.as_array(res.key_vals[c], (max(ng, 1),))[:ng].copy()
        valid = np.ctypeslib.as_array(res.key_valid[c], (max(ng, 1),))[:ng].copy().astype(bool)
        src = np.asarray(keys[c][0])
        if src.dtype.kind == "f":
            vals = vals.view(np.float64).astype(src.dtype)
        elif src.dtype == np.bool_:
            vals = vals.astype(bool)
        else:
            vals = vals.astype(src.dtype) if src.dtype != np.uint64 else vals.view(np.uint64)
        out_keys.append((vals, None if valid.all() else valid))
    out_aggs = []
    for a in range(len(aggs)):
        out_aggs.append(dict(
            i=np.ctypeslib.as_array(res.out_i[a], (max(ng, 1),))[:ng].copy(),
            f=np.ctypeslib.as_array(res.out_f[a], (max(ng, 1),))[:ng].copy(),
            c=np.ctypeslib.as_array(res.out_c[a], (max(ng, 1),))[:ng].copy(),
            valid=np.ctypeslib.as_array(res.out_valid[a], (max(ng, 1),))[:ng].copy().astype(bool)))
    L.oracle_free_group_result(C.byref(res))
    return out_keys, out_aggs


def agg_output_columns(func: int, r: dict, arg_dtype, state: bool) -> List[Col]:
    """Shape one aggregate's oracle result like AggregateExec's output (state() or evaluate())."""
    def nv(v):
        return None if v.all() else v
    if func == A_SUM and r.get("dec") is not None:
        return [(r["dec"], nv(r["valid"]))]
    if func == A_SUM:
        if np.dtype(arg_dtype).kind == "f":
            return [(r["f"], nv(r["valid"]))]
        if np.dtype(arg_dtype).kind == "u":
            return [(r["i"].view(np.uint64), nv(r["valid"]))]
        return [(r["i"], nv(r["valid"]))]
    if func in (A_COUNT, A_COUNT_STAR):
        return [(r["c"].astype(np.int64), None)]
    if func in (A_MIN, A_MAX):
        if np.dtype(arg_dtype).kind == "f":
            return [(r["f"].astype(arg_dtype), nv(r["valid"]))]
        if np.dtype(arg_dtype) == np.uint64:
            return [(r["i"].view(np.uint64), nv(r["valid"]))]
        return [(r["i"].astype(arg_dtype), nv(r["valid"]))]
    if func == A_AVG:
        if state:
            return [(r["c"].astype(np.uint64), None), (r["f"], None)]
        with np.errstate(divide="ignore", invalid="ignore"):
            return [(np.where(r["c"] > 0, r["f"] / np.maximum(r["c"], 1), 0.0), nv(r["c"] > 0))]
    raise ValueError(func)


def expand_grouping_sets(keys: Sequence[Col], masks: Sequence[Sequence[bool]]):
    """PhysicalGroupBy with grouping sets (aggregates/mod.rs:368-560 `PhysicalGroupBy { expr, null_expr, groups }`; evaluate_group_by
    :3149-3192): every input row is evaluated once per grouping set, with the group columns the set masks out replaced by NULL and an
    extra `__grouping_id` key (UInt8 for <= 8 group columns) whose bit (n-1-i) is set when column i is NULLed.
    Returns (expanded key columns + the grouping-id column, number of copies)."""
    n = len(keys[0][0])
    nk = len(keys)
    out = []
    for c in range(nk):
        vals = np.concatenate([np.asarray(keys[c][0]) for _ in masks])
        valid = np.concatenate([(np.zeros(n, bool) if m[c] else (np.ones(n, bool) if keys[c][1] is None else np.asarray(keys[c][1], bool))) for m in masks])
        out.append((vals, None if valid.all() else valid))
    gid = np.concatenate([np.full(n, sum((1 << (nk - 1 - i)) for i in range(nk) if m[i]), np.uint8) for m in masks])
    out.append((gid, None))
    return out, len(masks)


def partial_aggregate_with_skip(key_batches: Sequence[Sequence[Col]], arg_batches: Sequence[Col], func: int,
                                probe_rows_threshold: int = 100_000, probe_ratio_threshold: float = 0.8):
    """AggregateMode::Partial with the skip-partial-aggregation probe (aggregates/skip_partial.rs:69-110, the streams'
    SkippingAggregation state, convert_batch_to_state partial_table.rs:199-238), for ONE aggregate (SUM or COUNT).

    After every aggregated batch the probe adds the batch's rows and takes the current group count; once input_rows >=
    probe_rows_threshold it decides `should_skip = groups / rows > ratio` (and keeps re-deciding on later batches until it says
    skip).  On skip the stream emits all current groups, then every later batch is converted row by row into a state row
    (COUNT: 1 / 0 by validity, SUM: the value).  Returns (key columns, state column) in emission order."""
    assert func in (A_SUM, A_COUNT)
    nk = len(key_batches[0])
    out_keys = [[] for _ in range(nk)]; out_kvalid = [[] for _ in range(nk)]
    out_state, out_svalid = [], []
    rows_seen, should_skip, agg_upto = 0, False, 0

    def emit_groups(upto):
        if upto == 0:
            return
        keys = [(np.concatenate([np.asarray(b[c][0]) for b in key_batches[:upto]]),
                 None if all(b[c][1] is None for b in key_batches[:upto]) else np.concatenate([np.ones(len(b[c][0]), bool) if b[c][1] is None else b[c][1] for b in key_batches[:upto]]))
                for c in range(nk)]
        arg = (np.concatenate([np.asarray(a[0]) for a in arg_batches[:upto]]),
               None if all(a[1] is None for a in arg_batches[:upto]) else np.concatenate([np.ones(len(a[0]), bool) if a[1] is None else a[1] for a in arg_batches[:upto]]))
        gk, res = group_by(keys, [(func, arg, None)])
        for c in range(nk):
            out_keys[c].append(np.asarray(gk[c][0])); out_kvalid[c].append(np.ones(len(gk[c][0]), bool) if gk[c][1] is None else gk[c][1])
        st = agg_output_columns(func, res[0], np.asarray(arg[0]).dtype, True)[0]
        out_state.append(np.asarray(st[0]).astype(np.int64)); out_svalid.append(np.ones(len(st[0]), bool) if st[1] is None else st[1])

    for bi, (kb, ab) in enumerate(zip(key_batches, arg_batches)):
        n = len(kb[0][0])
        if should_skip:                                  # SkippingAggregation: one state row per input row
            for c in range(nk):
                out_keys[c].append(np.asarray(kb[c][0])); out_kvalid[c].append(np.ones(n, bool) if kb[c][1] is None else np.asarray(kb[c][1], bool))
            valid = np.ones(n, bool) if ab[1] is None else np.asarray(ab[1], bool)
            out_state.append(valid.astype(np.int64) if func == A_COUNT else np.asarray(ab[0]).astype(np.int64)); out_svalid.append(np.ones(n, bool) if func == A_COUNT else valid)
            continue
        agg_upto = bi + 1
        rows_seen += n
        if rows_seen >= probe_rows_threshold:
            keys = [(np.concatenate([np.asarray(b[c][0]) for b in key_batches[:agg_upto]]), None) for c in range(nk)]
            groups = len(group_by(keys, [])[0][0][0]) if nk else 1
            should_skip = groups / rows_seen > probe_ratio_threshold
            if should_skip:
                emit_groups(agg_upto)
    if not should_skip:
        emit_groups(agg_upto)
    cat = lambda xs, dt=None: np.concatenate(xs) if xs else np.zeros(0, dt or np.int64)
    keys = [(cat(out_keys[c]), None if all(v.all() for v in out_kvalid[c]) else cat(out_kvalid[c], bool)) for c in range(nk)]
    sv = cat(out_svalid, bool)
    return keys, (cat(out_state), None if sv.all() else sv)


# ---------------------------------------------------------------------------------------------
# expressions (numpy)
# ---------------------------------------------------------------------------------------------
(E_COLUMN, E_LITERAL, E_BINARY, E_NOT, E_IS_NULL, E_IS_NOT_NULL, E_NEGATIVE, E_CAST) = range(1, 9)
(OP_EQ, OP_NEQ, OP_LT, OP_LTEQ, OP_GT, OP_GTEQ, OP_PLUS, OP_MINUS, OP_MULTIPLY, OP_DIVIDE, OP_MODULO, OP_AND, OP_OR,
 OP_IS_DISTINCT_FROM, OP_IS_NOT_DISTINCT_FROM, OP_BITAND, OP_BITOR, OP_BITXOR, OP_SHIFT_LEFT, OP_SHIFT_RIGHT) = range(1, 21)


class ArrowArithmeticOverflow(ArithmeticError):
    """ArrowError::ArithmeticOverflow (checked i128 arithmetic of Decimal128 operands)"""


# ---------------------------------------------------------------------------------------------
# Decimal128 (arrow-arith 59.2.0 arithmetic.rs `decimal_op`, arrow-cast 59.2.0 cast/decimal.rs — third-party crates pinned by the
# reference's Cargo.lock and absent from /root/reference: their published algorithm is restated here; pinned by the reference's own
# vectors binary.rs:4355-5000 in tests/test_oracle_decimal.py)
# ---------------------------------------------------------------------------------------------
class Dec(np.ndarray):
    """Decimal128Array values: unscaled Python ints in an object ndarray + (precision p, scale s)"""

    def __new__(cls, values, precision: int, scale: int):
        vals = list(values)
        obj = np.empty(len(vals), dtype=object)
        obj[:] = [int(x) for x in vals]
        obj = obj.view(cls)
        obj.p, obj.s = int(precision), int(scale)
        return obj

    def __array_finalize__(self, obj):
        self.p = getattr(obj, "p", None)
        self.s = getattr(obj, "s", None)


def _arr(v):
    return v if isinstance(v, Dec) else np.asarray(v)


def decimal_dtype(p: int, s: int):
    """the `dt` of a Decimal128 literal / cast target node"""
    return ("decimal128", int(p), int(s))


_I128_MIN, _I128_MAX = -(1 << 127), (1 << 127) - 1


def _chk128(x: int) -> int:
    if not (_I128_MIN <= x <= _I128_MAX):
        raise ArrowArithmeticOverflow("Arithmetic overflow")
    return x


def _tdiv(a: int, b: int) -> int:      # Rust's `/` on integers truncates toward zero
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def decimal_result_type(op: int, p1: int, s1: int, p2: int, s2: int):
    """(precision, scale, l_exp, r_exp) of `decimal_op`: operands are multiplied by 10^l_exp / 10^r_exp before the operation"""
    if op in (OP_PLUS, OP_MINUS):
        rs = max(s1, s2)
        return min(38, rs + max(p1 - s1, p2 - s2) + 1), rs, rs - s1, rs - s2
    if op == OP_MULTIPLY:
        return min(38, p1 + p2 + 1), s1 + s2, 0, 0
    if op == OP_DIVIDE:
        rs = min(38, s1 + 4)                       # "a fixed scale increment of 4"
        mul_pow = rs - s1 + s2
        return min(38, mul_pow + p1), rs, max(mul_pow, 0), max(-mul_pow, 0)
    if op == OP_MODULO:
        rs = max(s1, s2)
        return min(38, rs + min(p1 - s1, p2 - s2)), rs, rs - s1, rs - s2
    raise ValueError(op)


def _dec_binary(op: int, l: "Dec", r: "Dec", act: np.ndarray):
    n = len(l)
    if op in (OP_EQ, OP_NEQ, OP_LT, OP_LTEQ, OP_GT, OP_GTEQ):
        assert (l.p, l.s) == (r.p, r.s), "Decimal128 comparison needs equal precision and scale (the planner coerces)"
        f = {OP_EQ: int.__eq__, OP_NEQ: int.__ne__, OP_LT: int.__lt__, OP_LTEQ: int.__le__, OP_GT: int.__gt__, OP_GTEQ: int.__ge__}[op]
        return np.array([bool(f(int(a), int(b))) for a, b in zip(l, r)], bool) if n else np.zeros(0, bool)
    rp, rs, le, re = decimal_result_type(op, l.p, l.s, r.p, r.s)
    lm, rm = 10 ** le, 10 ** re
    out = []
    for i in range(n):
        if not act[i]:
            out.append(0); continue
        x, y = _chk128(int(l[i]) * lm), _chk128(int(r[i]) * rm)
        if op == OP_PLUS: z = x + y
        elif op == OP_MINUS: z = x - y
        elif op == OP_MULTIPLY: z = x * y
        else:
            if y == 0:
                raise ArrowDivideByZero("Divide by zero error")
            q = _tdiv(x, y)
            z = q if op == OP_DIVIDE else x - q * y
        out.append(_chk128(z))
    return Dec(out, rp, rs)


def _dec_fits(x: int, precision: int) -> bool:
    return abs(x) < 10 ** precision


def _dec_cast(v, val, n, tgt):
    """CastExpr with a Decimal128 on either side (CastOptions safe = false: failures are errors)"""
    act = np.ones(n, bool) if val is None else np.asarray(val, bool)
    if isinstance(tgt, tuple):
        _, p, sc = tgt
        out = []
        for i in range(n):
            if not act[i]:
                out.append(0); continue
            if isinstance(v, Dec):
                x = int(v[i])
                if sc >= v.s:
                    x = x * 10 ** (sc - v.s)
                else:                                   # convert_to_smaller_scale_decimal: round half away from zero
                    div = 10 ** (v.s - sc); half = div // 2
                    d = _tdiv(x, div); rem = x - d * div
                    x = (d + 1 if rem >= half else d) if x >= 0 else (d - 1 if rem <= -half else d)
            elif np.asarray(v).dtype.kind == "f":
                prod = np.float64(v[i]) * np.float64(10.0 ** sc) if sc <= 22 else None
                if prod is None or not np.isfinite(prod):
                    raise ArrowCastError("Cannot cast to Decimal128")
                t = np.trunc(prod)                            # f64::round: half away from zero (np.round would round half to even)
                m = float(t + np.copysign(1.0, prod)) if abs(prod - t) >= 0.5 else float(t)
                x = int(abs(m)); x = -x if m < 0 else x
            else:
                x = int(v[i]) * 10 ** sc
            if not _dec_fits(x, p) or not (_I128_MIN <= x <= _I128_MAX):
                raise ArrowCastError(f"{x} is too large to store in a Decimal128 of precision {p}")
            out.append(x)
        return Dec(out, p, sc), val
    tgt = np.dtype(tgt)
    assert isinstance(v, Dec)
    if tgt.kind == "f":
        with np.errstate(all="ignore"):
            r = np.array([float(np.float64(int(x)) / np.float64(10.0 ** v.s)) for x in v], np.float64).astype(tgt)   # `x as f64 / 10f64.powi(s)`
        return np.where(act, r, 0).astype(tgt), val
    info = np.iinfo(tgt)
    out = np.zeros(n, tgt)
    for i in range(n):
        if act[i]:
            q = _tdiv(int(v[i]), 10 ** v.s)
            if not (info.min <= q <= info.max):
                raise ArrowCastError("Can't cast value to the target type")
            out[i] = q
    return out, val


class ArrowDivideByZero(ArithmeticError):
    pass


class ArrowCastError(ArithmeticError):
    """arrow-cast with CastOptions { safe: false } — DataFusion's DEFAULT_CAST_OPTIONS (expressions/cast.rs:37-40)"""


def _total_order_key(x: np.ndarray) -> np.ndarray:
    """IEEE-754 totalOrder as a sortable int64, after -0.0 -> +0.0 (datum.rs:88-105)"""
    x = np.asarray(x, dtype=np.float64).copy()
    x[x == 0] = 0.0
    b = x.view(np.int64)
    return b ^ ((b >> 63).astype(np.uint64) >> np.uint64(1)).astype(np.int64)


PRE_SELECTION_THRESHOLD = np.float32(0.2)   # binary.rs:1160


def _subtree_starts(nodes):
    st, start = [], [0] * len(nodes)
    for i, nd in enumerate(nodes):
        if nd[0] in (E_COLUMN, E_LITERAL):
            start[i] = i
        elif nd[0] == E_BINARY:
            start[i] = start[start[i - 1] - 1]
        else:
            start[i] = start[i - 1]
    return start


def eval_expr(cols: Sequence[Col], nodes: Sequence[tuple], col_dtypes: Optional[Sequence] = None) -> Col:
    """PhysicalExpr::evaluate over a batch.  nodes: [(kind, a, np dtype or None, is_null, lit)] in post-order; returns (values, valid).
    AND / OR follow BinaryExpr::evaluate (binary.rs:536-600): the LHS is evaluated first and check_short_circuit (:1182-1290) may return
    it as is, return the RHS, or evaluate the RHS only on the pre-selected rows (filter_record_batch + scatter) — which also decides on
    which rows an error inside the RHS (division by zero, failed cast) can surface."""
    nodes = list(nodes)
    starts = _subtree_starts(nodes)

    def ev(lo, hi, cs):
        kind, a = nodes[hi - 1][0], nodes[hi - 1][1]
        n = len(cs[0][0]) if cs else 0
        if kind == E_BINARY and a in (OP_AND, OP_OR):
            is_and = a == OP_AND
            rlo = starts[hi - 2]
            lhs = ev(lo, rlo, cs)
            lv, lval = lhs
            scalar_lhs = (rlo - lo == 1 and nodes[lo][0] == E_LITERAL)
            if scalar_lhs:
                if nodes[lo][3]:                       # NULL scalar: no short circuit
                    return _kleene(is_and, lhs, ev(rlo, hi - 1, cs))
                is_true = bool(nodes[lo][4])
                return lhs if (is_and and not is_true) or (not is_and and is_true) else ev(rlo, hi - 1, cs)
            if lval is not None and not np.asarray(lval, bool).all() or n == 0:
                return _kleene(is_and, lhs, ev(rlo, hi - 1, cs))          # arrays with nulls can't be short-circuited
            tc = int(np.count_nonzero(lv))
            if is_and and tc == 0 or (not is_and and tc == n):
                return (np.asarray(lv, bool), None)                          # ReturnLeft
            if is_and and tc == n or (not is_and and tc == 0):
                return ev(rlo, hi - 1, cs)                                   # ReturnRight
            rare = tc if is_and else n - tc
            if np.float32(rare) / np.float32(n) <= PRE_SELECTION_THRESHOLD:
                mask = np.asarray(lv, bool) if is_and else ~np.asarray(lv, bool)
                sel = [(_arr(v)[mask], None if val is None else np.asarray(val, bool)[mask]) for v, val in cs]
                rv, rval = ev(rlo, hi - 1, sel)
                out = np.full(n, not is_and, bool)                           # fill_value: false for AND, true for OR
                out[mask] = np.asarray(rv, bool)
                valid = None
                if rval is not None and not np.asarray(rval, bool).all():
                    valid = np.ones(n, bool); valid[mask] = rval
                    out[mask] &= rval
                return (out, valid)
            return _kleene(is_and, lhs, ev(rlo, hi - 1, cs))
        if kind in (E_COLUMN, E_LITERAL):
            return _eval_flat(cs, nodes[lo:hi])
        if kind == E_BINARY:
            rlo = starts[hi - 2]
            l, r = ev(lo, rlo, cs), ev(rlo, hi - 1, cs)
            return _eval_flat([l, r], [(E_COLUMN, 0, None, 0, 0), (E_COLUMN, 1, None, 0, 0), nodes[hi - 1]])
        c = ev(lo, hi - 1, cs)
        return _eval_flat([c], [(E_COLUMN, 0, None, 0, 0), nodes[hi - 1]])
    return ev(0, len(nodes), list(cols))


def _kleene(is_and, lhs, rhs):
    return _eval_flat([lhs, rhs], [(E_COLUMN, 0, None, 0, 0), (E_COLUMN, 1, None, 0, 0), (E_BINARY, OP_AND if is_and else OP_OR, None, 0, 0)])


def _eval_flat(cols: Sequence[Col], nodes: Sequence[tuple]) -> Col:
    """the straight stack machine (every node over every row)"""
    n = len(cols[0][0]) if cols else 0
    st: List[Col] = []
    for kind, a, dt, is_null, lit in nodes:
        if kind == E_COLUMN:
            v, val = cols[a]
            st.append((_arr(v), None if val is None else np.asarray(val, bool)))
        elif kind == E_LITERAL:
            if isinstance(dt, tuple):
                arr = Dec([0 if is_null else int(lit)] * n, dt[1], dt[2])
            else:
                arr = np.full(n, 0 if is_null else lit, dtype=dt)
            st.append((arr, np.zeros(n, bool) if is_null else None))
        elif kind == E_BINARY:
            (rv, rval), (lv, lval) = st.pop(), st.pop()
            both = None
            if lval is not None or rval is not None:
                both = (np.ones(n, bool) if lval is None else lval) & (np.ones(n, bool) if rval is None else rval)
            if a in (OP_AND, OP_OR):  # Kleene (binary.rs:1093-1116)
                lt = lv.astype(bool) & (lval if lval is not None else True)
                lf = ~lv.astype(bool) & (lval if lval is not None else True)
                rt = rv.astype(bool) & (rval if rval is not None else True)
                rf = ~rv.astype(bool) & (rval if rval is not None else True)
                if a == OP_AND:
                    res_t, res_f = lt & rt, lf | rf
                else:
                    res_t, res_f = lt | rt, lf & rf
                valid = res_t | res_f
                st.append((res_t, None if valid.all() else valid))
            elif isinstance(lv, Dec) or isinstance(rv, Dec):
                assert isinstance(lv, Dec) and isinstance(rv, Dec), "a Decimal128 operand needs a Decimal128 partner (the planner's coercion casts the other side)"
                act = np.ones(n, bool) if both is None else both
                if a in (OP_IS_DISTINCT_FROM, OP_IS_NOT_DISTINCT_FROM):
                    lvv = np.ones(n, bool) if lval is None else lval
                    rvv = np.ones(n, bool) if rval is None else rval
                    ne = _dec_binary(OP_NEQ, lv, rv, act)
                    distinct = (lvv != rvv) | (lvv & rvv & ne)
                    st.append((distinct if a == OP_IS_DISTINCT_FROM else ~distinct, None))
                else:
                    r = _dec_binary(a, lv, rv, act)
                    if not isinstance(r, Dec) and both is not None:
                        r = r & both
                    st.append((r, both))
            elif a in (OP_EQ, OP_NEQ, OP_LT, OP_LTEQ, OP_GT, OP_GTEQ, OP_IS_DISTINCT_FROM, OP_IS_NOT_DISTINCT_FROM):
                if lv.dtype.kind == "f":
                    x, y = _total_order_key(lv), _total_order_key(rv)
                else:
                    x, y = lv, rv
                if a in (OP_IS_DISTINCT_FROM, OP_IS_NOT_DISTINCT_FROM):
                    lvv = np.ones(n, bool) if lval is None else lval
                    rvv = np.ones(n, bool) if rval is None else rval
                    distinct = (lvv != rvv) | (lvv & rvv & (x != y))
                    st.append((distinct if a == OP_IS_DISTINCT_FROM else ~distinct, None))
                else:
                    r = {OP_EQ: x == y, OP_NEQ: x != y, OP_LT: x < y, OP_LTEQ: x <= y, OP_GT: x > y, OP_GTEQ: x >= y}[a]
                    if both is not None:
                        r = r & both
                    st.append((r, both))
            else:
                dtp = lv.dtype
                act = np.ones(n, bool) if both is None else both
                with np.errstate(all="ignore"):
                    if dtp.kind == "f":
                        if a == OP_PLUS: r = lv + rv
                        elif a == OP_MINUS: r = lv - rv
                        elif a == OP_MULTIPLY: r = lv * rv
                        elif a == OP_DIVIDE: r = lv / rv
                        elif a == OP_MODULO: r = np.fmod(lv, rv)
                        else: raise ValueError(a)
                    else:
                        if a in (OP_DIVIDE, OP_MODULO):
                            if np.any(act & (rv == 0)):
                                raise ArrowDivideByZero("Divide by zero error")
                            safe = np.where(rv == 0, 1, rv)
                            if dtp.kind == "i":
                                # Rust's truncating `/` and `%` on exact Python ints: MIN / -1 does not fit the type, and arrow's checked `div`
                                # reports ArithmeticOverflow there; `rem` gives 0 (MIN % -1 == 0)
                                lo = int(np.iinfo(dtp).min)
                                if a == OP_DIVIDE and np.any(act & (lv == lo) & (rv == -1)):
                                    raise ArrowArithmeticOverflow("Arithmetic overflow")
                                q = [_tdiv(x, y) for x, y in zip(lv.tolist(), safe.tolist())]
                                r = [qq if qq != -lo else 0 for qq in q] if a == OP_DIVIDE else [x - qq * y for x, y, qq in zip(lv.tolist(), safe.tolist(), q)]
                                r = np.array(r, np.int64).astype(dtp)
                            else:
                                r = (lv // safe) if a == OP_DIVIDE else (lv % safe)
                        elif a == OP_PLUS: r = lv + rv   # numpy integer arrays wrap
                        elif a == OP_MINUS: r = lv - rv
                        elif a == OP_MULTIPLY: r = lv * rv
                        elif a == OP_BITAND: r = lv & rv
                        elif a == OP_BITOR: r = lv | rv
                        elif a == OP_BITXOR: r = lv ^ rv
                        elif a in (OP_SHIFT_LEFT, OP_SHIFT_RIGHT):
                            # arrow-arith bitwise_shift_left/right = wrapping_shl / wrapping_shr: shift amount modulo the bit
                            # width (binary.rs:5073 bitwise_shift_array_overflow_test: 2 << 100 = 32 for Int32)
                            sh = (rv.astype(np.int64) & (dtp.itemsize * 8 - 1)).astype(dtp)
                            r = ((lv << sh) if a == OP_SHIFT_LEFT else (lv >> sh)).astype(dtp)
                        else: raise ValueError(a)
                if both is not None:
                    r = np.where(both, r, np.zeros((), r.dtype))
                st.append((r.astype(dtp), both))
        elif kind == E_NOT:
            v, val = st.pop()
            r = ~v.astype(bool)
            st.append((r & val if val is not None else r, val))
        elif kind == E_IS_NULL:
            v, val = st.pop()
            st.append((np.zeros(n, bool) if val is None else ~val, None))
        elif kind == E_IS_NOT_NULL:
            v, val = st.pop()
            st.append((np.ones(n, bool) if val is None else val.copy(), None))
        elif kind == E_NEGATIVE:
            v, val = st.pop()
            if isinstance(v, Dec):       # neg_wrapping
                st.append((Dec([((-int(x) + (1 << 127)) % (1 << 128)) - (1 << 127) for x in v], v.p, v.s), val))
                continue
            with np.errstate(all="ignore"):
                st.append((-v, val))
        elif kind == E_CAST:
            v, val = st.pop()
            if isinstance(v, Dec) or isinstance(dt, tuple):
                st.append(_dec_cast(v, val, n, dt))
                continue
            tgt = np.dtype(dt)
            act = np.ones(n, bool) if val is None else np.asarray(val, bool)
            if tgt.kind in "iu" and v.dtype.kind in "iuf":
                # out-of-range values fail the cast (they neither wrap nor become NULL); float -> int truncates toward zero
                info = np.iinfo(tgt)
                if v.dtype.kind == "f":
                    t = np.trunc(v.astype(np.float64))
                    fits = np.isfinite(v) & (t >= float(info.min)) & (t < float(info.max) + 1.0)
                else:
                    fits = np.array([info.min <= int(x) <= info.max for x in v.tolist()], bool) if len(v) else np.zeros(0, bool)
                if np.any(act & ~fits):
                    raise ArrowCastError("Can't cast value to the target type")
                with np.errstate(all="ignore"):
                    out = np.where(fits, np.trunc(v) if v.dtype.kind == "f" else v, 0).astype(tgt)
                st.append((out, val))
            else:
                with np.errstate(all="ignore"):
                    st.append((v.astype(tgt), val))
        else:
            raise ValueError(kind)
    assert len(st) == 1
    return st[0]


def coalesce_sizes(input_sizes: Sequence[int], target_batch_size: int, fetch: Optional[int] = None) -> List[int]:
    """LimitedBatchCoalescer (physical-plan/src/coalesce/mod.rs:27-147): row counts of the completed output batches for a stream
    of input batches — full `target_batch_size` batches while rows keep coming, the remainder at finish; `fetch` truncates the batch
    that crosses the limit and stops the stream (PushBatchStatus::LimitReached)."""
    out, buffered, total = [], 0, 0
    for n in input_sizes:
        if fetch is not None:
            if total >= fetch:
                break
            n = min(n, fetch - total)
        total += n
        buffered += n
        while buffered >= target_batch_size:
            out.append(target_batch_size); buffered -= target_batch_size
        if fetch is not None and total >= fetch:
            break
    if buffered:
        out.append(buffered)
    return out


def filter_batch(cols: Sequence[Col], pred: Col, projection: Optional[Sequence[int]] = None) -> List[Col]:
    """filter_record_batch: keep rows whose predicate is TRUE and non-NULL (filter.rs:1339-1361)."""
    pv, pval = pred
    keep = pv.astype(bool) & (pval if pval is not None else True)
    proj = range(len(cols)) if projection is None else projection
    out = []
    for i in proj:
        v, val = cols[i]
        nv = None if val is None else np.asarray(val, bool)[keep]
        out.append((_arr(v)[keep], None if nv is None or nv.all() else nv))
    return out


# ---------------------------------------------------------------------------------------------
# CPU baseline timing (bench.py only)
# ---------------------------------------------------------------------------------------------
def generate_i64(kind: int, seed: int, a: int, b: int, n: int, threads: int = 1) -> np.ndarray:
    out = np.empty(n, np.int64)
    lib().oracle_generate_i64(C.c_int(kind), C.c_uint64(seed), C.c_int64(a), C.c_int64(b), C.c_int64(n), C.c_int(threads),
                              out.ctypes.data_as(C.POINTER(C.c_int64)))
    return out


def bench_join(bk, bp, pk, pp, threads: int, batch_size: int = 8192, use_amap_rule: bool = True):
    out = (C.c_uint64 * 2)()
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    secs = lib().oracle_bench_join(p(bk), p(bp), C.c_int64(len(bk)), p(pk), p(pp), C.c_int64(len(pk)), C.c_int(threads), C.c_int64(batch_size),
                                   C.c_int(1 if use_amap_rule else 0), out)
    return secs, int(out[0]), int(out[1])


def bench_groupby(g, v, threads: int, batch_size: int = 8192):
    out = (C.c_uint64 * 2)()
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    secs = lib().oracle_bench_groupby(p(g), p(v), C.c_int64(len(g)), C.c_int(threads), C.c_int64(batch_size), out)
    return secs, int(out[0]), int(out[1])


# ---- TPC-H Q3-shaped pipeline (BASELINE config C4) ----
Q3_D0, Q3_D1, Q3_CUT = 8035, 10440, 9204    # days since epoch of 1992-01-01, 1998-08-02, 1995-03-15


def q3_generate(sf: float, seed: int = 1, threads: int = 1) -> dict:
    """host copy of scripts/q3_device_pipeline.py gen_tables (same counter-based formulae, bit-identical tables)"""
    nc, no, nl = int(150_000 * sf), int(1_500_000 * sf), int(6_000_000 * sf)
    t = {"c_custkey": np.empty(nc, np.int64), "c_mktsegment": np.empty(nc, np.int64),
         "o_orderkey": np.empty(no, np.int64), "o_custkey": np.empty(no, np.int64), "o_orderdate": np.empty(no, np.int32), "o_shippriority": np.empty(no, np.int32),
         "l_orderkey": np.empty(nl, np.int64), "l_extendedprice": np.empty(nl, np.int64), "l_discount": np.empty(nl, np.int64), "l_shipdate": np.empty(nl, np.int32)}
    p = lambda a: C.c_void_p(a.ctypes.data)
    L = lib()
    L.oracle_q3_generate.restype = None
    L.oracle_q3_generate(C.c_int64(nc), C.c_int64(no), C.c_int64(nl), C.c_uint64(seed), C.c_int64(Q3_D0), C.c_int64(Q3_D1), C.c_int(threads),
                         p(t["c_custkey"]), p(t["c_mktsegment"]), p(t["o_orderkey"]), p(t["o_custkey"]), p(t["o_orderdate"]), p(t["o_shippriority"]),
                         p(t["l_orderkey"]), p(t["l_extendedprice"]), p(t["l_discount"]), p(t["l_shipdate"]))
    return t


def bench_q3(t: dict, threads: int, batch_size: int = 8192, cut: int = Q3_CUT):
    """(seconds, fingerprint [groups, sum l_orderkey, sum o_orderdate, sum o_shippriority, sum revenue], stage rows dict)"""
    out = (C.c_uint64 * 9)()
    p = lambda a: C.c_void_p(a.ctypes.data)
    L = lib()
    L.oracle_bench_q3.restype = C.c_double
    secs = L.oracle_bench_q3(C.c_int64(len(t["c_custkey"])), C.c_int64(len(t["o_orderkey"])), C.c_int64(len(t["l_orderkey"])),
                             p(t["c_custkey"]), p(t["c_mktsegment"]), p(t["o_orderkey"]), p(t["o_custkey"]), p(t["o_orderdate"]), p(t["o_shippriority"]),
                             p(t["l_orderkey"]), p(t["l_extendedprice"]), p(t["l_discount"]), p(t["l_shipdate"]), C.c_int32(cut), C.c_int(threads),
                             C.c_int64(batch_size), out)
    o = [int(x) for x in out]
    return secs, o[:5], {"joined_rows": o[5], "customer_building": o[6], "orders_of_building_customers": o[7], "lineitem_after_cut": o[8]}


def q3_stream_fingerprint(sf_total: float, seed: int = 1, threads: int = 1, cut: int = Q3_CUT):
    """expected result fingerprint of the Q3-shaped query over the SF(sf_total) database, computed by streaming regeneration
    (no table in memory): ([groups, sum l_orderkey, sum o_orderdate, sum o_shippriority, sum revenue], joined rows, qualified orders)"""
    nc, no, nl = int(150_000 * sf_total), int(1_500_000 * sf_total), int(6_000_000 * sf_total)
    out = (C.c_uint64 * 7)()
    rc = lib().oracle_q3_stream_fingerprint(C.c_int64(nc), C.c_int64(no), C.c_int64(nl), C.c_uint64(seed), C.c_int64(Q3_D0), C.c_int64(Q3_D1),
                                           C.c_int32(cut), C.c_int(threads), out)
    if rc != 0:
        raise MemoryError("q3_stream_fingerprint: table allocation failed")
    o = [int(x) for x in out]
    return o[:5], o[5], o[6]


def scalar_aggregate(aggs: Sequence[tuple], state: bool = False) -> List[Col]:
    """AggregateStream (no GROUP BY; aggregates/aggregate_stream.rs:360-400 poll loop, aggregate_batch :437 + finalize_aggregation, aggregates/mod.rs:2993-3020):
    every input batch updates ONE accumulator per aggregate; at end of input exactly one row is emitted, also for empty input
    (fresh accumulators: SUM / MIN / MAX / AVG -> NULL, COUNT -> 0).  aggs: [(func, arg: Col | None, filter: Col | None)];
    state=True gives the Partial output (state columns) instead of the final values."""
    out: List[Col] = []
    for ag in aggs:
        func, arg, filt = ag[0], ag[1], ag[2] if len(ag) > 2 else None
        if arg is None:
            n = len(filt[0]) if filt is not None else ag[3]
            vals, act = np.zeros(n, np.int64), np.ones(n, bool)
        else:
            vals = np.asarray(arg[0]); act = np.ones(len(vals), bool) if arg[1] is None else np.asarray(arg[1], bool).copy()
        if filt is not None:
            act &= np.asarray(filt[0], bool) & (np.ones(len(act), bool) if filt[1] is None else np.asarray(filt[1], bool))
        sel = vals[act]
        cnt = int(act.sum())
        one = lambda v, dt, valid: (np.array([v], dt), None if valid else np.array([False]))
        if func in (A_COUNT, A_COUNT_STAR):
            out.append(one(cnt, np.int64, True))
        elif func == A_SUM:
            if vals.dtype.kind == "f":
                out.append(one(float(sel.astype(np.float64).sum()) if cnt else 0.0, np.float64, cnt > 0))
            else:
                dt = np.uint64 if vals.dtype.kind == "u" else np.int64
                with np.errstate(over="ignore"):
                    out.append(one(sel.astype(dt).sum(dtype=dt) if cnt else 0, dt, cnt > 0))
        elif func in (A_MIN, A_MAX):
            if vals.dtype.kind == "f" and cnt:   # IEEE totalOrder on the bits, as the grouped MIN / MAX
                u = np.ascontiguousarray(sel).view(np.uint64 if vals.dtype.itemsize == 8 else np.uint32)
                top = u.dtype.type(1 << (8 * u.dtype.itemsize - 1))
                k = np.where(u & top, ~u, u | top)
                out.append((sel[[np.argmin(k) if func == A_MIN else np.argmax(k)]], None))
                continue
            out.append(one((sel.min() if func == A_MIN else sel.max()) if cnt else 0, vals.dtype, cnt > 0))
        elif func == A_AVG:
            sm = float(sel.astype(np.float64).sum()) if cnt else 0.0
            if state:
                out.append(one(cnt, np.uint64, True)); out.append(one(sm, np.float64, cnt > 0))
            else:
                out.append(one(sm / cnt if cnt else 0.0, np.float64, cnt > 0))
        else:
            raise ValueError(func)
    return out
