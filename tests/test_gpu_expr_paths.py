"""Every expression-evaluation path against the oracle, and against each other, on generated typed programs (tests/expr_gen.py).

The same PhysicalExpr program runs in dfgpu_expr_evaluate_host / _device, FilterExec, the hash join's JoinFilter, the fused pipeline's
predicate, its stage filters and its aggregate arguments.  Each picks an evaluator from the program's shape, its types and the batch:
the local-memory interpreter (eval_nodes), the register-stack one (eval_nodes_reg<4>, stack depth <= 4), the integer fast paths
(eval_int_fast, and eval_int_gathered in the ring-fed kernel), the Decimal128 interpreter, the conjunction of `column <cmp> literal`
terms, the scalar Int64 compare, and payload-field nodes.  Each test counts the evaluators its programs reached, from the pipeline's
metrics where there is one (ring_launches) and from the planning predicates (expr_gen's depth / is_int_arith / has_decimal) elsewhere,
and asserts that none went unexercised.  Floats compare bit for bit; a NaN that arithmetic produced equals any NaN (expr_gen's rules).
"""
import collections
import ctypes as CT

import numpy as np
import pytest

import expr_gen as G
from datafusion_b200 import capi as D
from harness import batches_to_cols
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ERR_CLASS = {O.ArrowDivideByZero: "divide by zero", O.ArrowArithmeticOverflow: "arithmetic overflow", O.ArrowCastError: "cast error"}
N_PROGRAMS = 300
ROWS = (0, 1, 31, 33, 255, 257, 511, 513, 1023, 1025, 3001)
VALUE_ROOTS = G.INTS + G.FLOATS + (G.BOOL,)


# ---------------------------------------------------------------------------------------------
# running the paths
# ---------------------------------------------------------------------------------------------
def outcome(fn):
    """('ok', result) or ('err', message class) for a GPU call; any other GPU error fails the test"""
    try:
        return "ok", fn()
    except D.DfgpuError as ex:
        msg = str(ex).lower()
        assert ex.code == -4, f"unexpected error {ex}"                  # DFGPU_ERR_ARITH
        return "err", next(c for c in ERR_CLASS.values() if c in msg)


def oracle_outcome(prog, cols):
    try:
        return "ok", O.eval_expr(G.oracle_cols(prog, cols), prog.oracle_nodes())
    except tuple(ERR_CLASS) as ex:
        return "err", ERR_CLASS[type(ex)]


def slice_cols(cols, lo, hi):
    return [(v[lo:hi], None if val is None else val[lo:hi]) for v, val in cols]


def offset_column(ctx, t, v, val, off, device, keep):
    """a dfgpu_column whose logical row 0 is physical row `off` (Arrow's offset): the bitmaps are read through `voff`"""
    n = len(v)
    pad_v = (list(v[:1]) * off + list(v)) if t.kind == "x" else np.concatenate([np.zeros(off, np.asarray(v).dtype), np.asarray(v)])
    pad_val = None if val is None else np.concatenate([np.ones(off, bool), val])
    hc = D.HostColumn(pad_v, pad_val, t.code)
    keep.append(hc)
    src = hc
    if device:
        src = D.DeviceColumn.from_host(ctx, hc)
        keep.append(src)
    c = src.c()
    c.offset, c.length = off, n
    c.null_count = 0 if val is None else int(n - np.count_nonzero(val))
    return c


def gpu_columns(ctx, prog, cols, device, offset, keep):
    out = []
    for (t, _), (v, val) in zip(prog.cols, cols):
        if offset and (t.kind == "b" or val is not None):
            out.append(offset_column(ctx, t, v, val, offset, device, keep))
            continue
        hc = D.HostColumn(list(v) if t.kind == "x" else v, val, t.code)
        keep.append(hc)
        if device:
            dc = D.DeviceColumn.from_host(ctx, hc)
            keep.append(dc)
            out.append(dc.c())
        else:
            out.append(hc.c())
    return out


def run_evaluate(ctx, prog, cols, n, device=False, offset=0):
    keep = []
    arr = (D.Column * max(len(prog.cols), 1))(*gpu_columns(ctx, prog, cols, device, offset, keep))
    nodes = D.expr_nodes(prog.gpu_nodes())
    out = CT.c_void_p()
    fn = ctx.lib.dfgpu_expr_evaluate_device if device else ctx.lib.dfgpu_expr_evaluate_host
    ctx.check(fn(ctx.h, arr, len(prog.cols), n, nodes, len(nodes), CT.byref(out)))
    return D.Batch(ctx, out.value).column_numpy(0)


def as_py(t, col):
    """(values, valid) of type t -> list of Python values / None"""
    v, val = col
    if isinstance(v, O.Dec):
        vals = [int(x) for x in v]
    elif t.kind == "x":
        vals = D.words_to_decimal(v)
    else:
        vals = list(np.asarray(v))
    return [None if (val is not None and not val[i]) else vals[i] for i in range(len(vals))]


def same(t, a, b):
    if a is None or b is None:
        return a is None and b is None
    if t.kind == "f":
        a, b = t.np(a), t.np(b)
        if np.isnan(a) and np.isnan(b):
            return True
        u = np.uint64 if t.bits == 64 else np.uint32
        return np.array([a]).view(u)[0] == np.array([b]).view(u)[0]
    if t.kind == "b":
        return bool(a) == bool(b)
    return int(a) == int(b)


def fail(prog, path, cols, i, exp, got, extra=""):
    row = None if i is None else [as_py(t, (np.asarray(v[i:i + 1]) if t.kind != "x" else O.Dec(v[i:i + 1], t.p, t.s), None if val is None else val[i:i + 1]))[0]
                                  for (t, _), (v, val) in zip(prog.cols, cols)]
    raise AssertionError(f"{path}: {prog.describe()}\n first differing row {i}: inputs {row}\n expected {exp!r}\n got      {got!r}{extra}")


def compare_values(prog, path, cols, exp_col, got_col, t=None):
    t = t or prog.t
    e, g = as_py(t, exp_col), as_py(t, got_col)
    if len(e) != len(g):
        fail(prog, path, cols, None, f"{len(e)} rows", f"{len(g)} rows")
    for i, (a, b) in enumerate(zip(e, g)):
        if not same(t, a, b):
            fail(prog, path, cols, i, a, b)


def compare_outcomes(prog, path, cols, exp, got, t=None):
    if exp[0] != got[0] or (exp[0] == "err" and exp[1] != got[1]):
        fail(prog, path, cols, None, exp if exp[0] == "err" else "values", got if got[0] == "err" else "values")
    if exp[0] == "ok":
        compare_values(prog, path, cols, exp[1], got[1], t)


def truth(col):
    v, val = col
    m = np.asarray(v, bool).copy()
    if val is not None:
        m &= np.asarray(val, bool)
    return m


def pushes(n, rng):
    """1-3 pushes, their sizes not multiples of the tile widths"""
    if n < 2 or rng.random() < 0.4:
        return [(0, n)]
    cuts = sorted({int(x) for x in rng.integers(1, n, int(rng.integers(1, 3)))})
    b = [0] + cuts + [n]
    return list(zip(b[:-1], b[1:]))


def per_push_oracle(prog, cols, parts):
    """the oracle over each push (short-circuit guards are decided per batch): ('ok', TRUE mask) or the first push's error"""
    masks = []
    for lo, hi in parts:
        res = oracle_outcome(prog, slice_cols(cols, lo, hi))
        if res[0] == "err":
            return res
        masks.append(truth(res[1]))
    return "ok", np.concatenate(masks) if masks else np.zeros(0, bool)


def host_cols_with_rowid(prog, cols, lo, hi, rowid):
    return G.host_columns(prog, cols, lo, hi) + [D.HostColumn(rowid[lo:hi])]


def run_filter(ctx, prog, cols, parts, rowid):
    types = [t.code for t, _ in prog.cols] + [D.INT64]
    f = D.FilterHandle(ctx, types, prog.gpu_nodes(), [len(prog.cols)], 8192, -1)
    try:
        outs = []
        for lo, hi in parts:
            f.push_host(host_cols_with_rowid(prog, cols, lo, hi, rowid))
            outs += f.drain(host=True)
        f.finish()
        outs += f.drain(host=True)
        return batches_to_cols(outs, 1)[0][0].astype(np.int64), [o.num_rows for o in outs]
    finally:
        f.close()


def run_pipe_pred(ctx, prog, cols, parts, rowid, ordered):
    types = [t.code for t, _ in prog.cols] + [D.INT64]
    p = D.Pipeline(ctx, types, prog.gpu_nodes())
    try:
        p.sink_output([len(prog.cols)], ordered=ordered)
        for lo, hi in parts:
            p.push_host(host_cols_with_rowid(prog, cols, lo, hi, rowid))
        p.finish()
        got = batches_to_cols(p.drain(host=True), 1)[0][0].astype(np.int64)
        return got if ordered else np.sort(got)
    finally:
        p.close()


def agg_program(prog):
    """the aggregate argument and function for a value program: SUM over integers, MIN over Float64, Float32 / Boolean widened"""
    if prog.t.kind == "b":
        return G.Program(G.cast(prog.root, G.I32), prog.cols, prog.family, prog.seed), D.AGG_SUM
    if prog.t == G.F32:
        return G.Program(G.cast(prog.root, G.F64), prog.cols, prog.family, prog.seed), D.AGG_MIN
    return prog, D.AGG_MIN if prog.t.kind == "f" else D.AGG_SUM


def run_pipe_agg(ctx, prog, cols, parts, rowid):
    """the program as the argument of a hash-keyed aggregate grouped on a unique row id: {row id: value}"""
    aprog, func = agg_program(prog)
    types = [t.code for t, _ in prog.cols] + [D.INT64]
    p = D.Pipeline(ctx, types)
    try:
        p.sink_aggregate_hash([len(prog.cols)], [(func, aprog.gpu_nodes())], capacity_hint=max(len(rowid), 1))
        for lo, hi in parts:
            p.push_host(host_cols_with_rowid(prog, cols, lo, hi, rowid))
        p.finish()
        outs = p.drain(host=True)
        res = batches_to_cols(outs, 2)
        return aprog, dict(zip(res[0][0].tolist(), as_py(aprog.t if func == D.AGG_MIN else G.I64, res[1])))
    finally:
        p.close()


def small_mode(prog, cols):
    """pipeline.cu's choice for an aggregate argument: 3 Decimal128, 2 eval_int_fast, 1 eval_nodes_reg<4>, 0 eval_nodes"""
    if prog.has_decimal():
        return 3
    if prog.depth() > 4:
        return 0
    return 2 if prog.is_int_arith([val is not None for _, val in cols]) else 1


def pipe_refuses(prog):
    """the fused pipeline takes fixed-width input columns of 1-8 bytes (and Decimal128 ones inside expressions), not Boolean ones"""
    return any(t.kind == "b" for t, _ in prog.cols)


def assert_unsupported(fn, what):
    with pytest.raises(D.DfgpuError) as ei:
        fn()
    assert ei.value.code == -3, f"{what}: {ei.value}"                   # DFGPU_ERR_UNSUPPORTED


def pred_mode(prog):
    """pipeline.cu's predicate evaluator: conjunction, Decimal128, register stack or local-memory stack"""
    nodes = prog.gpu_nodes()
    i, depth, ok = 0, 0, True
    while i < len(nodes) and ok:
        if i + 2 < len(nodes) and nodes[i][0] == D.EXPR_COLUMN and nodes[i + 1][0] == D.EXPR_LITERAL and nodes[i + 2][0] == D.EXPR_BINARY \
                and D.OP_EQ <= nodes[i + 2][1] <= D.OP_GTEQ and not nodes[i + 1][3]:
            t = prog.cols[nodes[i][1]][0]
            if t.kind not in "iud" or prog.has_decimal():
                ok = False
                break
            depth += 1
            i += 3
        elif nodes[i][0] == D.EXPR_BINARY and nodes[i][1] == D.OP_AND and depth >= 2:
            depth -= 1
            i += 1
        else:
            ok = False
    if ok and depth == 1:
        return "conjunction"
    return "decimal" if prog.has_decimal() else ("reg4" if prog.depth() <= 4 else "stack")


def programs(family, count, seed0):
    """(program, n rows, rng) triples: Boolean and value programs, every depth around the register-stack limit, conjunctions"""
    for k in range(count):
        seed = seed0 + k
        gen = G.Gen(seed)
        rng = np.random.default_rng(seed)
        if family == "raising":
            prog = gen.raising(G.BOOL if k % 3 else VALUE_ROOTS[k % len(VALUE_ROOTS)])
        elif k % 10 == 0:
            prog = gen.conjunction(1 + k % 4)
        elif k % 10 == 1:
            prog = gen.int_arith(G.INTS[k % 8])
        elif k % 10 in (2, 3):
            prog = gen.at_depth(G.BOOL if k % 2 else VALUE_ROOTS[k % len(VALUE_ROOTS)], 4 + k % 2)
        else:
            prog = gen.total(G.BOOL if k % 2 else VALUE_ROOTS[k % len(VALUE_ROOTS)], 6)
        yield prog, ROWS[k % len(ROWS)], rng


# ---------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["total", "raising"])
def test_evaluate_host_and_device(gpu_ctx, family):
    """dfgpu_expr_evaluate_host and _device: values and validity (or the error) equal the oracle's, and each other's"""
    reached = collections.Counter()
    for k, (prog, n, rng) in enumerate(programs(family, N_PROGRAMS, 1000 if family == "total" else 5000)):
        cols = G.gen_columns(prog, n, rng)
        exp = oracle_outcome(prog, cols)
        host = outcome(lambda: run_evaluate(gpu_ctx, prog, cols, n, offset=(0, 13, 3)[k % 3]))
        compare_outcomes(prog, "dfgpu_expr_evaluate_host", cols, exp, host)
        if n > 0:
            dev = outcome(lambda: run_evaluate(gpu_ctx, prog, cols, n, device=True, offset=(0, 3, 13)[k % 3]))
            compare_outcomes(prog, "dfgpu_expr_evaluate_device", cols, exp, dev)
            compare_outcomes(prog, "host vs device", cols, host, dev)
        reached["decimal" if prog.has_decimal() else "eval_nodes"] += 1
        reached[exp[0] if exp[0] == "ok" else exp[1]] += 1
    want = {"decimal", "eval_nodes", "ok"} | ({"divide by zero", "arithmetic overflow", "cast error"} if family == "raising" else set())
    assert want <= set(reached), reached


def test_int64_to_float32_cast_rounds_once(gpu_ctx):
    """CAST(Int64 | UInt64 AS Float32) rounds once, like Rust's `as f32`, on every interpreter that evaluates it"""
    cases = [(G.I64, [G.W60, -G.W60, (1 << 24) + 3, -(1 << 63), (1 << 63) - 1], [0x5D800001, 0xDD800001, 0x4B800002, 0xDF000000, 0x5F000000]),
             (G.U64, [G.W63, (1 << 64) - 1, (1 << 53) + 1], [0x5F000001, 0x5F800000, 0x5A000000])]
    for t, xs, bits in cases:
        prog = G.Program(G.cast(G.Expr("col", t, col=0), G.F32), [(t, False)])
        cols = [(np.array(xs, t.np), None)]
        for device in (False, True):
            v, _ = run_evaluate(gpu_ctx, prog, cols, len(xs), device=device)
            assert v.view(np.uint32).tolist() == bits, (t.name, device, [hex(b) for b in v.view(np.uint32)])
        dec = G.Program(G.cast(G.Expr("col", t, col=0), G.F32), [(t, False), (G.DEC, False)])   # the Decimal128 interpreter casts too
        dprog = G.Program(G.binary(O.OP_AND, G.binary(O.OP_EQ, G.Expr("col", G.DEC, col=1), G.Expr("col", G.DEC, col=1)),
                                   G.binary(O.OP_EQ, dec.root, G.lit(float(np.array(xs, t.np).astype(np.float32)[0]), G.F32))), dec.cols)
        v, _ = run_evaluate(gpu_ctx, dprog, cols + [([0] * len(xs), None)], len(xs))
        assert bool(v[0]), (t.name, "decimal interpreter")
        for ordered in (True, False):      # the pipeline's register-stack interpreter, through a predicate
            got = run_pipe_pred(gpu_ctx, G.Program(dprog.root.kids[1], prog.cols), cols, [(0, len(xs))], np.arange(len(xs), dtype=np.int64), ordered)
            assert 0 in got.tolist(), (t.name, "pipeline predicate")


@pytest.mark.parametrize("family", ["total", "raising"])
def test_filter_and_pipeline_predicate(gpu_ctx, family):
    """Boolean programs as FilterExec's predicate and as the fused pipeline's (sink_output ordered and unordered), over 1-3 pushes:
    the kept row ids equal the oracle's, or both raise the same error class over the same push"""
    reached = collections.Counter()
    k = 0
    for prog, n, rng in programs(family, 2 * N_PROGRAMS, 20_000 if family == "total" else 30_000):
        if prog.t != G.BOOL:
            continue
        k += 1
        cols = G.gen_columns(prog, n, rng)
        parts = pushes(n, rng)
        rowid = np.arange(n, dtype=np.int64)
        exp = per_push_oracle(prog, cols, parts)
        got_f = outcome(lambda: run_filter(gpu_ctx, prog, cols, parts, rowid))
        if exp[0] != got_f[0] or (exp[0] == "err" and exp[1] != got_f[1]):
            fail(prog, f"FilterExec over pushes {parts}", cols, None, exp if exp[0] == "err" else "rows", got_f if got_f[0] == "err" else "rows")
        if exp[0] == "ok":
            want = rowid[exp[1]]
            ids, sizes = got_f[1]
            if not np.array_equal(ids, want):
                bad = next((i for i in range(min(len(ids), len(want))) if ids[i] != want[i]), min(len(ids), len(want)))
                fail(prog, f"FilterExec over pushes {parts}", cols, int(want[bad]) if bad < len(want) else None, want[bad:bad + 3].tolist(), ids[bad:bad + 3].tolist())
            assert all(s == 8192 for s in sizes[:-1]) and (not sizes or 0 < sizes[-1] <= 8192), sizes
        if pipe_refuses(prog):
            assert_unsupported(lambda: run_pipe_pred(gpu_ctx, prog, cols, parts, rowid, True), prog.describe())
            reached["refused"] += 1
            continue
        for ordered in (True, False):
            got_p = outcome(lambda: run_pipe_pred(gpu_ctx, prog, cols, parts, rowid, ordered))
            path = f"pipeline predicate ({pred_mode(prog)}, {'ordered' if ordered else 'unordered'}) over pushes {parts}"
            if exp[0] != got_p[0] or (exp[0] == "err" and exp[1] != got_p[1]):
                fail(prog, path, cols, None, exp if exp[0] == "err" else "rows", got_p if got_p[0] == "err" else "rows")
            if exp[0] == "ok" and not np.array_equal(got_p[1], rowid[exp[1]]):
                diff = np.setxor1d(got_p[1], rowid[exp[1]])
                fail(prog, path, cols, int(diff[0]) if len(diff) else None, "row kept" if len(diff) and exp[1][diff[0]] else "row dropped", "the other")
        reached[pred_mode(prog)] += 1
        nodes = prog.gpu_nodes()
        if len(nodes) == 3 and prog.cols[nodes[0][1]] == (G.I64, False) and nodes[1][0] == D.EXPR_LITERAL and not nodes[1][3] and D.OP_EQ <= nodes[2][1] <= D.OP_GTEQ:
            reached["cmp_i64_scalar"] += 1
        reached[exp[0] if exp[0] == "ok" else exp[1]] += 1
    want = {"decimal", "reg4", "ok"} | ({"divide by zero", "arithmetic overflow", "cast error"} if family == "raising" else {"conjunction", "stack"})
    assert want <= set(reached), reached


def test_scalar_int64_compare_paths(gpu_ctx):
    """`Int64 column <cmp> literal` without NULLs: FilterExec's scalar compare kernel, at row counts around its 512-row tiles"""
    rng = np.random.default_rng(7)
    for n in (1, 511, 512, 513, 1025, 8193):
        for op in (O.OP_EQ, O.OP_NEQ, O.OP_LT, O.OP_LTEQ, O.OP_GT, O.OP_GTEQ):
            edges = G.int_edges(G.I64)
            lv = edges[int(rng.integers(len(edges)))]
            prog = G.Program(G.binary(op, G.Expr("col", G.I64, col=0), G.lit(lv, G.I64)), [(G.I64, False)])
            cols = [(np.array([edges[i] if rng.random() < 0.5 else int(rng.integers(-5, 5)) for i in rng.integers(0, len(edges), n)], np.int64), None)]
            rowid = np.arange(n, dtype=np.int64)
            want = rowid[truth(O.eval_expr(G.oracle_cols(prog, cols), prog.oracle_nodes()))]
            ids, _ = run_filter(gpu_ctx, prog, cols, [(0, n)], rowid)
            assert np.array_equal(ids, want), prog.describe()
            assert np.array_equal(run_pipe_pred(gpu_ctx, prog, cols, [(0, n)], rowid, True), want), prog.describe()


@pytest.mark.parametrize("nulls", [False, True])
def test_pipeline_aggregate_argument(gpu_ctx, nulls):
    """value programs as the argument of a hash-keyed aggregate grouped on a unique row id, so each group holds one row: the group's
    SUM / MIN is the row's value.  Without NULLs in the batch, + - * programs take eval_int_fast; depth 4 and its padded depth-5 twin
    take eval_nodes_reg<4> and eval_nodes, and agree"""
    reached = collections.Counter()
    for k, (prog, n, rng) in enumerate(programs("total", N_PROGRAMS, 40_000 + 1000 * nulls)):
        if n == 0:
            continue
        cols = G.gen_columns(prog, n, rng, null_rate=0.2 if nulls else 0.0)
        if not nulls:
            cols = [(v, None) for v, _ in cols]
        if pipe_refuses(prog):
            assert_unsupported(lambda: run_pipe_agg(gpu_ctx, prog, cols, pushes(n, rng), np.arange(n, dtype=np.int64)), prog.describe())
            reached["refused"] += 1
            continue
        variants = [prog] + ([G.padded(prog)] if prog.depth() == 4 and prog.t.kind in "iufb" else [])
        results = []
        for pv in variants:
            parts = pushes(n, rng)
            rowid = np.arange(n, dtype=np.int64)
            aprog, got = run_pipe_agg(gpu_ctx, pv, cols, parts, rowid)
            exp = as_py(aprog.t, O.eval_expr(G.oracle_cols(aprog, cols), aprog.oracle_nodes()))
            mode = small_mode(aprog, cols if nulls else [(v, None) for v, _ in cols])
            path = f"pipeline aggregate argument (small {mode}) over pushes {parts}"
            t = aprog.t if aprog.t.kind == "f" else G.U64         # a one-row SUM: the value, compared modulo 2^64
            for i in range(n):
                e, g = exp[i], got.get(i)
                if t == G.U64:
                    e, g = (None if e is None else int(e) % (1 << 64)), (None if g is None else int(g) % (1 << 64))
                if not same(t, e, g):
                    fail(aprog, path, cols, i, e, g)
            reached[mode] += 1
            results.append(got)
        if len(results) == 2:
            for i in range(n):
                if not same(G.F64 if prog.t.kind == "f" else G.U64, results[0].get(i), results[1].get(i)):
                    fail(prog, "depth 4 vs depth 5", cols, i, results[0].get(i), results[1].get(i))
            reached["depth 4 vs 5"] += 1
    want = {0, 1, 3, "depth 4 vs 5"} | ({2} if not nulls else set())
    assert want <= set(reached), reached


# payload sets: every width and sign a 64-bit payload word carries
PAYLOADS = [[G.I8, G.I16, G.U8, G.U16], [G.F32, G.U32], [G.DATE32, G.I16, G.I8], [G.I32, G.U16, G.U8], [G.I64], [G.F64], [G.U64]]
PROBE = [(G.I8, True), (G.I16, False), (G.U8, False), (G.U16, True), (G.I32, False), (G.U32, True), (G.I64, True), (G.U64, False),
         (G.F32, False), (G.F64, True), (G.DATE32, False)]


def build_side(ctx, pays, nb, rng):
    """a lookup of the unique keys 0..nb-1 with payload columns of the given types (edge values included)"""
    vals = [G.gen_values(t, nb, rng) for t in pays]
    look = D.Lookup(ctx, D.INT64, [t.code for t in pays], expected_rows=nb)
    p = D.Pipeline(ctx, [D.INT64] + [t.code for t in pays])
    p.sink_build(look, 0, list(range(1, len(pays) + 1)))
    p.push_host([D.HostColumn(np.arange(nb, dtype=np.int64))] + [D.HostColumn(v, None, t.code) for v, t in zip(vals, pays)])
    p.finish()
    p.close()
    return look, vals


@pytest.mark.parametrize("pset", range(len(PAYLOADS)))
def test_stage_filter_and_payload_fields(gpu_ctx, pset):
    """filters of INNER and SEMI probe stages that read payload fields of every width and sign, and eval_int_fast aggregate arguments that
    read them over an INNER stage: joined rows and per-row values against the oracle over the joined columns"""
    pays = PAYLOADS[pset]
    rng = np.random.default_rng(70 + pset)
    nb, n = 700, 1537
    look, pvals = build_side(gpu_ctx, pays, nb, rng)
    probe_schema = [(t, nul) for t, nul in PROBE if rng.random() < 0.5][:6]
    nin = 1 + len(probe_schema)                       # the probe key, then the program's input columns
    schema = probe_schema + [(t, False) for t in pays]
    reached = collections.Counter()
    try:
        for k in range(40):
            gen = G.Gen(90_000 + 100 * pset + k, schema=schema, decimals=False)
            prog = gen.total(G.BOOL, 6) if k % 4 else gen.at_depth(G.BOOL, 4 + k % 8 // 4)
            if not any(e.kind == "col" and e.col >= len(probe_schema) for e in prog.root.post()):
                j = len(probe_schema) + k % len(pays)             # read a payload field: `p <op> (payload <cmp> literal)`
                cmp = G.binary(G.CMP_OPS[k % 6], G.Expr("col", pays[j - len(probe_schema)], col=j), gen.literal(pays[j - len(probe_schema)], allow_null=False))
                prog = G.Program(G.binary(O.OP_AND if k % 2 else O.OP_OR, prog.root, cmp), schema, "total", prog.seed)
            key = rng.integers(0, nb + 50, n).astype(np.int64)          # a few keys miss
            hit = key < nb
            icols = G.gen_columns(G.Program(prog.root, probe_schema), n, rng)
            joined = icols + [(np.asarray(v)[np.minimum(key, nb - 1)], None) for v in pvals]
            m = truth(O.eval_expr(G.oracle_cols(prog, joined), prog.oracle_nodes())) & hit
            col_map = [1 + c for c in range(len(probe_schema))] + [nin + 1 + j for j in range(len(pays))]   # row id sits at nin
            nodes = prog.gpu_nodes(col_map)
            types = [D.INT64] + [t.code for t, _ in probe_schema] + [D.INT64]
            rowid = np.arange(n, dtype=np.int64)
            if G.guarded(prog):
                p = D.Pipeline(gpu_ctx, types, None, [(D.STAGE_INNER, 0, look)])
                try:
                    assert_unsupported(lambda: p.set_stage_filter(0, nodes), prog.describe())
                finally:
                    p.close()
                reached["refused"] += 1
                continue
            for kind in (D.STAGE_INNER, D.STAGE_SEMI):
                p = D.Pipeline(gpu_ctx, types, None, [(kind, 0, look)])
                try:
                    p.set_stage_filter(0, nodes)
                    p.sink_output([nin] + ([nin + 1 + j for j in range(len(pays))] if kind == D.STAGE_INNER else []), ordered=True)
                    for lo, hi in pushes(n, rng):
                        p.push_host([D.HostColumn(key[lo:hi])] + G.host_columns(G.Program(prog.root, probe_schema), icols, lo, hi) + [D.HostColumn(rowid[lo:hi])])
                    p.finish()
                    out = batches_to_cols(p.drain(host=True), 1 + (len(pays) if kind == D.STAGE_INNER else 0))
                finally:
                    p.close()
                ids = out[0][0].astype(np.int64)
                path = f"{'INNER' if kind == D.STAGE_INNER else 'SEMI'} stage filter over payload {[t.name for t in pays]}"
                if not np.array_equal(ids, rowid[m]):
                    diff = np.setxor1d(ids, rowid[m])
                    fail(prog, path, joined, int(diff[0]), bool(m[diff[0]]), not m[diff[0]])
                if kind == D.STAGE_INNER:
                    for j, t in enumerate(pays):
                        compare_values(prog, path + f" (payload field {j} of the output)", joined, (np.asarray(pvals[j])[key[m]], None), out[1 + j], t)
                reached[("reg4" if prog.depth() <= 4 else "stack", kind)] += 1
        # eval_int_fast over payload fields: + - * programs over the integer payload fields and the non-NULL input columns
        in_sch = [(x, False) for x, nul in probe_schema if not nul]
        sch = in_sch + [(x, False) for x in pays]
        ints = [x for x in pays if x.is_int]
        for k in range(12 if ints else 0):
            t = ints[k % len(ints)]
            prog = G.Gen(95_000 + 100 * pset + k, schema=sch, decimals=False).int_arith(t, 3)
            if not any(e.kind == "col" and e.col >= len(in_sch) for e in prog.root.post()):
                continue
            key = rng.integers(0, nb, n).astype(np.int64)
            icols = G.gen_columns(G.Program(prog.root, in_sch), n, rng)
            joined = icols + [(np.asarray(v)[key], None) for v in pvals]
            exp = as_py(t, O.eval_expr(G.oracle_cols(prog, joined), prog.oracle_nodes()))
            nin2 = 1 + len(in_sch)
            col_map = [1 + c for c in range(len(in_sch))] + [nin2 + 1 + j for j in range(len(pays))]
            p = D.Pipeline(gpu_ctx, [D.INT64] + [x.code for x, _ in in_sch] + [D.INT64], None, [(D.STAGE_INNER, 0, look)])
            try:
                p.sink_aggregate_hash([nin2], [(D.AGG_SUM, prog.gpu_nodes(col_map))], capacity_hint=n)
                rowid = np.arange(n, dtype=np.int64)
                p.push_host([D.HostColumn(key)] + G.host_columns(G.Program(prog.root, in_sch), icols) + [D.HostColumn(rowid)])
                p.finish()
                res = batches_to_cols(p.drain(host=True), 2)
            finally:
                p.close()
            got = dict(zip(res[0][0].tolist(), res[1][0].tolist()))
            for i in range(n):
                if int(exp[i]) % (1 << 64) != int(got[i]) % (1 << 64):
                    fail(prog, "eval_int_fast aggregate argument over payload fields", joined, i, exp[i], got[i])
            reached["eval_int_fast"] += 1
    finally:
        look.close()
    assert any(k != "refused" for k in reached), reached
    if any(t.is_int for t in pays):
        assert reached["eval_int_fast"] > 0, reached


def test_stage_filter_rejects_guarded_programs(gpu_ctx):
    """a stage filter whose AND / OR has a right operand that can raise is refused with DFGPU_ERR_UNSUPPORTED"""
    look, _ = build_side(gpu_ctx, [G.I32], 10, np.random.default_rng(1))
    try:
        n_ok = 0
        for k in range(60):
            prog = G.Gen(7000 + k).raising(G.BOOL)
            guarded = G.guarded(prog)
            p = D.Pipeline(gpu_ctx, [D.INT64] + [t.code for t, _ in prog.cols], None, [(D.STAGE_INNER, 0, look)])
            try:
                try:
                    p.set_stage_filter(0, prog.gpu_nodes([1 + c for c in range(len(prog.cols))]))
                    assert not guarded, f"a guarded stage filter was accepted: {prog.describe()}"
                except D.DfgpuError as ex:
                    assert guarded and ex.code == -3, f"{ex}: {prog.describe()}"
                    n_ok += 1
            finally:
                p.close()
        assert n_ok > 0
    finally:
        look.close()


def test_hash_join_filter(gpu_ctx):
    """Boolean programs as a hash join's JoinFilter over build and probe columns: the joined pairs equal the oracle's over the pairs"""
    reached = collections.Counter()
    for k, (prog, n, rng) in enumerate(programs("total", 2 * N_PROGRAMS, 60_000)):
        if prog.t != G.BOOL or n == 0 or len(prog.cols) < 1:
            continue
        side = rng.integers(0, 2, len(prog.cols))                  # 0: the column comes from the build side, 1: from the probe side
        nb = max(1, n // 3)
        bcols = G.gen_columns(prog, nb, rng)
        pcols = G.gen_columns(prog, n, rng)
        key = rng.integers(0, nb, n).astype(np.int64)
        pair = [(bcols[c][0][key] if prog.cols[c][0].kind != "x" else [bcols[c][0][i] for i in key],
                 None if bcols[c][1] is None else bcols[c][1][key]) if side[c] == 0 else pcols[c] for c in range(len(prog.cols))]
        m = truth(O.eval_expr(G.oracle_cols(prog, pair), prog.oracle_nodes()))
        bt = [D.INT64] + [t.code for t, _ in prog.cols]
        pt = [D.INT64] + [t.code for t, _ in prog.cols] + [D.INT64]
        j = D.HashJoinHandle(gpu_ctx, bt, pt, [0], [0], [1, 0], [len(prog.cols) + 1, 0], D.JOIN_INNER)
        try:
            j.set_filter([int(s) for s in side], [1 + c for c in range(len(prog.cols))], prog.gpu_nodes())
            j.push_build_host([D.HostColumn(np.arange(nb, dtype=np.int64))] + G.host_columns(prog, bcols))
            j.finish_build()
            outs = []
            rowid = np.arange(n, dtype=np.int64)
            for lo, hi in pushes(n, rng):
                j.push_probe_host([D.HostColumn(key[lo:hi])] + G.host_columns(prog, pcols, lo, hi) + [D.HostColumn(rowid[lo:hi])])
                outs += j.drain(host=True)
            j.finish_probe()
            outs += j.drain(host=True)
            got = batches_to_cols(outs, 2)
        finally:
            j.close()
        ids = got[0][0].astype(np.int64)
        if not np.array_equal(np.sort(ids), rowid[m]) or not np.array_equal(got[1][0].astype(np.int64)[np.argsort(ids, kind="stable")], key[np.sort(ids)]):
            diff = np.setxor1d(ids, rowid[m])
            fail(G.Program(prog.root, prog.cols), f"hash join filter (sides {side.tolist()})", pair, int(diff[0]) if len(diff) else None,
                 "pair kept" if len(diff) and m[diff[0]] else "pair dropped", "the other")
        reached["join_filter"] += 1
        reached["decimal" if prog.has_decimal() else "eval_nodes"] += 1
    assert {"join_filter", "decimal", "eval_nodes"} <= set(reached), reached


def test_ring_fed_aggregate_gathered(gpu_ctx):
    """a Q3-shaped join-keyed aggregate over an INNER stage, with a conjunction predicate and a + - * SUM argument over narrow integer
    columns: the ring-fed kernel evaluates it with eval_int_gathered; group sums against the oracle"""
    rng = np.random.default_rng(11)
    nb, n = 3000, 50_003
    bk = np.arange(1, nb + 1, dtype=np.int64) * 3
    b8, b16 = G.gen_values(G.I8, nb, rng), G.gen_values(G.I16, nb, rng)

    def orders():
        """the build side; the aggregate accumulates into its records, so every program gets a fresh one"""
        look = D.Lookup(gpu_ctx, D.INT64, [D.INT8, D.INT16], n_acc_words=2, membership_filter=1)
        bp = D.Pipeline(gpu_ctx, [D.INT64, D.INT8, D.INT16])
        bp.sink_build(look, 0, [1, 2])
        bp.push_host([D.HostColumn(bk), D.HostColumn(b8, None, D.INT8), D.HostColumn(b16, None, D.INT16)])
        bp.finish()
        bp.close()
        return look

    schema = [(G.I64, False), (G.I8, False), (G.I16, False), (G.U16, False), (G.I32, False)]
    launches = 0
    for k in range(12):
        look = orders()
        try:
            gen = G.Gen(123_000 + k, schema=schema[1:], decimals=False)
            t = (G.I8, G.I16, G.U16, G.I32)[k % 4]
            prog = gen.int_arith(t, 3)
            cols = [(rng.integers(0, nb * 3 + 300, n).astype(np.int64), None)] + [(G.gen_values(x, n, rng), None) for x, _ in schema[1:]]
            lo8, hi16 = int(rng.integers(-100, 0)), int(rng.integers(0, 30000))
            pred = [(D.EXPR_COLUMN, 1, 0, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.INT8, 0, lo8, 0.0), (D.EXPR_BINARY, D.OP_GT, 0, 0, 0, 0.0),
                    (D.EXPR_COLUMN, 2, 0, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.INT16, 0, hi16, 0.0), (D.EXPR_BINARY, D.OP_LT, 0, 0, 0, 0.0),
                    (D.EXPR_BINARY, D.OP_AND, 0, 0, 0, 0.0)]
            p = D.Pipeline(gpu_ctx, [x.code for x, _ in schema], pred, [(D.STAGE_INNER, 0, look)])
            try:
                p.sink_aggregate([0], [(D.AGG_SUM, prog.gpu_nodes([1 + c for c in range(4)]))])
                p.push_host([D.HostColumn(v, None, x.code) for (x, _), (v, _) in zip(schema, cols)])
                p.finish()
                launches += p.metric("ring_launches")
                res = batches_to_cols(p.drain(host=True), 2)
            finally:
                p.close()
            keep = (cols[1][0].astype(np.int64) > lo8) & (cols[2][0].astype(np.int64) < hi16) & (cols[0][0] % 3 == 0) & (cols[0][0] >= 3) & (cols[0][0] <= 3 * nb)
            vals = as_py(t, O.eval_expr(G.oracle_cols(G.Program(prog.root, schema[1:]), cols[1:]), prog.oracle_nodes()))
            exp = collections.defaultdict(int)
            for i in np.nonzero(keep)[0]:
                exp[int(cols[0][0][i])] = (exp[int(cols[0][0][i])] + int(vals[i])) % (1 << 64)
            got = {int(a): int(b) % (1 << 64) for a, b in zip(res[0][0].tolist(), res[1][0].tolist())}
            assert got == dict(exp), f"ring-fed SUM: {G.Program(prog.root, schema[1:], seed=prog.seed).describe()}\n keys differing: {sorted(set(got.items()) ^ set(exp.items()))[:4]}"
        finally:
            look.close()
    assert launches > 0, "the ring-fed kernel never ran"
