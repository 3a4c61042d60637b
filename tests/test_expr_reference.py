"""A row-by-row scalar restatement of PhysicalExpr::evaluate, and the oracle's eval_expr checked against it on generated programs.

The scalar evaluator keeps integers as Python ints wrapped to their type's width after every operation, divides with Rust's truncation
on exact ints, runs float operations on np.float32 / np.float64 scalars, and rounds an integer -> float cast exactly once (Rust's
`as f32` / `as f64`).  AND / OR follow BinaryExpr::evaluate over the batch (binary.rs:536-600, check_short_circuit :1182-1290), which
decides on which rows an error inside the right operand can surface.  Within one operator, a zero divisor is reported before
`MIN / -1`, as the oracle and the GPU do.
"""
import math

import numpy as np
import pytest

import expr_gen as G
from oracle import oracle as O

I64_MIN = -(1 << 63)


class Div0(Exception):
    pass


class Overflow(Exception):
    pass


class CastErr(Exception):
    pass


ORACLE_ERR = {O.ArrowDivideByZero: Div0, O.ArrowArithmeticOverflow: Overflow, O.ArrowCastError: CastErr}


def wrap(x: int, t: G.Ty) -> int:
    m = 1 << t.bits
    return ((x - t.lo) % m) + t.lo


def int_to_f32(x: int) -> np.float32:
    """round an integer to the nearest Float32, ties to even, in one step"""
    a = abs(x)
    if a.bit_length() > 24:
        sh = a.bit_length() - 24
        q, r = divmod(a, 1 << sh)
        half = 1 << (sh - 1)
        if r > half or (r == half and q & 1):
            q += 1
        a = q << sh
    return np.float32(float(-a if x < 0 else a))     # <= 25 significant bits: exact in a double, exact in a float


def to_float(x, src: G.Ty, t: G.Ty):
    if src.kind == "f":
        with np.errstate(all="ignore"):
            return t.np(x)
    if src.kind == "x":
        with np.errstate(all="ignore"):
            return t.np(np.float64(float(x)) / np.float64(10.0 ** src.s))      # (x as f64 / 10^s) as f32: the reference rounds twice
    x = int(x)
    return int_to_f32(x) if t.bits == 32 else np.float64(float(x))           # Python's int -> float rounds once, ties to even


def total_key(x) -> int:
    x = np.float64(x)
    if x == 0:
        x = np.float64(0.0)
    b = int(np.array([x]).view(np.int64)[0])
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


def cast_scalar(v, src: G.Ty, t: G.Ty):
    if t.kind == "f":
        return to_float(v, src, t)
    if t.kind == "b":
        return bool(v != 0)
    if t.kind == "x":
        x = int(v) * 10 ** t.s
        if abs(x) >= 10 ** t.p:
            raise CastErr
        return x
    if src.kind == "f":
        if not math.isfinite(v):
            raise CastErr
        x = math.trunc(float(v))
    elif src.kind == "x":
        q = abs(int(v)) // 10 ** src.s
        x = q if v >= 0 else -q
    else:
        x = int(v)
    if not t.lo <= x <= t.hi:
        raise CastErr
    return x


def binary_scalar(op, t: G.Ty, a, b):
    """one row of a non-logical binary operator on non-NULL operands of type t"""
    if op in (O.OP_EQ, O.OP_NEQ, O.OP_LT, O.OP_LTEQ, O.OP_GT, O.OP_GTEQ):
        x, y = (total_key(a), total_key(b)) if t.kind == "f" else (a, b)
        return {O.OP_EQ: x == y, O.OP_NEQ: x != y, O.OP_LT: x < y, O.OP_LTEQ: x <= y, O.OP_GT: x > y, O.OP_GTEQ: x >= y}[op]
    if t.kind == "f":
        with np.errstate(all="ignore"):
            return {O.OP_PLUS: lambda: a + b, O.OP_MINUS: lambda: a - b, O.OP_MULTIPLY: lambda: a * b, O.OP_DIVIDE: lambda: a / b,
                    O.OP_MODULO: lambda: np.fmod(a, b)}[op]()
    if op == O.OP_PLUS:
        z = a + b
    elif op == O.OP_MINUS:
        z = a - b
    elif op == O.OP_MULTIPLY:
        z = a * b
    elif op in (O.OP_DIVIDE, O.OP_MODULO):
        q = abs(a) // abs(b)
        q = q if (a < 0) == (b < 0) else -q
        z = q if op == O.OP_DIVIDE else a - q * b
        if op == O.OP_DIVIDE and z > t.hi:
            raise Overflow
    elif op == O.OP_BITAND:
        z = a & b
    elif op == O.OP_BITOR:
        z = a | b
    elif op == O.OP_BITXOR:
        z = a ^ b
    elif op == O.OP_SHIFT_LEFT:
        z = a << (b & (t.bits - 1))
    else:
        z = a >> (b & (t.bits - 1))
    return wrap(z, t)


def dec_binary(op, lt: G.Ty, rt: G.Ty, a, b):
    if op in (O.OP_EQ, O.OP_NEQ, O.OP_LT, O.OP_LTEQ, O.OP_GT, O.OP_GTEQ):
        return binary_scalar(op, G.I64, a, b)
    _, _, le, re = O.decimal_result_type(op, lt.p, lt.s, rt.p, rt.s)
    x, y = a * 10 ** le, b * 10 ** re
    z = {O.OP_PLUS: x + y, O.OP_MINUS: x - y, O.OP_MULTIPLY: x * y}[op]
    if not -(1 << 127) <= z < (1 << 127):
        raise Overflow
    return z


def kleene(is_and, a, b):
    if is_and:
        return False if a is False or b is False else (True if a is True and b is True else None)
    return True if a is True or b is True else (False if a is False and b is False else None)


def evaluate(e: G.Expr, cols, n: int):
    """the values of e over a batch of n rows (None = NULL); cols[c] = list of n scalars.  Raises Div0 / Overflow / CastErr."""
    if e.kind == "col":
        return list(cols[e.col])
    if e.kind == "lit":
        v = None if e.null else (e.t.np(e.val) if e.t.kind == "f" else e.val)
        return [v] * n
    if e.kind == "bin" and e.op in (O.OP_AND, O.OP_OR):
        is_and = e.op == O.OP_AND
        l, r = e.kids
        lhs = evaluate(l, cols, n)
        if l.kind == "lit":                                       # a scalar left side always short-circuits unless NULL
            if l.null:
                return [kleene(is_and, a, b) for a, b in zip(lhs, evaluate(r, cols, n))]
            return lhs if l.val != is_and else evaluate(r, cols, n)
        if n == 0 or any(v is None for v in lhs):
            return [kleene(is_and, a, b) for a, b in zip(lhs, evaluate(r, cols, n))]
        tc = sum(1 for v in lhs if v)
        if (is_and and tc == 0) or (not is_and and tc == n):
            return lhs
        if (is_and and tc == n) or (not is_and and tc == 0):
            return evaluate(r, cols, n)
        rare = tc if is_and else n - tc
        if np.float32(rare) / np.float32(n) <= O.PRE_SELECTION_THRESHOLD:   # evaluate the right side on the pre-selected rows only
            sel = [i for i in range(n) if bool(lhs[i]) == is_and]
            rv = evaluate(r, [[c[i] for i in sel] for c in cols], len(sel))
            out = [not is_and] * n
            for i, v in zip(sel, rv):
                out[i] = v
            return out
        return [kleene(is_and, a, b) for a, b in zip(lhs, evaluate(r, cols, n))]
    if e.kind == "bin":
        l, r = e.kids
        a, b = evaluate(l, cols, n), evaluate(r, cols, n)
        if e.op in (O.OP_IS_DISTINCT_FROM, O.OP_IS_NOT_DISTINCT_FROM):
            out = []
            for x, y in zip(a, b):
                d = (x is None) != (y is None) or (x is not None and y is not None and
                                                     (dec_binary(O.OP_NEQ, l.t, r.t, x, y) if l.t.kind == "x" else binary_scalar(O.OP_NEQ, l.t, x, y)))
                out.append(d if e.op == O.OP_IS_DISTINCT_FROM else not d)
            return out
        if e.op in (O.OP_DIVIDE, O.OP_MODULO) and l.t.kind in "iu":
            if any(x is not None and y == 0 for x, y in zip(a, b)):
                raise Div0
            out = []
            for x, y in zip(a, b):
                out.append(None if x is None or y is None else binary_scalar(e.op, l.t, x, y))
            return out
        f = (lambda x, y: dec_binary(e.op, l.t, r.t, x, y)) if l.t.kind == "x" else (lambda x, y: binary_scalar(e.op, l.t, x, y))
        return [None if x is None or y is None else f(x, y) for x, y in zip(a, b)]
    a = evaluate(e.kids[0], cols, n)
    src = e.kids[0].t
    if e.kind == "not":
        return [None if x is None else not x for x in a]
    if e.kind == "is_null":
        return [x is None for x in a]
    if e.kind == "is_not_null":
        return [x is not None for x in a]
    if e.kind == "neg":
        return [None if x is None else (-x if src.kind in "fx" else wrap(-x, src)) for x in a]
    return [None if x is None else cast_scalar(x, src, e.t) for x in a]


def scalar_cols(prog: G.Program, cols):
    out = []
    for (t, _), (v, val) in zip(prog.cols, cols):
        vals = list(v) if t.kind == "x" else [bool(x) if t.kind == "b" else (x if t.kind == "f" else int(x)) for x in np.asarray(v)]
        out.append([None if (val is not None and not val[i]) else vals[i] for i in range(len(vals))])
    return out


def reference(prog: G.Program, cols, n: int):
    """('ok', [values]) or ('err', class)"""
    try:
        return "ok", evaluate(prog.root, scalar_cols(prog, cols), n)
    except (Div0, Overflow, CastErr) as ex:
        return "err", type(ex)


def oracle(prog: G.Program, cols):
    try:
        v, val = O.eval_expr(G.oracle_cols(prog, cols), prog.oracle_nodes())
    except tuple(ORACLE_ERR) as ex:
        return "err", ORACLE_ERR[type(ex)]
    n = len(v)
    if isinstance(v, O.Dec):
        vals = [int(x) for x in v]
    else:
        vals = list(np.asarray(v))
    return "ok", [None if (val is not None and not val[i]) else vals[i] for i in range(n)]


def same_value(t: G.Ty, a, b) -> bool:
    if a is None or b is None:
        return a is None and b is None
    if t.kind == "f":
        a, b = t.np(a), t.np(b)
        if np.isnan(a) and np.isnan(b):
            return True                  # NaN bits produced by arithmetic are unspecified (expr_gen's float rules)
        return np.array([a]).view(np.uint64 if t.bits == 64 else np.uint32)[0] == np.array([b]).view(np.uint64 if t.bits == 64 else np.uint32)[0]
    if t.kind == "b":
        return bool(a) == bool(b)
    return int(a) == int(b)


def check(prog, cols, n):
    exp = reference(prog, cols, n)
    got = oracle(prog, cols)
    assert exp[0] == got[0] and (exp[0] == "ok" or exp[1] == got[1]), f"{prog.describe()}\n reference {exp if exp[0] == 'err' else 'values'}, oracle {got if got[0] == 'err' else 'values'}"
    if exp[0] == "ok":
        for i, (a, b) in enumerate(zip(exp[1], got[1])):
            if not same_value(prog.t, a, b):
                row = [c[0][i] if c[1] is None or c[1][i] else None for c in cols]
                raise AssertionError(f"{prog.describe()}\n row {i}: inputs {row}\n reference {a!r}, oracle {b!r}")
    return exp[0] == "ok" or exp[1]


ROOTS = (G.BOOL,) * 4 + G.INTS + G.FLOATS


@pytest.mark.parametrize("chunk", range(8))
def test_oracle_matches_scalar_reference_total(chunk):
    """total programs never raise and the oracle's values equal the scalar reference's, row by row"""
    for seed in range(chunk * 250, (chunk + 1) * 250):
        gen = G.Gen(seed)
        rng = np.random.default_rng(seed)
        t = ROOTS[seed % len(ROOTS)]
        prog = gen.at_depth(t, 1 + seed % 6) if seed % 3 == 0 else gen.total(t, 6)
        n = (0, 1, 7, 40, 64)[seed % 5]
        assert check(prog, G.gen_columns(prog, n, rng), n) is True, prog.describe()


@pytest.mark.parametrize("chunk", range(4))
def test_oracle_matches_scalar_reference_raising(chunk):
    """raising programs: the oracle raises exactly when the scalar reference does, with the same error, over the same batch"""
    seen = set()
    for seed in range(chunk * 300, (chunk + 1) * 300):
        gen = G.Gen(100_000 + seed)
        rng = np.random.default_rng(seed)
        prog = gen.raising(G.BOOL if seed % 3 else G.I64)
        n = (1, 9, 40, 100)[seed % 4]
        seen.add(check(prog, G.gen_columns(prog, n, rng), n))
    assert seen >= {True, Div0, Overflow, CastErr}, seen       # every outcome occurs


def _lit(v, t):
    return G.lit(v, t)


def _run(root, cols):
    prog = G.Program(root, [(t, v[1] is not None) for t, v in cols])
    data = [v for _, v in cols]
    return reference(prog, data, len(data[0][0])), oracle(prog, data)


@pytest.mark.parametrize("x, y, q, r", [(I64_MIN, 2, -(1 << 62), 0), (I64_MIN, 3, -3074457345618258602, -2), (I64_MIN, -3, 3074457345618258602, -2),
                                        (I64_MIN + 1, -1, (1 << 63) - 1, 0), (I64_MIN, I64_MIN, 1, 0), (-7, 2, -3, -1)])
def test_int64_min_division_and_remainder(x, y, q, r):
    """truncating `/` and `%` at the type minimum, where np.abs overflows"""
    col = [(G.I64, (np.array([x], np.int64), None))]
    for op, want in ((O.OP_DIVIDE, q), (O.OP_MODULO, r)):
        ref, orc = _run(G.binary(op, G.Expr("col", G.I64, col=0), _lit(y, G.I64)), col)
        assert ref == ("ok", [want]) and orc[0] == "ok" and int(orc[1][0]) == want, (x, y, op, ref, orc)


@pytest.mark.parametrize("t", [G.I8, G.I16, G.I32, G.I64])
def test_min_divided_by_minus_one_overflows(t):
    """arrow's checked `div`: MIN / -1 is ArithmeticOverflow in every signed width; MIN % -1 is 0"""
    col = [(t, (np.array([t.lo, 5], t.np), None))]
    ref, orc = _run(G.binary(O.OP_DIVIDE, G.Expr("col", t, col=0), _lit(-1, t)), col)
    assert ref == ("err", Overflow) and orc == ("err", Overflow)
    with pytest.raises(O.ArrowArithmeticOverflow):
        O.eval_expr([(np.array([t.lo], t.np), None)], [(O.E_COLUMN, 0, None, 0, 0), (O.E_LITERAL, 0, np.dtype(t.np), 0, -1), (O.E_BINARY, O.OP_DIVIDE, None, 0, 0)])
    ref, orc = _run(G.binary(O.OP_MODULO, G.Expr("col", t, col=0), _lit(-1, t)), col)
    assert ref == ("ok", [0, 0]) and orc[0] == "ok" and [int(v) for v in orc[1]] == [0, 0]
    # a NULL row holding MIN does not raise
    col = [(t, (np.array([t.lo, 4], t.np), np.array([False, True])))]
    ref, orc = _run(G.binary(O.OP_DIVIDE, G.Expr("col", t, col=0), _lit(-1, t)), col)
    assert ref == ("ok", [None, -4]) and orc[0] == "ok" and orc[1][0] is None and int(orc[1][1]) == -4


@pytest.mark.parametrize("x, t, bits", [(G.W60, G.I64, 0x5D800001), (-G.W60, G.I64, 0xDD800001), (G.W63, G.U64, 0x5F000001),
                                        ((1 << 24) + 1, G.I32, 0x4B800000), ((1 << 24) + 3, G.I64, 0x4B800002), ((1 << 64) - 1, G.U64, 0x5F800000)])
def test_integer_to_float32_rounds_once(x, t, bits):
    """CAST(Int64 / UInt64 AS Float32) is Rust's `as f32`: one rounding.  Through a double, 2^60 + 2^36 + 1 would give 0x5d800000."""
    assert int(np.array([int_to_f32(x)]).view(np.uint32)[0]) == bits
    if abs(x) in (G.W60, G.W63):
        assert np.float32(float(x)).view(np.uint32) != bits                      # a double in between rounds these twice
    col = [(t, (np.array([x], t.np), None))]
    ref, orc = _run(G.cast(G.Expr("col", t, col=0), G.F32), col)
    assert ref[0] == orc[0] == "ok"
    assert int(np.array([ref[1][0]], np.float32).view(np.uint32)[0]) == bits
    assert int(np.array([orc[1][0]], np.float32).view(np.uint32)[0]) == bits


def test_int_to_f32_matches_numpy_on_random_integers():
    rng = np.random.default_rng(5)
    xs = [int(v) for v in rng.integers(-(1 << 63), (1 << 63) - 1, 20000, dtype=np.int64)] + [int(v) >> int(s) for v, s in
                                                                                              zip(rng.integers(-(1 << 63), (1 << 63) - 1, 5000, dtype=np.int64), rng.integers(0, 63, 5000))]
    got = np.array([int_to_f32(x) for x in xs], np.float32)
    assert np.array_equal(got.view(np.uint32), np.array(xs, np.int64).astype(np.float32).view(np.uint32))
    us = [int(v) for v in rng.integers(0, (1 << 64) - 1, 20000, dtype=np.uint64, endpoint=True)]
    got = np.array([int_to_f32(x) for x in us], np.float32)
    assert np.array_equal(got.view(np.uint32), np.array(us, np.uint64).astype(np.float32).view(np.uint32))


def test_generator_shapes():
    """the shapes the GPU paths are chosen by: a requested stack depth, plan_is_int_arith, a pure conjunction; and readable failures"""
    for seed in range(40):
        gen = G.Gen(seed)
        for d in (1, 2, 3, 4, 5, 6):
            p = gen.at_depth(G.BOOL if seed % 2 else G.I32, d)
            assert p.depth() == d and p.n_nodes() <= 40
            q = G.padded(p)
            assert q.depth() == d + 1
        assert gen.int_arith(G.INTS[seed % 8]).is_int_arith()
        c = gen.conjunction(1 + seed % 4)
        nodes = c.gpu_nodes()
        assert all(nodes[i][0] == 1 and nodes[i + 1][0] == 2 for i in range(0, 3, 3))
        r = gen.raising()
        assert r.family == "raising" and "RPN:" in r.describe() and str(seed) in r.describe()
