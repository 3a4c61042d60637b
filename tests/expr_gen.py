"""Seeded generator of typed PhysicalExpr programs and of the columns they run on (test infrastructure, no GPU).

A program is a typed expression tree.  It prints as infix and as the post-order (RPN) node lists of the C ABI and of the oracle.  Two
families:
- total: cannot raise.  An integer divisor is `((y & 7) | 1)`, never 0 or -1, and a cast to an integer type only sees values that fit.
- raising: exactly one node can raise (a division by a column holding 0, `MIN / -1`, or an out-of-range CAST), sometimes under an
  AND / OR whose left side decides per batch which rows the reference evaluates (binary.rs check_short_circuit).  One site per program
  keeps the error class determined: the reference reports the first failing row, the GPU the class of any failing row.

Float rules:
- the sign and payload of a NaN that arithmetic produces are not specified (x86 gives -NaN for inf - inf, the GPU +NaN), so a float
  comparison only sees columns, literals, casts and negations, and value results compare every NaN equal to every NaN;
- Float32 NaNs are quiet: whether a signalling NaN is quieted when it widens to f64 differs between paths and is out of scope.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from datafusion_b200 import capi as D
from oracle import oracle as O


@dataclass(frozen=True)
class Ty:
    name: str
    code: int                 # dfgpu type code
    kind: str                 # i signed int, u unsigned int, f float, b bool, d Date32, x Decimal128
    bits: int = 0
    p: int = 0
    s: int = 0

    @property
    def np(self):
        return {"b": np.bool_, "d": np.int32, "x": object}.get(self.kind) or np.dtype(f"{'int' if self.kind == 'i' else 'uint' if self.kind == 'u' else 'float'}{self.bits}").type

    @property
    def odt(self):            # the `dt` of an oracle literal / cast node
        return O.decimal_dtype(self.p, self.s) if self.kind == "x" else np.dtype(self.np)

    @property
    def lo(self):
        return -(1 << (self.bits - 1)) if self.kind in "id" else 0

    @property
    def hi(self):
        return (1 << (self.bits - 1)) - 1 if self.kind in "id" else (1 << self.bits) - 1

    @property
    def is_int(self):
        return self.kind in "iu"


I8, I16, I32, I64 = (Ty(f"Int{b}", c, "i", b) for b, c in ((8, D.INT8), (16, D.INT16), (32, D.INT32), (64, D.INT64)))
U8, U16, U32, U64 = (Ty(f"UInt{b}", c, "u", b) for b, c in ((8, D.UINT8), (16, D.UINT16), (32, D.UINT32), (64, D.UINT64)))
F32, F64 = Ty("Float32", D.FLOAT32, "f", 32), Ty("Float64", D.FLOAT64, "f", 64)
BOOL = Ty("Boolean", D.BOOL, "b", 1)
DATE32 = Ty("Date32", D.DATE32, "d", 32)
DEC = Ty("Decimal128(9, 2)", D.decimal128(9, 2), "x", 128, 9, 2)
INTS = (I8, I16, I32, I64, U8, U16, U32, U64)
FLOATS = (F32, F64)
ALL = INTS + FLOATS + (BOOL, DATE32, DEC)


def dec_ty(p, s):
    return DEC if (p, s) == (9, 2) else Ty(f"Decimal128({p}, {s})", D.decimal128(p, s), "x", 128, p, s)


CMP_OPS = (O.OP_EQ, O.OP_NEQ, O.OP_LT, O.OP_LTEQ, O.OP_GT, O.OP_GTEQ, O.OP_IS_DISTINCT_FROM, O.OP_IS_NOT_DISTINCT_FROM)
ARITH_OPS = (O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY, O.OP_DIVIDE, O.OP_MODULO)
BIT_OPS = (O.OP_BITAND, O.OP_BITOR, O.OP_BITXOR, O.OP_SHIFT_LEFT, O.OP_SHIFT_RIGHT)
OP_SYM = {O.OP_EQ: "=", O.OP_NEQ: "!=", O.OP_LT: "<", O.OP_LTEQ: "<=", O.OP_GT: ">", O.OP_GTEQ: ">=", O.OP_PLUS: "+", O.OP_MINUS: "-",
          O.OP_MULTIPLY: "*", O.OP_DIVIDE: "/", O.OP_MODULO: "%", O.OP_AND: "AND", O.OP_OR: "OR", O.OP_IS_DISTINCT_FROM: "IS DISTINCT FROM",
          O.OP_IS_NOT_DISTINCT_FROM: "IS NOT DISTINCT FROM", O.OP_BITAND: "&", O.OP_BITOR: "|", O.OP_BITXOR: "^", O.OP_SHIFT_LEFT: "<<",
          O.OP_SHIFT_RIGHT: ">>"}
UNARY = {"not": (O.E_NOT, D.EXPR_NOT), "is_null": (O.E_IS_NULL, D.EXPR_IS_NULL), "is_not_null": (O.E_IS_NOT_NULL, D.EXPR_IS_NOT_NULL),
         "neg": (O.E_NEGATIVE, D.EXPR_NEGATIVE)}


class Expr:
    __slots__ = ("kind", "op", "kids", "t", "col", "val", "null")

    def __init__(self, kind, t, op=0, kids=(), col=-1, val=None, null=False):
        self.kind, self.t, self.op, self.kids, self.col, self.val, self.null = kind, t, op, tuple(kids), col, val, null

    def infix(self, names=None) -> str:
        k = self.kind
        if k == "col":
            return names[self.col] if names else f"c{self.col}"
        if k == "lit":
            return f"NULL::{self.t.name}" if self.null else f"{self.val!r}::{self.t.name}"
        if k == "bin":
            return f"({self.kids[0].infix(names)} {OP_SYM[self.op]} {self.kids[1].infix(names)})"
        if k == "cast":
            return f"CAST({self.kids[0].infix(names)} AS {self.t.name})"
        a = self.kids[0].infix(names)
        return {"not": f"NOT {a}", "is_null": f"{a} IS NULL", "is_not_null": f"{a} IS NOT NULL", "neg": f"-{a}"}[k]

    def post(self):
        for c in self.kids:
            yield from c.post()
        yield self


def binary(op, l: Expr, r: Expr) -> Expr:
    assert l.t == r.t or (l.t.kind == "x" and r.t.kind == "x"), (OP_SYM[op], l.t, r.t)
    if op in CMP_OPS or op in (O.OP_AND, O.OP_OR):
        t = BOOL
    elif l.t.kind == "x":
        p, s, _, _ = O.decimal_result_type(op, l.t.p, l.t.s, r.t.p, r.t.s)
        t = dec_ty(p, s)
    else:
        t = l.t
    return Expr("bin", t, op, (l, r))


def cast(a: Expr, t: Ty) -> Expr:
    return Expr("cast", t, kids=(a,))


def lit(v, t: Ty, null=False) -> Expr:
    return Expr("lit", t, val=None if null else v, null=null)


def unary(kind, a: Expr) -> Expr:
    return Expr(kind, BOOL if kind in ("not", "is_null", "is_not_null") else a.t, kids=(a,))


def safe_divisor(y: Expr) -> Expr:
    """((y & 7) | 1): one of 1, 3, 5, 7 for every non-NULL y, so neither 0 nor -1"""
    return binary(O.OP_BITOR, binary(O.OP_BITAND, y, lit(7, y.t)), lit(1, y.t))


@dataclass
class Program:
    root: Expr
    cols: List[tuple]                     # [(Ty, nullable)] of the program's columns, by index
    family: str = "total"
    seed: int = 0
    zero_cols: tuple = ()                 # raising family: the divisor column, given extra zeros
    sel_cols: tuple = ()                  # raising family: the `sel < k` columns, given the values 0..99

    @property
    def t(self) -> Ty:
        return self.root.t

    def gpu_nodes(self, col_map=None):
        """[(kind, a, type, is_null, lit_i64, lit_f64)] for capi.expr_nodes; col_map renumbers the columns"""
        out = []
        for e in self.root.post():
            if e.kind == "col":
                out.append((D.EXPR_COLUMN, e.col if col_map is None else col_map[e.col], 0, 0, 0, 0.0))
            elif e.kind == "lit":
                if e.null:
                    out.append((D.EXPR_LITERAL, 0, e.t.code, 1, 0, 0.0))
                elif e.t.kind == "f":
                    out.append((D.EXPR_LITERAL, 0, e.t.code, 0, 0, float(e.val)))
                else:
                    v = int(e.val)
                    if e.t.kind != "x" and v >= 1 << 63:
                        v -= 1 << 64
                    out.append((D.EXPR_LITERAL, 0, e.t.code, 0, v, 0.0))
            elif e.kind == "bin":
                out.append((D.EXPR_BINARY, e.op, 0, 0, 0, 0.0))
            elif e.kind == "cast":
                out.append((D.EXPR_CAST, 0, e.t.code, 0, 0, 0.0))
            else:
                out.append((UNARY[e.kind][1], 0, 0, 0, 0, 0.0))
        return out

    def oracle_nodes(self, col_map=None):
        out = []
        for e in self.root.post():
            if e.kind == "col":
                out.append((O.E_COLUMN, e.col if col_map is None else col_map[e.col], None, 0, 0))
            elif e.kind == "lit":
                out.append((O.E_LITERAL, 0, e.t.odt, 1 if e.null else 0, 0 if e.null else (e.t.np(e.val) if e.t.kind == "f" else e.val)))
            elif e.kind == "bin":
                out.append((O.E_BINARY, e.op, None, 0, 0))
            elif e.kind == "cast":
                out.append((O.E_CAST, 0, e.t.odt, 0, 0))
            else:
                out.append((UNARY[e.kind][0], 0, None, 0, 0))
        return out

    def depth(self) -> int:
        """largest evaluation-stack depth (pipeline.cu plan_depth)"""
        sp = mx = 0
        for e in self.root.post():
            if e.kind in ("col", "lit"):
                sp += 1
            elif e.kind == "bin":
                sp -= 1
            mx = max(mx, sp)
        return mx

    def n_nodes(self) -> int:
        return sum(1 for _ in self.root.post())

    def is_int_arith(self, nullable_cols=None) -> bool:
        """pipeline.cu plan_is_int_arith: integer columns without NULLs in the batch, non-NULL literals, + - * only"""
        for e in self.root.post():
            if not e.t.is_int and e.t.kind != "d":
                return False
            if e.kind == "col":
                if (self.cols[e.col][1] if nullable_cols is None else nullable_cols[e.col]):
                    return False
            elif e.kind == "lit":
                if e.null:
                    return False
            elif e.kind == "bin":
                if e.op not in (O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY):
                    return False
            else:
                return False
        return True

    def has_decimal(self) -> bool:
        return any(e.t.kind == "x" or (e.kids and e.kids[0].t.kind == "x") for e in self.root.post())

    def describe(self) -> str:
        rpn = " ".join(_rpn_token(e, self) for e in self.root.post())
        cols = ", ".join(f"c{i}: {t.name}{'?' if nul else ''}" for i, (t, nul) in enumerate(self.cols))
        return f"[{self.family} program, seed {self.seed}] {self.root.infix()}\n  columns: {cols}\n  RPN: {rpn}"


def _rpn_token(e: Expr, prog: Program) -> str:
    if e.kind == "col":
        return f"c{e.col}"
    if e.kind == "lit":
        return "NULL" if e.null else repr(e.val)
    if e.kind == "bin":
        return OP_SYM[e.op].replace(" ", "_")
    if e.kind == "cast":
        return f"CAST:{e.t.name.replace(' ', '')}"
    return e.kind.upper()


# ---------------------------------------------------------------------------------------------
# column values
# ---------------------------------------------------------------------------------------------
W60 = (1 << 60) + (1 << 36) + 1              # Int64 -> Float32: one rounding gives 0x5d800001, two give 0x5d800000
W63 = (1 << 63) + (1 << 39) + 1              # UInt64 -> Float32: 9.2233731e18 against 9.2233720e18 through a double


def int_edges(t: Ty) -> List[int]:
    cand = [t.lo, t.lo + 1, -1, 0, 1, t.hi - 1, t.hi, 2, -2, 7, -8]
    for b in (24, 53, 63, 31, 15, 7):
        cand += [(1 << b) - 1, 1 << b, (1 << b) + 1, -(1 << b) - 1, -(1 << b), -(1 << b) + 1]
    cand += [W60, -W60, W63, (1 << 62) + 1]
    return sorted({v for v in cand if t.lo <= v <= t.hi})


def _f64_bits(b):
    return np.array([b], np.uint64).view(np.float64)[0]


F64_EDGES = [0.0, -0.0, 1.0, -1.0, 0.5, -2.5, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, 2.225073858507201e-308,
             3.4028234663852886e38, -3.4028234663852886e38, 3.5e38, -1e39, 1e300, 16777217.0, 9007199254740992.0, 9.223372036854775808e18,
             1.0000000596046448, 127.9, -128.9, 255.5, 1e-40, 4e9, -3e10]
F64_NANS = [_f64_bits(0x7FF8000000000000), _f64_bits(0xFFF8000000000000), _f64_bits(0x7FF8000000000123), _f64_bits(0xFFFC0000000ABCDE)]
F32_EDGES = [0.0, -0.0, 1.0, -1.0, 0.5, -2.5, math.inf, -math.inf, 1.401298464324817e-45, -1.401298464324817e-45, 1.1754943508222875e-38,
             3.4028234663852886e38, -3.4028234663852886e38, 16777216.0, 16777218.0, 127.5, -128.5, 1e-40]
F32_NANS = [np.array([0x7FC00000], np.uint32).view(np.float32)[0], np.array([0xFFC00000], np.uint32).view(np.float32)[0]]   # quiet only


def gen_values(t: Ty, n: int, rng, zero_rate: float = 0.0):
    """n values of type t: a third random over the whole domain, a third edge values, a third small values"""
    pick = rng.integers(0, 3, n)
    if t.kind in "iud":
        lo, hi = (t.lo, t.hi) if t.kind != "d" else (-200000, 200000)
        edges = int_edges(t)
        full = [int(x) for x in rng.integers(t.lo, t.hi, n, dtype=np.uint64 if t.kind == "u" else np.int64, endpoint=True)] if t.bits == 64 else \
            [int(x) for x in rng.integers(lo, hi + 1, n)]
        small = rng.integers(max(t.lo, -9), min(t.hi, 9) + 1, n)
        vals = [full[i] if pick[i] == 0 else (edges[rng.integers(len(edges))] if pick[i] == 1 else int(small[i])) for i in range(n)]
        out = np.array(vals, dtype=object).astype(t.np) if n else np.zeros(0, t.np)
    elif t.kind == "f":
        ft = t.np
        edges = [ft(x) for x in (F32_EDGES if t.bits == 32 else F64_EDGES)] + (F32_NANS if t.bits == 32 else F64_NANS)
        with np.errstate(all="ignore"):
            full = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 12, n)).astype(ft)
        small = rng.integers(-9, 10, n).astype(ft)
        out = np.empty(n, ft)
        for i in range(n):
            out[i] = full[i] if pick[i] == 0 else (edges[rng.integers(len(edges))] if pick[i] == 1 else small[i])
    elif t.kind == "b":
        out = rng.random(n) < 0.5
    else:
        lim = 10 ** t.p - 1
        out = [int(x) for x in rng.integers(-lim, lim + 1, n)]
        for i in range(n):
            if pick[i] == 1:
                out[i] = [lim, -lim, 0, 1, -1, 100, -100][rng.integers(7)]
            elif pick[i] == 2:
                out[i] = int(rng.integers(-999, 1000))
        return out
    if zero_rate and t.kind in "iuf":
        out[rng.random(n) < zero_rate] = 0
    return out


def gen_columns(prog: Program, n: int, rng, null_rate: float = 0.2):
    """[(values, valid or None)] for the program's columns (Decimal128 values are Python ints)"""
    cols = []
    for i, (t, nullable) in enumerate(prog.cols):
        v = gen_values(t, n, rng, 0.08 if i in prog.zero_cols else 0.0)
        if i in prog.sel_cols:              # `sel < k` is TRUE on about k % of the rows
            v = rng.integers(0, 100, n).astype(np.int32)
        cols.append((v, (rng.random(n) >= null_rate) if nullable else None))
    return cols


def oracle_cols(prog: Program, cols):
    out = []
    for (t, _), (v, val) in zip(prog.cols, cols):
        out.append((O.Dec(v, t.p, t.s) if t.kind == "x" else np.asarray(v), val))
    return out


def host_columns(prog: Program, cols, lo=0, hi=None):
    return [D.HostColumn(v[lo:hi] if t.kind != "x" else list(v[lo:hi]), None if val is None else val[lo:hi], t.code)
            for (t, _), (v, val) in zip(prog.cols, cols)]


# ---------------------------------------------------------------------------------------------
# programs
# ---------------------------------------------------------------------------------------------
class Gen:
    """gen = Gen(seed); gen.total(BOOL) / gen.total(I64) / gen.raising(BOOL) ...; schema= restricts the columns to a fixed list"""

    def __init__(self, seed: int, schema: Optional[Sequence[tuple]] = None, max_cols: int = 7, decimals: bool = True):
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.fixed = list(schema) if schema is not None else None
        self.max_cols = max_cols
        self.decimals = decimals
        self.cols: List[tuple] = []

    # -- leaves --
    def column(self, t: Ty, nullable=None) -> Optional[Expr]:
        r = self.rng
        if self.fixed is not None:
            idx = [i for i, (ct, nul) in enumerate(self.fixed) if ct == t and (nullable is None or nul == nullable)]
            return Expr("col", t, col=int(r.choice(idx))) if idx else None
        nul = bool(r.random() < 0.4) if nullable is None else nullable
        same = [i for i, c in enumerate(self.cols) if c == (t, nul)]
        if same and (r.random() < 0.5 or len(self.cols) >= self.max_cols):
            return Expr("col", t, col=int(r.choice(same)))
        if len(self.cols) >= self.max_cols:
            return None
        self.cols.append((t, nul))
        return Expr("col", t, col=len(self.cols) - 1)

    def literal(self, t: Ty, allow_null=True) -> Expr:
        r = self.rng
        if allow_null and r.random() < 0.05:
            return lit(None, t, null=True)
        if t.kind in "iu":
            e = int_edges(t)
            v = e[r.integers(len(e))] if r.random() < 0.4 else int(r.integers(max(t.lo, -20), min(t.hi, 20) + 1))
        elif t.kind == "d":
            v = int(r.integers(-200000, 200001))
        elif t.kind == "f":
            edges = [x for x in (F32_EDGES if t.bits == 32 else F64_EDGES) if not math.isnan(x)]
            v = float(t.np(edges[r.integers(len(edges))] if r.random() < 0.4 else round(float(r.standard_normal()) * 100, 2)))
        elif t.kind == "b":
            v = bool(r.random() < 0.5)
        else:
            v = int(r.integers(-10 ** t.p + 1, 10 ** t.p))
        return lit(v, t)

    def leaf(self, t: Ty, allow_null=True) -> Expr:
        if self.rng.random() < 0.7:
            c = self.column(t)
            if c is not None:
                return c
        return self.literal(t, allow_null)

    # -- typed expressions, total family --
    def expr(self, t: Ty, d: int, stable: bool = False) -> Expr:
        """an expression of type t and height <= d that cannot raise; stable = a float that may not come from arithmetic"""
        r = self.rng
        if d <= 1 or r.random() < 0.25:
            return self.leaf(t)
        if t.kind == "b":
            c = r.integers(7)
            if c <= 2:
                ot = self.comparable(r)
                l = self.expr(ot, d - 1, stable=True)
                rr = self.expr(ot, d - 2, stable=True) if r.random() < 0.5 else self.leaf(ot)
                return binary(CMP_OPS[r.integers(len(CMP_OPS))], l, rr)
            if c == 3:
                return binary(O.OP_AND if r.random() < 0.5 else O.OP_OR, self.expr(BOOL, d - 1), self.expr(BOOL, d - 2))
            if c == 4:
                return unary("not", self.expr(BOOL, d - 1))
            if c == 5:
                return unary("is_null" if r.random() < 0.5 else "is_not_null", self.expr(ALL[r.integers(len(ALL) - (0 if self.decimals else 1))], d - 1, stable=True))
            return cast(self.expr((INTS + FLOATS)[r.integers(10)], d - 1, stable=True), BOOL)
        if t.kind == "d":
            return cast(self.expr(I32, d - 1), DATE32) if r.random() < 0.5 else self.leaf(t)
        if t.kind == "x":
            if r.random() < 0.5:
                src = (I8, I16, U8)[r.integers(3)]
                return cast(self.expr(src, d - 1), DEC)
            return self.leaf(t)
        if t.kind == "f":
            c = r.integers(6 if not stable else 3)
            if c == 0:
                return unary("neg", self.expr(t, d - 1, stable))
            if c in (1, 2):
                return self.cast_to(t, d - 1)
            op = ARITH_OPS[r.integers(5)]
            return binary(op, self.expr(t, d - 1), self.expr(t, d - 2))
        # integers
        c = r.integers(8)
        if c <= 1:
            return binary((O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY)[r.integers(3)], self.expr(t, d - 1), self.expr(t, d - 2))
        if c == 2:
            if d < 4:
                return self.leaf(t)
            return binary(O.OP_DIVIDE if r.random() < 0.5 else O.OP_MODULO, self.expr(t, d - 1), safe_divisor(self.expr(t, d - 3)))
        if c == 3:
            return binary(BIT_OPS[r.integers(5)], self.expr(t, d - 1), self.expr(t, d - 2))
        if c == 4 and t.kind == "i":
            return unary("neg", self.expr(t, d - 1))
        return self.cast_to(t, d - 1)

    def comparable(self, r) -> Ty:
        pool = INTS + FLOATS + (BOOL, DATE32) + ((DEC,) if self.decimals else ())
        return pool[r.integers(len(pool))]

    def cast_to(self, t: Ty, d: int) -> Expr:
        """CAST(x AS t) for a source type and value range that always fit t"""
        r = self.rng
        if t.kind == "f":
            src = (INTS + FLOATS + (BOOL,) + ((DEC,) if self.decimals else ()))[r.integers(11 + self.decimals)]
            if src.kind == "x" and d > 1 and r.random() < 0.6:     # Decimal128 arithmetic: + - * never overflow at these precisions
                return cast(binary((O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY)[r.integers(3)], self.expr(DEC, d - 1), self.expr(DEC, d - 1)), t)
            return cast(self.expr(src, d, stable=True), t)
        if t.kind == "b":
            return cast(self.expr(I32, d), t)
        s = (INTS + (BOOL, F64, DATE32) + ((DEC,) if self.decimals else ()))[r.integers(11 + self.decimals)]
        if s.kind == "b":
            return cast(self.expr(s, d), t)
        if s.kind == "f":      # a float that holds a small integer: CAST(CAST(Int8 / UInt8 AS f) AS t)
            src = U8 if t.kind == "u" else I8
            if t.kind == "i" and t.bits == 8:
                src = I8
            return cast(cast(self.expr(src, max(d - 2, 1)), F64), t)
        if s.kind == "x":
            if t in (I32, I64):  # |x| < 10^7 once the 2 decimals are truncated
                return cast(self.expr(DEC, d), t)
            s = I16
        if s.kind == "d":
            s = I32
            x = cast(self.expr(DATE32, d - 1), I32) if d > 1 else self.leaf(I32)
        else:
            x = self.expr(s, d - 1)
        if s.lo >= t.lo and s.hi <= t.hi:
            return cast(x, t)
        mask = min(t.hi, s.hi)
        return cast(binary(O.OP_BITAND, x, lit(mask, s)), t)

    # -- public entry points --
    def _prog(self, root, family, zero_cols=(), sel_cols=()) -> Program:
        cols = list(self.fixed) if self.fixed is not None else list(self.cols)
        if not cols:                      # a program of literals still runs over a batch: one column gives it its row count
            cols = [(I8, False)]
        return Program(root, cols, family, self.seed, tuple(zero_cols), tuple(sel_cols))

    def total(self, t: Ty, height: int = 5) -> Program:
        self.cols = []
        return self._prog(self.expr(t, height), "total")

    def at_depth(self, t: Ty, depth: int, tries: int = 200) -> Program:
        """a total program whose evaluation stack is exactly `depth` deep"""
        for _ in range(tries):
            self.cols = []
            p = self._prog(self.deep(t, depth), "total")
            if p.depth() == depth and p.n_nodes() <= 40:
                return p
        raise RuntimeError(f"no {t.name} program of depth {depth} in {tries} tries (seed {self.seed})")

    def deep(self, t: Ty, d: int) -> Expr:
        """a total expression of stack depth d: the right operand of a binary node sits one slot above its left one"""
        r = self.rng
        if d <= 1:
            return self.leaf(t)
        left = self.expr(t, 2) if d >= 3 and r.random() < 0.5 else self.leaf(t)
        if t.kind == "b":
            if r.random() < 0.5:
                return binary(O.OP_AND if r.random() < 0.5 else O.OP_OR, left, self.deep(BOOL, d - 1))
            ot = INTS[r.integers(8)]
            return binary(CMP_OPS[r.integers(len(CMP_OPS))], self.leaf(ot), self.deep(ot, d - 1))
        ops = (O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY, O.OP_DIVIDE) if t.kind == "f" else (O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY, O.OP_BITAND, O.OP_BITXOR)
        return binary(ops[r.integers(len(ops))], left, self.deep(t, d - 1))

    def int_arith(self, t: Ty, height: int = 4) -> Program:
        """+ - * over non-NULL integer columns and literals: pipeline.cu plan_is_int_arith holds"""
        self.cols = []

        def go(d):
            if d <= 1 or self.rng.random() < 0.3:
                c = self.column(t, nullable=False) if self.rng.random() < 0.7 else None
                return c if c is not None else self.literal(t, allow_null=False)
            return binary((O.OP_PLUS, O.OP_MINUS, O.OP_MULTIPLY)[self.rng.integers(3)], go(d - 1), go(d - 1))
        return self._prog(go(height), "total")

    def conjunction(self, n_terms: int = 3) -> Program:
        """AND of `integer column <cmp> literal` terms, left-deep (pipeline.cu conjunction_terms / pred_mode 1)"""
        self.cols = []
        terms = []
        for _ in range(n_terms):
            t = (INTS + (DATE32,))[self.rng.integers(9)]
            c = self.column(t)
            terms.append(binary(CMP_OPS[self.rng.integers(6)], c, self.literal(t, allow_null=False)))
        root = terms[0]
        for x in terms[1:]:
            root = binary(O.OP_AND, root, x)
        return self._prog(root, "total")

    def raising(self, t: Ty = BOOL) -> Program:
        """one node that can raise, maybe under a short-circuiting AND / OR"""
        self.cols = []
        r = self.rng
        zero_cols, sel_cols = [], []
        kind = r.integers(3)
        if kind == 0:                            # division by a column holding 0
            it = INTS[r.integers(8)]
            y = self.column(it)
            zero_cols.append(y.col)
            site = binary(O.OP_DIVIDE if r.random() < 0.6 else O.OP_MODULO, self.expr(it, 3), y)
        elif kind == 1:                          # MIN / -1 (MIN % -1 = 0 never raises)
            it = (I8, I16, I32, I64)[r.integers(4)]
            site = binary(O.OP_DIVIDE if r.random() < 0.7 else O.OP_MODULO, self.column(it), lit(-1, it) if r.random() < 0.6 else self.column(it))
        else:                                    # out-of-range CAST
            src = (I16, I32, I64, U32, U64, F32, F64, DEC)[r.integers(8 if self.decimals else 7)]
            dst = (I8, I16, I32, I64, U8, U16, U32, U64)[r.integers(8)]
            if src == dst:
                dst = I8
            site = cast(self.column(src), dst)
        if t != BOOL:
            if site.t != t:
                site = cast(site, t) if t.kind == "f" else site
            return self._prog(site, "raising", zero_cols)
        core = binary(CMP_OPS[r.integers(6)], site, self.leaf(site.t, allow_null=False))
        wrap = r.integers(5)
        if wrap == 0:
            root = core
        else:
            # the left side: a scalar, or `sel < k` over a column whose values are 0..99 (~k % of the rows TRUE)
            if r.random() < 0.25:
                lhs = self.literal(BOOL)
            else:
                self.cols.append((I32, bool(r.random() < 0.3)))
                sel = Expr("col", I32, col=len(self.cols) - 1)
                sel_cols.append(sel.col)
                lhs = binary(O.OP_LT, sel, lit(int((0, 5, 15, 19, 50, 85, 100)[r.integers(7)]), I32))
            op = O.OP_AND if wrap in (1, 2) else O.OP_OR
            root = binary(op, lhs, core) if wrap != 4 else binary(op, core, lhs)
        return self._prog(root, "raising", zero_cols, sel_cols)


def guarded(prog: Program) -> bool:
    """an AND / OR whose right operand can raise (a CAST, an integer division or modulo, Decimal128 arithmetic): filter.cu plan_expr
    gives it a short-circuit guard, and a pipeline stage filter refuses it"""
    def can_raise(x):
        return x.kind == "cast" or (x.kind == "bin" and ((x.op in (O.OP_DIVIDE, O.OP_MODULO) and x.kids[0].t.kind != "f")
                                                         or (x.op in ARITH_OPS and x.kids[0].t.kind == "x")))
    return any(e.kind == "bin" and e.op in (O.OP_AND, O.OP_OR) and any(can_raise(x) for x in e.kids[1].post()) for e in prog.root.post())


def padded(prog: Program) -> Program:
    """the same values one stack slot deeper: TRUE AND p, 0 + p, -0.0 + p"""
    t = prog.t
    if t.kind == "b":
        root = binary(O.OP_AND, lit(True, BOOL), prog.root)
    elif t.kind in "iu":
        root = binary(O.OP_PLUS, lit(0, t), prog.root)
    elif t.kind == "f":
        root = binary(O.OP_PLUS, lit(-0.0, t), prog.root)
    else:
        raise ValueError(t)
    return Program(root, prog.cols, prog.family, prog.seed, prog.zero_cols, prog.sel_cols)
