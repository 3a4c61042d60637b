"""Host-side mirror of the reference's operator interface for the hot path.

The reference's operators implement `trait ExecutionPlan` (datafusion/physical-plan/src/execution_plan.rs:102;
`execute(partition, ctx) -> SendableRecordBatchStream` :696) and are driven by `collect(plan, ctx)` (:1752).
No Rust toolchain exists in this image, so this module is the Python stand-in for the Rust shim
(`GpuFilterExec` / `GpuHashJoinExec` / `GpuAggregateExec`, see INTEGRATION.md): same constructor
arguments, same output schemas, same error behaviour — all compute goes through the C ABI of
libdfgpu.so (capi.py); nothing here computes on the CPU.

Data model = pyarrow RecordBatch (crossing the boundary as Arrow C Data Interface structs, exactly as
datafusion/ffi/src/record_batch_stream.rs:101-167 does).
"""
from __future__ import annotations

from typing import Iterable, Iterator, List, NamedTuple, Optional, Sequence, Tuple, Union

import pyarrow as pa

from . import capi as D


# ---------------------------------------------------------------------------------------------
# types
# ---------------------------------------------------------------------------------------------
def type_id(t: pa.DataType) -> int:
    m = {pa.bool_(): D.BOOL, pa.int8(): D.INT8, pa.int16(): D.INT16, pa.int32(): D.INT32, pa.int64(): D.INT64,
         pa.uint8(): D.UINT8, pa.uint16(): D.UINT16, pa.uint32(): D.UINT32, pa.uint64(): D.UINT64,
         pa.float32(): D.FLOAT32, pa.float64(): D.FLOAT64, pa.date32(): D.DATE32, pa.date64(): D.DATE64}
    if t in m:
        return m[t]
    if pa.types.is_timestamp(t):
        return D.TIMESTAMP
    if pa.types.is_decimal128(t):
        return D.decimal128(t.precision, t.scale) if 0 <= t.scale <= t.precision else D.DECIMAL128
    raise NotImplementedError(f"This feature is not implemented: GPU operators do not support Arrow type {t}")


def arrow_type(tid: int) -> pa.DataType:
    if D.type_base(tid) == D.DECIMAL128:
        p, sc = D.decimal_precision_scale(tid)
        return pa.decimal128(p or 38, sc)
    return {D.BOOL: pa.bool_(), D.INT8: pa.int8(), D.INT16: pa.int16(), D.INT32: pa.int32(), D.INT64: pa.int64(), D.UINT8: pa.uint8(),
            D.UINT16: pa.uint16(), D.UINT32: pa.uint32(), D.UINT64: pa.uint64(), D.FLOAT32: pa.float32(), D.FLOAT64: pa.float64(),
            D.DATE32: pa.date32(), D.DATE64: pa.date64(), D.TIMESTAMP: pa.timestamp("ns")}[tid]


# ---------------------------------------------------------------------------------------------
# expressions — PhysicalExpr (physical-expr-common/src/physical_expr.rs:76)
# ---------------------------------------------------------------------------------------------
class Expr:
    def _bin(self, op, other):
        return BinaryExpr(self, op, other if isinstance(other, Expr) else lit(other))

    def __gt__(self, o): return self._bin(D.OP_GT, o)
    def __ge__(self, o): return self._bin(D.OP_GTEQ, o)
    def __lt__(self, o): return self._bin(D.OP_LT, o)
    def __le__(self, o): return self._bin(D.OP_LTEQ, o)
    def __eq__(self, o): return self._bin(D.OP_EQ, o)  # type: ignore[override]
    def __ne__(self, o): return self._bin(D.OP_NEQ, o)  # type: ignore[override]
    def __add__(self, o): return self._bin(D.OP_PLUS, o)
    def __sub__(self, o): return self._bin(D.OP_MINUS, o)
    def __mul__(self, o): return self._bin(D.OP_MULTIPLY, o)
    def __truediv__(self, o): return self._bin(D.OP_DIVIDE, o)
    def __mod__(self, o): return self._bin(D.OP_MODULO, o)
    def __and__(self, o): return self._bin(D.OP_AND, o)
    def __or__(self, o): return self._bin(D.OP_OR, o)
    def __invert__(self): return UnaryExpr(D.EXPR_NOT, self)
    def __neg__(self): return UnaryExpr(D.EXPR_NEGATIVE, self)
    def is_null(self): return UnaryExpr(D.EXPR_IS_NULL, self)
    def is_not_null(self): return UnaryExpr(D.EXPR_IS_NOT_NULL, self)
    def is_distinct_from(self, o): return self._bin(D.OP_IS_DISTINCT_FROM, o)
    def is_not_distinct_from(self, o): return self._bin(D.OP_IS_NOT_DISTINCT_FROM, o)
    def cast(self, t: pa.DataType): return CastExpr(self, t)
    __hash__ = None  # type: ignore[assignment]

    def data_type(self, schema: pa.Schema) -> pa.DataType:
        raise NotImplementedError

    def rpn(self, schema: pa.Schema, out: list) -> None:
        raise NotImplementedError


class Column(Expr):
    """expressions/column.rs:121"""

    def __init__(self, name: str):
        self.name = name

    def data_type(self, schema): return schema.field(self.name).type

    def rpn(self, schema, out):
        ix = schema.get_field_index(self.name)
        if ix < 0:
            raise KeyError(f"Schema error: No field named {self.name}")
        out.append((D.EXPR_COLUMN, ix, 0, 0, 0, 0.0))


class Literal(Expr):
    """expressions/literal.rs:106; value None = NULL of the given type.  A str value is a Utf8 literal."""

    def __init__(self, value, type: Optional[pa.DataType] = None):
        if type is None:
            type = (pa.bool_() if isinstance(value, bool) else pa.int64() if isinstance(value, int) else pa.string() if isinstance(value, str)
                    else pa.float64())
        self.value, self.type = value, type

    def data_type(self, schema): return self.type

    def rpn(self, schema, out):
        tid = type_id(self.type)
        isnull = 1 if self.value is None else 0
        v = 0 if self.value is None else self.value
        if tid in (D.FLOAT32, D.FLOAT64):
            out.append((D.EXPR_LITERAL, 0, tid, isnull, 0, float(v)))
        elif D.type_base(tid) == D.DECIMAL128:
            import decimal
            with decimal.localcontext() as dctx:
                dctx.prec = 80
                unscaled = int(decimal.Decimal(str(v)).scaleb(self.type.scale).to_integral_value(rounding=decimal.ROUND_HALF_UP))
            out.append((D.EXPR_LITERAL, 0, tid, isnull, unscaled, 0.0))   # capi.expr_nodes splits the 128-bit value
        else:
            if hasattr(v, "toordinal") and tid == D.DATE32:
                import datetime
                v = (v - datetime.date(1970, 1, 1)).days
            out.append((D.EXPR_LITERAL, 0, tid, isnull, int(v), 0.0))


class BinaryExpr(Expr):
    """expressions/binary.rs:536-676.  Operand types must already agree (the planner's type coercion);
    as a convenience an untyped Python literal adopts the other side's type."""

    def __init__(self, left: Expr, op: int, right: Expr):
        self.left, self.op, self.right = left, op, right

    def _coerced(self, schema):
        l, r = self.left, self.right
        if isinstance(r, Literal) and not isinstance(l, Literal):
            lt = l.data_type(schema)
            if r.type != lt and (pa.types.is_integer(r.type) or pa.types.is_floating(r.type)) and not pa.types.is_boolean(lt):
                if pa.types.is_decimal128(lt) and self.op in (D.OP_PLUS, D.OP_MINUS, D.OP_MULTIPLY, D.OP_DIVIDE, D.OP_MODULO) and pa.types.is_integer(r.type):
                    r = Literal(r.value, pa.decimal128(20, 0))    # Int64 -> Decimal128(20, 0) (type_coercion/binary.rs:1265)
                else:
                    r = Literal(r.value, lt)
        elif isinstance(l, Literal) and not isinstance(r, Literal):
            rt = r.data_type(schema)
            if l.type != rt and (pa.types.is_integer(l.type) or pa.types.is_floating(l.type)) and not pa.types.is_boolean(rt):
                if pa.types.is_decimal128(rt) and self.op in (D.OP_PLUS, D.OP_MINUS, D.OP_MULTIPLY, D.OP_DIVIDE, D.OP_MODULO) and pa.types.is_integer(l.type):
                    l = Literal(l.value, pa.decimal128(20, 0))
                else:
                    l = Literal(l.value, rt)
        return l, r

    def data_type(self, schema):
        if self.op in (D.OP_EQ, D.OP_NEQ, D.OP_LT, D.OP_LTEQ, D.OP_GT, D.OP_GTEQ, D.OP_AND, D.OP_OR, D.OP_IS_DISTINCT_FROM,
                       D.OP_IS_NOT_DISTINCT_FROM):
            return pa.bool_()
        l, r = self._coerced(schema)
        lt, rt = l.data_type(schema), r.data_type(schema)
        if pa.types.is_decimal128(lt) and pa.types.is_decimal128(rt):   # arrow-arith decimal_op result types (include/dfgpu.h)
            p1, s1, p2, s2 = lt.precision, lt.scale, rt.precision, rt.scale
            if self.op in (D.OP_PLUS, D.OP_MINUS):
                sc = max(s1, s2); return pa.decimal128(min(38, sc + max(p1 - s1, p2 - s2) + 1), sc)
            if self.op == D.OP_MULTIPLY:
                return pa.decimal128(min(38, p1 + p2 + 1), s1 + s2)
            if self.op == D.OP_DIVIDE:
                sc = min(38, s1 + 4); return pa.decimal128(min(38, sc - s1 + s2 + p1), sc)
            if self.op == D.OP_MODULO:
                sc = max(s1, s2); return pa.decimal128(min(38, sc + min(p1 - s1, p2 - s2)), sc)
        return lt

    def rpn(self, schema, out):
        l, r = self._coerced(schema)
        l.rpn(schema, out)
        r.rpn(schema, out)
        out.append((D.EXPR_BINARY, self.op, 0, 0, 0, 0.0))


class UnaryExpr(Expr):
    def __init__(self, kind: int, arg: Expr):
        self.kind, self.arg = kind, arg

    def data_type(self, schema):
        return self.arg.data_type(schema) if self.kind == D.EXPR_NEGATIVE else pa.bool_()

    def rpn(self, schema, out):
        self.arg.rpn(schema, out)
        out.append((self.kind, 0, 0, 0, 0, 0.0))


class CastExpr(Expr):
    def __init__(self, arg: Expr, to: pa.DataType):
        self.arg, self.to = arg, to

    def data_type(self, schema): return self.to

    def rpn(self, schema, out):
        self.arg.rpn(schema, out)
        out.append((D.EXPR_CAST, 0, type_id(self.to), 0, 0, 0.0))


class LikeExpr(Expr):
    """expressions/like.rs: `expr [NOT] [I]LIKE pattern`, evaluated by arrow-string's like / nlike / ilike / nilike.  Boolean.  It has no
    expression program of its own: plan_like_predicates computes a LIKE on a string column with a literal pattern as a UINT8 mask column
    (GpuLikeExec, libdfgpu_strings.so) and compares `mask = 1`.  A str pattern is a Utf8 literal."""

    def __init__(self, expr: Expr, pattern: Union[Expr, str, None], negated: bool = False, case_insensitive: bool = False):
        self.expr, self.negated, self.case_insensitive = expr, negated, case_insensitive
        self.pattern = pattern if isinstance(pattern, Expr) else Literal(pattern, pa.string())

    def data_type(self, schema): return pa.bool_()

    def rpn(self, schema, out):
        raise NotImplementedError("This feature is not implemented: LikeExpr has no GPU expression program (plan_like_predicates turns a LIKE "
                                  "on a string column with a literal pattern into a mask column)")


class InListExpr(Expr):
    """expressions/in_list.rs: `expr [NOT] IN (list)` with a static list, SQL's three-valued IN: NULL when expr is NULL, or when expr is
    found nowhere and the list holds a NULL.  Boolean.  It has no expression program of its own: plan_string_predicates computes an IN
    list of Utf8 literals over a string column as a UINT8 mask column (GpuLikeExec, libdfgpu_strings.so) and compares `mask = 1`.  A str
    or None item is a Utf8 literal."""

    def __init__(self, expr: Expr, list: Sequence[Union[Expr, str, None]], negated: bool = False):
        self.expr, self.negated = expr, negated
        self.list = [v if isinstance(v, Expr) else Literal(v, pa.string()) for v in list]

    def data_type(self, schema): return pa.bool_()

    def rpn(self, schema, out):
        raise NotImplementedError("This feature is not implemented: InListExpr has no GPU expression program (plan_string_predicates turns an "
                                  "IN list of Utf8 literals over a string column into a mask column)")


def col(name: str) -> Column: return Column(name)
def lit(value, type: Optional[pa.DataType] = None) -> Literal: return Literal(value, type)


# ---------------------------------------------------------------------------------------------
# plans
# ---------------------------------------------------------------------------------------------
class SessionConfig:
    """the execution.* keys that change hot-path behaviour (common/src/config.rs:904-923)"""

    def __init__(self, batch_size: int = 8192, perfect_hash_join_small_build_threshold: int = 1024,
                 perfect_hash_join_min_key_density: float = 0.15, force_hash_collisions: bool = False, device: int = 0):
        self.batch_size = batch_size
        self.perfect_hash_join_small_build_threshold = perfect_hash_join_small_build_threshold
        self.perfect_hash_join_min_key_density = perfect_hash_join_min_key_density
        self.force_hash_collisions = force_hash_collisions
        self.device = device


class TaskContext:
    """execution/src/task.rs:52 — owns the dfgpu context (device + stream)"""

    def __init__(self, config: Optional[SessionConfig] = None, ctx: Optional[D.Context] = None):
        self.config = config or SessionConfig()
        self.gpu = ctx or D.Context(self.config.device)


class ExecutionPlan:
    schema: pa.Schema

    def children(self) -> List["ExecutionPlan"]: return []
    def name(self) -> str: return type(self).__name__
    def execute(self, ctx: TaskContext) -> Iterator[pa.RecordBatch]: raise NotImplementedError
    def metrics(self) -> dict: return {}


class MemoryExec(ExecutionPlan):
    """TestMemoryExec (physical-plan/src/test.rs): yields the given batches of ONE partition"""

    def __init__(self, batches: Sequence[pa.RecordBatch], schema: Optional[pa.Schema] = None):
        self.batches = list(batches)
        self.schema = schema or self.batches[0].schema

    def execute(self, ctx):
        return iter(self.batches)


def _rename(rb: pa.RecordBatch, schema: pa.Schema) -> pa.RecordBatch:
    cols = []
    for c, f in zip(rb.columns, schema):
        cols.append(c if c.type == f.type else c.cast(f.type))
    return pa.RecordBatch.from_arrays(cols, schema=schema)


def _drain(op, schema, project: Optional[Sequence[int]] = None) -> Iterator[pa.RecordBatch]:
    """the operator's output batches as `schema`; `project`: the columns of each batch that form it (None = all, in order)"""
    while True:
        b = op.next(host=True)
        if b is None:
            return
        rb = b.to_arrow()
        yield _rename(rb if project is None else rb.select(list(project)), schema)


# ---------------------------------------------------------------------------------------------
# string keys — Utf8 / Utf8View / Dictionary(_, Utf8) columns as INT32 codes in ONE code space (dfgpu_dictionary)
# ---------------------------------------------------------------------------------------------
def _is_string_like(t: pa.DataType) -> bool:
    if pa.types.is_dictionary(t):
        t = t.value_type
    return pa.types.is_string(t) or pa.types.is_large_string(t) or (hasattr(pa.types, "is_string_view") and pa.types.is_string_view(t))


class StringDictionary:
    """the plan-wide code space: equal strings <=> equal codes in every column, every batch and on both sides of a join"""

    def __init__(self, ctx: TaskContext):
        self.ctx = ctx
        self.dic = D.Dictionary(ctx.gpu)

    def encode(self, arr: pa.Array) -> pa.Array:
        """string-like array -> int32 codes (NULL stays NULL): the batch's own dictionary is unified on the host (distinct values only),
        the row codes are rewritten on the device (dfgpu_dictionary_remap)"""
        import numpy as np
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        d = arr if pa.types.is_dictionary(arr.type) else arr.dictionary_encode()
        values = d.dictionary.cast(pa.string())
        bufs = values.buffers()
        offsets = np.frombuffer(bufs[1], np.int32, len(values) + 1, values.offset * 4) if len(values) else np.zeros(1, np.int32)
        data = np.frombuffer(bufs[2], np.uint8) if bufs[2] is not None else np.zeros(0, np.uint8)
        vvalid = None if values.null_count == 0 else np.asarray(values.is_valid())
        remap = self.dic.unify(offsets, data, vvalid)
        idx = d.indices.cast(pa.int32())
        codes = D.HostColumn(np.asarray(idx.fill_null(0)), None if idx.null_count == 0 else np.asarray(idx.is_valid()))
        b = self.dic.remap(codes, remap, on_host=True)
        v, valid = b.column_numpy(0)
        b.release()
        return pa.array(v, pa.int32(), mask=None if valid is None else ~valid)

    def decode(self, codes: pa.Array, to: pa.DataType) -> pa.Array:
        n = self.dic.size()
        values = pa.array([self.dic.value(i).decode() for i in range(n)], pa.string())
        if isinstance(codes, pa.ChunkedArray):
            codes = codes.combine_chunks()
        out = pa.DictionaryArray.from_arrays(codes.cast(pa.int32()), values)
        return out if pa.types.is_dictionary(to) else out.cast(to)

    def code(self, s: str) -> int:
        """the literal of `col = 'text'`: -1 when the string was never seen (matches nothing)"""
        return self.dic.code(s.encode())

    def close(self):
        self.dic.close()


class DictionaryEncodeExec(ExecutionPlan):
    """string-like columns of the input -> INT32 code columns (same names); everything else passes through"""

    def __init__(self, input: ExecutionPlan, dictionary_of: "callable"):
        self.input, self.dictionary_of = input, dictionary_of
        self.string_cols = [i for i, f in enumerate(input.schema) if _is_string_like(f.type)]
        self.schema = pa.schema([pa.field(f.name, pa.int32(), True) if i in self.string_cols else f for i, f in enumerate(input.schema)])

    def children(self): return [self.input]

    def execute(self, ctx):
        sd = self.dictionary_of(ctx)
        for rb in self.input.execute(ctx):
            cols = [sd.encode(rb.column(i)) if i in self.string_cols else rb.column(i) for i in range(rb.num_columns)]
            yield pa.RecordBatch.from_arrays(cols, schema=self.schema)


class DictionaryDecodeExec(ExecutionPlan):
    """INT32 code columns `names` of the input -> strings of type `to` (after the GPU operators)"""

    def __init__(self, input: ExecutionPlan, names: Sequence[str], dictionary_of: "callable", to: pa.DataType = pa.string()):
        self.input, self.names, self.dictionary_of, self.to = input, list(names), dictionary_of, to
        self.schema = pa.schema([pa.field(f.name, to, True) if f.name in self.names else f for f in input.schema])

    def children(self): return [self.input]

    def execute(self, ctx):
        sd = self.dictionary_of(ctx)
        for rb in self.input.execute(ctx):
            cols = [sd.decode(rb.column(i), self.to) if f.name in self.names else rb.column(i) for i, f in enumerate(rb.schema)]
            yield pa.RecordBatch.from_arrays(cols, schema=self.schema)


def _mask_column(e: Expr) -> Column:
    """the string column a mask predicate of GpuLikeExec reads"""
    return e.left if isinstance(e, BinaryExpr) else e.expr


class GpuLikeExec(ExecutionPlan):
    """String predicates over string columns -> one UINT8 mask column per predicate (`name`, appended; NULL where the predicate is NULL),
    and the input without the columns `drop`.  A predicate is a LikeExpr, a BinaryExpr(Column, comparison, Utf8 Literal) or an
    InListExpr(Column, Utf8 Literals); `likes` holds (predicate, mask name).  A Utf8 / LargeUtf8 / Utf8View column runs dfgpu_like,
    dfgpu_string_compare or dfgpu_string_in_list; an INT32 column of DictionaryEncodeExec codes (`dictionary_of` given) evaluates the
    predicate over the dictionary's distinct values, then maps each row's code with dfgpu_like_codes."""

    def __init__(self, input: ExecutionPlan, likes: Sequence[Tuple[LikeExpr, str]], drop: Sequence[str] = (), dictionary_of: Optional["callable"] = None):
        self.input, self.likes, self.drop, self.dictionary_of = input, list(likes), set(drop), dictionary_of
        self.schema = pa.schema([f for f in input.schema if f.name not in self.drop] + [pa.field(name, pa.uint8(), True) for _, name in self.likes])

    def children(self): return [self.input]

    @staticmethod
    def _predicate(ctx: TaskContext, strings, e: Expr) -> "D.DeviceColumn":
        if isinstance(e, LikeExpr):
            return D.like(ctx.gpu, strings, e.pattern.value, e.negated)
        if isinstance(e, BinaryExpr):
            return D.string_compare(ctx.gpu, strings, _STRING_CMP[e.op], e.right.value)
        return D.string_in_list(ctx.gpu, strings, [v.value for v in e.list], e.negated)

    def _mask(self, ctx: TaskContext, arr: pa.Array, e: Expr) -> pa.Array:
        import numpy as np
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        if _is_string_like(arr.type):
            m = self._predicate(ctx, arr, e)
        else:                                              # INT32 codes of DictionaryEncodeExec
            dic = self.dictionary_of(ctx).dic
            n = dic.size()
            values = pa.array([dic.value(i) for i in range(n)], pa.binary()).cast(pa.string())
            code_match = self._predicate(ctx, values, e)
            codes = D.DeviceColumn.from_host(ctx.gpu, D.HostColumn(np.asarray(arr.fill_null(0)), None if arr.null_count == 0 else np.asarray(arr.is_valid())))
            m = D.like_codes(ctx.gpu, codes, code_match, n)
        v, valid = D.device_column_numpy(m)
        return pa.array(v, pa.uint8(), mask=None if valid is None else ~valid)

    def execute(self, ctx):
        isch = self.input.schema
        for rb in self.input.execute(ctx):
            masks = [self._mask(ctx, rb.column(isch.get_field_index(_mask_column(e).name)), e) for e, _ in self.likes]
            cols = [rb.column(i) for i, f in enumerate(isch) if f.name not in self.drop]
            yield pa.RecordBatch.from_arrays(cols + masks, schema=self.schema)


def plan_string_dictionary():
    """a factory for the `dictionary_of` argument: one StringDictionary per TaskContext, created on first use"""
    cache = {}

    def get(ctx: TaskContext) -> StringDictionary:
        if id(ctx) not in cache:
            cache[id(ctx)] = StringDictionary(ctx)
        return cache[id(ctx)]
    return get


class GpuFilterExec(ExecutionPlan):
    """FilterExec (physical-plan/src/filter.rs:85): FilterExecBuilder::new(predicate, input).with_projection(..).with_fetch(..)"""

    def __init__(self, predicate: Expr, input: ExecutionPlan, projection: Optional[Sequence[int]] = None, fetch: Optional[int] = None):
        self.predicate, self.input, self.projection, self.fetch = predicate, input, projection, fetch
        if predicate.data_type(input.schema) != pa.bool_():
            # filter.rs:139-145
            raise ValueError(f"Error during planning: Filter predicate must return BOOLEAN values, got {predicate.data_type(input.schema)}")
        fields = list(input.schema) if projection is None else [input.schema.field(i) for i in projection]
        self.schema = pa.schema(fields)
        self._metrics = {}

    def children(self): return [self.input]

    def execute(self, ctx):
        nodes: list = []
        self.predicate.rpn(self.input.schema, nodes)
        types = [type_id(f.type) for f in self.input.schema]
        op = D.FilterHandle(ctx.gpu, types, nodes, self.projection, ctx.config.batch_size, -1 if self.fetch is None else self.fetch)
        try:
            for rb in self.input.execute(ctx):
                op.push_arrow(rb)
                yield from _drain(op, self.schema)
            op.finish()
            yield from _drain(op, self.schema)
            self._metrics = {k: op.metric(k) for k in ("input_rows", "output_rows", "selectivity_num", "selectivity_den")}
        finally:
            op.close()

    def metrics(self): return self._metrics


class GpuProjectionExec(ExecutionPlan):
    """ProjectionExec over PhysicalExpr::evaluate (physical-expr-common/src/physical_expr.rs:88): each output column is
    one expression evaluated on the GPU; plain `Column` expressions are passed through untouched (zero copy on the host)."""

    def __init__(self, exprs: Sequence[Tuple[Expr, str]], input: ExecutionPlan):
        self.exprs, self.input = list(exprs), input
        self.schema = pa.schema([pa.field(name, e.data_type(input.schema)) for e, name in self.exprs])

    def children(self): return [self.input]

    def execute(self, ctx):
        import ctypes as C
        import numpy as np
        isch = self.input.schema
        for rb in self.input.execute(ctx):
            cols = []
            for e, name in self.exprs:
                if isinstance(e, Column):
                    cols.append(rb.column(isch.get_field_index(e.name)))
                    continue
                nodes: list = []
                e.rpn(isch, nodes)
                hcols, keep = [], []
                for i, f in enumerate(isch):
                    arr = rb.column(i)
                    if pa.types.is_date32(f.type):
                        vals = np.asarray(arr.cast(pa.int32()).fill_null(0))
                    elif pa.types.is_boolean(f.type):
                        vals = np.asarray(arr.fill_null(False))
                    else:
                        vals = np.asarray(arr.fill_null(0))
                    valid = None if arr.null_count == 0 else ~np.asarray(arr.is_null())
                    keep.append(D.HostColumn(vals, valid, type_id(f.type)))
                arrc = (D.Column * len(keep))(*[k.c() for k in keep])
                na = D.expr_nodes(nodes)
                out = C.c_void_p()
                ctx.gpu.check(ctx.gpu.lib.dfgpu_expr_evaluate_host(ctx.gpu.h, arrc, len(keep), rb.num_rows, na, len(nodes), C.byref(out)))
                b = D.Batch(ctx.gpu, out.value)
                res = b.to_arrow().column(0)
                t = e.data_type(isch)
                cols.append(res if res.type == t else res.cast(t))
            yield pa.RecordBatch.from_arrays(cols, schema=self.schema)


_JOIN_TYPES = {"Inner": D.JOIN_INNER, "Left": D.JOIN_LEFT, "Right": D.JOIN_RIGHT, "Full": D.JOIN_FULL, "LeftSemi": D.JOIN_LEFT_SEMI,
               "RightSemi": D.JOIN_RIGHT_SEMI, "LeftAnti": D.JOIN_LEFT_ANTI, "RightAnti": D.JOIN_RIGHT_ANTI, "LeftMark": D.JOIN_LEFT_MARK,
               "RightMark": D.JOIN_RIGHT_MARK}


def build_join_schema(left: pa.Schema, right: pa.Schema, join_type: str) -> Tuple[pa.Schema, List[Tuple[int, int]]]:
    """joins/utils.rs build_join_schema: output fields + ColumnIndex (side, index); side 0=left 1=right 2=mark"""
    def nullable(fields): return [pa.field(f.name, f.type, True) for f in fields]
    l, r = list(left), list(right)
    if join_type in ("Inner", "Left", "Right", "Full"):
        lf = nullable(l) if join_type in ("Right", "Full") else l
        rf = nullable(r) if join_type in ("Left", "Full") else r
        return pa.schema(lf + rf), [(0, i) for i in range(len(l))] + [(1, i) for i in range(len(r))]
    if join_type in ("LeftSemi", "LeftAnti"):
        return pa.schema(l), [(0, i) for i in range(len(l))]
    if join_type in ("RightSemi", "RightAnti"):
        return pa.schema(r), [(1, i) for i in range(len(r))]
    if join_type == "LeftMark":
        return pa.schema(l + [pa.field("mark", pa.bool_(), False)]), [(0, i) for i in range(len(l))] + [(2, 0)]
    if join_type == "RightMark":
        return pa.schema(r + [pa.field("mark", pa.bool_(), False)]), [(1, i) for i in range(len(r))] + [(2, 0)]
    raise ValueError(join_type)


class JoinFilter:
    """joins/utils.rs JoinFilter: `expression` over an intermediate batch whose column c ("f0", "f1", ...) is
    column_indices[c] = (side "left"|"right", index)"""

    def __init__(self, expression: Expr, column_indices: Sequence[Tuple[str, int]]):
        self.expression, self.column_indices = expression, list(column_indices)


class GpuHashJoinExec(ExecutionPlan):
    """HashJoinExec::try_new(left, right, on, filter, join_type, projection, partition_mode, null_equality, null_aware)
    (physical-plan/src/joins/hash_join/exec.rs:752).  left = build side, right = probe side."""

    def __init__(self, left: ExecutionPlan, right: ExecutionPlan, on: Sequence[Tuple[str, str]], join_type: str = "Inner",
                 null_equality: str = "NullEqualsNothing", filter=None, projection: Optional[Sequence[int]] = None, null_aware: bool = False):
        if not on:
            raise ValueError("Error during planning: On constraints in HashJoinExec should be non-empty")  # exec.rs try_new
        self.filter, self.null_aware = filter, bool(null_aware)
        self.left, self.right, self.on, self.join_type, self.null_equality = left, right, list(on), join_type, null_equality
        full, idx = build_join_schema(left.schema, right.schema, join_type)
        if projection is not None:
            full = pa.schema([full.field(i) for i in projection])
            idx = [idx[i] for i in projection]
        self.schema, self.column_indices = full, idx
        self._metrics = {}

    def children(self): return [self.left, self.right]

    def execute(self, ctx):
        cfg = ctx.config
        bt = [type_id(f.type) for f in self.left.schema]
        pt = [type_id(f.type) for f in self.right.schema]
        ob = [self.left.schema.get_field_index(l) for l, _ in self.on]
        op_ = [self.right.schema.get_field_index(r) for _, r in self.on]
        if min(ob + op_) < 0:
            raise KeyError("Schema error: join key not found")
        op = D.HashJoinHandle(ctx.gpu, bt, pt, ob, op_, [s for s, _ in self.column_indices], [i for _, i in self.column_indices],
                              _JOIN_TYPES[self.join_type], D.NULL_EQUALS_NULL if self.null_equality == "NullEqualsNull" else D.NULL_EQUALS_NOTHING,
                              cfg.batch_size, cfg.perfect_hash_join_small_build_threshold, cfg.perfect_hash_join_min_key_density,
                              cfg.force_hash_collisions, self.null_aware)
        if self.filter is not None:
            fields = [(self.left.schema if sd == "left" else self.right.schema).field(ix) for sd, ix in self.filter.column_indices]
            inter = pa.schema([pa.field(f"f{i}", f.type) for i, f in enumerate(fields)])
            nodes: list = []
            self.filter.expression.rpn(inter, nodes)
            op.set_filter([0 if sd == "left" else 1 for sd, _ in self.filter.column_indices], [ix for _, ix in self.filter.column_indices], nodes)
        try:
            for rb in self.left.execute(ctx):     # collect_left_input
                op.push_build_arrow(rb)
            op.finish_build()
            for rb in self.right.execute(ctx):    # FetchProbeBatch / ProcessProbeBatch
                op.push_probe_arrow(rb)
                yield from _drain(op, self.schema)
            op.finish_probe()                     # ExhaustedProbeSide
            yield from _drain(op, self.schema)
            self._metrics = {k: op.metric(k) for k in ("build_input_rows", "input_rows", "output_rows", "array_map_created_count", "probe_hits")}
        finally:
            op.close()

    def metrics(self): return self._metrics


_AGG_FUNCS = {"sum": D.AGG_SUM, "count": D.AGG_COUNT, "min": D.AGG_MIN, "max": D.AGG_MAX, "avg": D.AGG_AVG, "count_star": D.AGG_COUNT_STAR}
_AGG_MODES = {"Partial": D.AGG_PARTIAL, "Final": D.AGG_FINAL, "FinalPartitioned": D.AGG_FINAL_PARTITIONED, "Single": D.AGG_SINGLE,
              "SinglePartitioned": D.AGG_SINGLE_PARTITIONED, "PartialReduce": D.AGG_PARTIAL_REDUCE}


class AggregateExpr:
    """AggregateFunctionExpr: func(arg) [FILTER (WHERE filter)] AS alias"""

    def __init__(self, func: str, arg: Optional[str], alias: Optional[str] = None, filter: Optional[str] = None):
        self.func, self.arg, self.filter = func.lower(), arg, filter
        self.alias = alias or f"{func.upper()}({arg or '*'})"

    def value_type(self, t: Optional[pa.DataType]) -> pa.DataType:
        if self.func in ("count", "count_star"):
            return pa.int64()
        if self.func == "avg":  # Avg::return_type (functions-aggregate average.rs): Decimal128(min(38, p + 4), min(38, s + 4))
            if pa.types.is_decimal128(t):
                return pa.decimal128(min(38, t.precision + 4), min(38, t.scale + 4))
            return pa.float64()
        if self.func == "sum":  # Sum::return_type, functions-aggregate/src/sum.rs:232-261
            if pa.types.is_decimal128(t):
                return pa.decimal128(min(38, t.precision + 10), t.scale)
            return pa.float64() if pa.types.is_floating(t) else pa.uint64() if pa.types.is_unsigned_integer(t) else pa.int64()
        return t

    def state_fields(self, t: Optional[pa.DataType]) -> List[pa.Field]:
        if self.func == "avg" and pa.types.is_decimal128(t):
            raise NotImplementedError(f"{self.alias}: AVG over {t} runs in Single modes only; its Partial state is not defined")
        if self.func == "avg":  # [count, sum] (aggregates/mod.rs:3591-3700 snapshots)
            return [pa.field(f"{self.alias}[count]", pa.uint64()), pa.field(f"{self.alias}[sum]", pa.float64())]
        return [pa.field(f"{self.alias}[{self.func}]", self.value_type(t))]


class GpuAggregateExec(ExecutionPlan):
    """AggregateExec::try_new(mode, group_by, aggr_expr, filter_expr, input, input_schema) (aggregates/mod.rs:930)."""

    def __init__(self, mode: str, group_by: Sequence[str], aggr_expr: Sequence[AggregateExpr], input: ExecutionPlan,
                 input_schema: Optional[pa.Schema] = None, capacity_hint: int = 0):
        self.mode, self.group_by, self.aggr_expr, self.input = mode, list(group_by), list(aggr_expr), input
        self.input_schema = input_schema or input.schema  # schema of the RAW input (needed in Final modes for value types)
        self.capacity_hint = capacity_hint
        self.state_input = mode in ("Final", "FinalPartitioned", "PartialReduce")
        self.state_output = mode in ("Partial", "PartialReduce")
        gfields = [input.schema.field(g) for g in self.group_by]
        afields: List[pa.Field] = []
        self._plan_error: Optional[NotImplementedError] = None
        for a in self.aggr_expr:
            t = self.input_schema.field(a.arg).type if a.arg is not None else None
            if self.state_output:
                try:
                    afields += a.state_fields(t)
                except NotImplementedError as e:   # the node stays inspectable by the optimizer rules; its schema and execution raise
                    self._plan_error = e
            else:
                afields.append(pa.field(a.alias, a.value_type(t)))
        self._schema = pa.schema([pa.field(f.name, f.type, True) for f in gfields] + afields)
        self._metrics = {}

    @property
    def schema(self) -> pa.Schema:
        if self._plan_error is not None:
            raise self._plan_error
        return self._schema

    def children(self): return [self.input]

    def execute(self, ctx):
        if self._plan_error is not None:
            raise self._plan_error
        isch = self.input.schema
        types = [type_id(f.type) for f in isch]
        gcols = [isch.get_field_index(g) for g in self.group_by]
        aggs = []
        for a in self.aggr_expr:
            if self.state_input:
                aggs.append((_AGG_FUNCS[a.func], -1, -1))
            else:
                aggs.append((_AGG_FUNCS[a.func], isch.get_field_index(a.arg) if a.arg is not None else -1,
                             isch.get_field_index(a.filter) if a.filter else -1))
        if self.state_input:  # layout contract: [group cols..., state cols...] in order
            assert gcols == list(range(len(gcols))), "state input must start with the group columns"
        op = D.AggHandle(ctx.gpu, types, gcols, aggs, _AGG_MODES[self.mode], ctx.config.batch_size, self.capacity_hint)
        try:
            for rb in self.input.execute(ctx):
                op.push_arrow(rb)
            op.finish()
            bs = ctx.config.batch_size
            for rb in _drain(op, self.schema):   # one big batch sliced by batch_size (aggregate_hash_table/common.rs:290)
                for s in range(0, rb.num_rows, bs):
                    yield rb.slice(s, bs)
            self._metrics = {k: op.metric(k) for k in ("num_groups", "input_rows", "output_rows", "rehashes")}
        finally:
            op.close()

    def metrics(self): return self._metrics


# ---------------------------------------------------------------------------------------------
# pipeline fusion — the executable twin of the second optimizer rule of INTEGRATION.md §2a
# ---------------------------------------------------------------------------------------------
class _Scan:
    """the probe-side chain of one pipeline: source plan, predicate over the source schema, probe stages, names visible downstream"""

    def __init__(self, source: ExecutionPlan, predicate: Optional[Expr] = None):
        self.source, self.predicate = source, predicate
        self.stages: List[Tuple[int, object, "GpuPipelineExec"]] = []  # (stage kind, probe key column — a list of them for a composite key, build pipeline)
        self.visible: List[str] = [f.name for f in source.schema]       # column names the operators above may still reference
        self.filters: dict = {}                                          # stage index -> its JoinFilter as stage-filter RPN nodes
        self.full = False                                                # the only stage is a Full join's

    def virtual_schema(self) -> pa.Schema:
        # a Full join's unmatched build rows carry every probe column NULL (build_join_schema(..., "Full"))
        fields = [f.with_nullable(True) for f in self.source.schema] if self.full else list(self.source.schema)
        for kind, _, build in self.stages:
            if kind in (D.STAGE_INNER, D.STAGE_LEFT, D.STAGE_LEFT_ANTI):
                fields += [build.scan_field(n) for n in build.payload]
            elif kind == D.STAGE_RIGHT:   # NULL on the probe rows no build row matched (build_join_schema(..., "Right"))
                fields += [build.scan_field(n).with_nullable(True) for n in build.payload]
        return pa.schema(fields)

    def has_right(self) -> bool:
        return any(kind == D.STAGE_RIGHT for kind, _, _ in self.stages)


class _Chain(NamedTuple):
    """what a probe chain may contain (_as_scan): the join types its stages come from, and whether a join may carry a JoinFilter"""
    joins: frozenset = frozenset({"Inner", "RightSemi", "RightAnti"})
    filters: bool = False

    def without_outer(self) -> "_Chain":
        return self._replace(joins=self.joins - {"Right", "Full"})


_FILTER_NODES = 128   # the node pool of a pipeline's stage filters (dfgpu_pipeline_set_stage_filter)


def _can_raise(e: Expr, schema: pa.Schema) -> bool:
    """CAST, integer ÷ / %, or Decimal128 arithmetic anywhere in e"""
    if isinstance(e, CastExpr):
        return True
    if isinstance(e, BinaryExpr):
        if e.op in (D.OP_DIVIDE, D.OP_MODULO) and not pa.types.is_floating(e.data_type(schema)):
            return True
        if e.op in (D.OP_PLUS, D.OP_MINUS, D.OP_MULTIPLY, D.OP_DIVIDE, D.OP_MODULO) and pa.types.is_decimal128(e.data_type(schema)):
            return True
        return _can_raise(e.left, schema) or _can_raise(e.right, schema)
    if isinstance(e, UnaryExpr):
        return _can_raise(e.arg, schema)
    return False


def _has_fallible_rhs(e: Expr, schema: pa.Schema) -> bool:
    """an AND / OR whose right operand can raise: its short-circuit is decided per batch on the host, which cannot see payload fields"""
    if isinstance(e, BinaryExpr):
        if e.op in (D.OP_AND, D.OP_OR) and _can_raise(e.right, schema):
            return True
        return _has_fallible_rhs(e.left, schema) or _has_fallible_rhs(e.right, schema)
    if isinstance(e, (UnaryExpr, CastExpr)):
        return _has_fallible_rhs(e.arg, schema)
    return False


_MAX_PIPE_COLS = 16   # input columns plus packed composite keys of one pipeline (dfgpu_pipeline_set_stage_keys)


def _room_for_composite(sc: _Scan) -> bool:
    """whether the pipeline of sc can pack one more composite key beside its source columns and the composite keys it packs already"""
    return len(sc.source.schema) + sum(isinstance(k, list) for _, k, _ in sc.stages) + 1 <= _MAX_PIPE_COLS


def _key_pairs(pkey, build: "GpuPipelineExec") -> List[Tuple[str, str]]:
    """(build key, probe key) of every key column of a stage: one pair, or one per component of a composite key"""
    if isinstance(pkey, list):
        return list(zip(build.key, pkey))
    return [(build.key, pkey)]


def _integer_like(t: pa.DataType) -> bool:
    return pa.types.is_integer(t) or pa.types.is_date32(t) or pa.types.is_date64(t) or pa.types.is_timestamp(t)


def _join_keys(join: GpuHashJoinExec, sc: _Scan):
    """(build keys, probe keys) of a join fused as one stage of the probe chain sc: the two names for one key (as they always were), two
    lists for a composite key of 2..4 pairs, or None.  A composite key needs pairs of the same integer-like Arrow type whose probe keys
    are source columns of the chain; whether the build keys pack (source columns with known bounds, domain <= 2^63 - 1) is _as_build's
    decision."""
    src = [f.name for f in sc.source.schema]
    if len(join.on) == 1:
        return join.on[0]
    if not 2 <= len(join.on) <= 4:
        return None
    for b, pk in join.on:
        if pk not in src or join.left.schema.get_field_index(b) < 0:
            return None
        bt, pt = join.left.schema.field(b).type, sc.source.schema.field(pk).type
        if bt != pt or not _integer_like(bt):
            return None
    if not _room_for_composite(sc):
        return None
    return [b for b, _ in join.on], [pk for _, pk in join.on]


def _stage_filter(sc: _Scan, join: GpuHashJoinExec, kind: int, payload: List[str]) -> Optional[list]:
    """The join's JoinFilter as the RPN program of the stage it becomes (appended next to sc.stages), or None when it cannot run there.
    Its columns: a probe-side column -> that column of the probe chain's virtual schema, the build key -> the probe key, any other build
    column -> the stage's payload field (`payload`, in order; a SEMI / ANTI stage's fields are seen by its filter only).  Each column of
    a composite key maps to its paired probe key.  None too when the pipeline's filters would exceed _FILTER_NODES nodes, or an AND / OR
    has a right operand that can raise (÷, %, CAST, Decimal128 arithmetic)."""
    f = join.filter
    vs = sc.virtual_schema()
    fields = list(vs) + [join.left.schema.field(n) for n in payload]
    paired = dict(join.on)
    where = []
    for side, ix in f.column_indices:
        if side == "left":
            name = join.left.schema.field(ix).name
            at = vs.get_field_index(paired[name]) if name in paired else (len(vs) + payload.index(name) if name in payload else -1)
        else:
            at = vs.get_field_index(join.right.schema.field(ix).name)   # -1 when missing or ambiguous
        if at < 0:
            return None
        where.append(at)
    inter = pa.schema([pa.field(f"f{i}", fields[at].type, fields[at].nullable) for i, at in enumerate(where)])
    try:
        if f.expression.data_type(inter) != pa.bool_() or _has_fallible_rhs(f.expression, inter):
            return None
        nodes: list = []
        f.expression.rpn(inter, nodes)
    except KeyError:
        return None
    if len(nodes) + sum(len(n) for n in sc.filters.values()) > _FILTER_NODES:
        return None
    return [(k, where[a], *rest) if k == D.EXPR_COLUMN else (k, a, *rest) for k, a, *rest in nodes]


def _expr_names(e: Expr) -> set:
    """the column names an expression reads"""
    if isinstance(e, Column):
        return {e.name}
    if isinstance(e, BinaryExpr):
        return _expr_names(e.left) | _expr_names(e.right)
    if isinstance(e, (UnaryExpr, CastExpr)):
        return _expr_names(e.arg)
    if isinstance(e, LikeExpr):
        return _expr_names(e.expr) | _expr_names(e.pattern)
    if isinstance(e, InListExpr):
        return _expr_names(e.expr).union(*[_expr_names(v) for v in e.list])
    return set()


def _settle_right(sc: _Scan, read: set) -> bool:
    """The RIGHT stages of sc (HashJoinExec(Right), planned by _as_scan with every build column) keep as payload exactly the build columns
    read above the join (`read`), a build key included: it is NULL on the probe rows nothing matched, so it cannot stand in for the probe
    key as an Inner join's can.  False when a RIGHT stage would carry no column (no payload lookup enforces unique keys then) or more than
    64 bits, or when the pipeline has stage filters (they do not run beside a RIGHT stage).  Call before reading the virtual schema."""
    if not sc.has_right():
        return True
    if sc.filters:
        return False
    for kind, _, build in sc.stages:
        if kind != D.STAGE_RIGHT:
            continue
        build.payload = [n for n in build.payload if n in read]
        if not build.payload or sum(D.WIDTH[type_id(build.scan_field(n).type)] * 8 for n in build.payload) > 64:
            return False
    return True


def _as_scan(plan: ExecutionPlan, ch: _Chain = _Chain()) -> Optional[_Scan]:
    """[ProjectionExec(columns only)]* over [FilterExec]? over [HashJoinExec(a join type of ch.joins, one key or a composite key
    (_join_keys), NullEqualsNothing, not null-aware, fusable build)]* over a source.  When ch.filters allows it, a join may carry a
    JoinFilter, which becomes its stage's filter (_stage_filter); a Right or Full join never does.  A Right join becomes a RIGHT stage
    (DFGPU_STAGE_RIGHT) whose payload fields are nullable, as build_join_schema(..., "Right") makes them; it carries every build column
    until _settle_right keeps those read above it.  A Full join becomes a RIGHT stage that also emits the unmatched build rows
    (dfgpu_pipeline_set_stage_full) when it is the chain's only join: its probe side is [FilterExec] over the source, and no join probes
    above it.  Those rows carry every probe column NULL, so the source columns are nullable in the virtual schema.  Its lookup takes one
    accumulator word, the visited marks."""
    if isinstance(plan, GpuProjectionExec):
        if not all(isinstance(e, Column) and e.name == name for e, name in plan.exprs):
            return None
        sc = _as_scan(plan.input, ch)
        if sc is not None:
            sc.visible = [name for _, name in plan.exprs]
        return sc
    if isinstance(plan, GpuFilterExec):
        if plan.fetch is not None:
            return None
        inner = plan.input
        if isinstance(inner, (GpuFilterExec, GpuHashJoinExec, GpuProjectionExec, GpuAggregateExec)):
            return None                                   # predicates are fused over the source columns only
        sc = _Scan(inner, plan.predicate)
        if plan.projection is not None:
            sc.visible = [inner.schema.field(i).name for i in plan.projection]
        return sc
    if isinstance(plan, GpuHashJoinExec):
        if plan.join_type not in ch.joins or (plan.filter is not None and (not ch.filters or plan.join_type in ("Right", "Full"))) or \
                plan.null_aware or plan.null_equality != "NullEqualsNothing":
            return None
        sc = _as_scan(plan.right, ch)
        if sc is not None and (sc.full or (plan.join_type == "Full" and sc.stages)):
            return None                                   # a FULL stage is the pipeline's only probe stage
        keys = None if sc is None else _join_keys(plan, sc)
        if keys is None or (isinstance(keys[1], str) and keys[1] not in [f.name for f in sc.source.schema]):
            return None
        bkey, pkey = keys
        bkeys = bkey if isinstance(bkey, list) else [bkey]
        kind = {"RightSemi": D.STAGE_SEMI, "RightAnti": D.STAGE_ANTI, "Inner": D.STAGE_INNER, "Right": D.STAGE_RIGHT, "Full": D.STAGE_RIGHT}[plan.join_type]
        payload = [f.name for f in plan.left.schema if f.name not in bkeys] if kind == D.STAGE_INNER else []
        if kind == D.STAGE_RIGHT:
            payload = [f.name for f in plan.left.schema]
        if plan.filter is not None and kind != D.STAGE_INNER:   # a semi / anti lookup carries the build columns its filter reads
            read = {plan.left.schema.field(ix).name for sd, ix in plan.filter.column_indices if sd == "left"}
            payload = [f.name for f in plan.left.schema if f.name not in bkeys and f.name in read]
        filt = None
        if plan.filter is not None:
            filt = _stage_filter(sc, plan, kind, payload)
            if filt is None:
                return None
        build = _as_build(plan.left, bkey, payload, ch, max_bits=None if kind == D.STAGE_RIGHT else 64)
        if build is None:
            return None
        if filt is not None:
            sc.filters[len(sc.stages)] = filt
        if plan.join_type == "Full":
            sc.full = True
            build.n_acc_words = 1                         # the visited marks (dfgpu_pipeline_set_stage_full)
        sc.stages.append((kind, pkey, build))
        names = [f.name for f in plan.schema]
        sc.visible = names
        return sc
    if isinstance(plan, (GpuAggregateExec,)):
        return None
    return _Scan(plan)


def _as_build(plan: ExecutionPlan, key, payload: List[str], ch: _Chain, max_bits: Optional[int] = 64) -> Optional["GpuPipelineExec"]:
    """the build pipeline of a fused join on `key` (a list of columns for a composite key: source columns with known bounds
    (_source_bounds) whose domain, the product of max - min + 1, is at most 2^63 - 1, so that the tuple packs into one 64-bit key).
    max_bits None: the payload is settled later (a Right join's, _settle_right).  A build side with a Right or Full join stays unfused:
    its NULL payload fields cannot enter a lookup."""
    sc = _as_scan(plan, ch.without_outer())
    if sc is None or len(sc.stages) >= 3:
        return None
    vs = sc.virtual_schema()
    keys = key if isinstance(key, list) else [key]
    if any(vs.get_field_index(k) < 0 or vs.get_field_index(k) >= len(sc.source.schema) for k in keys) or any(vs.get_field_index(n) < 0 for n in payload):
        return None
    bits = sum(D.WIDTH[type_id(vs.field(n).type)] * 8 for n in payload)
    if max_bits is not None and bits > max_bits:
        return None
    ranges = []
    if isinstance(key, list):
        if not _room_for_composite(sc):
            return None
        dom = 1
        for k in keys:
            b = _source_bounds(sc.source, k)
            if b is None:
                return None
            dom *= b[1] - b[0] + 1
            ranges.append(b)
        if dom > (1 << 63) - 1:
            return None
    build = GpuPipelineExec(sc, sink="build", key=key, payload=payload)
    build.key_ranges = ranges
    return build


class GpuPipelineExec(ExecutionPlan):
    """One fused pipeline (dfgpu_pipeline): source -> predicate -> probe stages -> {build | aggregate | output}.  Built by fuse_pipelines()."""

    def __init__(self, scan: _Scan, sink: str, key: Optional[str] = None, payload: Sequence[str] = (), group_by: Sequence[str] = (),
                 aggs: Sequence[Tuple[str, Optional[Expr], str]] = (), mode: str = "Single", out_schema: Optional[pa.Schema] = None,
                 key_range: Sequence[Tuple[int, int]] = (), nullable: Sequence[bool] = (), project: Optional[Sequence[int]] = None,
                 out_cols: Sequence[int] = (), fallback: Optional[ExecutionPlan] = None):
        self.scan, self.sink, self.key, self.payload, self.group_by, self.aggs, self.mode = scan, sink, key, list(payload), list(group_by), list(aggs), mode
        self.key_range = list(key_range)   # dense sink: the declared (min, max) of every group column
        self.nullable = list(nullable)     # hash sink: the declared nullability of every group column
        self.project = None if project is None else list(project)   # the emitted columns that form the output (a LeftSemi / LeftAnti join's projection)
        self.out_cols = list(out_cols)     # output sink: the virtual columns of the scan that form the output, in order
        self.fallback = fallback           # output sink: the unfused plan, run when a build side cannot be fused (_execute_output)
        self.schema = out_schema if out_schema is not None else pa.schema([])
        self.n_acc_words = 0
        self.key_ranges: List[Tuple[int, int]] = []   # build sink of a composite key: the declared (min, max) of every component
        self._metrics = {}

    def children(self): return [self.scan.source] + [b for _, _, b in self.scan.stages]
    def scan_field(self, name: str) -> pa.Field: return self.scan.virtual_schema().field(name)
    def metrics(self): return self._metrics

    # ---- build side: run the pipeline into a dfgpu_lookup ----
    def build_lookup(self, ctx: TaskContext) -> D.Lookup:
        vs = self.scan.virtual_schema()
        batches = list(self.scan.source.execute(ctx))
        if isinstance(self.key, list):
            look = D.Lookup(ctx.gpu, key_types=[type_id(vs.field(k).type) for k in self.key], key_ranges=self.key_ranges,
                            payload_types=[type_id(vs.field(n).type) for n in self.payload], n_acc_words=self.n_acc_words)
            return self._run_build(ctx, look, batches, dict(key_cols=[vs.get_field_index(k) for k in self.key]))
        key_range = None
        ktype = vs.field(self.key).type
        if not self.payload and self.n_acc_words == 0 and pa.types.is_integer(ktype) and batches:   # statistics: the bounds collect_left_input tracks
            import pyarrow.compute as pc
            mm = [pc.min_max(b.column(self.scan.source.schema.get_field_index(self.key))) for b in batches if b.num_rows]
            lo = [m["min"].as_py() for m in mm if m["min"].is_valid]; hi = [m["max"].as_py() for m in mm if m["max"].is_valid]
            if lo:
                key_range = (min(lo), max(hi))
        look = D.Lookup(ctx.gpu, type_id(ktype), [type_id(vs.field(n).type) for n in self.payload], key_range=key_range, n_acc_words=self.n_acc_words)
        return self._run_build(ctx, look, batches, dict(key_col=vs.get_field_index(self.key)))

    def _run_build(self, ctx: TaskContext, look: D.Lookup, batches, key: dict) -> D.Lookup:
        vs = self.scan.virtual_schema()
        try:
            pipe, keep = self._make_pipeline(ctx)
        except BaseException:
            look.close()
            raise
        try:
            pipe.sink_build(look, payload_cols=[vs.get_field_index(n) for n in self.payload], **key)
            for rb in batches:
                pipe.push_arrow(rb)
            pipe.finish()
            self._metrics = {"input_rows": pipe.metric("input_rows"), "build_rows": pipe.metric("sink_rows"), "lookup_mode": look.metric("mode")}
        except BaseException:
            look.close()
            raise
        finally:
            pipe.close()
            for l in keep:
                l.close()
        return look

    def _make_pipeline(self, ctx: TaskContext):
        ssch = self.scan.source.schema
        nodes = None
        if self.scan.predicate is not None:
            nodes = []
            self.scan.predicate.rpn(ssch, nodes)
        stages, keep = [], []
        try:
            for kind, pkey, build in self.scan.stages:
                look = build.build_lookup(ctx)                  # the pipeline breaker: WaitBuildSide (hash_join/stream.rs:117-140)
                keep.append(look)
                stages.append((kind, [ssch.get_field_index(k) for k in pkey] if isinstance(pkey, list) else ssch.get_field_index(pkey), look))
        except BaseException:
            for l in keep:
                l.close()
            raise
        pipe = D.Pipeline(ctx.gpu, [type_id(f.type) for f in ssch], nodes, stages)
        try:
            if self.scan.full:
                pipe.set_stage_full(0)
            for s, fnodes in sorted(self.scan.filters.items()):
                pipe.set_stage_filter(s, fnodes)
        except BaseException:
            pipe.close()
            for l in keep:
                l.close()
            raise
        return pipe, keep

    def execute(self, ctx):
        assert self.sink in ("aggregate", "dense", "hash", "output"), "build pipelines are driven by their consumer"
        if self.sink == "output":
            yield from self._execute_output(ctx)
            return
        if self.fallback is not None:   # a RIGHT stage: its build's keys are known unique only once it ran; the sinks emit after finish
            try:
                out = list(self._execute_aggregate(ctx))
            except D.DfgpuError as e:
                yield from self._fall_back(ctx, e)
                return
            yield from out
            return
        yield from self._execute_aggregate(ctx)

    def _execute_aggregate(self, ctx):
        vs = self.scan.virtual_schema()
        pipe, keep = self._make_pipeline(ctx)
        try:
            aggs = []
            for func, expr, _ in self.aggs:
                if expr is None:
                    aggs.append((D.AGG_COUNT_STAR if self.sink in ("dense", "hash") else _AGG_FUNCS[func], None))
                else:
                    nodes: list = []
                    expr.rpn(vs, nodes)
                    aggs.append((_AGG_FUNCS[func], nodes))
            gcols = [vs.get_field_index(g) for g in self.group_by]
            if self.sink == "dense":
                pipe.sink_aggregate_dense(gcols, self.key_range, aggs, _AGG_MODES[self.mode], 0)
            elif self.sink == "hash":
                pipe.sink_aggregate_hash(gcols, aggs, _AGG_MODES[self.mode], 0, 0, self.nullable)
            else:
                pipe.sink_aggregate(gcols, aggs, _AGG_MODES[self.mode], 0)
            for rb in self.scan.source.execute(ctx):
                pipe.push_arrow(rb)
            pipe.finish()
            bs = ctx.config.batch_size
            for rb in _drain(pipe, self.schema, self.project):
                for s in range(0, rb.num_rows, bs):
                    yield rb.slice(s, bs)
            self._metrics = {k: pipe.metric(k) for k in ("input_rows", "sink_rows", "num_groups")}
        finally:
            pipe.close()
            for l in keep:
                l.close()


    def _execute_output(self, ctx):
        """the ordered output sink (dfgpu_pipeline_sink_output): the surviving rows in input order, sliced by batch_size.  The sink
        emits nothing before finish, so every refusal comes first: when the library refuses the fused plan (DFGPU_ERR_UNSUPPORTED, e.g.
        duplicate keys in an Inner stage's build, a NULL in a payload column, a Boolean input column) the unfused plan runs instead and
        the metric "fallback" holds the reason.  Other errors (arithmetic, state) propagate."""
        try:
            pipe, keep = self._make_pipeline(ctx)
        except D.DfgpuError as e:
            yield from self._fall_back(ctx, e)
            return
        try:
            try:
                pipe.sink_output(self.out_cols, batch_size=ctx.config.batch_size)
                for rb in self.scan.source.execute(ctx):
                    pipe.push_arrow(rb)
                pipe.finish()
            except D.DfgpuError as e:
                refused = e
            else:
                refused = None
                yield from _drain(pipe, self.schema)
                self._metrics = {k: pipe.metric(k) for k in ("input_rows", "sink_rows", "output_rows")}
        finally:
            pipe.close()
            for l in keep:
                l.close()
        if refused is not None:
            yield from self._fall_back(ctx, refused)

    def _fall_back(self, ctx, e: "D.DfgpuError"):
        if self.fallback is None or e.code != _ERR_UNSUPPORTED:
            raise e
        yield from self.fallback.execute(ctx)
        self._metrics = {"fallback": str(e)}


_ERR_UNSUPPORTED = -3   # DFGPU_ERR_UNSUPPORTED (include/dfgpu.h)


def _source_bounds(source: ExecutionPlan, name: str) -> Optional[Tuple[int, int]]:
    """(min, max) of an integer-like source column, when known at planning time.  The twin reads a MemoryExec's batches; DataFusion
    has them as ColumnStatistics::{min_value, max_value} of partition_statistics.  None when unknown (or no non-NULL value)."""
    if isinstance(source, GpuLikeExec) and source.input.schema.get_field_index(name) >= 0:
        return _source_bounds(source.input, name)        # a column the LIKE pass carries through
    if not isinstance(source, MemoryExec):
        return None
    t = source.schema.field(name).type
    if not (pa.types.is_integer(t) or pa.types.is_date32(t)):
        return None
    import pyarrow.compute as pc
    i = source.schema.get_field_index(name)
    lo = hi = None
    for b in source.batches:
        c = b.column(i)
        if c.null_count == len(c):
            continue
        mm = pc.min_max(c.cast(pa.int32()).cast(pa.int64()) if pa.types.is_date32(t) else c)   # date32 casts to int64 through int32 only
        lo = mm["min"].as_py() if lo is None else min(lo, mm["min"].as_py())
        hi = mm["max"].as_py() if hi is None else max(hi, mm["max"].as_py())
    if lo is None or hi > (1 << 63) - 1:
        return None
    return lo, hi


def _agg_input(plan: "GpuAggregateExec") -> Tuple[ExecutionPlan, dict]:
    """the plan under an aggregate and its optional ProjectionExec, and the expression over that plan of every column of the aggregate's
    input"""
    below = plan.input
    if isinstance(below, GpuProjectionExec):
        return below.input, {name: e for e, name in below.exprs}
    return below, {f.name: Column(f.name) for f in below.schema}


def _agg_args(plan: "GpuAggregateExec", exprs: dict, vs: pa.Schema) -> Optional[list]:
    """(aggregate, argument expression, its type, its RPN nodes over the virtual schema vs) of every aggregate of plan, the last three None
    for COUNT(*); None when an aggregate has a FILTER clause or an argument that is no input column (`exprs`) or reads a name vs lacks,
    or is an AVG whose state no sink holds: AVG(Decimal128) has no pinned Partial state, and any other AVG argument must be Float64"""
    args = []
    for a in plan.aggr_expr:
        if a.filter is not None:
            return None
        if a.arg is None:
            args.append((a, None, None, None))
            continue
        e = exprs.get(a.arg)
        if e is None:
            return None
        nodes: list = []
        try:
            e.rpn(vs, nodes)
            t = e.data_type(vs)
        except KeyError:
            return None
        if a.func == "avg" and t != pa.float64() and not (pa.types.is_decimal128(t) and plan.mode != "Partial"):
            return None
        args.append((a, e, t, nodes))
    return args


def _fuse_dense(plan: "GpuAggregateExec", ch: _Chain) -> Optional["GpuPipelineExec"]:
    """AggregateExec over [ProjectionExec] over FilterExec over a source (no join: TPC-H Q1, Q6), or over a chain that ch allows topped by
    a Right or Full join, with no JoinFilter anywhere, whose GROUP BY columns have known bounds (_field_bounds) spanning at most
    DENSE_MAX_GROUPS slots (NULL included); at most 8 aggregates, no Float32 MIN / MAX -> a GpuPipelineExec with the dense sink; None
    otherwise"""
    below, exprs = _agg_input(plan)
    if not (isinstance(below, GpuFilterExec) or (isinstance(below, GpuHashJoinExec) and below.join_type in ("Right", "Full"))):
        return None
    sc = _as_scan(below, ch._replace(filters=False))
    if sc is None or not _settle_right(sc, _read_names(plan, exprs)):
        return None
    vs = sc.virtual_schema()
    group, ranges, slots = [], [], 1
    for g in plan.group_by:
        e = exprs.get(g)
        if not isinstance(e, Column) or e.name not in sc.visible or vs.get_field_index(e.name) < 0:
            return None
        b = _field_bounds(sc, e.name)
        if b is None:
            return None
        slots *= b[1] - b[0] + 2
        if slots > D.DENSE_MAX_GROUPS:
            return None
        group.append(e.name)
        ranges.append(b)
    if len(plan.aggr_expr) > 8:
        return None
    args = _agg_args(plan, exprs, vs)
    if args is None or any(a.func in ("min", "max") and t == pa.float32() for a, _, t, _ in args):
        return None
    return GpuPipelineExec(sc, sink="dense", group_by=group, aggs=[(a.func, e, a.alias) for a, e, _, _ in args], mode=plan.mode,
                           out_schema=plan.schema, key_range=ranges, fallback=plan if sc.has_right() else None)


def _read_names(plan: "GpuAggregateExec", exprs: dict) -> set:
    """the input column names an aggregate's GROUP BY and arguments read (through its projection's expressions)"""
    read = set()
    for n in list(plan.group_by) + [a.arg for a in plan.aggr_expr if a.arg is not None]:
        if n in exprs:
            read |= _expr_names(exprs[n])
    return read


def _field_bounds(sc: _Scan, name: str) -> Optional[Tuple[int, int]]:
    """(min, max) of a column of sc's virtual schema: a source column's (_source_bounds), or a RIGHT stage's payload field taken from a
    source column of its build side (a NULL field goes to its own dense slot)"""
    if sc.source.schema.get_field_index(name) >= 0:
        return _source_bounds(sc.source, name)
    for kind, _, build in sc.stages:
        if kind == D.STAGE_RIGHT and name in build.payload and build.scan.source.schema.get_field_index(name) >= 0:
            return _source_bounds(build.scan.source, name)
    return None


def _acc_words(funcs: Sequence[str], types: Sequence[Optional[pa.DataType]], has_payload: bool) -> int:
    """n_acc_words of the build lookup that a join-keyed aggregate sink accumulates into (dfgpu.h, dfgpu_pipeline_sink_aggregate): the
    row counter; per aggregate 1 word (2 for AVG over Float64), and a Decimal128 SUM, MIN or MAX 2, a Decimal128 AVG 3; one non-null
    counter per SUM, MIN and MAX.  A Decimal128 MIN / MAX pair is 16-byte aligned: one padding word, and a record of an even number of
    words (key + accumulators) when the build has no payload."""
    n, pairs = 1, False
    for f, t in zip(funcs, types):
        dec = t is not None and pa.types.is_decimal128(t)
        if f == "avg":
            n += 3 if dec else 2
        elif f in ("sum", "min", "max"):
            n += (2 if dec else 1) + 1
            pairs = pairs or (dec and f != "sum")
        else:
            n += 1
    if pairs:
        n += 1
        if not has_payload and n % 2 == 0:
            n += 1
    return n


def _fuse_inner(plan: "GpuAggregateExec", ch: _Chain) -> Optional["GpuPipelineExec"]:
    """AggregateExec over [ProjectionExec] over HashJoinExec(Inner), a chain that ch allows without its Right and Full joins, whose GROUP BY
    is the probe key of that last Inner stage (or the equal build key; every component of a composite key) plus its payload fields ->
    ONE GpuPipelineExec with the join-keyed sink, its build side (filters, semi joins, column projections) a build pipeline; at most 12
    accumulator words (_acc_words); None otherwise"""
    below, exprs = _agg_input(plan)
    if not isinstance(below, GpuHashJoinExec) or below.join_type != "Inner":
        return None
    sc = _as_scan(below, ch.without_outer())
    if sc is None:
        return None
    _, pkey, build = sc.stages[-1]
    vs = sc.virtual_schema()
    paired = dict(_key_pairs(pkey, build))
    pkeys = list(paired.values())
    group = []
    for g in plan.group_by:
        e = exprs.get(g)
        if not isinstance(e, Column):
            return None
        n = paired.get(e.name, e.name)
        if n not in pkeys and n not in build.payload:
            return None
        group.append(n)
    if any(k not in group for k in pkeys):
        return None
    args = _agg_args(plan, exprs, vs)
    if args is None:
        return None
    n_acc = _acc_words([a.func for a, _, _, _ in args], [t for _, _, t, _ in args], bool(build.payload))
    if n_acc > 12:
        return None
    build.n_acc_words = n_acc
    return GpuPipelineExec(sc, sink="aggregate", group_by=group, aggs=[(a.func, e, a.alias) for a, e, _, _ in args], mode=plan.mode,
                           out_schema=plan.schema)


def _left_join_scan(join: GpuHashJoinExec, kind: int, ch: _Chain) -> Optional[_Scan]:
    """The probe chain of a Left / LeftSemi / LeftAnti join with the join as its last stage (kind), or None.  Conditions: one key or a
    composite key (_join_keys), NullEqualsNothing, not null-aware; the right side is a chain that ch allows without its Right and Full
    joins, probing on its source columns; the left side is a fusable build whose key fields are declared non-nullable (a NULL build key
    is never in the lookup, but Left / LeftAnti emit its row) and have the probe keys' types.  The build's payload is every other left
    column.  A JoinFilter, when ch allows one, becomes the stage's filter.  The fused join emits its rows in slot order: the reference
    does not keep the build side's order either (maintains_input_order is false for it)."""
    if (join.filter is not None and not ch.filters) or join.null_aware or join.null_equality != "NullEqualsNothing":
        return None
    sc = _as_scan(join.right, ch.without_outer())
    keys = None if sc is None or len(sc.stages) >= 3 else _join_keys(join, sc)
    if keys is None:
        return None
    bkey, pkey = keys
    ls = join.left.schema
    for b, pk in (zip(bkey, pkey) if isinstance(bkey, list) else [(bkey, pkey)]):
        if sc.source.schema.get_field_index(pk) < 0 or ls.get_field_index(b) < 0:
            return None
        kf = ls.field(b)
        if kf.nullable or kf.type != sc.source.schema.field(pk).type:
            return None
    bkeys = bkey if isinstance(bkey, list) else [bkey]
    payload = [f.name for f in ls if f.name not in bkeys]
    filt = None
    if join.filter is not None:
        filt = _stage_filter(sc, join, kind, payload)
        if filt is None:
            return None
    build = _as_build(join.left, bkey, payload, ch)
    if build is None:
        return None
    if filt is not None:
        sc.filters[len(sc.stages)] = filt
    sc.stages.append((kind, pkey, build))
    return sc


def _fuse_left(plan: "GpuAggregateExec", ch: _Chain) -> Optional["GpuPipelineExec"]:
    """AggregateExec over [ProjectionExec] over HashJoinExec(Left) -> the join-keyed sink over a LEFT stage (TPC-H Q13), or None.  GROUP BY
    the build key (not the probe key: NULL on a padded row) plus build columns; every aggregate COUNT(*) or an argument over right-side
    columns that reads a probe source column and propagates NULL, so that it is NULL on a build row's padded row; no Float32 MIN / MAX;
    at most 12 accumulator words (_acc_words)."""
    join, exprs = _agg_input(plan)
    if not isinstance(join, GpuHashJoinExec) or join.join_type != "Left":
        return None
    sc = _left_join_scan(join, D.STAGE_LEFT, ch)
    if sc is None:
        return None
    _, pkey, build = sc.stages[-1]
    vs = sc.virtual_schema()
    paired = dict(_key_pairs(pkey, build))
    group = []
    for g in plan.group_by:
        e = exprs.get(g)
        if not isinstance(e, Column) or (e.name not in paired and e.name not in build.payload):
            return None
        group.append(paired.get(e.name, e.name))
    if any(k not in group for k in paired.values()):
        return None
    args = _agg_args(plan, exprs, vs)                      # the build key is not in the virtual schema
    if args is None:
        return None
    n_src, left_payload = len(sc.source.schema), range(len(vs) - len(build.payload), len(vs))
    for a, e, t, nodes in args:
        if e is None:
            continue
        if not any(n[0] == D.EXPR_COLUMN and n[1] < n_src for n in nodes):
            return None
        for n in nodes:
            if (n[0] == D.EXPR_COLUMN and n[1] in left_payload) or n[0] in (D.EXPR_IS_NULL, D.EXPR_IS_NOT_NULL) or \
                    (n[0] == D.EXPR_BINARY and n[1] in (D.OP_AND, D.OP_OR, D.OP_IS_DISTINCT_FROM, D.OP_IS_NOT_DISTINCT_FROM)):
                return None
        if a.func in ("min", "max") and t == pa.float32():
            return None
    aggs = [("count_star" if e is None else a.func, e, a.alias) for a, e, _, _ in args]
    n_acc = _acc_words([f for f, _, _ in aggs], [t for _, _, t, _ in args], bool(build.payload))
    if n_acc > 12:
        return None
    build.n_acc_words = n_acc
    return GpuPipelineExec(sc, sink="aggregate", group_by=group, aggs=aggs, mode=plan.mode, out_schema=plan.schema)


def _fuse_left_filter(join: GpuHashJoinExec, ch: _Chain) -> Optional["GpuPipelineExec"]:
    """HashJoinExec(LeftSemi / LeftAnti) -> the join-keyed sink without aggregates, grouped on every left column, or None (TPC-H Q18, Q20,
    Q22).  LeftSemi is an INNER stage over the unique build keys (the records a probe row reached), LeftAnti a LEFT_ANTI stage (the
    records none reached)."""
    sc = _left_join_scan(join, D.STAGE_INNER if join.join_type == "LeftSemi" else D.STAGE_LEFT_ANTI, ch)
    if sc is None:
        return None
    _, pkey, build = sc.stages[-1]
    paired = dict(_key_pairs(pkey, build))
    group = [paired.get(f.name, f.name) for f in join.left.schema]
    build.n_acc_words = _acc_words([], [], bool(build.payload))
    project = [i for _, i in join.column_indices]          # the join's projection: left columns only
    if project == list(range(len(group))):
        project = None
    return GpuPipelineExec(sc, sink="aggregate", group_by=group, mode="Single", out_schema=join.schema, project=project)


def _fuse_hash(plan: "GpuAggregateExec", ch: _Chain) -> Optional["GpuPipelineExec"]:
    """AggregateExec over [ProjectionExec] over an Inner, Right or Full join chain or a FilterExec (as _as_scan accepts them under ch) ->
    ONE GpuPipelineExec with the hash-keyed sink (dfgpu_pipeline_sink_aggregate_hash: TPC-H Q15's revenue0, Q3 grouped by o_custkey), or
    None.  Every group key must be a plain integer-like column of the virtual schema, the packed key (each column at its width, one more
    bit per nullable column) at most 128 bits; at most 4 aggregates, no Float32 MIN / MAX and no SUM / MIN / MAX / AVG over Boolean."""
    below, exprs = _agg_input(plan)
    if not ((isinstance(below, GpuHashJoinExec) and below.join_type in ("Inner", "Right", "Full")) or isinstance(below, GpuFilterExec)):
        return None
    sc = _as_scan(below, ch)
    # a composite-key stage under the hash-keyed sink (TPC-H Q9's lineitem x partsupp profit by supplier) measured slower than the
    # unfused dfgpu_hashjoin -> dfgpu_agg (README): that shape stays unfused
    if sc is None or any(isinstance(k, list) for _, k, _ in sc.stages):
        return None
    if not _settle_right(sc, _read_names(plan, exprs)):
        return None
    vs = sc.virtual_schema()
    group, nullable, bits = [], [], 0
    for g in plan.group_by:
        e = exprs.get(g)
        if not isinstance(e, Column) or e.name not in sc.visible or vs.get_field_index(e.name) < 0:
            return None
        f = vs.field(e.name)
        if not _integer_like(f.type):
            return None
        bits += D.WIDTH[type_id(f.type)] * 8 + (1 if f.nullable else 0)
        group.append(e.name)
        nullable.append(f.nullable)
    if bits > 128 or len(plan.aggr_expr) > 4:
        return None
    args = _agg_args(plan, exprs, vs)
    if args is None or any(a.func in ("min", "max") and t == pa.float32() for a, _, t, _ in args):
        return None
    if any(t is not None and pa.types.is_boolean(t) and a.func != "count" for a, _, t, _ in args):
        return None
    return GpuPipelineExec(sc, sink="hash", group_by=group, aggs=[(a.func, e, a.alias) for a, e, _, _ in args], mode=plan.mode,
                           out_schema=plan.schema, nullable=nullable, fallback=plan if sc.has_right() else None)


def _fuse_output(plan: ExecutionPlan, ch: _Chain) -> Optional["GpuPipelineExec"]:
    """A top-level [ProjectionExec(columns only)] over a HashJoinExec chain that ch allows -> ONE GpuPipelineExec over the ordered output
    sink (dfgpu_pipeline_sink_output) that emits the plan's schema: a probe-side column comes from the input, the build key of an Inner
    stage from its probe key (only when the two have the same type), any other build column from the stage's payload field.  The fused
    lookups need unique build keys: an Inner stage without payload gets a row-counter word, so its build refuses duplicate keys like one
    with payload.  Whether the keys are unique is known only once the build side has run, so the fused node keeps the plan as its
    fallback: a build the library refuses (duplicate keys, NULL payloads) runs the unfused joins instead, before any row is emitted.  The
    fused Inner join emits its rows in probe order, the reference's order for unique build keys.  None for anything else (a bare
    FilterExec, a Left join, a computed projection)."""
    join = plan.input if isinstance(plan, GpuProjectionExec) else plan
    if not isinstance(join, GpuHashJoinExec):
        return None
    sc = _as_scan(join, ch)
    if sc is None:
        return None
    pick = list(range(len(join.column_indices)))                                # the join's columns that form the output
    if isinstance(plan, GpuProjectionExec):
        names = [f.name for f in join.schema]
        if not all(isinstance(e, Column) and names.count(e.name) == 1 for e, _ in plan.exprs):
            return None
        pick = [names.index(e.name) for e, _ in plan.exprs]
    if not _settle_right(sc, {join.schema.field(i).name for i in pick}):
        return None
    vs = sc.virtual_schema()
    kind, pkey, build = sc.stages[-1]
    n_below = len(vs) - (len(build.payload) if kind in (D.STAGE_INNER, D.STAGE_RIGHT) else 0)   # the virtual columns the top join's probe side sees
    keys = {bk: (pk, b) for k, p, b in sc.stages if k == D.STAGE_INNER for bk, pk in _key_pairs(p, b)}   # an Inner stage's build key -> its probe key

    def probe_col(name: str) -> int:
        at = [i for i in range(n_below) if vs.field(i).name == name]
        if len(at) == 1:
            return at[0]
        if not at and name in keys:                                             # a lower Inner stage's build key
            p, b = keys[name]
            i = probe_col(p) if p != name else -1
            return i if i >= 0 and b.scan_field(name).type == vs.field(i).type else -1
        return -1

    cols = []
    for side, ix in (join.column_indices[i] for i in pick):
        if side == 1:
            at = probe_col(join.right.schema.field(ix).name)
        else:
            name = join.left.schema.field(ix).name
            paired = dict(_key_pairs(pkey, build)) if kind != D.STAGE_RIGHT else {}   # a Right join's build key is NULL when unmatched
            if name in paired:
                at = probe_col(paired[name])
                at = at if at >= 0 and join.left.schema.field(ix).type == vs.field(at).type else -1
            else:
                at = n_below + build.payload.index(name) if name in build.payload else -1
        if at < 0:
            return None
        cols.append(at)
    for k, _, b in sc.stages:
        if k == D.STAGE_INNER and not b.payload:
            b.n_acc_words = max(b.n_acc_words, 1)
    return GpuPipelineExec(sc, sink="output", out_schema=plan.schema, out_cols=cols, fallback=plan)


# the levels of the fusion rule, each fusing what the level before it does and more
_JOIN_KEYED, _HASH_SINK, _JOIN_FILTERS, _OUTPUT_SINK, _RIGHT_JOINS, _FULL_JOINS = range(6)


def _fuse(plan: ExecutionPlan, level: int) -> ExecutionPlan:
    """PhysicalOptimizerRule twin (INTEGRATION.md §2a) at `level`: a top-level HashJoinExec(LeftSemi / LeftAnti) onto the join-keyed sink
    (_fuse_left_filter); an AggregateExec(Single / SinglePartitioned / Partial) onto the first sink that takes it: the dense sink, the
    join-keyed sink over a Left or an Inner join, and from _HASH_SINK on the hash sink; from _OUTPUT_SINK on, a plan none of those takes
    onto the ordered output sink.  From _JOIN_FILTERS on a probe chain's joins may carry JoinFilters, from _RIGHT_JOINS on it may
    contain Right joins, and at _FULL_JOINS a Full join.  Anything else is returned unchanged (the unfused Gpu*Exec operators run)."""
    if isinstance(plan, GpuStringTakeExec):        # the gather of plan_string_payloads: fuse the plan of row ids under it
        return _with_children(plan, lambda p: _fuse(p, level))
    joins = _Chain().joins | ({"Right"} if level >= _RIGHT_JOINS else set()) | ({"Full"} if level >= _FULL_JOINS else set())
    ch = _Chain(joins, filters=level >= _JOIN_FILTERS)
    fused = None
    if isinstance(plan, GpuHashJoinExec) and plan.join_type in ("LeftSemi", "LeftAnti"):
        fused = _fuse_left_filter(plan, ch)
    elif isinstance(plan, GpuAggregateExec) and plan.mode in ("Single", "SinglePartitioned", "Partial"):
        fused = _fuse_dense(plan, ch)
        if fused is None and plan.group_by:
            fused = _fuse_left(plan, ch) or _fuse_inner(plan, ch) or (_fuse_hash(plan, ch) if level >= _HASH_SINK else None)
    if fused is None and level >= _OUTPUT_SINK:
        fused = _fuse_output(plan, ch)
    return plan if fused is None else fused


def fuse_pipelines(plan: ExecutionPlan) -> ExecutionPlan:
    """The fusion rule's first level (_fuse): the dense and join-keyed sinks"""
    return _fuse(plan, _JOIN_KEYED)


def fuse_hash_aggregates(plan: ExecutionPlan) -> ExecutionPlan:
    """The fusion rule (_fuse) with the hash-keyed sink too"""
    return _fuse(plan, _HASH_SINK)


def fuse_join_filters(plan: ExecutionPlan) -> ExecutionPlan:
    """The fusion rule (_fuse) with the hash-keyed sink and JoinFilters too"""
    return _fuse(plan, _JOIN_FILTERS)


def fuse_output_pipelines(plan: ExecutionPlan) -> ExecutionPlan:
    """The fusion rule (_fuse) with the hash-keyed sink, JoinFilters and the ordered output sink too"""
    return _fuse(plan, _OUTPUT_SINK)


def fuse_right_joins(plan: ExecutionPlan) -> ExecutionPlan:
    """The fusion rule (_fuse) with the hash-keyed sink, JoinFilters, the ordered output sink and Right joins too: DataFusion's join
    selection puts the smaller input on the build side, so `fact LEFT JOIN dimension` arrives as a Right join with the dimension as the
    build"""
    return _fuse(plan, _RIGHT_JOINS)


def fuse_full_joins(plan: ExecutionPlan) -> ExecutionPlan:
    """The fusion rule (_fuse) at its widest: the hash-keyed sink, JoinFilters, the ordered output sink, Right joins and a Full join too"""
    return _fuse(plan, _FULL_JOINS)


# ---------------------------------------------------------------------------------------------
# string predicates — a mask column computed ahead of the filter (libdfgpu_strings.so)
# ---------------------------------------------------------------------------------------------
_STRING_CMP = {D.OP_EQ: "=", D.OP_NEQ: "<>", D.OP_LT: "<", D.OP_LTEQ: "<=", D.OP_GT: ">", D.OP_GTEQ: ">="}
_MIRRORED = {D.OP_EQ: D.OP_EQ, D.OP_NEQ: D.OP_NEQ, D.OP_LT: D.OP_GT, D.OP_LTEQ: D.OP_GTEQ, D.OP_GT: D.OP_LT, D.OP_GTEQ: D.OP_LTEQ}


def _string_column(e: Expr, schema: pa.Schema, coded: set) -> bool:
    """a Utf8, LargeUtf8 or Utf8View column of schema (not a raw Arrow dictionary), or a column DictionaryEncodeExec coded (`coded`)"""
    if not isinstance(e, Column):
        return False
    ix = schema.get_field_index(e.name)
    return ix >= 0 and (e.name in coded or (_is_string_like(schema.field(ix).type) and not pa.types.is_dictionary(schema.field(ix).type)))


def _utf8_literal(e: Expr) -> bool:
    """a Utf8 literal: a str or NULL of a string type whose text encodes as UTF-8"""
    if not isinstance(e, Literal) or not _is_string_like(e.type) or pa.types.is_dictionary(e.type):
        return False
    if e.value is None:
        return True
    try:
        return isinstance(e.value, str) and e.value.encode("utf-8") is not None
    except UnicodeEncodeError:
        return False


def _like_on_gpu(e: LikeExpr, schema: pa.Schema, coded: set) -> bool:
    """LIKE / NOT LIKE of a Utf8, LargeUtf8 or Utf8View column (or one DictionaryEncodeExec coded: `coded`) with a Utf8 literal pattern
    without `\\`; a NULL pattern too (the predicate folds to NULL)"""
    if e.case_insensitive or not isinstance(e.pattern, Literal):
        return False
    p = e.pattern.value
    if p is not None and (not isinstance(p, str) or "\\" in p):
        return False
    return _string_column(e.expr, schema, coded)


def _string_comparison(e: BinaryExpr, schema: pa.Schema, coded: set) -> Optional[BinaryExpr]:
    """a comparison of a string column with a Utf8 literal as BinaryExpr(column, op, literal), a literal on the left swapped to the right
    with its operator mirrored; None when e is not one or the literal is longer than the library takes"""
    l, op, r = e.left, e.op, e.right
    if isinstance(l, Literal) and not isinstance(r, Literal):
        l, op, r = r, _MIRRORED[op], l
    if not (_string_column(l, schema, coded) and _utf8_literal(r)):
        return None
    if r.value is not None and len(r.value.encode("utf-8")) > D.STRING_MAX_LITERAL_BYTES:
        return None
    return e if l is e.left else BinaryExpr(l, op, r)


def _in_list_on_gpu(e: InListExpr, schema: pa.Schema, coded: set) -> bool:
    """an IN list of Utf8 literals and NULLs over a string column, within the library's caps on distinct values and their bytes"""
    if not _string_column(e.expr, schema, coded) or not all(_utf8_literal(v) for v in e.list):
        return False
    vals = {v.value.encode("utf-8") for v in e.list if v.value is not None}
    return len(vals) <= D.STRING_IN_MAX_VALUES and sum(len(v) for v in vals) <= D.STRING_IN_MAX_BYTES


def _string_operand(e: Expr, schema: pa.Schema) -> bool:
    """a column of a string type, or a literal of one: a comparison reading it must become a mask or stay off the GPU"""
    if isinstance(e, Column):
        ix = schema.get_field_index(e.name)
        return ix >= 0 and _is_string_like(schema.field(ix).type)
    return isinstance(e, Literal) and _is_string_like(e.type)


def _mask_eq(e: Expr, prefix: str, taken: set, likes: list) -> Expr:
    """`mask = 1` for a new mask column computing e (appended to likes as (e, mask name))"""
    name = f"{prefix}_{len(likes)}"
    while name in taken:
        name = "_" + name
    taken.add(name)
    likes.append((e, name))
    return BinaryExpr(Column(name), D.OP_EQ, Literal(1, pa.uint8()))


def _rewrite_likes(e: Expr, schema: pa.Schema, coded: set, taken: set, likes: list, strings: bool = False) -> Optional[Expr]:
    """e with every LIKE that runs on the GPU replaced by `mask = 1` (appended to likes as (predicate, mask name)); None when a LIKE that
    cannot run there remains.  With `strings`, also every comparison of a string column with a Utf8 literal and every IN list of Utf8
    literals over a string column; None when a comparison reading a string, or an IN list, that cannot run there remains."""
    if isinstance(e, LikeExpr):
        if not _like_on_gpu(e, schema, coded):
            return None
        if e.pattern.value is None:
            return Literal(None, pa.bool_())
        return _mask_eq(e, "__like", taken, likes)
    if strings and isinstance(e, InListExpr):
        if not _in_list_on_gpu(e, schema, coded):
            return None
        vals = [v for v in e.list if v.value is not None]
        pred = _mask_eq(InListExpr(e.expr, vals, e.negated), "__in", taken, likes)
        if len(vals) == len(e.list):
            return pred
        # a NULL in the list: a string found nowhere gives NULL.  Kleene logic adds it to the mask of the non-NULL values: IN is
        # `found OR NULL`, NOT IN is `not found AND NULL`.  So the mask stays a plain map of each distinct string (dictionary codes too).
        return BinaryExpr(pred, D.OP_AND if e.negated else D.OP_OR, Literal(None, pa.bool_()))
    if strings and isinstance(e, BinaryExpr) and e.op in _STRING_CMP and (_string_operand(e.left, schema) or _string_operand(e.right, schema)):
        c = _string_comparison(e, schema, coded)
        if c is None:
            return None
        if c.right.value is None:
            return Literal(None, pa.bool_())
        return _mask_eq(c, "__cmp", taken, likes)
    if isinstance(e, BinaryExpr):
        l = _rewrite_likes(e.left, schema, coded, taken, likes, strings)
        r = None if l is None else _rewrite_likes(e.right, schema, coded, taken, likes, strings)
        return None if r is None else (e if (l is e.left and r is e.right) else BinaryExpr(l, e.op, r))
    if isinstance(e, (UnaryExpr, CastExpr)):
        a = _rewrite_likes(e.arg, schema, coded, taken, likes, strings)
        if a is None:
            return None
        if a is e.arg:
            return e
        return UnaryExpr(e.kind, a) if isinstance(e, UnaryExpr) else CastExpr(a, e.to)
    return e


def _with_children(plan: ExecutionPlan, fn) -> ExecutionPlan:
    """plan with fn applied to its input / left / right children (a shallow copy when one changes)"""
    import copy
    changed = {}
    for attr in ("input", "left", "right"):
        ch = getattr(plan, attr, None)
        if isinstance(ch, ExecutionPlan):
            new = fn(ch)
            if new is not ch:
                changed[attr] = new
    if not changed:
        return plan
    out = copy.copy(plan)
    for k, v in changed.items():
        setattr(out, k, v)
    if hasattr(out, "_metrics"):
        out._metrics = {}
    return out


def _plan_masks(plan: ExecutionPlan, strings: bool) -> ExecutionPlan:
    plan = _with_children(plan, lambda p: _plan_masks(p, strings))
    if not isinstance(plan, GpuFilterExec):
        return plan
    inner = plan.input
    isch = inner.schema
    coded = {isch.field(i).name for i in inner.string_cols} if isinstance(inner, DictionaryEncodeExec) else set()
    likes: list = []
    pred = _rewrite_likes(plan.predicate, isch, coded, set(isch.names), likes, strings)
    if pred is None or pred is plan.predicate:
        return plan
    out_names = [f.name for f in plan.schema]
    raw = {_mask_column(e).name for e, _ in likes if _mask_column(e).name not in coded}
    if raw & set(out_names):
        return plan                                       # a string column read above the filter
    drop = raw - _expr_names(pred)
    below = GpuLikeExec(inner, likes, drop, inner.dictionary_of if coded else None) if likes else inner
    projection = [below.schema.get_field_index(n) for n in out_names]
    return GpuFilterExec(pred, below, projection, plan.fetch)


def plan_like_predicates(plan: ExecutionPlan) -> ExecutionPlan:
    """PhysicalOptimizerRule twin (INTEGRATION.md §2c), ahead of the fusion rules: every FilterExec whose predicate holds LikeExpr(column,
    Utf8 literal) over a Utf8, LargeUtf8 or Utf8View column, or over a column DictionaryEncodeExec coded, gets a GpuLikeExec under it that
    appends one UINT8 mask per LIKE and drops the string columns nothing else reads; each LIKE becomes `mask = 1` (Kleene logic holds: a
    NULL mask gives NULL) and the filter projects exactly its old output, so its schema is unchanged.  A filter stays as it was when its
    predicate holds any other LIKE (ILIKE, a column pattern, a `\\` in the pattern) or when a Utf8 column a LIKE reads is also read
    above the filter.  A NULL literal pattern folds to a NULL predicate.  The fusion rules then treat the GpuLikeExec as the pipeline's
    source, as they treat any other node under a filter."""
    return _plan_masks(plan, strings=False)


def plan_string_predicates(plan: ExecutionPlan) -> ExecutionPlan:
    """PhysicalOptimizerRule twin (INTEGRATION.md §3b), ahead of the fusion rules, in place of plan_like_predicates: everything that rule
    rewrites, and also, over the same string columns (Utf8, LargeUtf8, Utf8View, or coded by DictionaryEncodeExec):
      - BinaryExpr(column, =, <>, <, <=, >, >=, Utf8 literal), a literal on the left swapped to the right with its operator mirrored;
        a NULL literal folds to a NULL predicate;
      - InListExpr(column, Utf8 literals and NULLs), [NOT] IN, within the library's caps (64 distinct values, 1024 bytes); a NULL in the
        list becomes `mask OR NULL` (IN) / `mask AND NULL` (NOT IN) over the mask of the non-NULL values.
    Each becomes a GpuLikeExec mask and `mask = 1`, and the filter keeps its schema.  A filter stays as it was when its predicate holds a
    string predicate that cannot run on the GPU (a column compared with a column, an IN list of anything but Utf8 literals or over the
    caps, a LIKE plan_like_predicates leaves), or when a raw string column a predicate reads is also read above the filter."""
    return _plan_masks(plan, strings=True)


# ---------------------------------------------------------------------------------------------
# string payloads — carried string columns as row ids, gathered after the operators (late materialisation, libdfgpu_strings.so)
# ---------------------------------------------------------------------------------------------
def _carried_type(t: pa.DataType) -> bool:
    return pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_string_view(t)


def _compact(a: pa.Array) -> pa.Array:
    """a copy of a string array holding only its own rows' bytes: a batch sliced from a larger array shares the parent's buffers, and
    uploading those would put the whole column on the device once per batch"""
    if pa.types.is_string_view(a.type):
        return a.cast(pa.large_string()).cast(pa.string_view())
    return pa.concat_arrays([a])


class StringPayloadStore:
    """The device-resident strings of the sources GpuStringRowIdExec replaced, for one TaskContext.  A build-side source's batches are
    concatenated into one array per column at its first gather (its ids are UINT32 rows of that array, as collect_left_input
    concatenates the build); a streamed source keeps one array per column per batch (ids: batch << 32 | row).
    Every batch is compacted to its own rows before it is uploaded.
    Memory rule: a build-side source is held until the gather's execute ends, which is when its join's probe side has ended.  A streamed
    source whose ids reach the gather in nondecreasing order releases every batch below the smallest id of each gathered batch: its path
    to the gather runs through filters, projections, mask nodes and the probe side of joins that keep probe order (Inner, Left, Right,
    Full, RightSemi, RightAnti, RightMark; the fused ordered output sink keeps it too).  Any other streamed source is held until the
    gather's execute ends."""

    def __init__(self):
        self.sources: dict = {}     # key -> {"build": bool, "batches": {batch: [DeviceStrings]}, "host": [[pa.Array]], "whole": [DeviceStrings]}
        self.held = self.peak = 0

    def _add_bytes(self, n: int):
        self.held += n
        self.peak = max(self.peak, self.held)

    def open(self, key, build: bool):
        self.release(key)
        self.sources[key] = {"build": build, "batches": {}, "host": [], "whole": None, "released": 0}

    def push(self, ctx: TaskContext, key, batch: int, arrays: List[pa.Array]):
        s = self.sources[key]
        if s["build"]:
            s["host"].append(arrays)                      # uploaded once, concatenated, at the first gather
            return
        ds = [D.DeviceStrings(ctx.gpu, _compact(a)) for a in arrays]
        self._add_bytes(sum(d.nbytes for d in ds))
        s["batches"][batch] = ds

    def build_arrays(self, ctx: TaskContext, key) -> list:
        s = self.sources[key]
        if s["whole"] is None:
            cols = list(zip(*s["host"])) if s["host"] else []
            s["whole"] = [D.DeviceStrings(ctx.gpu, _compact(pa.concat_arrays(list(c)))) for c in cols]
            s["host"] = []
            self._add_bytes(sum(d.nbytes for d in s["whole"]))
        return s["whole"]

    def batches(self, key, lo: int, hi: int, col: int) -> list:
        s = self.sources[key]
        if lo < s["released"]:
            raise RuntimeError(f"string payload batch {lo} of source {key} was released before its gather")
        return [s["batches"][b][col] for b in range(lo, hi + 1)]

    def release_below(self, key, batch: int):
        s = self.sources[key]
        for b in [b for b in s["batches"] if b < batch]:
            self.held -= sum(d.nbytes for d in s["batches"].pop(b))
        s["released"] = max(s["released"], batch)

    def release(self, key):
        s = self.sources.pop(key, None)
        if s is None:
            return
        for ds in s["batches"].values():
            self.held -= sum(d.nbytes for d in ds)
        if s["whole"] is not None:
            self.held -= sum(d.nbytes for d in s["whole"])


def plan_string_payloads_store():
    """a factory for the `store_of` argument: one StringPayloadStore per TaskContext, created on first use"""
    cache = {}

    def get(ctx: TaskContext) -> StringPayloadStore:
        if id(ctx) not in cache:
            cache[id(ctx)] = StringPayloadStore()
        return cache[id(ctx)]
    return get


class GpuStringRowIdExec(ExecutionPlan):
    """A source's carried string columns -> one row-id column (`id_name`, appended) and the strings kept on the device in the
    StringPayloadStore; the columns `drop` (indices) leave the batch, and of them `keep` (indices) are stored.  build: UINT32 rows of
    the concatenated source (a join's build side), else INT64 batch << 32 | row.  With no `keep` no id is made: the columns only go."""

    def __init__(self, input: ExecutionPlan, drop: Sequence[int], keep: Sequence[int], id_name: str, build: bool, key, store_of):
        self.input, self.drop, self.keep, self.id_name, self.build, self.key, self.store_of = input, list(drop), list(keep), id_name, build, key, store_of
        fields = [f for i, f in enumerate(input.schema) if i not in self.drop]
        if self.keep:
            fields.append(pa.field(id_name, pa.uint32() if build else pa.int64(), False))
        self.schema = pa.schema(fields)

    def children(self): return [self.input]

    def execute(self, ctx):
        import numpy as np
        store = self.store_of(ctx)
        if self.keep:
            store.open(self.key, self.build)
        rows = 0
        for b, rb in enumerate(self.input.execute(ctx)):
            cols = [rb.column(i) for i in range(rb.num_columns) if i not in self.drop]
            if self.keep:
                store.push(ctx, self.key, b, [rb.column(i) for i in self.keep])
                n = rb.num_rows
                if self.build:
                    if rows + n > 0xFFFFFFFF:
                        raise NotImplementedError("This feature is not implemented: a build side of more than 2^32 - 1 rows carrying strings")
                    cols.append(pa.array(np.arange(rows, rows + n, dtype=np.uint32)))
                else:
                    cols.append(pa.array((np.int64(b) << 32) | np.arange(n, dtype=np.int64)))
                rows += n
            yield pa.RecordBatch.from_arrays(cols, schema=self.schema)


class GpuStringTakeExec(ExecutionPlan):
    """The gather over a plan whose carried string columns travel as row ids: each output column is an input column (`('col', i)`)
    or the strings its id column names (`('take', id column, source key, stored column)`), by dfgpu_string_take.  schema: the plan's
    schema before plan_string_payloads.  ordered: the streamed source keys whose ids arrive nondecreasing (the store's release rule)."""

    def __init__(self, input: ExecutionPlan, schema: pa.Schema, spec: Sequence[tuple], sources: dict, ordered: Sequence, store_of):
        self.input, self.schema, self.spec, self.sources, self.ordered, self.store_of = input, schema, list(spec), dict(sources), set(ordered), store_of
        self._metrics = {}

    def children(self): return [self.input]

    def _take(self, ctx, store, rb, idx: int, key, col: int) -> pa.Array:
        import numpy as np
        ids = rb.column(idx)
        if ids.null_count == len(ids):                           # no id names a string (an empty batch, an unmatched outer side)
            return pa.nulls(len(ids), self._type_of(key, col))
        if self.sources[key]:                                    # a build side: UINT32 rows of one array
            return D.string_take(ctx.gpu, [store.build_arrays(ctx, key)[col]], ids).to_arrow()
        v = np.asarray(ids.fill_null(0)).astype(np.int64)
        valid = np.asarray(ids.is_valid())
        batch = v[valid] >> 32
        lo, hi = int(batch.min()), int(batch.max())
        packed = pa.array(v - (np.int64(lo) << 32), pa.int64(), mask=None if valid.all() else ~valid)
        return D.string_take(ctx.gpu, store.batches(key, lo, hi, col), packed).to_arrow()

    def _type_of(self, key, col):
        for j, s in enumerate(self.spec):
            if s[0] == "take" and s[2] == key and s[3] == col:
                return self.schema.field(j).type

    def execute(self, ctx):
        import numpy as np
        store = self.store_of(ctx)
        store.peak = store.held
        rows = 0
        try:
            for rb in self.input.execute(ctx):
                cols = [rb.column(s[1]) if s[0] == "col" else self._take(ctx, store, rb, *s[1:]) for s in self.spec]
                rows += rb.num_rows
                yield pa.RecordBatch.from_arrays(cols, schema=self.schema)
                for key in self.ordered:                         # nondecreasing ids: no later batch reaches below this one's smallest
                    idx = next(s[1] for s in self.spec if s[0] == "take" and s[2] == key)
                    ids = rb.column(idx).drop_null()
                    if len(ids):
                        store.release_below(key, int(np.asarray(ids).min()) >> 32)
        finally:
            for key in self.sources:
                store.release(key)
            self._metrics = {"output_rows": rows, "string_bytes_held": store.held, "peak_string_bytes_held": store.peak}

    def metrics(self): return self._metrics


_PAYLOAD_NODES = (GpuFilterExec, GpuHashJoinExec, GpuProjectionExec, GpuLikeExec)


def _payload_origins(plan: ExecutionPlan, leaves: list, reads: set) -> list:
    """the origin (leaf number, leaf column) of each output column of plan, None for a computed one; the leaves in visiting order; the
    origins an operator reads (join keys and JoinFilter operands, predicate and mask inputs, computed projections)"""
    def names(schema, origins, ns):
        return {origins[i] for i, f in enumerate(schema) if f.name in ns}
    if isinstance(plan, GpuFilterExec):
        o = _payload_origins(plan.input, leaves, reads)
        reads |= names(plan.input.schema, o, _expr_names(plan.predicate))
        return o if plan.projection is None else [o[i] for i in plan.projection]
    if isinstance(plan, GpuProjectionExec):
        o = _payload_origins(plan.input, leaves, reads)
        isch = plan.input.schema
        out = []
        for e, _ in plan.exprs:
            if isinstance(e, Column):
                out.append(o[isch.get_field_index(e.name)] if isch.get_field_index(e.name) >= 0 else None)
            else:
                reads |= names(isch, o, _expr_names(e))
                out.append(None)
        return out
    if isinstance(plan, GpuLikeExec):
        o = _payload_origins(plan.input, leaves, reads)
        isch = plan.input.schema
        reads |= names(isch, o, {_mask_column(e).name for e, _ in plan.likes})
        return [o[i] for i, f in enumerate(isch) if f.name not in plan.drop] + [None] * len(plan.likes)
    if isinstance(plan, GpuHashJoinExec):
        lo = _payload_origins(plan.left, leaves, reads)
        ro = _payload_origins(plan.right, leaves, reads)
        reads |= names(plan.left.schema, lo, {l for l, _ in plan.on}) | names(plan.right.schema, ro, {r for _, r in plan.on})
        if plan.filter is not None:
            reads |= {(lo if sd == "left" else ro)[ix] for sd, ix in plan.filter.column_indices}
        return [lo[i] if sd == 0 else ro[i] if sd == 1 else None for sd, i in plan.column_indices]
    leaves.append(plan)
    return [(len(leaves) - 1, i) for i in range(len(plan.schema))]


_PROBE_ORDER = {"Inner", "Left", "Right", "Full", "RightSemi", "RightAnti", "RightMark"}   # joins whose output keeps probe order
_PAYLOAD_REGIONS = iter(range(1 << 62))                                                    # store keys: (region, leaf)


class _PayloadRewrite:
    def __init__(self, carried: set, needed: set, store_of):
        self.carried, self.needed, self.store_of = carried, needed, store_of
        self.region = next(_PAYLOAD_REGIONS)
        self.leaf = 0
        self.kinds: dict = {}       # leaf -> build side?
        self.ordered: set = set()   # streamed leaves whose ids reach the root in order

    def id_name(self, leaf: int) -> str:
        return f"__string_row_id_{leaf}"

    def rewrite(self, plan: ExecutionPlan, build: bool, ordered: bool):
        """-> (plan', tags): tags[i] = ('o', i of plan's output) or ('id', leaf) for each column of plan'"""
        if isinstance(plan, GpuHashJoinExec):
            return self.join(plan, ordered)
        if not isinstance(plan, _PAYLOAD_NODES):
            return self.source(plan, build, ordered)
        new_in, it = self.rewrite(plan.input, build, ordered)
        same = [("o", i) for i in range(len(plan.schema))]
        if new_in is plan.input:
            return plan, same
        ids = [t for t in it if t[0] == "id"]
        if isinstance(plan, GpuFilterExec):
            if plan.projection is None:
                return GpuFilterExec(plan.predicate, new_in, None, plan.fetch), it
            keep = [(j, it.index(("o", i))) for j, i in enumerate(plan.projection) if ("o", i) in it]
            proj = [p for _, p in keep] + [it.index(t) for t in ids]
            return GpuFilterExec(plan.predicate, new_in, proj, plan.fetch), [("o", j) for j, _ in keep] + ids
        if isinstance(plan, GpuProjectionExec):
            isch = plan.input.schema
            keep = [(j, e, n) for j, (e, n) in enumerate(plan.exprs)
                    if not isinstance(e, Column) or ("o", isch.get_field_index(e.name)) in it]
            exprs = [(e, n) for _, e, n in keep] + [(Column(self.id_name(t[1])), self.id_name(t[1])) for t in ids]
            return GpuProjectionExec(exprs, new_in), [("o", j) for j, _, _ in keep] + ids
        # GpuLikeExec: the input minus `drop`, then the masks
        isch = plan.input.schema
        out_of = {i: j for j, i in enumerate(i for i, f in enumerate(isch) if f.name not in plan.drop)}
        tags = [("o", out_of[t[1]]) if t[0] == "o" else t for t in it if t[0] == "id" or isch.field(t[1]).name not in plan.drop]
        n_in = len(out_of)
        return GpuLikeExec(new_in, plan.likes, plan.drop, plan.dictionary_of), tags + [("o", n_in + k) for k in range(len(plan.likes))]

    def source(self, plan: ExecutionPlan, build: bool, ordered: bool):
        leaf = self.leaf
        self.leaf += 1
        inner = plan_string_payloads(plan, self.store_of)   # the operators under a node the rule does not pass through; same schema
        drop = [i for i in range(len(plan.schema)) if (leaf, i) in self.carried]
        if not drop:
            return inner, [("o", i) for i in range(len(plan.schema))]
        keep = [i for i in drop if (leaf, i) in self.needed]
        node = GpuStringRowIdExec(inner, drop, keep, self.id_name(leaf), build, (self.region, leaf), self.store_of)
        if keep:
            self.kinds[leaf] = build
            if ordered and not build:
                self.ordered.add(leaf)
        return node, [("o", i) for i in range(len(plan.schema)) if i not in drop] + ([("id", leaf)] if keep else [])

    def join(self, plan: GpuHashJoinExec, ordered: bool):
        nl, lt = self.rewrite(plan.left, True, False)
        nr, rt = self.rewrite(plan.right, False, ordered and plan.join_type in _PROBE_ORDER)
        if nl is plan.left and nr is plan.right:
            return plan, [("o", i) for i in range(len(plan.schema))]
        _, old_idx = build_join_schema(plan.left.schema, plan.right.schema, plan.join_type)
        _, new_idx = build_join_schema(nl.schema, nr.schema, plan.join_type)
        child = {0: lt, 1: rt}

        def new_pos(sd, i):             # the new natural-output position of old child column (sd, i), -1 when it left
            if sd == 2:
                return new_idx.index((2, 0))
            t = ("o", i)
            return new_idx.index((sd, child[sd].index(t))) if t in child[sd] else -1
        filt = plan.filter
        if filt is not None:
            filt = JoinFilter(filt.expression, [(sd, (lt if sd == "left" else rt).index(("o", ix))) for sd, ix in filt.column_indices])
        id_pos = [p for p, (sd, i) in enumerate(new_idx) if sd != 2 and child[sd][i][0] == "id"]
        if list(plan.column_indices) == old_idx:      # no projection
            def tag(sd, i):
                if sd == 2:
                    return ("o", old_idx.index((2, 0)))
                t = child[sd][i]
                return ("o", old_idx.index((sd, t[1]))) if t[0] == "o" else t
            tags = [tag(sd, i) for sd, i in new_idx]
            return GpuHashJoinExec(nl, nr, plan.on, plan.join_type, plan.null_equality, filt, None, plan.null_aware), tags
        keep = [(j, new_pos(sd, i)) for j, (sd, i) in enumerate(plan.column_indices)]
        keep = [(j, p) for j, p in keep if p >= 0]
        proj = [p for _, p in keep] + id_pos
        tags = [("o", j) for j, _ in keep] + [child[new_idx[p][0]][new_idx[p][1]] for p in id_pos]
        return GpuHashJoinExec(nl, nr, plan.on, plan.join_type, plan.null_equality, filt, proj, plan.null_aware), tags


def plan_string_payloads(plan: ExecutionPlan, store_of=None) -> ExecutionPlan:
    """PhysicalOptimizerRule twin (INTEGRATION.md §3c), after plan_string_predicates and ahead of the fusion rules: late materialisation
    of the string columns a plan of GPU operators (GpuFilterExec, GpuHashJoinExec, GpuProjectionExec column pass-throughs, GpuLikeExec)
    only carries.  Every Utf8, LargeUtf8 or Utf8View column of a source that no operator reads (not a join key, JoinFilter operand,
    predicate or mask input, computed-projection input) leaves at the source: when some output needs one of a source's columns, a
    GpuStringRowIdExec replaces them by one row-id column (UINT32 rows of the concatenated build on a join's build side, else INT64
    batch << 32 | row) and keeps their strings on the device; else they are dropped outright.  The operators carry the ids as any
    fixed-width column (NULL on the outer side of Left / Right / Full joins) and a GpuStringTakeExec at the plan's root gathers the
    strings (dfgpu_string_take), emitting the plan's schema exactly.  A column an operator reads stays as it is.  Under a
    GpuAggregateExec (not a Final mode) the operators' output is what the aggregate reads: its group and argument columns stay as they
    are, the strings it does not read are dropped at their sources, and no gather is needed.  Any other node the rule does not pass
    through gets the rule on its children.  A plan with no carried string column is returned as it is.  store_of: the
    StringPayloadStore factory (plan_string_payloads_store())."""
    store_of = store_of or plan_string_payloads_store()
    if isinstance(plan, GpuAggregateExec) and not plan.state_input and isinstance(plan.input, _PAYLOAD_NODES):
        read = set(plan.group_by) | {a.arg for a in plan.aggr_expr if a.arg} | {a.filter for a in plan.aggr_expr if a.filter}
        new_in = _plan_payloads(plan.input, store_of, {i for i, f in enumerate(plan.input.schema) if f.name in read})
        if new_in is plan.input:
            return plan
        return GpuAggregateExec(plan.mode, plan.group_by, plan.aggr_expr, new_in,
                                None if plan.input_schema is plan.input.schema else plan.input_schema, plan.capacity_hint)
    if not isinstance(plan, _PAYLOAD_NODES):
        return _with_children(plan, lambda p: plan_string_payloads(p, store_of))
    return _plan_payloads(plan, store_of, None)


def _plan_payloads(plan: ExecutionPlan, store_of, read_above: Optional[set]) -> ExecutionPlan:
    """plan_string_payloads on a plan whose root is one of its operators.  read_above: the output columns the node above reads, which
    stay as they are while the other carried strings leave (None: the node above needs every output column as it is now)"""
    leaves: list = []
    reads: set = set()
    origins = _payload_origins(plan, leaves, reads)
    if read_above is not None:
        reads |= {origins[j] for j in read_above if origins[j] is not None}
    carried = {(k, i) for k, leaf in enumerate(leaves) for i, f in enumerate(leaf.schema) if _carried_type(f.type) and (k, i) not in reads}
    wanted = range(len(origins)) if read_above is None else read_above
    needed = {origins[j] for j in wanted if origins[j] in carried}
    rw = _PayloadRewrite(carried, needed, store_of)
    new, tags = rw.rewrite(plan, False, True)
    if new is plan:
        return plan
    stored = {k: [i for i in range(len(leaves[k].schema)) if (k, i) in needed] for k in rw.kinds}
    spec, fields = [], []
    for j, o in enumerate(origins):
        if ("o", j) in tags:
            spec.append(("col", tags.index(("o", j))))
        elif o in needed:
            spec.append(("take", tags.index(("id", o[0])), (rw.region, o[0]), stored[o[0]].index(o[1])))
        else:
            continue                                     # a carried string nothing above reads: dropped at its source
        fields.append(plan.schema.field(j))
    if all(s[0] == "col" for s in spec):                 # no id was made, nothing to gather
        return new
    return GpuStringTakeExec(new, pa.schema(fields), spec, {(rw.region, k): b for k, b in rw.kinds.items()},
                             {(rw.region, k) for k in rw.ordered}, store_of)


def collect(plan: ExecutionPlan, ctx: Optional[TaskContext] = None) -> List[pa.RecordBatch]:
    """physical-plan/src/execution_plan.rs:1752"""
    ctx = ctx or TaskContext()
    return [b for b in plan.execute(ctx) if b.num_rows > 0]
