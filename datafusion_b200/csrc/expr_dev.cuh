// expr_dev.cuh — the device-side PhysicalExpr interpreter (post-order program evaluated per row in registers),
// shared by FilterExec (filter.cu), the JoinFilter (hash_join.cu) and the fused pipeline (pipeline.cu).
// Reference semantics: BinaryExpr::evaluate physical-expr/src/expressions/binary.rs:536-676, datum.rs:36-105,
// and_kleene / or_kleene binary.rs:1093-1116, CastExpr expressions/cast.rs:37-40.
#pragma once
#include "batch.cuh"

namespace dfgpu {

// internal node kind (never crosses the C ABI): a field of a 64-bit payload word fetched by a fused join probe.
// voff = index of the payload word in the per-row `ext` array, lit = bit shift, out_type = field type.
constexpr int kExprExt = 100;
// The interpreters' XN parameter (nullable payload fields: the fused pipeline's RIGHT stages): ext[kExtValid], behind the payload words,
// holds the row's validity bits, bit s = the fields of payload word s are valid.  Without XN a payload field is never NULL.
constexpr int kExtValid = 3;

constexpr int kMaxNodes = 48;
constexpr int kMaxStack = 16;

struct ENode {
  int kind, op;
  int in_type;   // operand type (binary / unary / cast source)
  int out_type;
  const void* col; const uint8_t* valid; int64_t voff;  // COLUMN (BOOL: voff is also the value bit offset)
  uint64_t lit; int lit_null;
  // short-circuit guards (BinaryExpr::evaluate, binary.rs:536-600 + check_short_circuit :1182): when this node lies in the RHS of an
  // AND / OR whose LHS lets the reference skip or pre-select the RHS for this batch, an error raised here counts only on the rows the
  // reference would have evaluated: bit s of g_and = "stack slot s (that AND's LHS) must be TRUE", of g_or = "... must be FALSE".
  uint16_t g_and, g_or;
};
struct EProgram { int n; ENode node[kMaxNodes]; };

enum Cls : int { C_I64 = 0, C_U64 = 1, C_F64 = 2, C_BOOL = 3, C_DEC = 4 /* Decimal128: 128-bit stack, expr_dec.cuh */ };
// class of a primitive (non-decimal) type: what the 64-bit interpreter dispatches on
__host__ __device__ inline int cls_of_prim(int t) {
  if (t == DFGPU_BOOL) return C_BOOL;
  if (type_is_float(t)) return C_F64;
  if (type_is_unsigned_int(t)) return C_U64;
  return C_I64;
}
__host__ __device__ inline int cls_of(int t) { return type_is_decimal(t) ? C_DEC : cls_of_prim(t); }

// values travel on the evaluation stack as 64-bit payloads: ints sign/zero-extended, floats as
// f64 bits (f32 widened exactly), bools as 0/1.
__device__ __forceinline__ uint64_t load_col_value(const ENode& nd, int64_t row) {
  switch (nd.out_type) {
    case DFGPU_BOOL: return bit_get((const uint8_t*)nd.col, nd.voff + row) ? 1ull : 0ull;
    case DFGPU_INT8: return (uint64_t)(int64_t)((const int8_t*)nd.col)[row];
    case DFGPU_INT16: return (uint64_t)(int64_t)((const int16_t*)nd.col)[row];
    case DFGPU_INT32: case DFGPU_DATE32: return (uint64_t)(int64_t)((const int32_t*)nd.col)[row];
    case DFGPU_UINT8: return ((const uint8_t*)nd.col)[row];
    case DFGPU_UINT16: return ((const uint16_t*)nd.col)[row];
    case DFGPU_UINT32: return ((const uint32_t*)nd.col)[row];
    case DFGPU_FLOAT32: { double d = (double)((const float*)nd.col)[row]; return (uint64_t)__double_as_longlong(d); }
    default: return ((const uint64_t*)nd.col)[row];
  }
}

// wrap an integer result to the width of its Arrow type (add_wrapping on Int32 wraps at 32 bits)
__device__ __forceinline__ uint64_t wrap_to_type(uint64_t v, int t) {
  switch (t) {
    case DFGPU_INT8: return (uint64_t)(int64_t)(int8_t)v;
    case DFGPU_INT16: return (uint64_t)(int64_t)(int16_t)v;
    case DFGPU_INT32: case DFGPU_DATE32: return (uint64_t)(int64_t)(int32_t)v;
    case DFGPU_UINT8: return v & 0xFFull;
    case DFGPU_UINT16: return v & 0xFFFFull;
    case DFGPU_UINT32: return v & 0xFFFFFFFFull;
    case DFGPU_FLOAT32: { float f = (float)__longlong_as_double((long long)v); return (uint64_t)__double_as_longlong((double)f); }
    default: return v;
  }
}

// IEEE-754 totalOrder compare after -0.0 -> +0.0 normalisation (datum.rs:88-105)
__device__ __forceinline__ int cmp_f64_total(double a, double b) {
  long long x = __double_as_longlong(a), y = __double_as_longlong(b);
  if ((x << 1) == 0) x = 0;
  if ((y << 1) == 0) y = 0;
  x ^= (long long)((unsigned long long)(x >> 63) >> 1);
  y ^= (long long)((unsigned long long)(y >> 63) >> 1);
  return x < y ? -1 : (x > y ? 1 : 0);
}

enum ErrBits : int { ERR_DIV_ZERO = 1, ERR_OVERFLOW = 2, ERR_CAST = 4 };

__device__ __forceinline__ void eval_binary(const ENode& nd, uint64_t a, bool av, uint64_t b, bool bv, uint64_t* r, bool* rv, int* err) {
  const int op = nd.op;
  const int c = cls_of_prim(nd.in_type);
  // ---- Kleene logic (and_kleene / or_kleene) ----
  if (op == DFGPU_OP_AND) {
    bool at = av && a, af = av && !a, bt = bv && b, bf = bv && !b;
    if (af || bf) { *r = 0; *rv = true; } else if (at && bt) { *r = 1; *rv = true; } else { *r = 0; *rv = false; }
    return;
  }
  if (op == DFGPU_OP_OR) {
    bool at = av && a, af = av && !a, bt = bv && b, bf = bv && !b;
    if (at || bt) { *r = 1; *rv = true; } else if (af && bf) { *r = 0; *rv = true; } else { *r = 0; *rv = false; }
    return;
  }
  // ---- comparisons ----
  if (op <= DFGPU_OP_GTEQ || op == DFGPU_OP_IS_DISTINCT_FROM || op == DFGPU_OP_IS_NOT_DISTINCT_FROM) {
    int cmp;
    if (c == C_F64) cmp = cmp_f64_total(__longlong_as_double((long long)a), __longlong_as_double((long long)b));
    else if (c == C_U64 || c == C_BOOL) cmp = a < b ? -1 : (a > b ? 1 : 0);
    else cmp = (long long)a < (long long)b ? -1 : ((long long)a > (long long)b ? 1 : 0);
    if (op == DFGPU_OP_IS_DISTINCT_FROM || op == DFGPU_OP_IS_NOT_DISTINCT_FROM) {
      bool distinct = (av != bv) || (av && bv && cmp != 0);
      *r = (op == DFGPU_OP_IS_DISTINCT_FROM) ? distinct : !distinct;
      *rv = true;  // never NULL (arrow-ord distinct / not_distinct)
      return;
    }
    bool res;
    switch (op) {
      case DFGPU_OP_EQ: res = cmp == 0; break;
      case DFGPU_OP_NEQ: res = cmp != 0; break;
      case DFGPU_OP_LT: res = cmp < 0; break;
      case DFGPU_OP_LTEQ: res = cmp <= 0; break;
      case DFGPU_OP_GT: res = cmp > 0; break;
      default: res = cmp >= 0; break;
    }
    *r = res; *rv = av && bv;  // result null = union of operand nulls (datum.rs:36-58)
    return;
  }
  // ---- arithmetic / bitwise: null if either side is null; kernels run only on valid slots ----
  *rv = av && bv;
  if (!*rv) { *r = 0; return; }
  if (c == C_F64) {
    double x = __longlong_as_double((long long)a), y = __longlong_as_double((long long)b), z;
    switch (op) {
      case DFGPU_OP_PLUS: z = x + y; break;
      case DFGPU_OP_MINUS: z = x - y; break;
      case DFGPU_OP_MULTIPLY: z = x * y; break;
      case DFGPU_OP_DIVIDE: z = x / y; break;
      case DFGPU_OP_MODULO: z = fmod(x, y); break;
      default: z = 0; break;
    }
    if (nd.out_type == DFGPU_FLOAT32) {
      // f32 arithmetic happens in f32 in the reference: both inputs are exact f32 values, so round once
      float xf = (float)x, yf = (float)y, zf;
      switch (op) {
        case DFGPU_OP_PLUS: zf = xf + yf; break;
        case DFGPU_OP_MINUS: zf = xf - yf; break;
        case DFGPU_OP_MULTIPLY: zf = xf * yf; break;
        case DFGPU_OP_DIVIDE: zf = xf / yf; break;
        case DFGPU_OP_MODULO: zf = fmodf(xf, yf); break;
        default: zf = 0; break;
      }
      z = (double)zf;
    }
    *r = (uint64_t)__double_as_longlong(z);
    return;
  }
  uint64_t z = 0;
  switch (op) {
    case DFGPU_OP_PLUS: z = a + b; break;       // add_wrapping
    case DFGPU_OP_MINUS: z = a - b; break;      // sub_wrapping
    case DFGPU_OP_MULTIPLY: z = a * b; break;   // mul_wrapping
    case DFGPU_OP_DIVIDE:
    case DFGPU_OP_MODULO:
      if (b == 0) { *err |= ERR_DIV_ZERO; z = 0; break; }  // ArrowError::DivideByZero
      if (c == C_I64) {
        long long x = (long long)a, y = (long long)b;
        // MIN / -1 overflows the type: arrow's checked `div` reports ArithmeticOverflow; `rem` yields 0
        bool ovf = (y == -1) && (wrap_to_type((uint64_t)(-x), nd.out_type) == (uint64_t)x) && x != 0;
        if (ovf) { if (op == DFGPU_OP_DIVIDE) *err |= ERR_OVERFLOW; z = 0; }
        else z = (uint64_t)(op == DFGPU_OP_DIVIDE ? x / y : x % y);
      } else z = op == DFGPU_OP_DIVIDE ? a / b : a % b;
      break;
    case DFGPU_OP_BITAND: z = a & b; break;
    case DFGPU_OP_BITOR: z = a | b; break;
    case DFGPU_OP_BITXOR: z = a ^ b; break;
    // arrow's bitwise_shift_left / _right are `wrapping_shl` / `wrapping_shr`: the shift amount is taken modulo the bit width
    // (binary.rs bitwise_shift_array_overflow_test: 2 << 100 = 32 for Int32), sign-propagating for signed types
    case DFGPU_OP_SHIFT_LEFT: { const int w = type_width_prim(nd.out_type) * 8; z = a << (b & (uint64_t)(w - 1)); break; }
    case DFGPU_OP_SHIFT_RIGHT: {
      const int w = type_width_prim(nd.out_type) * 8;
      const uint64_t sh = b & (uint64_t)(w - 1);
      if (c == C_I64) z = (uint64_t)((long long)a >> sh);
      else z = a >> sh;
      break;
    }
  }
  *r = wrap_to_type(z, nd.out_type);
}

// CastExpr with the default CastOptions { safe: false } (expressions/cast.rs:37-40): a value that does not fit the integer target is
// an error ("Can't cast value ..."), not a wrapped or NULL result; NULL slots never raise.  Float -> int truncates toward zero.
__device__ __forceinline__ uint64_t cast_value(uint64_t v, int from, int to, bool valid, int* err) {
  int cf = cls_of_prim(from), ct = cls_of_prim(to);
  if (ct == C_F64) {
    // an integer -> Float32 cast is Rust's `as f32` (arrow-cast's numeric cast): one rounding, straight from the integer.  Through a
    // double it would round twice: Int64 2^60 + 2^36 + 1 would give 0x5d800000 instead of 0x5d800001.
    if (to == DFGPU_FLOAT32 && cf != C_F64) {
      const float f = cf == C_I64 ? __ll2float_rn((long long)v) : __ull2float_rn(v);
      return (uint64_t)__double_as_longlong((double)f);
    }
    double d = cf == C_F64 ? __longlong_as_double((long long)v) : (cf == C_U64 || cf == C_BOOL ? (double)v : (double)(long long)v);
    if (to == DFGPU_FLOAT32) d = (double)(float)d;
    return (uint64_t)__double_as_longlong(d);
  }
  if (ct == C_BOOL) return cf == C_F64 ? (__longlong_as_double((long long)v) != 0.0) : (v != 0);
  const int w = type_width_prim(to) * 8;
  uint64_t iv = v;
  bool fits = true;
  if (cf == C_F64) {
    const double d = __longlong_as_double((long long)v);
    const double t = trunc(d);
    fits = isfinite(d) && (ct == C_U64 ? (t >= 0.0 && t < ldexp(1.0, w)) : (t >= -ldexp(1.0, w - 1) && t < ldexp(1.0, w - 1)));
    iv = !fits ? 0ull : (ct == C_U64 ? (uint64_t)t : (uint64_t)(long long)t);
  } else if (cf == C_I64) {
    const long long x = (long long)v;
    fits = ct == C_I64 ? (w == 64 || (x >= -(1ll << (w - 1)) && x < (1ll << (w - 1)))) : (x >= 0 && (w == 64 || x < (1ll << w)));
  } else if (cf == C_U64) {
    fits = ct == C_I64 ? (v < (1ull << (w - 1))) : (w == 64 || v < (1ull << w));
  }
  if (!fits) { if (valid) *err |= ERR_CAST; return 0; }
  return wrap_to_type(iv, to);
}

// evaluate the post-order program for one row: value bits + validity
template <bool XN = false>
__device__ __forceinline__ uint64_t eval_nodes(const ENode* __restrict__ nodes, int n_nodes, int64_t row, bool* ok_out, int* err, const uint64_t* ext = nullptr) {
  uint64_t sv[kMaxStack];
  bool sk[kMaxStack];
  int sp = 0;
#pragma unroll 1
  for (int i = 0; i < n_nodes; ++i) {
    const ENode& nd = nodes[i];
    switch (nd.kind) {
      case DFGPU_EXPR_COLUMN:
    sk[sp] = !(nd.valid && !bit_get(nd.valid, nd.voff + row));
    sv[sp] = load_col_value(nd, row);
    ++sp;
    break;
      case DFGPU_EXPR_LITERAL:
    sk[sp] = !nd.lit_null; sv[sp] = nd.lit; ++sp;
    break;
      case kExprExt: {
    uint64_t v = ext[nd.voff] >> (int)nd.lit;
    const int w = type_width_prim(nd.out_type);
    if (w < 8) { v &= (1ull << (8 * w)) - 1ull; if (type_is_signed_int(nd.out_type)) v = (uint64_t)(((int64_t)(v << (64 - 8 * w))) >> (64 - 8 * w)); }
    if (nd.out_type == DFGPU_FLOAT32) { float f = __uint_as_float((uint32_t)v); v = (uint64_t)__double_as_longlong((double)f); }
    sk[sp] = XN ? ((ext[kExtValid] >> nd.voff) & 1ull) != 0 : true; sv[sp] = v; ++sp;
    break;
      }
      case DFGPU_EXPR_BINARY: {
    uint64_t r; bool ok;
    int e = 0;
    eval_binary(nd, sv[sp - 2], sk[sp - 2], sv[sp - 1], sk[sp - 1], &r, &ok, &e);
    if (e) {
      bool counts = true;
      for (int g = 0; g < kMaxStack; ++g) {
        if ((nd.g_and >> g) & 1) counts = counts && sk[g] && sv[g];
        if ((nd.g_or >> g) & 1) counts = counts && sk[g] && !sv[g];
      }
      if (counts) *err |= e;
    }
    sp -= 1; sv[sp - 1] = r; sk[sp - 1] = ok;
    break;
      }
      case DFGPU_EXPR_NOT: sv[sp - 1] = sv[sp - 1] ? 0 : 1; break;  // NULL stays NULL
      case DFGPU_EXPR_IS_NULL: sv[sp - 1] = sk[sp - 1] ? 0 : 1; sk[sp - 1] = true; break;
      case DFGPU_EXPR_IS_NOT_NULL: sv[sp - 1] = sk[sp - 1] ? 1 : 0; sk[sp - 1] = true; break;
      case DFGPU_EXPR_NEGATIVE:
    if (cls_of_prim(nd.out_type) == C_F64) sv[sp - 1] ^= 0x8000000000000000ull;
    else sv[sp - 1] = wrap_to_type(0ull - sv[sp - 1], nd.out_type);  // neg_wrapping
    break;
      case DFGPU_EXPR_CAST: {
    int e = 0;
    sv[sp - 1] = cast_value(sv[sp - 1], nd.in_type, nd.out_type, sk[sp - 1], &e);
    if (e) {
      bool counts = true;
      for (int g = 0; g < kMaxStack; ++g) {
        if ((nd.g_and >> g) & 1) counts = counts && sk[g] && sv[g];
        if ((nd.g_or >> g) & 1) counts = counts && sk[g] && !sv[g];
      }
      if (counts) *err |= e;
    }
    break;
      }
    }
  }
  *ok_out = sk[0];
  return sv[0];
}
// Register-resident variant for shallow programs (stack depth <= DEPTH): every stack slot is addressed through fully
// unrolled selects, so the stack never leaves the register file (the indexed arrays of eval_nodes live in local memory,
// which costs an L1 round trip per push / pop and — in divergent consumers — real L2 / DRAM traffic).
template <int DEPTH, bool XN = false>
__device__ __forceinline__ uint64_t eval_nodes_reg(const ENode* __restrict__ nodes, int n_nodes, int64_t row, bool* ok_out, int* err, const uint64_t* ext = nullptr) {
  uint64_t sv[DEPTH];
  bool sk[DEPTH];
#pragma unroll
  for (int d = 0; d < DEPTH; ++d) { sv[d] = 0; sk[d] = false; }
  int sp = 0;
#define DF_PUSH(V, K) do { const uint64_t _v = (V); const bool _k = (K); _Pragma("unroll") for (int d = 0; d < DEPTH; ++d) if (d == sp) { sv[d] = _v; sk[d] = _k; } ++sp; } while (0)
#define DF_GET(I, V, K) do { _Pragma("unroll") for (int d = 0; d < DEPTH; ++d) if (d == (I)) { V = sv[d]; K = sk[d]; } } while (0)
#define DF_SET(I, V, K) do { const uint64_t _v = (V); const bool _k = (K); _Pragma("unroll") for (int d = 0; d < DEPTH; ++d) if (d == (I)) { sv[d] = _v; sk[d] = _k; } } while (0)
#pragma unroll 1
  for (int i = 0; i < n_nodes; ++i) {
    const ENode& nd = nodes[i];
    if (nd.kind == DFGPU_EXPR_COLUMN) {
      DF_PUSH(load_col_value(nd, row), !(nd.valid && !bit_get(nd.valid, nd.voff + row)));
    } else if (nd.kind == DFGPU_EXPR_LITERAL) {
      DF_PUSH(nd.lit, !nd.lit_null);
    } else if (nd.kind == kExprExt) {
      uint64_t v = ext[nd.voff] >> (int)nd.lit;
      const int w = type_width_prim(nd.out_type);
      if (w < 8) { v &= (1ull << (8 * w)) - 1ull; if (type_is_signed_int(nd.out_type)) v = (uint64_t)(((int64_t)(v << (64 - 8 * w))) >> (64 - 8 * w)); }
      if (nd.out_type == DFGPU_FLOAT32) { float f = __uint_as_float((uint32_t)v); v = (uint64_t)__double_as_longlong((double)f); }
      DF_PUSH(v, XN ? ((ext[kExtValid] >> nd.voff) & 1ull) != 0 : true);
    } else if (nd.kind == DFGPU_EXPR_BINARY) {
      uint64_t a = 0, b = 0, r; bool ak = false, bk = false, ok;
      DF_GET(sp - 2, a, ak); DF_GET(sp - 1, b, bk);
      int e = 0;
      eval_binary(nd, a, ak, b, bk, &r, &ok, &e);
      if (e) {
        bool counts = true;
#pragma unroll
        for (int d = 0; d < DEPTH; ++d) {
          if ((nd.g_and >> d) & 1) counts = counts && sk[d] && sv[d];
          if ((nd.g_or >> d) & 1) counts = counts && sk[d] && !sv[d];
        }
        if (counts) *err |= e;
      }
      sp -= 1;
      DF_SET(sp - 1, r, ok);
    } else {
      uint64_t a = 0; bool ak = false;
      DF_GET(sp - 1, a, ak);
      switch (nd.kind) {
        case DFGPU_EXPR_NOT: a = a ? 0 : 1; break;  // NULL stays NULL
        case DFGPU_EXPR_IS_NULL: a = ak ? 0 : 1; ak = true; break;
        case DFGPU_EXPR_IS_NOT_NULL: a = ak ? 1 : 0; ak = true; break;
        case DFGPU_EXPR_NEGATIVE:
          if (cls_of_prim(nd.out_type) == C_F64) a ^= 0x8000000000000000ull;
          else a = wrap_to_type(0ull - a, nd.out_type);  // neg_wrapping
          break;
        case DFGPU_EXPR_CAST: {
          int e = 0;
          a = cast_value(a, nd.in_type, nd.out_type, ak, &e);
          if (e) {
            bool counts = true;
#pragma unroll
            for (int d = 0; d < DEPTH; ++d) {
              if ((nd.g_and >> d) & 1) counts = counts && sk[d] && sv[d];
              if ((nd.g_or >> d) & 1) counts = counts && sk[d] && !sv[d];
            }
            if (counts) *err |= e;
          }
          break;
        }
      }
      DF_SET(sp - 1, a, ak);
    }
  }
#undef DF_PUSH
#undef DF_GET
#undef DF_SET
  *ok_out = sk[0];
  return sv[0];
}

__device__ __forceinline__ uint64_t eval_row(const EProgram& p, int64_t row, bool* ok_out, int* err) { return eval_nodes(p.node, p.n, row, ok_out, err); }

}  // namespace dfgpu
