// expr_dec.cuh — the 128-bit variant of the device PhysicalExpr interpreter: programs that touch Decimal128 values.
//
// Reference semantics: BinaryExpr::evaluate (physical-expr/src/expressions/binary.rs:536-676) hands decimal operands to
// arrow-arith's `decimal_op` and CastExpr to arrow-cast's decimal casts.  Both crates are third-party (arrow-arith / arrow-cast
// 59.2.0, pinned by the reference's Cargo.lock, absent from its tree): the published algorithm is restated here and in
// oracle/oracle.py (`_dec_binary`, `_dec_cast`) and anchored on the reference's own vectors binary.rs:4355-5000
// (comparison_decimal_expr_test, arithmetic_decimal_expr_test, arithmetic_divide_zero).
//
// Every stack slot is a 128-bit integer; non-decimal values (ints, float bits, booleans) travel in its low 64 bits and are
// handled by the same eval_binary / cast_value as the 64-bit interpreter.  The planner (filter.cu plan_expr) has already
// derived the result type of every node and the power-of-ten rescale exponents, which ride in ENode::voff:
//   BINARY on decimals: voff = l_exp | r_exp << 8  (operands are multiplied by 10^l_exp / 10^r_exp before the operation)
//   CAST              : voff = |scale delta| (10^voff is the multiplier or divisor)
//   LITERAL           : lit = low 64 bits, voff = high 64 bits
#pragma once
#include "expr_dev.cuh"

namespace dfgpu {

typedef __int128 i128;
typedef unsigned __int128 u128;

// 10^0 .. 10^38 as {lo, hi}
__device__ const unsigned long long kPow10Tab[39][2] = {
    {0x0000000000000001ull, 0x0ull}, {0x000000000000000aull, 0x0ull}, {0x0000000000000064ull, 0x0ull}, {0x00000000000003e8ull, 0x0ull},
    {0x0000000000002710ull, 0x0ull}, {0x00000000000186a0ull, 0x0ull}, {0x00000000000f4240ull, 0x0ull}, {0x0000000000989680ull, 0x0ull},
    {0x0000000005f5e100ull, 0x0ull}, {0x000000003b9aca00ull, 0x0ull}, {0x00000002540be400ull, 0x0ull}, {0x000000174876e800ull, 0x0ull},
    {0x000000e8d4a51000ull, 0x0ull}, {0x000009184e72a000ull, 0x0ull}, {0x00005af3107a4000ull, 0x0ull}, {0x00038d7ea4c68000ull, 0x0ull},
    {0x002386f26fc10000ull, 0x0ull}, {0x016345785d8a0000ull, 0x0ull}, {0x0de0b6b3a7640000ull, 0x0ull}, {0x8ac7230489e80000ull, 0x0ull},
    {0x6bc75e2d63100000ull, 0x5ull}, {0x35c9adc5dea00000ull, 0x36ull}, {0x19e0c9bab2400000ull, 0x21eull}, {0x02c7e14af6800000ull, 0x152dull},
    {0x1bcecceda1000000ull, 0xd3c2ull}, {0x161401484a000000ull, 0x84595ull}, {0xdcc80cd2e4000000ull, 0x52b7d2ull}, {0x9fd0803ce8000000ull, 0x33b2e3cull},
    {0x3e25026110000000ull, 0x204fce5eull}, {0x6d7217caa0000000ull, 0x1431e0faeull}, {0x4674edea40000000ull, 0xc9f2c9cd0ull}, {0xc0914b2680000000ull, 0x7e37be2022ull},
    {0x85acef8100000000ull, 0x4ee2d6d415bull}, {0x38c15b0a00000000ull, 0x314dc6448d93ull}, {0x378d8e6400000000ull, 0x1ed09bead87c0ull}, {0x2b878fe800000000ull, 0x13426172c74d82ull},
    {0xb34b9f1000000000ull, 0xc097ce7bc90715ull}, {0x00f436a000000000ull, 0x785ee10d5da46d9ull}, {0x098a224000000000ull, 0x4b3b4ca85a86c47aull}};
__device__ __forceinline__ i128 pow10_i128(int e) { return (i128)(((u128)kPow10Tab[e][1] << 64) | (u128)kPow10Tab[e][0]); }

// checked arithmetic on i128 (ArrowNativeTypeOp::{add,sub,mul,div,mod}_checked): true = overflow
__device__ __forceinline__ bool add_ovf128(i128 a, i128 b, i128* r) { *r = (i128)((u128)a + (u128)b); return ((a ^ *r) & (b ^ *r)) < 0; }
__device__ __forceinline__ bool sub_ovf128(i128 a, i128 b, i128* r) { *r = (i128)((u128)a - (u128)b); return ((a ^ b) & (a ^ *r)) < 0; }
__device__ __forceinline__ bool mul_ovf128(i128 a, i128 b, i128* r) {
  const bool neg = (a < 0) != (b < 0);
  const u128 ua = a < 0 ? (u128)0 - (u128)a : (u128)a, ub = b < 0 ? (u128)0 - (u128)b : (u128)b;
  const uint64_t a0 = (uint64_t)ua, a1 = (uint64_t)(ua >> 64), b0 = (uint64_t)ub, b1 = (uint64_t)(ub >> 64);
  *r = 0;
  if (a1 && b1) return true;
  const u128 cross = (u128)a1 * b0 + (u128)a0 * b1;   // at most one term is non-zero
  if (cross >> 64) return true;
  const u128 lo = (u128)a0 * b0;
  const u128 mag = lo + (cross << 64);
  if (mag < lo) return true;
  const u128 lim = (u128)1 << 127;
  if (neg ? mag > lim : mag >= lim) return true;
  *r = neg ? (i128)((u128)0 - mag) : (i128)mag;
  return false;
}
__device__ __forceinline__ bool is_min128(i128 a) { return (u128)a == ((u128)1 << 127); }

// ---- 16-byte {lo, hi} pairs in memory: Decimal128 accumulators (and 128-bit keys / record heads), always accessed as ONE 128-bit unit ----
struct alignas(16) Rec128 { unsigned long long lo, hi; };
// 128-bit compare-and-swap on a global address; GENERIC: on a generic one (shared memory as well)
template <bool GENERIC = false>
__device__ __forceinline__ Rec128 cas128(void* addr, Rec128 cmp, Rec128 val) {
  Rec128 old;
  if constexpr (GENERIC)
    asm volatile("{\n\t.reg .b128 c, v, o;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 v, {%4, %5};\n\tatom.cas.b128 o, [%6], c, v;\n\tmov.b128 {%0, %1}, o;\n\t}"
                 : "=l"(old.lo), "=l"(old.hi) : "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi), "l"(addr) : "memory");
  else
    asm volatile("{\n\t.reg .b128 c, v, o;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 v, {%4, %5};\n\tatom.global.cas.b128 o, [%6], c, v;\n\tmov.b128 {%0, %1}, o;\n\t}"
                 : "=l"(old.lo), "=l"(old.hi) : "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi), "l"(addr) : "memory");
  return old;
}
// a {lo, hi} pair in global memory in one 128-bit access: never a mix of two CAS results
__device__ __forceinline__ Rec128 ld_pair(const void* addr) {
  Rec128 v;
  asm volatile("{\n\t.reg .b128 t;\n\tld.relaxed.gpu.global.b128 t, [%2];\n\tmov.b128 {%0, %1}, t;\n\t}" : "=l"(v.lo), "=l"(v.hi) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ bool lt_i128(Rec128 a, Rec128 b) { return (long long)a.hi < (long long)b.hi || (a.hi == b.hi && a.lo < b.lo); }
// Decimal128 MIN / MAX of v into the 16-byte aligned pair at w (global memory), signed i128 order.  Once a group has a few rows most
// values are not better than the pair: one load, no atomic.  The load is one 128-bit access and the pair only ever improves, so "not
// better" than it is final (a torn read could show a value below anything ever stored and skip a needed update).
__device__ __forceinline__ void minmax_i128(void* w, Rec128 v, bool is_min) {
  Rec128 cur = ld_pair(w);
  while (is_min ? lt_i128(v, cur) : lt_i128(cur, v)) {
    const Rec128 prev = cas128(w, cur, v);
    if (prev.lo == cur.lo && prev.hi == cur.hi) break;
    cur = prev;
  }
}

__device__ __forceinline__ i128 load_dec(const void* col, int64_t row) {
  const unsigned long long* p = (const unsigned long long*)col + 2 * row;   // 8-byte aligned is all Arrow promises for a sliced buffer
  return (i128)(((u128)p[1] << 64) | (u128)p[0]);
}

// Decimal128::validate_decimal_precision: |v| <= 10^p - 1
__device__ __forceinline__ bool dec_fits(i128 v, int precision) {
  const i128 lim = pow10_i128(precision);
  return v < lim && v > -lim;
}

// AVG over Decimal128(p, s) into Decimal128(tp, ts) (DecimalAverager::avg): sum.mul_checked(10^mul) / count, mul = ts - s, truncated
// toward zero and validated against tp.  count > 0.  Returns false on either overflow ("Arithmetic Overflow in AvgAccumulator").
__device__ __forceinline__ bool dec_avg(i128 sum, unsigned long long count, int mul, int tp, i128* q) {
  i128 m;
  *q = 0;
  if (mul_ovf128(sum, pow10_i128(mul), &m)) return false;
  const i128 r = m / (i128)count;
  if (!dec_fits(r, tp)) return false;
  *q = r;
  return true;
}

// i128 -> f64 (`as f64`, round to nearest even)
__device__ __forceinline__ double i128_to_f64(i128 v) {
  const bool neg = v < 0;
  u128 m = neg ? (u128)0 - (u128)v : (u128)v;
  double d;
  if ((m >> 64) == 0) d = (double)(uint64_t)m;
  else {
    // normalise to 64 significant bits + sticky so that the single hardware rounding below is the only one
    const int lz = __clzll((long long)(uint64_t)(m >> 64));
    const int sh = 64 - lz;                                  // bits to drop
    uint64_t top = (uint64_t)(m >> sh);
    const bool sticky = (m & (((u128)1 << sh) - 1)) != 0;
    if (sticky) top |= 1ull;                                 // top has 64 bits: bit 0 lies far below the 53-bit cut, a safe sticky
    d = ldexp((double)top, sh);
  }
  return neg ? -d : d;
}

__device__ __forceinline__ void eval_binary_dec(const ENode& nd, i128 a, bool av, i128 b, bool bv, i128* r, bool* rv, int* err) {
  const int op = nd.op;
  if (op <= DFGPU_OP_GTEQ || op == DFGPU_OP_IS_DISTINCT_FROM || op == DFGPU_OP_IS_NOT_DISTINCT_FROM) {
    const int cmp = a < b ? -1 : (a > b ? 1 : 0);
    if (op == DFGPU_OP_IS_DISTINCT_FROM || op == DFGPU_OP_IS_NOT_DISTINCT_FROM) {
      const bool distinct = (av != bv) || (av && bv && cmp != 0);
      *r = (op == DFGPU_OP_IS_DISTINCT_FROM) ? distinct : !distinct;
      *rv = true;
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
    *r = res; *rv = av && bv;
    return;
  }
  *rv = av && bv;
  *r = 0;
  if (!*rv) return;
  const int le = (int)(nd.voff & 0xff), re = (int)((nd.voff >> 8) & 0xff);
  i128 x = a, y = b, z = 0;
  bool ovf = false;
  if (le) ovf |= mul_ovf128(a, pow10_i128(le), &x);
  if (re) ovf |= mul_ovf128(b, pow10_i128(re), &y);
  if (!ovf) {
    switch (op) {
      case DFGPU_OP_PLUS: ovf = add_ovf128(x, y, &z); break;
      case DFGPU_OP_MINUS: ovf = sub_ovf128(x, y, &z); break;
      case DFGPU_OP_MULTIPLY: ovf = mul_ovf128(x, y, &z); break;
      case DFGPU_OP_DIVIDE:
      case DFGPU_OP_MODULO:
        if (y == 0) { *err |= ERR_DIV_ZERO; return; }
        if (y == -1 && is_min128(x)) { ovf = true; break; }
        z = op == DFGPU_OP_DIVIDE ? x / y : x % y;
        break;
      default: break;
    }
  }
  if (ovf) { *err |= ERR_OVERFLOW; z = 0; }
  *r = z;
}

// CastExpr touching a decimal on either side (arrow-cast cast/decimal.rs; CastOptions { safe: false }: failures are errors)
__device__ __forceinline__ i128 cast_value_dec(const ENode& nd, i128 v, bool valid, int* err) {
  const int from = nd.in_type, to = nd.out_type;
  if (!valid) return 0;
  const int e = (int)(nd.voff & 0xff);
  if (type_is_decimal(to)) {
    i128 x = 0;
    if (type_is_decimal(from)) {
      const int s1 = dec_scale(from), s2 = dec_scale(to);
      if (s2 >= s1) { if (mul_ovf128(v, pow10_i128(e), &x)) { *err |= ERR_CAST; return 0; } }
      else {
        // convert_to_smaller_scale_decimal: divide, round half away from zero
        const i128 div = pow10_i128(e), half = div / 2;
        const i128 d = v / div, rem = v % div;
        x = v >= 0 ? (rem >= half ? d + 1 : d) : (rem <= -half ? d - 1 : d);
      }
    } else if (cls_of(from) == C_F64) {
      // cast_floating_point_to_decimal128: (v * 10^scale).round() -> i128
      const double f = __longlong_as_double((long long)(uint64_t)v);
      const double m = round(f * i128_to_f64(pow10_i128(e)));
      if (!isfinite(m) || fabs(m) >= 1.7014118346046923e38) { *err |= ERR_CAST; return 0; }
      const bool neg = m < 0;
      const double am = fabs(m);
      u128 mag;
      if (am < 18446744073709551616.0) mag = (u128)(uint64_t)am;
      else { const double hi = floor(ldexp(am, -64)); mag = ((u128)(uint64_t)hi << 64) | (u128)(uint64_t)(am - ldexp(hi, 64)); }
      x = neg ? (i128)((u128)0 - mag) : (i128)mag;
    } else {
      // cast_integer_to_decimal: v * 10^scale, checked
      const i128 iv = cls_of(from) == C_U64 || cls_of(from) == C_BOOL ? (i128)(u128)(uint64_t)v : (i128)(long long)(uint64_t)v;
      if (mul_ovf128(iv, pow10_i128(e), &x)) { *err |= ERR_CAST; return 0; }
    }
    if (!dec_fits(x, dec_precision(to))) { *err |= ERR_CAST; return 0; }
    return x;
  }
  // decimal -> float64 / float32 / integer
  if (cls_of(to) == C_F64) {
    double d = i128_to_f64(v) / i128_to_f64(pow10_i128(e));
    if (to == DFGPU_FLOAT32) d = (double)(float)d;
    return (i128)(u128)(uint64_t)__double_as_longlong(d);
  }
  const i128 q = v / pow10_i128(e);   // cast_decimal_to_integer: truncating division by 10^scale, then a checked narrowing
  const int w = type_width(to) * 8;
  bool fits;
  if (cls_of(to) == C_U64) fits = q >= 0 && (w == 64 ? q <= (i128)(u128)~0ull : q < ((i128)1 << w));
  else fits = q >= -((i128)1 << (w - 1)) && q < ((i128)1 << (w - 1));
  if (!fits) { *err |= ERR_CAST; return 0; }
  return (i128)(u128)(uint64_t)wrap_to_type((uint64_t)q, to);
}

// one row of a program that touches decimals: value (128 bits) + validity; XN: nullable payload fields (expr_dev.cuh)
template <bool XN = false>
__device__ __forceinline__ i128 eval_nodes_dec(const ENode* __restrict__ nodes, int n_nodes, int64_t row, bool* ok_out, int* err, const uint64_t* ext = nullptr) {
  i128 sv[kMaxStack];
  bool sk[kMaxStack];
  int sp = 0;
#pragma unroll 1
  for (int i = 0; i < n_nodes; ++i) {
    const ENode& nd = nodes[i];
    int e = 0;
    switch (nd.kind) {
      case DFGPU_EXPR_COLUMN:
        sk[sp] = !(nd.valid && !bit_get(nd.valid, nd.voff + row));
        sv[sp] = type_is_decimal(nd.out_type) ? load_dec(nd.col, row) : (i128)(u128)load_col_value(nd, row);
        ++sp;
        break;
      case DFGPU_EXPR_LITERAL:
        sk[sp] = !nd.lit_null;
        sv[sp] = type_is_decimal(nd.out_type) ? (i128)(((u128)(uint64_t)nd.voff << 64) | (u128)nd.lit) : (i128)(u128)nd.lit;
        ++sp;
        break;
      case kExprExt: {
        uint64_t v = ext[nd.voff] >> (int)nd.lit;
        const int w = type_width(nd.out_type);
        if (w < 8) { v &= (1ull << (8 * w)) - 1ull; if (type_is_signed_int(nd.out_type)) v = (uint64_t)(((int64_t)(v << (64 - 8 * w))) >> (64 - 8 * w)); }
        if (nd.out_type == DFGPU_FLOAT32) { float f = __uint_as_float((uint32_t)v); v = (uint64_t)__double_as_longlong((double)f); }
        sk[sp] = XN ? ((ext[kExtValid] >> nd.voff) & 1ull) != 0 : true; sv[sp] = (i128)(u128)v; ++sp;
        break;
      }
      case DFGPU_EXPR_BINARY: {
        i128 r; bool ok;
        if (type_is_decimal(nd.in_type)) eval_binary_dec(nd, sv[sp - 2], sk[sp - 2], sv[sp - 1], sk[sp - 1], &r, &ok, &e);
        else { uint64_t r64; eval_binary(nd, (uint64_t)sv[sp - 2], sk[sp - 2], (uint64_t)sv[sp - 1], sk[sp - 1], &r64, &ok, &e); r = (i128)(u128)r64; }
        sp -= 1; sv[sp - 1] = r; sk[sp - 1] = ok;
        break;
      }
      case DFGPU_EXPR_NOT: sv[sp - 1] = sv[sp - 1] ? 0 : 1; break;
      case DFGPU_EXPR_IS_NULL: sv[sp - 1] = sk[sp - 1] ? 0 : 1; sk[sp - 1] = true; break;
      case DFGPU_EXPR_IS_NOT_NULL: sv[sp - 1] = sk[sp - 1] ? 1 : 0; sk[sp - 1] = true; break;
      case DFGPU_EXPR_NEGATIVE:
        if (type_is_decimal(nd.out_type)) sv[sp - 1] = (i128)((u128)0 - (u128)sv[sp - 1]);   // neg_wrapping
        else if (cls_of(nd.out_type) == C_F64) sv[sp - 1] = (i128)(u128)((uint64_t)sv[sp - 1] ^ 0x8000000000000000ull);
        else sv[sp - 1] = (i128)(u128)wrap_to_type(0ull - (uint64_t)sv[sp - 1], nd.out_type);
        break;
      case DFGPU_EXPR_CAST:
        if (type_is_decimal(nd.in_type) || type_is_decimal(nd.out_type)) sv[sp - 1] = cast_value_dec(nd, sv[sp - 1], sk[sp - 1], &e);
        else sv[sp - 1] = (i128)(u128)cast_value((uint64_t)sv[sp - 1], nd.in_type, nd.out_type, sk[sp - 1], &e);
        break;
    }
    if (e) {
      // an error inside the RHS of a short-circuited AND / OR counts only on the rows the reference evaluates (expr_dev.cuh)
      bool counts = true;
      const int top = sp;   // the guard slots lie below the operands of this node
      for (int g = 0; g < kMaxStack; ++g) {
        if (g >= top) break;
        if ((nd.g_and >> g) & 1) counts = counts && sk[g] && sv[g] != 0;
        if ((nd.g_or >> g) & 1) counts = counts && sk[g] && sv[g] == 0;
      }
      if (counts) *err |= e;
    }
  }
  *ok_out = sk[0];
  return sv[0];
}

}  // namespace dfgpu
