// filter.cu — PhysicalExpr::evaluate + GpuFilterExec.
//
// Reference path being replaced (SURVEY.md §8a rows a1–a7):
//   FilterExecStream::poll_next       physical-plan/src/filter.rs:1364-1445
//   filter_and_project                physical-plan/src/filter.rs:1339-1361
//   BinaryExpr::evaluate              physical-expr/src/expressions/binary.rs:536-676
//   apply / apply_cmp (+ float zero normalisation)   physical-expr-common/src/datum.rs:36-105
//   and_kleene / or_kleene            physical-expr/src/expressions/binary.rs:1093-1116
//   filter_record_batch (arrow-select 59.2.0; null mask entries count as false)  filter.rs:1412
//   LimitedBatchCoalescer             physical-plan/src/coalesce/mod.rs:27-147
//
// GPU design: the reference walks the expression tree once per node per batch and allocates an
// Arrow array for every intermediate.  Here the whole tree is a post-order program evaluated per
// row in registers by ONE kernel (no intermediate arrays in HBM); a warp owns 32 consecutive rows
// so Boolean results and validity leave as one ballot word per warp (Arrow's LSB bitmaps for free).
// Selection = that bitmap -> popcount/scan -> index list -> one gather per projected column.
#include "batch.cuh"
#include "scan.cuh"
#include "expr.cuh"
#include "expr_dev.cuh"
#include "expr_dec.cuh"

namespace dfgpu {


// One kernel evaluates the whole expression.  Outputs: typed values (or bit-packed booleans),
// validity words, and — for predicates — the selection words (valid AND true).
__global__ void __launch_bounds__(256) expr_eval_kernel(EProgram p, int64_t n, void* __restrict__ out_values, uint32_t* __restrict__ out_boolwords,
                                                     uint32_t* __restrict__ out_valid, uint32_t* __restrict__ out_select, int* __restrict__ err_flag) {
  const int64_t nw = (n + 31) / 32;
  const int lane = threadIdx.x & 31;
  const int root_type = p.node[p.n - 1].out_type;
  int err = 0;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t row = wi * 32 + lane;
    uint64_t rv = 0;
    bool rok = false;
    if (row < n) {
      rv = eval_row(p, row, &rok, &err);
      if (!rok) rv = 0;
      if (out_values) {
        switch (root_type) {
          case DFGPU_INT8: case DFGPU_UINT8: ((uint8_t*)out_values)[row] = (uint8_t)rv; break;
          case DFGPU_INT16: case DFGPU_UINT16: ((uint16_t*)out_values)[row] = (uint16_t)rv; break;
          case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_DATE32: ((uint32_t*)out_values)[row] = (uint32_t)rv; break;
          case DFGPU_FLOAT32: ((float*)out_values)[row] = (float)__longlong_as_double((long long)rv); break;
          default: ((uint64_t*)out_values)[row] = rv; break;
        }
      }
    }
    uint32_t vw = __ballot_sync(0xffffffffu, rok);
    uint32_t bw = __ballot_sync(0xffffffffu, rok && (rv & 1));
    if (lane == 0) {
      if (out_valid) out_valid[wi] = vw;
      if (out_boolwords) out_boolwords[wi] = bw;  // NULL slots hold 0
      if (out_select) out_select[wi] = bw;
    }
  }
  if (err) atomicOr(err_flag, err);
}

// the same for programs that touch Decimal128 values: 128-bit evaluation stack (expr_dec.cuh)
__global__ void __launch_bounds__(256) expr_eval_dec_kernel(EProgram p, int64_t n, void* __restrict__ out_values, uint32_t* __restrict__ out_boolwords,
                                                         uint32_t* __restrict__ out_valid, uint32_t* __restrict__ out_select, int* __restrict__ err_flag) {
  const int64_t nw = (n + 31) / 32;
  const int lane = threadIdx.x & 31;
  const int root_type = p.node[p.n - 1].out_type;
  int err = 0;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t row = wi * 32 + lane;
    i128 rv = 0;
    bool rok = false;
    if (row < n) {
      rv = eval_nodes_dec(p.node, p.n, row, &rok, &err);
      if (!rok) rv = 0;
      if (out_values) {
        const uint64_t lo = (uint64_t)rv;
        if (type_is_decimal(root_type)) { ((unsigned long long*)out_values)[2 * row] = lo; ((unsigned long long*)out_values)[2 * row + 1] = (uint64_t)((u128)rv >> 64); }
        else switch (root_type) {
          case DFGPU_INT8: case DFGPU_UINT8: ((uint8_t*)out_values)[row] = (uint8_t)lo; break;
          case DFGPU_INT16: case DFGPU_UINT16: ((uint16_t*)out_values)[row] = (uint16_t)lo; break;
          case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_DATE32: ((uint32_t*)out_values)[row] = (uint32_t)lo; break;
          case DFGPU_FLOAT32: ((float*)out_values)[row] = (float)__longlong_as_double((long long)lo); break;
          default: ((uint64_t*)out_values)[row] = lo; break;
        }
      }
    }
    uint32_t vw = __ballot_sync(0xffffffffu, rok);
    uint32_t bw = __ballot_sync(0xffffffffu, rok && ((uint64_t)rv & 1));
    if (lane == 0) {
      if (out_valid) out_valid[wi] = vw;
      if (out_boolwords) out_boolwords[wi] = bw;
      if (out_select) out_select[wi] = bw;
    }
  }
  if (err) atomicOr(err_flag, err);
}

// ---- fast path: `column <cmp> literal` on an 8-byte integer column without NULLs ------------
// 128-bit vectorised loads, two rows per load, 8 loads in flight per thread; each warp emits whole
// 32-bit selection words.  (C1: `x:int64 > c`.)
__device__ __forceinline__ uint32_t spread16(uint32_t x) {  // bit i -> bit 2i
  x &= 0xFFFFu;
  x = (x | (x << 8)) & 0x00FF00FFu;
  x = (x | (x << 4)) & 0x0F0F0F0Fu;
  x = (x | (x << 2)) & 0x33333333u;
  x = (x | (x << 1)) & 0x55555555u;
  return x;
}
template <int OP>
__device__ __forceinline__ bool cmp_i64(int64_t a, int64_t lit) {
  if (OP == DFGPU_OP_EQ) return a == lit;
  if (OP == DFGPU_OP_NEQ) return a != lit;
  if (OP == DFGPU_OP_LT) return a < lit;
  if (OP == DFGPU_OP_LTEQ) return a <= lit;
  if (OP == DFGPU_OP_GT) return a > lit;
  return a >= lit;
}
// A warp owns 512 consecutive rows per iteration: 8 coalesced 512-byte wavefronts of int4 loads in
// flight, two ballots per wavefront, bit-interleaved into two selection words.
template <int OP>
__global__ void __launch_bounds__(256) cmp_i64_scalar_kernel(const int64_t* __restrict__ col, int64_t n, int64_t lit, uint32_t* __restrict__ select_words) {
  constexpr int K = 8;
  const int lane = threadIdx.x & 31;
  const int64_t nchunks = n / (64 * K);
  const int64_t warp_id = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp_id; c < nchunks; c += nwarps) {
    const int4* p = reinterpret_cast<const int4*>(col + c * 64 * K);
    int4 v[K];
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = ld_stream_16(p + k * 32 + lane);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      int64_t a = (int64_t)(((uint64_t)(uint32_t)v[k].y << 32) | (uint32_t)v[k].x);
      int64_t b = (int64_t)(((uint64_t)(uint32_t)v[k].w << 32) | (uint32_t)v[k].z);
      uint32_t ba = __ballot_sync(0xffffffffu, cmp_i64<OP>(a, lit));  // even rows
      uint32_t bb = __ballot_sync(0xffffffffu, cmp_i64<OP>(b, lit));  // odd rows
      if (lane < 2) {
        uint32_t ha = lane ? (ba >> 16) : ba, hb = lane ? (bb >> 16) : bb;
        select_words[c * 2 * K + k * 2 + lane] = spread16(ha) | (spread16(hb) << 1);
      }
    }
  }
  // tail (< 512 rows): one word per thread of the first block
  if (blockIdx.x == 0) {
    const int64_t tail0 = nchunks * 64 * K;
    const int64_t nw = (n + 31) / 32;
    for (int64_t w = tail0 / 32 + threadIdx.x; w < nw; w += blockDim.x) {
      uint32_t word = 0;
      for (int k = 0; k < 32 && w * 32 + k < n; ++k) word |= (uint32_t)cmp_i64<OP>(col[w * 32 + k], lit) << k;
      select_words[w] = word;
    }
  }
}

// ------------------------------------------------------------------------------------------
// fused FilterExec: predicate -> ordered compaction -> projected columns, ONE pass over the batch
// (tile = 256 threads x 4 consecutive rows; selected rows ranked by a block scan, tile offsets by decoupled
// look-back, every projected column written with coalesced stores).  No selection bitmap, index list or
// per-column gather kernels touch HBM.
// ------------------------------------------------------------------------------------------
constexpr int kFiltThreads = 256;
constexpr int kFiltItems = 4;
constexpr int kFiltTile = kFiltThreads * kFiltItems;
constexpr int kMaxFiltCols = 16;
struct FilterCols { int n; const void* src[kMaxFiltCols]; void* dst[kMaxFiltCols]; int width[kMaxFiltCols]; };

template <int FAST>
__global__ void __launch_bounds__(kFiltThreads) filter_fused_kernel(const EProgram* __restrict__ prog, const int64_t* __restrict__ fast_col, int fast_op, int64_t fast_lit,
                                                                  int64_t n, FilterCols fc, unsigned long long* __restrict__ tile_desc,
                                                                  unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ totals, int* __restrict__ err_flag) {
  __shared__ uint32_t s_p[kFiltTile];
  __shared__ unsigned int s_tile;
  __shared__ unsigned long long s_base;
  if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);
  __syncthreads();
  const int64_t tile = s_tile;
  const int64_t row0 = tile * kFiltTile + (int64_t)threadIdx.x * kFiltItems;
  bool keep[kFiltItems];
  uint32_t m = 0;
  int err = 0;
  if (FAST == 1) {
    int64_t v[kFiltItems];
#pragma unroll
    for (int k = 0; k < kFiltItems; ++k) v[k] = row0 + k < n ? fast_col[row0 + k] : 0;
#pragma unroll
    for (int k = 0; k < kFiltItems; ++k) {
      bool r;
      switch (fast_op) {
        case DFGPU_OP_EQ: r = v[k] == fast_lit; break;
        case DFGPU_OP_NEQ: r = v[k] != fast_lit; break;
        case DFGPU_OP_LT: r = v[k] < fast_lit; break;
        case DFGPU_OP_LTEQ: r = v[k] <= fast_lit; break;
        case DFGPU_OP_GT: r = v[k] > fast_lit; break;
        default: r = v[k] >= fast_lit; break;
      }
      keep[k] = r && row0 + k < n;
      m += keep[k] ? 1u : 0u;
    }
  } else {
#pragma unroll 1
    for (int k = 0; k < kFiltItems; ++k) {
      keep[k] = false;
      if (row0 + k < n) {
        bool ok;
        uint64_t val;
        if (FAST == 2) val = (uint64_t)eval_nodes_dec(prog->node, prog->n, row0 + k, &ok, &err);   // the predicate touches Decimal128 values
        else val = eval_row(*prog, row0 + k, &ok, &err);
        keep[k] = ok && (val & 1);   // NULL predicate rows are dropped (filter_record_batch)
      }
      m += keep[k] ? 1u : 0u;
    }
  }
  uint32_t tot;
  uint32_t ex = block_exclusive_scan<kFiltThreads, uint32_t>(m, &tot);
#pragma unroll
  for (int k = 0; k < kFiltItems; ++k) if (keep[k]) s_p[ex++] = (uint32_t)(threadIdx.x * kFiltItems + k);
  if (threadIdx.x < 32) {
    unsigned long long exclusive = tile_lookback(tile, tot, tile_desc);
    if (threadIdx.x == 0) {
      s_base = exclusive;
      if ((tile + 1) * (int64_t)kFiltTile >= n) totals[0] = exclusive + tot;
    }
  }
  __syncthreads();
  const unsigned long long base = s_base;
  const int64_t prow0 = tile * kFiltTile;
  for (int c = 0; c < fc.n; ++c) {
    switch (fc.width[c]) {
      case 8: { const uint64_t* src = (const uint64_t*)fc.src[c]; uint64_t* dst = (uint64_t*)fc.dst[c] + base;
                for (uint32_t j = threadIdx.x; j < tot; j += kFiltThreads) dst[j] = src[prow0 + s_p[j]]; break; }
      case 4: { const uint32_t* src = (const uint32_t*)fc.src[c]; uint32_t* dst = (uint32_t*)fc.dst[c] + base;
                for (uint32_t j = threadIdx.x; j < tot; j += kFiltThreads) dst[j] = src[prow0 + s_p[j]]; break; }
      case 2: { const uint16_t* src = (const uint16_t*)fc.src[c]; uint16_t* dst = (uint16_t*)fc.dst[c] + base;
                for (uint32_t j = threadIdx.x; j < tot; j += kFiltThreads) dst[j] = src[prow0 + s_p[j]]; break; }
      case 1: { const uint8_t* src = (const uint8_t*)fc.src[c]; uint8_t* dst = (uint8_t*)fc.dst[c] + base;
                for (uint32_t j = threadIdx.x; j < tot; j += kFiltThreads) dst[j] = src[prow0 + s_p[j]]; break; }
      default: { const uint4* src = (const uint4*)fc.src[c]; uint4* dst = (uint4*)fc.dst[c] + base;
                for (uint32_t j = threadIdx.x; j < tot; j += kFiltThreads) dst[j] = src[prow0 + s_p[j]]; break; }
    }
  }
  if (err) atomicOr(err_flag, err);
}

// ------------------------------------------------------------------------------------------
// host side: type inference + program binding
// ------------------------------------------------------------------------------------------
static bool is_cmp_op(int op) { return (op >= DFGPU_OP_EQ && op <= DFGPU_OP_GTEQ) || op == DFGPU_OP_IS_DISTINCT_FROM || op == DFGPU_OP_IS_NOT_DISTINCT_FROM; }
static bool is_arith_op(int op) { return op >= DFGPU_OP_PLUS && op <= DFGPU_OP_MODULO; }
static bool is_bit_op(int op) { return op >= DFGPU_OP_BITAND && op <= DFGPU_OP_SHIFT_RIGHT; }
static bool expr_type_ok(int t) {
  if (type_is_decimal(t)) return dec_precision(t) >= 1 && dec_precision(t) <= 38 && dec_scale(t) >= 0 && dec_scale(t) <= dec_precision(t);
  return t == DFGPU_BOOL || type_is_int(t) || type_is_float(t);
}

ExprPlan plan_expr(const int32_t* schema_types, int n_cols, const dfgpu_expr_node* nodes, int n_nodes, int max_nodes) {
  DF_CHECK(n_nodes >= 1 && n_nodes <= max_nodes, DFGPU_ERR_UNSUPPORTED, max_nodes == kMaxNodes ? "expression: 1..48 nodes supported" : "expression: too many nodes");
  ExprPlan p;
  p.nodes.assign(nodes, nodes + n_nodes);
  p.in_type.assign(n_nodes, 0);
  p.out_type.assign(n_nodes, 0);
  p.aux.assign(n_nodes, 0);
  std::vector<int> stack;       // node index of each stack entry
  for (int i = 0; i < n_nodes; ++i) {
    const dfgpu_expr_node& nd = nodes[i];
    switch (nd.kind) {
      case DFGPU_EXPR_COLUMN:
        DF_CHECK(nd.a >= 0 && nd.a < n_cols, DFGPU_ERR_INVALID, "expression: column index out of range");
        DF_CHECK(expr_type_ok(schema_types[nd.a]), DFGPU_ERR_UNSUPPORTED, "expression: column type not supported on the GPU");
        p.out_type[i] = schema_types[nd.a];
        stack.push_back(i);
        break;
      case DFGPU_EXPR_LITERAL:
        DF_CHECK(expr_type_ok(nd.type), DFGPU_ERR_UNSUPPORTED, "expression: literal type not supported on the GPU");
        p.out_type[i] = nd.type;
        stack.push_back(i);
        break;
      case DFGPU_EXPR_BINARY: {
        DF_CHECK(stack.size() >= 2, DFGPU_ERR_INVALID, "expression: malformed program (binary needs two operands)");
        int r = stack.back(); stack.pop_back();
        int l = stack.back(); stack.pop_back();
        int lt = p.out_type[l], rt = p.out_type[r];
        if (type_is_decimal(lt) || type_is_decimal(rt)) {
          // arrow-arith decimal_op (arithmetic.rs): result precision / scale and the rescale multipliers per operator
          DF_CHECK(type_is_decimal(lt) && type_is_decimal(rt), DFGPU_ERR_INVALID, "expression: a Decimal128 operand needs a Decimal128 partner (the planner's coercion casts the other side)");
          const int p1 = dec_precision(lt), s1 = dec_scale(lt), p2 = dec_precision(rt), s2 = dec_scale(rt);
          p.in_type[i] = lt;
          p.has_decimal = true;
          if (is_cmp_op(nd.a)) {
            DF_CHECK(lt == rt, DFGPU_ERR_INVALID, "expression: Decimal128 comparison needs equal precision and scale on both sides");
            p.out_type[i] = DFGPU_BOOL;
          } else if (is_arith_op(nd.a)) {
            int rp, rs, le = 0, re = 0;
            switch (nd.a) {
              case DFGPU_OP_PLUS: case DFGPU_OP_MINUS:
                rs = std::max(s1, s2); rp = std::min(38, rs + std::max(p1 - s1, p2 - s2) + 1); le = rs - s1; re = rs - s2; break;
              case DFGPU_OP_MULTIPLY:
                rp = std::min(38, p1 + p2 + 1); rs = s1 + s2;
                DF_CHECK(rs <= 38, DFGPU_ERR_INVALID, "expression: Decimal128 multiply: output scale exceeds 38");
                break;
              case DFGPU_OP_DIVIDE: {
                rs = std::min(38, s1 + 4);                 // "a fixed scale increment of 4" (postgres / MySQL)
                const int mul_pow = rs - s1 + s2;
                rp = std::min(38, mul_pow + p1);
                if (mul_pow >= 0) le = mul_pow; else re = -mul_pow;
                break;
              }
              default:  // MODULO
                rs = std::max(s1, s2); rp = std::min(38, rs + std::min(p1 - s1, p2 - s2)); le = rs - s1; re = rs - s2; break;
            }
            DF_CHECK(le <= 38 && re <= 38, DFGPU_ERR_INVALID, "expression: Decimal128 rescale exceeds 10^38");
            p.out_type[i] = dec_type(rp, rs);
            p.aux[i] = (int64_t)le | ((int64_t)re << 8);
          } else throw Error(DFGPU_ERR_UNSUPPORTED, "expression: operator not supported on Decimal128");
          stack.push_back(i);
          break;
        }
        // the planner coerces both sides to one type (expr-common type_coercion); we insist on it
        DF_CHECK(lt == rt || (cls_of(lt) == cls_of(rt) && type_width(lt) == type_width(rt)), DFGPU_ERR_INVALID,
                 "expression: binary operands must already be coerced to a common type");
        p.in_type[i] = lt;
        if (nd.a == DFGPU_OP_AND || nd.a == DFGPU_OP_OR) {
          DF_CHECK(lt == DFGPU_BOOL, DFGPU_ERR_INVALID, "expression: AND/OR need Boolean operands");
          p.out_type[i] = DFGPU_BOOL;
        } else if (is_cmp_op(nd.a)) p.out_type[i] = DFGPU_BOOL;
        else if (is_arith_op(nd.a)) {
          DF_CHECK(lt != DFGPU_BOOL, DFGPU_ERR_INVALID, "expression: arithmetic on Boolean");
          DF_CHECK(!(lt == DFGPU_DATE32 || lt == DFGPU_DATE64 || lt == DFGPU_TIMESTAMP), DFGPU_ERR_UNSUPPORTED, "expression: temporal arithmetic stays on the CPU operator");
          p.out_type[i] = lt;
        } else if (is_bit_op(nd.a)) {
          DF_CHECK(type_is_int(lt), DFGPU_ERR_INVALID, "expression: bitwise operators need integer operands");
          p.out_type[i] = lt;
        } else throw Error(DFGPU_ERR_UNSUPPORTED, "expression: operator not supported on the GPU");
        stack.push_back(i);
        break;
      }
      case DFGPU_EXPR_NOT:
        DF_CHECK(!stack.empty() && p.out_type[stack.back()] == DFGPU_BOOL, DFGPU_ERR_INVALID, "expression: NOT needs a Boolean operand");
        p.in_type[i] = DFGPU_BOOL; p.out_type[i] = DFGPU_BOOL; stack.back() = i;
        break;
      case DFGPU_EXPR_IS_NULL: case DFGPU_EXPR_IS_NOT_NULL:
        DF_CHECK(!stack.empty(), DFGPU_ERR_INVALID, "expression: malformed program");
        p.in_type[i] = p.out_type[stack.back()]; p.out_type[i] = DFGPU_BOOL; stack.back() = i;
        break;
      case DFGPU_EXPR_NEGATIVE:
        DF_CHECK(!stack.empty() && p.out_type[stack.back()] != DFGPU_BOOL, DFGPU_ERR_INVALID, "expression: negative needs a numeric operand");
        p.in_type[i] = p.out_type[stack.back()]; p.out_type[i] = p.in_type[i]; stack.back() = i;
        break;
      case DFGPU_EXPR_CAST:
        DF_CHECK(!stack.empty() && expr_type_ok(nd.type), DFGPU_ERR_UNSUPPORTED, "expression: cast target not supported");
        p.in_type[i] = p.out_type[stack.back()]; p.out_type[i] = nd.type; stack.back() = i;
        if (type_is_decimal(p.in_type[i]) || type_is_decimal(nd.type)) {
          const int from = p.in_type[i], to = nd.type;
          p.has_decimal = true;
          DF_CHECK(from != DFGPU_BOOL && to != DFGPU_BOOL, DFGPU_ERR_UNSUPPORTED, "expression: Boolean <-> Decimal128 cast is not supported");
          int e;
          if (type_is_decimal(from) && type_is_decimal(to)) e = std::abs(dec_scale(to) - dec_scale(from));
          else if (type_is_decimal(to)) e = dec_scale(to);
          else e = dec_scale(from);
          // float <-> decimal goes through 10^scale as an f64, exact up to 10^22 (beyond that the reference's powi rounding would have to be reproduced)
          if (type_is_float(from) || type_is_float(to)) DF_CHECK(e <= 22, DFGPU_ERR_UNSUPPORTED, "expression: float <-> Decimal128 cast with scale > 22 stays on the CPU operator");
          p.aux[i] = e;
        }
        break;
      default: throw Error(DFGPU_ERR_INVALID, "expression: unknown node kind");
    }
    DF_CHECK((int)stack.size() <= kMaxStack, DFGPU_ERR_UNSUPPORTED, "expression: too deep");
  }
  DF_CHECK(stack.size() == 1, DFGPU_ERR_INVALID, "expression: malformed program (stack must end with one value)");
  p.root_type = p.out_type[n_nodes - 1];
  for (int i = 0; i < n_nodes; ++i) if (type_is_decimal(p.out_type[i]) || type_is_decimal(p.in_type[i])) p.has_decimal = true;
  // ---- short-circuit guards: AND / OR nodes whose RHS can raise an error ----
  {
    std::vector<int> start(n_nodes), depth_before(n_nodes);
    int sp = 0;
    for (int i = 0; i < n_nodes; ++i) {
      depth_before[i] = sp;
      const int k = nodes[i].kind;
      if (k == DFGPU_EXPR_COLUMN || k == DFGPU_EXPR_LITERAL) { start[i] = i; sp++; }
      else if (k == DFGPU_EXPR_BINARY) { const int rhs_start = start[i - 1]; start[i] = start[rhs_start - 1]; sp--; }
      else start[i] = start[i - 1];
    }
    for (int i = 0; i < n_nodes; ++i) {
      if (nodes[i].kind != DFGPU_EXPR_BINARY || (nodes[i].a != DFGPU_OP_AND && nodes[i].a != DFGPU_OP_OR)) continue;
      const int rhs_start = start[i - 1], lhs_start = start[rhs_start - 1];
      bool can_error = false;
      for (int j = rhs_start; j < i; ++j) {
        if (nodes[j].kind == DFGPU_EXPR_CAST) can_error = true;
        if (nodes[j].kind == DFGPU_EXPR_BINARY && (nodes[j].a == DFGPU_OP_DIVIDE || nodes[j].a == DFGPU_OP_MODULO) && !type_is_float(p.in_type[j])) can_error = true;
        if (nodes[j].kind == DFGPU_EXPR_BINARY && is_arith_op(nodes[j].a) && type_is_decimal(p.in_type[j])) can_error = true;   // checked 128-bit arithmetic
      }
      if (!can_error) continue;
      ExprGuard g;
      g.op_idx = i; g.lhs_start = lhs_start; g.rhs_start = rhs_start; g.slot = depth_before[lhs_start]; g.is_and = nodes[i].a == DFGPU_OP_AND;
      if (g.slot < 16) p.guards.push_back(g);
    }
  }
  return p;
}

// check_short_circuit (binary.rs:1182-1290) per batch: the RHS of AND is skipped when the LHS has no NULLs and is all false, and evaluated
// only on the LHS-true rows when at most 20 % of them are true (PRE_SELECTION_THRESHOLD); OR symmetrically; a scalar LHS always
// short-circuits.  In those cases an error raised inside the RHS counts only on the rows the reference evaluates.
std::vector<std::pair<uint16_t, uint16_t>> resolve_guards(dfgpu_ctx* ctx, const ExprPlan& plan, const std::vector<DCol>& cols, int64_t n) {
  std::vector<std::pair<uint16_t, uint16_t>> masks(plan.nodes.size(), {0, 0});
  if (plan.guards.empty() || n <= 0) return masks;
  std::vector<int32_t> types;
  for (auto& c : cols) types.push_back(c.type);
  for (const ExprGuard& g : plan.guards) {
    bool active = false;
    const int lhs_n = g.rhs_start - g.lhs_start;
    if (lhs_n == 1 && plan.nodes[g.lhs_start].kind == DFGPU_EXPR_LITERAL) active = !plan.nodes[g.lhs_start].is_null;   // scalar LHS: ReturnLeft / ReturnRight
    else {
      bool evaluable = true;
      for (int j = g.lhs_start; j < g.rhs_start; ++j) if (plan.nodes[j].kind == DFGPU_EXPR_COLUMN && plan.nodes[j].a >= (int)cols.size()) evaluable = false;
      if (evaluable) {
        ExprPlan sub = plan_expr(types.data(), (int)types.size(), plan.nodes.data() + g.lhs_start, lhs_n);
        EvalResult ev = evaluate_expr(ctx, sub, cols, n, true, false);
        const int64_t nulls = ev.column.validity ? n - count_set_bits(ctx, ev.column.validity, ev.column.offset, n) : 0;
        if (nulls == 0) {
          const int64_t t = count_set_bits(ctx, (const uint8_t*)ev.column.values, ev.column.offset, n);
          const int64_t rare = g.is_and ? t : n - t;          // the rows that still depend on the RHS
          active = rare == 0 || ((float)rare / (float)n <= 0.2f);
        }
      }
    }
    if (!active) continue;
    for (int j = g.rhs_start; j < g.op_idx; ++j) {
      if (g.is_and) masks[j].first |= (uint16_t)(1u << g.slot); else masks[j].second |= (uint16_t)(1u << g.slot);
    }
  }
  return masks;
}

uint64_t literal_bits(const dfgpu_expr_node& nd) {
  if (type_is_float(nd.type)) {
    double d = nd.lit_f64;
    if (nd.type == DFGPU_FLOAT32) d = (double)(float)d;
    uint64_t b; memcpy(&b, &d, 8); return b;
  }
  if (nd.type == DFGPU_BOOL) return nd.lit_i64 ? 1 : 0;
  if (type_is_decimal(nd.type)) return (uint64_t)nd.lit_i64;   // low half; the high half rides in the bytes of lit_f64 (bind_program)
  switch (nd.type) {
    case DFGPU_INT8: return (uint64_t)(int64_t)(int8_t)nd.lit_i64;
    case DFGPU_INT16: return (uint64_t)(int64_t)(int16_t)nd.lit_i64;
    case DFGPU_INT32: case DFGPU_DATE32: return (uint64_t)(int64_t)(int32_t)nd.lit_i64;
    case DFGPU_UINT8: return (uint64_t)nd.lit_i64 & 0xFFull;
    case DFGPU_UINT16: return (uint64_t)nd.lit_i64 & 0xFFFFull;
    case DFGPU_UINT32: return (uint64_t)nd.lit_i64 & 0xFFFFFFFFull;
    default: return (uint64_t)nd.lit_i64;
  }
}

void bind_program(const ExprPlan& plan, const std::vector<DCol>& cols, EProgram* prog, const std::vector<std::pair<uint16_t, uint16_t>>* gmasks) {
  memset(prog, 0, sizeof(*prog));
  prog->n = (int)plan.nodes.size();
  for (int i = 0; i < prog->n; ++i) {
    const dfgpu_expr_node& nd = plan.nodes[i];
    ENode& e = prog->node[i];
    e.kind = nd.kind; e.op = nd.a; e.in_type = plan.in_type[i]; e.out_type = plan.out_type[i];
    if (nd.kind == DFGPU_EXPR_COLUMN) {
      const DCol& c = cols[nd.a];
      DF_CHECK(c.type == plan.out_type[i], DFGPU_ERR_INVALID, "expression: batch column type differs from the planned schema");
      e.col = c.values; e.valid = c.validity; e.voff = c.offset;
    } else if (nd.kind == DFGPU_EXPR_LITERAL) {
      e.lit = literal_bits(nd); e.lit_null = nd.is_null;
      if (type_is_decimal(nd.type)) memcpy(&e.voff, &nd.lit_f64, 8);
    } else if ((nd.kind == DFGPU_EXPR_BINARY || nd.kind == DFGPU_EXPR_CAST) && plan.has_decimal) {
      e.voff = plan.aux[i];   // power-of-ten rescale exponents (expr_dec.cuh)
    }
    if (gmasks) { e.g_and = (*gmasks)[i].first; e.g_or = (*gmasks)[i].second; }
  }
}

// Evaluate `plan` over device columns.  want_select: also produce selection words (valid & true).

EvalResult evaluate_expr(dfgpu_ctx* ctx, const ExprPlan& plan, const std::vector<DCol>& cols, int64_t n, bool want_column, bool want_select) {
  EvalResult res;
  const int64_t nw = (n + 31) / 32;
  if (want_select) res.select_words.alloc(ctx, (size_t)std::max<int64_t>(nw, 1) * 4);
  // fast path: Column(int64-like, no nulls) cmp Literal(non-null)
  if (want_select && !want_column && plan.nodes.size() == 3 && plan.nodes[0].kind == DFGPU_EXPR_COLUMN && plan.nodes[1].kind == DFGPU_EXPR_LITERAL &&
      plan.nodes[2].kind == DFGPU_EXPR_BINARY && plan.nodes[2].a >= DFGPU_OP_EQ && plan.nodes[2].a <= DFGPU_OP_GTEQ && !plan.nodes[1].is_null) {
    const DCol& c = cols[plan.nodes[0].a];
    if (cls_of(c.type) == C_I64 && type_width(c.type) == 8 && !c.validity && ((uintptr_t)c.values % 16 == 0)) {
      if (n > 0) {
        const int64_t* p = (const int64_t*)c.values;
        int64_t lit = (int64_t)literal_bits(plan.nodes[1]);
        int grid = grid_for((n + 511) / 512 * 32, 256, kNumSMs * 8);
        uint32_t* sw = res.select_words.as<uint32_t>();
        switch (plan.nodes[2].a) {
          case DFGPU_OP_EQ: cmp_i64_scalar_kernel<DFGPU_OP_EQ><<<grid, 256, 0, ctx->stream>>>(p, n, lit, sw); break;
          case DFGPU_OP_NEQ: cmp_i64_scalar_kernel<DFGPU_OP_NEQ><<<grid, 256, 0, ctx->stream>>>(p, n, lit, sw); break;
          case DFGPU_OP_LT: cmp_i64_scalar_kernel<DFGPU_OP_LT><<<grid, 256, 0, ctx->stream>>>(p, n, lit, sw); break;
          case DFGPU_OP_LTEQ: cmp_i64_scalar_kernel<DFGPU_OP_LTEQ><<<grid, 256, 0, ctx->stream>>>(p, n, lit, sw); break;
          case DFGPU_OP_GT: cmp_i64_scalar_kernel<DFGPU_OP_GT><<<grid, 256, 0, ctx->stream>>>(p, n, lit, sw); break;
          default: cmp_i64_scalar_kernel<DFGPU_OP_GTEQ><<<grid, 256, 0, ctx->stream>>>(p, n, lit, sw); break;
        }
        DF_LAUNCH_CHECK(ctx);
      }
      return res;
    }
  }
  EProgram prog;
  const auto gmasks = resolve_guards(ctx, plan, cols, n);
  bind_program(plan, cols, &prog, &gmasks);
  const int rt = plan.root_type;
  if (want_column) {
    res.column = alloc_col(ctx, rt, n, true);
  }
  DevBuf err(ctx, 4);
  err.zero();
  if (n > 0) {
    auto kern = plan.has_decimal ? expr_eval_dec_kernel : expr_eval_kernel;
    kern<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(
        prog, n, (want_column && rt != DFGPU_BOOL) ? res.column.own_values->ptr : nullptr,
        (want_column && rt == DFGPU_BOOL) ? res.column.own_values->as<uint32_t>() : nullptr,
        want_column ? res.column.own_validity->as<uint32_t>() : nullptr, want_select ? res.select_words.as<uint32_t>() : nullptr, err.as<int>());
    DF_LAUNCH_CHECK(ctx);
    int e = read_scalar<int>(ctx, err.as<int>());
    if (e & ERR_DIV_ZERO) throw Error(DFGPU_ERR_ARITH, "Arrow error: Divide by zero error");
    if (e & ERR_OVERFLOW) throw Error(DFGPU_ERR_ARITH, "Arrow error: Arithmetic overflow");
    if (e & ERR_CAST) throw Error(DFGPU_ERR_ARITH, "Arrow error: Cast error: Can't cast value to the target type (out of range or beyond the Decimal128 precision)");
  }
  if (want_column) {
    // an expression over columns that carry no validity bitmap in THIS batch and without NULL literals cannot produce a NULL
    // (errors, not NULLs, come out of division by zero): drop the all-ones bitmap so consumers keep their no-NULL fast paths
    bool can_null = false;
    for (const auto& nd : plan.nodes) {
      if (nd.kind == DFGPU_EXPR_COLUMN && cols[nd.a].validity) can_null = true;
      if (nd.kind == DFGPU_EXPR_LITERAL && nd.is_null) can_null = true;
    }
    if (can_null) res.column.null_count = -1;
    else { res.column.null_count = 0; res.column.validity = nullptr; res.column.own_validity.reset(); }
  }
  return res;
}

}  // namespace dfgpu

// ==========================================================================================
// GpuFilterExec
// ==========================================================================================
using namespace dfgpu;

struct dfgpu_filter {
  dfgpu_ctx* ctx = nullptr;
  std::vector<int> schema, projection;
  ExprPlan plan;
  int64_t batch_size = 8192, fetch = -1;
  bool finished = false, limit_reached = false;
  // coalescer state: pending filtered parts (LimitedBatchCoalescer, coalesce/mod.rs:27-147)
  std::vector<std::vector<DCol>> pending;
  int64_t pending_rows = 0, total_rows = 0;
  std::deque<BatchPtr> outq;
  int64_t m_input_rows = 0, m_output_rows = 0, m_input_batches = 0, m_output_batches = 0;
};

namespace dfgpu {

static void filter_flush(dfgpu_filter* f, bool final_flush) {
  dfgpu_ctx* ctx = f->ctx;
  if (f->pending_rows == 0) return;
  if (!final_flush && f->batch_size > 0 && f->pending_rows < f->batch_size) return;
  // concatenate the buffered parts, then cut batch_size-row batches (BatchCoalescer emits exactly target-size batches)
  size_t ncols = f->projection.size();
  std::vector<DCol> merged;
  for (size_t c = 0; c < ncols; ++c) {
    std::vector<DCol> parts;
    for (auto& b : f->pending) parts.push_back(b[c]);
    merged.push_back(concat_columns(ctx, parts, f->schema[f->projection[c]]));
  }
  int64_t rows = f->pending_rows;
  f->pending.clear();
  f->pending_rows = 0;
  int64_t pos = 0;
  const int64_t bs = f->batch_size > 0 ? f->batch_size : rows;
  while (rows - pos >= bs || (final_flush && pos < rows)) {
    int64_t len = std::min<int64_t>(bs, rows - pos);
    BatchPtr b(new dfgpu_batch());
    b->ctx = ctx; b->rows = len; b->host = false;
    for (size_t c = 0; c < ncols; ++c) b->cols.push_back((pos == 0 && len == rows) ? merged[c] : slice_column(merged[c], pos, len));
    f->m_output_rows += len;
    f->m_output_batches++;
    f->outq.push_back(std::move(b));
    pos += len;
  }
  if (pos < rows) {
    std::vector<DCol> rest;
    for (size_t c = 0; c < ncols; ++c) rest.push_back(slice_column(merged[c], pos, rows - pos));
    f->pending.push_back(std::move(rest));
    f->pending_rows = rows - pos;
  }
}

static void filter_push(dfgpu_filter* f, const std::vector<DCol>& cols) {
  DF_CHECK(!f->finished, DFGPU_ERR_STATE, "push after finish");
  DF_CHECK(cols.size() == f->schema.size(), DFGPU_ERR_INVALID, "filter input column count mismatch");
  dfgpu_ctx* ctx = f->ctx;
  set_device(ctx);
  int64_t n = cols.empty() ? 0 : cols[0].length;
  for (size_t c = 0; c < cols.size(); ++c) {
    DF_CHECK(cols[c].type == f->schema[c], DFGPU_ERR_INVALID, "filter input column type mismatch");
    DF_CHECK(cols[c].length == n, DFGPU_ERR_INVALID, "filter input ragged columns");
  }
  f->m_input_rows += n;
  f->m_input_batches++;
  if (n == 0 || f->limit_reached) return;
  DF_CHECK(n < 0xFFFFFFFFll, DFGPU_ERR_UNSUPPORTED, "filter: a batch must have < 2^32-1 rows");
  // ---- fused single-pass path: plain projected columns, no fetch limit ----
  bool fusable = f->fetch < 0 && f->projection.size() <= (size_t)kMaxFiltCols;
  for (int pc : f->projection) if (cols[pc].validity || cols[pc].type == DFGPU_BOOL) fusable = false;
  static const int fused_enabled = getenv("DFGPU_FILTER_FUSED") ? atoi(getenv("DFGPU_FILTER_FUSED")) : 1;
  if (fusable && fused_enabled) {
    FilterCols fc;
    memset(&fc, 0, sizeof(fc));
    fc.n = (int)f->projection.size();
    std::vector<DCol> part;
    for (int c = 0; c < fc.n; ++c) {
      const DCol& src = cols[f->projection[c]];
      DCol d = alloc_col(ctx, src.type, n, false);
      fc.src[c] = src.values; fc.dst[c] = d.own_values->ptr; fc.width[c] = type_width(src.type);
      part.push_back(std::move(d));
    }
    const int64_t nt = (n + kFiltTile - 1) / kFiltTile;
    DevBuf desc(ctx, (size_t)nt * 8 + 32), progbuf, err(ctx, 4);
    desc.zero();
    err.zero();
    unsigned long long* totals = (unsigned long long*)((char*)desc.ptr + (size_t)nt * 8);
    unsigned int* counter = (unsigned int*)(totals + 2);
    const ExprPlan& plan = f->plan;
    bool fast = plan.nodes.size() == 3 && plan.nodes[0].kind == DFGPU_EXPR_COLUMN && plan.nodes[1].kind == DFGPU_EXPR_LITERAL && plan.nodes[2].kind == DFGPU_EXPR_BINARY &&
                plan.nodes[2].a >= DFGPU_OP_EQ && plan.nodes[2].a <= DFGPU_OP_GTEQ && !plan.nodes[1].is_null;
    if (fast) {
      const DCol& c = cols[plan.nodes[0].a];
      fast = cls_of(c.type) == C_I64 && type_width(c.type) == 8 && !c.validity;
    }
    {
      KernelTimer kt(ctx, "filter_fused");
      if (fast) {
        filter_fused_kernel<1><<<(int)nt, kFiltThreads, 0, ctx->stream>>>(nullptr, (const int64_t*)cols[plan.nodes[0].a].values, plan.nodes[2].a, (int64_t)literal_bits(plan.nodes[1]), n,
                                                                          fc, desc.as<unsigned long long>(), counter, totals, err.as<int>());
      } else {
        EProgram prog;
        const auto gmasks = resolve_guards(ctx, plan, cols, n);
        bind_program(plan, cols, &prog, &gmasks);
        progbuf.alloc(ctx, sizeof(EProgram));
        DF_CUDA(cudaMemcpyAsync(progbuf.ptr, &prog, sizeof(EProgram), cudaMemcpyHostToDevice, ctx->stream));
        DF_CUDA(cudaStreamSynchronize(ctx->stream));  // `prog` lives on this stack frame
        if (plan.has_decimal) filter_fused_kernel<2><<<(int)nt, kFiltThreads, 0, ctx->stream>>>((const EProgram*)progbuf.ptr, nullptr, 0, 0, n, fc, desc.as<unsigned long long>(), counter, totals, err.as<int>());
        else filter_fused_kernel<0><<<(int)nt, kFiltThreads, 0, ctx->stream>>>((const EProgram*)progbuf.ptr, nullptr, 0, 0, n, fc, desc.as<unsigned long long>(), counter, totals, err.as<int>());
      }
      DF_LAUNCH_CHECK(ctx);
    }
    unsigned long long h[2];
    int herr = 0;
    DF_CUDA(cudaMemcpyAsync(h, totals, 16, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaMemcpyAsync(&herr, err.ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    if (herr & ERR_DIV_ZERO) throw Error(DFGPU_ERR_ARITH, "Arrow error: Divide by zero error");
    if (herr & ERR_OVERFLOW) throw Error(DFGPU_ERR_ARITH, "Arrow error: Arithmetic overflow");
    if (herr & ERR_CAST) throw Error(DFGPU_ERR_ARITH, "Arrow error: Cast error: Can't cast value to the target type (out of range)");
    const int64_t kept = (int64_t)h[0];
    if (kept == 0) return;
    for (auto& c : part) c.length = kept;
    f->total_rows += kept;
    f->pending.push_back(std::move(part));
    f->pending_rows += kept;
    filter_flush(f, false);
    return;
  }
  EvalResult ev = evaluate_expr(ctx, f->plan, cols, n, false, true);
  DevBuf idx;
  int64_t kept = compact_flag_indices(ctx, ev.select_words.as<uint32_t>(), n, 1, &idx);
  if (kept == 0) return;
  if (f->fetch >= 0 && f->total_rows + kept >= f->fetch) {  // LimitReached: keep only the head (coalesce/mod.rs:100-112)
    kept = f->fetch - f->total_rows;
    f->limit_reached = true;
  }
  f->total_rows += kept;
  if (kept == 0) return;
  std::vector<DCol> part;
  for (int pc : f->projection) part.push_back(take_column(ctx, cols[pc], idx.as<uint32_t>(), kept, false));
  f->pending.push_back(std::move(part));
  f->pending_rows += kept;
  filter_flush(f, false);
}

}  // namespace dfgpu

extern "C" {

int dfgpu_filter_create(dfgpu_ctx* ctx, const int32_t* schema_types, int32_t n_cols, const dfgpu_expr_node* predicate, int32_t n_nodes,
                        const int32_t* projection, int32_t n_projection, int64_t batch_size, int64_t fetch, dfgpu_filter** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && out && schema_types && predicate, DFGPU_ERR_INVALID, "null argument");
  std::unique_ptr<dfgpu_filter> f(new dfgpu_filter());
  f->ctx = ctx;
  f->schema.assign(schema_types, schema_types + n_cols);
  f->plan = plan_expr(schema_types, n_cols, predicate, n_nodes);
  DF_CHECK(f->plan.root_type == DFGPU_BOOL, DFGPU_ERR_INVALID, "Cannot create filter_array from non-boolean predicates");  // filter.rs:1355-1359
  if (projection) {
    for (int i = 0; i < n_projection; ++i) {
      DF_CHECK(projection[i] >= 0 && projection[i] < n_cols, DFGPU_ERR_INVALID, "projection index out of range");
      f->projection.push_back(projection[i]);
    }
  } else for (int i = 0; i < n_cols; ++i) f->projection.push_back(i);
  for (int pc : f->projection) DF_CHECK(type_width(f->schema[pc]) >= 0, DFGPU_ERR_UNSUPPORTED, "filter: column type not supported");
  f->batch_size = batch_size;
  f->fetch = fetch;
  *out = f.release();
  DF_API_END
}
int dfgpu_filter_push_host(dfgpu_filter* f, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(f ? f->ctx : nullptr)
  set_device(f->ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(upload_column(f->ctx, cols[i]));
  filter_push(f, v);
  DF_API_END
}
int dfgpu_filter_push_device(dfgpu_filter* f, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(f ? f->ctx : nullptr)
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(device_view(cols[i]));
  filter_push(f, v);
  DF_API_END
}
int dfgpu_filter_finish(dfgpu_filter* f) {
  DF_API_BEGIN(f ? f->ctx : nullptr)
  DF_CHECK(!f->finished, DFGPU_ERR_STATE, "finish called twice");
  f->finished = true;
  set_device(f->ctx);
  filter_flush(f, true);
  DF_API_END
}
int dfgpu_filter_next(dfgpu_filter* f, int host, dfgpu_batch** out) {
  dfgpu_ctx* _ctx = f ? f->ctx : nullptr;
  try {
    DF_CHECK(f && out, DFGPU_ERR_INVALID, "null argument");
    if (f->outq.empty()) { *out = nullptr; return DFGPU_END; }
    BatchPtr b = std::move(f->outq.front());
    f->outq.pop_front();
    if (host) { set_device(f->ctx); b = to_host_batch(f->ctx, *b); }
    *out = b.release();
    return DFGPU_OK;
  } catch (const dfgpu::Error& e) { if (_ctx) _ctx->last_error = e.what(); return e.code; }
  catch (const std::exception& e) { if (_ctx) _ctx->last_error = e.what(); return DFGPU_ERR_INVALID; }
}
int64_t dfgpu_filter_metric(dfgpu_filter* f, const char* name) {
  if (!f || !name) return -1;
  std::string s(name);
  if (s == "input_rows") return f->m_input_rows;
  if (s == "output_rows") return f->m_output_rows;
  if (s == "input_batches") return f->m_input_batches;
  if (s == "output_batches") return f->m_output_batches;
  if (s == "selectivity_num") return f->total_rows;   // filter.rs:1312-1330: selectivity = output_rows / input_rows
  if (s == "selectivity_den") return f->m_input_rows;
  return -1;
}
void dfgpu_filter_destroy(dfgpu_filter* f) {
  if (!f) return;
  cudaSetDevice(f->ctx->device);
  delete f;
}

static int expr_evaluate_common(dfgpu_ctx* ctx, std::vector<DCol>& v, int64_t n_rows, const dfgpu_expr_node* expr, int32_t n_nodes, dfgpu_batch** out) {
  std::vector<int32_t> types;
  for (auto& c : v) types.push_back(c.type);
  ExprPlan plan = plan_expr(types.data(), (int)types.size(), expr, n_nodes);
  EvalResult ev = evaluate_expr(ctx, plan, v, n_rows, true, false);
  BatchPtr b(new dfgpu_batch());
  b->ctx = ctx; b->rows = n_rows; b->host = false;
  b->cols.push_back(std::move(ev.column));
  *out = b.release();
  return DFGPU_OK;
}
int dfgpu_expr_evaluate_device(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, int64_t n_rows, const dfgpu_expr_node* expr, int32_t n_nodes, dfgpu_batch** out) {
  DF_API_BEGIN(ctx)
  set_device(ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(device_view(cols[i]));
  expr_evaluate_common(ctx, v, n_rows, expr, n_nodes, out);
  DF_API_END
}
int dfgpu_expr_evaluate_host(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, int64_t n_rows, const dfgpu_expr_node* expr, int32_t n_nodes, dfgpu_batch** out) {
  DF_API_BEGIN(ctx)
  set_device(ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(upload_column(ctx, cols[i]));
  dfgpu_batch* dev = nullptr;
  expr_evaluate_common(ctx, v, n_rows, expr, n_nodes, &dev);
  BatchPtr devp(dev);
  *out = to_host_batch(ctx, *devp).release();
  DF_API_END
}

}  // extern "C"
