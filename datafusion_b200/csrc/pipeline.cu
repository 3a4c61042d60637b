// pipeline.cu — fused pipelines: FilterExec -> HashJoinExec probe side(s) -> {join build | AggregateExec | output}.
//
// Reference path being replaced (SURVEY.md §8a rows a1-a3, a12-a15, a19-a24, a27; §8f rank 3):
//   FilterExecStream::poll_next                 physical-plan/src/filter.rs:1364-1445
//   HashJoinStream::process_probe_batch         physical-plan/src/joins/hash_join/stream.rs:740-1000
//   lookup_join_hashmap / equal_rows_arr        stream.rs:396-438, joins/utils.rs:2191-2257
//   adjust_indices_by_join_type (RightSemi/Anti) joins/utils.rs:1432-1490
//   AggregateHashTable::aggregate_batch_inner   aggregates/aggregate_hash_table/common.rs:205-236
//   PrimitiveGroupsAccumulator / CountGroupsAccumulator  prim_op.rs:41-195, count.rs:631-780
//   dynamic filter pushdown (bounds + membership) joins/hash_join/shared_bounds.rs, partitioned_hash_eval.rs
// and the plan shape it serves: sqllogictest/test_files/tpch/plans/q3.slt.part:60-76.
//
// GPU design.  The reference keeps a pipeline's intermediates in CPU cache by streaming 8192-row batches through
// the operators; on the GPU the same effect needs ONE kernel per pipeline: a thread block walks 1024-row tiles of the
// probe-side table, evaluates the predicate from coalesced column loads, probes the build-side structures and feeds
// the sink, so every input byte crosses HBM once and no filtered copy / join output / projection is materialised.
//   * a build side is a `dfgpu_lookup`: an open-addressing table of fixed-stride records
//       {key:u64 | payload:u64 | accumulator words...}   (exact key in the record: no equal_rows re-check),
//     or — for key sets over a dense range — a bitmap (the reference's ArrayMap idea at one bit per key).
//   * a blocked Bloom filter (one 64-bit block per lookup, 16 bits per key, 4 probes) sits in front of tables that
//     exceed L2: it is the device form of the reference's dynamic filter pushdown (membership test pushed into the
//     probe-side scan) and turns nine out of ten random DRAM accesses of a low-hit-rate join into L2 hits.
//   * when the GROUP BY keys are the join key plus build-side columns (TPC-H Q3: l_orderkey, o_orderdate,
//     o_shippriority) the group id IS the build row, so the accumulators live inside the matched record and an
//     update is one or two RED operations on the sector the probe just fetched — no second hash table.
#include "batch.cuh"
#include "scan.cuh"
#include "expr.cuh"
#include "expr_dev.cuh"
#include "expr_dec.cuh"
#include "bloom.cuh"
#include "tma.cuh"
#include <climits>
#include <algorithm>
#include <array>

namespace dfgpu {

std::vector<dfgpu_column> arrow_to_columns(const ArrowArray* batch, const ArrowSchema* schema);  // arrow_io.cu

constexpr uint64_t kEmptyKey = ~0ull;
constexpr int kMaxPipeCols = 16, kMaxStages = 3, kMaxPipeAggs = 4, kMaxExt = 8, kMaxTerms = 4, kPoolNodes = 56, kMaxBuildPay = 8;
constexpr int kPipeThreads = 256, kPipeItems = 4, kPipeTile = kPipeThreads * kPipeItems;
enum LookupMode : int { LK_HASH = 0, LK_BITMAP = 1 };
enum SinkKind : int { SINK_NONE = 0, SINK_COUNT = 1, SINK_BUILD = 2, SINK_AGG = 3, SINK_OUTPUT = 4, SINK_OUTPUT_ANY = 5 /* row order unspecified */,
                      SINK_PACK = 6 /* build sink, table size unknown: {key, payload} records to a staging buffer, inserted afterwards */,
                      SINK_DENSE = 7 /* aggregate over group keys in small declared domains: slot arithmetic, shared-memory accumulators */,
                      SINK_HASH = 8 /* aggregate over a packed group key: find-or-claim in the sink's own table */ };
constexpr int kStageMaybe = 3;   // DFGPU_STAGE_MAYBE
static_assert(kExtValid == kMaxStages, "the payload validity word follows the kMaxStages payload words (expr_dev.cuh)");
constexpr int kPipeVarDefault = 11;   // pipe_kernel's VAR when DFGPU_PIPE_VAR is not set (H100 SXM at 400 W, Q3 SF100 lineitem pass: 17.5 ms; 43 20.4-20.9 ms)
// ring-fed phase A: at most kMaxRing streamed columns, kMaxRingStages tiles per warp ring, the mbarriers in the first kRingBarBytes of the
// dynamic shared memory; kGather gathered argument columns
constexpr int kMaxRing = 4, kMaxRingStages = 4, kRingBarBytes = 256, kGather = 2;
constexpr int kErrRingAgg = 8;   // error bit (next to ErrBits): the ring kernel met an aggregate that fill_ring should not have admitted
// bytes of rings per block.  The aggregate sink runs three blocks per SM with 2-tile rings: its phase B lookups need the warps (Q3 SF100
// lineitem pass on an H100 SXM at 700 W: 15.0 ms, against 18.5 ms with two blocks and 4-tile rings).  The pack sink runs two blocks with
// 4-tile rings (orders pass: 1.71 ms, against 1.78 ms with 3-tile rings).
constexpr int ring_smem(int sink) { return sink == SINK_AGG ? 48 * 1024 : 96 * 1024; }

struct LookupDev {
  int mode, stride /* 8-byte words per record */, has_payload, pad;
  unsigned long long* recs; uint64_t cap;
  unsigned long long* bloom; uint64_t bloom_blocks;
  uint32_t* coarse; uint64_t coarse_words;   // optional first level (4 bits per key, L2-resident) in front of a filter that exceeds L2
  uint32_t* bits; uint64_t kmin, ksize;
};
struct ColRef { const void* ptr; const uint8_t* valid; int64_t voff; int width, sgn, vec /* base pointer 16-byte aligned: 128-bit loads allowed */, pad; };
struct StageDev { int kind, key_col; LookupDev lk; };
struct ExtDef { int stage, shift, width, type; };
struct AggDef { int func, cls, word, nn_word, start, n, small, pad; };
struct PipeParams {
  int n_cols, hints; ColRef col[kMaxPipeCols];
  int pred_mode /* 0 none, 1 conjunction of col <cmp> literal, 2 interpreter */, n_terms, pred_start, pred_n, pred_small, first_hash /* first stage backed by a hash table, -1 = none */;
  int term_col[kMaxTerms], term_op[kMaxTerms], term_uns[kMaxTerms]; long long term_lit[kMaxTerms];
  int n_stages; StageDev stage[kMaxStages];
  int n_ext; ExtDef ext[kMaxExt];
  // build sink
  LookupDev target; int bkey_col, target_unique, n_bpay, bpay_src[kMaxBuildPay], bpay_shift[kMaxBuildPay], bpay_width[kMaxBuildPay];
  // aggregate sink (group id == record of stage `agg_stage`)
  int agg_stage, rows_word, n_aggs; AggDef agg[kMaxPipeAggs];
  // unordered output sink; the partitioned aggregate sink (pipe_kernel VAR bit 128) writes its {key, value} records to out_dst[0] / out_dst[1],
  // reserved through out_counter, at most target.cap of them
  int n_out, out_src[kMaxPipeCols], out_width[kMaxPipeCols]; void* out_dst[kMaxPipeCols]; unsigned long long* out_counter;
  ENode pool[kPoolNodes];
  // ring-fed phase A (pipe_kernel VAR bit 64): ring_stages > 0 when this batch qualifies (fill_params)
  int ring_stages, ring_bytes /* one stage: a 256-row warp tile of every ring column */, ring_n, ring_col[kMaxRing], ring_off[kMaxPipeCols] /* byte offset in a stage */;
  int n_gather, gather_node[kGather];   // pool nodes of agg[0]'s column operands, loaded for all survivors of a round before evaluating
};

// ---- cache-policy loads: the table scan is read-once (evict first), the lookup structures should stay in L2 ----
__device__ __forceinline__ uint64_t policy_evict_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t policy_normal() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t policy_evict_last() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t ld_stream_int(const void* base, int width, int sgn, int64_t row, uint64_t pol) {
  switch (width) {
    case 1: { uint32_t v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"((const uint8_t*)base + row), "l"(pol)); return sgn ? (uint64_t)(int64_t)(int8_t)v : (uint64_t)v; }
    case 2: { uint32_t v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %2;" : "=r"(v) : "l"((const uint16_t*)base + row), "l"(pol)); return sgn ? (uint64_t)(int64_t)(int16_t)v : (uint64_t)v; }
    case 4: { uint32_t v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"((const uint32_t*)base + row), "l"(pol)); return sgn ? (uint64_t)(int64_t)(int32_t)v : (uint64_t)v; }
    default: { uint64_t v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"((const uint64_t*)base + row), "l"(pol)); return v; }
  }
}
__device__ __forceinline__ void st_stream_u64(unsigned long long* p, unsigned long long v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" :: "l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ unsigned long long ld_keep_u64(const unsigned long long* p, uint64_t pol) {
  unsigned long long v; asm volatile("ld.global.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol)); return v;
}

__device__ __forceinline__ uint64_t lk_hash(uint64_t key) { return hash_u64(key, kSeedJoin); }
// Coarse first level for filters that do not fit L2 (a join's filter shared by 4-8 GPUs is hundreds of MB): 4 bits per key, two probe
// bits in one 32-bit word.  It stays L2-resident and rejects ~85 % of the keys without a partner, so only ~1 probe in 4 pays the DRAM
// access of the exact (16 bits per key) level behind it.
struct CoarsePos { uint32_t word, mask; };
__device__ __forceinline__ CoarsePos coarse_pos(uint64_t key, uint64_t words) {
  uint32_t h = ((uint32_t)key * 0x27D4EB2Fu) ^ ((uint32_t)(key >> 32) * 0x165667B1u);
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13;
  CoarsePos p;
  p.word = __umulhi(h, (uint32_t)words);
  const uint32_t t = h * 0xC2B2AE35u;
  p.mask = (1u << (t >> 27)) | (1u << ((t >> 22) & 31));
  return p;
}
__device__ __forceinline__ void filter_set(const LookupDev& t, uint64_t key) {
  bloom_set(t.bloom, t.bloom_blocks, key);
  if (t.coarse) { const CoarsePos c = coarse_pos(key, t.coarse_words); atomicOr(&t.coarse[c.word], c.mask); }
}

// insert one record; returns 0 inserted, 1 duplicate key, 2 cannot store this key
__device__ __forceinline__ int lk_insert(const LookupDev& t, uint64_t key, uint64_t pay) {
  if (t.mode == LK_BITMAP) {
    const uint64_t i = key - t.kmin;
    if (i >= t.ksize) return 2;          // outside the promised range
    atomicOr(&t.bits[i >> 5], 1u << (i & 31));
    return 0;
  }
  if (key == kEmptyKey) return 2;
  const uint64_t h = lk_hash(key);
  if (t.cap == 0) {   // filter-only lookup: membership bits, no table
    filter_set(t, key);
    return 0;
  }
  uint64_t s = __umul64hi(h, t.cap);
  int rc = 0;
  while (true) {
    unsigned long long* r = t.recs + s * (uint64_t)t.stride;
    unsigned long long prev;
    if (t.has_payload) prev = cas128(r, Rec128{kEmptyKey, 0ull}, Rec128{key, pay}).lo;
    else prev = atomicCAS(r, (unsigned long long)kEmptyKey, (unsigned long long)key);
    if (prev == kEmptyKey) break;
    if (prev == key) { rc = 1; break; }
    if (++s == t.cap) s = 0;
  }
  if (rc == 0 && t.bloom) filter_set(t, key);
  return rc;
}

__device__ __forceinline__ uint64_t ext_field(uint64_t word, int shift, int width, int type) {
  uint64_t v = word >> shift;
  if (width < 8) { v &= (1ull << (8 * width)) - 1ull; if (type_is_signed_int(type)) v = (uint64_t)(((int64_t)(v << (64 - 8 * width))) >> (64 - 8 * width)); }
  return v;
}

// ------------------------------------------------------------------------------------------
// the pipeline kernel.  Every WARP runs the pipeline on its own 256-row tiles, in two phases, with no block barrier:
//   phase A (every row, cheap, coalesced): a lane owns 8 consecutive rows and reads them with 128-bit loads (a warp request
//     is 512 contiguous bytes per instruction); it evaluates the predicate, the bitmap stages and the Bloom pre-test of the
//     hash stages, and appends the surviving row numbers to the warp's queue in shared memory;
//   phase B (survivors only, dense): whenever the queue holds >= 128 entries every lane takes four of them — all lanes busy,
//     four table lookups in flight per lane — resolves the hash stages and feeds the sink (record insert / accumulator RED).
// Without the queue the expensive tail (a DRAM lookup, the argument interpreter, an insert CAS) runs at warp granularity for
// the few live lanes of every warp: that cost 27 warp-instructions and 143 B of DRAM traffic per row on Q3's lineitem pass.
// ------------------------------------------------------------------------------------------
constexpr int kWarpRows = 8, kWarpTile = 32 * kWarpRows, kPhaseB = 2, kPhaseBGroup = 32 * kPhaseB, kQueueCap = kPhaseBGroup + kWarpTile;
constexpr int kPipeWarps = kPipeThreads / 32;

__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v) { asm volatile("red.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_add_f64(unsigned long long* p, double v) { asm volatile("red.global.add.f64 [%0], %1;" :: "l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ void red_min_s64(unsigned long long* p, long long v) { asm volatile("red.global.min.s64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_max_s64(unsigned long long* p, long long v) { asm volatile("red.global.max.s64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_min_u64(unsigned long long* p, unsigned long long v) { asm volatile("red.global.min.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_max_u64(unsigned long long* p, unsigned long long v) { asm volatile("red.global.max.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }

// Pure 64-bit integer arithmetic (integer columns without NULLs in this batch, integer literals, payload fields, + - *): nothing can be
// NULL, nothing can fail — a four-register stack and ~10 instructions per node instead of the general interpreter's ~100.
__device__ __forceinline__ uint64_t eval_int_fast(const ENode* __restrict__ nodes, int n, int64_t row, const uint64_t* ext) {
  uint64_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;   // s0 = top of stack
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const ENode& nd = nodes[i];
    if (nd.kind == DFGPU_EXPR_BINARY) {
      uint64_t r = nd.op == DFGPU_OP_PLUS ? s1 + s0 : (nd.op == DFGPU_OP_MINUS ? s1 - s0 : s1 * s0);
      if (type_width_prim(nd.out_type) < 8) r = wrap_to_type(r, nd.out_type);
      s0 = r; s1 = s2; s2 = s3;
    } else {
      uint64_t v;
      if (nd.kind == DFGPU_EXPR_COLUMN) v = load_col_value(nd, row);
      else if (nd.kind == DFGPU_EXPR_LITERAL) v = nd.lit;
      else { v = ext[nd.voff] >> (int)nd.lit; const int w = type_width_prim(nd.out_type); if (w < 8) { v &= (1ull << (8 * w)) - 1ull; if (type_is_signed_int(nd.out_type)) v = (uint64_t)(((int64_t)(v << (64 - 8 * w))) >> (64 - 8 * w)); } }
      s3 = s2; s2 = s1; s1 = s0; s0 = v;
    }
  }
  return s0;
}
// the same program with its first `ng` column operands already loaded (g0 first): the loads of a round were all issued before the first
// evaluation instead of one dependent access per node; same operations in the same order
__device__ __forceinline__ uint64_t eval_int_gathered(const ENode* __restrict__ nodes, int n, int64_t row, const uint64_t* ext, int ng, uint64_t g0, uint64_t g1) {
  uint64_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const ENode& nd = nodes[i];
    if (nd.kind == DFGPU_EXPR_BINARY) {
      uint64_t r = nd.op == DFGPU_OP_PLUS ? s1 + s0 : (nd.op == DFGPU_OP_MINUS ? s1 - s0 : s1 * s0);
      if (type_width_prim(nd.out_type) < 8) r = wrap_to_type(r, nd.out_type);
      s0 = r; s1 = s2; s2 = s3;
    } else {
      uint64_t v;
      if (nd.kind == DFGPU_EXPR_COLUMN) {
        if (ng > 0) { v = g0; g0 = g1; --ng; }
        else v = load_col_value(nd, row);
      } else if (nd.kind == DFGPU_EXPR_LITERAL) v = nd.lit;
      else { v = ext[nd.voff] >> (int)nd.lit; const int w = type_width_prim(nd.out_type); if (w < 8) { v &= (1ull << (8 * w)) - 1ull; if (type_is_signed_int(nd.out_type)) v = (uint64_t)(((int64_t)(v << (64 - 8 * w))) >> (64 - 8 * w)); } }
      s3 = s2; s2 = s1; s1 = s0; s0 = v;
    }
  }
  return s0;
}

// programs that touch Decimal128 values (small == 3): the 128-bit interpreter; returns the low word, *hi the high word.
// XN (and in the functions below): nullable payload fields, ext[kExtValid] holds their validity bits (pipe_kernel VAR bit 1024)
template <bool XN = false>
__device__ __noinline__ uint64_t pipe_eval_dec(const ENode* nodes, int n, int64_t row, const uint64_t* ext, int* err_ok, unsigned long long* hi) {
  bool ok;
  int err = 0;
  const i128 v = eval_nodes_dec<XN>(nodes, n, row, &ok, &err, ext);
  err_ok[0] |= err; err_ok[1] = ok ? 1 : 0;
  *hi = (unsigned long long)((u128)v >> 64);
  return (uint64_t)v;
}
// one out-of-line copy of each interpreter: the kernel stays small enough for the instruction cache
template <bool DEC, bool XN = false>
__device__ __noinline__ uint64_t pipe_eval(const ENode* nodes, int n, int small, int64_t row, const uint64_t* ext, int* err_ok /* [0]=err bits (or-ed), [1]=valid */) {
  if (DEC && small == 3) { unsigned long long hi; return pipe_eval_dec<XN>(nodes, n, row, ext, err_ok, &hi); }
  bool ok;
  int err = 0;
  const uint64_t v = small ? eval_nodes_reg<4, XN>(nodes, n, row, &ok, &err, ext) : eval_nodes<XN>(nodes, n, row, &ok, &err, ext);
  err_ok[0] |= err; err_ok[1] = ok ? 1 : 0;
  return v;
}
// SUM over a Decimal128 argument, evaluated and accumulated out of line (the hot integer path of the aggregate sink stays as it was):
// i128 add_wrapping over two accumulator words — the carry out of the low word is decided by this add alone
template <bool XN = false>
__device__ __noinline__ void pipe_sum_dec(const ENode* nodes, int n, int64_t row, const uint64_t* ext, int* err_ok, unsigned long long* acc, unsigned long long* nn) {
  unsigned long long hi;
  const unsigned long long lo = pipe_eval_dec<XN>(nodes, n, row, ext, err_ok, &hi);
  if (!err_ok[1]) return;                                  // NULL inputs are skipped (accumulate.rs:373-470)
  if (nn) atomicAdd(nn, 1ull);
  const unsigned long long old = atomicAdd(acc, lo);
  const unsigned long long add_hi = hi + ((old + lo) < old ? 1ull : 0ull);
  if (add_hi) atomicAdd(acc + 1, add_hi);
}
// MIN / MAX over a Decimal128 argument, out of line like SUM: the {lo, hi} pair at acc (16-byte aligned in the record) is read in one
// 128-bit load and replaced by a 128-bit CAS only when the value is better
template <bool XN = false>
__device__ __noinline__ void pipe_minmax_dec(const ENode* nodes, int n, int64_t row, const uint64_t* ext, int* err_ok, unsigned long long* acc, unsigned long long* nn,
                                             bool is_min) {
  unsigned long long hi;
  const unsigned long long lo = pipe_eval_dec<XN>(nodes, n, row, ext, err_ok, &hi);
  if (!err_ok[1]) return;                                  // NULL inputs are skipped
  if (nn) atomicAdd(nn, 1ull);
  minmax_i128(acc, Rec128{lo, hi}, is_min);
}

__device__ __forceinline__ uint4 ld_stream_v4(const void* p, uint64_t pol) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint2 ld_stream_v2(const void* p, uint64_t pol) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(r.x), "=r"(r.y) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint64_t ext32(uint32_t x, int sgn) { return sgn ? (uint64_t)(int64_t)(int32_t)x : (uint64_t)x; }
__device__ __forceinline__ uint64_t ext16(uint32_t x, int sgn) { return sgn ? (uint64_t)(int64_t)(int16_t)x : (uint64_t)(x & 0xFFFFu); }
__device__ __forceinline__ uint64_t ext8(uint32_t x, int sgn) { return sgn ? (uint64_t)(int64_t)(int8_t)x : (uint64_t)(x & 0xFFu); }
// 8 consecutive elements starting at row0 (a multiple of 8), sign / zero extended to 64 bits
// one whole 32-byte sector (p 32-byte aligned): a lane's 8 rows of a 4-byte column are one sector, of an 8-byte column two.  sm_90 has
// no 256-bit load, so these are the same two 128-bit loads the vec == 1 path below issues: on Hopper a warp instruction asks L2 for
// half sectors either way, and VAR bit 5 changes the code but not the requests
__device__ __forceinline__ void ld_stream_v4x64(const void* p, uint64_t pol, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;" : "=l"(a), "=l"(b) : "l"(p), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;" : "=l"(c), "=l"(d) : "l"((const char*)p + 16), "l"(pol));
}
template <bool WIDE = false>
__device__ __forceinline__ void load8(const ColRef& c, int64_t row0, int64_t n, uint64_t v[kWarpRows], uint64_t pol) {
  if (WIDE && c.vec == 2 && row0 + kWarpRows <= n && (c.width == 8 || c.width == 4)) {   // vec == 2: base pointer 32-byte aligned
    if (c.width == 8) {
      const char* p = (const char*)c.ptr + row0 * 8;
      ld_stream_v4x64(p, pol, v[0], v[1], v[2], v[3]);
      ld_stream_v4x64(p + 32, pol, v[4], v[5], v[6], v[7]);
    } else {
      uint64_t a, b, cc, d;
      ld_stream_v4x64((const char*)c.ptr + row0 * 4, pol, a, b, cc, d);
      v[0] = ext32((uint32_t)a, c.sgn); v[1] = ext32((uint32_t)(a >> 32), c.sgn); v[2] = ext32((uint32_t)b, c.sgn); v[3] = ext32((uint32_t)(b >> 32), c.sgn);
      v[4] = ext32((uint32_t)cc, c.sgn); v[5] = ext32((uint32_t)(cc >> 32), c.sgn); v[6] = ext32((uint32_t)d, c.sgn); v[7] = ext32((uint32_t)(d >> 32), c.sgn);
    }
    return;
  }
  if (c.vec && row0 + kWarpRows <= n) {
    switch (c.width) {
      case 8: {
        const char* p = (const char*)c.ptr + row0 * 8;
#pragma unroll
        for (int q = 0; q < 4; ++q) { const uint4 x = ld_stream_v4(p + 16 * q, pol); v[2 * q] = (uint64_t)x.x | ((uint64_t)x.y << 32); v[2 * q + 1] = (uint64_t)x.z | ((uint64_t)x.w << 32); }
        break;
      }
      case 4: {
        const char* p = (const char*)c.ptr + row0 * 4;
        const uint4 x = ld_stream_v4(p, pol), y = ld_stream_v4(p + 16, pol);
        v[0] = ext32(x.x, c.sgn); v[1] = ext32(x.y, c.sgn); v[2] = ext32(x.z, c.sgn); v[3] = ext32(x.w, c.sgn);
        v[4] = ext32(y.x, c.sgn); v[5] = ext32(y.y, c.sgn); v[6] = ext32(y.z, c.sgn); v[7] = ext32(y.w, c.sgn);
        break;
      }
      case 2: {
        const uint4 x = ld_stream_v4((const char*)c.ptr + row0 * 2, pol);
        v[0] = ext16(x.x, c.sgn); v[1] = ext16(x.x >> 16, c.sgn); v[2] = ext16(x.y, c.sgn); v[3] = ext16(x.y >> 16, c.sgn);
        v[4] = ext16(x.z, c.sgn); v[5] = ext16(x.z >> 16, c.sgn); v[6] = ext16(x.w, c.sgn); v[7] = ext16(x.w >> 16, c.sgn);
        break;
      }
      default: {
        const uint2 x = ld_stream_v2((const char*)c.ptr + row0, pol);
        v[0] = ext8(x.x, c.sgn); v[1] = ext8(x.x >> 8, c.sgn); v[2] = ext8(x.x >> 16, c.sgn); v[3] = ext8(x.x >> 24, c.sgn);
        v[4] = ext8(x.y, c.sgn); v[5] = ext8(x.y >> 8, c.sgn); v[6] = ext8(x.y >> 16, c.sgn); v[7] = ext8(x.y >> 24, c.sgn);
        break;
      }
    }
  } else {   // unaligned base or ragged tail: one scalar load site, results routed by selects (keeps v[] in registers, the code small)
#pragma unroll 1
    for (int j = 0; j < kWarpRows; ++j) {
      const uint64_t x = row0 + j < n ? ld_stream_int(c.ptr, c.width, c.sgn, row0 + j, pol) : 0ull;
#pragma unroll
      for (int k = 0; k < kWarpRows; ++k) if (k == j) v[k] = x;
    }
  }
}
// ring-fed phase A: the lane's 8 rows are row0 + 32 j (row0 = tile start + lane), so every shared-memory load of the warp reads
// consecutive elements (no bank conflicts).  `src` is the column's slice of the ring stage; a tile that is not full was not streamed
// and is read from global memory.
__device__ __forceinline__ void ring_load8(const ColRef& c, const unsigned char* src, bool full, int64_t row0, int64_t n, uint64_t v[kWarpRows], uint64_t pol) {
  if (full) {
    const int lane = (int)(row0 & 31);
    switch (c.width) {
      case 8:
#pragma unroll
        for (int j = 0; j < kWarpRows; ++j) v[j] = ((const uint64_t*)src)[32 * j + lane];
        break;
      case 4:
#pragma unroll
        for (int j = 0; j < kWarpRows; ++j) v[j] = ext32(((const uint32_t*)src)[32 * j + lane], c.sgn);
        break;
      case 2:
#pragma unroll
        for (int j = 0; j < kWarpRows; ++j) v[j] = ext16(((const uint16_t*)src)[32 * j + lane], c.sgn);
        break;
      default:
#pragma unroll
        for (int j = 0; j < kWarpRows; ++j) v[j] = ext8(((const uint8_t*)src)[32 * j + lane], c.sgn);
        break;
    }
  } else {
#pragma unroll 1
    for (int j = 0; j < kWarpRows; ++j) {
      const int64_t r = row0 + 32 * j;
      const uint64_t x = r < n ? ld_stream_int(c.ptr, c.width, c.sgn, r, pol) : 0ull;
#pragma unroll
      for (int k = 0; k < kWarpRows; ++k) if (k == j) v[k] = x;
    }
  }
}
// validity bits of the same 8 rows (bit j = row0 + j is non-NULL)
__device__ __forceinline__ uint32_t valid8(const ColRef& c, int64_t row0, int64_t n) {
  if (!c.valid) return 0xFFu;
  const int nb = (int)min((int64_t)kWarpRows, n - row0);
  return nb > 0 ? load_bits32(c.valid, c.voff + row0, nb) : 0u;
}

// VAR (compile-time, so that an instantiation which has been measured stays byte for byte what it was while others are tried against it):
//   bit 0 (1)  at the start of phase B, prefetch.global.L2 the survivors' argument sectors (the integer evaluator would read them one
//              dependent DRAM access after the other);
//   bit 1 (2)  at the start of phase A, prefetch this tile's key column of the first stage (its load is issued only after the predicate's
//              column has arrived and been compared);
//   bit 3 (8)  lane-paired REDs in the aggregate sink: a record's row counter and sum share a sector, so the even lane adds its row's count
//              while its odd neighbour adds the same row's value (then the roles swap) — one reduction request per row instead of two;
//   bit 5 (32) sector-aligned column loads in phase A: a lane's 8 rows are read as one or two whole 32-byte sectors (each as two
//              back-to-back 128-bit loads, the widest sm_90 has: the same requests as without the bit) when the column base is 32-byte aligned.
//   bit 6 (64) ring-fed phase A: the columns phase A reads for every row (predicate terms, keys of the filter / bitmap stages) arrive by
//              TMA bulk copies in a ring of ring_stages warp tiles per warp in dynamic shared memory; lane 0 refills the ring S - 1 tiles
//              ahead, so a warp in phase B keeps its next tiles in flight.  Phase B loads agg[0]'s column operands of the whole round
//              before evaluating (replaces bit 0).  Blocks per SM and ring sizes: ring_smem.  Chosen by launch_pipe, not by DFGPU_PIPE_VAR.
//   bit 7 (128) partitioned aggregate (with bit 6; pipeline_push decides, partitioned_parts): the aggregate stage's table exceeds L2, so
//              phase B makes no lookup — it writes each survivor's {key, SUM argument} to the record buffer (out_dst, out_counter), and
//              pipe_probe_agg_kernel probes them once they are radix-partitioned.  Rows past the buffer's end probe and RED right here.
//   bit 8 (256) stage filters (FiltParams; launch_pipe picks it whenever a stage has one, on top of the sink's default bits, never with
//              bits 6 / 7): phase B evaluates a stage's JoinFilter on the rows whose key matched there, and a row that fails counts as
//              not matched; a filtered bitmap ANTI stage is decided in phase B instead of phase A.
//   bit 9 (512) output columns with validity bitmaps or 16 bytes wide, unordered output sink only (OutValid; pipeline_push picks it when a
//              column of the push needs it, on top of the sink's default or filtered bits).
//   bit 10 (1024) RIGHT stages (Right joins; launch_pipe, hash_push, launch_dense pick it whenever the pipeline has one, never with bits 6,
//              7, 8 or DFGPU_PIPE_VAR): phase A skips a RIGHT stage (it drops nothing); phase B probes it like an INNER hash stage but keeps
//              every row, with the stage's bit of pvalid cleared and its payload word 0 on a miss.  pvalid rides behind the payload words as
//              ext[kExtValid], so the interpreters' XN instantiations see the fields as NULL; the output (with bit 9), dense and hash
//              sinks read it for the fields they take directly.  A FULL stage (kStageFull: a RIGHT stage turned into a Full join by
//              dfgpu_pipeline_set_stage_full) runs the same path and also marks each record it matches (mark_visited).
// DFGPU_PIPE_VAR selects the instantiation (aggregate sink; bits 1 and 5 also for the pack sink, bit 1 for the unordered-output sink); 0 is the
// kernel without any of them, 11 the default.  Tried and removed: four instead of two survivors per lane and phase-B round; prefetching the
// table record and the argument sectors already when a row passes the membership filter in phase A (the prefetches of five tiles queue up
// in front of the column stream).
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

// ------------------------------------------------------------------------------------------
// dense-group aggregate sink (SINK_DENSE): AggregateExec over a FilterExec (and probe stages) whose GROUP BY keys lie in small
// declared domains (TPC-H Q1: l_returnflag x l_linestatus; Q4: o_orderpriority; Q6: no GROUP BY).  The group id is arithmetic:
//   slot = sum_g stride_g * idx_g,  idx_g = key - min_g (a value) or max_g - min_g + 1 (NULL),  row-major strides,
// at most kDenseMaxSlots slots, so no hash table.  The sink's parameters (DenseParams) sit right behind PipeParams in the same device
// allocation; PipeParams and the other sinks' code are unchanged.  Accumulators are privatised per BLOCK in dynamic shared memory
// (a 256-slot domain with 8 aggregates is up to 80 KB: per-warp copies do not fit); before touching them the lanes of a phase-B
// round that share a slot are combined (__match_any_sync + a shuffle tree), so a warp issues one shared atomic per distinct slot
// and aggregate instead of 32.  At kernel end every block adds its slots into the pipeline's global accumulator array (acc), which
// persists across pushes; the row loop makes no global atomics.
// ------------------------------------------------------------------------------------------
constexpr int kDenseMaxSlots = 256, kDenseMaxKeys = 8, kDenseMaxAggs = 8, kDenseMaxWords = 40, kDenseMaxXTerms = 4;
constexpr int kDenseWarpBytes = 48 * 1024;   // per-warp accumulator copies when all eight fit in this many bytes
// how one aggregate's value combines: none (COUNT: only the non-null counter), add, min, max over u64 / i64 / f64 / i128 words
enum DenseOp : int { DO_NONE = 0, DO_ADD_U64, DO_ADD_F64, DO_ADD_128, DO_MIN_S64, DO_MAX_S64, DO_MIN_U64, DO_MAX_U64, DO_MIN_128, DO_MAX_128 };
struct DenseKey { int src /* virtual column */, pad; unsigned long long kmin, nvals /* max - min + 1: the index of NULL */, stride; };
struct DenseAgg { int func, op, small, start, n, word /* value word(s) in a slot, -1 none */, nn_word /* non-null counter, -1 none */,
                  f64_key /* Float64 MIN / MAX: the word holds f64_to_ordered of the value */; };
struct DenseParams {
  int n_keys, n_aggs, n_slots, n_words /* per slot, even: the 128-bit fields are 16-byte aligned; word 0 counts the rows */;
  DenseKey key[kDenseMaxKeys];
  DenseAgg agg[kDenseMaxAggs];
  unsigned long long ident[kDenseMaxWords];   // initial value of each word of a slot (0, or the MIN / MAX identity)
  unsigned long long* acc;                    // [n_slots][n_words] in global memory
  int per_warp;                               // 1: one copy of the slots per warp, updated by plain loads and stores; 0: one per block, atomics
  // `column <cmp> literal` terms of the predicate's conjunction beyond PipeParams' kMaxTerms (TPC-H Q6 has five), tested after them
  int n_xterms, xterm_col[kDenseMaxXTerms], xterm_op[kDenseMaxXTerms], xterm_uns[kDenseMaxXTerms]; long long xterm_lit[kDenseMaxXTerms];
};
constexpr int kDenseParamsOff = (int)((sizeof(PipeParams) + 15) / 16 * 16);   // DenseParams (or HashParams) behind PipeParams in the parameter buffer
constexpr int kDenseAccOff = (int)((sizeof(DenseParams) + 15) / 16 * 16);     // dynamic shared memory: DenseParams, then the slots

// ------------------------------------------------------------------------------------------
// hash-keyed aggregate sink (SINK_HASH): AggregateExec over a FilterExec (and probe stages) whose GROUP BY keys the join key does not
// determine (TPC-H Q15's revenue0: l_suppkey; Q3 grouped by o_custkey).  The group columns of a row are packed into a 128-bit tag
// {lo, hi} (each column at its width, one NULL bit per nullable column) and the sink finds or claims the record
//   {tag_lo | tag_hi | row counter | accumulator words...}
// of that tag in its own open-addressing table (one 16-byte CAS claims a slot); the accumulate block of the join-keyed sink then runs on
// that record.  The table grows between launches: a claim beyond the budget (group_limit) or a probe longer than kHashMaxProbe defers
// the row to the overflow list before it touches any accumulator, and the host grows the table and pushes the deferred rows again.
// The one tag equal to the empty marker {~0, ~0} lives in the side record behind the cap regular slots.  HashParams sit behind
// PipeParams in the parameter buffer, as DenseParams do, and are copied to dynamic shared memory.
// ------------------------------------------------------------------------------------------
constexpr int kHashMaxKeys = 8, kHashMaxWords = 16, kHashMaxProbe = 256;
struct HashKey { int src /* virtual column */, shift /* bit offset in the tag */, bits, null_bit /* -1: declared non-nullable */; };
struct HashParams {
  int n_keys, stride /* words per record, even */, pad0, pad1;
  HashKey key[kHashMaxKeys];
  unsigned long long* recs; uint64_t cap;        // cap regular records, then the side record
  unsigned long long* ngroups; uint64_t group_limit;   // claimed regular records; no claims at or beyond the limit
  uint32_t* overflow; unsigned long long* overflow_count;   // deferred input rows of this launch
};
struct HashIdent { unsigned long long w[kHashMaxWords]; };   // initial value of each record word (tag words ~0, MIN / MAX identities)

// ------------------------------------------------------------------------------------------
// stage filters (pipe_kernel VAR bit 256, pipe_output_kernel<true>): the JoinFilter of a probe stage, a Boolean program evaluated on each
// row whose key matched at that stage.  The programs have a node pool of their own; the block sits behind DenseParams / HashParams in the
// parameter buffer and is copied to dynamic shared memory at smem_off (behind the sink's own block there), so PipeParams and every
// instantiation without the bit are unchanged.
// ------------------------------------------------------------------------------------------
constexpr int kFiltPoolNodes = 128, kVarFilt = 256;
struct FiltParams {
  int smem_off;                                                  // byte offset of this block in the kernel's dynamic shared memory
  int start[kMaxStages], n[kMaxStages] /* 0: no filter */, small[kMaxStages];
  ENode pool[kFiltPoolNodes];
};
constexpr int kFiltParamsOff = kDenseParamsOff + (int)(((sizeof(DenseParams) > sizeof(HashParams) ? sizeof(DenseParams) : sizeof(HashParams)) + 15) / 16 * 16);

// ------------------------------------------------------------------------------------------
// output columns with validity bitmaps or 16 bytes wide (pipe_kernel VAR bit 512 on the unordered output sink, pipe_output_cols_kernel on
// the ordered one): the output bitmaps, zeroed before the launch, sit in the sink's block behind PipeParams (where DenseParams / HashParams
// sit for their sinks), so PipeParams, OutCols and every instantiation without them are unchanged.  An output column has a bitmap exactly
// when its input column has one in this push; payload fields never do.
// ------------------------------------------------------------------------------------------
constexpr int kVarOutCols = 512;
constexpr int kVarRight = 1024, kStageRight = 6;   // pipe_kernel VAR bit 10; DFGPU_STAGE_RIGHT
// a RIGHT stage of a Full join (dfgpu_pipeline_set_stage_full), a kind private to the library: StageDev.kind of that stage, which the host
// keeps as DFGPU_STAGE_RIGHT.  The RIGHT instantiations treat both kinds alike (kind >= kStageRight)
constexpr int kStageFull = 7, kVisitedWord = 2;   // the visited mark: word 2 of the {key, payload, acc...} record, the first accumulator word
// a FULL stage's match: mark the record visited.  The word shares the 32-byte sector of the {key, payload} just read; the store is made
// only while the word is 0 (once per record, not once per matching row) and needs no atomic, as every writer stores the same 1
__device__ __forceinline__ void mark_visited(unsigned long long* rec) {
  if (__ldcg(rec + kVisitedWord) == 0ull) __stcg(rec + kVisitedWord, 1ull);
}
struct OutValid { uint32_t* valid[kMaxPipeCols]; /* nullptr: the column leaves without a bitmap */ };
static_assert(kDenseParamsOff + (int)sizeof(OutValid) <= kFiltParamsOff, "OutValid fits the sink's block");
// one 16-byte value (Decimal128): Arrow promises only 8-byte alignment of a sliced input buffer
__device__ __forceinline__ void copy16(const ColRef& c, int64_t row, void* dst, uint64_t pol) {
  uint4 v;
  if (c.vec) v = ld_stream_v4((const char*)c.ptr + row * 16, pol);
  else {
    const uint64_t lo = ld_stream_int(c.ptr, 8, 0, 2 * row, pol), hi = ld_stream_int(c.ptr, 8, 0, 2 * row + 1, pol);
    v = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
  }
  *(uint4*)dst = v;
}
// stage s's filter on one candidate pair (ext: the payload words of stages 0..s): TRUE passes, NULL and FALSE do not; errors are or-ed
// into err_ok[0], so only candidate pairs raise
template <bool DEC>
__device__ __forceinline__ bool stage_filter_pass(const FiltParams& fp, int s, int64_t row, const uint64_t* ext, int* err_ok) {
  if (fp.n[s] == 0) return true;
  const uint64_t v = pipe_eval<DEC>(fp.pool + fp.start[s], fp.n[s], fp.small[s], row, ext, err_ok);
  return err_ok[1] && (v & 1);
}

__device__ __forceinline__ uint64_t hash_tag_slot(uint64_t lo, uint64_t hi, uint64_t cap) { return __umul64hi(hash_combine(hash_u64(lo, kSeedAgg), hi), cap); }
// the record of tag {lo, hi}, claimed when absent; nullptr when the row must be deferred (claim budget exhausted or probe too long)
__device__ __forceinline__ unsigned long long* hash_find_or_claim(const HashParams& hp, uint64_t lo, uint64_t hi) {
  if (lo == kEmptyKey && hi == kEmptyKey) return hp.recs + hp.cap * (uint64_t)hp.stride;   // the side record
  uint64_t s = hash_tag_slot(lo, hi, hp.cap);
#pragma unroll 1
  for (int probe = 0; probe < kHashMaxProbe; ++probe) {
    unsigned long long* r = hp.recs + s * (uint64_t)hp.stride;
    const uint4 v = __ldcg((const uint4*)r);
    const uint64_t clo = (uint64_t)v.x | ((uint64_t)v.y << 32), chi = (uint64_t)v.z | ((uint64_t)v.w << 32);
    if (clo == lo && chi == hi) return r;
    if (clo == kEmptyKey && chi == kEmptyKey) {
      if (__ldcg(hp.ngroups) >= hp.group_limit) return nullptr;
      const Rec128 prev = cas128(r, Rec128{kEmptyKey, kEmptyKey}, Rec128{lo, hi});
      if (prev.lo == kEmptyKey && prev.hi == kEmptyKey) { atomicAdd(hp.ngroups, 1ull); return r; }
      if (prev.lo == lo && prev.hi == hi) return r;
    }
    if (++s == hp.cap) s = 0;
  }
  return nullptr;
}

__device__ __forceinline__ bool lt128(unsigned long long alo, unsigned long long ahi, unsigned long long blo, unsigned long long bhi) {
  return (long long)ahi < (long long)bhi || (ahi == bhi && alo < blo);   // signed 128-bit a < b
}
// true when value (lo, hi) replaces the current (clo, chi) under a MIN / MAX op
__device__ __forceinline__ bool dense_better(int op, unsigned long long lo, unsigned long long hi, unsigned long long clo, unsigned long long chi) {
  switch (op) {
    case DO_MIN_S64: return (long long)lo < (long long)clo;
    case DO_MAX_S64: return (long long)lo > (long long)clo;
    case DO_MIN_U64: return lo < clo;
    case DO_MAX_U64: return lo > clo;
    case DO_MIN_128: return lt128(lo, hi, clo, chi);
    case DO_MAX_128: return lt128(clo, chi, lo, hi);
    default: return false;
  }
}
__device__ __forceinline__ void dense_combine(int op, unsigned long long& lo, unsigned long long& hi, unsigned long long olo, unsigned long long ohi) {
  if (op == DO_ADD_U64) lo += olo;   // add_wrapping
  else if (op == DO_ADD_F64) lo = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)lo) + __longlong_as_double((long long)olo));
  else if (op == DO_ADD_128) { const unsigned long long s = lo + olo; hi += ohi + (s < lo ? 1ull : 0ull); lo = s; }   // i128 add_wrapping
  else if (dense_better(op, olo, ohi, lo, hi)) { lo = olo; hi = ohi; }
}
// add / min / max (lo, hi) into the word(s) at w
__device__ __forceinline__ void dense_update(int op, unsigned long long* w, unsigned long long lo, unsigned long long hi) {
  switch (op) {
    case DO_ADD_U64: atomicAdd(w, lo); break;
    case DO_ADD_F64: atomicAdd((double*)w, __longlong_as_double((long long)lo)); break;
    case DO_ADD_128: {   // the carry out of the low word is decided by this add alone
      const unsigned long long old = atomicAdd(w, lo);
      const unsigned long long add_hi = hi + ((old + lo) < old ? 1ull : 0ull);
      if (add_hi) atomicAdd(w + 1, add_hi);
      break;
    }
    case DO_MIN_S64: atomicMin((long long*)w, (long long)lo); break;
    case DO_MAX_S64: atomicMax((long long*)w, (long long)lo); break;
    case DO_MIN_U64: atomicMin(w, lo); break;
    case DO_MAX_U64: atomicMax(w, lo); break;
    case DO_MIN_128: case DO_MAX_128: {
      // w is a generic address: shared memory in the row loop, global memory at the flush
      Rec128 cur = cas128<true>(w, Rec128{lo, hi}, Rec128{lo, hi});   // an atomic read of both words (stores only what is already there)
      while (dense_better(op, lo, hi, cur.lo, cur.hi)) {
        const Rec128 prev = cas128<true>(w, cur, Rec128{lo, hi});
        if (prev.lo == cur.lo && prev.hi == cur.hi) break;
        cur = prev;
      }
      break;
    }
    default: break;
  }
}
// the same for a slot only this lane writes (per-warp copies): a plain read-modify-write
__device__ __forceinline__ void dense_apply(int op, unsigned long long* w, unsigned long long lo, unsigned long long hi) {
  const bool wide = op == DO_ADD_128 || op == DO_MIN_128 || op == DO_MAX_128;
  unsigned long long clo = w[0], chi = wide ? w[1] : 0ull;
  dense_combine(op, clo, chi, lo, hi);
  w[0] = clo;
  if (wide) w[1] = chi;
}
// combine (lo, hi) and the non-null counts over the lanes of each peer group (lanes with the same slot): a tree over the group's
// lanes, log2(group size) shuffle steps; the group's lowest lane ends with the result
__device__ __forceinline__ void dense_reduce_peers(unsigned peers, int op, unsigned long long& lo, unsigned long long& hi, unsigned& cnt) {
  const int lane = threadIdx.x & 31;
  const bool wide = op == DO_ADD_128 || op == DO_MIN_128 || op == DO_MAX_128;   // warp-uniform
  unsigned rel = __popc(peers & ((1u << lane) - 1u));   // rank in the group
  unsigned rest = peers & (0xfffffffeu << lane);          // the group's lanes above this one
  while (__any_sync(0xffffffffu, rest != 0)) {
    const int next = __ffs(rest);                         // the next one still in play (1-based, 0 = none)
    const int src = next ? next - 1 : lane;
    const unsigned long long tlo = __shfl_sync(0xffffffffu, lo, src);
    const unsigned long long thi = wide ? __shfl_sync(0xffffffffu, hi, src) : 0ull;
    const unsigned tc = __shfl_sync(0xffffffffu, cnt, src);
    if (next) { if (op != DO_NONE) dense_combine(op, lo, hi, tlo, thi); cnt += tc; }
    rest &= ~__ballot_sync(0xffffffffu, rel & 1u);        // odd ranks have been read: out of play
    rel >>= 1;
  }
}

template <int SINK, bool DEC, int VAR = 0>
__global__ void __launch_bounds__(kPipeThreads, (((VAR & 64) && SINK == SINK_PACK) || SINK == SINK_DENSE) ? 2 : 3) pipe_kernel(const PipeParams* __restrict__ gp, int64_t n, unsigned long long* __restrict__ counters /* [alive, inserted, fail, err] */) {
  constexpr int PB = kPhaseB, PBG = kPhaseBGroup, QC = kQueueCap;
  constexpr bool RING = (VAR & 64) != 0, PART = (VAR & 128) != 0, FILT = (VAR & kVarFilt) != 0, OUTV = (VAR & kVarOutCols) != 0;
  static_assert(!FILT || !(RING || PART), "stage filters do not run on the ring-fed or partitioned paths");
  static_assert(!OUTV || SINK == SINK_OUTPUT_ANY, "output bitmaps and 16-byte columns belong to the unordered output sink");
  constexpr bool RIGHT = (VAR & kVarRight) != 0;
  static_assert(!RIGHT || (!RING && !PART && !FILT && (SINK == SINK_DENSE || SINK == SINK_HASH || (SINK == SINK_OUTPUT_ANY && OUTV))),
                "RIGHT stages run with the dense, hash and unordered output (bitmap) sinks only");
  constexpr int NX = kMaxStages + (RIGHT ? 1 : 0);   // a row's ext words: the stages' payload words, then (RIGHT) their validity bits
  __shared__ PipeParams sp;
  __shared__ uint32_t q_rows[kPipeWarps][QC];
  extern __shared__ __align__(128) unsigned char dyn_smem[];   // RING: mbarriers [warp][stage], then the rings [warp][stage][ring_bytes]
  for (int i = threadIdx.x; i < (int)(sizeof(PipeParams) / 4); i += kPipeThreads) ((uint32_t*)&sp)[i] = ((const uint32_t*)gp)[i];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  uint64_t* ring_bar = (uint64_t*)dyn_smem + wib * kMaxRingStages;
  if (RING && lane == 0) {
#pragma unroll 1
    for (int s = 0; s < kMaxRingStages; ++s) mbar_init(&ring_bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if constexpr (SINK == SINK_DENSE) {   // dynamic shared memory: DenseParams, then this block's slots
    const uint32_t* src = (const uint32_t*)((const char*)gp + kDenseParamsOff);
    for (int i = threadIdx.x; i < (int)(sizeof(DenseParams) / 4); i += kPipeThreads) ((uint32_t*)dyn_smem)[i] = src[i];
  }
  if constexpr (SINK == SINK_HASH) {   // dynamic shared memory: HashParams
    const uint32_t* src = (const uint32_t*)((const char*)gp + kDenseParamsOff);
    for (int i = threadIdx.x; i < (int)(sizeof(HashParams) / 4); i += kPipeThreads) ((uint32_t*)dyn_smem)[i] = src[i];
  }
  const FiltParams* fpp = nullptr;   // FILT: the stage filters, in dynamic shared memory behind the sink's block
  if constexpr (FILT) {
    const FiltParams* g = (const FiltParams*)((const char*)gp + kFiltParamsOff);
    fpp = (const FiltParams*)(dyn_smem + g->smem_off);
    for (int i = threadIdx.x; i < (int)(sizeof(FiltParams) / 4); i += kPipeThreads) ((uint32_t*)fpp)[i] = ((const uint32_t*)g)[i];
  }
  __syncthreads();
  if constexpr (SINK == SINK_DENSE) {
    const DenseParams& dp = *(const DenseParams*)dyn_smem;
    unsigned long long* sacc = (unsigned long long*)(dyn_smem + kDenseAccOff);
    const int words = (dp.per_warp ? kPipeWarps : 1) * dp.n_slots * dp.n_words;
    for (int i = threadIdx.x; i < words; i += kPipeThreads) sacc[i] = dp.ident[i % dp.n_words];
    __syncthreads();
  }
  const uint64_t pol_stream = (sp.hints & 1) ? policy_evict_first() : policy_normal();
  const uint64_t pol_keep = (sp.hints & 2) ? policy_evict_last() : policy_normal();
  uint32_t* q_row = q_rows[wib];
  unsigned int alive_cnt = 0, ins_cnt = 0;
  int err_ok[2] = {0, 0};
  int fail = 0;
  unsigned int qn = 0;   // queue length (warp-uniform)
  const int64_t ntiles = (n + kWarpTile - 1) / kWarpTile;
  const int64_t gwarp = (int64_t)blockIdx.x * kPipeWarps + wib, nwarps = (int64_t)gridDim.x * kPipeWarps;
  // RING: the warp's i-th tile (gwarp + i nwarps) lives in stage i % S; only full tiles are streamed (bulk copies move multiples of 16 bytes)
  const int S = sp.ring_stages;
  auto ring_stage = [&](int s) { return dyn_smem + kRingBarBytes + (size_t)(wib * S + s) * sp.ring_bytes; };
  auto ring_issue = [&](int64_t t, int s) {
    if (t < ntiles && (t + 1) * kWarpTile <= n) {
      mbar_expect_tx(&ring_bar[s], (uint32_t)sp.ring_bytes);
      unsigned char* dst = ring_stage(s);
#pragma unroll 1
      for (int k = 0; k < sp.ring_n; ++k) {
        const ColRef& c = sp.col[sp.ring_col[k]];
        tma_load_1d_hint(dst + sp.ring_off[sp.ring_col[k]], (const char*)c.ptr + t * kWarpTile * c.width, (uint32_t)(kWarpTile * c.width), &ring_bar[s], pol_stream);
      }
    }
  };
  if (RING && lane == 0) {
#pragma unroll 1
    for (int k = 0; k + 1 < S; ++k) ring_issue(gwarp + k * nwarps, k);
  }
  unsigned int it = 0;     // RING: tiles of this warp so far: stage it % S, mbarrier phase parity (it / S) & 1
  for (int64_t tile = gwarp; tile < ntiles + nwarps; tile += nwarps) {   // one extra trip per warp drains its queue
    const bool draining = tile >= ntiles;
    if (!draining) {
      // =============================== phase A ===============================
      const int64_t row0 = RING ? tile * kWarpTile + lane : tile * kWarpTile + (int64_t)lane * kWarpRows;
      uint32_t mask = 0;
      const unsigned char* stage = nullptr;
      bool full = false;
      if (RING) {
#pragma unroll
        for (int j = 0; j < kWarpRows; ++j) mask |= (uint32_t)(row0 + 32 * j < n) << j;
        const int rs = (int)(it % (unsigned)S);
        if (lane == 0) ring_issue(tile + (int64_t)(S - 1) * nwarps, rs == 0 ? S - 1 : rs - 1);   // the stage the previous tile used: every lane has read it
        full = (tile + 1) * kWarpTile <= n;
        if (full) mbar_wait(&ring_bar[rs], (it / (unsigned)S) & 1u);
        stage = ring_stage(rs);
        ++it;
      } else {
        mask = row0 + kWarpRows <= n ? 0xFFu : (row0 < n ? (1u << (int)(n - row0)) - 1u : 0u);
      }
      if ((VAR & 2) && !RING && sp.n_stages > 0 && row0 < n) {
        const ColRef& kc0 = sp.col[sp.stage[0].key_col];
        prefetch_l2((const char*)kc0.ptr + row0 * kc0.width);
      }
      if (sp.pred_mode == 1) {   // FilterExec, conjunction of `column <cmp> literal`
#pragma unroll 1
        for (int t = 0; t < sp.n_terms; ++t) {
          const ColRef c = sp.col[sp.term_col[t]];
          uint64_t v[kWarpRows];
          if (RING) ring_load8(c, stage + sp.ring_off[sp.term_col[t]], full, row0, n, v, pol_stream);
          else load8<(VAR & 32) != 0>(c, row0, n, v, pol_stream);
          mask &= valid8(c, row0, n);            // a NULL predicate drops the row
          const int op = sp.term_op[t];
          const long long lit = sp.term_lit[t];
          uint32_t lt = 0, eq = 0;
          if (sp.term_uns[t]) {
#pragma unroll
            for (int j = 0; j < kWarpRows; ++j) { lt |= (uint32_t)(v[j] < (uint64_t)lit) << j; eq |= (uint32_t)(v[j] == (uint64_t)lit) << j; }
          } else {
#pragma unroll
            for (int j = 0; j < kWarpRows; ++j) { lt |= (uint32_t)((long long)v[j] < lit) << j; eq |= (uint32_t)((long long)v[j] == lit) << j; }
          }
          uint32_t r;
          switch (op) {
            case DFGPU_OP_EQ: r = eq; break;
            case DFGPU_OP_NEQ: r = ~eq; break;
            case DFGPU_OP_LT: r = lt; break;
            case DFGPU_OP_LTEQ: r = lt | eq; break;
            case DFGPU_OP_GT: r = ~(lt | eq); break;
            default: r = ~lt; break;
          }
          mask &= r;
        }
      } else if (!RING && sp.pred_mode == 2) {   // FilterExec, general expression
#pragma unroll 1
        for (int j = 0; j < kWarpRows; ++j) {
          if (!((mask >> j) & 1u)) continue;
          const uint64_t val = pipe_eval<DEC>(sp.pool + sp.pred_start, sp.pred_n, sp.pred_small, row0 + j, nullptr, err_ok);
          if (!(err_ok[1] && (val & 1))) mask &= ~(1u << j);
        }
      }
      if constexpr (SINK == SINK_DENSE) {   // the conjunction's terms beyond kMaxTerms
        const DenseParams& dp = *(const DenseParams*)dyn_smem;
#pragma unroll 1
        for (int t = 0; t < dp.n_xterms; ++t) {
          const ColRef c = sp.col[dp.xterm_col[t]];
          uint64_t v[kWarpRows];
          load8<false>(c, row0, n, v, pol_stream);
          const long long lit = dp.xterm_lit[t];
          uint32_t lt = 0, eq = 0;
          if (dp.xterm_uns[t]) {
#pragma unroll
            for (int j = 0; j < kWarpRows; ++j) { lt |= (uint32_t)(v[j] < (uint64_t)lit) << j; eq |= (uint32_t)(v[j] == (uint64_t)lit) << j; }
          } else {
#pragma unroll
            for (int j = 0; j < kWarpRows; ++j) { lt |= (uint32_t)((long long)v[j] < lit) << j; eq |= (uint32_t)((long long)v[j] == lit) << j; }
          }
          uint32_t r;
          switch (dp.xterm_op[t]) {
            case DFGPU_OP_EQ: r = eq; break;
            case DFGPU_OP_NEQ: r = ~eq; break;
            case DFGPU_OP_LT: r = lt; break;
            case DFGPU_OP_LTEQ: r = lt | eq; break;
            case DFGPU_OP_GT: r = ~(lt | eq); break;
            default: r = ~lt; break;
          }
          mask &= r & valid8(c, row0, n);
        }
      }
      // bitmap stages decide here; hash stages get their Bloom pre-test (the pushed-down membership filter)
#pragma unroll 1
      for (int s = 0; s < sp.n_stages; ++s) {
        const StageDev& st = sp.stage[s];
        if constexpr (RIGHT) if (st.kind >= kStageRight) continue;   // RIGHT / FULL drop nothing: no NULL-key mask, no membership test
        const bool bitmap = st.lk.mode == LK_BITMAP;
        if constexpr (FILT) if (bitmap && st.kind == DFGPU_STAGE_ANTI && fpp->n[s] > 0) continue;   // a key match alone drops nothing: phase B
        if (!bitmap && !(st.lk.bloom && st.kind != DFGPU_STAGE_ANTI)) {   // nothing cheap to test; NULL keys of an inner / semi stage still drop here
          if (st.kind != DFGPU_STAGE_ANTI && sp.col[st.key_col].valid) mask &= valid8(sp.col[st.key_col], row0, n);
          continue;
        }
        if (!bitmap && st.kind == kStageMaybe && !st.lk.bloom) continue;                                // may-contain without a filter: everything may
        if (!__any_sync(0xffffffffu, mask != 0)) continue;
        const ColRef kc = sp.col[st.key_col];
        uint64_t key[kWarpRows];
        if (RING) ring_load8(kc, stage + sp.ring_off[st.key_col], full, row0, n, key, pol_stream);
        else load8<(VAR & 32) != 0>(kc, row0, n, key, pol_stream);
        const uint32_t kvalid = valid8(kc, row0, n);
        if (bitmap) {
          uint32_t w[kWarpRows];
#pragma unroll
          for (int j = 0; j < kWarpRows; ++j) {
            const uint64_t i = key[j] - st.lk.kmin;
            w[j] = (((mask & kvalid) >> j) & 1u) && i < st.lk.ksize ? __ldg(&st.lk.bits[i >> 5]) : 0u;
          }
          uint32_t found = 0;
#pragma unroll
          for (int j = 0; j < kWarpRows; ++j) found |= ((w[j] >> ((key[j] - st.lk.kmin) & 31)) & 1u) << j;   // NULL keys never match (w = 0)
          mask &= st.kind == DFGPU_STAGE_ANTI ? ~found : found;
        } else {
          if (st.kind != DFGPU_STAGE_ANTI) {
            mask &= kvalid;                      // NULL keys never match
            if (st.lk.coarse) {   // first level: L2-resident, removes most rows before the exact level's DRAM access
              uint32_t cw[kWarpRows], cm[kWarpRows];
#pragma unroll
              for (int j = 0; j < kWarpRows; ++j) {
                const CoarsePos cp = coarse_pos(key[j], st.lk.coarse_words);
                cm[j] = cp.mask;
                cw[j] = ((mask >> j) & 1u) ? __ldg(&st.lk.coarse[cp.word]) : 0u;
              }
              uint32_t cpass = 0;
#pragma unroll
              for (int j = 0; j < kWarpRows; ++j) cpass |= (uint32_t)((cw[j] & cm[j]) == cm[j]) << j;
              mask &= cpass;
            }
            if (st.lk.bloom) {
              unsigned long long bw[kWarpRows];
              uint32_t bt[kWarpRows];
#pragma unroll
              for (int j = 0; j < kWarpRows; ++j) {
                const BloomPos bp = bloom_pos(key[j], st.lk.bloom_blocks);
                bt[j] = bp.t;
                bw[j] = ((mask >> j) & 1u) ? ld_keep_u64(&st.lk.bloom[bp.block], pol_keep) : 0ull;
              }
              uint32_t pass = 0;
#pragma unroll
              for (int j = 0; j < kWarpRows; ++j) pass |= (uint32_t)bloom_test(bw[j], bt[j]) << j;
              mask &= pass;
            }
          }
        }
      }
      // append the survivors to the warp's queue (exclusive scan of the per-lane counts)
      const unsigned int cnt = __popc(mask);
      unsigned int incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
      unsigned int pos = qn + incl - cnt;
#pragma unroll
      for (int j = 0; j < kWarpRows; ++j)
        if ((mask >> j) & 1u) { q_row[pos] = (uint32_t)(row0 + (RING ? 32 : 1) * j); ++pos; }
      qn += __shfl_sync(0xffffffffu, incl, 31);
      __syncwarp();
    }
    // =============================== phase B ===============================
    while (qn >= (unsigned)PBG || (draining && qn > 0)) {
      const unsigned int take = qn >= (unsigned)PBG ? (unsigned)PBG : qn;
      const unsigned int qbase = qn - take;   // consume from the tail: nothing has to move
      bool live[PB];
      int64_t row[PB];
      uint64_t pay[kMaxStages][PB], pkey[PB];   // pkey: PART, the aggregate stage's key
      unsigned long long* arec[PB];
      uint32_t pvalid[PB];                      // RIGHT: bit s = stage s's payload fields are valid (cleared by a RIGHT stage's miss)
#pragma unroll
      for (int u = 0; u < PB; ++u) {
        const unsigned int e = u * 32 + lane;
        live[u] = e < take; row[u] = live[u] ? (int64_t)q_row[qbase + e] : 0; arec[u] = nullptr; pkey[u] = 0;
        if constexpr (RIGHT) pvalid[u] = ~0u;
      }
      if ((VAR & 1) && SINK == SINK_AGG) {
#pragma unroll 1
        for (int a = 0; a < sp.n_aggs; ++a) {
          const AggDef& ag = sp.agg[a];
          if (ag.small != 2) continue;
#pragma unroll 1
          for (int i = 0; i < ag.n; ++i) {
            const ENode& nd = sp.pool[ag.start + i];
            if (nd.kind != DFGPU_EXPR_COLUMN) continue;
            const int w = type_width_prim(nd.out_type);
#pragma unroll
            for (int u = 0; u < PB; ++u) if (live[u]) prefetch_l2((const char*)nd.col + row[u] * w);
          }
        }
      }
      uint64_t g[kGather][PB];   // RING: agg[0]'s column operands, all issued before the stages' table lookups
#pragma unroll
      for (int k = 0; k < kGather; ++k) {
#pragma unroll
        for (int u = 0; u < PB; ++u) g[k][u] = 0;
        if (RING && SINK == SINK_AGG && k < sp.n_gather) {
          const ENode& nd = sp.pool[sp.gather_node[k]];
          if (PART) {   // read once, evict first: the lines around the survivors must not push the Bloom filter out of L2
#pragma unroll
            for (int u = 0; u < PB; ++u) if (live[u]) g[k][u] = ld_stream_int(nd.col, type_width_prim(nd.out_type), type_is_signed_int(nd.out_type) ? 1 : 0, row[u], pol_stream);
          } else
#pragma unroll
          for (int u = 0; u < PB; ++u) if (live[u]) g[k][u] = load_col_value(nd, row[u]);
        }
      }
#pragma unroll
      for (int s = 0; s < kMaxStages; ++s) {
#pragma unroll
        for (int u = 0; u < PB; ++u) pay[s][u] = 0;
        if (s >= sp.n_stages) continue;
        const StageDev& st = sp.stage[s];
        if constexpr (FILT) {
          if (st.lk.mode == LK_BITMAP && fpp->n[s] > 0) {   // phase A kept the matches of an INNER / SEMI stage; an ANTI stage is probed here
#pragma unroll
            for (int u = 0; u < PB; ++u) {
              if (!live[u]) continue;
              bool found = true;
              if (st.kind == DFGPU_STAGE_ANTI) {
                const ColRef& kc = sp.col[st.key_col];
                const uint64_t i = ld_stream_int(kc.ptr, kc.width, kc.sgn, row[u], pol_stream) - st.lk.kmin;
                found = !(kc.valid && !bit_get(kc.valid, kc.voff + row[u])) && i < st.lk.ksize && ((__ldg(&st.lk.bits[i >> 5]) >> (i & 31)) & 1u);
              }
              if (found) {
                uint64_t ext[kMaxStages];
#pragma unroll
                for (int k = 0; k < kMaxStages; ++k) ext[k] = k < s ? pay[k][u] : 0ull;
                found = stage_filter_pass<DEC>(*fpp, s, row[u], ext, err_ok);
              }
              live[u] = st.kind == DFGPU_STAGE_ANTI ? !found : found;
            }
            continue;
          }
        }
        if (st.lk.mode == LK_BITMAP || st.kind == kStageMaybe) continue;   // decided in phase A
        const ColRef kc = sp.col[st.key_col];
        uint64_t key[PB], slot[PB], ck[PB], cp[PB];
        bool look[PB], found[PB];
#pragma unroll
        for (int u = 0; u < PB; ++u) {
          found[u] = false; look[u] = live[u]; key[u] = 0;
          if constexpr (RIGHT) if (st.lk.cap == 0) look[u] = false;   // an empty build side has no table (a Right join keeps its rows)
          if (look[u]) {
            key[u] = ld_stream_int(kc.ptr, kc.width, kc.sgn, row[u], pol_stream);   // streamed in moments ago by phase A: an L2 hit (not for a RIGHT stage, which phase A skips)
            if ((kc.valid && !bit_get(kc.valid, kc.voff + row[u])) || key[u] == kEmptyKey) look[u] = false;   // NULL keys never match
          }
          slot[u] = __umul64hi(lk_hash(key[u]), st.lk.cap); ck[u] = kEmptyKey; cp[u] = 0;
          if (look[u] && !PART) {
            const unsigned long long* r = st.lk.recs + slot[u] * (uint64_t)st.lk.stride;
            if (st.lk.has_payload) { const uint4 v = __ldcg((const uint4*)r); ck[u] = (uint64_t)v.x | ((uint64_t)v.y << 32); cp[u] = (uint64_t)v.z | ((uint64_t)v.w << 32); }
            else ck[u] = __ldcg(r);
          }
        }
        if (PART) {   // the aggregate stage, the only hash stage here: resolved by pipe_probe_agg_kernel (or the sink's fallback below)
#pragma unroll
          for (int u = 0; u < PB; ++u) { pkey[u] = key[u]; live[u] = look[u]; }
          continue;
        }
#pragma unroll
        for (int u = 0; u < PB; ++u) {
          if (look[u]) {
            while (true) {   // linear probing continues only past a foreign key (load factor <= 0.5)
              if (ck[u] == key[u]) { found[u] = true; break; }
              if (ck[u] == kEmptyKey) break;
              if (++slot[u] == st.lk.cap) slot[u] = 0;
              const unsigned long long* r = st.lk.recs + slot[u] * (uint64_t)st.lk.stride;
              if (st.lk.has_payload) { const uint4 v = __ldcg((const uint4*)r); ck[u] = (uint64_t)v.x | ((uint64_t)v.y << 32); cp[u] = (uint64_t)v.z | ((uint64_t)v.w << 32); }
              else ck[u] = __ldcg(r);
            }
            if (found[u]) {
              pay[s][u] = cp[u];
              if constexpr (FILT) {   // a candidate pair the filter rejects is no match: a LEFT stage's record is not touched
                uint64_t ext[kMaxStages];
#pragma unroll
                for (int k = 0; k < kMaxStages; ++k) ext[k] = k <= s ? pay[k][u] : 0ull;
                found[u] = stage_filter_pass<DEC>(*fpp, s, row[u], ext, err_ok);
              }
              if (SINK == SINK_AGG && s == sp.agg_stage && (!FILT || found[u])) arec[u] = st.lk.recs + slot[u] * (uint64_t)st.lk.stride;
            }
          }
          if constexpr (RIGHT) if (st.kind >= kStageRight) { if (!found[u]) pvalid[u] &= ~(1u << s); continue; }   // keeps the row
          live[u] = live[u] && (st.kind == DFGPU_STAGE_ANTI ? !found[u] : found[u]);
        }
        if constexpr (RIGHT) if (st.kind == kStageFull) {   // a FULL stage's matches mark their records
#pragma unroll
          for (int u = 0; u < PB; ++u) if (found[u]) mark_visited(st.lk.recs + slot[u] * (uint64_t)st.lk.stride);
        }
      }
      // ---- sink ----
      if (SINK == SINK_OUTPUT_ANY) {   // rows leave in arrival order: one global reservation per 128-row group, coalesced column writes
        unsigned int tot = 0, mypos[PB];
#pragma unroll
        for (int u = 0; u < PB; ++u) { const unsigned m = __ballot_sync(0xffffffffu, live[u]); mypos[u] = tot + __popc(m & ((1u << lane) - 1u)); tot += __popc(m); }
        unsigned long long obase = 0;
        if (lane == 0 && tot) obase = atomicAdd(sp.out_counter, (unsigned long long)tot);
        obase = __shfl_sync(0xffffffffu, obase, 0);
#pragma unroll
        for (int u = 0; u < PB; ++u) {
          if (!live[u]) continue;
          alive_cnt++;
          for (int c = 0; c < sp.n_out; ++c) {
            const int src = sp.out_src[c], w = sp.out_width[c];
            if (OUTV && w == 16) { copy16(sp.col[src], row[u], (char*)sp.out_dst[c] + (obase + mypos[u]) * 16, pol_stream); continue; }   // inputs only
            uint64_t v;
            if (src < sp.n_cols) v = ld_stream_int(sp.col[src].ptr, w, 0, row[u], pol_stream);
            else { const ExtDef e = sp.ext[src - sp.n_cols]; uint64_t wd = 0;
#pragma unroll
                   for (int s = 0; s < kMaxStages; ++s) if (s == e.stage) wd = pay[s][u];
                   v = ext_field(wd, e.shift, e.width, DFGPU_UINT64); }
            const unsigned long long o = obase + mypos[u];
            switch (w) {
              case 1: ((uint8_t*)sp.out_dst[c])[o] = (uint8_t)v; break;
              case 2: ((uint16_t*)sp.out_dst[c])[o] = (uint16_t)v; break;
              case 4: ((uint32_t*)sp.out_dst[c])[o] = (uint32_t)v; break;
              default: ((uint64_t*)sp.out_dst[c])[o] = v; break;
            }
          }
        }
        if constexpr (OUTV) {   // the live lanes of item u hold the lane-ordered range [obase + at, obase + at + popc(m)): at most two words
          const OutValid* ov = (const OutValid*)((const char*)gp + kDenseParamsOff);
          unsigned int at = 0;
#pragma unroll
          for (int u = 0; u < PB; ++u) {
            const unsigned m = __ballot_sync(0xffffffffu, live[u]);
            const unsigned rank = __popc(m & ((1u << lane) - 1u));
            const unsigned long long start = obase + at;
#pragma unroll 1
            for (int c = 0; m && c < sp.n_out; ++c) {
              uint32_t* dv = ov->valid[c];
              if (!dv) continue;
              unsigned bits;
              if constexpr (RIGHT) {   // a payload field's bit: its stage matched
                const int src = sp.out_src[c];
                const bool ok = live[u] && (src < sp.n_cols ? bit_get(sp.col[src].valid, sp.col[src].voff + row[u]) : ((pvalid[u] >> sp.ext[src - sp.n_cols].stage) & 1u) != 0);
                bits = __reduce_or_sync(0xffffffffu, ok ? 1u << rank : 0u);
              } else {
                const ColRef& col = sp.col[sp.out_src[c]];
                bits = __reduce_or_sync(0xffffffffu, live[u] && bit_get(col.valid, col.voff + row[u]) ? 1u << rank : 0u);
              }
              const int sh = (int)(start & 31);
              if (lane == 0 && bits) {
                atomicOr(dv + (start >> 5), bits << sh);
                if (sh && (bits >> (32 - sh))) atomicOr(dv + (start >> 5) + 1, bits >> (32 - sh));
              }
            }
            at += __popc(m);
          }
        }
      }
      bool sunk = false;
      if (PART && SINK == SINK_AGG) {
        // {key, value} records through one reservation per warp and round; no table access.  A Bloom false positive costs one record
        // (its key finds no partner later).  Reservations past the buffer's end (target.cap records) probe and RED here instead.
        sunk = true;
        const AggDef& ag0 = sp.agg[0];
        unsigned int tot = 0, mypos[PB];
#pragma unroll
        for (int u = 0; u < PB; ++u) { const unsigned m = __ballot_sync(0xffffffffu, live[u]); mypos[u] = tot + __popc(m & ((1u << lane) - 1u)); tot += __popc(m); }
        unsigned long long obase = 0;
        if (lane == 0 && tot) obase = atomicAdd(sp.out_counter, (unsigned long long)tot);
        obase = __shfl_sync(0xffffffffu, obase, 0);
#pragma unroll
        for (int u = 0; u < PB; ++u) {
          if (!live[u]) continue;
          const uint64_t ext[kMaxStages] = {0, 0, 0};   // the program reads no payload field (partitioned_parts)
          const unsigned long long v = eval_int_gathered(sp.pool + ag0.start, ag0.n, row[u], ext, sp.n_gather, g[0][u], g[1][u]);
          const unsigned long long o = obase + mypos[u];
          if (o < sp.target.cap) {
            st_stream_u64((unsigned long long*)sp.out_dst[0] + o, pkey[u], pol_stream);   // the records, too, are read again only after this pass
            st_stream_u64((unsigned long long*)sp.out_dst[1] + o, v, pol_stream);
            continue;
          }
          const LookupDev& lk = sp.stage[sp.agg_stage].lk;
          uint64_t slot = __umul64hi(lk_hash(pkey[u]), lk.cap);
          while (true) {
            unsigned long long* r = lk.recs + slot * (uint64_t)lk.stride;
            const unsigned long long ck = __ldcg(r);
            if (ck == pkey[u]) { red_add_u64(r + sp.rows_word, 1ull); red_add_u64(r + ag0.word, v); alive_cnt++; break; }
            if (ck == kEmptyKey) break;
            if (++slot == lk.cap) slot = 0;
          }
        }
      }
      if ((VAR & 8) && SINK == SINK_AGG) {
        // one RED instruction per lane PAIR and row: the row counter and the sum word of a record share a sector, so the even lane adds
        // its row's count while the odd neighbour adds the same row's value (then the roles swap) — half the L2 reduction requests
        const AggDef& ag0 = sp.agg[0];
        if (sp.n_aggs == 1 && ag0.small == 2 && ag0.func == DFGPU_AGG_SUM && ag0.cls != C_F64 && ag0.cls != C_DEC && ag0.nn_word < 0) {
          sunk = true;
          const bool even = !(lane & 1);
#pragma unroll
          for (int u = 0; u < PB; ++u) {
            uint64_t ext[kMaxStages];
#pragma unroll
            for (int s = 0; s < kMaxStages; ++s) ext[s] = pay[s][u];
            unsigned long long v = 0;
            if (live[u]) {
              alive_cnt++;
              v = RING ? eval_int_gathered(sp.pool + ag0.start, ag0.n, row[u], ext, sp.n_gather, g[0][u], g[1][u])
                       : eval_int_fast(sp.pool + ag0.start, ag0.n, row[u], ext);
            }
            __syncwarp();
            const unsigned long long rp = (unsigned long long)arec[u];
            const unsigned long long prp = __shfl_xor_sync(0xffffffffu, rp, 1);
            const unsigned long long pv = __shfl_xor_sync(0xffffffffu, v, 1);
            const bool pl = __shfl_xor_sync(0xffffffffu, live[u] ? 1 : 0, 1) != 0;
            unsigned long long* const mine = (unsigned long long*)rp + sp.rows_word;    // this lane's row: the row counter
            unsigned long long* const theirs = (unsigned long long*)prp + ag0.word;     // the neighbour's row: the sum
            if (even ? live[u] : pl) red_add_u64(even ? mine : theirs, even ? 1ull : pv);     // rows of the even lanes
            if (even ? pl : live[u]) red_add_u64(even ? theirs : mine, even ? pv : 1ull);     // rows of the odd lanes
          }
        }
      }
      if constexpr (SINK == SINK_DENSE) {   // every lane takes part in each step: the combining is warp-collective
        const DenseParams& dp = *(const DenseParams*)dyn_smem;
        unsigned long long* sacc = (unsigned long long*)(dyn_smem + kDenseAccOff);
#pragma unroll 1
        for (int u = 0; u < PB; ++u) {
          if (!__any_sync(0xffffffffu, live[u])) continue;
          uint64_t ext[NX];
#pragma unroll
          for (int s = 0; s < kMaxStages; ++s) ext[s] = pay[s][u];
          if constexpr (RIGHT) ext[kExtValid] = pvalid[u];
          int slot = -1;
          if (live[u]) {
            alive_cnt++;
            unsigned long long sl = 0;
            bool inside = true;
#pragma unroll 1
            for (int k = 0; k < dp.n_keys; ++k) {
              const DenseKey& dk = dp.key[k];
              bool isnull = false;
              uint64_t key;
              if (dk.src < sp.n_cols) {
                const ColRef& c = sp.col[dk.src];
                isnull = c.valid && !bit_get(c.valid, c.voff + row[u]);
                key = isnull ? 0ull : ld_stream_int(c.ptr, c.width, c.sgn, row[u], pol_stream);
              } else {
                const ExtDef e = sp.ext[dk.src - sp.n_cols];
                uint64_t wd = 0;
#pragma unroll
                for (int s = 0; s < kMaxStages; ++s) if (s == e.stage) wd = ext[s];
                key = ext_field(wd, e.shift, e.width, e.type);
                if constexpr (RIGHT) isnull = !((pvalid[u] >> e.stage) & 1u);
              }
              const uint64_t idx = isnull ? dk.nvals : key - dk.kmin;   // modular: one unsigned compare checks both bounds
              if (idx > dk.nvals || (!isnull && idx == dk.nvals)) { inside = false; break; }
              sl += idx * dk.stride;
            }
            if (inside) slot = (int)sl;
            else fail |= 2;                                            // a key outside its declared range
          }
          const unsigned peers = __match_any_sync(0xffffffffu, slot);
          const bool lead = slot >= 0 && lane == __ffs(peers) - 1;
          unsigned long long* const sw = sacc + ((size_t)(dp.per_warp ? wib * dp.n_slots : 0) + (slot < 0 ? 0 : slot)) * dp.n_words;
          if (lead) {   // word 0: the group's rows (COUNT(*))
            if (dp.per_warp) sw[0] += (unsigned long long)__popc(peers);
            else atomicAdd(sw, (unsigned long long)__popc(peers));
          }
#pragma unroll 1
          for (int a = 0; a < dp.n_aggs; ++a) {
            const DenseAgg& ag = dp.agg[a];
            if (ag.func == DFGPU_AGG_COUNT_STAR) continue;
            unsigned long long lo = 0, hi = 0;
            unsigned ok = 0;
            if (slot >= 0) {
              if (ag.small == 2) { lo = eval_int_fast(sp.pool + ag.start, ag.n, row[u], ext); ok = 1; }
              else if (DEC && ag.small == 3) { lo = pipe_eval_dec<RIGHT>(sp.pool + ag.start, ag.n, row[u], ext, err_ok, &hi); ok = err_ok[1] ? 1 : 0; }
              else { lo = pipe_eval<DEC, RIGHT>(sp.pool + ag.start, ag.n, ag.small, row[u], ext, err_ok); ok = err_ok[1] ? 1 : 0; }
              if (ag.f64_key) lo = f64_to_ordered(__longlong_as_double((long long)lo));
            }
            if (!ok && ag.word >= 0) { lo = dp.ident[ag.word]; hi = ag.op == DO_MIN_128 || ag.op == DO_MAX_128 ? dp.ident[ag.word + 1] : 0ull; }
            dense_reduce_peers(peers, ag.op, lo, hi, ok);
            if (lead && ok) {
              if (dp.per_warp) {
                if (ag.nn_word >= 0) sw[ag.nn_word] += (unsigned long long)ok;
                if (ag.op != DO_NONE) dense_apply(ag.op, sw + ag.word, lo, hi);
              } else {
                if (ag.nn_word >= 0) atomicAdd(sw + ag.nn_word, (unsigned long long)ok);
                dense_update(ag.op, sw + ag.word, lo, hi);
              }
            }
          }
          __syncwarp();   // per-warp copies: this round's stores are seen by the next round's leaders
        }
      }
      if constexpr (SINK == SINK_HASH) {   // the record of each survivor's packed group tag; a deferred row leaves the round untouched
        const HashParams& hp = *(const HashParams*)dyn_smem;
#pragma unroll
        for (int u = 0; u < PB; ++u) {
          if (!live[u]) continue;
          u128 tag = 0;
#pragma unroll 1
          for (int k = 0; k < hp.n_keys; ++k) {
            const HashKey& hk = hp.key[k];
            bool isnull = false;
            uint64_t v;
            if (hk.src < sp.n_cols) {
              const ColRef& c = sp.col[hk.src];
              isnull = c.valid && !bit_get(c.valid, c.voff + row[u]);
              v = isnull ? 0ull : ld_stream_int(c.ptr, c.width, 0, row[u], pol_stream);
            } else {
              const ExtDef e = sp.ext[hk.src - sp.n_cols];
              uint64_t wd = 0;
#pragma unroll
              for (int s = 0; s < kMaxStages; ++s) if (s == e.stage) wd = pay[s][u];
              v = ext_field(wd, e.shift, e.width, DFGPU_UINT64);
              if constexpr (RIGHT) isnull = !((pvalid[u] >> e.stage) & 1u);   // v is 0 then: the payload word of a miss
            }
            if (isnull && hk.null_bit < 0) fail |= 4;   // a NULL in a column declared non-nullable
            if (hk.bits < 64) v &= (1ull << hk.bits) - 1ull;
            tag |= (u128)v << hk.shift;
            if (isnull && hk.null_bit >= 0) tag |= (u128)1 << hk.null_bit;
          }
          arec[u] = hash_find_or_claim(hp, (uint64_t)tag, (uint64_t)(tag >> 64));
          if (!arec[u]) { hp.overflow[atomicAdd(hp.overflow_count, 1ull)] = (uint32_t)row[u]; live[u] = false; }
        }
      }
#pragma unroll
      for (int u = 0; u < PB; ++u) {
        if (SINK == SINK_OUTPUT_ANY || SINK == SINK_DENSE || sunk) break;
        uint64_t ext[NX];
#pragma unroll
        for (int s = 0; s < kMaxStages; ++s) ext[s] = pay[s][u];
        if constexpr (RIGHT) ext[kExtValid] = pvalid[u];
        if (!live[u]) continue;
        alive_cnt++;
        if (SINK == SINK_BUILD || SINK == SINK_PACK) {
          const ColRef kc = sp.col[sp.bkey_col];
          if (kc.valid && !bit_get(kc.valid, kc.voff + row[u])) continue;   // NULL build keys are not inserted (utils.rs:2146-2155)
          const uint64_t key = ld_stream_int(kc.ptr, kc.width, kc.sgn, row[u], pol_stream);
          uint64_t p = 0;
          for (int c = 0; c < sp.n_bpay; ++c) {
            const int src = sp.bpay_src[c];
            uint64_t v;
            if (src < sp.n_cols) v = ld_stream_int(sp.col[src].ptr, sp.col[src].width, 0, row[u], pol_stream);
            else { const ExtDef e = sp.ext[src - sp.n_cols]; v = ext_field(ext[e.stage], e.shift, e.width, DFGPU_UINT64); }
            if (sp.bpay_width[c] < 8) v &= (1ull << (8 * sp.bpay_width[c])) - 1ull;
            p |= v << sp.bpay_shift[c];
          }
          if (SINK == SINK_PACK) {   // one reservation per warp and round (the lanes still active here), coalesced 16-byte stores
            const unsigned am = __activemask();
            const int leader = __ffs(am) - 1;
            unsigned long long o = 0;
            if (lane == leader) o = atomicAdd(sp.out_counter, (unsigned long long)__popc(am));
            o = __shfl_sync(am, o, leader) + __popc(am & ((1u << lane) - 1u));
            ((ulonglong2*)sp.out_dst[0])[o] = make_ulonglong2(key, p);
            ins_cnt++;
          } else {
            const int rc = lk_insert(sp.target, key, p);
            if (rc == 0) ins_cnt++;
            else if (rc == 2 || sp.target_unique) fail |= rc;
          }
        } else if (SINK == SINK_AGG || SINK == SINK_HASH) {
          unsigned long long* rec = arec[u];
          red_add_u64(rec + sp.rows_word, 1ull);
          for (int a = 0; a < sp.n_aggs; ++a) {
            const AggDef ag = sp.agg[a];
            if (ag.func == DFGPU_AGG_COUNT_STAR) continue;   // = the row counter
            uint64_t v;
            if (ag.small == 2) v = RING && a == 0 ? eval_int_gathered(sp.pool + ag.start, ag.n, row[u], ext, sp.n_gather, g[0][u], g[1][u])
                                                  : eval_int_fast(sp.pool + ag.start, ag.n, row[u], ext);
            else if (DEC && ag.cls == C_DEC && ag.func != DFGPU_AGG_COUNT) {
              unsigned long long* nn = ag.nn_word >= 0 ? rec + ag.nn_word : nullptr;   // AVG: its count word
              if (ag.func == DFGPU_AGG_MIN || ag.func == DFGPU_AGG_MAX) pipe_minmax_dec<RIGHT>(sp.pool + ag.start, ag.n, row[u], ext, err_ok, rec + ag.word, nn, ag.func == DFGPU_AGG_MIN);
              else pipe_sum_dec<RIGHT>(sp.pool + ag.start, ag.n, row[u], ext, err_ok, rec + ag.word, nn);   // SUM, and the sum of AVG
              continue;
            } else {
              if (RING) { atomicOr(&counters[3], (unsigned long long)kErrRingAgg); continue; }   // fill_ring admits integer programs and COUNT(*) only
              v = pipe_eval<DEC, RIGHT>(sp.pool + ag.start, ag.n, ag.small, row[u], ext, err_ok);
              if (!err_ok[1]) continue;                      // NULL inputs are skipped (accumulate.rs:373-470)
            }
            if (ag.nn_word >= 0) red_add_u64(rec + ag.nn_word, 1ull);
            switch (ag.func) {
              case DFGPU_AGG_COUNT: red_add_u64(rec + ag.word, 1ull); break;
              case DFGPU_AGG_SUM: case DFGPU_AGG_AVG:
                if (ag.cls == C_F64) red_add_f64(rec + ag.word, __longlong_as_double((long long)v));
                else red_add_u64(rec + ag.word, (unsigned long long)v);   // add_wrapping (sum.rs:316)
                break;
              case DFGPU_AGG_MIN:
                if (ag.cls == C_F64) red_min_u64(rec + ag.word, f64_to_ordered(__longlong_as_double((long long)v)));
                else if (ag.cls == C_U64) red_min_u64(rec + ag.word, (unsigned long long)v);
                else red_min_s64(rec + ag.word, (long long)v);
                break;
              case DFGPU_AGG_MAX:
                if (ag.cls == C_F64) red_max_u64(rec + ag.word, f64_to_ordered(__longlong_as_double((long long)v)));
                else if (ag.cls == C_U64) red_max_u64(rec + ag.word, (unsigned long long)v);
                else red_max_s64(rec + ag.word, (long long)v);
                break;
            }
          }
        }
      }
      qn = qbase;
      __syncwarp();
    }
  }
  if constexpr (SINK == SINK_DENSE) {   // flush: this block's slots into the pipeline's accumulators, one thread per slot
    __syncthreads();
    const DenseParams& dp = *(const DenseParams*)dyn_smem;
    unsigned long long* sacc = (unsigned long long*)(dyn_smem + kDenseAccOff);
    for (int s = threadIdx.x; s < dp.n_slots; s += kPipeThreads) {
      unsigned long long* w = sacc + (size_t)s * dp.n_words;
#pragma unroll 1
      for (int c = 1; dp.per_warp && c < kPipeWarps; ++c) {   // fold the other warps' copies of this slot into warp 0's
        const unsigned long long* o = w + (size_t)c * dp.n_slots * dp.n_words;
        if (o[0] == 0ull) continue;
        w[0] += o[0];
#pragma unroll 1
        for (int a = 0; a < dp.n_aggs; ++a) {
          const DenseAgg& ag = dp.agg[a];
          if (ag.nn_word >= 0) {
            if (o[ag.nn_word] == 0ull) continue;
            w[ag.nn_word] += o[ag.nn_word];
          }
          const bool wide = ag.op == DO_ADD_128 || ag.op == DO_MIN_128 || ag.op == DO_MAX_128;
          if (ag.op != DO_NONE) dense_apply(ag.op, w + ag.word, o[ag.word], wide ? o[ag.word + 1] : 0ull);
        }
      }
      if (w[0] == 0ull) continue;
      unsigned long long* g = dp.acc + (size_t)s * dp.n_words;
      atomicAdd(g, w[0]);
#pragma unroll 1
      for (int a = 0; a < dp.n_aggs; ++a) {
        const DenseAgg& ag = dp.agg[a];
        if (ag.nn_word >= 0) {
          if (w[ag.nn_word] == 0ull) continue;   // no value: the slot's word still holds the identity
          atomicAdd(g + ag.nn_word, w[ag.nn_word]);
        }
        if (ag.op == DO_NONE) continue;
        const bool wide = ag.op == DO_ADD_128 || ag.op == DO_MIN_128 || ag.op == DO_MAX_128;
        dense_update(ag.op, g + ag.word, w[ag.word], wide ? w[ag.word + 1] : 0ull);
      }
    }
  }
  // block-level counter reduction: one atomic per block and counter
  __shared__ unsigned int s_red[2][kPipeWarps];
  __shared__ int s_flag[2];
  if (threadIdx.x == 0) { s_flag[0] = 0; s_flag[1] = 0; }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { alive_cnt += __shfl_xor_sync(0xffffffffu, alive_cnt, d); ins_cnt += __shfl_xor_sync(0xffffffffu, ins_cnt, d); }
  __syncthreads();
  if (lane == 0) { s_red[0][wib] = alive_cnt; s_red[1][wib] = ins_cnt; }
  if (fail) atomicOr(&s_flag[0], fail);
  if (err_ok[0]) atomicOr(&s_flag[1], err_ok[0]);
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long a = 0, b = 0;
    for (int w = 0; w < kPipeWarps; ++w) { a += s_red[0][w]; b += s_red[1][w]; }
    if (a) atomicAdd(&counters[0], a);
    if (b) atomicAdd(&counters[1], b);
    if (s_flag[0]) atomicOr(&counters[2], (unsigned long long)s_flag[0]);
    if (s_flag[1]) atomicOr(&counters[3], (unsigned long long)s_flag[1]);
  }
}

// ------------------------------------------------------------------------------------------
// partitioned aggregate, second half: the {key, value} records of pipe_kernel VAR bit 128, radix-partitioned (radix_partition), probe the
// aggregate stage's table and RED into the matched record.  Tiles are taken in record order from one counter, so the running blocks
// share one ~16 MB slot range of the table and its lookups and REDs are L2 hits instead of DRAM misses (radix_probe_kernel's scheme).
// Matches add to counters[0], the sink's row count.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pipe_probe_agg_kernel(const ulonglong2* __restrict__ recs, int64_t n, LookupDev t, int rows_word, int sum_word,
                                                             unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ counters) {
  constexpr int ITEMS = 4, TILE = 256 * ITEMS;
  __shared__ unsigned int s_tile;
  const int lane = threadIdx.x & 31;
  const bool even = !(lane & 1);
  const int64_t ntiles = (n + TILE - 1) / TILE;
  unsigned int hits = 0;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);   // tiles in record order: the running blocks share one sub-table
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;
    unsigned long long key[ITEMS], val[ITEMS], slot[ITEMS], cur[ITEMS];
    unsigned pend = 0, hit = 0;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int64_t i = tile * TILE + k * 256 + threadIdx.x;
      key[k] = kEmptyKey; val[k] = 0; cur[k] = kEmptyKey;
      if (i < n) { const int4 r = ld_stream_16(recs + i); key[k] = (uint64_t)(uint32_t)r.x | ((uint64_t)(uint32_t)r.y << 32); val[k] = (uint64_t)(uint32_t)r.z | ((uint64_t)(uint32_t)r.w << 32); }
      slot[k] = __umul64hi(lk_hash(key[k]), t.cap);
      if (i < n) { cur[k] = __ldcg(t.recs + slot[k] * (uint64_t)t.stride); pend |= 1u << k; }
    }
    // lockstep linear probing: the (rare) second probes of the thread's rows overlap
    while (pend) {
#pragma unroll
      for (int k = 0; k < ITEMS; ++k) {
        if (!((pend >> k) & 1u)) continue;
        if (cur[k] == key[k]) { hit |= 1u << k; pend &= ~(1u << k); }
        else if (cur[k] == kEmptyKey) pend &= ~(1u << k);
        else {
          if (++slot[k] == t.cap) slot[k] = 0;
          cur[k] = __ldcg(t.recs + slot[k] * (uint64_t)t.stride);
        }
      }
    }
    // lane-paired REDs (pipe_kernel VAR bit 3): the even lane adds its row's count while the odd neighbour adds the same row's value
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const bool h = (hit >> k) & 1u;
      hits += h ? 1u : 0u;
      const unsigned long long rp = h ? (unsigned long long)(t.recs + slot[k] * (uint64_t)t.stride) : 0ull;
      const unsigned long long prp = __shfl_xor_sync(0xffffffffu, rp, 1);
      const unsigned long long pv = __shfl_xor_sync(0xffffffffu, val[k], 1);
      const bool pl = __shfl_xor_sync(0xffffffffu, h ? 1 : 0, 1) != 0;
      unsigned long long* const mine = (unsigned long long*)rp + rows_word;
      unsigned long long* const theirs = (unsigned long long*)prp + sum_word;
      if (even ? h : pl) red_add_u64(even ? mine : theirs, even ? 1ull : pv);
      if (even ? pl : h) red_add_u64(even ? theirs : mine, even ? pv : 1ull);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, d);
  if (lane == 0 && hits) atomicAdd(&counters[0], (unsigned long long)hits);
}

// ------------------------------------------------------------------------------------------
// output sink: surviving rows in input order (ordered compaction: block scan + decoupled look-back, as filter_fused_kernel)
// ------------------------------------------------------------------------------------------
struct OutCols { int n; int src[kMaxPipeCols]; int width[kMaxPipeCols]; void* dst[kMaxPipeCols]; };

// FILT: the stage filters (FiltParams at offset 0 of the dynamic shared memory), evaluated on each candidate pair with the interpreter of
// pipe_kernel's DEC instantiations.  COLS: output columns with bitmaps or 16 bytes wide (OutValid behind PipeParams; pipe_output_cols_kernel).
// RIGHT (with COLS, without FILT): RIGHT stages keep every row; each survivor's payload validity bits (bit s = stage s matched) are staged
// in the dynamic shared memory next to s_pay, and a RIGHT payload column's bitmap takes them (pipe_output_right_kernel)
template <bool FILT, bool COLS, bool RIGHT = false>
__device__ __forceinline__ void pipe_output_tile(const PipeParams* __restrict__ gp, int64_t n, const OutCols& oc, unsigned long long* __restrict__ tile_desc,
                                                 unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ totals, unsigned long long* __restrict__ counters) {
  __shared__ PipeParams sp;
  __shared__ uint32_t s_p[kPipeTile];
  __shared__ unsigned long long s_pay[kMaxStages][kPipeTile];
  __shared__ unsigned int s_tile;
  __shared__ unsigned long long s_base;
  extern __shared__ __align__(128) unsigned char dyn_smem[];
  for (int i = threadIdx.x; i < (int)(sizeof(PipeParams) / 4); i += kPipeThreads) ((uint32_t*)&sp)[i] = ((const uint32_t*)gp)[i];
  if constexpr (FILT) {
    const uint32_t* src = (const uint32_t*)((const char*)gp + kFiltParamsOff);
    for (int i = threadIdx.x; i < (int)(sizeof(FiltParams) / 4); i += kPipeThreads) ((uint32_t*)dyn_smem)[i] = src[i];
  }
  if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);
  __syncthreads();
  const int64_t tile = s_tile;
  const int64_t row0 = tile * kPipeTile + (int64_t)threadIdx.x * kPipeItems;   // consecutive rows per thread: rank order == row order
  static_assert(!RIGHT || (COLS && !FILT), "RIGHT stages: output bitmaps, no stage filters");
  int err = 0;
  bool alive[kPipeItems];
  uint64_t pay[kMaxStages][kPipeItems];
  uint32_t pvalid[kPipeItems];   // RIGHT: bit s = stage s's payload fields are valid
#pragma unroll
  for (int k = 0; k < kPipeItems; ++k) {
    const int64_t row = row0 + k;
    alive[k] = row < n;
    if constexpr (RIGHT) pvalid[k] = ~0u;
#pragma unroll
    for (int s = 0; s < kMaxStages; ++s) pay[s][k] = 0;
    if (!alive[k]) continue;
    if (sp.pred_mode == 1) {
      for (int t = 0; t < sp.n_terms && alive[k]; ++t) {
        const ColRef c = sp.col[sp.term_col[t]];
        if (c.valid && !bit_get(c.valid, c.voff + row)) { alive[k] = false; break; }
        const uint64_t v = ld_stream_int(c.ptr, c.width, c.sgn, row, policy_evict_first());
        const long long lit = sp.term_lit[t];
        int cmp;
        if (sp.term_uns[t]) cmp = v < (uint64_t)lit ? -1 : (v > (uint64_t)lit ? 1 : 0);
        else cmp = (long long)v < lit ? -1 : ((long long)v > lit ? 1 : 0);
        switch (sp.term_op[t]) {
          case DFGPU_OP_EQ: alive[k] = cmp == 0; break;
          case DFGPU_OP_NEQ: alive[k] = cmp != 0; break;
          case DFGPU_OP_LT: alive[k] = cmp < 0; break;
          case DFGPU_OP_LTEQ: alive[k] = cmp <= 0; break;
          case DFGPU_OP_GT: alive[k] = cmp > 0; break;
          default: alive[k] = cmp >= 0; break;
        }
      }
    } else if (sp.pred_mode == 2) {
      bool ok;
      uint64_t val;
      if (sp.pred_small == 3) {   // Decimal128 nodes: the 128-bit interpreter, as in pipe_kernel's DEC instantiations
        int eo[2] = {0, 0};
        val = pipe_eval<true>(sp.pool + sp.pred_start, sp.pred_n, 3, row, nullptr, eo);
        err |= eo[0]; ok = eo[1] != 0;
      } else {
        val = eval_nodes(sp.pool + sp.pred_start, sp.pred_n, row, &ok, &err);
      }
      alive[k] = ok && (val & 1);
    }
  }
#pragma unroll
  for (int s = 0; s < kMaxStages; ++s) {
    if (s >= sp.n_stages) continue;
    const StageDev& st = sp.stage[s];
    const ColRef kc = sp.col[st.key_col];
#pragma unroll
    for (int k = 0; k < kPipeItems; ++k) {
      if (!alive[k]) continue;
      const int64_t row = row0 + k;
      bool found = false;
      const bool knull = kc.valid && !bit_get(kc.valid, kc.voff + row);
      const uint64_t key = ld_stream_int(kc.ptr, kc.width, kc.sgn, row, policy_evict_first());
      if (!knull) {
        if (st.lk.mode == LK_BITMAP) {
          const uint64_t i = key - st.lk.kmin;
          found = i < st.lk.ksize && ((__ldg(&st.lk.bits[i >> 5]) >> (i & 31)) & 1u);
        } else if (key != kEmptyKey && (!RIGHT || st.lk.cap > 0)) {   // RIGHT: an empty build side has no table
          const uint64_t h = lk_hash(key);
          bool maybe = true;
          if (st.lk.coarse) { const CoarsePos cp = coarse_pos(key, st.lk.coarse_words); maybe = (st.lk.coarse[cp.word] & cp.mask) == cp.mask; }
          if (maybe && st.lk.bloom) { const BloomPos bp = bloom_pos(key, st.lk.bloom_blocks); maybe = bloom_test(st.lk.bloom[bp.block], bp.t); }
          if (maybe) {
            uint64_t slot = __umul64hi(h, st.lk.cap);
            while (true) {
              const unsigned long long* r = st.lk.recs + slot * (uint64_t)st.lk.stride;
              const unsigned long long ck = __ldcg(r);
              if (ck == key) {
                found = true;
                if (st.lk.has_payload) pay[s][k] = __ldcg(r + 1);
                if constexpr (RIGHT) if (st.kind == kStageFull) mark_visited(st.lk.recs + slot * (uint64_t)st.lk.stride);
                break;
              }
              if (ck == kEmptyKey) break;
              if (++slot == st.lk.cap) slot = 0;
            }
          }
        }
      }
      if constexpr (FILT) {
        if (found) {
          uint64_t ext[kMaxStages];
#pragma unroll
          for (int q = 0; q < kMaxStages; ++q) ext[q] = pay[q][k];
          int eo[2] = {err, 0};
          found = stage_filter_pass<true>(*(const FiltParams*)dyn_smem, s, row, ext, eo);
          err = eo[0];
        }
      }
      if constexpr (RIGHT) if (st.kind >= kStageRight) { if (!found) pvalid[k] &= ~(1u << s); continue; }   // keeps the row
      alive[k] = st.kind == DFGPU_STAGE_ANTI ? !found : found;
    }
  }
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < kPipeItems; ++k) m += alive[k] ? 1u : 0u;
  uint32_t tot;
  uint32_t ex = block_exclusive_scan<kPipeThreads, uint32_t>(m, &tot);
#pragma unroll
  for (int k = 0; k < kPipeItems; ++k)
    if (alive[k]) {
      s_p[ex] = (uint32_t)(threadIdx.x * kPipeItems + k);
#pragma unroll
      for (int s = 0; s < kMaxStages; ++s) s_pay[s][ex] = pay[s][k];
      if constexpr (RIGHT) dyn_smem[ex] = (unsigned char)pvalid[k];
      ++ex;
    }
  if (threadIdx.x < 32) {
    unsigned long long exclusive = tile_lookback(tile, tot, tile_desc);
    if (threadIdx.x == 0) {
      s_base = exclusive;
      if ((tile + 1) * (int64_t)kPipeTile >= n) totals[0] = exclusive + tot;
    }
  }
  __syncthreads();
  const unsigned long long obase = s_base;
  const int64_t prow0 = tile * kPipeTile;
  for (int c = 0; c < oc.n; ++c) {
    const int src = oc.src[c], w = oc.width[c];
    for (uint32_t j = threadIdx.x; j < tot; j += kPipeThreads) {
      if (COLS && w == 16) { copy16(sp.col[src], prow0 + s_p[j], (char*)oc.dst[c] + (obase + j) * 16, policy_evict_first()); continue; }   // inputs only
      uint64_t v;
      if (src < sp.n_cols) v = ld_stream_int(sp.col[src].ptr, w, 0, prow0 + s_p[j], policy_evict_first());
      else { const ExtDef e = sp.ext[src - sp.n_cols]; v = ext_field(s_pay[e.stage][j], e.shift, e.width, DFGPU_UINT64); }
      switch (w) {
        case 1: ((uint8_t*)oc.dst[c])[obase + j] = (uint8_t)v; break;
        case 2: ((uint16_t*)oc.dst[c])[obase + j] = (uint16_t)v; break;
        case 4: ((uint32_t*)oc.dst[c])[obase + j] = (uint32_t)v; break;
        default: ((uint64_t*)oc.dst[c])[obase + j] = v; break;
      }
    }
  }
  if constexpr (COLS) {
    // the tile's output bits [obase, obase + tot), staged as whole words in shared memory: a warp's 32 survivors are one ballot, or-ed
    // into at most two staged words.  The first and the last word may be shared with the neighbouring tiles: atomicOr into the zeroed
    // bitmap; the words in between belong to this tile alone: plain stores.
    __shared__ uint32_t s_vw[kPipeTile / 32 + 2];
    const OutValid* ov = (const OutValid*)((const char*)gp + kDenseParamsOff);
    const int sh = (int)(obase & 31), lane = threadIdx.x & 31;
    const int nw = tot ? (int)((sh + tot + 31) >> 5) : 0;
    for (int c = 0; c < oc.n; ++c) {
      uint32_t* dv = ov->valid[c];
      if (!dv || nw == 0) continue;
      const int src = oc.src[c];
      for (int i = threadIdx.x; i < nw; i += kPipeThreads) s_vw[i] = 0;
      __syncthreads();
      for (uint32_t j0 = 0; j0 < tot; j0 += kPipeThreads) {
        const uint32_t j = j0 + threadIdx.x;
        bool ok;
        if constexpr (RIGHT) ok = j < tot && (src < sp.n_cols ? bit_get(sp.col[src].valid, sp.col[src].voff + prow0 + s_p[j]) : ((dyn_smem[j] >> sp.ext[src - sp.n_cols].stage) & 1u) != 0);
        else { const ColRef& col = sp.col[src]; ok = j < tot && bit_get(col.valid, col.voff + prow0 + s_p[j]); }
        const unsigned bits = __ballot_sync(0xffffffffu, ok);
        const uint32_t first = (uint32_t)sh + j0 + (threadIdx.x & ~31u);   // staged bit of this warp's lane 0
        if (lane == 0 && bits) {
          atomicOr(&s_vw[first >> 5], bits << (first & 31));
          if ((first & 31) && (bits >> (32 - (first & 31)))) atomicOr(&s_vw[(first >> 5) + 1], bits >> (32 - (first & 31)));
        }
      }
      __syncthreads();
      uint32_t* g = dv + (obase >> 5);
      for (int i = threadIdx.x; i < nw; i += kPipeThreads) {
        if (i == 0 || i == nw - 1) { if (s_vw[i]) atomicOr(g + i, s_vw[i]); }
        else g[i] = s_vw[i];
      }
      __syncthreads();   // s_vw is staged again for the next column
    }
  }
  if (err) atomicOr(&counters[3], (unsigned long long)err);
}

template <bool FILT>
__global__ void __launch_bounds__(kPipeThreads) pipe_output_kernel(const PipeParams* __restrict__ gp, int64_t n, OutCols oc, unsigned long long* __restrict__ tile_desc,
                                                                  unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ totals, unsigned long long* __restrict__ counters) {
  pipe_output_tile<FILT, false>(gp, n, oc, tile_desc, tile_counter, totals, counters);
}
// the same for output columns with validity bitmaps or 16 bytes wide
template <bool FILT>
__global__ void __launch_bounds__(kPipeThreads) pipe_output_cols_kernel(const PipeParams* __restrict__ gp, int64_t n, OutCols oc, unsigned long long* __restrict__ tile_desc,
                                                                       unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ totals, unsigned long long* __restrict__ counters) {
  pipe_output_tile<FILT, true>(gp, n, oc, tile_desc, tile_counter, totals, counters);
}
// the same for a pipeline with RIGHT stages (kPipeTile bytes of dynamic shared memory: the survivors' payload validity bits)
__global__ void __launch_bounds__(kPipeThreads) pipe_output_right_kernel(const PipeParams* __restrict__ gp, int64_t n, OutCols oc, unsigned long long* __restrict__ tile_desc,
                                                                        unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ totals, unsigned long long* __restrict__ counters) {
  pipe_output_tile<false, true, true>(gp, n, oc, tile_desc, tile_counter, totals, counters);
}

// ------------------------------------------------------------------------------------------
// lookup maintenance kernels
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lookup_init_kernel(unsigned long long* recs, uint64_t cap, int stride) {
  const uint64_t total = cap * (uint64_t)stride;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x)
    recs[i] = (i % (uint64_t)stride) == 0 ? kEmptyKey : 0ull;
}
__global__ void __launch_bounds__(256) lookup_rehash_kernel(LookupDev old_t, LookupDev new_t) {
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < old_t.cap; s += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long* r = old_t.recs + s * (uint64_t)old_t.stride;
    const unsigned long long key = r[0];
    if (key == kEmptyKey) continue;
    const uint64_t h = lk_hash(key);
    uint64_t d = __umul64hi(h, new_t.cap);
    while (true) {
      unsigned long long* q = new_t.recs + d * (uint64_t)new_t.stride;
      if (atomicCAS(q, (unsigned long long)kEmptyKey, key) == kEmptyKey) { for (int w = 1; w < new_t.stride; ++w) q[w] = r[w]; break; }
      if (++d == new_t.cap) d = 0;
    }
    if (new_t.bloom) filter_set(new_t, key);
  }
}
// second half of a build whose size was unknown: the packed {key, payload} records of the survivors go into the (now sized) table
__global__ void __launch_bounds__(256) lookup_insert_records_kernel(LookupDev t, const ulonglong2* __restrict__ recs, int64_t n, int unique, unsigned long long* __restrict__ counters /* [_, inserted, fail] */) {
  unsigned int ins = 0; int fail = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const ulonglong2 r = recs[i];
    const int rc = lk_insert(t, r.x, r.y);
    if (rc == 0) ins++;
    else if (rc == 2 || unique) fail |= rc;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) ins += __shfl_xor_sync(0xffffffffu, ins, d);
  fail = __any_sync(0xffffffffu, fail & 1) | (__any_sync(0xffffffffu, fail & 2) << 1);
  if ((threadIdx.x & 31) == 0) { if (ins) atomicAdd(&counters[1], (unsigned long long)ins); if (fail) atomicOr(&counters[2], (unsigned long long)fail); }
}
// the same insert for records radix-partitioned by slot range (radix_partition_records), with the same counters.  Tiles are taken in
// record order from one counter (pipe_probe_agg_kernel's scheme), so the running blocks insert into one ~16 MB slot range of the table at
// a time and its sectors come from DRAM about once.  A thread first prefetches the start slots of its tile's four records into L2, so
// their misses overlap instead of stalling one 128-bit CAS after the other.  The caller detaches the membership filter from `t`
// (lookup_filter_records_kernel sets it): lk_insert then makes no filter update.
__global__ void __launch_bounds__(256) lookup_insert_part_kernel(LookupDev t, const ulonglong2* __restrict__ recs, int64_t n, int unique,
                                                                 unsigned int* __restrict__ tile_counter, unsigned long long* __restrict__ counters /* [_, inserted, fail] */) {
  constexpr int ITEMS = 4, TILE = 256 * ITEMS;
  __shared__ unsigned int s_tile;
  const int64_t ntiles = (n + TILE - 1) / TILE;
  unsigned int ins = 0; int fail = 0;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);   // tiles in record order: the running blocks share one slot range
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;
    ulonglong2 r[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int64_t i = tile * TILE + k * 256 + threadIdx.x;
      if (i < n) { const int4 v = ld_stream_16(recs + i); r[k].x = (uint64_t)(uint32_t)v.x | ((uint64_t)(uint32_t)v.y << 32); r[k].y = (uint64_t)(uint32_t)v.z | ((uint64_t)(uint32_t)v.w << 32); }
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k)
      if (tile * TILE + k * 256 + threadIdx.x < n) asm volatile("prefetch.global.L2 [%0];" :: "l"(t.recs + __umul64hi(lk_hash(r[k].x), t.cap) * (uint64_t)t.stride));
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      if (tile * TILE + k * 256 + threadIdx.x >= n) continue;
      const int rc = lk_insert(t, r[k].x, r[k].y);
      if (rc == 0) ins++;
      else if (rc == 2 || unique) fail |= rc;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) ins += __shfl_xor_sync(0xffffffffu, ins, d);
  fail = __any_sync(0xffffffffu, fail & 1) | (__any_sync(0xffffffffu, fail & 2) << 1);
  if ((threadIdx.x & 31) == 0) { if (ins) atomicAdd(&counters[1], (unsigned long long)ins); if (fail) atomicOr(&counters[2], (unsigned long long)fail); }
}
// the membership filter of n packed records, set in a sweep of its own: inside lookup_insert_part_kernel its random updates would compete
// with the table's slot range for L2, while here the filter (Q3 SF100: 29 MB) stays in L2 and the records stream past it at evict-first
// priority.  The bits equal lk_insert's: a duplicate key sets the bits its first copy set, and the reserved all-ones key, which lk_insert
// rejects, sets none.
__global__ void __launch_bounds__(256) lookup_filter_records_kernel(LookupDev t, const ulonglong2* __restrict__ recs, int64_t n) {
  const uint64_t pol = policy_evict_first();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t key = ld_stream_int(recs + i, 8, 0, 0, pol);
    if (key != kEmptyKey) filter_set(t, key);
  }
}
// the membership filter folded to half its blocks: out[i] = in[2i] | in[2i+1].  bloom_pos places a key by fastrange, block =
// umulhi(h1, blocks) = floor(h1 * blocks / 2^32), and its bit positions t do not depend on `blocks`.  For blocks = 2b,
// umulhi(h1, 2b) >> 1 = floor(floor(h1 * b / 2^31) / 2) = floor(h1 * b / 2^32) = umulhi(h1, b): a key of exact block k lands in folded
// block k >> 1, which holds k's bits, so probing `out` with b blocks has no false negatives for any key of the exact filter.
__global__ void __launch_bounds__(256) bloom_fold_kernel(const ulonglong2* __restrict__ in, unsigned long long* __restrict__ out, uint64_t half) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < half; i += (uint64_t)gridDim.x * blockDim.x) {
    const ulonglong2 v = in[i];
    out[i] = v.x | v.y;
  }
}
// accumulator identities for MIN / MAX (SUM / COUNT start at 0: the table's initialisation, or claim_acc_words on a reused lookup)
__global__ void __launch_bounds__(256) lookup_init_acc_kernel(LookupDev t, int word, unsigned long long value) {
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < t.cap; s += (uint64_t)gridDim.x * blockDim.x) t.recs[s * (uint64_t)t.stride + word] = value;
}
// the hash sink's table: every record (the side record included) starts as its identity words
__global__ void __launch_bounds__(256) hash_init_kernel(unsigned long long* recs, uint64_t n_recs, int stride, HashIdent id) {
  const uint64_t total = n_recs * (uint64_t)stride;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) recs[i] = id.w[i % (uint64_t)stride];
}
// the hash sink's growth: the claimed regular records of the old table move to the (initialised) new one, every word as it is
__global__ void __launch_bounds__(256) hash_rehash_kernel(const unsigned long long* __restrict__ old_recs, uint64_t old_cap, unsigned long long* new_recs, uint64_t new_cap, int stride) {
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < old_cap; s += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long* r = old_recs + s * (uint64_t)stride;
    const uint64_t lo = r[0], hi = r[1];
    if (lo == kEmptyKey && hi == kEmptyKey) continue;
    uint64_t d = hash_tag_slot(lo, hi, new_cap);
    while (true) {
      unsigned long long* q = new_recs + d * (uint64_t)stride;
      const Rec128 prev = cas128(q, Rec128{kEmptyKey, kEmptyKey}, Rec128{lo, hi});
      if (prev.lo == kEmptyKey && prev.hi == kEmptyKey) { for (int w = 2; w < stride; ++w) q[w] = r[w]; break; }
      if (++d == new_cap) d = 0;
    }
  }
}
// the records to emit -> occupancy bitmap (one ballot word per warp).  sel 0: rows_word > 0 (the records a row reached);
// 1: occupied records with rows_word == 0 (LEFT_ANTI: the build rows no probe row reached); 2: every occupied record (LEFT)
__global__ void __launch_bounds__(256) lookup_groups_kernel(LookupDev t, int rows_word, int sel, uint32_t* __restrict__ words) {
  const uint64_t nw = (t.cap + 31) / 32;
  const int lane = threadIdx.x & 31;
  for (uint64_t w = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; w < nw; w += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const uint64_t s = w * 32 + lane;
    bool occ = false;
    if (s < t.cap) {
      const unsigned long long* r = t.recs + s * (uint64_t)t.stride;
      const bool hit = r[rows_word] != 0ull;
      occ = sel == 0 ? hit : (r[0] != kEmptyKey && (sel == 2 || !hit));
    }
    const uint32_t b = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) words[w] = b;
  }
}
struct EmitCol {
  int kind /* 0 key, 1 payload field, 2 accumulator word, 3 AVG value, 4 count as u64, 5 Decimal128 sum / min / max (two words),
              6 dense group key decoded from the slot number, 7 Decimal128 AVG value, 8 packed group field of a 128-bit tag in words 0 and 1,
              9 COUNT(*) of a LEFT join's build row: the row counter, at least 1 (the NULL-padded row of a record no probe row reached),
              10 component of a composite key decoded from the packed key in word 0 */,
      width, shift, word, nn_word, cnt_word, f64_key /* kind 2: the word holds f64_to_ordered of a Float64 MIN / MAX */;
  void* dst; uint32_t* valid;
  long long kmin; int kstride, kradix;   // kind 6: key = kmin + (slot / kstride) % kradix, NULL when that index is kradix - 1
  int avg_mul, avg_prec;                  // kind 7: sum * 10^avg_mul / count must fit Decimal128(avg_prec, _)
  int tag_null;                           // kind 8: the field starts at bit `shift`; NULL when bit tag_null (>= 0) is set
  unsigned long long cstride, cradix;     // kind 10: component = kmin + (key / cstride) % cradix
};
struct EmitCols { int n; EmitCol c[kMaxPipeCols]; unsigned long long* err /* kind 7: set to 1 on overflow */; };
__global__ void __launch_bounds__(256) lookup_emit_kernel(LookupDev t, const uint32_t* __restrict__ slots, int64_t n, int rows_word, EmitCols ec) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (n + 31) / 32;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t i = wi * 32 + lane;
    const unsigned long long* r = i < n ? t.recs + (uint64_t)slots[i] * (uint64_t)t.stride : nullptr;
    for (int c = 0; c < ec.n; ++c) {
      const EmitCol e = ec.c[c];
      uint64_t v = 0;
      bool ok = false;
      if (r) {
        ok = true;
        switch (e.kind) {
          case 0: v = r[0]; break;
          case 1: v = r[1] >> e.shift; break;
          case 2:
            v = e.f64_key ? (uint64_t)__double_as_longlong(ordered_to_f64(r[e.word])) : r[e.word];
            ok = e.nn_word >= 0 ? r[e.nn_word] != 0ull : true;
            break;
          case 4: v = r[e.word]; break;
          case 9: v = max(r[e.word], 1ull); break;
          case 10: v = (uint64_t)e.kmin + (r[0] / e.cstride) % e.cradix; break;
          case 5:
            ok = e.nn_word >= 0 ? r[e.nn_word] != 0ull : true;
            ((unsigned long long*)e.dst)[2 * i] = ok ? r[e.word] : 0ull;
            ((unsigned long long*)e.dst)[2 * i + 1] = ok ? r[e.word + 1] : 0ull;
            break;
          case 6: {
            const uint64_t q = ((uint64_t)slots[i] / (uint64_t)e.kstride) % (uint64_t)e.kradix;
            ok = q + 1 != (uint64_t)e.kradix;
            v = (uint64_t)e.kmin + q;
            break;
          }
          case 7: {   // DecimalAverager::avg (expr_dec.cuh dec_avg)
            const unsigned long long cnt = r[e.cnt_word];
            ok = cnt != 0ull;
            i128 q = 0;
            if (ok && !dec_avg((i128)(((u128)r[e.word + 1] << 64) | (u128)r[e.word]), cnt, e.avg_mul, e.avg_prec, &q)) atomicOr(ec.err, 1ull);
            ((unsigned long long*)e.dst)[2 * i] = (unsigned long long)(u128)q;
            ((unsigned long long*)e.dst)[2 * i + 1] = (unsigned long long)((u128)q >> 64);
            break;
          }
          case 8: {
            const u128 tag = ((u128)r[1] << 64) | (u128)r[0];
            ok = e.tag_null < 0 || !(uint64_t)((tag >> e.tag_null) & 1u);
            v = (uint64_t)(tag >> e.shift);   // the store below keeps the column's width: no sign extension needed
            break;
          }
          default: {   // AVG = sum / count over Float64 (functions-aggregate/src/average.rs)
            const unsigned long long cnt = r[e.cnt_word];
            ok = cnt != 0ull;
            const double d = ok ? __longlong_as_double((long long)r[e.word]) / (double)cnt : 0.0;
            v = (uint64_t)__double_as_longlong(d);
          }
        }
        if (!ok) v = 0;
        if (e.kind != 5 && e.kind != 7) switch (e.width) {
          case 1: ((uint8_t*)e.dst)[i] = (uint8_t)v; break;
          case 2: ((uint16_t*)e.dst)[i] = (uint16_t)v; break;
          case 4: ((uint32_t*)e.dst)[i] = (uint32_t)v; break;
          default: ((uint64_t*)e.dst)[i] = v; break;
        }
      }
      if (e.valid) { const uint32_t b = __ballot_sync(0xffffffffu, ok); if (lane == 0) e.valid[wi] = b; }
    }
  }
}

// lookup_groups_kernel (sel 0) -> compact -> lookup_emit_kernel in one pass over the table, for emissions whose every column is a word of
// the record (kinds 0, 1, 4, and 2 without a non-null counter or a Float64 key) without a validity bitmap: each 1024-slot tile finds its
// records with a non-zero rows_word, ranks them in slot order (ballots, then decoupled look-back across tiles taken in order), and writes
// their columns at those ranks, so the groups come out in the order of the three-kernel path.  The table is read once, with no bitmap,
// index array or host round trip in between.  total[0]: the group count; the columns hold max_out rows, and rows past them are not written.
__global__ void __launch_bounds__(256) lookup_scan_emit_kernel(LookupDev t, int rows_word, EmitCols ec, unsigned int* __restrict__ tile_counter,
                                                               unsigned long long* __restrict__ tile_desc, unsigned long long* __restrict__ total, uint64_t max_out) {
  constexpr int ITEMS = 4, TILE = 256 * ITEMS;
  __shared__ unsigned int s_tile;
  __shared__ uint32_t s_rank[ITEMS * 8];   // exclusive rank of (item k, warp w) at [k * 8 + w]
  __shared__ unsigned long long s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t ntiles = (t.cap + TILE - 1) / TILE;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);   // tiles in slot order: look-back waits on earlier tiles only
    __syncthreads();
    const uint64_t tile = s_tile;
    if (tile >= ntiles) break;
    unsigned bal[ITEMS];
    bool occ[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const uint64_t slot = tile * TILE + k * 256 + threadIdx.x;
      occ[k] = slot < t.cap && t.recs[slot * (uint64_t)t.stride + rows_word] != 0ull;
      bal[k] = __ballot_sync(0xffffffffu, occ[k]);
      if (lane == 0) s_rank[k * 8 + warp] = __popc(bal[k]);
    }
    __syncthreads();
    if (warp == 0) {
      const uint32_t c = s_rank[lane];
      uint32_t inc = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += v; }
      s_rank[lane] = inc - c;
      const uint32_t tot = __shfl_sync(0xffffffffu, inc, 31);
      const unsigned long long ex = tile_lookback((int64_t)tile, tot, tile_desc);
      if (lane == 0) { s_base = ex; if (tile == ntiles - 1) total[0] = ex + tot; }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const uint64_t i = s_base + s_rank[k * 8 + warp] + __popc(bal[k] & ((1u << lane) - 1u));
      if (!occ[k] || i >= max_out) continue;
      const unsigned long long* r = t.recs + (tile * TILE + k * 256 + threadIdx.x) * (uint64_t)t.stride;
      for (int c = 0; c < ec.n; ++c) {
        const EmitCol& e = ec.c[c];
        const uint64_t v = e.kind == 0 ? r[0] : (e.kind == 1 ? r[1] >> e.shift : r[e.word]);
        switch (e.width) {
          case 1: ((uint8_t*)e.dst)[i] = (uint8_t)v; break;
          case 2: ((uint16_t*)e.dst)[i] = (uint16_t)v; break;
          case 4: ((uint32_t*)e.dst)[i] = (uint32_t)v; break;
          default: ((uint64_t*)e.dst)[i] = v; break;
        }
      }
    }
  }
}

// OR-all-reduce of n_ranks membership filters of identical geometry over peer memory (NVLink): this rank merges slice
// `rank` of every filter (reads of the peers' slices travel over NVLink) and writes the merged slice into every rank's
// filter.  Slice r of rank q's buffer is read only by rank r, and written by rank r only after it has read it.
constexpr int kMaxPeers = 8;
struct PeerWords { unsigned long long* p[kMaxPeers]; };
__global__ void __launch_bounds__(256) filter_allreduce_peer_kernel(PeerWords pw, int rank, int n_ranks, uint64_t blocks) {
  const uint64_t lo = blocks * (uint64_t)rank / (uint64_t)n_ranks, hi = blocks * (uint64_t)(rank + 1) / (uint64_t)n_ranks;
  for (uint64_t i = lo + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < hi; i += (uint64_t)gridDim.x * blockDim.x) {
    unsigned long long acc = 0;
#pragma unroll
    for (int q = 0; q < kMaxPeers; ++q) if (q < n_ranks) acc |= pw.p[q][i];
#pragma unroll
    for (int q = 0; q < kMaxPeers; ++q) if (q < n_ranks) pw.p[q][i] = acc;
  }
}

__global__ void __launch_bounds__(256) col_minmax_kernel(ColRef c, int64_t n, int uns, unsigned long long* mm /* [min,max,valid] */) {
  unsigned long long kmin = ~0ull, kmax = 0, cnt = 0;   // order-preserving map of signed keys onto unsigned
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (c.valid && !bit_get(c.valid, c.voff + i)) continue;
    uint64_t v;
    switch (c.width) {
      case 1: v = c.sgn ? (uint64_t)(int64_t)((const int8_t*)c.ptr)[i] : ((const uint8_t*)c.ptr)[i]; break;
      case 2: v = c.sgn ? (uint64_t)(int64_t)((const int16_t*)c.ptr)[i] : ((const uint16_t*)c.ptr)[i]; break;
      case 4: v = c.sgn ? (uint64_t)(int64_t)((const int32_t*)c.ptr)[i] : ((const uint32_t*)c.ptr)[i]; break;
      default: v = ((const uint64_t*)c.ptr)[i]; break;
    }
    if (!uns) v ^= 1ull << 63;
    kmin = min(kmin, (unsigned long long)v); kmax = max(kmax, (unsigned long long)v); cnt++;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, d));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, d));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  }
  if ((threadIdx.x & 31) == 0 && cnt) { atomicMin(&mm[0], kmin); atomicMax(&mm[1], kmax); atomicAdd(&mm[2], cnt); }
}

// wrapping sum of an integer column (sign / zero extended to 64 bits): order-independent fingerprints of large results
__global__ void __launch_bounds__(256) col_sum_kernel(ColRef c, int64_t n, unsigned long long* out /* [sum, valid] */) {
  unsigned long long s = 0, cnt = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (c.valid && !bit_get(c.valid, c.voff + i)) continue;
    switch (c.width) {
      case 1: s += c.sgn ? (uint64_t)(int64_t)((const int8_t*)c.ptr)[i] : ((const uint8_t*)c.ptr)[i]; break;
      case 2: s += c.sgn ? (uint64_t)(int64_t)((const int16_t*)c.ptr)[i] : ((const uint16_t*)c.ptr)[i]; break;
      case 4: s += c.sgn ? (uint64_t)(int64_t)((const int32_t*)c.ptr)[i] : ((const uint32_t*)c.ptr)[i]; break;
      case 16: s += ((const uint64_t*)c.ptr)[2 * i] + 3ull * ((const uint64_t*)c.ptr)[2 * i + 1]; break;   // Decimal128: low word + 3 x high word
      default: s += ((const uint64_t*)c.ptr)[i]; break;
    }
    cnt++;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, d); cnt += __shfl_xor_sync(0xffffffffu, cnt, d); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&out[0], s); atomicAdd(&out[1], cnt); }
}

}  // namespace dfgpu

// ==========================================================================================
// host side
// ==========================================================================================
using namespace dfgpu;

struct dfgpu_lookup {
  dfgpu_ctx* ctx = nullptr;
  int key_type = 0;
  std::vector<int> pay_types, pay_shift;
  dfgpu_lookup_options opt{};
  int mode = LK_HASH, stride = 1;
  bool has_payload = false;
  DevBuf recs, bloom, bits;
  uint64_t cap = 0, bloom_blocks = 0, coarse_words = 0, kmin = 0, ksize = 0;   // the coarse level lives behind the exact blocks in `bloom`
  int64_t rows = 0, rehashes = 0;
  int64_t null_keys = 0;   // build rows pushed with a NULL key (counted before the predicate): never inserted, so a LEFT / LEFT_ANTI stage cannot emit them
  bool acc_claimed = false, filter_only = false;
  bool marks_taken = false;   // a FULL stage's visited marks live in the first accumulator word: one FULL pipeline, until dfgpu_lookup_clear
  // a join-keyed aggregate sink or a FULL stage pushed into the accumulator words since creation or dfgpu_lookup_clear: the next one to
  // claim them zeroes them first (claim_acc_words)
  bool acc_written = false;
  // composite key (dfgpu_lookup_create_composite): the key is the packed tuple of these components, in [0, domain)
  std::vector<int> comp_types; std::vector<int64_t> comp_min; std::vector<uint64_t> comp_range, comp_stride; uint64_t domain = 0;
};

struct PipeAgg { int func; ExprPlan plan; bool has_expr = false; int word = -1, nn_word = -1, cnt_word = -1, cls = C_I64, arg_type = 0; };

struct dfgpu_pipeline {
  dfgpu_ctx* ctx = nullptr;
  std::vector<int> in_types, vtypes;                 // input schema, virtual schema (input + payload fields)
  std::vector<ExtDef> exts;
  bool has_pred = false;
  ExprPlan pred;
  std::vector<dfgpu_pipeline_stage> stages;
  bool has_right = false;   // a RIGHT stage: every kernel runs its VAR bit 1024 / pipe_output_right_kernel instantiation
  // Full join (dfgpu_pipeline_set_stage_full): the RIGHT stage that marks its records (kStageFull on the device), or -1.  in_tail: the push
  // of the unmatched build rows at finish, whose FULL stage reads the emitted keys from the hidden column behind the inputs
  int full_stage = -1; bool in_tail = false; int64_t m_unmatched_build_rows = 0;
  std::vector<DCol> tail_part; int64_t tail_rows = 0;   // output sinks: the tail push's columns, emitted after the probe rows' batches
  // stage filters (dfgpu_pipeline_set_stage_filter): per stage the program and the payload fields its virtual columns past the inputs name
  ExprPlan filt[kMaxStages]; bool has_filt[kMaxStages] = {false, false, false}; std::vector<ExtDef> filt_ext[kMaxStages]; int filt_nodes = 0;
  std::unique_ptr<FiltParams> filt_host;   // staging copy of the bound programs (upload_filters)
  bool pushed = false;
  int sink = SINK_NONE;
  // build sink
  dfgpu_lookup* target = nullptr; int bkey_col = -1; std::vector<int> bpay_cols;
  // composite keys: the component input columns of each stage (dfgpu_pipeline_set_stage_keys) and of the build sink
  // (dfgpu_pipeline_sink_build_composite); `packed` holds the current batch's packed keys in that order (stages, then the build sink),
  // in PipeParams' column array behind the input columns; key_flags: [out-of-domain build key seen, NULL build keys], read at finish
  std::vector<int> stage_keys[kMaxStages]; std::vector<int> bkey_cols;
  std::vector<DCol> packed; DevBuf key_flags;
  // aggregate sink
  std::vector<int> group_cols; std::vector<PipeAgg> aggs; int agg_mode = DFGPU_AGG_SINGLE, agg_stage = -1, rows_word = -1; bool acc_ready = false;
  int left_kind = 0;   // DFGPU_STAGE_LEFT / DFGPU_STAGE_LEFT_ANTI when the last stage is one (it is then agg_stage), else 0
  // dense-group aggregate sink (group_cols, aggs and agg_mode as above; the aggregates' words address a slot of dense_acc)
  std::vector<DenseKey> dense_keys; std::vector<int> dense_radix; std::vector<unsigned long long> dense_ident;
  int dense_slots = 0, dense_words = 0; DevBuf dense_acc;
  // hash-keyed aggregate sink (group_cols, aggs, agg_mode and rows_word as above; the aggregates' words address a record of hash_recs)
  std::vector<HashKey> hash_keys; std::vector<unsigned long long> hash_ident; int hash_stride = 0; int64_t hash_cap_hint = 0;
  uint64_t hash_cap = 0; DevBuf hash_recs /* hash_cap records, then the side record */, hash_ngroups;
  int64_t m_group_rehashes = 0, m_replayed_rows = 0;
  // output sink
  std::vector<int> out_cols; bool out_ordered = true;
  std::vector<std::vector<DCol>> out_parts; int64_t out_rows_pending = 0;
  int64_t batch_size = 0;
  bool finished = false;
  DevBuf params_dev, counters;
  std::deque<BatchPtr> outq;
  int64_t m_input_rows = 0, m_sink_rows = 0, m_output_rows = 0, m_groups = 0, m_ring_launches = 0, m_dense_block_launches = 0, m_partitioned_launches = 0,
          m_partitioned_inserts = 0, m_partitioned_records = 0;
  std::string name;   // optional label: the kernel-timing family becomes "pipe:<name>" (dfgpu_kernel_time)
};

namespace dfgpu {

static LookupDev lookup_dev(const dfgpu_lookup* l) {
  LookupDev d;
  memset(&d, 0, sizeof(d));
  d.mode = l->mode; d.stride = l->stride; d.has_payload = l->has_payload ? 1 : 0;
  d.recs = l->recs.as<unsigned long long>(); d.cap = l->cap;
  d.bloom = l->bloom.ptr ? l->bloom.as<unsigned long long>() : nullptr; d.bloom_blocks = l->bloom_blocks;
  d.coarse = (l->bloom.ptr && l->coarse_words) ? (uint32_t*)(l->bloom.as<unsigned long long>() + l->bloom_blocks) : nullptr; d.coarse_words = l->coarse_words;
  d.bits = l->bits.ptr ? l->bits.as<uint32_t>() : nullptr; d.kmin = l->kmin; d.ksize = l->ksize;
  return d;
}

static bool key_type_ok(int t) { int w = type_width(t); return w >= 1 && w <= 8 && !type_is_float(t) && t != DFGPU_BOOL; }

// A lookup table larger than this does not stay in the 50 MB L2: it gets a Bloom filter (membership_filter < 0), and the fused pipeline
// partitions its build records (pipeline_push) and the probe records of its aggregate sink (partitioned_table_bytes) by slot range.
constexpr size_t kL2TableBytes = 40ull << 20;

// (re)allocate a hash lookup for at least `rows` records at load factor <= 0.5; existing records are rehashed
static void lookup_reserve(dfgpu_lookup* l, int64_t rows) {
  if (l->mode != LK_HASH || l->filter_only) return;
  dfgpu_ctx* ctx = l->ctx;
  const uint64_t need = std::max<uint64_t>(1024, (uint64_t)rows * 2);
  if (l->cap >= need) return;
  const uint64_t new_cap = l->cap == 0 ? need : std::max<uint64_t>(need, l->cap * 2);
  DF_CHECK(new_cap < 0xFFFFFFFFull, DFGPU_ERR_UNSUPPORTED, "lookup: more than 2^31 build rows");
  DevBuf nrecs(ctx, (size_t)new_cap * l->stride * 8), nbloom;
  lookup_init_kernel<<<grid_for((int64_t)new_cap * l->stride, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(nrecs.as<unsigned long long>(), new_cap, l->stride);
  DF_LAUNCH_CHECK(ctx);
  uint64_t nblocks = 0;
  const size_t table_bytes = (size_t)new_cap * l->stride * 8;
  if (l->opt.membership_filter == 1 || (l->opt.membership_filter < 0 && table_bytes > kL2TableBytes)) {
    // 16 bits per key at load factor 0.5; an even count lets the partitioned aggregate fold the filter to half size (bloom_fold_kernel)
    nblocks = (std::max<uint64_t>(1024, new_cap / 8) + 1) & ~1ull;
    nbloom.alloc(ctx, (size_t)nblocks * 8);
    nbloom.zero();
  }
  LookupDev old_t = lookup_dev(l);
  LookupDev new_t = old_t;
  new_t.recs = nrecs.as<unsigned long long>(); new_t.cap = new_cap; new_t.bloom = nbloom.ptr ? nbloom.as<unsigned long long>() : nullptr; new_t.bloom_blocks = nblocks;
  if (l->cap > 0 && l->rows > 0) {
    lookup_rehash_kernel<<<grid_for((int64_t)l->cap, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(old_t, new_t);
    DF_LAUNCH_CHECK(ctx);
    l->rehashes++;
  }
  l->recs = std::move(nrecs); l->bloom = std::move(nbloom); l->cap = new_cap; l->bloom_blocks = nblocks;
}

static ColRef col_ref(const DCol& c) {
  ColRef r;
  r.ptr = c.values; r.valid = c.validity; r.voff = c.offset; r.width = type_width(c.type); r.sgn = type_is_signed_int(c.type) ? 1 : 0;
  r.vec = ((uintptr_t)c.values % 32 == 0) ? 2 : (((uintptr_t)c.values % 16 == 0) ? 1 : 0); r.pad = 0;   // 2: whole-sector loads allowed too
  return r;
}

// bind a planned expression into nodes at `out`; virtual columns >= n_cols become the payload fields exts[column - n_cols]
static void bind_nodes(const ExprPlan& plan, const std::vector<DCol>& cols, const std::vector<ExtDef>& exts, const std::vector<std::pair<uint16_t, uint16_t>>& gmasks,
                       ENode* out) {
  for (size_t i = 0; i < plan.nodes.size(); ++i) {
    const dfgpu_expr_node& nd = plan.nodes[i];
    ENode& e = out[i];
    memset(&e, 0, sizeof(e));
    e.kind = nd.kind; e.op = nd.a; e.in_type = plan.in_type[i]; e.out_type = plan.out_type[i];
    if (nd.kind == DFGPU_EXPR_COLUMN) {
      if (nd.a < (int)cols.size()) {
        const DCol& c = cols[nd.a];
        e.col = c.values; e.valid = c.validity; e.voff = c.offset;
      } else {
        const ExtDef& x = exts[nd.a - (int)cols.size()];
        e.kind = kExprExt; e.voff = x.stage; e.lit = (uint64_t)x.shift;
      }
    } else if (nd.kind == DFGPU_EXPR_LITERAL) {
      e.lit = literal_bits(nd); e.lit_null = nd.is_null;
      if (type_is_decimal(nd.type)) memcpy(&e.voff, &nd.lit_f64, 8);
    } else if ((nd.kind == DFGPU_EXPR_BINARY || nd.kind == DFGPU_EXPR_CAST) && plan.has_decimal) {
      e.voff = plan.aux[i];   // power-of-ten rescale exponents (expr_dec.cuh)
    }
    e.g_and = gmasks[i].first; e.g_or = gmasks[i].second;
  }
}

// bind a planned expression into pool nodes; virtual columns >= n_cols become payload-field nodes
static int bind_pool(const dfgpu_pipeline* p, const ExprPlan& plan, const std::vector<DCol>& cols, PipeParams* pp, int* pool_used) {
  const int start = *pool_used;
  const int64_t n_rows = cols.empty() ? 0 : cols[0].length;
  const auto gmasks = resolve_guards(p->ctx, plan, cols, n_rows);   // short-circuit AND / OR: which RHS errors count on which rows (binary.rs:1182)
  DF_CHECK(start + (int)plan.nodes.size() <= kPoolNodes, DFGPU_ERR_UNSUPPORTED, "pipeline: expressions too large (56 nodes in total)");
  bind_nodes(plan, cols, p->exts, gmasks, pp->pool + start);
  *pool_used = start + (int)plan.nodes.size();
  return start;
}

static bool pipeline_has_filters(const dfgpu_pipeline* p) { return p->filt_nodes > 0; }

// byte offset of FiltParams in pipe_kernel's dynamic shared memory: behind the hash sink's HashParams or the dense sink's slots
static int filt_smem_off(const dfgpu_pipeline* p);
static int plan_depth(const ExprPlan& plan);

// the stage filters for one batch, into the parameter buffer behind PipeParams and the sink's block (the pointers address `cols`)
static void upload_filters(dfgpu_pipeline* p, const std::vector<DCol>& cols) {
  FiltParams& fp = *p->filt_host;
  memset(&fp, 0, sizeof(fp));
  fp.smem_off = filt_smem_off(p);
  int used = 0;
  for (int s = 0; s < kMaxStages; ++s) {
    if (!p->has_filt[s]) continue;
    const ExprPlan& plan = p->filt[s];
    // no guards: set_stage_filter admits no AND / OR whose right operand can raise
    bind_nodes(plan, cols, p->filt_ext[s], std::vector<std::pair<uint16_t, uint16_t>>(plan.nodes.size(), {0, 0}), fp.pool + used);
    fp.start[s] = used; fp.n[s] = (int)plan.nodes.size();
    fp.small[s] = plan.has_decimal ? 3 : (plan_depth(plan) <= 4 ? 1 : 0);
    used += fp.n[s];
  }
  const size_t bytes = kFiltParamsOff + sizeof(FiltParams);
  if (p->params_dev.bytes < bytes) p->params_dev.alloc(p->ctx, bytes);
  // filt_host lives as long as the pipeline, and every push synchronises before the next batch rewrites it
  DF_CUDA(cudaMemcpyAsync((char*)p->params_dev.ptr + kFiltParamsOff, &fp, sizeof(FiltParams), cudaMemcpyHostToDevice, p->ctx->stream));
}

// largest evaluation-stack depth of a post-order program (the register-resident interpreter handles <= 4)
static int plan_depth(const ExprPlan& plan) {
  int sp = 0, mx = 0;
  for (const auto& nd : plan.nodes) {
    if (nd.kind == DFGPU_EXPR_COLUMN || nd.kind == DFGPU_EXPR_LITERAL) sp++;
    else if (nd.kind == DFGPU_EXPR_BINARY) sp--;
    mx = std::max(mx, sp);
  }
  return mx;
}

// virtual column c is a payload field of a RIGHT stage: NULL on the rows that stage did not match
static bool is_right_field(const dfgpu_pipeline* p, int c) {
  const int nin = (int)p->in_types.size();
  return c >= nin && p->stages[p->exts[c - nin].stage].kind == DFGPU_STAGE_RIGHT;
}

// only integer columns without NULLs (in THIS batch), non-NULL integer literals, payload fields (not a RIGHT stage's: they can be NULL) and
// + - *: eval_int_fast applies
static bool plan_is_int_arith(const dfgpu_pipeline* p, const ExprPlan& plan, const std::vector<DCol>& cols) {
  for (size_t i = 0; i < plan.nodes.size(); ++i) {
    const dfgpu_expr_node& nd = plan.nodes[i];
    const int t = plan.out_type[i];
    if (!type_is_int(t)) return false;
    if (nd.kind == DFGPU_EXPR_COLUMN) { if ((nd.a < (int)cols.size() && cols[nd.a].validity) || is_right_field(p, nd.a)) return false; }
    else if (nd.kind == DFGPU_EXPR_LITERAL) { if (nd.is_null) return false; }
    else if (nd.kind == DFGPU_EXPR_BINARY) { if (nd.a != DFGPU_OP_PLUS && nd.a != DFGPU_OP_MINUS && nd.a != DFGPU_OP_MULTIPLY) return false; }
    else return false;
  }
  return true;
}

static bool expr_can_be_null(const dfgpu_pipeline* p, const ExprPlan& plan, const std::vector<DCol>& cols) {
  for (const auto& nd : plan.nodes) {
    if (nd.kind == DFGPU_EXPR_COLUMN && nd.a < (int)cols.size() && cols[nd.a].validity) return true;
    if (nd.kind == DFGPU_EXPR_COLUMN && is_right_field(p, nd.a)) return true;
    if (nd.kind == DFGPU_EXPR_LITERAL && nd.is_null) return true;
  }
  return false;
}

// The ring-fed phase A (pipe_kernel VAR bit 64) serves batches whose phase A is a conjunction of `column <cmp> literal` terms (or no
// predicate) plus filter / bitmap stage tests, over columns without validity bitmaps, and whose aggregates (if any) are COUNT(*) or
// integer programs (eval_int_fast); the streamed columns need 16-byte-aligned bases and at least two 256-row tiles per warp ring must
// fit ring_smem(sink).  Everything else keeps ring_stages = 0 and runs the other instantiations.
static void fill_ring(PipeParams* pp, int ring_bytes_budget) {
  if (pp->pred_mode == 2) return;
  std::vector<int> ring;
  auto add = [&](int c) { if (std::find(ring.begin(), ring.end(), c) == ring.end()) ring.push_back(c); };
  if (pp->pred_mode == 1)
    for (int t = 0; t < pp->n_terms; ++t) add(pp->term_col[t]);
  for (int s = 0; s < pp->n_stages; ++s) {
    const StageDev& st = pp->stage[s];
    if (pp->col[st.key_col].valid) return;
    if (st.lk.mode == LK_BITMAP || (st.lk.bloom && st.kind != DFGPU_STAGE_ANTI)) add(st.key_col);   // the keys phase A tests
  }
  for (int a = 0; a < pp->n_aggs; ++a) if (pp->agg[a].func != DFGPU_AGG_COUNT_STAR && pp->agg[a].small != 2) return;   // the general interpreters stay out of the ring kernel
  if (ring.empty() || (int)ring.size() > kMaxRing) return;
  int bytes = 0;
  for (int c : ring) {
    if (pp->col[c].valid || !pp->col[c].vec) return;
    pp->ring_off[c] = bytes;
    bytes += kWarpTile * pp->col[c].width;
  }
  const int stages = std::min(kMaxRingStages, ring_bytes_budget / (kPipeWarps * bytes));
  if (stages < 2) return;
  pp->ring_stages = stages; pp->ring_bytes = bytes; pp->ring_n = (int)ring.size();
  for (size_t k = 0; k < ring.size(); ++k) pp->ring_col[k] = ring[k];
}

// the predicate as a conjunction of at most max_terms `column <cmp> literal` terms over integer-class columns: {col, op, uns, lit} each
static bool conjunction_terms(const dfgpu_pipeline* p, int max_terms, std::vector<std::array<long long, 4>>* terms) {
  const auto& nd = p->pred.nodes;
  terms->clear();
  bool fast = true;
  size_t i = 0;
  int depth = 0;
  while (i < nd.size() && fast) {
    if (i + 2 < nd.size() && nd[i].kind == DFGPU_EXPR_COLUMN && nd[i + 1].kind == DFGPU_EXPR_LITERAL && nd[i + 2].kind == DFGPU_EXPR_BINARY &&
        nd[i + 2].a >= DFGPU_OP_EQ && nd[i + 2].a <= DFGPU_OP_GTEQ && !nd[i + 1].is_null) {
      const int ct = p->in_types[nd[i].a];
      const int cls = cls_of(ct);
      if ((cls != C_I64 && cls != C_U64) || p->pred.has_decimal || (int)terms->size() >= max_terms) { fast = false; break; }
      terms->push_back({(long long)nd[i].a, (long long)nd[i + 2].a, (long long)(cls == C_U64), (long long)literal_bits(nd[i + 1])});
      depth++; i += 3;
    } else if (nd[i].kind == DFGPU_EXPR_BINARY && nd[i].a == DFGPU_OP_AND && depth >= 2) { depth--; i++; }
    else fast = false;
  }
  return fast && depth == 1 && !terms->empty();
}

// the column of PipeParams' array that stage s (s == kMaxStages: the build sink) reads its key from: a composite key's packed column
// behind the input columns (pack_batch_keys' order), else the key column itself
static int key_slot(const dfgpu_pipeline* p, int s) {
  int k = (int)p->in_types.size();
  if (p->in_tail && s == p->full_stage) return k;   // the Full join's tail: the emitted keys, the only hidden column (its stage is the only one)
  for (int t = 0; t < (int)p->stages.size() && t < s; ++t) k += p->stage_keys[t].empty() ? 0 : 1;
  if (s == kMaxStages) return p->bkey_cols.empty() ? p->bkey_col : k;
  return p->stage_keys[s].empty() ? p->stages[s].key_col : k;
}

static void fill_params(dfgpu_pipeline* p, const std::vector<DCol>& cols, PipeParams* pp) {
  memset(pp, 0, sizeof(*pp));
  pp->n_cols = (int)cols.size();
  static const int hints_env = getenv("DFGPU_PIPE_HINTS") ? atoi(getenv("DFGPU_PIPE_HINTS")) : 3;
  pp->hints = hints_env;
  for (size_t c = 0; c < cols.size(); ++c) pp->col[c] = col_ref(cols[c]);
  for (size_t k = 0; k < p->packed.size(); ++k) pp->col[cols.size() + k] = col_ref(p->packed[k]);   // hidden: n_cols stays the inputs'
  int pool_used = 0;
  pp->pred_mode = 0;
  if (p->has_pred && !p->in_tail) {   // the Full join's tail rows are build rows: the predicate over the probe side does not apply
    // fast path: conjunction of `column <cmp> literal` terms over integer-class columns
    std::vector<std::array<long long, 4>> terms;  // col, op, uns, lit
    if (conjunction_terms(p, kMaxTerms, &terms)) {
      pp->pred_mode = 1; pp->n_terms = (int)terms.size();
      for (size_t t = 0; t < terms.size(); ++t) { pp->term_col[t] = (int)terms[t][0]; pp->term_op[t] = (int)terms[t][1]; pp->term_uns[t] = (int)terms[t][2]; pp->term_lit[t] = terms[t][3]; }
    } else {
      pp->pred_mode = 2;
      pp->pred_start = bind_pool(p, p->pred, cols, pp, &pool_used);
      pp->pred_n = (int)p->pred.nodes.size();
      pp->pred_small = p->pred.has_decimal ? 3 : (plan_depth(p->pred) <= 4 ? 1 : 0);
    }
  }
  pp->n_stages = (int)p->stages.size();
  pp->first_hash = -1;
  for (size_t s = 0; s < p->stages.size(); ++s) if (p->stages[s].lookup->mode == LK_HASH && p->stages[s].kind != DFGPU_STAGE_MAYBE && pp->first_hash < 0) pp->first_hash = (int)s;
  for (size_t s = 0; s < p->stages.size(); ++s) {
    // a LEFT / LEFT_ANTI stage probes as an INNER one: the build rows no probe row reached are found in the records at finish
    const int kind = p->stages[s].kind;
    pp->stage[s].kind = kind == DFGPU_STAGE_LEFT || kind == DFGPU_STAGE_LEFT_ANTI ? DFGPU_STAGE_INNER : kind; pp->stage[s].key_col = key_slot(p, (int)s); pp->stage[s].lk = lookup_dev(p->stages[s].lookup);
    if ((int)s == p->full_stage) pp->stage[s].kind = kStageFull;
  }
  pp->n_ext = (int)p->exts.size();
  for (size_t e = 0; e < p->exts.size(); ++e) pp->ext[e] = p->exts[e];
  pp->agg_stage = -1;
  if (p->sink == SINK_BUILD) {
    pp->target = lookup_dev(p->target);
    pp->bkey_col = key_slot(p, kMaxStages);
    pp->target_unique = (p->target->has_payload || p->target->opt.n_acc_words > 0) ? 1 : 0;
    pp->n_bpay = (int)p->bpay_cols.size();
    for (size_t c = 0; c < p->bpay_cols.size(); ++c) {
      pp->bpay_src[c] = p->bpay_cols[c]; pp->bpay_shift[c] = p->target->pay_shift[c]; pp->bpay_width[c] = type_width(p->target->pay_types[c]);
      if (p->bpay_cols[c] < (int)cols.size()) DF_CHECK(!cols[p->bpay_cols[c]].validity, DFGPU_ERR_UNSUPPORTED, "pipeline: nullable build payload columns stay on the unfused join");
    }
  } else if (p->sink == SINK_AGG || p->sink == SINK_HASH) {
    pp->agg_stage = p->agg_stage; pp->rows_word = p->rows_word; pp->n_aggs = (int)p->aggs.size();
    for (size_t a = 0; a < p->aggs.size(); ++a) {
      const PipeAgg& ag = p->aggs[a];
      AggDef& d = pp->agg[a];
      d.func = ag.func; d.cls = ag.cls; d.word = ag.word; d.nn_word = ag.nn_word; d.start = 0; d.n = 0;
      if (ag.has_expr) {
        d.start = bind_pool(p, ag.plan, cols, pp, &pool_used); d.n = (int)ag.plan.nodes.size();
        d.small = plan_depth(ag.plan) <= 4 ? 1 : 0;
        if (d.small && plan_is_int_arith(p, ag.plan, cols)) d.small = 2;
        if (ag.plan.has_decimal) d.small = 3;
        if (ag.nn_word < 0 && ag.func != DFGPU_AGG_COUNT)
          DF_CHECK(!expr_can_be_null(p, ag.plan, cols), DFGPU_ERR_UNSUPPORTED, "pipeline: nullable aggregate input needs one more accumulator word in the lookup (n_acc_words)");
      }
    }
    if (pp->n_aggs > 0 && pp->agg[0].small == 2) {
      const AggDef& d = pp->agg[0];
      int ng = 0;
      for (int i = 0; i < d.n; ++i) if (pp->pool[d.start + i].kind == DFGPU_EXPR_COLUMN) ng++;
      if (ng <= kGather) {
        for (int i = 0; i < d.n; ++i) if (pp->pool[d.start + i].kind == DFGPU_EXPR_COLUMN) pp->gather_node[pp->n_gather++] = d.start + i;
      }
    }
  }
  if (pipeline_has_filters(p)) upload_filters(p, cols);   // the ring-fed and partitioned paths take no stage filters
  else fill_ring(pp, ring_smem(p->sink));
}

static void check_errors(unsigned long long err) {
  if (err & ERR_DIV_ZERO) throw Error(DFGPU_ERR_ARITH, "Arrow error: Divide by zero error");
  if (err & ERR_OVERFLOW) throw Error(DFGPU_ERR_ARITH, "Arrow error: Arithmetic overflow");
  if (err & ERR_CAST) throw Error(DFGPU_ERR_ARITH, "Arrow error: Cast error: Can't cast value to the target type (out of range)");
  if (err & kErrRingAgg) throw Error(DFGPU_ERR_INVALID, "internal: the ring-fed pipeline kernel was given an aggregate it does not evaluate");
}

static bool pipeline_has_decimal(const dfgpu_pipeline* p);

// the sink's default VAR bits (launch_pipe below) plus the stage filters
constexpr int filt_var(int sink) { return kVarFilt | (sink == SINK_AGG ? kPipeVarDefault : (sink == SINK_PACK || sink == SINK_OUTPUT_ANY ? 2 : 0)); }

// the timing family of a push's pipeline kernel: "pipe:<name>" (`unnamed` without a name); the Full join's tail push at finish is timed
// as its own family, "pipe_full_tail[:<name>]", so it is not counted in the probe pushes' family
static std::string tail_timer(const dfgpu_pipeline* p) { return p->name.empty() ? std::string("pipe_full_tail") : "pipe_full_tail:" + p->name; }
static std::string pipe_timer(const dfgpu_pipeline* p, const char* unnamed) {
  if (p->in_tail) return tail_timer(p);
  return p->name.empty() ? std::string(unnamed) : "pipe:" + p->name;
}

template <int SINK>
static void launch_pipe(dfgpu_pipeline* p, const PipeParams& pp, int64_t n, const char* timer_name, bool part = false, bool out_cols = false) {
  dfgpu_ctx* ctx = p->ctx;
  const int64_t ntiles = (n + kPipeTile - 1) / kPipeTile;
  // FiltParams in dynamic shared memory; Decimal128 programs anywhere take the 128-bit interpreter.  There is one filtered instantiation
  // per sink and interpreter, so DFGPU_PIPE_VAR (which picks among the unfiltered ones) does not apply; DFGPU_PIPE_BLOCKS_PER_SM does.
  if (pipeline_has_filters(p)) {
    DF_CHECK(!part, DFGPU_ERR_INVALID, "internal: the partitioned aggregate takes no stage filters");
    void (*kern)(const PipeParams*, int64_t, unsigned long long*) =
        pipeline_has_decimal(p) ? pipe_kernel<SINK, true, kVarFilt> : pipe_kernel<SINK, false, filt_var(SINK)>;
    if constexpr (SINK == SINK_OUTPUT_ANY)   // output bitmaps or 16-byte columns (OutValid)
      if (out_cols) kern = pipeline_has_decimal(p) ? pipe_kernel<SINK, true, kVarFilt | kVarOutCols> : pipe_kernel<SINK, false, filt_var(SINK) | kVarOutCols>;
    DF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FiltParams)));   // per device: on every launch
    static const int blocks_env_f = getenv("DFGPU_PIPE_BLOCKS_PER_SM") ? atoi(getenv("DFGPU_PIPE_BLOCKS_PER_SM")) : 0;
    int blocks_per_sm = blocks_env_f;
    if (blocks_per_sm <= 0) DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, kPipeThreads, sizeof(FiltParams)));
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)kNumSMs * std::max(1, blocks_per_sm));
    const std::string tname = pipe_timer(p, timer_name);
    KernelTimer kt(ctx, tname.c_str());
    kern<<<grid, kPipeThreads, sizeof(FiltParams), ctx->stream>>>((const PipeParams*)p->params_dev.ptr, n, p->counters.as<unsigned long long>());
    DF_LAUNCH_CHECK(ctx);
    return;
  }
  // programs that touch Decimal128 values run a second instantiation of the kernel (128-bit interpreter linked in): the integer
  // instantiation stays byte for byte what it was
  bool dec = p->has_pred && p->pred.has_decimal;
  for (const auto& ag : p->aggs) dec = dec || (ag.has_expr && ag.plan.has_decimal);
  const PipeParams* gp = (const PipeParams*)p->params_dev.ptr;
  unsigned long long* cnt = p->counters.as<unsigned long long>();
  const std::string tname = pipe_timer(p, timer_name);
  if constexpr (SINK == SINK_AGG || SINK == SINK_PACK) if (!dec && pp.ring_stages > 0 && !getenv("DFGPU_PIPE_VAR")) {
    constexpr int RV = SINK == SINK_AGG ? 64 | 8 : 64;   // ring + lane-paired REDs for the aggregate sink, ring alone for the pack sink
    // the partitioned aggregate: ring + records instead of lookups
    void (*kern)(const PipeParams*, int64_t, unsigned long long*) = SINK == SINK_AGG && part ? pipe_kernel<SINK_AGG, false, 64 | 128> : pipe_kernel<SINK, false, RV>;
    const int smem = kRingBarBytes + kPipeWarps * pp.ring_stages * pp.ring_bytes;
    // the attribute belongs to the current device: set on every launch (a host-side call), so any device and thread may launch
    DF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kRingBarBytes + ring_smem(SINK)));
    int blocks_per_sm = 0;
    DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, kPipeThreads, smem));
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)kNumSMs * std::max(1, blocks_per_sm));
    KernelTimer kt(ctx, tname.c_str());
    kern<<<grid, kPipeThreads, smem, ctx->stream>>>(gp, n, cnt);
    DF_LAUNCH_CHECK(ctx);
    p->m_ring_launches++;
    return;
  }
  DF_CHECK(!part, DFGPU_ERR_INVALID, "internal: the partitioned aggregate needs the ring-fed pipeline kernel");
  DF_CHECK(!p->has_right || (SINK == SINK_OUTPUT_ANY && out_cols), DFGPU_ERR_INVALID, "internal: RIGHT stages run the output kernel with bitmaps");
  if constexpr (SINK == SINK_OUTPUT_ANY) if (out_cols) {   // output bitmaps or 16-byte columns: the default bits of this sink plus OutValid
    void (*kern)(const PipeParams*, int64_t, unsigned long long*) = dec ? pipe_kernel<SINK, true, kVarOutCols> : pipe_kernel<SINK, false, 2 | kVarOutCols>;
    if (p->has_right) kern = dec ? pipe_kernel<SINK, true, kVarOutCols | kVarRight> : pipe_kernel<SINK, false, 2 | kVarOutCols | kVarRight>;
    int blocks_per_sm = 0;
    DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, kPipeThreads, 0));
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)kNumSMs * std::max(1, blocks_per_sm));
    KernelTimer kt(ctx, tname.c_str());
    kern<<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
    DF_LAUNCH_CHECK(ctx);
    return;
  }
  static const int blocks_env = getenv("DFGPU_PIPE_BLOCKS_PER_SM") ? atoi(getenv("DFGPU_PIPE_BLOCKS_PER_SM")) : 0;
  int blocks_per_sm = blocks_env;
  if (blocks_per_sm <= 0) {   // persistent blocks: exactly one resident wave (a second wave would start after the first finished)
    if (dec) DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, pipe_kernel<SINK, true>, kPipeThreads, 0));
    else DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, pipe_kernel<SINK, false>, kPipeThreads, 0));
    blocks_per_sm = std::max(1, blocks_per_sm);
  }
  const int grid = (int)std::min<int64_t>(ntiles, (int64_t)kNumSMs * blocks_per_sm);
  KernelTimer kt(ctx, tname.c_str());
  const int var_env = getenv("DFGPU_PIPE_VAR") ? atoi(getenv("DFGPU_PIPE_VAR")) : kPipeVarDefault;
  if (dec) pipe_kernel<SINK, true><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 1) pipe_kernel<SINK_AGG, false, 1><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 2) pipe_kernel<SINK_AGG, false, 2><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 3) pipe_kernel<SINK_AGG, false, 3><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 8) pipe_kernel<SINK_AGG, false, 8><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 9) pipe_kernel<SINK_AGG, false, 9><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 11) pipe_kernel<SINK_AGG, false, 11><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_AGG && var_env == 43) pipe_kernel<SINK_AGG, false, 43><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_PACK && (var_env & 32)) pipe_kernel<SINK_PACK, false, 34><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_PACK && (var_env & 2)) pipe_kernel<SINK_PACK, false, 2><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  else if (SINK == SINK_OUTPUT_ANY && (var_env & 2)) pipe_kernel<SINK_OUTPUT_ANY, false, 2><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);   // the multi-GPU plan's scans (the 256-bit loads were not measured on this sink)
  else pipe_kernel<SINK, false><<<grid, kPipeThreads, 0, ctx->stream>>>(gp, n, cnt);
  DF_LAUNCH_CHECK(ctx);
}

static void read_counters(dfgpu_pipeline* p, unsigned long long h[4]) {
  DF_CUDA(cudaMemcpyAsync(h, p->counters.ptr, 32, cudaMemcpyDeviceToHost, p->ctx->stream));
  DF_CUDA(cudaStreamSynchronize(p->ctx->stream));
}

static void upload_params(dfgpu_pipeline* p, const PipeParams& pp) {
  if (!p->params_dev.ptr) p->params_dev.alloc(p->ctx, sizeof(PipeParams));
  DF_CUDA(cudaMemcpyAsync(p->params_dev.ptr, &pp, sizeof(PipeParams), cudaMemcpyHostToDevice, p->ctx->stream));
  DF_CUDA(cudaStreamSynchronize(p->ctx->stream));   // `pp` lives on the caller's stack frame
}

// the output sink's columns for one push of n rows: a column has a (zeroed) bitmap exactly when its input column has one in this push
static std::vector<DCol> alloc_output(dfgpu_pipeline* p, const std::vector<DCol>& cols, int64_t n, OutValid* ov) {
  memset(ov, 0, sizeof(*ov));
  std::vector<DCol> part;
  for (size_t c = 0; c < p->out_cols.size(); ++c) {
    const int src = p->out_cols[c];
    const bool nullable = (src < (int)cols.size() && cols[src].validity) || is_right_field(p, src);
    DCol d = alloc_col(p->ctx, p->vtypes[src], n, nullable);
    if (nullable) { d.own_validity->zero(); ov->valid[c] = d.own_validity->as<uint32_t>(); }
    part.push_back(std::move(d));
  }
  return part;
}
// the output kernels with bitmaps and 16-byte columns (pipe_kernel VAR bit 512, pipe_output_cols_kernel) run only when a column needs them
static bool output_needs_cols(const dfgpu_pipeline* p, const OutValid* ov) {
  if (p->has_right) return true;   // the RIGHT instantiations are the bitmap ones
  for (size_t c = 0; c < p->out_cols.size(); ++c)
    if (ov->valid[c] || type_width(p->vtypes[p->out_cols[c]]) == 16) return true;
  return false;
}
// OutValid into the sink's block behind PipeParams (after fill_params: the stage filters' upload sizes the buffer past this block)
static void upload_out_valid(dfgpu_pipeline* p, const OutValid& ov) {
  const size_t bytes = kDenseParamsOff + sizeof(OutValid);
  if (p->params_dev.bytes < bytes) p->params_dev.alloc(p->ctx, bytes);
  DF_CUDA(cudaMemcpyAsync((char*)p->params_dev.ptr + kDenseParamsOff, &ov, sizeof(OutValid), cudaMemcpyHostToDevice, p->ctx->stream));
}

static void prepare_acc(dfgpu_pipeline* p) {
  if (p->acc_ready) return;
  dfgpu_lookup* l = p->stages[p->agg_stage].lookup;
  dfgpu_ctx* ctx = p->ctx;
  LookupDev t = lookup_dev(l);
  for (const PipeAgg& ag : p->aggs) {
    if (ag.func != DFGPU_AGG_MIN && ag.func != DFGPU_AGG_MAX) continue;
    unsigned long long init, init_hi = 0;
    const bool is_min = ag.func == DFGPU_AGG_MIN;
    if (ag.cls == C_DEC) { init = is_min ? ~0ull : 0ull; init_hi = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN; }   // i128::MAX / MIN
    else if (ag.cls == C_U64 || ag.cls == C_F64) init = is_min ? ~0ull : 0ull;   // Float64: f64_to_ordered keys
    else init = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN;
    if (l->cap) {
      lookup_init_acc_kernel<<<grid_for((int64_t)l->cap, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, ag.word, init); DF_LAUNCH_CHECK(ctx);
      if (ag.cls == C_DEC) { lookup_init_acc_kernel<<<grid_for((int64_t)l->cap, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, ag.word + 1, init_hi); DF_LAUNCH_CHECK(ctx); }
    }
  }
  p->acc_ready = true;
}

// A join-keyed aggregate sink or a FULL stage takes the accumulator words of `l`.  When an earlier one pushed into them (acc_written), its
// row counters, SUM / COUNT words and visited marks are still there: they go back to 0 here, one pass over the table timed as
// "lookup_acc_reset".  A lookup fresh from creation or dfgpu_lookup_clear launches nothing.  The pass is a strided memset: words
// [1 + payload, stride) of each record are one row of a 2D region whose pitch is the record (no kernel of the library's own).
static void claim_acc_words(dfgpu_lookup* l) {
  if (!l->acc_written) return;
  dfgpu_ctx* ctx = l->ctx;
  set_device(ctx);
  const int base = 1 + (l->has_payload ? 1 : 0);
  if (l->cap && base < l->stride) {
    KernelTimer kt(ctx, "lookup_acc_reset");
    DF_CUDA(cudaMemset2DAsync((char*)l->recs.ptr + (size_t)base * 8, (size_t)l->stride * 8, 0, (size_t)(l->stride - base) * 8, (size_t)l->cap, ctx->stream));
  }
  l->acc_written = false;
}

// ---- dense-group aggregate sink ----
static int dense_op(const PipeAgg& ag) {
  const bool wide = ag.cls == C_DEC, f = ag.cls == C_F64, u = ag.cls == C_U64;
  switch (ag.func) {
    case DFGPU_AGG_SUM: case DFGPU_AGG_AVG: return wide ? DO_ADD_128 : (f ? DO_ADD_F64 : DO_ADD_U64);
    case DFGPU_AGG_MIN: return wide ? DO_MIN_128 : (f || u ? DO_MIN_U64 : DO_MIN_S64);   // Float64: its f64_to_ordered key
    case DFGPU_AGG_MAX: return wide ? DO_MAX_128 : (f || u ? DO_MAX_U64 : DO_MAX_S64);
    default: return DO_NONE;
  }
}

// small domains keep one copy of the slots per warp: no atomics in the row loop, the warps of a block are folded at the flush
static bool dense_per_warp(const dfgpu_pipeline* p) { return (size_t)kPipeWarps * p->dense_slots * p->dense_words * 8 <= (size_t)kDenseWarpBytes; }

static void prepare_dense(dfgpu_pipeline* p) {
  if (p->dense_acc.ptr) return;
  const size_t words = (size_t)p->dense_slots * p->dense_words;
  std::vector<unsigned long long> init(words);
  for (size_t i = 0; i < words; ++i) init[i] = p->dense_ident[i % p->dense_words];
  p->dense_acc.alloc(p->ctx, words * 8);
  DF_CUDA(cudaMemcpyAsync(p->dense_acc.ptr, init.data(), words * 8, cudaMemcpyHostToDevice, p->ctx->stream));
  DF_CUDA(cudaStreamSynchronize(p->ctx->stream));   // `init` lives on this stack frame
}

// the dense sink's parameters for one batch: its aggregate programs are bound behind the predicate in pp's pool
static void fill_dense(dfgpu_pipeline* p, const std::vector<DCol>& cols, PipeParams* pp, DenseParams* dp) {
  memset(dp, 0, sizeof(*dp));
  std::vector<std::array<long long, 4>> terms;
  if (pp->pred_mode == 2 && conjunction_terms(p, kMaxTerms + kDenseMaxXTerms, &terms)) {   // a longer conjunction: the rest in DenseParams
    pp->pred_mode = 1; pp->n_terms = kMaxTerms; pp->pred_start = 0; pp->pred_n = 0;
    for (size_t t = 0; t < terms.size(); ++t) {
      const int k = (int)t - kMaxTerms;
      if (k < 0) { pp->term_col[t] = (int)terms[t][0]; pp->term_op[t] = (int)terms[t][1]; pp->term_uns[t] = (int)terms[t][2]; pp->term_lit[t] = terms[t][3]; }
      else { dp->xterm_col[k] = (int)terms[t][0]; dp->xterm_op[k] = (int)terms[t][1]; dp->xterm_uns[k] = (int)terms[t][2]; dp->xterm_lit[k] = terms[t][3]; }
    }
    dp->n_xterms = (int)terms.size() - kMaxTerms;
  }
  dp->per_warp = dense_per_warp(p) ? 1 : 0;
  int pool_used = pp->pred_mode == 2 ? pp->pred_start + pp->pred_n : 0;
  dp->n_keys = (int)p->dense_keys.size(); dp->n_aggs = (int)p->aggs.size(); dp->n_slots = p->dense_slots; dp->n_words = p->dense_words;
  for (size_t k = 0; k < p->dense_keys.size(); ++k) dp->key[k] = p->dense_keys[k];
  for (int w = 0; w < p->dense_words; ++w) dp->ident[w] = p->dense_ident[w];
  dp->acc = p->dense_acc.as<unsigned long long>();
  for (size_t a = 0; a < p->aggs.size(); ++a) {
    const PipeAgg& ag = p->aggs[a];
    DenseAgg& d = dp->agg[a];
    d.func = ag.func; d.op = dense_op(ag);
    d.f64_key = ag.cls == C_F64 && (ag.func == DFGPU_AGG_MIN || ag.func == DFGPU_AGG_MAX) ? 1 : 0;
    d.word = ag.func == DFGPU_AGG_COUNT ? -1 : ag.word;   // COUNT(x) is its non-null counter
    d.nn_word = ag.func == DFGPU_AGG_COUNT ? ag.word : ag.nn_word;
    if (ag.has_expr) {
      d.start = bind_pool(p, ag.plan, cols, pp, &pool_used); d.n = (int)ag.plan.nodes.size();
      d.small = plan_depth(ag.plan) <= 4 ? 1 : 0;
      if (d.small && plan_is_int_arith(p, ag.plan, cols)) d.small = 2;
      if (ag.plan.has_decimal) d.small = 3;
    }
  }
}

static bool pipeline_has_decimal(const dfgpu_pipeline* p) {
  bool dec = p->has_pred && p->pred.has_decimal;
  for (const auto& ag : p->aggs) dec = dec || (ag.has_expr && ag.plan.has_decimal);
  for (int s = 0; s < kMaxStages; ++s) dec = dec || (p->has_filt[s] && p->filt[s].has_decimal);
  return dec;
}

static int dense_smem(const dfgpu_pipeline* p) { return kDenseAccOff + (dense_per_warp(p) ? kPipeWarps : 1) * p->dense_slots * p->dense_words * 8; }

static int filt_smem_off(const dfgpu_pipeline* p) {
  if (p->sink == SINK_DENSE) return (dense_smem(p) + 15) / 16 * 16;
  if (p->sink == SINK_HASH) return (int)((sizeof(HashParams) + 15) / 16 * 16);
  return 0;
}

static void launch_dense(dfgpu_pipeline* p, const PipeParams& pp, const DenseParams& dp, int64_t n) {
  dfgpu_ctx* ctx = p->ctx;
  if (!p->params_dev.ptr) p->params_dev.alloc(ctx, kDenseParamsOff + sizeof(DenseParams));
  DF_CUDA(cudaMemcpyAsync(p->params_dev.ptr, &pp, sizeof(PipeParams), cudaMemcpyHostToDevice, ctx->stream));
  DF_CUDA(cudaMemcpyAsync((char*)p->params_dev.ptr + kDenseParamsOff, &dp, sizeof(DenseParams), cudaMemcpyHostToDevice, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));   // `pp` and `dp` live on the caller's stack frame
  // programs that touch Decimal128 values run the instantiation with the 128-bit interpreter
  void (*kern)(const PipeParams*, int64_t, unsigned long long*) = pipeline_has_decimal(p) ? pipe_kernel<SINK_DENSE, true> : pipe_kernel<SINK_DENSE, false>;
  if (p->has_right) kern = pipeline_has_decimal(p) ? pipe_kernel<SINK_DENSE, true, kVarRight> : pipe_kernel<SINK_DENSE, false, kVarRight>;   // no stage filters
  int smem = kDenseAccOff + (dp.per_warp ? kPipeWarps : 1) * p->dense_slots * p->dense_words * 8;
  if (pipeline_has_filters(p)) {   // the stage filters behind the slots
    kern = pipeline_has_decimal(p) ? pipe_kernel<SINK_DENSE, true, kVarFilt> : pipe_kernel<SINK_DENSE, false, filt_var(SINK_DENSE)>;
    smem = filt_smem_off(p) + (int)sizeof(FiltParams);
  }
  DF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));   // per device: set on every launch
  int blocks_per_sm = 0;
  DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, kPipeThreads, smem));
  const int64_t ntiles = (n + kPipeTile - 1) / kPipeTile;
  const int grid = (int)std::min<int64_t>(ntiles, (int64_t)kNumSMs * std::max(1, blocks_per_sm));
  const std::string tname = pipe_timer(p, "pipeline_dense");
  KernelTimer kt(ctx, tname.c_str());
  kern<<<grid, kPipeThreads, smem, ctx->stream>>>((const PipeParams*)p->params_dev.ptr, n, p->counters.as<unsigned long long>());
  DF_LAUNCH_CHECK(ctx);
  if (!dp.per_warp) p->m_dense_block_launches++;
}

// The partitioned aggregate (pipe_kernel VAR bit 128, then radix_partition and pipe_probe_agg_kernel) trades phase B's dependent DRAM
// lookup + RED per survivor for streamed records and L2-resident probes.  It serves a batch that takes the ring kernel, whose aggregate
// stage is the only hash stage phase B probes and exceeds L2 (the rule that gives it a Bloom filter), with one integer SUM over this
// batch's columns: no payload field, no NULLs, no non-null counter — TPC-H Q3 over Int64 money.  Returns the stage's table bytes, 0 when
// the batch keeps the direct probe.  force_parts >= 2 (a test hook) admits tables of any size.
static size_t partitioned_table_bytes(const dfgpu_pipeline* p, const PipeParams& pp, int force_parts) {
  if (pp.ring_stages == 0 || pipeline_has_decimal(p) || getenv("DFGPU_PIPE_VAR")) return 0;   // launch_pipe's ring kernel runs
  if (pipeline_has_filters(p)) return 0;
  if (pp.agg_stage < 0 || p->left_kind) return 0;
  for (int s = 0; s < pp.n_stages; ++s)
    if (s != pp.agg_stage && pp.stage[s].lk.mode == LK_HASH && pp.stage[s].kind != kStageMaybe) return 0;
  const StageDev& st = pp.stage[pp.agg_stage];
  if (st.kind != DFGPU_STAGE_INNER || st.lk.mode != LK_HASH || st.lk.cap == 0) return 0;
  const AggDef& a = pp.agg[0];
  if (pp.n_aggs != 1 || a.small != 2 || a.func != DFGPU_AGG_SUM || a.cls == C_F64 || a.cls == C_DEC || a.nn_word >= 0) return 0;
  for (int i = 0; i < a.n; ++i) if (pp.pool[a.start + i].kind == kExprExt) return 0;
  const size_t bytes = (size_t)st.lk.cap * st.lk.stride * 8;
  return bytes > kL2TableBytes || force_parts >= 2 ? bytes : 0;
}

// ---- hash-keyed aggregate sink ----
// (re)allocate the table with new_cap regular records: every record starts as the identity words, then the claimed records and the
// side record of the old table move over
static void hash_grow(dfgpu_pipeline* p, uint64_t new_cap) {
  dfgpu_ctx* ctx = p->ctx;
  DF_CHECK(new_cap < 0xFFFFFFFEull, DFGPU_ERR_UNSUPPORTED, "pipeline hash aggregate: the group table would exceed 2^32 records");
  const int st = p->hash_stride;
  HashIdent id;
  memset(&id, 0, sizeof(id));
  for (int w = 0; w < st; ++w) id.w[w] = p->hash_ident[w];
  DevBuf nrecs(ctx, (size_t)(new_cap + 1) * st * 8);
  hash_init_kernel<<<grid_for((int64_t)(new_cap + 1) * st, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(nrecs.as<unsigned long long>(), new_cap + 1, st, id);
  DF_LAUNCH_CHECK(ctx);
  if (p->hash_cap > 0) {
    hash_rehash_kernel<<<grid_for((int64_t)p->hash_cap, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(p->hash_recs.as<unsigned long long>(), p->hash_cap,
                                                                                                  nrecs.as<unsigned long long>(), new_cap, st);
    DF_LAUNCH_CHECK(ctx);
    DF_CUDA(cudaMemcpyAsync(nrecs.as<unsigned long long>() + new_cap * st, p->hash_recs.as<unsigned long long>() + p->hash_cap * st, (size_t)st * 8,
                            cudaMemcpyDeviceToDevice, ctx->stream));
    p->m_group_rehashes++;
  }
  p->hash_recs = std::move(nrecs); p->hash_cap = new_cap;
}

// One push in row chunks (the overflow list holds one chunk's row numbers).  Before a chunk the table grows x4 once groups x 2 > capacity;
// after a launch that deferred rows the table grows x4 and those rows, gathered into one compact batch, go through the same kernel again
// (each round raises the claim budget to 5/8 of four times the capacity, above the groups already claimed, so every round claims more).
static void hash_push(dfgpu_pipeline* p, const std::vector<DCol>& cols, int64_t n) {
  dfgpu_ctx* ctx = p->ctx;
  DF_CHECK(n < 0xFFFFFFFFll, DFGPU_ERR_UNSUPPORTED, "pipeline: a batch must have < 2^32-1 rows");
  if (!p->hash_recs.ptr) {
    p->hash_ngroups.alloc(ctx, 8);
    p->hash_ngroups.zero();
    hash_grow(p, std::max<uint64_t>(1024, (uint64_t)p->hash_cap_hint * 2));
  }
  const size_t pbytes = kDenseParamsOff + sizeof(HashParams);
  if (p->params_dev.bytes < pbytes) p->params_dev.alloc(ctx, pbytes);
  // programs that touch Decimal128 values run the instantiation with the 128-bit interpreter
  void (*kern)(const PipeParams*, int64_t, unsigned long long*) = pipeline_has_decimal(p) ? pipe_kernel<SINK_HASH, true> : pipe_kernel<SINK_HASH, false>;
  if (p->has_right) kern = pipeline_has_decimal(p) ? pipe_kernel<SINK_HASH, true, kVarRight> : pipe_kernel<SINK_HASH, false, kVarRight>;   // no stage filters
  int smem = (int)sizeof(HashParams);
  if (pipeline_has_filters(p)) {   // the stage filters behind HashParams
    kern = pipeline_has_decimal(p) ? pipe_kernel<SINK_HASH, true, kVarFilt> : pipe_kernel<SINK_HASH, false, filt_var(SINK_HASH)>;
    smem = filt_smem_off(p) + (int)sizeof(FiltParams);
    DF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));   // per device: on every launch
  }
  int blocks_per_sm = 0;
  DF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, kPipeThreads, smem));
  const std::string tname = pipe_timer(p, "pipeline_hash");
  constexpr int64_t kMaxChunk = 1ll << 26;
  int64_t chunk = std::max<int64_t>((int64_t)p->hash_cap / 2, 1 << 20);
  DevBuf overflow;
  unsigned long long groups = 0;
  DF_CUDA(cudaMemcpyAsync(&groups, p->hash_ngroups.ptr, 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  const std::vector<DCol> packed = p->packed;   // the batch's packed keys, sliced and replayed with the input columns
  for (int64_t done = 0; done < n; done += chunk, chunk = std::min(chunk * 4, kMaxChunk)) {
    const int64_t m = std::min(chunk, n - done);
    if (groups * 2 > p->hash_cap) hash_grow(p, p->hash_cap * 4);
    if (overflow.bytes < (size_t)m * 4) overflow.alloc(ctx, (size_t)m * 4);
    std::vector<DCol> batch;
    for (const DCol& c : cols) batch.push_back(m == n ? c : slice_column(c, done, m));
    p->packed.clear();
    for (const DCol& c : packed) p->packed.push_back(m == n ? c : slice_column(c, done, m));
    int64_t rows = m;
    while (true) {
      PipeParams pp;
      fill_params(p, batch, &pp);
      pp.ring_stages = 0;
      HashParams hp;
      memset(&hp, 0, sizeof(hp));
      hp.n_keys = (int)p->hash_keys.size(); hp.stride = p->hash_stride;
      for (size_t k = 0; k < p->hash_keys.size(); ++k) hp.key[k] = p->hash_keys[k];
      hp.recs = p->hash_recs.as<unsigned long long>(); hp.cap = p->hash_cap;
      hp.ngroups = p->hash_ngroups.as<unsigned long long>(); hp.group_limit = p->hash_cap / 8 * 5;   // the claim budget, as dfgpu_agg's
      hp.overflow = overflow.as<uint32_t>(); hp.overflow_count = p->counters.as<unsigned long long>() + 4;
      DF_CUDA(cudaMemcpyAsync(p->params_dev.ptr, &pp, sizeof(PipeParams), cudaMemcpyHostToDevice, ctx->stream));
      DF_CUDA(cudaMemcpyAsync((char*)p->params_dev.ptr + kDenseParamsOff, &hp, sizeof(HashParams), cudaMemcpyHostToDevice, ctx->stream));
      p->counters.zero();
      const int grid = (int)std::min<int64_t>((rows + kPipeTile - 1) / kPipeTile, (int64_t)kNumSMs * std::max(1, blocks_per_sm));
      {
        KernelTimer kt(ctx, tname.c_str());
        kern<<<grid, kPipeThreads, smem, ctx->stream>>>((const PipeParams*)p->params_dev.ptr, rows, p->counters.as<unsigned long long>());
        DF_LAUNCH_CHECK(ctx);
      }
      unsigned long long h8[8];
      DF_CUDA(cudaMemcpyAsync(h8, p->counters.ptr, 64, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaMemcpyAsync(&groups, p->hash_ngroups.ptr, 8, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));   // also: `pp` and `hp` live on this stack frame
      check_errors(h8[3]);
      if (h8[2] & 4) throw Error(DFGPU_ERR_INVALID, "pipeline hash aggregate: a group column declared non-nullable holds a NULL");
      p->m_sink_rows += (int64_t)h8[0];
      const int64_t deferred = (int64_t)h8[4];
      if (deferred == 0) break;
      hash_grow(p, p->hash_cap * 4);   // x4 per round: the deferred rows may hold few groups, so their count does not size the table
      std::vector<DCol> replay;
      for (const DCol& c : batch) replay.push_back(take_column(ctx, c, overflow.as<uint32_t>(), deferred, false));
      batch = std::move(replay);
      for (DCol& c : p->packed) c = take_column(ctx, c, overflow.as<uint32_t>(), deferred, false);
      rows = deferred;
      p->m_replayed_rows += deferred;
    }
  }
}

// A LEFT / LEFT_ANTI join emits its build rows with a NULL key too, but the build sink never inserts them
static void check_left_build(const dfgpu_pipeline* p) {
  if (p->left_kind)
    DF_CHECK(p->stages[p->agg_stage].lookup->null_keys == 0, DFGPU_ERR_UNSUPPORTED,
             "pipeline: a LEFT / LEFT_ANTI stage needs a build side without NULL keys (they are not in the lookup) — use dfgpu_hashjoin");
  if (p->full_stage >= 0)   // the same for a Full join's build rows
    DF_CHECK(p->stages[p->full_stage].lookup->null_keys == 0, DFGPU_ERR_UNSUPPORTED,
             "pipeline: a FULL stage needs a build side without NULL keys (they are not in the lookup) — use dfgpu_hashjoin");
}

// rows of a build push whose key is NULL, from the key column's validity (before the predicate: an upper bound of the rows dropped for it)
static int64_t count_null_keys(dfgpu_ctx* ctx, const DCol& c) {
  if (!c.validity || c.length == 0) return 0;
  DevBuf mm(ctx, 24);
  mm.zero();
  col_minmax_kernel<<<grid_for(c.length, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(col_ref(c), c.length, type_is_unsigned_int(c.type) ? 1 : 0,
                                                                                  mm.as<unsigned long long>());
  DF_LAUNCH_CHECK(ctx);
  unsigned long long h[3];
  DF_CUDA(cudaMemcpyAsync(h, mm.ptr, 24, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  return c.length - (int64_t)h[2];
}

// One launch packs every composite key of the batch (composite_key.cu) into p->packed, timed as "pipe_keys:<name>"
static void pack_batch_keys(dfgpu_pipeline* p, const std::vector<DCol>& cols, int64_t n) {
  p->packed.clear();
  PackKeysParams kp;
  memset(&kp, 0, sizeof(kp));
  auto add = [&](const dfgpu_lookup* l, const std::vector<int>& key_cols, bool build) {
    PackedKey& k = kp.key[kp.n_keys++];
    k.n_parts = (int)key_cols.size();
    for (size_t g = 0; g < key_cols.size(); ++g) {
      const DCol& c = cols[key_cols[g]];
      KeyPart& kc = k.part[g];
      kc.ptr = c.values; kc.valid = c.validity; kc.voff = c.offset; kc.width = type_width(c.type); kc.sgn = type_is_signed_int(c.type) ? 1 : 0;
      kc.kmin = (unsigned long long)l->comp_min[g]; kc.range = l->comp_range[g]; kc.stride = l->comp_stride[g];
    }
    DCol d = alloc_col(p->ctx, DFGPU_INT64, n, build);
    if (build) d.null_count = -1;
    k.out = d.own_values->as<unsigned long long>(); k.out_valid = build ? d.own_validity->as<uint8_t>() : nullptr; k.domain = l->domain;
    p->packed.push_back(std::move(d));
  };
  for (size_t s = 0; s < p->stages.size(); ++s)
    if (!p->stage_keys[s].empty()) add(p->stages[s].lookup, p->stage_keys[s], false);
  if (!p->bkey_cols.empty()) {
    add(p->target, p->bkey_cols, true);
    if (!p->key_flags.ptr) { p->key_flags.alloc(p->ctx, 16); p->key_flags.zero(); }
    kp.flags = p->key_flags.as<unsigned long long>();
  }
  if (kp.n_keys == 0) return;
  const std::string tname = p->name.empty() ? std::string("pipe_keys") : "pipe_keys:" + p->name;
  KernelTimer kt(p->ctx, tname.c_str());
  pack_keys(p->ctx, kp, n);
}

static void pipeline_push(dfgpu_pipeline* p, const std::vector<DCol>& cols) {
  DF_CHECK(!p->finished, DFGPU_ERR_STATE, "push after finish");
  DF_CHECK(p->sink != SINK_NONE, DFGPU_ERR_STATE, "pipeline: choose a sink before the first push");
  DF_CHECK(cols.size() == p->in_types.size(), DFGPU_ERR_INVALID, "pipeline input column count mismatch");
  for (size_t s = 0; s < p->stages.size(); ++s)
    DF_CHECK(p->stages[s].lookup->comp_types.empty() || !p->stage_keys[s].empty(), DFGPU_ERR_STATE,
             "pipeline: a stage over a composite-key lookup needs dfgpu_pipeline_set_stage_keys before the first push");
  check_left_build(p);
  p->pushed = true;
  dfgpu_ctx* ctx = p->ctx;
  set_device(ctx);
  const int64_t n = cols.empty() ? 0 : cols[0].length;
  for (size_t c = 0; c < cols.size(); ++c) {
    DF_CHECK(cols[c].type == p->in_types[c], DFGPU_ERR_INVALID, "pipeline input column type mismatch");
    DF_CHECK(cols[c].length == n, DFGPU_ERR_INVALID, "pipeline input ragged columns");
    DF_CHECK(cols[c].type != DFGPU_BOOL && (type_width(cols[c].type) <= 8 || type_is_decimal(cols[c].type)), DFGPU_ERR_UNSUPPORTED,
             "pipeline: fixed-width columns of <= 8 bytes (and Decimal128 inside expressions) only");
  }
  if (!p->in_tail) p->m_input_rows += n;   // the Full join's unmatched build rows are not input rows
  if (n == 0) return;
  if (p->sink == SINK_AGG) p->stages[p->agg_stage].lookup->acc_written = true;
  if (p->full_stage >= 0) p->stages[p->full_stage].lookup->acc_written = true;
  if (!p->counters.ptr) p->counters.alloc(ctx, 64);
  if (!p->in_tail) pack_batch_keys(p, cols, n);   // the tail brings its keys in p->packed
  PipeParams pp;
  unsigned long long h[4];
  if (p->sink == SINK_BUILD) {
    dfgpu_lookup* t = p->target;
    if (p->bkey_cols.empty()) t->null_keys += count_null_keys(ctx, cols[p->bkey_col]);   // a composite key's: pack_keys counts them
    if (t->mode == LK_HASH && !t->filter_only && (uint64_t)(t->rows + n) * 2 > t->cap) {
      // the batch may not fit at load factor 0.5 and nobody knows how many rows survive: ONE pass evaluates the pipeline and leaves
      // the survivors as packed {key, payload} records; the table is sized for exactly that many and the records are inserted by a
      // dense kernel (no second scan of the input).
      fill_params(p, cols, &pp);
      DevBuf recs(ctx, (size_t)n * 16);
      p->counters.zero();
      pp.out_dst[0] = recs.ptr;
      pp.out_counter = p->counters.as<unsigned long long>() + 4;
      upload_params(p, pp);
      launch_pipe<SINK_PACK>(p, pp, n, "pipeline_build");
      unsigned long long h8[8];
      DF_CUDA(cudaMemcpyAsync(h8, p->counters.ptr, 64, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
      check_errors(h8[3]);
      const int64_t packed = (int64_t)h8[4];
      lookup_reserve(t, t->rows + packed);
      p->counters.zero();
      const int unique = (t->has_payload || t->opt.n_acc_words > 0) ? 1 : 0;
      // a table larger than L2 takes its records one slot range at a time: partitioned first, like the aggregate sink's probe records
      // (DFGPU_PIPE_RADIX_PARTS, a test hook, forces P and this path on small tables)
      const size_t table_bytes = (size_t)t->cap * t->stride * 8;
      const int force_parts = getenv("DFGPU_PIPE_RADIX_PARTS") ? atoi(getenv("DFGPU_PIPE_RADIX_PARTS")) : 0;
      DevBuf parts, meta;   // released after read_counters' synchronise
      if (packed > 0 && (table_bytes > kL2TableBytes || force_parts >= 2)) {
        parts.alloc(ctx, (size_t)packed * 16); meta.alloc(ctx, (size_t)(kRadixMetaWords + 1) * 8);
        meta.zero();
        {
          KernelTimer kt(ctx, "lookup_partition");
          radix_partition_records(ctx, recs.ptr, packed, table_bytes, force_parts, parts.ptr, meta.as<unsigned long long>());
        }
        recs.release();
        KernelTimer kt(ctx, "lookup_insert");   // both kernels: the time of the insert the unpartitioned path makes in one
        LookupDev d = lookup_dev(t);
        if (d.bloom) {
          lookup_filter_records_kernel<<<grid_for(packed, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(d, parts.as<ulonglong2>(), packed);
          DF_LAUNCH_CHECK(ctx);
          d.bloom = nullptr; d.coarse = nullptr;
        }
        lookup_insert_part_kernel<<<kNumSMs * 8, 256, 0, ctx->stream>>>(d, parts.as<ulonglong2>(), packed, unique, (unsigned int*)(meta.as<unsigned long long>() + kRadixMetaWords),
                                                                     p->counters.as<unsigned long long>());
        DF_LAUNCH_CHECK(ctx);
        p->m_partitioned_inserts++;
      } else if (packed > 0) {
        KernelTimer kt(ctx, "lookup_insert");
        lookup_insert_records_kernel<<<grid_for(packed, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(lookup_dev(t), (const ulonglong2*)recs.ptr, packed, unique,
                                                                                                   p->counters.as<unsigned long long>());
        DF_LAUNCH_CHECK(ctx);
      }
      read_counters(p, h);
      h[0] = h8[0];
    } else {
      fill_params(p, cols, &pp);
      upload_params(p, pp);
      p->counters.zero();
      launch_pipe<SINK_BUILD>(p, pp, n, "pipeline_build");
      read_counters(p, h);
      check_errors(h[3]);
    }
    if (h[2] & 2) throw Error(DFGPU_ERR_INVALID, "lookup build: a key lies outside the declared key range (or is the reserved all-ones value)");
    if (h[2] & 1) throw Error(DFGPU_ERR_UNSUPPORTED, "lookup build: duplicate build keys — the fused lookup needs unique keys, use dfgpu_hashjoin");
    t->rows += (int64_t)h[1];
    p->m_sink_rows += (int64_t)h[0];
  } else if (p->sink == SINK_AGG) {
    prepare_acc(p);
    fill_params(p, cols, &pp);
    // test hooks: DFGPU_PIPE_RADIX_PARTS forces the partition count (and the partitioned path on small tables), DFGPU_PIPE_RADIX_CAP the
    // record buffer's capacity
    const int force_parts = getenv("DFGPU_PIPE_RADIX_PARTS") ? atoi(getenv("DFGPU_PIPE_RADIX_PARTS")) : 0;
    const size_t part_bytes = partitioned_table_bytes(p, pp, force_parts);
    DevBuf rkeys, rvals, recs, meta, folded;   // released after read_counters' synchronise
    if (part_bytes) {
      // survivors are a fraction of the rows (Q3: ~5 %); the buffer holds one in eight, rows past it take the in-kernel fallback
      int64_t cap = std::min<int64_t>(n, std::max<int64_t>(n / 8, 1 << 20));
      if (getenv("DFGPU_PIPE_RADIX_CAP")) cap = std::min<int64_t>(cap, atoll(getenv("DFGPU_PIPE_RADIX_CAP")));
      cap = std::max<int64_t>(cap, 1);
      rkeys.alloc(ctx, (size_t)cap * 8); rvals.alloc(ctx, (size_t)cap * 8);
      pp.out_dst[0] = rkeys.ptr; pp.out_dst[1] = rvals.ptr; pp.out_counter = p->counters.as<unsigned long long>() + 4; pp.target.cap = (uint64_t)cap;
      // Pass 1 tests the filter once per date-qualified row, a random 8-byte load each.  At 16 bits per key the filter (Q3 SF100:
      // 29 MB) does not stay in L2 beside the stream; folded once to 8 bits per key it does, and a false positive here costs only a
      // record that finds nothing in an L2-resident probe.  The lookup keeps the exact filter for the direct probe, where a false
      // positive costs a DRAM access.  Folding twice (4 bits per key, ~18 % false positives) would overflow Q3 SF100's record buffer.
      LookupDev& lk = pp.stage[pp.agg_stage].lk;
      if (lk.bloom) {
        DF_CHECK(lk.bloom_blocks % 2 == 0 && !lk.coarse, DFGPU_ERR_INVALID, "internal: the partitioned aggregate folds an even-sized exact filter");
        const uint64_t half = lk.bloom_blocks / 2;
        folded.alloc(ctx, (size_t)half * 8);
        {
          KernelTimer kt(ctx, "pipe_filter_fold");
          bloom_fold_kernel<<<grid_for((int64_t)half, 256, kNumSMs * 8), 256, 0, ctx->stream>>>((const ulonglong2*)lk.bloom, folded.as<unsigned long long>(), half);
          DF_LAUNCH_CHECK(ctx);
        }
        lk.bloom = folded.as<unsigned long long>(); lk.bloom_blocks = half;
      }
    }
    upload_params(p, pp);
    p->counters.zero();
    launch_pipe<SINK_AGG>(p, pp, n, "pipeline_agg", part_bytes != 0);
    if (part_bytes) {
      unsigned long long h8[8];
      DF_CUDA(cudaMemcpyAsync(h8, p->counters.ptr, 64, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
      check_errors(h8[3]);
      const int64_t m = std::min<int64_t>((int64_t)h8[4], (int64_t)pp.target.cap);
      p->m_partitioned_records += m;
      if (m > 0) {
        recs.alloc(ctx, (size_t)m * 16); meta.alloc(ctx, (size_t)(kRadixMetaWords + 1) * 8);
        meta.zero();
        {
          KernelTimer kt(ctx, "pipe_partition");
          radix_partition(ctx, rkeys.as<unsigned long long>(), rvals.as<unsigned long long>(), m, part_bytes, force_parts, recs.ptr, meta.as<unsigned long long>());
        }
        {
          KernelTimer kt(ctx, "pipe_probe_agg");
          pipe_probe_agg_kernel<<<kNumSMs * 8, 256, 0, ctx->stream>>>(recs.as<ulonglong2>(), m, pp.stage[pp.agg_stage].lk, pp.rows_word, pp.agg[0].word,
                                                                      (unsigned int*)(meta.as<unsigned long long>() + kRadixMetaWords), p->counters.as<unsigned long long>());
          DF_LAUNCH_CHECK(ctx);
        }
      }
      p->m_partitioned_launches++;
    }
    read_counters(p, h);
    check_errors(h[3]);
    p->m_sink_rows += (int64_t)h[0];
  } else if (p->sink == SINK_HASH) {
    hash_push(p, cols, n);
  } else if (p->sink == SINK_DENSE) {
    prepare_dense(p);
    fill_params(p, cols, &pp);
    DenseParams dp;
    fill_dense(p, cols, &pp, &dp);
    p->counters.zero();
    launch_dense(p, pp, dp, n);
    read_counters(p, h);
    check_errors(h[3]);
    if (h[2] & 2) throw Error(DFGPU_ERR_INVALID, "pipeline dense aggregate: a group key lies outside its declared range");
    p->m_sink_rows += (int64_t)h[0];
  } else if (!p->out_ordered) {   // SINK_OUTPUT, row order unspecified: the two-phase kernel, one global reservation per 128 survivors
    DF_CHECK(n < 0xFFFFFFFFll, DFGPU_ERR_UNSUPPORTED, "pipeline: a batch must have < 2^32-1 rows");
    fill_params(p, cols, &pp);
    OutValid ov;
    std::vector<DCol> part = alloc_output(p, cols, n, &ov);
    pp.n_out = (int)p->out_cols.size();
    for (int c = 0; c < pp.n_out; ++c) {
      const int src = p->out_cols[c];
      pp.out_src[c] = src; pp.out_width[c] = type_width(p->vtypes[src]); pp.out_dst[c] = part[c].own_values->ptr;
    }
    const bool out_cols = output_needs_cols(p, &ov);
    if (out_cols) upload_out_valid(p, ov);
    p->counters.zero();
    pp.out_counter = p->counters.as<unsigned long long>() + 4;
    upload_params(p, pp);
    launch_pipe<SINK_OUTPUT_ANY>(p, pp, n, "pipeline_output", false, out_cols);
    unsigned long long h8[8];
    DF_CUDA(cudaMemcpyAsync(h8, p->counters.ptr, 64, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    check_errors(h8[3]);
    const int64_t kept = (int64_t)h8[4];
    p->m_sink_rows += kept;
    if (kept > 0) {
      for (auto& c : part) c.length = kept;
      p->out_parts.push_back(std::move(part));
      p->out_rows_pending += kept;
    }
  } else {  // SINK_OUTPUT, input order preserved
    DF_CHECK(n < 0xFFFFFFFFll, DFGPU_ERR_UNSUPPORTED, "pipeline: a batch must have < 2^32-1 rows");
    for (auto& st : p->stages) DF_CHECK(st.kind != DFGPU_STAGE_MAYBE, DFGPU_ERR_UNSUPPORTED, "pipeline: MAYBE stages feed an exchange — use the unordered output sink");
    fill_params(p, cols, &pp);
    OutValid ov;
    std::vector<DCol> part = alloc_output(p, cols, n, &ov);
    const bool out_cols = output_needs_cols(p, &ov);
    if (out_cols) upload_out_valid(p, ov);
    upload_params(p, pp);
    p->counters.zero();
    OutCols oc;
    memset(&oc, 0, sizeof(oc));
    oc.n = (int)p->out_cols.size();
    for (int c = 0; c < oc.n; ++c) {
      const int src = p->out_cols[c];
      oc.src[c] = src; oc.width[c] = type_width(p->vtypes[src]); oc.dst[c] = part[c].own_values->ptr;
    }
    const int64_t nt = (n + kPipeTile - 1) / kPipeTile;
    DevBuf desc(ctx, (size_t)nt * 8 + 32);
    desc.zero();
    unsigned long long* totals = (unsigned long long*)((char*)desc.ptr + (size_t)nt * 8);
    unsigned int* counter = (unsigned int*)(totals + 2);
    {
      const std::string tname = p->in_tail ? tail_timer(p) : std::string("pipeline_output");
      KernelTimer kt(ctx, tname.c_str());
      if (p->has_right) {   // RIGHT stages: the survivors' payload validity bits in the dynamic shared memory
        pipe_output_right_kernel<<<(int)nt, kPipeThreads, kPipeTile, ctx->stream>>>((const PipeParams*)p->params_dev.ptr, n, oc, desc.as<unsigned long long>(), counter, totals,
                                                                                   p->counters.as<unsigned long long>());
      } else if (out_cols) {   // the instantiations above stay as they were for columns without bitmaps, <= 8 bytes wide
        const bool filt = pipeline_has_filters(p);
        void (*kern)(const PipeParams*, int64_t, OutCols, unsigned long long*, unsigned int*, unsigned long long*, unsigned long long*) =
            filt ? pipe_output_cols_kernel<true> : pipe_output_cols_kernel<false>;
        if (filt) DF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FiltParams)));
        kern<<<(int)nt, kPipeThreads, filt ? sizeof(FiltParams) : 0, ctx->stream>>>((const PipeParams*)p->params_dev.ptr, n, oc, desc.as<unsigned long long>(), counter, totals,
                                                                                   p->counters.as<unsigned long long>());
      } else if (pipeline_has_filters(p)) {
        DF_CUDA(cudaFuncSetAttribute(pipe_output_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FiltParams)));
        pipe_output_kernel<true><<<(int)nt, kPipeThreads, sizeof(FiltParams), ctx->stream>>>((const PipeParams*)p->params_dev.ptr, n, oc, desc.as<unsigned long long>(), counter,
                                                                                           totals, p->counters.as<unsigned long long>());
      } else
        pipe_output_kernel<false><<<(int)nt, kPipeThreads, 0, ctx->stream>>>((const PipeParams*)p->params_dev.ptr, n, oc, desc.as<unsigned long long>(), counter, totals, p->counters.as<unsigned long long>());
      DF_LAUNCH_CHECK(ctx);
    }
    unsigned long long tot[2];
    DF_CUDA(cudaMemcpyAsync(tot, totals, 16, cudaMemcpyDeviceToHost, ctx->stream));
    read_counters(p, h);
    check_errors(h[3]);
    const int64_t kept = (int64_t)tot[0];
    p->m_sink_rows += kept;
    if (kept > 0) {
      for (auto& c : part) c.length = kept;
      p->out_parts.push_back(std::move(part));
      p->out_rows_pending += kept;
    }
  }
}

static void emit_sliced(dfgpu_pipeline* p, std::vector<DCol>& merged, int64_t rows) {
  const int64_t bs = p->batch_size > 0 ? p->batch_size : std::max<int64_t>(rows, 1);
  for (int64_t pos = 0; pos < rows; pos += bs) {
    const int64_t len = std::min<int64_t>(bs, rows - pos);
    BatchPtr b(new dfgpu_batch());
    b->ctx = p->ctx; b->rows = len; b->host = false;
    for (auto& c : merged) b->cols.push_back((pos == 0 && len == rows) ? c : slice_column(c, pos, len));
    p->m_output_rows += len;
    p->outq.push_back(std::move(b));
  }
}

// one column (Single) or the state columns (Partial) per aggregate, read from the accumulator words the aggregate addresses.  `left`: the
// records are a LEFT join's build rows, and one no probe row reached stands for its NULL-padded row: COUNT(*) 1, COUNT(x) 0 and every other
// value NULL (the arguments propagate NULL).  Such a record's row counter is 0, so the counter serves as the non-null counter of a SUM /
// MIN / MAX that has none; AVG's count is 0 anyway.
template <class Add>
static void add_agg_columns(const std::vector<PipeAgg>& aggs, int rows_word, bool partial, bool left, Add& add) {
  for (const PipeAgg& ag : aggs) {
    EmitCol e; memset(&e, 0, sizeof(e));
    e.nn_word = -1;
    const int sum_type = ag.cls == C_F64 ? DFGPU_FLOAT64 : (ag.cls == C_U64 ? DFGPU_UINT64 : DFGPU_INT64);   // sum.rs:232-261
    const int nn_word = left && ag.nn_word < 0 ? rows_word : ag.nn_word;
    switch (ag.func) {
      case DFGPU_AGG_COUNT_STAR: e.kind = left ? 9 : 4; e.word = rows_word; add(DFGPU_INT64, false, e); break;
      case DFGPU_AGG_COUNT: e.kind = 4; e.word = ag.word; add(DFGPU_INT64, false, e); break;
      case DFGPU_AGG_SUM:
        if (ag.cls == C_DEC) {   // Sum::return_type: Decimal128(min(38, p + 10), s) (sum.rs:247-249); the Partial state has the same type
          e.kind = 5; e.word = ag.word; e.nn_word = nn_word;
          add(dec_type(std::min(38, dec_precision(ag.arg_type) + 10), dec_scale(ag.arg_type)), nn_word >= 0, e);
        } else { e.kind = 2; e.word = ag.word; e.nn_word = nn_word; add(sum_type, nn_word >= 0, e); }
        break;
      case DFGPU_AGG_MIN: case DFGPU_AGG_MAX:   // the argument's type; Decimal128 takes two words
        e.kind = ag.cls == C_DEC ? 5 : 2; e.word = ag.word; e.nn_word = nn_word; e.f64_key = ag.cls == C_F64;
        add(ag.arg_type, nn_word >= 0, e);
        break;
      case DFGPU_AGG_AVG:
        if (ag.cls == C_DEC) {   // Avg::return_type: Decimal128(min(38, p + 4), min(38, s + 4)) (average.rs); Single modes only
          const int tp = std::min(38, dec_precision(ag.arg_type) + 4), ts = std::min(38, dec_scale(ag.arg_type) + 4);
          e.kind = 7; e.word = ag.word; e.cnt_word = ag.cnt_word; e.avg_mul = ts - dec_scale(ag.arg_type); e.avg_prec = tp;
          add(dec_type(tp, ts), true, e);
        } else if (partial) {   // state = [count: UInt64, sum: Float64] (aggregates/mod.rs:3591-3700)
          EmitCol c1 = e; c1.kind = 4; c1.word = ag.cnt_word; add(DFGPU_UINT64, false, c1);
          EmitCol c2 = e; c2.kind = 2; c2.word = ag.word; c2.nn_word = ag.cnt_word; add(DFGPU_FLOAT64, true, c2);
        } else { e.kind = 3; e.word = ag.word; e.cnt_word = ag.cnt_word; add(DFGPU_FLOAT64, true, e); }
        break;
    }
  }
}

static void dense_finish(dfgpu_pipeline* p);

// Full join, second part: the build rows no probe row matched go once more through the pipeline, as one push at finish (timed as
// "pipe_full_tail:<name>").  Their records are the occupied ones whose visited word is still 0 (lookup_groups_kernel's LEFT_ANTI
// selection); their keys, emitted in slot order, are the FULL stage's hidden key column.  Every input column is NULL (zeroed values, an
// all-zero bitmap) and the predicate is off, so each row finds its record and carries its payload fields, and the sink takes it like any
// other row: the output sinks write it with bitmaps, the dense and hash sinks put its NULL probe columns in their NULL groups, and the
// aggregate arguments are evaluated on it.
static void full_tail(dfgpu_pipeline* p) {
  check_left_build(p);
  dfgpu_lookup* l = p->stages[p->full_stage].lookup;
  if (l->cap == 0 || l->rows == 0) return;
  dfgpu_ctx* ctx = p->ctx;
  DCol keys;
  int64_t m = 0;
  {   // the selection and the key emission; the push below times its kernels under the same family, one timer after the other
    const std::string tname = tail_timer(p);
    KernelTimer kt(ctx, tname.c_str());
    const LookupDev t = lookup_dev(l);
    const uint64_t nw = (t.cap + 31) / 32;
    DevBuf words(ctx, (size_t)nw * 4 + 8), idx;
    lookup_groups_kernel<<<grid_for((int64_t)nw * 32, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, kVisitedWord, 1, words.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
    m = compact_flag_indices(ctx, words.as<uint32_t>(), (int64_t)t.cap, 1, &idx);
    p->m_unmatched_build_rows = m;
    if (m == 0) return;
    keys = alloc_col(ctx, DFGPU_INT64, m, false);   // the record's key word as stored: a composite key's packed tuple
    EmitCols ec;
    memset(&ec, 0, sizeof(ec));
    ec.n = 1; ec.c[0].kind = 0; ec.c[0].width = 8; ec.c[0].nn_word = -1; ec.c[0].dst = keys.own_values->ptr;
    lookup_emit_kernel<<<grid_for(m, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, idx.as<uint32_t>(), m, kVisitedWord, ec);
    DF_LAUNCH_CHECK(ctx);
  }
  std::vector<DCol> cols;
  for (int type : p->in_types) {
    DCol c = alloc_col(ctx, type, m, true);
    c.own_values->zero(); c.own_validity->zero();
    c.null_count = m;
    cols.push_back(std::move(c));
  }
  p->packed.clear();
  p->packed.push_back(std::move(keys));
  const size_t parts = p->out_parts.size();
  const int64_t pending = p->out_rows_pending;
  p->in_tail = true;
  try { pipeline_push(p, cols); } catch (...) { p->in_tail = false; throw; }
  p->in_tail = false;
  if (p->sink == SINK_OUTPUT && p->out_parts.size() > parts) {   // the output sinks emit the tail's rows as batches of their own
    p->tail_part = std::move(p->out_parts.back());
    p->out_parts.pop_back();
    p->tail_rows = p->out_rows_pending - pending;
    p->out_rows_pending = pending;
  }
}

static void pipeline_finish(dfgpu_pipeline* p) {
  DF_CHECK(!p->finished, DFGPU_ERR_STATE, "finish called twice");
  if (p->full_stage >= 0) {   // a tail that fails leaves the pipeline finished: a second finish must not push the rows again
    set_device(p->ctx);
    try { full_tail(p); } catch (...) { p->finished = true; throw; }
  }
  p->finished = true;
  dfgpu_ctx* ctx = p->ctx;
  set_device(ctx);
  if (p->sink == SINK_OUTPUT) {
    if (p->out_rows_pending > 0) {
      std::vector<DCol> merged;
      for (size_t c = 0; c < p->out_cols.size(); ++c) {
        std::vector<DCol> parts;
        for (auto& b : p->out_parts) parts.push_back(b[c]);
        merged.push_back(parts.size() == 1 ? parts[0] : concat_columns(ctx, parts, p->vtypes[p->out_cols[c]]));
      }
      p->out_parts.clear();
      emit_sliced(p, merged, p->out_rows_pending);
    }
    if (p->tail_rows > 0) emit_sliced(p, p->tail_part, p->tail_rows);   // behind the probe rows, not copied into their columns
    return;
  }
  if (p->sink == SINK_DENSE) { dense_finish(p); return; }
  if (p->sink == SINK_BUILD && p->key_flags.ptr) {   // a composite build key: what the packing passes saw, read once
    unsigned long long f[2];
    DF_CUDA(cudaMemcpyAsync(f, p->key_flags.ptr, 16, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    p->target->null_keys += (int64_t)f[1];
    if (f[0]) throw Error(DFGPU_ERR_INVALID, "lookup build: a composite key has a component outside its declared domain");
  }
  if (p->sink != SINK_AGG && p->sink != SINK_HASH) return;
  check_left_build(p);
  LookupDev t;
  if (p->sink == SINK_AGG) {
    dfgpu_lookup* l = p->stages[p->agg_stage].lookup;
    if (l->cap == 0) return;
    t = lookup_dev(l);
  } else {   // the hash sink's table: the regular records, then the side record
    if (!p->hash_recs.ptr) return;
    memset(&t, 0, sizeof(t));
    t.recs = p->hash_recs.as<unsigned long long>(); t.cap = p->hash_cap + 1; t.stride = p->hash_stride;
  }
  const int sel = p->left_kind == DFGPU_STAGE_LEFT ? 2 : (p->left_kind == DFGPU_STAGE_LEFT_ANTI ? 1 : 0);
  // the join-keyed sink's groups are at most the lookup's records: columns of that length let lookup_scan_emit_kernel find and emit the
  // groups in one pass, when every column is one it emits
  const bool try_scan = p->sink == SINK_AGG && sel == 0;
  int64_t groups = try_scan ? p->stages[p->agg_stage].lookup->rows : 0;
  DevBuf idx;
  auto scan_groups = [&]() {
    const uint64_t nw = (t.cap + 31) / 32;
    DevBuf words(ctx, (size_t)nw * 4 + 8);
    lookup_groups_kernel<<<grid_for((int64_t)nw * 32, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, p->rows_word, sel, words.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
    groups = compact_flag_indices(ctx, words.as<uint32_t>(), (int64_t)t.cap, 1, &idx);
  };
  if (!try_scan) {
    scan_groups();
    p->m_groups = groups;
    if (groups == 0) return;
  }
  // output schema: group columns, then one (Single) or the state (Partial) columns per aggregate
  const bool partial = p->agg_mode == DFGPU_AGG_PARTIAL;
  EmitCols ec;
  memset(&ec, 0, sizeof(ec));
  // AVG over Decimal128 (emission kind 7): the error word is set when a group's value overflows
  bool dec_avg = false;
  for (const PipeAgg& ag : p->aggs) dec_avg = dec_avg || (ag.func == DFGPU_AGG_AVG && ag.cls == C_DEC);
  DevBuf err;
  if (dec_avg) { err.alloc(ctx, 8); err.zero(); ec.err = err.as<unsigned long long>(); }
  std::vector<DCol> out;
  const int key_col = p->sink == SINK_AGG ? p->stages[p->agg_stage].key_col : -1;
  const std::vector<int> no_keys, &comp_cols = p->sink == SINK_AGG ? p->stage_keys[p->agg_stage] : no_keys;
  auto add = [&](int type, bool nullable, EmitCol e) {
    DF_CHECK(ec.n < kMaxPipeCols, DFGPU_ERR_UNSUPPORTED, "pipeline: too many output columns");
    DCol d = alloc_col(ctx, type, groups, nullable);
    e.width = type_width(type); e.dst = d.own_values->ptr; e.valid = nullable ? d.own_validity->as<uint32_t>() : nullptr;
    d.null_count = nullable ? -1 : 0;
    ec.c[ec.n++] = e;
    out.push_back(std::move(d));
  };
  auto add_columns = [&]() {
    for (size_t k = 0; k < p->hash_keys.size(); ++k) {   // hash sink: the fields of the packed tag
      const HashKey& hk = p->hash_keys[k];
      EmitCol e; memset(&e, 0, sizeof(e));
      e.kind = 8; e.shift = hk.shift; e.tag_null = hk.null_bit;
      add(p->vtypes[hk.src], hk.null_bit >= 0, e);
    }
    for (int g : p->group_cols) {
      if (p->sink == SINK_HASH) break;
      EmitCol e; memset(&e, 0, sizeof(e));
      const auto comp = std::find(comp_cols.begin(), comp_cols.end(), g);
      if (comp != comp_cols.end()) {   // a component of the composite key, decoded from the packed key
        const dfgpu_lookup* l = p->stages[p->agg_stage].lookup;
        const size_t c = comp - comp_cols.begin();
        e.kind = 10; e.kmin = l->comp_min[c]; e.cstride = l->comp_stride[c]; e.cradix = l->comp_range[c];
        add(p->in_types[g], false, e);
      } else if (g == key_col) { e.kind = 0; add(p->in_types[g], false, e); }
      else { const ExtDef& x = p->exts[g - (int)p->in_types.size()]; e.kind = 1; e.shift = x.shift; add(x.type, false, e); }
    }
    add_agg_columns(p->aggs, p->rows_word, partial, p->left_kind == DFGPU_STAGE_LEFT, add);
  };
  add_columns();
  bool scan = try_scan && !dec_avg;
  for (int c = 0; c < ec.n && scan; ++c) {
    const EmitCol& e = ec.c[c];
    scan = !e.valid && (e.kind == 0 || e.kind == 1 || e.kind == 4 || (e.kind == 2 && e.nn_word < 0 && !e.f64_key));
  }
  if (scan) {
    const uint64_t ntiles = (t.cap + 1023) / 1024;
    DevBuf desc(ctx, (size_t)(ntiles + 2) * 8);   // tile descriptors, then the tile counter and the group count
    desc.zero();
    unsigned long long* d = desc.as<unsigned long long>();
    lookup_scan_emit_kernel<<<kNumSMs * 8, 256, 0, ctx->stream>>>(t, p->rows_word, ec, (unsigned int*)(d + ntiles), d, d + ntiles + 1, (uint64_t)groups);
    DF_LAUNCH_CHECK(ctx);
    const int64_t found = (int64_t)read_scalar(ctx, d + ntiles + 1);
    scan = found <= groups;   // more records reached than the lookup holds rows: emit through the index path instead
    if (scan) {
      groups = found;
      for (DCol& c : out) c.length = groups;
      p->m_groups = groups;
      if (groups == 0) return;
    }
  }
  if (!scan) {
    if (try_scan) {   // an emission the single pass does not make: the columns again, at the group count
      out.clear(); ec.n = 0;
      scan_groups();
      p->m_groups = groups;
      if (groups == 0) return;
      add_columns();
    }
    lookup_emit_kernel<<<grid_for(groups, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, idx.as<uint32_t>(), groups, p->rows_word, ec);
    DF_LAUNCH_CHECK(ctx);
  }
  if (dec_avg) {
    unsigned long long h_err = 0;
    DF_CUDA(cudaMemcpyAsync(&h_err, err.ptr, 8, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    if (h_err) throw Error(DFGPU_ERR_ARITH, "Arithmetic Overflow in AvgAccumulator");
  }
  emit_sliced(p, out, groups);
}

// the dense sink's output: one row per slot that received a row (exactly one row without GROUP BY, also for empty input), in slot
// order = ascending key order with NULL after the values of its column
static void dense_finish(dfgpu_pipeline* p) {
  dfgpu_ctx* ctx = p->ctx;
  prepare_dense(p);
  LookupDev t;
  memset(&t, 0, sizeof(t));
  t.recs = p->dense_acc.as<unsigned long long>(); t.cap = (uint64_t)p->dense_slots; t.stride = p->dense_words;
  DevBuf idx, err(ctx, 8);
  err.zero();
  int64_t groups = 1;
  if (p->dense_keys.empty()) {   // AggregateStream: the single slot
    idx.alloc(ctx, 8);
    idx.zero();
  } else {
    const uint64_t nw = (t.cap + 31) / 32;
    DevBuf words(ctx, (size_t)nw * 4 + 8);
    lookup_groups_kernel<<<grid_for((int64_t)nw * 32, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, 0, 0, words.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
    groups = compact_flag_indices(ctx, words.as<uint32_t>(), (int64_t)t.cap, 1, &idx);
  }
  p->m_groups = groups;
  if (groups == 0) return;
  EmitCols ec;
  memset(&ec, 0, sizeof(ec));
  ec.err = err.as<unsigned long long>();
  std::vector<DCol> out;
  auto add = [&](int type, bool nullable, EmitCol e) {
    DF_CHECK(ec.n < kMaxPipeCols, DFGPU_ERR_UNSUPPORTED, "pipeline: too many output columns");
    DCol d = alloc_col(ctx, type, groups, nullable);
    e.width = type_width(type); e.dst = d.own_values->ptr; e.valid = nullable ? d.own_validity->as<uint32_t>() : nullptr;
    d.null_count = nullable ? -1 : 0;
    ec.c[ec.n++] = e;
    out.push_back(std::move(d));
  };
  for (size_t k = 0; k < p->dense_keys.size(); ++k) {
    EmitCol e; memset(&e, 0, sizeof(e));
    e.kind = 6; e.kmin = (long long)p->dense_keys[k].kmin; e.kstride = (int)p->dense_keys[k].stride; e.kradix = p->dense_radix[k];
    add(p->vtypes[p->group_cols[k]], true, e);
  }
  add_agg_columns(p->aggs, 0, p->agg_mode == DFGPU_AGG_PARTIAL, false, add);
  lookup_emit_kernel<<<grid_for(groups, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(t, idx.as<uint32_t>(), groups, 0, ec);
  DF_LAUNCH_CHECK(ctx);
  unsigned long long h_err = 0;
  DF_CUDA(cudaMemcpyAsync(&h_err, err.ptr, 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  if (h_err) throw Error(DFGPU_ERR_ARITH, "Arithmetic Overflow in AvgAccumulator");
  emit_sliced(p, out, groups);
}

// the aggregates of the join-keyed and the hash-keyed sink: functions, argument programs and the types each accepts
static std::vector<PipeAgg> parse_pipe_aggs(const dfgpu_pipeline* p, const dfgpu_pipeline_agg* aggs, int n_aggs, int mode) {
  DF_CHECK(n_aggs >= 0 && n_aggs <= kMaxPipeAggs && (n_aggs == 0 || aggs), DFGPU_ERR_UNSUPPORTED, "pipeline: 0..4 aggregates");
  std::vector<PipeAgg> out;
  for (int a = 0; a < n_aggs; ++a) {
    PipeAgg ag;
    ag.func = aggs[a].func;
    DF_CHECK(ag.func >= DFGPU_AGG_SUM && ag.func <= DFGPU_AGG_COUNT_STAR, DFGPU_ERR_INVALID, "pipeline aggregate: unknown function");
    if (ag.func != DFGPU_AGG_COUNT_STAR) {
      DF_CHECK(aggs[a].expr && aggs[a].n_nodes > 0, DFGPU_ERR_INVALID, "pipeline aggregate: missing argument expression");
      ag.plan = plan_expr(p->vtypes.data(), (int)p->vtypes.size(), aggs[a].expr, aggs[a].n_nodes);
      ag.has_expr = true;
      ag.arg_type = ag.plan.root_type;
      ag.cls = cls_of(ag.arg_type);
      DF_CHECK(ag.cls != C_BOOL || ag.func == DFGPU_AGG_COUNT, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: Boolean arguments only for COUNT");
      if (ag.func == DFGPU_AGG_AVG) {
        DF_CHECK(ag.arg_type == DFGPU_FLOAT64 || ag.cls == C_DEC, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: AVG takes a Float64 (the planner casts) or Decimal128 argument");
        DF_CHECK(ag.cls != C_DEC || mode != DFGPU_AGG_PARTIAL, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: AVG over Decimal128 runs in Single modes only");
      }
      if ((ag.func == DFGPU_AGG_MIN || ag.func == DFGPU_AGG_MAX)) DF_CHECK(ag.arg_type != DFGPU_FLOAT32, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: MIN/MAX over Float32 stays on dfgpu_agg");
    }
    out.push_back(std::move(ag));
  }
  return out;
}

// accumulator words of a record, taken from word `next` (the row counter already taken) up to `budget` (exclusive); `next` ends past the
// last word taken.  Without pairs: every aggregate's words in order.  With pairs (a Decimal128 MIN / MAX is a {lo, hi} pair updated by one
// 16-byte CAS, so it sits on an even word of a record of an even number of words, `even_record`): at most one padding word to reach an
// even word, the pairs, then the other aggregates in order.  Spare words (the padding word first) become non-null counters.
static void layout_agg_words(std::vector<PipeAgg>& aggs, int& next, int budget, bool even_record) {
  auto is_pair = [](const PipeAgg& ag) { return ag.cls == C_DEC && (ag.func == DFGPU_AGG_MIN || ag.func == DFGPU_AGG_MAX); };
  bool pairs = false;
  for (const auto& ag : aggs) pairs = pairs || (ag.has_expr && is_pair(ag));
  auto take = [&](const char* what) { DF_CHECK(next < budget, DFGPU_ERR_UNSUPPORTED, what); return next++; };
  int pad = -1;
  if (pairs) {
    DF_CHECK(even_record, DFGPU_ERR_UNSUPPORTED,
             "pipeline aggregate: a Decimal128 MIN / MAX needs a record of an even number of words: a lookup without payload takes an odd n_acc_words");
    if (next & 1) pad = take("pipeline aggregate: not enough accumulator words in the lookup (n_acc_words)");
    for (auto& ag : aggs) {
      if (!is_pair(ag)) continue;
      ag.word = take("pipeline aggregate: not enough accumulator words in the lookup (n_acc_words)");
      take("pipeline aggregate: a Decimal128 MIN / MAX takes two accumulator words (n_acc_words)");
    }
  }
  for (auto& ag : aggs) {
    if (ag.func == DFGPU_AGG_COUNT_STAR || is_pair(ag)) continue;
    ag.word = take("pipeline aggregate: not enough accumulator words in the lookup (n_acc_words)");
    if (ag.cls == C_DEC && ag.func == DFGPU_AGG_SUM) take("pipeline aggregate: a Decimal128 SUM takes two accumulator words (n_acc_words)");
    if (ag.cls == C_DEC && ag.func == DFGPU_AGG_AVG) take("pipeline aggregate: a Decimal128 AVG takes three accumulator words (n_acc_words)");
    if (ag.func == DFGPU_AGG_AVG) { ag.cnt_word = take("pipeline aggregate: not enough accumulator words in the lookup (n_acc_words)"); ag.nn_word = ag.cnt_word; }
  }
  // spare words become non-null counters (SUM / MIN / MAX of a nullable argument are NULL until a value arrives, accumulate.rs:164-188)
  for (auto& ag : aggs) {
    if (ag.func != DFGPU_AGG_SUM && ag.func != DFGPU_AGG_MIN && ag.func != DFGPU_AGG_MAX) continue;
    if (pad >= 0) { ag.nn_word = pad; pad = -1; }
    else if (next < budget) ag.nn_word = next++;
  }
}

static bool is_left_kind(int kind) { return kind == DFGPU_STAGE_LEFT || kind == DFGPU_STAGE_LEFT_ANTI; }

// a LEFT / LEFT_ANTI stage emits its build rows from the join-keyed aggregate sink's records; every other sink is UNSUPPORTED
static void check_no_left_stage(const dfgpu_pipeline* p) {
  for (const auto& st : p->stages)
    DF_CHECK(!is_left_kind(st.kind), DFGPU_ERR_UNSUPPORTED, "pipeline: a LEFT / LEFT_ANTI stage runs only with the join-keyed aggregate sink grouped on it");
}

// a RIGHT stage runs with the output, dense and hash sinks only
static void check_no_right_stage(const dfgpu_pipeline* p, const char* what) {
  DF_CHECK(!p->has_right, DFGPU_ERR_UNSUPPORTED, what);
}

// LEFT: a build row no probe row reached is emitted as one NULL-padded row without evaluating anything, so an aggregate argument must be
// NULL on that row: it reads at least one probe-side input column, no payload field of the LEFT stage (that is the padded row's own
// value), and every node propagates NULL (no IS [NOT] NULL, IS [NOT] DISTINCT FROM, AND, OR)
static void check_left_args(const dfgpu_pipeline* p, const std::vector<PipeAgg>& aggs, int stage) {
  const int nin = (int)p->in_types.size();
  for (const PipeAgg& ag : aggs) {
    if (!ag.has_expr) continue;
    bool probe_col = false;
    for (const auto& nd : ag.plan.nodes) {
      bool ok = true;
      if (nd.kind == DFGPU_EXPR_COLUMN) {
        if (nd.a < nin) probe_col = true;
        else ok = p->exts[nd.a - nin].stage != stage;
      } else if (nd.kind == DFGPU_EXPR_BINARY) {
        ok = nd.a != DFGPU_OP_AND && nd.a != DFGPU_OP_OR && nd.a != DFGPU_OP_IS_DISTINCT_FROM && nd.a != DFGPU_OP_IS_NOT_DISTINCT_FROM;
      } else {
        ok = nd.kind == DFGPU_EXPR_LITERAL || nd.kind == DFGPU_EXPR_CAST || nd.kind == DFGPU_EXPR_NEGATIVE || nd.kind == DFGPU_EXPR_NOT;
      }
      DF_CHECK(ok, DFGPU_ERR_UNSUPPORTED,
               "pipeline aggregate: under a LEFT stage an argument must propagate NULL and read no build-side column — use dfgpu_hashjoin + dfgpu_agg");
    }
    DF_CHECK(probe_col, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: under a LEFT stage every argument reads a probe-side input column");
  }
}

}  // namespace dfgpu

extern "C" {

void dfgpu_lookup_default_options(dfgpu_lookup_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->membership_filter = -1;
}

int dfgpu_lookup_create(dfgpu_ctx* ctx, int32_t key_type, const int32_t* payload_types, int32_t n_payload, const dfgpu_lookup_options* opts, dfgpu_lookup** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && out, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(key_type_ok(key_type), DFGPU_ERR_UNSUPPORTED, "lookup: the key must be one integer-like column of <= 64 bits");
  DF_CHECK(n_payload >= 0 && n_payload <= kMaxBuildPay && (n_payload == 0 || payload_types), DFGPU_ERR_INVALID, "lookup: 0..8 payload columns");
  set_device(ctx);
  std::unique_ptr<dfgpu_lookup> l(new dfgpu_lookup());
  l->ctx = ctx; l->key_type = key_type;
  if (opts) l->opt = *opts; else dfgpu_lookup_default_options(&l->opt);
  DF_CHECK(l->opt.n_acc_words >= 0 && l->opt.n_acc_words <= 12, DFGPU_ERR_INVALID, "lookup: 0..12 accumulator words");
  int bits = 0;
  for (int i = 0; i < n_payload; ++i) {
    const int w = type_width(payload_types[i]);
    DF_CHECK(w >= 1 && w <= 8 && payload_types[i] != DFGPU_BOOL, DFGPU_ERR_UNSUPPORTED, "lookup: payload columns must be fixed-width, <= 8 bytes");
    l->pay_types.push_back(payload_types[i]); l->pay_shift.push_back(bits);
    bits += 8 * w;
  }
  DF_CHECK(bits <= 64, DFGPU_ERR_UNSUPPORTED, "lookup: payload columns wider than 64 bits together stay on the unfused join");
  l->has_payload = n_payload > 0;
  l->stride = 1 + (l->has_payload ? 1 : 0) + l->opt.n_acc_words;
  if (l->has_payload && (l->stride & 1)) l->stride++;   // {key,payload} is claimed with one 16-byte CAS
  l->mode = LK_HASH;
  if (!l->has_payload && l->opt.n_acc_words == 0 && l->opt.has_key_range && l->opt.key_max >= l->opt.key_min) {
    const uint64_t range = (uint64_t)l->opt.key_max - (uint64_t)l->opt.key_min;
    if (range < (1ull << 32)) {   // <= 512 MiB of bits
      l->mode = LK_BITMAP; l->kmin = (uint64_t)l->opt.key_min; l->ksize = range + 1;
      l->bits.alloc(ctx, (size_t)((l->ksize + 31) / 32) * 4 + 8);
      l->bits.zero();
    }
  }
  if (l->opt.filter_only) {
    DF_CHECK(l->mode == LK_HASH && !l->has_payload && l->opt.n_acc_words == 0, DFGPU_ERR_INVALID, "lookup: a filter-only lookup is a key set without payload");
    DF_CHECK(l->opt.expected_rows > 0, DFGPU_ERR_INVALID, "lookup: a filter-only lookup needs expected_rows (its geometry is fixed up front)");
    l->filter_only = true;
    l->bloom_blocks = std::max<uint64_t>(1024, (uint64_t)l->opt.expected_rows / 4);   // 16 bits per key
    DF_CHECK(l->bloom_blocks < (1ull << 32), DFGPU_ERR_UNSUPPORTED, "lookup: filter too large");
    // a filter larger than L2 gets the coarse first level (4 bits per key) in the same allocation: one buffer to share and to all-reduce
    static const int coarse_mb = getenv("DFGPU_FILTER_COARSE_MB") ? atoi(getenv("DFGPU_FILTER_COARSE_MB")) : 20;
    if (coarse_mb >= 0 && (size_t)l->bloom_blocks * 8 > ((size_t)coarse_mb << 20)) l->coarse_words = (std::max<uint64_t>(4096, (uint64_t)l->opt.expected_rows / 8) + 1) & ~1ull;
    l->bloom.alloc(ctx, (size_t)l->bloom_blocks * 8 + (size_t)l->coarse_words * 4);
    l->bloom.zero();
  }
  if (l->mode == LK_HASH && !l->filter_only && l->opt.expected_rows > 0) lookup_reserve(l.get(), l->opt.expected_rows);
  *out = l.release();
  DF_API_END
}
int dfgpu_lookup_create_composite(dfgpu_ctx* ctx, const int32_t* key_types, const int64_t* key_min, const int64_t* key_max, int32_t n_keys,
                                  const int32_t* payload_types, int32_t n_payload, const dfgpu_lookup_options* opts, dfgpu_lookup** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && out && key_types && key_min && key_max, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(n_keys >= 2 && n_keys <= kMaxKeyParts, DFGPU_ERR_INVALID, "lookup: a composite key has 2..4 components");
  dfgpu_lookup_options o;
  if (opts) o = *opts; else dfgpu_lookup_default_options(&o);
  DF_CHECK(!o.has_key_range, DFGPU_ERR_INVALID, "lookup: a composite key's range is its declared domains (has_key_range must be 0)");
  // r_g = max_g - min_g + 1, stride_0 = 1, stride_{g+1} = stride_g r_g; D = prod r_g <= 2^63 - 1 (so no packed key is kEmptyKey)
  std::vector<uint64_t> range(n_keys), stride(n_keys);
  uint64_t domain = 1;
  for (int g = 0; g < n_keys; ++g) {
    DF_CHECK(key_type_ok(key_types[g]), DFGPU_ERR_UNSUPPORTED, "lookup: composite key components must be integer-like columns of <= 64 bits");
    DF_CHECK(key_min[g] <= key_max[g], DFGPU_ERR_INVALID, "lookup: composite key domain with min > max");
    DF_CHECK(!type_is_unsigned_int(key_types[g]) || key_min[g] >= 0, DFGPU_ERR_INVALID, "lookup: an unsigned component's domain starts at 0 or above");
    const uint64_t span = (uint64_t)key_max[g] - (uint64_t)key_min[g];
    DF_CHECK(span < (uint64_t)INT64_MAX, DFGPU_ERR_UNSUPPORTED, "lookup: the composite key's domain exceeds 2^63 - 1 values");
    range[g] = span + 1;
    stride[g] = domain;
    DF_CHECK(domain <= (uint64_t)INT64_MAX / range[g], DFGPU_ERR_UNSUPPORTED, "lookup: the composite key's domain exceeds 2^63 - 1 values");
    domain *= range[g];
  }
  // the packed key is an Int64 in [0, D - 1]: the bitmap / hash / Bloom rules of dfgpu_lookup_create apply to that range (a filter-only
  // lookup is a Bloom filter whatever its range)
  if (!o.filter_only) { o.has_key_range = 1; o.key_min = 0; o.key_max = (int64_t)(domain - 1); }
  dfgpu_lookup* l = nullptr;
  const int rc = dfgpu_lookup_create(ctx, DFGPU_INT64, payload_types, n_payload, &o, &l);
  if (rc != DFGPU_OK) return rc;
  l->opt.has_key_range = 0;
  l->comp_types.assign(key_types, key_types + n_keys); l->comp_min.assign(key_min, key_min + n_keys);
  l->comp_range = range; l->comp_stride = stride; l->domain = domain;
  *out = l;
  DF_API_END
}
int64_t dfgpu_lookup_metric(dfgpu_lookup* l, const char* name) {
  if (!l || !name) return -1;
  std::string s(name);
  if (s == "rows") return l->rows;
  if (s == "capacity") return l->mode == LK_BITMAP ? (int64_t)l->ksize : (int64_t)l->cap;
  if (s == "mode") return l->mode;
  if (s == "table_bytes") return l->mode == LK_BITMAP ? (int64_t)l->bits.bytes : (int64_t)l->recs.bytes;
  if (s == "filter_bytes") return (int64_t)l->bloom.bytes;
  if (s == "rehashes") return l->rehashes;
  if (s == "stride_bytes") return l->stride * 8;
  if (s == "null_keys") return l->null_keys;
  if (s == "key_domain") return l->comp_types.empty() ? -1 : (int64_t)l->domain;
  return -1;
}
int dfgpu_lookup_clear(dfgpu_lookup* l) {
  DF_API_BEGIN(l ? l->ctx : nullptr)
  DF_CHECK(l, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(!l->acc_claimed, DFGPU_ERR_STATE, "lookup: accumulators in use by a pipeline");
  dfgpu_ctx* ctx = l->ctx;
  set_device(ctx);
  if (l->mode == LK_BITMAP) l->bits.zero();
  else {
    if (l->cap) { lookup_init_kernel<<<grid_for((int64_t)l->cap * l->stride, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(l->recs.as<unsigned long long>(), l->cap, l->stride); DF_LAUNCH_CHECK(ctx); }
    if (l->bloom.ptr) l->bloom.zero();
  }
  l->rows = 0; l->null_keys = 0; l->marks_taken = false; l->acc_written = false;   // every accumulator word (visited marks included) is 0 again
  DF_API_END
}
int dfgpu_lookup_filter_buffer(dfgpu_lookup* l, void** words_dev, uint64_t* n_bytes) {
  DF_API_BEGIN(l ? l->ctx : nullptr)
  DF_CHECK(l && words_dev && n_bytes, DFGPU_ERR_INVALID, "null argument");
  *words_dev = l->bloom.ptr; *n_bytes = (uint64_t)l->bloom_blocks * 8 + (uint64_t)l->coarse_words * 4;
  DF_API_END
}
int dfgpu_lookup_filter_allreduce_peer(dfgpu_lookup* l, void* const* peer_words, int32_t rank, int32_t n_ranks) {
  DF_API_BEGIN(l ? l->ctx : nullptr)
  DF_CHECK(l && peer_words, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(n_ranks >= 1 && n_ranks <= kMaxPeers && rank >= 0 && rank < n_ranks, DFGPU_ERR_INVALID, "filter all-reduce: 1..8 ranks of one box");
  DF_CHECK(l->bloom.ptr && l->bloom_blocks > 0, DFGPU_ERR_STATE, "filter all-reduce: the lookup has no membership filter");
  dfgpu_ctx* ctx = l->ctx;
  set_device(ctx);
  PeerWords pw;
  memset(&pw, 0, sizeof(pw));
  for (int q = 0; q < n_ranks; ++q) { DF_CHECK(peer_words[q], DFGPU_ERR_INVALID, "filter all-reduce: null peer pointer"); pw.p[q] = (unsigned long long*)peer_words[q]; }
  DF_CHECK(pw.p[rank] == l->bloom.as<unsigned long long>(), DFGPU_ERR_INVALID, "filter all-reduce: peer_words[rank] must be this lookup's own filter");
  const uint64_t words64 = l->bloom_blocks + l->coarse_words / 2;   // exact blocks + coarse level, merged as one array of 64-bit words
  const uint64_t slice = words64 / (uint64_t)n_ranks + 1;
  KernelTimer kt(ctx, "filter_allreduce");
  filter_allreduce_peer_kernel<<<grid_for((int64_t)slice, 256, kNumSMs * 4), 256, 0, ctx->stream>>>(pw, rank, n_ranks, words64);
  DF_LAUNCH_CHECK(ctx);
  DF_API_END
}
void dfgpu_lookup_destroy(dfgpu_lookup* l) {
  if (!l) return;
  cudaSetDevice(l->ctx->device);
  delete l;
}

int dfgpu_column_minmax_device(dfgpu_ctx* ctx, const dfgpu_column* col, int64_t* min_out, int64_t* max_out, int64_t* valid_out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && col && min_out && max_out, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(key_type_ok(col->type), DFGPU_ERR_UNSUPPORTED, "minmax: integer-like columns only");
  set_device(ctx);
  DCol c = device_view(*col);
  const int uns = type_is_unsigned_int(c.type) ? 1 : 0;
  DevBuf mm(ctx, 24);
  unsigned long long init[3] = {~0ull, 0ull, 0ull};
  DF_CUDA(cudaMemcpyAsync(mm.ptr, init, 24, cudaMemcpyHostToDevice, ctx->stream));
  if (c.length > 0) {
    col_minmax_kernel<<<grid_for(c.length, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(col_ref(c), c.length, uns, mm.as<unsigned long long>());
    DF_LAUNCH_CHECK(ctx);
  }
  unsigned long long h[3];
  DF_CUDA(cudaMemcpyAsync(h, mm.ptr, 24, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  if (valid_out) *valid_out = (int64_t)h[2];
  if (h[2] == 0) { *min_out = 0; *max_out = -1; }
  else if (uns) { *min_out = (int64_t)h[0]; *max_out = (int64_t)h[1]; }
  else { *min_out = (int64_t)(h[0] ^ (1ull << 63)); *max_out = (int64_t)(h[1] ^ (1ull << 63)); }
  DF_API_END
}

int dfgpu_column_sum_device(dfgpu_ctx* ctx, const dfgpu_column* col, uint64_t* sum_out, int64_t* valid_out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && col && sum_out, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(key_type_ok(col->type) || type_is_decimal(col->type), DFGPU_ERR_UNSUPPORTED, "column sum: integer-like and Decimal128 columns only");
  set_device(ctx);
  DCol c = device_view(*col);
  DevBuf acc(ctx, 16);
  acc.zero();
  if (c.length > 0) {
    col_sum_kernel<<<grid_for(c.length, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(col_ref(c), c.length, acc.as<unsigned long long>());
    DF_LAUNCH_CHECK(ctx);
  }
  unsigned long long h[2];
  DF_CUDA(cudaMemcpyAsync(h, acc.ptr, 16, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  *sum_out = h[0];
  if (valid_out) *valid_out = (int64_t)h[1];
  DF_API_END
}

int dfgpu_pipeline_create(dfgpu_ctx* ctx, const int32_t* input_types, int32_t n_cols, const dfgpu_expr_node* predicate, int32_t n_pred_nodes,
                          const dfgpu_pipeline_stage* stages, int32_t n_stages, dfgpu_pipeline** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && out && input_types, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(n_cols >= 1 && n_cols <= kMaxPipeCols, DFGPU_ERR_UNSUPPORTED, "pipeline: 1..16 input columns");
  DF_CHECK(n_stages >= 0 && n_stages <= kMaxStages && (n_stages == 0 || stages), DFGPU_ERR_UNSUPPORTED, "pipeline: 0..3 probe stages");
  std::unique_ptr<dfgpu_pipeline> p(new dfgpu_pipeline());
  p->ctx = ctx;
  p->in_types.assign(input_types, input_types + n_cols);
  p->vtypes = p->in_types;
  if (predicate && n_pred_nodes > 0) {
    p->pred = plan_expr(input_types, n_cols, predicate, n_pred_nodes);
    DF_CHECK(p->pred.root_type == DFGPU_BOOL, DFGPU_ERR_INVALID, "Cannot create filter_array from non-boolean predicates");
    p->has_pred = true;
  }
  for (int s = 0; s < n_stages; ++s) {
    const dfgpu_pipeline_stage& st = stages[s];
    DF_CHECK(st.lookup, DFGPU_ERR_INVALID, "pipeline: stage without a lookup");
    DF_CHECK(st.kind >= DFGPU_STAGE_INNER && st.kind <= DFGPU_STAGE_RIGHT, DFGPU_ERR_INVALID, "pipeline: unknown stage kind");
    // a RIGHT stage keeps the row count only over unique keys: a lookup with payload (its build refuses duplicate keys)
    DF_CHECK(st.kind != DFGPU_STAGE_RIGHT || (st.lookup->has_payload && st.lookup->mode == LK_HASH && !st.lookup->filter_only), DFGPU_ERR_UNSUPPORTED,
             "pipeline: a RIGHT stage needs a lookup with payload (unique keys), not a key set, bitmap or filter-only lookup — use dfgpu_hashjoin");
    DF_CHECK(!st.lookup->filter_only || st.kind == DFGPU_STAGE_MAYBE, DFGPU_ERR_INVALID, "pipeline: a filter-only lookup can only back a MAYBE stage");
    DF_CHECK(st.key_col >= 0 && st.key_col < n_cols, DFGPU_ERR_INVALID, "pipeline: stage key column out of range");
    const int kt = input_types[st.key_col], lt = st.lookup->key_type;
    if (!st.lookup->comp_types.empty())   // a composite key: key_col is its first component (dfgpu_pipeline_set_stage_keys names them all)
      DF_CHECK(kt == st.lookup->comp_types[0], DFGPU_ERR_INVALID, "pipeline: probe key type differs from the lookup's first key component");
    else
      DF_CHECK(key_type_ok(kt) && type_width(kt) == type_width(lt) && type_is_signed_int(kt) == type_is_signed_int(lt), DFGPU_ERR_INVALID,
               "pipeline: probe key type differs from the lookup's key type");
    DF_CHECK(st.lookup->ctx->device == ctx->device, DFGPU_ERR_INVALID, "pipeline: lookup lives on another device");
    p->stages.push_back(st);
    p->has_right = p->has_right || st.kind == DFGPU_STAGE_RIGHT;
    if (st.kind == DFGPU_STAGE_INNER || st.kind == DFGPU_STAGE_LEFT || st.kind == DFGPU_STAGE_LEFT_ANTI || st.kind == DFGPU_STAGE_RIGHT)
      for (size_t f = 0; f < st.lookup->pay_types.size(); ++f) {
        DF_CHECK(p->exts.size() < (size_t)kMaxExt, DFGPU_ERR_UNSUPPORTED, "pipeline: at most 8 payload fields");
        ExtDef e; e.stage = s; e.shift = st.lookup->pay_shift[f]; e.width = type_width(st.lookup->pay_types[f]); e.type = st.lookup->pay_types[f];
        p->exts.push_back(e);
        p->vtypes.push_back(e.type);
      }
  }
  *out = p.release();
  DF_API_END
}

// the input columns key_cols[0 .. n_keys) as the components of a composite-key lookup, in order and of the same types (a stage's or the
// build sink's); the hidden packed columns and the inputs share PipeParams' 16 column slots
static void check_composite_keys(const dfgpu_pipeline* p, const dfgpu_lookup* l, const int32_t* key_cols, int32_t n_keys, int extra_packed) {
  DF_CHECK(!l->comp_types.empty(), DFGPU_ERR_INVALID, "pipeline: composite key columns for a lookup with a one-column key");
  DF_CHECK(key_cols && n_keys == (int)l->comp_types.size(), DFGPU_ERR_INVALID, "pipeline: the key column count differs from the lookup's components");
  for (int g = 0; g < n_keys; ++g) {
    DF_CHECK(key_cols[g] >= 0 && key_cols[g] < (int)p->in_types.size(), DFGPU_ERR_INVALID, "pipeline: a composite key component must be an input column");
    DF_CHECK(p->in_types[key_cols[g]] == l->comp_types[g], DFGPU_ERR_INVALID, "pipeline: a key column's type differs from the lookup's component type");
  }
  int packed = extra_packed + (p->bkey_cols.empty() ? 0 : 1);
  for (int s = 0; s < kMaxStages; ++s) packed += p->stage_keys[s].empty() ? 0 : 1;
  DF_CHECK((int)p->in_types.size() + packed <= kMaxPipeCols, DFGPU_ERR_UNSUPPORTED,
           "pipeline: the input columns and the packed composite keys exceed 16 columns");
}

static void set_build_sink(dfgpu_pipeline* p, dfgpu_lookup* target, int32_t key_col, const int32_t* payload_cols, int32_t n_payload) {
  DF_CHECK(n_payload == (int)target->pay_types.size(), DFGPU_ERR_INVALID, "pipeline build sink: payload column count differs from the lookup's");
  for (int c = 0; c < n_payload; ++c) {
    DF_CHECK(payload_cols[c] >= 0 && payload_cols[c] < (int)p->vtypes.size(), DFGPU_ERR_INVALID, "pipeline build sink: payload column out of range");
    DF_CHECK(type_width(p->vtypes[payload_cols[c]]) == type_width(target->pay_types[c]), DFGPU_ERR_INVALID, "pipeline build sink: payload column width differs from the lookup's");
    p->bpay_cols.push_back(payload_cols[c]);
  }
  for (auto& st : p->stages) DF_CHECK(st.lookup != target, DFGPU_ERR_INVALID, "pipeline: cannot build the lookup it probes");
  p->target = target; p->bkey_col = key_col; p->sink = SINK_BUILD;
}

int dfgpu_pipeline_sink_build(dfgpu_pipeline* p, dfgpu_lookup* target, int32_t key_col, const int32_t* payload_cols, int32_t n_payload) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && target, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(p->sink == SINK_NONE && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline: the sink is chosen once, before the first push");
  check_no_left_stage(p);
  check_no_right_stage(p, "pipeline build sink: a RIGHT stage's NULL payload fields cannot enter a lookup — use dfgpu_hashjoin");
  DF_CHECK(target->comp_types.empty(), DFGPU_ERR_INVALID, "pipeline build sink: a composite-key lookup is built by dfgpu_pipeline_sink_build_composite");
  DF_CHECK(key_col >= 0 && key_col < (int)p->in_types.size(), DFGPU_ERR_INVALID, "pipeline build sink: the key must be an input column");
  const int kt = p->in_types[key_col];
  DF_CHECK(type_width(kt) == type_width(target->key_type) && type_is_signed_int(kt) == type_is_signed_int(target->key_type), DFGPU_ERR_INVALID,
           "pipeline build sink: key type differs from the lookup's key type");
  set_build_sink(p, target, key_col, payload_cols, n_payload);
  DF_API_END
}

int dfgpu_pipeline_sink_build_composite(dfgpu_pipeline* p, dfgpu_lookup* target, const int32_t* key_cols, int32_t n_keys, const int32_t* payload_cols,
                                        int32_t n_payload) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && target, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(p->sink == SINK_NONE && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline: the sink is chosen once, before the first push");
  check_no_left_stage(p);
  check_no_right_stage(p, "pipeline build sink: a RIGHT stage's NULL payload fields cannot enter a lookup — use dfgpu_hashjoin");
  check_composite_keys(p, target, key_cols, n_keys, 1);
  set_build_sink(p, target, key_cols[0], payload_cols, n_payload);
  p->bkey_cols.assign(key_cols, key_cols + n_keys);
  DF_API_END
}

int dfgpu_pipeline_set_stage_keys(dfgpu_pipeline* p, int32_t stage, const int32_t* key_cols, int32_t n_keys) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(stage >= 0 && stage < (int)p->stages.size(), DFGPU_ERR_INVALID, "pipeline stage keys: stage out of range");
  DF_CHECK(!p->pushed && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline stage keys: set before the first push");
  DF_CHECK(p->stage_keys[stage].empty(), DFGPU_ERR_STATE, "pipeline stage keys: the stage already has them");
  check_composite_keys(p, p->stages[stage].lookup, key_cols, n_keys, 1);
  DF_CHECK(key_cols[0] == p->stages[stage].key_col, DFGPU_ERR_INVALID, "pipeline stage keys: the stage's key_col must be the first component");
  p->stage_keys[stage].assign(key_cols, key_cols + n_keys);
  DF_API_END
}

int dfgpu_pipeline_set_stage_full(dfgpu_pipeline* p, int32_t stage) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(stage >= 0 && stage < (int)p->stages.size(), DFGPU_ERR_INVALID, "pipeline full stage: stage out of range");
  DF_CHECK(p->stages[stage].kind == DFGPU_STAGE_RIGHT, DFGPU_ERR_INVALID, "pipeline full stage: only a RIGHT stage becomes a Full join");
  DF_CHECK(p->sink == SINK_NONE && !p->pushed && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline full stage: set before the sink and the first push");
  DF_CHECK(p->full_stage < 0, DFGPU_ERR_STATE, "pipeline full stage: the stage already is one");
  // the unmatched build rows are pushed with every input column NULL: past other probe stages they would have to skip those stages
  DF_CHECK(p->stages.size() == 1, DFGPU_ERR_UNSUPPORTED, "pipeline full stage: a FULL stage must be the pipeline's only probe stage — use dfgpu_hashjoin");
  dfgpu_lookup* l = p->stages[stage].lookup;
  DF_CHECK(l->has_payload && l->opt.n_acc_words >= 1, DFGPU_ERR_UNSUPPORTED,
           "pipeline full stage: the lookup needs payload and an accumulator word for the visited marks (n_acc_words >= 1)");
  DF_CHECK((int)p->in_types.size() + 1 <= kMaxPipeCols, DFGPU_ERR_UNSUPPORTED, "pipeline full stage: the input columns and the emitted build keys exceed 16 columns");
  DF_CHECK(!l->marks_taken && !l->acc_claimed, DFGPU_ERR_STATE,
           "pipeline full stage: the lookup's marks are taken by another pipeline (dfgpu_lookup_clear frees them)");
  claim_acc_words(l);
  l->marks_taken = true;
  p->full_stage = stage;
  DF_API_END
}

int dfgpu_pipeline_sink_aggregate(dfgpu_pipeline* p, const int32_t* group_cols, int32_t n_group, const dfgpu_pipeline_agg* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && group_cols && n_group >= 1, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(p->sink == SINK_NONE && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline: the sink is chosen once, before the first push");
  DF_CHECK(n_aggs >= 0 && n_aggs <= kMaxPipeAggs && (n_aggs == 0 || aggs), DFGPU_ERR_UNSUPPORTED, "pipeline: 0..4 aggregates");
  DF_CHECK(mode == DFGPU_AGG_SINGLE || mode == DFGPU_AGG_SINGLE_PARTITIONED || mode == DFGPU_AGG_PARTIAL, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: Single / SinglePartitioned / Partial");
  check_no_right_stage(p, "pipeline aggregate: the join-keyed sink does not run with a RIGHT stage — use the dense or hash aggregate sink");
  // a LEFT / LEFT_ANTI stage must be the last one, and the records grouped on are its own
  const int n_stages = (int)p->stages.size();
  int left = -1;
  for (int s = 0; s < n_stages; ++s) {
    if (!is_left_kind(p->stages[s].kind)) continue;
    DF_CHECK(s == n_stages - 1, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: a LEFT / LEFT_ANTI stage must be the last stage");
    left = s;
  }
  for (int s = 0; s < n_stages; ++s)   // the group columns name a composite key's components
    DF_CHECK(p->stages[s].lookup->comp_types.empty() || !p->stage_keys[s].empty(), DFGPU_ERR_STATE,
             "pipeline aggregate: set a composite-key stage's keys (dfgpu_pipeline_set_stage_keys) before this sink");
  // functional dependence: every group column is the probe key (every component of a composite one) of ONE inner stage or a payload
  // field of that stage
  const int nin = (int)p->in_types.size();
  int stage = -1;
  for (int s = 0; s < n_stages && stage < 0; ++s) {
    if (left >= 0 ? s != left : p->stages[s].kind != DFGPU_STAGE_INNER) continue;
    // the key: the probe key column, or every component of a composite key
    const std::vector<int> keys = p->stage_keys[s].empty() ? std::vector<int>{p->stages[s].key_col} : p->stage_keys[s];
    size_t has_keys = 0;
    bool ok = true;
    for (int g = 0; g < n_group; ++g) {
      const int c = group_cols[g];
      DF_CHECK(c >= 0 && c < (int)p->vtypes.size(), DFGPU_ERR_INVALID, "pipeline aggregate: group column out of range");
      if (std::find(keys.begin(), keys.end(), c) != keys.end()) has_keys++;
      else if (c >= nin && p->exts[c - nin].stage == (int)s) {}
      else ok = false;
    }
    bool all_keys = true;
    for (int k : keys) all_keys = all_keys && std::find(group_cols, group_cols + n_group, k) != group_cols + n_group;
    if (ok && has_keys > 0 && all_keys) stage = (int)s;
  }
  DF_CHECK(stage >= 0, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: group keys are not determined by one join key — use the unfused dfgpu_agg");
  dfgpu_lookup* l = p->stages[stage].lookup;
  DF_CHECK(!l->acc_claimed && !l->marks_taken, DFGPU_ERR_STATE, "pipeline aggregate: the lookup's accumulators are already in use");
  const int base = 1 + (l->has_payload ? 1 : 0);
  int next = base;
  DF_CHECK(next < base + l->opt.n_acc_words, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: the lookup reserves no accumulator words (n_acc_words)");
  const int rows_word = next++;
  std::vector<PipeAgg> new_aggs = parse_pipe_aggs(p, aggs, n_aggs, mode);   // committed only when every check has passed
  const int left_kind = left >= 0 ? p->stages[left].kind : 0;
  DF_CHECK(left_kind != DFGPU_STAGE_LEFT_ANTI || n_aggs == 0, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: a LEFT_ANTI stage emits its build rows without aggregates");
  if (left_kind == DFGPU_STAGE_LEFT) check_left_args(p, new_aggs, left);
  layout_agg_words(new_aggs, next, base + l->opt.n_acc_words, l->stride % 2 == 0);
  claim_acc_words(l);
  p->rows_word = rows_word;
  p->group_cols.assign(group_cols, group_cols + n_group);
  p->aggs = std::move(new_aggs);
  l->acc_claimed = true;
  p->left_kind = left_kind;
  p->agg_stage = stage; p->agg_mode = mode; p->batch_size = batch_size; p->sink = SINK_AGG;
  DF_API_END
}

int dfgpu_pipeline_sink_aggregate_hash(dfgpu_pipeline* p, const int32_t* group_cols, const int32_t* group_nullable, int32_t n_group,
                                       const dfgpu_pipeline_agg* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size, int64_t capacity_hint) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && group_cols && n_group >= 1, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(p->sink == SINK_NONE && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline: the sink is chosen once, before the first push");
  check_no_left_stage(p);
  DF_CHECK(n_group <= kHashMaxKeys, DFGPU_ERR_UNSUPPORTED, "pipeline hash aggregate: 1..8 group columns");
  DF_CHECK(mode == DFGPU_AGG_SINGLE || mode == DFGPU_AGG_SINGLE_PARTITIONED || mode == DFGPU_AGG_PARTIAL, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: Single / SinglePartitioned / Partial");
  DF_CHECK(capacity_hint >= 0, DFGPU_ERR_INVALID, "pipeline hash aggregate: negative capacity_hint");
  for (auto& st : p->stages) DF_CHECK(st.kind != DFGPU_STAGE_MAYBE, DFGPU_ERR_UNSUPPORTED, "pipeline hash aggregate: a MAYBE stage's false positives would be counted");
  // the packed tag: each column at its width, then its NULL bit when it is nullable; at most 128 bits
  std::vector<HashKey> keys(n_group);
  int bit = 0;
  for (int g = 0; g < n_group; ++g) {
    const int c = group_cols[g];
    DF_CHECK(c >= 0 && c < (int)p->vtypes.size(), DFGPU_ERR_INVALID, "pipeline hash aggregate: group column out of range");
    DF_CHECK(key_type_ok(p->vtypes[c]), DFGPU_ERR_UNSUPPORTED, "pipeline hash aggregate: group keys must be integer-like columns of <= 64 bits");
    keys[g].src = c; keys[g].bits = 8 * type_width(p->vtypes[c]); keys[g].shift = bit;
    bit += keys[g].bits;
    keys[g].null_bit = (group_nullable && group_nullable[g]) ? bit++ : -1;
  }
  DF_CHECK(bit <= 128, DFGPU_ERR_UNSUPPORTED, "pipeline hash aggregate: the group key is wider than 128 bits — use the unfused dfgpu_agg");
  std::vector<PipeAgg> new_aggs = parse_pipe_aggs(p, aggs, n_aggs, mode);
  int next = 3;   // words 0 and 1: the tag; word 2: the row counter
  layout_agg_words(new_aggs, next, kHashMaxWords, true);
  p->hash_stride = next + (next & 1);
  p->hash_ident.assign(p->hash_stride, 0ull);
  p->hash_ident[0] = p->hash_ident[1] = kEmptyKey;
  for (const PipeAgg& ag : new_aggs) {   // MIN / MAX identities
    if (ag.func != DFGPU_AGG_MIN && ag.func != DFGPU_AGG_MAX) continue;
    const bool is_min = ag.func == DFGPU_AGG_MIN;
    unsigned long long& lo = p->hash_ident[ag.word];
    if (ag.cls == C_DEC) { lo = is_min ? ~0ull : 0ull; p->hash_ident[ag.word + 1] = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN; }
    else if (ag.cls == C_U64 || ag.cls == C_F64) lo = is_min ? ~0ull : 0ull;   // Float64: f64_to_ordered keys
    else lo = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN;
  }
  p->hash_keys = std::move(keys);
  p->hash_cap_hint = capacity_hint;
  p->rows_word = 2;
  p->group_cols.assign(group_cols, group_cols + n_group);
  p->aggs = std::move(new_aggs);
  p->agg_mode = mode; p->batch_size = batch_size; p->sink = SINK_HASH;
  DF_API_END
}

int dfgpu_pipeline_sink_aggregate_dense(dfgpu_pipeline* p, const int32_t* group_cols, const int64_t* key_min, const int64_t* key_max, int32_t n_group,
                                        const dfgpu_pipeline_agg* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && n_group >= 0 && (n_group == 0 || (group_cols && key_min && key_max)), DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(p->sink == SINK_NONE && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline: the sink is chosen once, before the first push");
  check_no_left_stage(p);
  DF_CHECK(n_group <= kDenseMaxKeys, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: 0..8 group columns");
  DF_CHECK(n_aggs >= 0 && n_aggs <= kDenseMaxAggs && (n_aggs == 0 || aggs), DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: 0..8 aggregates");
  DF_CHECK(mode == DFGPU_AGG_SINGLE || mode == DFGPU_AGG_SINGLE_PARTITIONED || mode == DFGPU_AGG_PARTIAL, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: Single / SinglePartitioned / Partial");
  for (auto& st : p->stages) DF_CHECK(st.kind != DFGPU_STAGE_MAYBE, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: a MAYBE stage's false positives would be counted");
  // group keys: slot = sum_g stride_g * idx_g, row-major over radix_g = max - min + 2 (the values, then NULL)
  std::vector<DenseKey> keys(n_group);
  std::vector<int> radix(n_group);
  uint64_t slots = 1;
  for (int g = 0; g < n_group; ++g) {
    const int c = group_cols[g];
    DF_CHECK(c >= 0 && c < (int)p->vtypes.size(), DFGPU_ERR_INVALID, "pipeline dense aggregate: group column out of range");
    const int t = p->vtypes[c];
    DF_CHECK(key_type_ok(t), DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: group keys must be integer-like columns of <= 64 bits");
    const bool uns = type_is_unsigned_int(t);
    DF_CHECK(uns ? (uint64_t)key_min[g] <= (uint64_t)key_max[g] : key_min[g] <= key_max[g], DFGPU_ERR_INVALID, "pipeline dense aggregate: key_min > key_max");
    const uint64_t span = (uint64_t)key_max[g] - (uint64_t)key_min[g];
    DF_CHECK(span < (uint64_t)kDenseMaxSlots, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: more than 256 groups (DFGPU_DENSE_MAX_GROUPS)");
    radix[g] = (int)span + 2;
    slots *= (uint64_t)radix[g];
    DF_CHECK(slots <= (uint64_t)kDenseMaxSlots, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: more than 256 groups (DFGPU_DENSE_MAX_GROUPS)");
    memset(&keys[g], 0, sizeof(DenseKey));
    keys[g].src = c; keys[g].kmin = (unsigned long long)key_min[g]; keys[g].nvals = span + 1;
  }
  uint64_t stride = 1;
  for (int g = n_group - 1; g >= 0; --g) { keys[g].stride = stride; stride *= (uint64_t)radix[g]; }
  // accumulator words of a slot: word 0 counts the rows; every SUM / MIN / MAX / AVG has its own non-null counter
  std::vector<unsigned long long> ident(1, 0ull);
  auto take = [&](int nw, unsigned long long lo, unsigned long long hi) {
    if (nw == 2 && (ident.size() & 1)) ident.push_back(0ull);   // 128-bit fields 16-byte aligned
    const int w = (int)ident.size();
    ident.push_back(lo);
    if (nw == 2) ident.push_back(hi);
    return w;
  };
  std::vector<PipeAgg> new_aggs;
  for (int a = 0; a < n_aggs; ++a) {
    PipeAgg ag;
    ag.func = aggs[a].func;
    DF_CHECK(ag.func >= DFGPU_AGG_SUM && ag.func <= DFGPU_AGG_COUNT_STAR, DFGPU_ERR_INVALID, "pipeline aggregate: unknown function");
    if (ag.func != DFGPU_AGG_COUNT_STAR) {
      DF_CHECK(aggs[a].expr && aggs[a].n_nodes > 0, DFGPU_ERR_INVALID, "pipeline aggregate: missing argument expression");
      ag.plan = plan_expr(p->vtypes.data(), (int)p->vtypes.size(), aggs[a].expr, aggs[a].n_nodes);
      ag.has_expr = true;
      ag.arg_type = ag.plan.root_type;
      ag.cls = cls_of(ag.arg_type);
      DF_CHECK(ag.cls != C_BOOL || ag.func == DFGPU_AGG_COUNT, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: Boolean arguments only for COUNT");
      if (ag.func == DFGPU_AGG_AVG) {
        DF_CHECK(ag.arg_type == DFGPU_FLOAT64 || ag.cls == C_DEC, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: AVG takes a Float64 (the planner casts) or Decimal128 argument");
        DF_CHECK(ag.cls != C_DEC || mode != DFGPU_AGG_PARTIAL, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: AVG over Decimal128 runs in Single modes only");
      }
      if (ag.func == DFGPU_AGG_MIN || ag.func == DFGPU_AGG_MAX) DF_CHECK(ag.arg_type != DFGPU_FLOAT32, DFGPU_ERR_UNSUPPORTED, "pipeline aggregate: MIN/MAX over Float32 stays on dfgpu_agg");
      const int nw = ag.cls == C_DEC ? 2 : 1;
      const bool is_min = ag.func == DFGPU_AGG_MIN;
      unsigned long long lo = 0, hi = 0;   // MIN / MAX identities
      if (ag.func == DFGPU_AGG_MIN || ag.func == DFGPU_AGG_MAX) {
        if (ag.cls == C_DEC) { lo = is_min ? ~0ull : 0ull; hi = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN; }
        else if (ag.cls == C_U64 || ag.cls == C_F64) lo = is_min ? ~0ull : 0ull;   // Float64: f64_to_ordered keys
        else lo = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN;
      }
      if (ag.func == DFGPU_AGG_COUNT) ag.word = take(1, 0, 0);
      else {
        ag.word = take(nw, lo, hi);
        ag.nn_word = take(1, 0, 0);
        if (ag.func == DFGPU_AGG_AVG) ag.cnt_word = ag.nn_word;
      }
    }
    new_aggs.push_back(std::move(ag));
  }
  if (ident.size() & 1) ident.push_back(0ull);
  DF_CHECK((int)ident.size() <= kDenseMaxWords, DFGPU_ERR_UNSUPPORTED, "pipeline dense aggregate: too many accumulator words");
  p->dense_keys = std::move(keys); p->dense_radix = std::move(radix); p->dense_ident = std::move(ident);
  p->dense_slots = (int)slots; p->dense_words = (int)p->dense_ident.size();
  p->group_cols.assign(group_cols, group_cols + n_group);
  p->aggs = std::move(new_aggs);
  p->agg_mode = mode; p->batch_size = batch_size; p->sink = SINK_DENSE;
  DF_API_END
}

int dfgpu_pipeline_sink_output(dfgpu_pipeline* p, const int32_t* out_cols, int32_t n_out, int64_t batch_size) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && out_cols && n_out >= 1 && n_out <= kMaxPipeCols, DFGPU_ERR_INVALID, "pipeline output: 1..16 columns");
  DF_CHECK(p->sink == SINK_NONE && p->m_input_rows == 0, DFGPU_ERR_STATE, "pipeline: the sink is chosen once, before the first push");
  check_no_left_stage(p);
  for (int c = 0; c < n_out; ++c) {
    DF_CHECK(out_cols[c] >= 0 && out_cols[c] < (int)p->vtypes.size(), DFGPU_ERR_INVALID, "pipeline output: column out of range");
    p->out_cols.push_back(out_cols[c]);
  }
  p->batch_size = batch_size; p->sink = SINK_OUTPUT;
  DF_API_END
}

int dfgpu_pipeline_sink_output_unordered(dfgpu_pipeline* p, const int32_t* out_cols, int32_t n_out, int64_t batch_size) {
  const int rc = dfgpu_pipeline_sink_output(p, out_cols, n_out, batch_size);
  if (rc == DFGPU_OK) p->out_ordered = false;
  return rc;
}

int dfgpu_pipeline_set_name(dfgpu_pipeline* p, const char* name) {
  if (!p || !name) return DFGPU_ERR_INVALID;
  p->name = name;
  return DFGPU_OK;
}

int dfgpu_pipeline_set_stage_filter(dfgpu_pipeline* p, int32_t stage, const dfgpu_expr_node* expr, int32_t n_nodes) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && expr && n_nodes > 0, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(stage >= 0 && stage < (int)p->stages.size(), DFGPU_ERR_INVALID, "pipeline stage filter: stage out of range");
  DF_CHECK(!p->pushed, DFGPU_ERR_STATE, "pipeline stage filter: set before the first push");
  DF_CHECK(!p->has_filt[stage], DFGPU_ERR_STATE, "pipeline stage filter: the stage already has one");
  const dfgpu_pipeline_stage& st = p->stages[stage];
  DF_CHECK(st.kind != DFGPU_STAGE_MAYBE, DFGPU_ERR_UNSUPPORTED, "pipeline stage filter: a MAYBE stage has no candidate row to test");
  check_no_right_stage(p, "pipeline stage filter: a pipeline with a RIGHT stage takes no stage filters — use dfgpu_hashjoin");
  // the filter's columns: the inputs, the payload fields of the INNER / LEFT / LEFT_ANTI stages 0..stage, then a SEMI / ANTI stage's own
  const int nin = (int)p->in_types.size();
  std::vector<int> types(p->in_types);
  std::vector<ExtDef> exts;
  for (size_t e = 0; e < p->exts.size() && p->exts[e].stage <= stage; ++e) { exts.push_back(p->exts[e]); types.push_back(p->vtypes[nin + e]); }
  if (st.kind == DFGPU_STAGE_SEMI || st.kind == DFGPU_STAGE_ANTI)
    for (size_t f = 0; f < st.lookup->pay_types.size(); ++f) {
      ExtDef e; e.stage = stage; e.shift = st.lookup->pay_shift[f]; e.width = type_width(st.lookup->pay_types[f]); e.type = st.lookup->pay_types[f];
      exts.push_back(e); types.push_back(e.type);
    }
  DF_CHECK(p->filt_nodes + n_nodes <= kFiltPoolNodes, DFGPU_ERR_UNSUPPORTED, "pipeline stage filter: the filters of a pipeline hold at most 128 nodes");
  ExprPlan plan = plan_expr(types.data(), (int)types.size(), expr, n_nodes, kFiltPoolNodes);   // the filters' own pool, not EProgram
  DF_CHECK(plan.root_type == DFGPU_BOOL, DFGPU_ERR_INVALID, "pipeline stage filter: the filter must be Boolean");
  // the short-circuit guards are resolved per batch on the host, which cannot see payload fields
  DF_CHECK(plan.guards.empty(), DFGPU_ERR_UNSUPPORTED,
           "pipeline stage filter: an AND / OR whose right operand can raise (division, modulo, CAST, Decimal128 arithmetic) stays on dfgpu_hashjoin");
  if (!p->filt_host) p->filt_host.reset(new FiltParams());
  p->filt[stage] = std::move(plan); p->filt_ext[stage] = std::move(exts); p->has_filt[stage] = true;
  p->filt_nodes += n_nodes;
  DF_API_END
}

int dfgpu_pipeline_push_device(dfgpu_pipeline* p, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && cols, DFGPU_ERR_INVALID, "null argument");
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(device_view(cols[i]));
  pipeline_push(p, v);   // consumed (stream-synchronised) before returning
  DF_API_END
}
int dfgpu_pipeline_push_host(dfgpu_pipeline* p, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p && cols, DFGPU_ERR_INVALID, "null argument");
  set_device(p->ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(upload_column(p->ctx, cols[i]));
  pipeline_push(p, v);
  DF_API_END
}
int dfgpu_pipeline_push_arrow(dfgpu_pipeline* p, const struct ArrowArray* batch, const struct ArrowSchema* schema) {
  try {
    std::vector<dfgpu_column> cols = arrow_to_columns(batch, schema);
    return dfgpu_pipeline_push_host(p, cols.data(), (int32_t)cols.size());
  } catch (const Error& e) { if (p) p->ctx->last_error = e.what(); return e.code; }
}
int dfgpu_pipeline_finish(dfgpu_pipeline* p) {
  DF_API_BEGIN(p ? p->ctx : nullptr)
  DF_CHECK(p, DFGPU_ERR_INVALID, "null argument");
  pipeline_finish(p);
  DF_API_END
}
int dfgpu_pipeline_next(dfgpu_pipeline* p, int host, dfgpu_batch** out) {
  dfgpu_ctx* _ctx = p ? p->ctx : nullptr;
  try {
    DF_CHECK(p && out, DFGPU_ERR_INVALID, "null argument");
    if (p->outq.empty()) { *out = nullptr; return DFGPU_END; }
    BatchPtr b = std::move(p->outq.front());
    p->outq.pop_front();
    if (host) { set_device(p->ctx); b = to_host_batch(p->ctx, *b); }
    *out = b.release();
    return DFGPU_OK;
  } catch (const dfgpu::Error& e) { if (_ctx) _ctx->last_error = e.what(); return e.code; }
  catch (const std::exception& e) { if (_ctx) _ctx->last_error = e.what(); return DFGPU_ERR_INVALID; }
}
int64_t dfgpu_pipeline_metric(dfgpu_pipeline* p, const char* name) {
  if (!p || !name) return -1;
  std::string s(name);
  if (s == "input_rows") return p->m_input_rows;
  if (s == "sink_rows") return p->m_sink_rows;
  if (s == "output_rows") return p->m_output_rows;
  if (s == "num_groups") return p->m_groups;
  if (s == "ring_launches") return p->m_ring_launches;   // launches of the ring-fed pipeline kernel
  if (s == "dense_block_launches") return p->m_dense_block_launches;   // dense sink launches with one accumulator copy per block (shared atomics)
  if (s == "partitioned_launches") return p->m_partitioned_launches;   // aggregate sink pushes probed from radix-partitioned records
  if (s == "partitioned_inserts") return p->m_partitioned_inserts;     // build sink pushes inserted from radix-partitioned records
  if (s == "partitioned_records") return p->m_partitioned_records;     // {key, value} records the partitioned aggregate's pass 1 wrote
  if (s == "group_rehashes") return p->m_group_rehashes;               // hash aggregate sink: times its group table grew
  if (s == "replayed_rows") return p->m_replayed_rows;                 // hash aggregate sink: rows deferred by the claim budget and pushed again
  if (s == "unmatched_build_rows") return p->m_unmatched_build_rows;   // FULL stage: build rows no probe row matched, pushed at finish
  return -1;
}
void dfgpu_pipeline_destroy(dfgpu_pipeline* p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);
  if (p->sink == SINK_AGG && p->agg_stage >= 0) p->stages[p->agg_stage].lookup->acc_claimed = false;
  delete p;
}

}  // extern "C"
