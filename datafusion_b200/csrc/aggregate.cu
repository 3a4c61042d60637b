// aggregate.cu — GpuAggregateExec: hash group-by with partial -> final merge.
//
// Reference path being replaced (SURVEY.md §8a rows a17–a25):
//   stream selection / modes      aggregates/mod.rs:289-362, 1167-1253
//   AggregateHashTable            aggregates/aggregate_hash_table/common.rs:169-366
//   GroupValuesPrimitive::intern  aggregates/group_values/single_group_by/primitive.rs:138-181
//   GroupValuesColumn (multi-col) aggregates/group_values/multi_group_by/mod.rs:455-512
//   SUM  PrimitiveGroupsAccumulator + add_wrapping   functions-aggregate-common/.../prim_op.rs:41-195, functions-aggregate/src/sum.rs:308-321
//   COUNT CountGroupsAccumulator  functions-aggregate/src/count.rs:631-780
//   NullState (seen values)       functions-aggregate-common/.../accumulate.rs:114-334
//
// GPU design: the reference interns keys to dense group ids (hashbrown + Vec) and then scatters
// into per-aggregate Vecs.  Here one kernel does both: every input row finds-or-claims an
// open-addressing slot whose tag IS the (bit-packed, exact, <= 128-bit) group key, and applies its
// aggregate updates with L2 atomics straight into struct-of-arrays accumulators indexed by slot.
// The fewer bytes the table takes, the more of it stays in L2 (50 MB on an H100) and the closer the kernel
// comes to its only necessary HBM traffic, the 16 B/row input stream.  The table grows by rehash between chunks; rows
// that cannot be placed (group budget reached) are deferred to an overflow list and replayed after
// the grow, so every row is accumulated exactly once.
// Partial/Final use the same table: Final consumes [group cols, state cols] and merges.
#include "batch.cuh"
#include "expr_dec.cuh"
#include "scan.cuh"

namespace dfgpu {

constexpr int kMaxGroupCols = 8;
constexpr int kMaxAggs = 8;
constexpr int kMaxProbe = 512;
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

using Key2 = Rec128;   // a group key of up to 128 bits, or a Decimal128 accumulator pair (expr_dec.cuh)

struct GroupCols {
  int n;
  int kw;                 // key words: 1 (<= 64 bits) or 2 (<= 128 bits)
  int single_null_slot;   // n == 1 and nullable: NULL keys go to the dedicated null-group slot
  const void* ptr[kMaxGroupCols];
  const uint8_t* valid[kMaxGroupCols];
  int64_t voff[kMaxGroupCols];
  int width[kMaxGroupCols];     // bytes; 0 = BOOL (1 bit)
  int64_t boff[kMaxGroupCols];  // BOOL value bit offset
  int shift[kMaxGroupCols];     // bit position of the value inside the 128-bit key
  int null_bit[kMaxGroupCols];  // bit position of the null flag or -1
  int is_float[kMaxGroupCols];  // canonicalise -0.0 -> +0.0 (primitive.rs:75-98)
  // wide keys (> 128 bits together): the table tag is a 64-bit hash of the key tuple, the tuple itself is stored per slot by the thread
  // that claims it (two 64-bit words per column + a NULL mask) and every row of the batch is compared against it afterwards
  // (GroupValuesColumn: hash, then vectorized_equal_to against the stored group values, group_values/multi_group_by/mod.rs:628)
  int wide;
  unsigned long long* kstore[kMaxGroupCols * 2];
  uint8_t* knull;
};

// one group column's value as stored / hashed in the wide-key path: raw bits widened to 64 (+ a second word for 16-byte types), floats
// with -0.0 folded into +0.0
__device__ __forceinline__ bool load_group_col(const GroupCols& g, int c, int64_t row, uint64_t* v, uint64_t* v2) {
  *v = 0; *v2 = 0;
  if (g.valid[c] && !bit_get(g.valid[c], g.voff[c] + row)) return false;
  switch (g.width[c]) {
    case 0: *v = bit_get((const uint8_t*)g.ptr[c], g.boff[c] + row) ? 1ull : 0ull; break;
    case 1: *v = ((const uint8_t*)g.ptr[c])[row]; break;
    case 2: *v = ((const uint16_t*)g.ptr[c])[row]; break;
    case 4: *v = ((const uint32_t*)g.ptr[c])[row]; if (g.is_float[c] && (*v & 0x7FFFFFFFull) == 0) *v = 0; break;
    case 16: *v = ((const uint64_t*)g.ptr[c])[2 * row]; *v2 = ((const uint64_t*)g.ptr[c])[2 * row + 1]; break;
    default: *v = ((const uint64_t*)g.ptr[c])[row]; if (g.is_float[c] && (*v << 1) == 0) *v = 0; break;
  }
  return true;
}
__device__ __forceinline__ uint64_t wide_group_hash(const GroupCols& g, int64_t row) {
  uint64_t h = kSeedAgg;
#pragma unroll 1
  for (int c = 0; c < g.n; ++c) {
    uint64_t v, v2;
    if (!load_group_col(g, c, row, &v, &v2)) { h = hash_combine(h, 0x6E756C6Cull + (uint64_t)c); continue; }   // NULL is a group value
    h = hash_combine(h, v);
    if (g.width[c] == 16) h = hash_combine(h, v2);
  }
  return h == kEmptyKey ? 0x5bd1e995ull : h;
}
__device__ __forceinline__ void store_group_key(const GroupCols& g, int64_t row, uint64_t slot) {
  unsigned int nullmask = 0;
#pragma unroll 1
  for (int c = 0; c < g.n; ++c) {
    uint64_t v, v2;
    if (!load_group_col(g, c, row, &v, &v2)) nullmask |= 1u << c;
    g.kstore[2 * c][slot] = v;
    if (g.width[c] == 16) g.kstore[2 * c + 1][slot] = v2;
  }
  g.knull[slot] = (uint8_t)nullmask;
}
__device__ __forceinline__ bool equal_group_key(const GroupCols& g, int64_t row, uint64_t slot) {
  const unsigned int nullmask = g.knull[slot];
#pragma unroll 1
  for (int c = 0; c < g.n; ++c) {
    uint64_t v, v2;
    const bool ok = load_group_col(g, c, row, &v, &v2);
    if (ok == (((nullmask >> c) & 1u) != 0)) return false;
    if (!ok) continue;
    if (g.kstore[2 * c][slot] != v) return false;
    if (g.width[c] == 16 && g.kstore[2 * c + 1][slot] != v2) return false;
  }
  return true;
}

__device__ __forceinline__ void key_or(Key2& k, uint64_t v, int shift) {
  // v < 2^width and shift + width <= 128, so nothing is lost
  if (shift < 64) {
    k.lo |= v << shift;
    if (shift > 0) k.hi |= v >> (64 - shift);
  } else {
    k.hi |= v << (shift - 64);
  }
}

// returns true when the row belongs to the single-column NULL group
__device__ __forceinline__ bool load_group_key(const GroupCols& g, int64_t row, Key2* out) {
  if (g.wide) { *out = Key2{wide_group_hash(g, row), 0ull}; return false; }
  Key2 k{0ull, 0ull};
  bool null_group = false;
#pragma unroll
  for (int c = 0; c < kMaxGroupCols; ++c) {
    if (c >= g.n) break;
    bool ok = !(g.valid[c] && !bit_get(g.valid[c], g.voff[c] + row));
    uint64_t v = 0;
    if (ok) {
      switch (g.width[c]) {
        case 0: v = bit_get((const uint8_t*)g.ptr[c], g.boff[c] + row) ? 1ull : 0ull; break;
        case 1: v = ((const uint8_t*)g.ptr[c])[row]; break;
        case 2: v = ((const uint16_t*)g.ptr[c])[row]; break;
        case 4: v = ((const uint32_t*)g.ptr[c])[row]; if (g.is_float[c] && (v & 0x7FFFFFFFull) == 0) v = 0; break;  // f32 -0.0 -> +0.0
        case 16: k.lo |= ((const uint64_t*)g.ptr[c])[2 * row]; k.hi |= ((const uint64_t*)g.ptr[c])[2 * row + 1]; continue;   // Decimal128: the whole 128-bit key (single group column)
        default: v = ((const uint64_t*)g.ptr[c])[row]; if (g.is_float[c] && (v << 1) == 0) v = 0; break;     // f64 -0.0 -> +0.0
      }
      key_or(k, v, g.shift[c]);
    } else {
      if (g.single_null_slot) null_group = true;
      else key_or(k, 1ull, g.null_bit[c]);
    }
  }
  *out = k;
  return null_group;
}

struct AggDev {
  int func;   // dfgpu_agg_func
  int cls;    // 0 signed int, 1 unsigned int, 2 float  (class of the accumulated value)
  int merge;  // 1 = inputs are partial states
  int in0_type, in1_type;
  const void* in0; const uint8_t* in0_valid; int64_t in0_voff;  // BOOL in0: in0_voff doubles as value offset
  const void* in1; const uint8_t* in1_valid; int64_t in1_voff;
  const uint8_t* filt; int64_t filt_off; const uint8_t* filt_valid; int64_t filt_voff;
  unsigned long long* acc0;  // sum / min / max / count; Decimal128 SUM: low words; Decimal128 MIN / MAX / AVG: one {lo, hi} pair per slot
  unsigned long long* acc1;  // AVG: count; Decimal128 SUM: high words
  uint8_t* seen;             // NullState::seen_values (nullptr = SeenValues::All)
};
struct AggSet { int n; AggDev a[kMaxAggs]; };

__device__ __forceinline__ int64_t load_as_i64(const void* p, int type, int64_t i) {
  switch (type) {
    case DFGPU_INT8: return ((const int8_t*)p)[i];
    case DFGPU_INT16: return ((const int16_t*)p)[i];
    case DFGPU_INT32: case DFGPU_DATE32: return ((const int32_t*)p)[i];
    case DFGPU_UINT8: return ((const uint8_t*)p)[i];
    case DFGPU_UINT16: return ((const uint16_t*)p)[i];
    case DFGPU_UINT32: return ((const uint32_t*)p)[i];
    case DFGPU_FLOAT32: return (int64_t)((const float*)p)[i];
    case DFGPU_FLOAT64: return (int64_t)((const double*)p)[i];
    default: return ((const int64_t*)p)[i];
  }
}
__device__ __forceinline__ double load_as_f64(const void* p, int type, int64_t i) {
  switch (type) {
    case DFGPU_FLOAT32: return (double)((const float*)p)[i];
    case DFGPU_FLOAT64: return ((const double*)p)[i];
    case DFGPU_UINT64: return (double)((const uint64_t*)p)[i];
    default: return (double)load_as_i64(p, type, i);
  }
}
// order-preserving map double -> uint64 (IEEE total order: -NaN < -inf < ... < +inf < +NaN)
__host__ __device__ __forceinline__ uint64_t f64_to_ordered(double d) {
  uint64_t b;
  memcpy(&b, &d, 8);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double ordered_to_f64(uint64_t u) {
  uint64_t b = (u & 0x8000000000000000ull) ? (u & 0x7FFFFFFFFFFFFFFFull) : ~u;
  double d;
  memcpy(&d, &b, 8);
  return d;
}

// i128 add_wrapping as two 64-bit atomics: the carry out of the low word is a function of this add alone (old + lo overflowed), so the
// high words sum to the right value in any interleaving
__device__ __forceinline__ void add_i128(unsigned long long* lo_word, unsigned long long* hi_word, unsigned long long lo, unsigned long long hi) {
  const unsigned long long old = atomicAdd(lo_word, lo);
  const unsigned long long carry = (old + lo) < old ? 1ull : 0ull;
  if (hi + carry) atomicAdd(hi_word, hi + carry);
}

// PAIR: the aggregate set has a Decimal128 MIN / MAX / AVG ({lo, hi} pair accumulators).  Only those update kernels compile their
// updates: in the others the CAS loop would cost registers on every path (the 128-bit-key kernel would spill)
template <bool PAIR>
__device__ __forceinline__ void apply_agg(const AggDev& a, int64_t row, uint64_t slot) {
  // opt_filter: only rows whose filter is Some(true) contribute (accumulate.rs:373-470)
  if (a.filt) {
    if (a.filt_valid && !bit_get(a.filt_valid, a.filt_voff + row)) return;
    if (!bit_get(a.filt, a.filt_off + row)) return;
  }
  if (a.func == DFGPU_AGG_COUNT_STAR && !a.merge) { atomicAdd(&a.acc0[slot], 1ull); return; }
  if (a.in0_valid && !bit_get(a.in0_valid, a.in0_voff + row)) {
    if (!(a.func == DFGPU_AGG_AVG && a.merge)) return;  // NULL input: skipped
  }
  switch (a.func) {
    case DFGPU_AGG_COUNT:
    case DFGPU_AGG_COUNT_STAR:
      // update: +1 per non-null row (count.rs:648-672); merge: + partial count (count.rs:675-698)
      atomicAdd(&a.acc0[slot], a.merge ? (unsigned long long)((const int64_t*)a.in0)[row] : 1ull);
      break;
    case DFGPU_AGG_SUM:
      if (a.cls == 3) {   // Decimal128: i128 add_wrapping (sum.rs:316 on Decimal128Type)
        const unsigned long long* p = (const unsigned long long*)a.in0 + 2 * row;
        add_i128(&a.acc0[slot], &a.acc1[slot], p[0], p[1]);
      } else if (a.cls == 2) atomicAdd((double*)&a.acc0[slot], load_as_f64(a.in0, a.in0_type, row));
      else if (a.in0_type == DFGPU_UINT64) atomicAdd(&a.acc0[slot], (unsigned long long)((const uint64_t*)a.in0)[row]);
      else atomicAdd(&a.acc0[slot], (unsigned long long)load_as_i64(a.in0, a.in0_type, row));  // add_wrapping (sum.rs:316)
      if (a.seen) a.seen[slot] = 1;
      break;
    case DFGPU_AGG_MIN:
    case DFGPU_AGG_MAX: {
      const bool is_min = a.func == DFGPU_AGG_MIN;
      if (PAIR && a.cls == 3) {
        Key2* w = (Key2*)a.acc0 + slot;
        const unsigned long long* p = (const unsigned long long*)a.in0 + 2 * row;
        minmax_i128(w, Key2{p[0], p[1]}, is_min);
      }
      else if (a.cls == 0) {
        long long v = load_as_i64(a.in0, a.in0_type, row);
        if (is_min) atomicMin((long long*)&a.acc0[slot], v); else atomicMax((long long*)&a.acc0[slot], v);
      } else {
        unsigned long long v = a.cls == 2 ? f64_to_ordered(load_as_f64(a.in0, a.in0_type, row))
                               : (a.in0_type == DFGPU_UINT64 ? ((const uint64_t*)a.in0)[row] : (unsigned long long)load_as_i64(a.in0, a.in0_type, row));
        if (is_min) atomicMin(&a.acc0[slot], v); else atomicMax(&a.acc0[slot], v);
      }
      if (a.seen) a.seen[slot] = 1;
      break;
    }
    case DFGPU_AGG_AVG:
      if (PAIR && a.cls == 3) {
        // Decimal128: i128 add_wrapping of the sum into the slot's {lo, hi} pair + a count (DecimalAverager's inputs).  The merge reads the
        // no-GROUP-BY composite's internal state [count: UInt64, sum: Decimal128]
        if (!(a.merge && a.in1_valid && !bit_get(a.in1_valid, a.in1_voff + row))) {
          const unsigned long long* p = (const unsigned long long*)(a.merge ? a.in1 : a.in0) + 2 * row;
          add_i128(&a.acc0[2 * slot], &a.acc0[2 * slot + 1], p[0], p[1]);
        }
        atomicAdd(&a.acc1[slot], a.merge ? (unsigned long long)((const uint64_t*)a.in0)[row] : 1ull);
      } else if (a.merge) {
        // state = [count: UInt64, sum: Float64]
        unsigned long long c = ((const uint64_t*)a.in0)[row];
        atomicAdd(&a.acc1[slot], c);
        if (!(a.in1_valid && !bit_get(a.in1_valid, a.in1_voff + row))) atomicAdd((double*)&a.acc0[slot], ((const double*)a.in1)[row]);
      } else {
        atomicAdd((double*)&a.acc0[slot], load_as_f64(a.in0, a.in0_type, row));
        atomicAdd(&a.acc1[slot], 1ull);
      }
      break;
  }
}

struct TableDev {
  void* tags;                 // KW=1: uint64[cap+2]; KW=2: Key2[cap+2]
  uint64_t cap;
  unsigned long long* ngroups;  // claimed regular slots
  uint64_t group_limit;         // stop claiming beyond this (load-factor guard)
  uint32_t* special_used;       // [0]: slot cap (key == all-ones), [1]: slot cap+1 (NULL group)
  int bucketed;                 // probe sequences start on a 32-byte boundary (4 x 8-byte tags): one sector holds the first 4 candidates
};

// find-or-claim; returns slot or ~0ull when the row must be deferred (table budget exhausted)
template <int KW>
__device__ __forceinline__ uint64_t start_slot(const TableDev& t, const Key2& k) {
  uint64_t h = KW == 1 ? hash_u64(k.lo, kSeedAgg) : hash_combine(hash_u64(k.lo, kSeedAgg), k.hi);
  if (KW == 1 && t.bucketed) return __umul64hi(h, t.cap >> 2) << 2;
  return __umul64hi(h, t.cap);
}
template <int KW>
__device__ __forceinline__ Key2 load_tag_at(const TableDev& t, uint64_t s) {
  if (KW == 1) return Key2{__ldcg((const unsigned long long*)t.tags + s), 0ull};
  uint4 raw = __ldcg((const uint4*)((const Key2*)t.tags + s));
  return Key2{(unsigned long long)raw.x | ((unsigned long long)raw.y << 32), (unsigned long long)raw.z | ((unsigned long long)raw.w << 32)};
}
__device__ __forceinline__ bool key_is_empty(const Key2& k, int kw) { return k.lo == kEmptyKey && (kw == 1 || k.hi == kEmptyKey); }

// find-or-claim starting at slot s with the tag already fetched in `cur` (the caller issues the first-probe
// loads of several rows back to back).  Returns the slot or ~0ull when the row must be deferred.
template <int KW>
__device__ __forceinline__ uint64_t find_or_claim_from(const TableDev& t, const Key2& k, uint64_t s, Key2 cur, bool* claimed) {
  *claimed = false;
  for (int probe = 0; probe < kMaxProbe; ++probe) {
    if (cur.lo == k.lo && (KW == 1 || cur.hi == k.hi)) return s;
    if (key_is_empty(cur, KW)) {
      if (__ldcg(t.ngroups) >= t.group_limit) return ~0ull;
      Key2 prev;
      if (KW == 1) prev = Key2{atomicCAS((unsigned long long*)t.tags + s, (unsigned long long)kEmptyKey, k.lo), 0ull};
      else prev = cas128((Key2*)t.tags + s, Key2{kEmptyKey, kEmptyKey}, k);
      if (key_is_empty(prev, KW)) { *claimed = true; return s; }
      if (prev.lo == k.lo && (KW == 1 || prev.hi == k.hi)) return s;
    }
    if (++s == t.cap) s = 0;
    cur = load_tag_at<KW>(t, s);
  }
  return ~0ull;
}
template <int KW>
__device__ __forceinline__ uint64_t find_or_claim(const TableDev& t, Key2 k, bool null_group, bool may_claim, bool* claimed) {
  *claimed = false;
  if (null_group) { if (!t.special_used[1]) t.special_used[1] = 1; return t.cap + 1; }
  if (key_is_empty(k, KW)) { if (!t.special_used[0]) t.special_used[0] = 1; return t.cap; }
  const uint64_t s = start_slot<KW>(t, k);
  return find_or_claim_from<KW>(t, k, s, load_tag_at<KW>(t, s), claimed);
}

// the hot kernel: intern + accumulate.  Each thread owns R independent rows per iteration: their keys, then
// their first-probe tags, are loaded back to back BEFORE any is consumed — the loop is latency-bound
// (DRAM stream -> L2 tag -> RED), so memory-level parallelism per thread is what sets the rate.
template <int KW, int R, bool PAIR>
__global__ void __launch_bounds__(256) agg_update_kernel(GroupCols g, AggSet aggs, TableDev t, int64_t row0, int64_t n,
                                                      const uint32_t* __restrict__ row_list, uint32_t* __restrict__ overflow,
                                                      unsigned long long* __restrict__ overflow_count) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < n; i0 += stride * R) {
    int64_t row[R];
    Key2 k[R], cur[R];
    uint64_t s[R];
    bool live[R], ng[R], special[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t i = i0 + r * stride;
      live[r] = i < n;
      row[r] = live[r] ? row0 + (row_list ? (int64_t)row_list[i] : i) : 0;
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      ng[r] = false; special[r] = false; s[r] = 0; k[r] = Key2{0, 0};
      if (live[r]) {
        ng[r] = load_group_key(g, row[r], &k[r]);
        special[r] = ng[r] || key_is_empty(k[r], KW);
        if (!special[r]) s[r] = start_slot<KW>(t, k[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      cur[r] = Key2{0, 0};
      if (live[r] && !special[r]) cur[r] = load_tag_at<KW>(t, s[r]);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      bool claimed = false;
      uint64_t slot = ~0ull;
      if (live[r]) {
        if (special[r]) slot = find_or_claim<KW>(t, k[r], ng[r], true, &claimed);
        else slot = find_or_claim_from<KW>(t, k[r], s[r], cur[r], &claimed);
      }
      {  // one atomic per warp for the group counter (1M claims on one address would serialise otherwise)
        const unsigned act = __activemask();
        const unsigned m = __ballot_sync(act, claimed);
        if (m && (threadIdx.x & 31) == (unsigned)(__ffs(m) - 1)) atomicAdd(t.ngroups, (unsigned long long)__popc(m));
      }
      if (!live[r]) continue;
      if (slot == ~0ull) {
        unsigned long long pos = atomicAdd(overflow_count, 1ull);
        overflow[pos] = (uint32_t)(row[r] - row0);
        continue;
      }
      if (KW == 1 && claimed && g.wide) store_group_key(g, row[r], slot);   // read back only by later kernels (verify, rehash, emit)
#pragma unroll 1
      for (int a = 0; a < aggs.n; ++a) apply_agg<PAIR>(aggs.a[a], row[r], slot);
    }
  }
}
// wide keys: every row of the chunk against the key tuple stored in its slot.  Runs after the update kernel (and its replays) finished, so
// every claim and its stored tuple is visible; a mismatch means two distinct tuples share a 64-bit hash.
__global__ void __launch_bounds__(256) agg_verify_wide_kernel(GroupCols g, TableDev t, int64_t row0, int64_t n, int* __restrict__ mismatch) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = row0 + i;
    const uint64_t h = wide_group_hash(g, row);
    uint64_t s = start_slot<1>(t, Key2{h, 0ull});
    bool found = false;
    for (int probe = 0; probe < kMaxProbe; ++probe) {
      const unsigned long long tag = ((const unsigned long long*)t.tags)[s];
      if (tag == h) { found = true; break; }
      if (tag == kEmptyKey) break;
      if (++s == t.cap) s = 0;
    }
    if (!found || !equal_group_key(g, row, s)) *mismatch = 1;
  }
}

// ---- fast path: one non-null 8-byte key, every aggregate of the form acc[slot] += (column ? column[row] : 1) ----
// (SUM over a non-null 8-byte integer column, COUNT / COUNT(*) without NULLs or FILTER, and their Final-mode
// merges) — the C3 shape.  No type switches, no validity reads; 4 rows per thread with the loads hoisted.
constexpr int kMaxFastAggs = 4;
constexpr int kAggPairedDefault = 4;   // DFGPU_AGG_PAIRED when not set: agg_update_pair_kernel<3, true>
struct FastAggs { int n; const unsigned long long* col[kMaxFastAggs]; unsigned long long* acc[kMaxFastAggs]; };

template <int R, int NA, int B>
__global__ void __launch_bounds__(256) agg_update_fast_kernel(const unsigned long long* __restrict__ keys, FastAggs fa, TableDev t, int64_t row0, int64_t n,
                                                           const uint32_t* __restrict__ row_list, uint32_t* __restrict__ overflow,
                                                           unsigned long long* __restrict__ overflow_count) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < n; i0 += stride * R) {
    int64_t row[R];
    unsigned long long k[R], cur[R], v[R][NA];
    uint4 bk0[B ? R : 1], bk1[B ? R : 1];
    uint64_t s[R];
    bool live[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t i = i0 + r * stride;
      live[r] = i < n;
      row[r] = live[r] ? row0 + (row_list ? (int64_t)row_list[i] : i) : row0;
    }
#pragma unroll
    for (int r = 0; r < R; ++r) k[r] = live[r] ? keys[row[r]] : 0ull;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int a = 0; a < NA; ++a) v[r][a] = (fa.col[a] && live[r]) ? fa.col[a][row[r]] : 1ull;
#pragma unroll
    for (int r = 0; r < R; ++r) { s[r] = start_slot<1>(t, Key2{k[r], 0ull}); cur[r] = 0; }
    if (B) {
      // the 32-byte sector at the (aligned) start slot holds the first four candidates: fetch it whole
#pragma unroll
      for (int r = 0; r < R; ++r) {
        bk0[r] = make_uint4(0, 0, 0, 0); bk1[r] = bk0[r];
        if (live[r] && k[r] != kEmptyKey) { const uint4* bp = (const uint4*)((const unsigned long long*)t.tags + s[r]); bk0[r] = __ldcg(bp); bk1[r] = __ldcg(bp + 1); }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        if (!(live[r] && k[r] != kEmptyKey)) continue;
        const unsigned long long t0 = (unsigned long long)bk0[r].x | ((unsigned long long)bk0[r].y << 32), t1 = (unsigned long long)bk0[r].z | ((unsigned long long)bk0[r].w << 32);
        const unsigned long long t2 = (unsigned long long)bk1[r].x | ((unsigned long long)bk1[r].y << 32), t3 = (unsigned long long)bk1[r].z | ((unsigned long long)bk1[r].w << 32);
        // first slot that either holds the key or is empty (linear-probing order inside the sector)
        if (t0 == k[r] || t0 == kEmptyKey) { cur[r] = t0; }
        else if (t1 == k[r] || t1 == kEmptyKey) { cur[r] = t1; s[r] += 1; }
        else if (t2 == k[r] || t2 == kEmptyKey) { cur[r] = t2; s[r] += 2; }
        else { cur[r] = t3; s[r] += 3; }
      }
    } else {
#pragma unroll
      for (int r = 0; r < R; ++r) if (live[r] && k[r] != kEmptyKey) cur[r] = __ldcg((const unsigned long long*)t.tags + s[r]);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      bool claimed = false;
      uint64_t slot = ~0ull;
      if (live[r]) {
        if (k[r] == kEmptyKey) slot = find_or_claim<1>(t, Key2{k[r], 0ull}, false, true, &claimed);
        else slot = find_or_claim_from<1>(t, Key2{k[r], 0ull}, s[r], Key2{cur[r], 0ull}, &claimed);
      }
      {
        const unsigned act = __activemask();
        const unsigned m = __ballot_sync(act, claimed);
        if (m && (threadIdx.x & 31) == (unsigned)(__ffs(m) - 1)) atomicAdd(t.ngroups, (unsigned long long)__popc(m));
      }
      if (!live[r]) continue;
      if (slot == ~0ull) {
        unsigned long long pos = atomicAdd(overflow_count, 1ull);
        overflow[pos] = (uint32_t)(row[r] - row0);
        continue;
      }
#pragma unroll
      for (int a = 0; a < NA; ++a) atomicAdd(&fa.acc[a][slot], v[r][a]);
    }
  }
}

// ---- paired accumulators: the two-aggregate fast path (SUM + COUNT, the C3 shape) with ONE L2 reduction request per row ----
// The kernel above is bound by the number of L2 atomic requests (two RED instructions per row, 32 distinct sectors each).  Here the
// slot's two accumulators are adjacent — pairs[slot] = {acc of aggregate 0, acc of aggregate 1}, one 16-byte half-sector — and a lane
// PAIR updates one slot with one RED instruction: in the first instruction the even lane adds its row's first value while its odd
// neighbour adds the same row's second value (same sector, same instruction: the LSU hands L2 one sector request with two active
// words); the second instruction does the odd lanes' rows.  A warp's RED instruction touches 16 sectors instead of 32.
// `pairs` holds additive deltas only; agg_fold_pairs_kernel adds them into the per-aggregate arrays before anything else reads those.
__device__ __forceinline__ void red_add_u64_pred(unsigned long long* p, unsigned long long v, bool on) {
  if (on) asm volatile("red.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
// the 32-byte sector of a bucket (four tags).  sm_90 has no 256-bit load, so this issues the same two 128-bit loads as WIDE = false:
// on Hopper both instantiations ask L2 for two half-sector requests per bucket
__device__ __forceinline__ void ld_bucket_256(const unsigned long long* p, unsigned long long t[4]) {
  asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(t[0]), "=l"(t[1]) : "l"(p));
  asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(t[2]), "=l"(t[3]) : "l"(p + 2));
}
template <int R, bool WIDE>
__global__ void __launch_bounds__(256) agg_update_pair_kernel(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ col0,
                                                           const unsigned long long* __restrict__ col1, ulonglong2* __restrict__ pairs, TableDev t,
                                                           int64_t row0, int64_t n, const uint32_t* __restrict__ row_list, uint32_t* __restrict__ overflow,
                                                           unsigned long long* __restrict__ overflow_count) {
  const int lane = threadIdx.x & 31;
  const bool even = !(lane & 1);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  // the trip count is warp-uniform (lanes past the end stay in the loop, dead): the lane pairs exchange values with full-mask shuffles
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 - lane < n; i0 += stride * R) {
    int64_t row[R];
    unsigned long long k[R], cur[R], v0[R], v1[R], tg[R][4];
    uint64_t s[R];
    bool live[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t i = i0 + r * stride;
      live[r] = i < n;
      row[r] = live[r] ? row0 + (row_list ? (int64_t)row_list[i] : i) : row0;
    }
#pragma unroll
    for (int r = 0; r < R; ++r) k[r] = live[r] ? keys[row[r]] : 0ull;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      v0[r] = (col0 && live[r]) ? col0[row[r]] : 1ull;
      v1[r] = (col1 && live[r]) ? col1[row[r]] : 1ull;
    }
#pragma unroll
    for (int r = 0; r < R; ++r) { s[r] = start_slot<1>(t, Key2{k[r], 0ull}); cur[r] = 0; }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      tg[r][0] = tg[r][1] = tg[r][2] = tg[r][3] = 0ull;
      if (live[r] && k[r] != kEmptyKey) {
        const unsigned long long* bp = (const unsigned long long*)t.tags + s[r];   // start slots are multiples of four: 32-byte aligned
        if (WIDE) ld_bucket_256(bp, tg[r]);
        else {
          const uint4 b0 = __ldcg((const uint4*)bp), b1 = __ldcg((const uint4*)bp + 1);
          tg[r][0] = (unsigned long long)b0.x | ((unsigned long long)b0.y << 32); tg[r][1] = (unsigned long long)b0.z | ((unsigned long long)b0.w << 32);
          tg[r][2] = (unsigned long long)b1.x | ((unsigned long long)b1.y << 32); tg[r][3] = (unsigned long long)b1.z | ((unsigned long long)b1.w << 32);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (!(live[r] && k[r] != kEmptyKey)) continue;
      const unsigned long long t0 = tg[r][0], t1 = tg[r][1], t2 = tg[r][2], t3 = tg[r][3];
      if (t0 == k[r] || t0 == kEmptyKey) { cur[r] = t0; }
      else if (t1 == k[r] || t1 == kEmptyKey) { cur[r] = t1; s[r] += 1; }
      else if (t2 == k[r] || t2 == kEmptyKey) { cur[r] = t2; s[r] += 2; }
      else { cur[r] = t3; s[r] += 3; }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      bool claimed = false;
      uint64_t slot = ~0ull;
      if (live[r]) {
        if (k[r] == kEmptyKey) slot = find_or_claim<1>(t, Key2{k[r], 0ull}, false, true, &claimed);
        else slot = find_or_claim_from<1>(t, Key2{k[r], 0ull}, s[r], Key2{cur[r], 0ull}, &claimed);
      }
      __syncwarp();
      const unsigned m = __ballot_sync(0xffffffffu, claimed);
      if (m && lane == __ffs(m) - 1) atomicAdd(t.ngroups, (unsigned long long)__popc(m));
      const bool ok = live[r] && slot != ~0ull;
      if (live[r] && !ok) {   // table budget exhausted: the host grows the table and replays the row
        const unsigned long long pos = atomicAdd(overflow_count, 1ull);
        overflow[pos] = (uint32_t)(row[r] - row0);
      }
      __syncwarp();
      const uint32_t ms = (uint32_t)slot;                                       // the launcher guarantees cap + 2 < 2^32
      const uint32_t ps = __shfl_xor_sync(0xffffffffu, ms, 1);                  // the neighbour's slot, second value, row state
      const unsigned long long pv1 = __shfl_xor_sync(0xffffffffu, v1[r], 1);
      const bool pok = __shfl_xor_sync(0xffffffffu, ok ? 1 : 0, 1) != 0;
      unsigned long long* const mine = &pairs[ok ? ms : 0u].x;                  // this lane's row, first accumulator
      unsigned long long* const theirs = &pairs[pok ? ps : 0u].y;               // the neighbour's row, second accumulator
      red_add_u64_pred(even ? mine : theirs, even ? v0[r] : pv1, even ? ok : pok);    // rows of the even lanes
      red_add_u64_pred(even ? theirs : mine, even ? pv1 : v0[r], even ? pok : ok);    // rows of the odd lanes
    }
  }
}
__global__ void __launch_bounds__(256) agg_fold_pairs_kernel(ulonglong2* __restrict__ pairs, unsigned long long* __restrict__ acc_a, unsigned long long* __restrict__ acc_b, uint64_t n) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const ulonglong2 p = pairs[i];
    if (p.x | p.y) { acc_a[i] += p.x; acc_b[i] += p.y; pairs[i] = make_ulonglong2(0ull, 0ull); }
  }
}

// per aggregate at most acc0, acc1 and seen (a Decimal128 MIN / MAX has acc0 + seen, a Decimal128 AVG acc0 + acc1); wide keys add two
// stored words per group column and the NULL masks
struct AccArrays { int n; void* ptr[kMaxAggs * 3 + kMaxGroupCols * 2 + 1]; void* new_ptr[kMaxAggs * 3 + kMaxGroupCols * 2 + 1]; int elem[kMaxAggs * 3 + kMaxGroupCols * 2 + 1]; };

// grow: re-insert every occupied slot of the old table into the new one and move its accumulators
template <int KW>
__global__ void __launch_bounds__(256) agg_rehash_kernel(TableDev old_t, TableDev new_t, AccArrays acc) {
  const uint64_t total = old_t.cap + 2;
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < total; s += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t ns;
    if (s >= old_t.cap) {
      if (!old_t.special_used[s - old_t.cap]) continue;
      ns = new_t.cap + (s - old_t.cap);
      new_t.special_used[s - old_t.cap] = 1;
    } else {
      Key2 k;
      if (KW == 1) { k.lo = ((const unsigned long long*)old_t.tags)[s]; k.hi = 0; if (k.lo == kEmptyKey) continue; }
      else { k = ((const Key2*)old_t.tags)[s]; if (k.lo == kEmptyKey && k.hi == kEmptyKey) continue; }
      bool claimed;
      ns = find_or_claim<KW>(new_t, k, false, true, &claimed);  // the group count is copied over by the host
    }
    for (int a = 0; a < acc.n; ++a) {
      if (acc.elem[a] == 8) ((uint64_t*)acc.new_ptr[a])[ns] = ((const uint64_t*)acc.ptr[a])[s];
      else if (acc.elem[a] == 16) ((ulonglong2*)acc.new_ptr[a])[ns] = ((const ulonglong2*)acc.ptr[a])[s];
      else ((uint8_t*)acc.new_ptr[a])[ns] = ((const uint8_t*)acc.ptr[a])[s];
    }
  }
}

template <int KW>
__global__ void agg_occupancy_kernel(TableDev t, uint32_t* __restrict__ words) {
  const uint64_t total = t.cap + 2;
  const uint64_t nw = (total + 31) / 32;
  int lane = threadIdx.x & 31;
  for (uint64_t wi = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    uint64_t s = wi * 32 + lane;
    bool occ = false;
    if (s < t.cap) {
      if (KW == 1) occ = ((const unsigned long long*)t.tags)[s] != kEmptyKey;
      else { Key2 k = ((const Key2*)t.tags)[s]; occ = !(k.lo == kEmptyKey && k.hi == kEmptyKey); }
    } else if (s < total) occ = t.special_used[s - t.cap] != 0;
    uint32_t w = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) words[wi] = w;
  }
}

// seen[] materialisation when the first batch with NULLs / a filter arrives: every existing group
// has seen a value (SeenValues::All -> Some, accumulate.rs:59-82)
template <int KW>
__global__ void agg_init_seen_kernel(TableDev t, uint8_t* __restrict__ seen) {
  const uint64_t total = t.cap + 2;
  for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < total; s += (uint64_t)gridDim.x * blockDim.x) {
    bool occ;
    if (s < t.cap) {
      if (KW == 1) occ = ((const unsigned long long*)t.tags)[s] != kEmptyKey;
      else { Key2 k = ((const Key2*)t.tags)[s]; occ = !(k.lo == kEmptyKey && k.hi == kEmptyKey); }
    } else occ = t.special_used[s - t.cap] != 0;
    seen[s] = occ ? 1 : 0;
  }
}

// ---- emit kernels: one per output column, 32 consecutive outputs per warp ----
enum EmitKind : int { EK_KEY = 0, EK_COPY64 = 1, EK_AVG = 2, EK_MINMAX = 3, EK_DEC128 = 4, EK_WIDEKEY = 5, EK_PAIR128 = 6, EK_AVG_DEC = 7 };
struct EmitDesc {
  int kind;
  int out_type;        // output column type
  int kw;
  const void* tags;
  uint64_t cap;
  int shift, width_bits, null_bit, single_null_slot;  // EK_KEY
  const unsigned long long* acc0;
  const unsigned long long* acc1;
  const uint8_t* seen;
  int cls;             // EK_MINMAX: 0 signed, 1 unsigned, 2 float
  int avg_mul, avg_prec;           // EK_AVG_DEC: sum * 10^avg_mul / count must fit Decimal128(avg_prec, _)
  unsigned long long* err;         // EK_AVG_DEC: set to 1 on overflow
};

__device__ __forceinline__ void store_typed(void* out, int type, int64_t i, uint64_t bits) {
  switch (type_width(type)) {
    case 1: ((uint8_t*)out)[i] = (uint8_t)bits; break;
    case 2: ((uint16_t*)out)[i] = (uint16_t)bits; break;
    case 4: ((uint32_t*)out)[i] = (uint32_t)bits; break;
    default: ((uint64_t*)out)[i] = bits; break;
  }
}

__global__ void __launch_bounds__(256) agg_emit_kernel(EmitDesc d, const uint32_t* __restrict__ slot_idx, int64_t n, void* __restrict__ out,
                                                    uint32_t* __restrict__ out_valid, uint32_t* __restrict__ out_boolbits) {
  const int64_t nw = (n + 31) / 32;
  int lane = threadIdx.x & 31;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    int64_t i = wi * 32 + lane;
    bool ok = false, bval = false;
    if (i < n) {
      uint64_t s = slot_idx[i];
      ok = true;
      uint64_t bits = 0;
      switch (d.kind) {
        case EK_KEY: {
          if (s == d.cap + 1) { ok = false; break; }  // the NULL group (primitive.rs:195-249 build_primitive)
          unsigned long long lo, hi = 0;
          if (s == d.cap) { lo = kEmptyKey; hi = kEmptyKey; }
          else if (d.kw == 1) lo = ((const unsigned long long*)d.tags)[s];
          else { Key2 k = ((const Key2*)d.tags)[s]; lo = k.lo; hi = k.hi; }
          if (d.null_bit >= 0) {
            bool isnull = d.null_bit < 64 ? ((lo >> d.null_bit) & 1) : ((hi >> (d.null_bit - 64)) & 1);
            if (isnull) { ok = false; break; }
          }
          if (d.width_bits == 128) { ((unsigned long long*)out)[2 * i] = lo; ((unsigned long long*)out)[2 * i + 1] = hi; break; }   // Decimal128 key
          if (d.shift < 64) {
            bits = lo >> d.shift;
            if (d.shift > 0 && d.shift + d.width_bits > 64) bits |= hi << (64 - d.shift);
          } else bits = hi >> (d.shift - 64);
          if (d.width_bits < 64) bits &= (1ull << d.width_bits) - 1ull;
          break;
        }
        case EK_COPY64:
          bits = d.acc0[s];
          if (d.seen) ok = d.seen[s] != 0;
          break;
        case EK_WIDEKEY:   // acc0 / acc1: the column's stored words, seen: the slots' NULL masks, null_bit: this column's bit
          ok = ((d.seen[s] >> d.null_bit) & 1) == 0;
          bits = d.acc0[s];
          if (type_width(d.out_type) == 16) { ((unsigned long long*)out)[2 * i] = ok ? d.acc0[s] : 0ull; ((unsigned long long*)out)[2 * i + 1] = ok ? d.acc1[s] : 0ull; }
          break;
        case EK_DEC128:
          if (d.seen) ok = d.seen[s] != 0;
          ((unsigned long long*)out)[2 * i] = ok ? d.acc0[s] : 0ull;
          ((unsigned long long*)out)[2 * i + 1] = ok ? d.acc1[s] : 0ull;
          break;
        case EK_PAIR128:   // the slot's {lo, hi} pair: Decimal128 MIN / MAX, the AVG sum state
          if (d.seen) ok = d.seen[s] != 0;
          ((unsigned long long*)out)[2 * i] = ok ? d.acc0[2 * s] : 0ull;
          ((unsigned long long*)out)[2 * i + 1] = ok ? d.acc0[2 * s + 1] : 0ull;
          break;
        case EK_AVG_DEC: {   // DecimalAverager::avg (expr_dec.cuh dec_avg); no value -> NULL
          const unsigned long long c = d.acc1[s];
          ok = c != 0ull;
          i128 q = 0;
          if (ok && !dec_avg((i128)(((u128)d.acc0[2 * s + 1] << 64) | (u128)d.acc0[2 * s]), c, d.avg_mul, d.avg_prec, &q)) atomicOr(d.err, 1ull);
          ((unsigned long long*)out)[2 * i] = (unsigned long long)(u128)q;
          ((unsigned long long*)out)[2 * i + 1] = (unsigned long long)((u128)q >> 64);
          break;
        }
        case EK_AVG: {
          unsigned long long c = d.acc1[s];
          if (c == 0) { ok = false; break; }
          double sum;
          memcpy(&sum, &d.acc0[s], 8);
          double r = sum / (double)c;
          memcpy(&bits, &r, 8);
          break;
        }
        case EK_MINMAX: {
          if (d.seen) ok = d.seen[s] != 0;
          unsigned long long v = d.acc0[s];
          if (d.cls == 2) {
            double dv = ordered_to_f64(v);
            if (d.out_type == DFGPU_FLOAT32) { float f = (float)dv; uint32_t fb; memcpy(&fb, &f, 4); bits = fb; }
            else memcpy(&bits, &dv, 8);
          } else bits = v;
          break;
        }
      }
      if (!ok) bits = 0;
      if (d.out_type == DFGPU_BOOL) bval = bits & 1;
      else if (type_width(d.out_type) == 16) { if (!ok && d.kind != EK_WIDEKEY) { ((unsigned long long*)out)[2 * i] = 0ull; ((unsigned long long*)out)[2 * i + 1] = 0ull; } }   // 16-byte values were stored above
      else store_typed(out, d.out_type, i, bits);
    }
    uint32_t vw = __ballot_sync(0xffffffffu, ok);
    uint32_t bw = __ballot_sync(0xffffffffu, bval);
    if (lane == 0) {
      if (out_valid) out_valid[wi] = vw;
      if (out_boolbits) out_boolbits[wi] = bw;
    }
  }
}

// convert_to_state (GroupsAccumulator::convert_to_state, prim_op.rs / count.rs:722 / average.rs; partial_table.rs:199-238): in
// SkippingAggregation mode every input row becomes its own state row — SUM / MIN / MAX state = the value (NULL when the value is NULL
// or the FILTER rejects the row), COUNT state = 1 / 0, AVG state = [count 1 / 0, sum value].  One warp owns 32 rows: validity leaves
// as ballot words.
struct StateOut { void* v0; uint32_t* valid0; void* v1; uint32_t* valid1; int t0; };
struct StateOuts { StateOut o[kMaxAggs]; };
__global__ void __launch_bounds__(256) agg_convert_state_kernel(AggSet aggs, StateOuts outs, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (n + 31) / 32;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t row = wi * 32 + lane;
    for (int i = 0; i < aggs.n; ++i) {
      const AggDev& a = aggs.a[i];
      const StateOut& o = outs.o[i];
      bool pass = row < n;
      if (pass && a.filt) pass = !(a.filt_valid && !bit_get(a.filt_valid, a.filt_voff + row)) && bit_get(a.filt, a.filt_off + row);
      bool ok = pass && (a.func == DFGPU_AGG_COUNT_STAR || !(a.in0_valid && !bit_get(a.in0_valid, a.in0_voff + row)));
      if (row < n) {
        switch (a.func) {
          case DFGPU_AGG_COUNT: case DFGPU_AGG_COUNT_STAR: ((int64_t*)o.v0)[row] = ok ? 1 : 0; break;
          case DFGPU_AGG_SUM:
            if (a.cls == 3) {
              const unsigned long long* p = (const unsigned long long*)a.in0 + 2 * row;
              ((unsigned long long*)o.v0)[2 * row] = ok ? p[0] : 0ull; ((unsigned long long*)o.v0)[2 * row + 1] = ok ? p[1] : 0ull;
            } else if (a.cls == 2) ((double*)o.v0)[row] = ok ? load_as_f64(a.in0, a.in0_type, row) : 0.0;
            else ((uint64_t*)o.v0)[row] = !ok ? 0ull : (a.in0_type == DFGPU_UINT64 ? ((const uint64_t*)a.in0)[row] : (uint64_t)load_as_i64(a.in0, a.in0_type, row));
            break;
          case DFGPU_AGG_MIN: case DFGPU_AGG_MAX: {
            if (type_width(o.t0) == 16) {   // Decimal128
              const unsigned long long* p = (const unsigned long long*)a.in0 + 2 * row;
              ((unsigned long long*)o.v0)[2 * row] = ok ? p[0] : 0ull; ((unsigned long long*)o.v0)[2 * row + 1] = ok ? p[1] : 0ull;
              break;
            }
            uint64_t v = 0;
            if (ok) {
              if (a.in0_type == DFGPU_FLOAT64) { double d = ((const double*)a.in0)[row]; memcpy(&v, &d, 8); }
              else if (a.in0_type == DFGPU_FLOAT32) { float f = ((const float*)a.in0)[row]; uint32_t b; memcpy(&b, &f, 4); v = b; }
              else if (a.in0_type == DFGPU_UINT64) v = ((const uint64_t*)a.in0)[row];
              else v = (uint64_t)load_as_i64(a.in0, a.in0_type, row);
            }
            switch (type_width(o.t0)) {
              case 1: ((uint8_t*)o.v0)[row] = (uint8_t)v; break;
              case 2: ((uint16_t*)o.v0)[row] = (uint16_t)v; break;
              case 4: ((uint32_t*)o.v0)[row] = (uint32_t)v; break;
              default: ((uint64_t*)o.v0)[row] = v; break;
            }
            break;
          }
          case DFGPU_AGG_AVG:
            ((uint64_t*)o.v0)[row] = ok ? 1ull : 0ull;
            ((double*)o.v1)[row] = ok ? load_as_f64(a.in0, a.in0_type, row) : 0.0;
            break;
        }
      }
      const uint32_t b = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) {
        if (o.valid0) o.valid0[wi] = b;
        if (o.valid1) o.valid1[wi] = b;
      }
    }
  }
}

__global__ void __launch_bounds__(256) salt_kernel(uint16_t* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (uint16_t)(i & 1023);
}
__global__ void fill_u64_kernel(unsigned long long* p, uint64_t n, unsigned long long v) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill_pair_kernel(ulonglong2* p, uint64_t n, ulonglong2 v) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}

}  // namespace dfgpu

// ==========================================================================================
// operator state
// ==========================================================================================
using namespace dfgpu;

struct AggState {
  int func, cls;
  int arg_col, filter_col;
  int in_type;          // raw input type (raw modes) or state value type
  int out_type;         // final value type
  int first_state_col;  // state modes: index of this aggregate's first state column in the input
  DevBuf acc0, acc1, seen;
  bool track_seen = false;
  unsigned long long init0 = 0, init1 = 0;   // init1: high word of a {lo, hi} pair accumulator
  // Decimal128 MIN / MAX / AVG keep one 16-byte {lo, hi} pair per slot in acc0 (atom.cas.b128 swaps both words at once)
  bool pair_acc() const { return cls == 3 && func != DFGPU_AGG_SUM; }
};

struct dfgpu_agg {
  dfgpu_ctx* ctx = nullptr;
  std::vector<int> input_types, group_cols;
  std::vector<AggState> aggs;
  int mode = DFGPU_AGG_SINGLE;
  bool state_input = false, state_output = false;
  int64_t batch_size = 8192;
  int kw = 1;
  int key_bits = 0;
  bool finished = false, emitted = false, hinted = false, bucketed = false;
  // key packing
  std::vector<int> g_shift, g_width_bits, g_null_bit;
  bool single_null_slot = false;
  // wide keys (> 128 bits together): hash tag + stored key tuples (GroupCols::wide)
  bool wide = false;
  std::vector<DevBuf> kstore;   // 2 per group column (second word only for 16-byte types)
  DevBuf knull;
  // table
  DevBuf tags, counters /* [ngroups, overflow_count] */, special_used;
  uint64_t cap = 0;
  // paired accumulators of the two-aggregate fast path (agg_update_pair_kernel): additive deltas, folded into aggs[0/1].acc0 before those are read
  DevBuf pairs;
  uint64_t pairs_cap = 0;
  bool pairs_dirty = false;
  int fast_r4 = 0;       // DFGPU_AGG_R4 at create (A/B switch): the two-aggregate fast kernel with 4 instead of 2 rows in flight per thread
  int paired_mode = 0;   // DFGPU_AGG_PAIRED at create: 0 = one RED per aggregate and row; agg_update_pair_kernel: 1 = 2 rows in flight per thread, 2 = 4 rows, 3 / 4 = 2 / 3 rows + whole-sector bucket load (4 is the default)
  std::deque<BatchPtr> outq;
  int64_t m_input_rows = 0, m_output_rows = 0, m_rehashes = 0, m_num_groups = 0, m_input_batches = 0;
  // skip-partial-aggregation probe (aggregates/skip_partial.rs:69-110; config.rs skip_partial_aggregation_probe_*)
  int64_t probe_rows_threshold = 100000; double probe_ratio_threshold = 0.8;
  int64_t probe_rows = 0, m_skipped_rows = 0;
  bool skipping = false;
  // no GROUP BY (AggregateStream, aggregates/aggregate_stream.rs): a composite of two grouped handles, see scalar_* below
  bool scalar = false;
  dfgpu_agg* inner1 = nullptr;   // rows -> 1024 partial states (hidden key = row & 1023: a single accumulator would serialise every atomic)
  dfgpu_agg* inner2 = nullptr;   // <= 1024 states -> the one output row
  std::vector<int> scalar_state_types;
};

namespace dfgpu {

static TableDev table_dev(dfgpu_agg* a, DevBuf& tags, uint64_t cap, DevBuf& counters, DevBuf& special) {
  TableDev t;
  t.tags = tags.ptr;
  t.cap = cap;
  t.ngroups = counters.as<unsigned long long>();
  t.group_limit = cap / 8 * 5;  // claims stop at load factor 0.625; the host grows the table beyond 0.5
  t.special_used = special.as<uint32_t>();
  t.bucketed = a->bucketed ? 1 : 0;
  return t;
}

static void fill_u64(dfgpu_ctx* ctx, void* p, uint64_t n, unsigned long long v) {
  if (n == 0) return;
  if (v == 0) { DF_CUDA(cudaMemsetAsync(p, 0, n * 8, ctx->stream)); return; }
  if (v == ~0ull) { DF_CUDA(cudaMemsetAsync(p, 0xFF, n * 8, ctx->stream)); return; }
  fill_u64_kernel<<<grid_for((int64_t)n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>((unsigned long long*)p, n, v);
  DF_LAUNCH_CHECK(ctx);
}

static void alloc_table(dfgpu_agg* a, uint64_t cap, DevBuf* tags, std::vector<DevBuf>* acc0, std::vector<DevBuf>* acc1, std::vector<DevBuf>* seen,
                        std::vector<DevBuf>* kstore = nullptr, DevBuf* knull = nullptr) {
  dfgpu_ctx* ctx = a->ctx;
  tags->alloc(ctx, (size_t)(cap + 2) * 8 * a->kw);
  tags->fill(0xFF);
  if (a->wide && kstore && knull) {
    kstore->resize(a->group_cols.size() * 2);
    for (size_t c = 0; c < a->group_cols.size(); ++c) {
      (*kstore)[2 * c].alloc(ctx, (size_t)(cap + 2) * 8);
      if (type_width(a->input_types[a->group_cols[c]]) == 16) (*kstore)[2 * c + 1].alloc(ctx, (size_t)(cap + 2) * 8);
    }
    knull->alloc(ctx, (size_t)(cap + 2));
    knull->zero();
  }
  acc0->resize(a->aggs.size()); acc1->resize(a->aggs.size()); seen->resize(a->aggs.size());
  for (size_t i = 0; i < a->aggs.size(); ++i) {
    const AggState& st = a->aggs[i];
    if (st.pair_acc()) {
      (*acc0)[i].alloc(ctx, (size_t)(cap + 2) * 16);
      fill_pair_kernel<<<grid_for((int64_t)cap + 2, 256, kNumSMs * 8), 256, 0, ctx->stream>>>((*acc0)[i].as<ulonglong2>(), cap + 2, make_ulonglong2(st.init0, st.init1));
      DF_LAUNCH_CHECK(ctx);
    } else {
      (*acc0)[i].alloc(ctx, (size_t)(cap + 2) * 8);
      fill_u64(ctx, (*acc0)[i].ptr, cap + 2, st.init0);
    }
    if (st.func == DFGPU_AGG_AVG || (st.cls == 3 && st.func == DFGPU_AGG_SUM)) { (*acc1)[i].alloc(ctx, (size_t)(cap + 2) * 8); (*acc1)[i].zero(); }   // AVG: count; Decimal128 SUM: high word
    if (a->aggs[i].track_seen) { (*seen)[i].alloc(ctx, (size_t)(cap + 2)); (*seen)[i].zero(); }
  }
}

// add the paired fast path's deltas into the per-aggregate accumulator arrays (every reader of those arrays calls this first)
static void fold_pairs(dfgpu_agg* a) {
  if (!a->pairs_dirty) return;
  dfgpu_ctx* ctx = a->ctx;
  const uint64_t total = a->pairs_cap + 2;
  agg_fold_pairs_kernel<<<grid_for((int64_t)total, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(a->pairs.as<ulonglong2>(), a->aggs[0].acc0.as<unsigned long long>(),
                                                                                          a->aggs[1].acc0.as<unsigned long long>(), total);
  DF_LAUNCH_CHECK(ctx);
  a->pairs_dirty = false;
}

static void grow_table(dfgpu_agg* a, uint64_t new_cap) {
  dfgpu_ctx* ctx = a->ctx;
  fold_pairs(a);
  DevBuf ntags, ncounters(ctx, 16), nspecial(ctx, 8);
  std::vector<DevBuf> nacc0, nacc1, nseen, nkstore;
  DevBuf nknull;
  alloc_table(a, new_cap, &ntags, &nacc0, &nacc1, &nseen, &nkstore, &nknull);
  ncounters.zero();
  nspecial.zero();
  TableDev old_t = table_dev(a, a->tags, a->cap, a->counters, a->special_used);
  TableDev new_t = table_dev(a, ntags, new_cap, ncounters, nspecial);
  new_t.group_limit = new_cap;  // the rehash itself may always claim
  AccArrays arr;
  arr.n = 0;
  for (size_t i = 0; i < a->aggs.size(); ++i) {
    arr.ptr[arr.n] = a->aggs[i].acc0.ptr; arr.new_ptr[arr.n] = nacc0[i].ptr; arr.elem[arr.n++] = a->aggs[i].pair_acc() ? 16 : 8;
    if (a->aggs[i].acc1.ptr) { arr.ptr[arr.n] = a->aggs[i].acc1.ptr; arr.new_ptr[arr.n] = nacc1[i].ptr; arr.elem[arr.n++] = 8; }
    if (a->aggs[i].seen.ptr) { arr.ptr[arr.n] = a->aggs[i].seen.ptr; arr.new_ptr[arr.n] = nseen[i].ptr; arr.elem[arr.n++] = 1; }
  }
  if (a->wide) {
    for (size_t k = 0; k < a->kstore.size(); ++k)
      if (a->kstore[k].ptr) { arr.ptr[arr.n] = a->kstore[k].ptr; arr.new_ptr[arr.n] = nkstore[k].ptr; arr.elem[arr.n++] = 8; }
    arr.ptr[arr.n] = a->knull.ptr; arr.new_ptr[arr.n] = nknull.ptr; arr.elem[arr.n++] = 1;
  }
  int grid = grid_for((int64_t)a->cap + 2, 256, kNumSMs * 8);
  if (a->kw == 1) agg_rehash_kernel<1><<<grid, 256, 0, ctx->stream>>>(old_t, new_t, arr);
  else agg_rehash_kernel<2><<<grid, 256, 0, ctx->stream>>>(old_t, new_t, arr);
  DF_LAUNCH_CHECK(ctx);
  DF_CUDA(cudaMemcpyAsync(ncounters.ptr, a->counters.ptr, 8, cudaMemcpyDeviceToDevice, ctx->stream));  // ngroups carries over
  a->tags = std::move(ntags);
  a->counters = std::move(ncounters);
  a->special_used = std::move(nspecial);
  for (size_t i = 0; i < a->aggs.size(); ++i) {
    a->aggs[i].acc0 = std::move(nacc0[i]);
    a->aggs[i].acc1 = std::move(nacc1[i]);
    a->aggs[i].seen = std::move(nseen[i]);
  }
  if (a->wide) { a->kstore = std::move(nkstore); a->knull = std::move(nknull); }
  a->cap = new_cap;
  a->m_rehashes++;
}

static void ensure_seen(dfgpu_agg* a, AggState& s) {
  if (s.track_seen) return;
  if (!(s.func == DFGPU_AGG_SUM || s.func == DFGPU_AGG_MIN || s.func == DFGPU_AGG_MAX)) return;
  dfgpu_ctx* ctx = a->ctx;
  s.track_seen = true;
  s.seen.alloc(ctx, (size_t)(a->cap + 2));
  TableDev t = table_dev(a, a->tags, a->cap, a->counters, a->special_used);
  int grid = grid_for((int64_t)a->cap + 2, 256, kNumSMs * 8);
  if (a->kw == 1) agg_init_seen_kernel<1><<<grid, 256, 0, ctx->stream>>>(t, s.seen.as<uint8_t>());
  else agg_init_seen_kernel<2><<<grid, 256, 0, ctx->stream>>>(t, s.seen.as<uint8_t>());
  DF_LAUNCH_CHECK(ctx);
}

static void agg_finish(dfgpu_agg* a);
static void agg_emit_table(dfgpu_agg* a);

// SkippingAggregation: the batch leaves as one state row per input row (convert_batch_to_state, partial_table.rs:199-238)
static void agg_convert_batch_to_state(dfgpu_agg* a, const std::vector<DCol>& cols, const AggSet& set, int64_t n) {
  dfgpu_ctx* ctx = a->ctx;
  BatchPtr out(new dfgpu_batch());
  out->ctx = ctx; out->rows = n; out->host = false;
  for (int gc : a->group_cols) out->cols.push_back(copy_column_device(ctx, cols[gc]));
  StateOuts so;
  memset(&so, 0, sizeof(so));
  for (size_t i = 0; i < a->aggs.size(); ++i) {
    const AggState& st = a->aggs[i];
    switch (st.func) {
      case DFGPU_AGG_COUNT: case DFGPU_AGG_COUNT_STAR: {
        DCol c = alloc_col(ctx, DFGPU_INT64, n, false);
        so.o[i].v0 = c.own_values->ptr; so.o[i].t0 = DFGPU_INT64;
        out->cols.push_back(std::move(c));
        break;
      }
      case DFGPU_AGG_AVG: {
        DCol c = alloc_col(ctx, DFGPU_UINT64, n, false), sm = alloc_col(ctx, DFGPU_FLOAT64, n, true);
        so.o[i].v0 = c.own_values->ptr; so.o[i].v1 = sm.own_values->ptr; so.o[i].valid1 = sm.own_validity->as<uint32_t>(); so.o[i].t0 = DFGPU_UINT64;
        sm.null_count = -1;
        out->cols.push_back(std::move(c)); out->cols.push_back(std::move(sm));
        break;
      }
      default: {   // SUM / MIN / MAX
        const int t = st.func == DFGPU_AGG_SUM ? (st.cls == 3 ? st.out_type : (st.cls == 2 ? DFGPU_FLOAT64 : (st.cls == 1 ? DFGPU_UINT64 : DFGPU_INT64))) : st.out_type;
        DCol c = alloc_col(ctx, t, n, true);
        so.o[i].v0 = c.own_values->ptr; so.o[i].valid0 = c.own_validity->as<uint32_t>(); so.o[i].t0 = t;
        c.null_count = -1;
        out->cols.push_back(std::move(c));
      }
    }
  }
  agg_convert_state_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(set, so, n);
  DF_LAUNCH_CHECK(ctx);
  DF_CUDA(cudaStreamSynchronize(ctx->stream));   // the caller's input columns are consumed before the push returns
  a->m_output_rows += n;
  a->m_skipped_rows += n;
  a->outq.push_back(std::move(out));
}

static void agg_push(dfgpu_agg* a, const std::vector<DCol>& cols) {
  DF_CHECK(!a->finished, DFGPU_ERR_STATE, "push after finish");
  if (a->scalar) {
    DF_CHECK(cols.size() == a->input_types.size(), DFGPU_ERR_INVALID, "aggregate input column count mismatch");
    dfgpu_ctx* ctx = a->ctx;
    set_device(ctx);
    const int64_t n = cols.empty() ? 0 : cols[0].length;
    a->m_input_rows += n; a->m_input_batches++;
    if (n == 0) return;
    DCol salt = alloc_col(ctx, DFGPU_UINT16, n, false);
    salt_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>((uint16_t*)salt.own_values->ptr, n);
    DF_LAUNCH_CHECK(ctx);
    std::vector<DCol> v{salt};
    v.insert(v.end(), cols.begin(), cols.end());
    agg_push(a->inner1, v);
    return;
  }
  DF_CHECK(cols.size() == a->input_types.size(), DFGPU_ERR_INVALID, "aggregate input column count mismatch");
  dfgpu_ctx* ctx = a->ctx;
  set_device(ctx);
  const int64_t n = cols.empty() ? 0 : cols[0].length;
  for (size_t c = 0; c < cols.size(); ++c) {
    DF_CHECK(cols[c].type == a->input_types[c], DFGPU_ERR_INVALID, "aggregate input column type mismatch");
    DF_CHECK(cols[c].length == n, DFGPU_ERR_INVALID, "aggregate input ragged columns");
  }
  a->m_input_rows += n;
  a->m_input_batches++;
  if (n == 0) return;
  // group key columns
  GroupCols g;
  memset(&g, 0, sizeof(g));
  g.n = (int)a->group_cols.size();
  g.kw = a->kw;
  g.single_null_slot = a->single_null_slot ? 1 : 0;
  for (int c = 0; c < g.n; ++c) {
    const DCol& col = cols[a->group_cols[c]];
    g.ptr[c] = col.values; g.valid[c] = col.validity; g.voff[c] = col.offset;
    g.width[c] = type_width(col.type); g.boff[c] = col.offset;
    g.shift[c] = a->g_shift[c]; g.null_bit[c] = a->g_null_bit[c];
    g.is_float[c] = type_is_float(col.type) ? 1 : 0;
    DF_CHECK(a->wide || !(col.validity && a->g_null_bit[c] < 0 && !a->single_null_slot), DFGPU_ERR_INVALID, "group column declared non-nullable has a validity bitmap");
  }
  g.wide = a->wide ? 1 : 0;
  // aggregates
  AggSet set;
  memset(&set, 0, sizeof(set));
  set.n = (int)a->aggs.size();
  for (int i = 0; i < set.n; ++i) {
    AggState& s = a->aggs[i];
    AggDev& d = set.a[i];
    d.func = s.func; d.cls = s.cls; d.merge = a->state_input ? 1 : 0;
    const DCol* in0 = nullptr; const DCol* in1 = nullptr; const DCol* filt = nullptr;
    if (a->state_input) {
      in0 = &cols[s.first_state_col];
      if (s.func == DFGPU_AGG_AVG) in1 = &cols[s.first_state_col + 1];
    } else {
      if (s.func != DFGPU_AGG_COUNT_STAR) in0 = &cols[s.arg_col];
      if (s.filter_col >= 0) filt = &cols[s.filter_col];
    }
    if (in0) { d.in0 = in0->values; d.in0_type = in0->type; d.in0_valid = in0->validity; d.in0_voff = in0->offset; }
    if (in1) { d.in1 = in1->values; d.in1_type = in1->type; d.in1_valid = in1->validity; d.in1_voff = in1->offset; }
    if (filt) { d.filt = (const uint8_t*)filt->values; d.filt_off = filt->offset; d.filt_valid = filt->validity; d.filt_voff = filt->offset; }
    // NullState: switch to explicit seen tracking once nulls or a filter show up (accumulate.rs:164-188)
    if ((in0 && in0->validity) || filt) ensure_seen(a, s);
  }
  if (a->skipping) { agg_convert_batch_to_state(a, cols, set, n); return; }
  bool pair = false;
  for (const AggState& s : a->aggs) pair |= s.pair_acc();
  // fast-path eligibility (decided per batch: it depends on the validity of THIS batch's columns)
  static const int fast_enabled = getenv("DFGPU_AGG_FAST") ? atoi(getenv("DFGPU_AGG_FAST")) : 1;
  bool fast = fast_enabled && a->kw == 1 && g.n == 1 && g.width[0] == 8 && !g.valid[0] && !g.is_float[0] && set.n >= 1 && set.n <= kMaxFastAggs;
  FastAggs fa;
  memset(&fa, 0, sizeof(fa));
  for (int i = 0; i < set.n && fast; ++i) {
    const AggDev& d = set.a[i];
    const bool sum_like = (d.func == DFGPU_AGG_SUM && d.cls != 2 && type_width(d.in0_type) == 8) || ((d.func == DFGPU_AGG_COUNT || d.func == DFGPU_AGG_COUNT_STAR) && d.merge);
    const bool count_like = (d.func == DFGPU_AGG_COUNT || d.func == DFGPU_AGG_COUNT_STAR) && !d.merge;
    if (d.filt || d.in0_valid || a->aggs[i].track_seen || !(sum_like || count_like)) { fast = false; break; }
    fa.col[i] = sum_like ? (const unsigned long long*)d.in0 : nullptr;
  }
  fa.n = set.n;
  const int paired_env = a->paired_mode;
  const int fast_r4 = a->fast_r4;
  const bool use_pair = fast && paired_env > 0 && fa.n == 2 && a->bucketed;
  if (!use_pair) fold_pairs(a);   // the kernels below update the per-aggregate arrays directly
  auto refresh_ptrs = [&]() {
    for (int i = 0; i < set.n; ++i) {
      set.a[i].acc0 = a->aggs[i].acc0.as<unsigned long long>();
      set.a[i].acc1 = a->aggs[i].acc1.as<unsigned long long>();
      set.a[i].seen = a->aggs[i].seen.as<uint8_t>();
      if (i < kMaxFastAggs) fa.acc[i] = a->aggs[i].acc0.as<unsigned long long>();
    }
    if (a->wide) {
      for (size_t k = 0; k < a->kstore.size(); ++k) g.kstore[k] = a->kstore[k].as<unsigned long long>();
      g.knull = a->knull.as<uint8_t>();
    }
  };
  // chunked processing with ramp-up so an undersized table is discovered cheaply
  int64_t done = 0;
  // without a capacity hint the table starts small: ramp the chunk size so an undersized table is discovered
  // after a few million rows; with a hint the table is pre-sized and whole batches go in one launch
  int64_t chunk = a->hinted ? (1ll << 28) : std::max<int64_t>((int64_t)a->cap / 2, 1 << 20);
  const int64_t kMaxChunk = 1ll << 28;
  DevBuf overflow;
  while (done < n) {
    int64_t m = std::min<int64_t>(std::min(chunk, kMaxChunk), n - done);
    if (overflow.bytes < (size_t)m * 4) overflow.alloc(ctx, (size_t)m * 4);
    const uint32_t* list = nullptr;
    int64_t work = m;
    DevBuf replay;
    while (true) {
      refresh_ptrs();
      TableDev t = table_dev(a, a->tags, a->cap, a->counters, a->special_used);
      DF_CUDA(cudaMemsetAsync(a->counters.as<unsigned long long>() + 1, 0, 8, ctx->stream));
      int grid = grid_for((work + 3) / 4, 256, kNumSMs * 8);
      {
        KernelTimer kt(ctx, "agg_update");
        if (fast) {
          const unsigned long long* kp = (const unsigned long long*)g.ptr[0];
          uint32_t* ov = overflow.as<uint32_t>();
          unsigned long long* oc = a->counters.as<unsigned long long>() + 1;
          if (use_pair && a->cap + 2 < (1ull << 32)) {
            if (a->pairs_cap != a->cap || !a->pairs.ptr) {   // first use, or the table grew (grow_table folded the old deltas)
              a->pairs.alloc(ctx, (size_t)(a->cap + 2) * 16);
              a->pairs.zero();
              a->pairs_cap = a->cap;
            }
            a->pairs_dirty = true;
            const int grid2 = grid_for((work + 1) / 2, 256, kNumSMs * 8);
            ulonglong2* pr = a->pairs.as<ulonglong2>();
            if (paired_env == 2) agg_update_pair_kernel<4, false><<<grid, 256, 0, ctx->stream>>>(kp, fa.col[0], fa.col[1], pr, t, done, work, list, ov, oc);
            else if (paired_env == 3) agg_update_pair_kernel<2, true><<<grid2, 256, 0, ctx->stream>>>(kp, fa.col[0], fa.col[1], pr, t, done, work, list, ov, oc);
            else if (paired_env == 4) agg_update_pair_kernel<3, true><<<grid_for((work + 2) / 3, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(kp, fa.col[0], fa.col[1], pr, t, done, work, list, ov, oc);
            else agg_update_pair_kernel<2, false><<<grid2, 256, 0, ctx->stream>>>(kp, fa.col[0], fa.col[1], pr, t, done, work, list, ov, oc);
          } else if (a->bucketed) {
            if (use_pair) fold_pairs(a);
            const int grid2 = grid_for((work + 1) / 2, 256, kNumSMs * 8);
            switch (fa.n) {
              case 1: agg_update_fast_kernel<2, 1, 1><<<grid2, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
              case 2:
                if (fast_r4) agg_update_fast_kernel<4, 2, 1><<<grid, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc);   // A/B switch: 4 rows in flight per thread
                else agg_update_fast_kernel<2, 2, 1><<<grid2, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc);
                break;
              case 3: agg_update_fast_kernel<2, 3, 1><<<grid2, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
              default: agg_update_fast_kernel<2, 4, 1><<<grid2, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
            }
          } else {
            switch (fa.n) {
              case 1: agg_update_fast_kernel<4, 1, 0><<<grid, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
              case 2: agg_update_fast_kernel<4, 2, 0><<<grid, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
              case 3: agg_update_fast_kernel<4, 3, 0><<<grid, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
              default: agg_update_fast_kernel<4, 4, 0><<<grid, 256, 0, ctx->stream>>>(kp, fa, t, done, work, list, ov, oc); break;
            }
          }
        } else {
          uint32_t* ov = overflow.as<uint32_t>();
          unsigned long long* oc = a->counters.as<unsigned long long>() + 1;
          if (a->kw == 1) {
            if (pair) agg_update_kernel<1, 4, true><<<grid, 256, 0, ctx->stream>>>(g, set, t, done, work, list, ov, oc);
            else agg_update_kernel<1, 4, false><<<grid, 256, 0, ctx->stream>>>(g, set, t, done, work, list, ov, oc);
          } else {
            if (pair) agg_update_kernel<2, 4, true><<<grid, 256, 0, ctx->stream>>>(g, set, t, done, work, list, ov, oc);
            else agg_update_kernel<2, 4, false><<<grid, 256, 0, ctx->stream>>>(g, set, t, done, work, list, ov, oc);
          }
        }
        DF_LAUNCH_CHECK(ctx);
      }
      unsigned long long hc[2];
      DF_CUDA(cudaMemcpyAsync(hc, a->counters.ptr, 16, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
      a->m_num_groups = (int64_t)hc[0];
      if (hc[1] == 0) {
        // grow once the load factor passes 1/2 (probe length and the claim budget of the next chunk)
        if (hc[0] * 2 > a->cap) grow_table(a, a->cap * 4);
        break;
      }
      // deferred rows: grow, then replay just those rows
      replay = std::move(overflow);
      overflow.alloc(ctx, (size_t)hc[1] * 4);
      list = replay.as<uint32_t>();
      work = (int64_t)hc[1];
      uint64_t want = std::max<uint64_t>(a->cap * 4, (hc[0] + hc[1]) * 2);
      grow_table(a, (want + 3) & ~3ull);
    }
    if (a->wide) {
      // vectorized_equal_to: every row of the chunk against its group's stored tuple (all claims of the chunk are complete by now)
      refresh_ptrs();
      TableDev t = table_dev(a, a->tags, a->cap, a->counters, a->special_used);
      DevBuf mism(ctx, 4);
      mism.zero();
      agg_verify_wide_kernel<<<grid_for(m, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(g, t, done, m, mism.as<int>());
      DF_LAUNCH_CHECK(ctx);
      const int bad = read_scalar<int>(ctx, mism.as<int>());
      DF_CHECK(!bad, DFGPU_ERR_UNSUPPORTED, "aggregate: two distinct wide group keys share a 64-bit hash (expected once in ~2^64 / groups^2 runs): keep the CPU operator for this input");
    }
    done += m;
    chunk = std::min<int64_t>(chunk * 4, kMaxChunk);
  }
  // SkipAggregationProbe::update_state (skip_partial.rs:69-110), Partial mode only: once probe_rows_threshold rows are in, a
  // groups / rows ratio above the threshold means aggregating here does not pay — emit the groups and pass later batches through
  if (a->mode == DFGPU_AGG_PARTIAL && a->probe_rows_threshold > 0 && !a->group_cols.empty()) {
    a->probe_rows += n;
    if (a->probe_rows >= a->probe_rows_threshold && (double)a->m_num_groups / (double)a->probe_rows > a->probe_ratio_threshold) {
      a->skipping = true;
      agg_emit_table(a);
      a->emitted = true;
    }
  }
}

// one all-NULL / zero state row: what fresh accumulators report (SUM / MIN / MAX / AVG sum: NULL, counts: 0)
static std::vector<DCol> scalar_empty_state(dfgpu_agg* a) {
  dfgpu_ctx* ctx = a->ctx;
  std::vector<DCol> v;
  DCol key = alloc_col(ctx, DFGPU_UINT16, 1, false);
  key.own_values->zero();
  v.push_back(key);
  size_t k = 0;
  for (auto& st : a->inner1->aggs) {
    const int n_state = st.func == DFGPU_AGG_AVG ? 2 : 1;
    for (int j = 0; j < n_state; ++j, ++k) {
      const int t = a->scalar_state_types[k];
      const bool is_count = st.func == DFGPU_AGG_COUNT || st.func == DFGPU_AGG_COUNT_STAR || (st.func == DFGPU_AGG_AVG && j == 0);
      DCol c = alloc_col(ctx, t, 1, !is_count);
      c.own_values->zero();
      if (!is_count) { c.own_validity->zero(); c.null_count = 1; }
      v.push_back(c);
    }
  }
  return v;
}

static void agg_finish(dfgpu_agg* a) {
  DF_CHECK(!a->finished, DFGPU_ERR_STATE, "finish called twice");
  if (a->scalar) {
    a->finished = true;
    dfgpu_ctx* ctx = a->ctx;
    set_device(ctx);
    agg_finish(a->inner1);
    bool any = false;
    while (!a->inner1->outq.empty()) {
      BatchPtr b = std::move(a->inner1->outq.front());
      a->inner1->outq.pop_front();
      if (b->rows == 0) continue;
      any = true;
      std::vector<DCol> v = b->cols;
      DCol key = alloc_col(ctx, DFGPU_UINT16, b->rows, false);   // every partial state merges into ONE group
      key.own_values->zero();
      v[0] = key;
      agg_push(a->inner2, v);
    }
    if (!any) agg_push(a->inner2, scalar_empty_state(a));
    agg_finish(a->inner2);
    while (!a->inner2->outq.empty()) {
      BatchPtr b = std::move(a->inner2->outq.front());
      a->inner2->outq.pop_front();
      b->cols.erase(b->cols.begin());                            // drop the hidden key
      a->m_output_rows += b->rows;
      a->outq.push_back(std::move(b));
    }
    a->m_num_groups = 1;
    return;
  }
  a->finished = true;
  set_device(a->ctx);
  if (!a->emitted) agg_emit_table(a);   // SkippingAggregation already emitted the groups when it switched (hash_stream.rs SkippingAggregation)
}

static void agg_emit_table(dfgpu_agg* a) {
  dfgpu_ctx* ctx = a->ctx;
  fold_pairs(a);
  // emit = group_values.emit(EmitTo::All) ++ acc.state()/evaluate() (common.rs:247-297)
  TableDev t = table_dev(a, a->tags, a->cap, a->counters, a->special_used);
  const uint64_t total = a->cap + 2;
  DevBuf occ(ctx, (size_t)((total + 31) / 32) * 4);
  int grid = grid_for((int64_t)total, 256, kNumSMs * 8);
  if (a->kw == 1) agg_occupancy_kernel<1><<<grid, 256, 0, ctx->stream>>>(t, occ.as<uint32_t>());
  else agg_occupancy_kernel<2><<<grid, 256, 0, ctx->stream>>>(t, occ.as<uint32_t>());
  DF_LAUNCH_CHECK(ctx);
  DevBuf idx;
  int64_t ng = compact_flag_indices(ctx, occ.as<uint32_t>(), (int64_t)total, 1, &idx);
  a->m_num_groups = ng;
  // a global aggregate (no GROUP BY) over empty input still yields one row in Final/Single modes; grouped: zero rows.
  BatchPtr out(new dfgpu_batch());
  out->ctx = ctx; out->rows = ng; out->host = false;
  DevBuf avg_err;   // Decimal128 AVG overflow flag
  auto run_emit =[&](EmitDesc& d, int out_type, bool with_valid) -> DCol {
    DCol col = alloc_col(ctx, out_type, ng, with_valid);
    if (ng > 0) {
      d.out_type = out_type; d.kw = a->kw; d.tags = a->tags.ptr; d.cap = a->cap;
      agg_emit_kernel<<<grid_for(ng, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(
          d, idx.as<uint32_t>(), ng, out_type == DFGPU_BOOL ? nullptr : col.own_values->ptr,
          with_valid ? col.own_validity->as<uint32_t>() : nullptr, out_type == DFGPU_BOOL ? col.own_values->as<uint32_t>() : nullptr);
      DF_LAUNCH_CHECK(ctx);
    }
    col.null_count = with_valid ? -1 : 0;
    return col;
  };
  for (size_t c = 0; c < a->group_cols.size(); ++c) {
    EmitDesc d;
    memset(&d, 0, sizeof(d));
    if (a->wide) {   // the stored tuple: column c's words + bit c of the NULL mask
      d.kind = EK_WIDEKEY; d.acc0 = a->kstore[2 * c].as<unsigned long long>(); d.acc1 = a->kstore[2 * c + 1].as<unsigned long long>();
      d.seen = a->knull.as<uint8_t>(); d.null_bit = (int)c;
      out->cols.push_back(run_emit(d, a->input_types[a->group_cols[c]], true));
      continue;
    }
    d.kind = EK_KEY; d.shift = a->g_shift[c]; d.width_bits = a->g_width_bits[c]; d.null_bit = a->g_null_bit[c];
    d.single_null_slot = a->single_null_slot;
    bool nullable = a->g_null_bit[c] >= 0 || a->single_null_slot;
    out->cols.push_back(run_emit(d, a->input_types[a->group_cols[c]], nullable));
  }
  for (auto& s : a->aggs) {
    EmitDesc d;
    memset(&d, 0, sizeof(d));
    d.acc0 = s.acc0.as<unsigned long long>(); d.acc1 = s.acc1.as<unsigned long long>(); d.seen = s.seen.as<uint8_t>(); d.cls = s.cls;
    d.null_bit = -1;
    switch (s.func) {
      case DFGPU_AGG_SUM: {
        d.kind = s.cls == 3 ? EK_DEC128 : EK_COPY64;
        int t2 = s.cls == 3 ? s.out_type : (s.cls == 2 ? DFGPU_FLOAT64 : (s.cls == 1 ? DFGPU_UINT64 : DFGPU_INT64));  // Sum::return_type, sum.rs:232-261
        out->cols.push_back(run_emit(d, t2, s.track_seen));
        break;
      }
      case DFGPU_AGG_COUNT: case DFGPU_AGG_COUNT_STAR:
        d.kind = EK_COPY64; d.seen = nullptr;
        out->cols.push_back(run_emit(d, DFGPU_INT64, false));  // COUNT is never NULL (count.rs:700-708)
        break;
      case DFGPU_AGG_MIN: case DFGPU_AGG_MAX:
        d.kind = s.pair_acc() ? EK_PAIR128 : EK_MINMAX;
        out->cols.push_back(run_emit(d, s.out_type, s.track_seen));
        break;
      case DFGPU_AGG_AVG:
        if (s.cls == 3 && a->state_output) {   // the no-GROUP-BY composite's internal state [count: UInt64, sum: the argument's type]
          EmitDesc dc = d; dc.kind = EK_COPY64; dc.acc0 = s.acc1.as<unsigned long long>(); dc.seen = nullptr;
          out->cols.push_back(run_emit(dc, DFGPU_UINT64, false));
          EmitDesc ds = d; ds.kind = EK_PAIR128; ds.seen = nullptr;
          out->cols.push_back(run_emit(ds, s.in_type, false));
        } else if (s.cls == 3) {
          if (!avg_err.ptr) { avg_err.alloc(ctx, 8); avg_err.zero(); }
          d.kind = EK_AVG_DEC; d.avg_mul = dec_scale(s.out_type) - dec_scale(s.in_type); d.avg_prec = dec_precision(s.out_type);
          d.err = avg_err.as<unsigned long long>();
          out->cols.push_back(run_emit(d, s.out_type, true));
        } else if (a->state_output) {
          EmitDesc dc = d; dc.kind = EK_COPY64; dc.acc0 = s.acc1.as<unsigned long long>(); dc.seen = nullptr;
          out->cols.push_back(run_emit(dc, DFGPU_UINT64, false));
          EmitDesc ds = d; ds.kind = EK_COPY64; ds.seen = nullptr;
          out->cols.push_back(run_emit(ds, DFGPU_FLOAT64, false));
        } else {
          d.kind = EK_AVG;
          out->cols.push_back(run_emit(d, DFGPU_FLOAT64, true));
        }
        break;
    }
  }
  if (avg_err.ptr && read_scalar<unsigned long long>(ctx, avg_err.as<unsigned long long>()))
    throw Error(DFGPU_ERR_ARITH, "Arithmetic Overflow in AvgAccumulator");
  a->m_output_rows += ng;
  if (ng > 0 || a->group_cols.empty()) a->outq.push_back(std::move(out));
}

// dec_avg_state: AVG over Decimal128 may take or emit the state [count: UInt64, sum: Decimal128(p, s)], where the sum is the i128
// add_wrapping sum labelled with the argument's type.  Only the no-GROUP-BY composite sets it, between its two inner handles: DataFusion
// pins no public Partial state for this AVG, so dfgpu_agg_create rejects it in the state modes.
static dfgpu_agg* agg_create(dfgpu_ctx* ctx, const int32_t* input_types, int32_t n_cols, const int32_t* group_cols, int32_t n_group,
                             const dfgpu_agg_desc* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size, int64_t capacity_hint, bool dec_avg_state) {
  DF_CHECK(n_group >= 0 && n_group <= kMaxGroupCols, DFGPU_ERR_UNSUPPORTED, "aggregate: at most 8 group columns");
  if (n_group == 0) {
    // ---- AggregateStream (no GROUP BY, aggregates/aggregate_stream.rs): exactly one output row, also for empty input ----
    DF_CHECK(n_aggs >= 1 && n_aggs <= kMaxAggs, DFGPU_ERR_INVALID, "aggregate without GROUP BY needs 1..8 aggregate expressions");
    const bool state_in = (mode == DFGPU_AGG_FINAL || mode == DFGPU_AGG_FINAL_PARTITIONED || mode == DFGPU_AGG_PARTIAL_REDUCE);
    const bool state_out = (mode == DFGPU_AGG_PARTIAL || mode == DFGPU_AGG_PARTIAL_REDUCE);
    std::unique_ptr<dfgpu_agg> a(new dfgpu_agg());
    a->ctx = ctx; a->scalar = true; a->mode = mode; a->state_input = state_in; a->state_output = state_out;
    a->input_types.assign(input_types, input_types + n_cols);
    std::vector<int32_t> t1{DFGPU_UINT16};
    t1.insert(t1.end(), input_types, input_types + n_cols);
    std::vector<dfgpu_agg_desc> d1(aggs, aggs + n_aggs);
    if (!state_in) for (auto& d : d1) { if (d.func != DFGPU_AGG_COUNT_STAR) d.arg_col += 1; if (d.filter_col >= 0) d.filter_col += 1; }
    const int32_t g0 = 0;
    const bool single = !state_in && !state_out;   // the inner state of a Decimal128 AVG never leaves the composite
    a->inner1 = agg_create(ctx, t1.data(), (int)t1.size(), &g0, 1, d1.data(), n_aggs, state_in ? DFGPU_AGG_PARTIAL_REDUCE : DFGPU_AGG_PARTIAL, batch_size, 1024, single);
    // state schema emitted by inner1: [salt, state columns...]
    std::vector<int32_t> t2{DFGPU_UINT16};
    for (auto& st : a->inner1->aggs) {
      switch (st.func) {
        case DFGPU_AGG_SUM: t2.push_back(st.cls == 3 ? st.out_type : (st.cls == 2 ? DFGPU_FLOAT64 : (st.cls == 1 ? DFGPU_UINT64 : DFGPU_INT64))); break;
        case DFGPU_AGG_COUNT: case DFGPU_AGG_COUNT_STAR: t2.push_back(DFGPU_INT64); break;
        case DFGPU_AGG_MIN: case DFGPU_AGG_MAX: t2.push_back(st.out_type); break;
        case DFGPU_AGG_AVG: t2.push_back(DFGPU_UINT64); t2.push_back(st.cls == 3 ? st.in_type : DFGPU_FLOAT64); break;
      }
    }
    a->scalar_state_types.assign(t2.begin() + 1, t2.end());
    std::vector<dfgpu_agg_desc> d2(aggs, aggs + n_aggs);
    for (auto& d : d2) { d.arg_col = -1; d.filter_col = -1; }
    try {
      a->inner2 = agg_create(ctx, t2.data(), (int)t2.size(), &g0, 1, d2.data(), n_aggs, state_out ? DFGPU_AGG_PARTIAL_REDUCE : DFGPU_AGG_FINAL, batch_size, 16, single);
    } catch (...) { dfgpu_agg_destroy(a->inner1); a->inner1 = nullptr; throw; }
    return a.release();
  }
  DF_CHECK(n_aggs >= 0 && n_aggs <= kMaxAggs, DFGPU_ERR_UNSUPPORTED, "aggregate: at most 8 aggregate expressions");
  set_device(ctx);
  std::unique_ptr<dfgpu_agg> a(new dfgpu_agg());
  a->ctx = ctx;
  a->input_types.assign(input_types, input_types + n_cols);
  a->group_cols.assign(group_cols, group_cols + n_group);
  a->mode = mode;
  a->batch_size = batch_size > 0 ? batch_size : 8192;
  a->state_input = (mode == DFGPU_AGG_FINAL || mode == DFGPU_AGG_FINAL_PARTITIONED || mode == DFGPU_AGG_PARTIAL_REDUCE);
  a->state_output = (mode == DFGPU_AGG_PARTIAL || mode == DFGPU_AGG_PARTIAL_REDUCE);
  // key packing: values first, then one null flag per (multi-column) group column.  All group
  // columns are treated as nullable: the schema-level nullability is not part of this ABI.
  int bits = 0;
  bool wide = false;
  for (int c = 0; c < n_group; ++c) {
    DF_CHECK(group_cols[c] >= 0 && group_cols[c] < n_cols, DFGPU_ERR_INVALID, "group column index out of range");
    int t = input_types[group_cols[c]];
    int w = type_width(t);
    DF_CHECK(w >= 0 && w <= 16, DFGPU_ERR_UNSUPPORTED, "aggregate: group column type not supported");
    if (w == 16 && n_group > 1) wide = true;   // a 16-byte Decimal128 key next to other group columns
    int wb = (t == DFGPU_BOOL) ? 1 : 8 * w;
    a->g_shift.push_back(bits);
    a->g_width_bits.push_back(wb);
    bits += wb;
  }
  a->single_null_slot = (n_group == 1);
  for (int c = 0; c < n_group; ++c) {
    if (a->single_null_slot) a->g_null_bit.push_back(-1);
    else { a->g_null_bit.push_back(bits); bits += 1; }
  }
  if (!a->single_null_slot && bits > 128) {
    // retry without null flags when the values alone fill 128 bits (e.g. TPC-H Q3: int64 + date32 + int32):
    // NULL group keys are then rejected at push time.
    bits -= n_group;
    for (int c = 0; c < n_group; ++c) a->g_null_bit[c] = -1;
  }
  if (bits > 128 || wide) {
    // keys beyond the exact 128-bit tag: hash tag + stored tuples + a verification pass per batch (GroupCols::wide)
    a->wide = true;
    a->single_null_slot = false;
    for (int c = 0; c < n_group; ++c) { a->g_shift[c] = 0; a->g_null_bit[c] = c; }   // NULL is part of the tuple: bit c of the slot's NULL mask
    bits = 64;
  }
  a->key_bits = bits;
  a->kw = bits <= 64 ? 1 : 2;
  int next_state_col = n_group;
  for (int i = 0; i < n_aggs; ++i) {
    AggState s;
    s.func = aggs[i].func; s.arg_col = aggs[i].arg_col; s.filter_col = aggs[i].filter_col;
    s.first_state_col = next_state_col;
    int vt;
    if (a->state_input) {
      DF_CHECK(next_state_col < n_cols, DFGPU_ERR_INVALID, "aggregate: state columns missing from input schema");
      vt = input_types[s.func == DFGPU_AGG_AVG ? next_state_col + 1 : next_state_col];
      next_state_col += (s.func == DFGPU_AGG_AVG) ? 2 : 1;
    } else {
      if (s.func == DFGPU_AGG_COUNT_STAR) vt = DFGPU_INT64;
      else {
        DF_CHECK(s.arg_col >= 0 && s.arg_col < n_cols, DFGPU_ERR_INVALID, "aggregate argument column out of range");
        vt = input_types[s.arg_col];
      }
      if (s.filter_col >= 0) DF_CHECK(s.filter_col < n_cols && input_types[s.filter_col] == DFGPU_BOOL, DFGPU_ERR_INVALID, "aggregate FILTER column must be Boolean");
    }
    s.in_type = vt;
    s.out_type = vt;
    s.cls = type_is_float(vt) ? 2 : (type_is_unsigned_int(vt) ? 1 : 0);
    switch (s.func) {
      case DFGPU_AGG_SUM:
        if (type_is_decimal(vt)) {
          // Sum::return_type (sum.rs:247-249): Decimal128(min(38, precision + 10), scale); the state column already carries that type
          DF_CHECK(dec_precision(vt) >= 1, DFGPU_ERR_UNSUPPORTED, "SUM: Decimal128 argument needs its precision and scale (DFGPU_DECIMAL128_TYPE)");
          s.cls = 3;
          s.out_type = a->state_input ? vt : dec_type(std::min(38, dec_precision(vt) + 10), dec_scale(vt));
        } else DF_CHECK(type_is_int(vt) || type_is_float(vt), DFGPU_ERR_UNSUPPORTED, "SUM: numeric argument required");
        s.init0 = 0; break;
      case DFGPU_AGG_COUNT: case DFGPU_AGG_COUNT_STAR: s.init0 = 0; break;
      case DFGPU_AGG_AVG:
        if (type_is_decimal(vt)) {
          // Avg::return_type (average.rs): Decimal128(min(38, p + 4), min(38, s + 4)), the value by DecimalAverager::avg at emission
          DF_CHECK(dec_precision(vt) >= 1, DFGPU_ERR_UNSUPPORTED, "AVG: Decimal128 argument needs its precision and scale (DFGPU_DECIMAL128_TYPE)");
          DF_CHECK(dec_avg_state || !(a->state_input || a->state_output), DFGPU_ERR_UNSUPPORTED,
                   "AVG over Decimal128 runs in Single modes only: its Partial state is not defined");
          s.cls = 3;
          s.out_type = dec_type(std::min(38, dec_precision(vt) + 4), std::min(38, dec_scale(vt) + 4));
        } else {
          DF_CHECK(type_is_int(vt) || type_is_float(vt), DFGPU_ERR_UNSUPPORTED, "AVG: numeric argument required");
          s.cls = 2;
        }
        s.init0 = 0; break;
      case DFGPU_AGG_MIN:
      case DFGPU_AGG_MAX: {
        const bool is_min = s.func == DFGPU_AGG_MIN;
        if (type_is_decimal(vt)) {   // signed i128 order; identity i128::MAX / i128::MIN as {lo, hi}
          s.cls = 3;
          s.init0 = is_min ? ~0ull : 0ull;
          s.init1 = is_min ? (unsigned long long)LLONG_MAX : (unsigned long long)LLONG_MIN;
          break;
        }
        DF_CHECK(type_is_int(vt) || type_is_float(vt), DFGPU_ERR_UNSUPPORTED, is_min ? "MIN: numeric argument required" : "MAX: numeric argument required");
        if (is_min) s.init0 = s.cls == 0 ? (unsigned long long)LLONG_MAX : ~0ull;
        else s.init0 = s.cls == 0 ? (unsigned long long)LLONG_MIN : 0ull;
        break;
      }
      default: throw Error(DFGPU_ERR_INVALID, "unknown aggregate function");
    }
    a->aggs.push_back(std::move(s));
  }
  // table
  uint64_t cap = 1 << 16;
  // with a hint the table is sized at 3 slots per hinted group: a sparser table costs L2 capacity (at load
  // factor 0.25 the table's DRAM reads were twice the input bytes).  The C3 shape (1M groups: 3M slots x 24 B of
  // tag + {sum, count} = 72 MB) does not fit the H100's 50 MB L2 even so: its lookups and REDs reach DRAM
  static const int cap_mult = getenv("DFGPU_AGG_CAPMULT") ? atoi(getenv("DFGPU_AGG_CAPMULT")) : 3;
  static const int bucket_env = getenv("DFGPU_AGG_BUCKET") ? atoi(getenv("DFGPU_AGG_BUCKET")) : 1;
  a->bucketed = bucket_env != 0;
  a->fast_r4 = getenv("DFGPU_AGG_R4") ? atoi(getenv("DFGPU_AGG_R4")) : 0;
  a->paired_mode = getenv("DFGPU_AGG_PAIRED") ? atoi(getenv("DFGPU_AGG_PAIRED")) : kAggPairedDefault;
  if (capacity_hint > 0) { cap = std::max<uint64_t>(cap, (uint64_t)capacity_hint * cap_mult); a->hinted = true; }
  cap = (cap + 3) & ~3ull;
  a->cap = cap;
  a->counters.alloc(ctx, 16); a->counters.zero();
  a->special_used.alloc(ctx, 8); a->special_used.zero();
  {
    std::vector<DevBuf> acc0, acc1, seen;
    alloc_table(a.get(), cap, &a->tags, &acc0, &acc1, &seen, &a->kstore, &a->knull);
    for (size_t i = 0; i < a->aggs.size(); ++i) { a->aggs[i].acc0 = std::move(acc0[i]); a->aggs[i].acc1 = std::move(acc1[i]); a->aggs[i].seen = std::move(seen[i]); }
  }
  return a.release();
}

}  // namespace dfgpu

extern "C" {

int dfgpu_agg_create(dfgpu_ctx* ctx, const int32_t* input_types, int32_t n_cols, const int32_t* group_cols, int32_t n_group,
                     const dfgpu_agg_desc* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size, int64_t capacity_hint, dfgpu_agg** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && out, DFGPU_ERR_INVALID, "null argument");
  *out = agg_create(ctx, input_types, n_cols, group_cols, n_group, aggs, n_aggs, mode, batch_size, capacity_hint, false);
  DF_API_END
}

int dfgpu_agg_push_host(dfgpu_agg* a, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(a ? a->ctx : nullptr)
  set_device(a->ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(upload_column(a->ctx, cols[i]));
  agg_push(a, v);
  DF_API_END
}
int dfgpu_agg_push_device(dfgpu_agg* a, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(a ? a->ctx : nullptr)
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(device_view(cols[i]));
  agg_push(a, v);  // fully consumed (stream-synchronised) before returning
  DF_API_END
}
int dfgpu_agg_set_skip_partial(dfgpu_agg* a, int64_t probe_rows_threshold, double probe_ratio_threshold) {
  DF_API_BEGIN(a ? a->ctx : nullptr)
  DF_CHECK(a, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(a->m_input_rows == 0, DFGPU_ERR_STATE, "set_skip_partial must be called before the first push");
  dfgpu_agg* t = a->scalar ? nullptr : a;
  if (t) { t->probe_rows_threshold = probe_rows_threshold; t->probe_ratio_threshold = probe_ratio_threshold; }
  DF_API_END
}
int dfgpu_agg_finish(dfgpu_agg* a) {
  DF_API_BEGIN(a ? a->ctx : nullptr)
  agg_finish(a);
  DF_API_END
}
int dfgpu_agg_next(dfgpu_agg* a, int host, dfgpu_batch** out) {
  dfgpu_ctx* _ctx = a ? a->ctx : nullptr;
  try {
    DF_CHECK(a && out, DFGPU_ERR_INVALID, "null argument");
    if (a->outq.empty()) { *out = nullptr; return DFGPU_END; }
    BatchPtr b = std::move(a->outq.front());
    a->outq.pop_front();
    if (host) { set_device(a->ctx); b = to_host_batch(a->ctx, *b); }
    *out = b.release();
    return DFGPU_OK;
  } catch (const dfgpu::Error& e) { if (_ctx) _ctx->last_error = e.what(); return e.code; }
  catch (const std::exception& e) { if (_ctx) _ctx->last_error = e.what(); return DFGPU_ERR_INVALID; }
}
int64_t dfgpu_agg_metric(dfgpu_agg* a, const char* name) {
  if (!a || !name) return -1;
  std::string s(name);
  if (s == "num_groups") return a->m_num_groups;
  if (s == "input_rows") return a->m_input_rows;
  if (s == "input_batches") return a->m_input_batches;
  if (s == "output_rows") return a->m_output_rows;
  if (s == "table_capacity") return (int64_t)a->cap;
  if (s == "rehashes") return a->m_rehashes;
  if (s == "key_words") return a->kw;
  if (s == "skipped_aggregation_rows") return a->m_skipped_rows;
  return -1;
}
void dfgpu_agg_destroy(dfgpu_agg* a) {
  if (!a) return;
  cudaSetDevice(a->ctx->device);
  if (a->inner1) dfgpu_agg_destroy(a->inner1);
  if (a->inner2) dfgpu_agg_destroy(a->inner2);
  delete a;
}

}  // extern "C"
