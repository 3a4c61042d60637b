// hash_join.cu — GpuHashJoinExec: build-side table construction + probe-side lookup/emit.
//
// Reference path being replaced (SURVEY.md §8a rows a9–a16):
//   build : collect_left_input            joins/hash_join/exec.rs:2569-2776
//           try_create_array_map          joins/hash_join/exec.rs:111-191   (perfect-hash / ArrayMap)
//           update_hash / update_from_iter joins/utils.rs:2127-2165, joins/join_hash_map.rs:307-337
//   probe : lookup_join_hashmap           joins/hash_join/stream.rs:396-438
//           get_matched_indices_with_limit_offset  joins/join_hash_map.rs:389-484, chain.rs:29-70
//           ArrayMap::lookup_and_get_indices       joins/array_map.rs:247-372
//           equal_rows_arr                joins/utils.rs:2191-2257
//           adjust_indices_by_join_type   joins/utils.rs:1432-1490
//           build_batch_from_indices      joins/utils.rs:1332-1387
//   final : process_unmatched_build_batch joins/hash_join/stream.rs:1002-1100
//
// GPU design (not a translation of the hashbrown + next[] structure):
//   * one open-addressing table of 16-byte slots {tag:u64, head:u32, cnt:u32} sized 2x the build
//     rows, or — when the reference would pick its ArrayMap — a direct-address array of
//     {head,cnt}.  The join key (all key columns, <= 64 bits together) is stored *exactly* in the
//     tag, so a probe needs one 16-byte load and no equal_rows_arr re-check.
//   * duplicates: lock-free *sorted* chains through next[] built with atomicMin, so a probe walks
//     matches in ascending build-row order == the reference's emission order
//     (exec.rs:634-640 "Inner join output is expected to preserve both inputs order").
//   * probe = count kernel (one table lookup per probe row, per-tile totals) -> single-block scan of
//     tile totals -> emit kernel writing (build_idx, probe_idx) pairs in reference order ->
//     one gather (`take`) kernel per output column.
#include "batch.cuh"
#include "scan.cuh"
#include "expr.cuh"
#include "bloom.cuh"

namespace dfgpu {

constexpr uint32_t kEmpty32 = 0xFFFFFFFFu;
constexpr uint64_t kEmpty64 = 0xFFFFFFFFFFFFFFFFull;
constexpr uint32_t kVisitedBit = 0x80000000u;
constexpr int kMaxKeys = 4;

struct KeyCols {
  int n;
  const void* ptr[kMaxKeys];
  const uint8_t* valid[kMaxKeys];
  int64_t voff[kMaxKeys];
  int width[kMaxKeys];   // bytes
  int sgn[kMaxKeys];     // sign-extend (single-key mode: mirrors `as u64` of array_map.rs:123-135)
  int shift[kMaxKeys];   // bit position when packing several columns
};

// returns false when any key column is NULL at `row`.
// null_as_key: NullEqualsNull single-column mode — reported through *is_null instead.
__device__ __forceinline__ bool load_tag(const KeyCols& kc, int64_t row, uint64_t* tag) {
  uint64_t t = 0;
  bool ok = true;
#pragma unroll
  for (int c = 0; c < kMaxKeys; ++c) {
    if (c >= kc.n) break;
    if (kc.valid[c] && !bit_get(kc.valid[c], kc.voff[c] + row)) ok = false;
    uint64_t v;
    switch (kc.width[c]) {
      case 1: v = kc.sgn[c] ? (uint64_t)(int64_t)((const int8_t*)kc.ptr[c])[row] : (uint64_t)((const uint8_t*)kc.ptr[c])[row]; break;
      case 2: v = kc.sgn[c] ? (uint64_t)(int64_t)((const int16_t*)kc.ptr[c])[row] : (uint64_t)((const uint16_t*)kc.ptr[c])[row]; break;
      case 4: v = kc.sgn[c] ? (uint64_t)(int64_t)((const int32_t*)kc.ptr[c])[row] : (uint64_t)((const uint32_t*)kc.ptr[c])[row]; break;
      default: v = ((const uint64_t*)kc.ptr[c])[row]; break;
    }
    if (kc.n > 1) { if (kc.width[c] < 8) v &= (1ull << (8 * kc.width[c])) - 1ull; v <<= kc.shift[c]; }
    t |= v;
  }
  *tag = t;
  return ok;
}

struct TableRef {
  uint4* slots;       // hash mode: cap slots + 1 special slot (tag == all-ones) at index cap
  uint64_t cap;
  uint2* amap;        // array-map mode: {head,cnt} per key value in [amin, amin+arange]
  uint64_t amin;
  uint64_t asize;     // arange + 1
  uint32_t* next;     // sorted chain links (kEmpty32 terminates)
  uint2* null_slot;   // NullEqualsNull: the entry that collects NULL-key rows (else nullptr)
  int force_collisions;  // mirror of feature force_hash_collisions: every key hashes to slot 0
};

__device__ __forceinline__ uint64_t slot_of(uint64_t tag, const TableRef& t) {
  if (t.force_collisions) return 0;
  return __umul64hi(hash_u64(tag, kSeedJoin), t.cap);  // fastrange on the upper hash bits
}

// find-or-claim the entry for `tag` (build side). Returns pointer to {head,cnt}.
__device__ __forceinline__ uint32_t* claim_entry(const TableRef& t, uint64_t tag) {
  if (t.amap) return (uint32_t*)&t.amap[tag - t.amin];
  if (tag == kEmpty64) return ((uint32_t*)&t.slots[t.cap]) + 2;
  uint64_t s = slot_of(tag, t);
  while (true) {
    unsigned long long* tp = (unsigned long long*)&t.slots[s];
    unsigned long long cur = __ldcg(tp);
    if (cur == kEmpty64) {
      unsigned long long prev = atomicCAS(tp, (unsigned long long)kEmpty64, (unsigned long long)tag);
      cur = (prev == kEmpty64) ? (unsigned long long)tag : prev;
    }
    if (cur == tag) return ((uint32_t*)tp) + 2;
    if (++s == t.cap) s = 0;
  }
}

// read-only lookup (probe side / final pass). Returns pointer to {head,cnt} or nullptr.
__device__ __forceinline__ uint32_t* find_entry(const TableRef& t, uint64_t tag) {
  if (t.amap) {
    uint64_t i = tag - t.amin;  // wrapping: key_to_index of array_map.rs:159-166
    if (i >= t.asize) return nullptr;
    return (uint32_t*)&t.amap[i];
  }
  if (tag == kEmpty64) return ((uint32_t*)&t.slots[t.cap]) + 2;
  uint64_t s = slot_of(tag, t);
  while (true) {
    const uint4 v = __ldcg(&t.slots[s]);
    uint64_t cur = (uint64_t)v.x | ((uint64_t)v.y << 32);
    if (cur == tag) return ((uint32_t*)&t.slots[s]) + 2;
    if (cur == kEmpty64) return nullptr;
    if (++s == t.cap) s = 0;
  }
}

// lock-free sorted insert of `row` into the chain rooted at *head (all links only ever decrease)
__device__ __forceinline__ void chain_insert(uint32_t* head, uint32_t* next, uint32_t row) {
  uint32_t* p = head;
  uint32_t x = row;
  while (true) {
    uint32_t old = atomicMin(p, x);
    if (old == kEmpty32) return;
    if (old > x) { p = &next[x]; x = old; }  // we displaced `old`: carry it behind x
    else { p = &next[old]; }                 // keep walking
  }
}

// null-aware LeftAnti: build rows whose key is NULL are treated as visited, so the final pass does not emit them
__global__ void __launch_bounds__(256) mark_null_keys_kernel(const uint8_t* __restrict__ valid, int64_t voff, int64_t n, uint32_t* __restrict__ vis) {
  const int64_t nw = (n + 31) / 32;
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nw; w += (int64_t)gridDim.x * blockDim.x) {
    uint32_t m = 0;
    for (int b = 0; b < 32; ++b) {
      const int64_t row = w * 32 + b;
      if (row < n && !bit_get(valid, voff + row)) m |= 1u << b;
    }
    if (m) vis[w] |= m;
  }
}

// ------------------------------------------------------------------------------------------
// build
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) join_minmax_kernel(KeyCols kc, int64_t n, int sgn, unsigned long long* mm /* [min,max,valid] */) {
  // min/max of a single integer key, as collect_left_input tracks for the perfect-hash decision (exec.rs:2585-2619)
  long long lmin_s = LLONG_MAX, lmax_s = LLONG_MIN;
  unsigned long long lmin_u = ~0ull, lmax_u = 0, cnt = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t t;
    if (!load_tag(kc, i, &t)) continue;
    cnt++;
    if (sgn) { long long v = (long long)t; lmin_s = min(lmin_s, v); lmax_s = max(lmax_s, v); }
    else { lmin_u = min(lmin_u, (unsigned long long)t); lmax_u = max(lmax_u, (unsigned long long)t); }
  }
  // block-level reduction first: one atomic triple per block, not per thread (the same three addresses serialise in L2)
  unsigned long long kmin = sgn ? (unsigned long long)lmin_s ^ (1ull << 63) : lmin_u;   // order-preserving map of signed keys onto unsigned
  unsigned long long kmax = sgn ? (unsigned long long)lmax_s ^ (1ull << 63) : lmax_u;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, d));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, d));
    cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  }
  __shared__ unsigned long long s_red[3][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_red[0][warp] = kmin; s_red[1][warp] = kmax; s_red[2][warp] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) { kmin = min(kmin, s_red[0][w]); kmax = max(kmax, s_red[1][w]); cnt += s_red[2][w]; }
    if (cnt) {
      if (sgn) { atomicMin((long long*)&mm[0], (long long)(kmin ^ (1ull << 63))); atomicMax((long long*)&mm[1], (long long)(kmax ^ (1ull << 63))); }
      else { atomicMin(&mm[0], kmin); atomicMax(&mm[1], kmax); }
      atomicAdd(&mm[2], cnt);
    }
  }
}

struct alignas(16) Slot128 { unsigned long long lo, hi; };
__device__ __forceinline__ Slot128 cas128(void* addr, Slot128 cmp, Slot128 val) {
  Slot128 old;
  asm volatile("{\n\t.reg .b128 c, v, o;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 v, {%4, %5};\n\tatom.global.cas.b128 o, [%6], c, v;\n\tmov.b128 {%0, %1}, o;\n\t}"
               : "=l"(old.lo), "=l"(old.hi) : "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi), "l"(addr) : "memory");
  return old;
}

// Insert `row` under `tag`.  The common case (first row of its key) is ONE 128-bit CAS that claims the
// slot and installs {tag, head=row, cnt=0} together; only duplicates take the counter + sorted-chain path.
// Returns true when this row created the key.
__device__ __forceinline__ bool insert_row(const TableRef& t, uint64_t tag, uint32_t row) {
  uint32_t* e = nullptr;
  if (t.amap) {
    unsigned long long* ep = (unsigned long long*)&t.amap[tag - t.amin];
    unsigned long long prev = atomicCAS(ep, (unsigned long long)kEmpty64, (unsigned long long)row /* head=row, cnt=0 */);
    if (prev == kEmpty64) return true;
    e = (uint32_t*)ep;
  } else if (tag == kEmpty64) {
    e = ((uint32_t*)&t.slots[t.cap]) + 2;  // dedicated slot for the all-ones key
  } else {
    uint64_t s = slot_of(tag, t);
    while (true) {
      const uint4 v = __ldcg(&t.slots[s]);
      uint64_t cur = (uint64_t)v.x | ((uint64_t)v.y << 32);
      if (cur == kEmpty64) {
        Slot128 prev = cas128(&t.slots[s], Slot128{kEmpty64, kEmpty64}, Slot128{tag, (unsigned long long)row /* head=row, cnt=0 */});
        if (prev.lo == kEmpty64) return true;
        cur = prev.lo;
      }
      if (cur == tag) { e = ((uint32_t*)&t.slots[s]) + 2; break; }
      if (++s == t.cap) s = 0;
    }
  }
  uint32_t old = atomicAdd(e + 1, 1u);
  chain_insert(e, t.next, row);
  return old == kEmpty32;  // only possible on the special / NULL slots (memset state)
}

__global__ void __launch_bounds__(256) join_build_kernel(KeyCols kc, int64_t n, TableRef t, unsigned long long* counters /* [distinct, valid_rows, null_rows] */) {
  unsigned int distinct = 0, valid = 0, nulls = 0;
  // rows are visited in DESCENDING order: a later (smaller) row then usually becomes the new chain
  // head with two atomics, mirroring the reference's reverse iteration (exec.rs:2684-2702, array_map.rs:213)
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t row = n - 1 - i;
    uint64_t tag;
    bool ok = load_tag(kc, row, &tag);
    if (!ok) nulls++;
    if (ok) {
      distinct += insert_row(t, tag, (uint32_t)row) ? 1u : 0u;
      valid++;
    } else if (t.null_slot) {  // NullEqualsNull: NULL keys collect in their own entry
      uint32_t* e = (uint32_t*)t.null_slot;
      uint32_t old = atomicAdd(e + 1, 1u);
      chain_insert(e, t.next, (uint32_t)row);
      distinct += old == kEmpty32 ? 1u : 0u;
      valid++;
    }  // else: NULL key under NullEqualsNothing is not inserted (utils.rs:2146-2155)
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    distinct += __shfl_xor_sync(0xffffffffu, distinct, d);
    valid += __shfl_xor_sync(0xffffffffu, valid, d);
    nulls += __shfl_xor_sync(0xffffffffu, nulls, d);
  }
  if ((threadIdx.x & 31) == 0) {
    if (distinct) atomicAdd(&counters[0], (unsigned long long)distinct);
    if (valid) atomicAdd(&counters[1], (unsigned long long)valid);
    if (nulls) atomicAdd(&counters[2], (unsigned long long)nulls);
  }
}

// ------------------------------------------------------------------------------------------
// probe
// ------------------------------------------------------------------------------------------
constexpr int kProbeThreads = 256;
constexpr int kProbeItems = 4;
constexpr int kProbeTile = kProbeThreads * kProbeItems;

enum EmitMode : int {
  EMIT_PAIRS = 0,        // Inner / Left: one output row per match
  EMIT_PAIRS_OUTER = 1,  // Right / Full: matches, or (NULL, probe) when none
  EMIT_SEMI = 2,         // RightSemi: probe rows with >= 1 match
  EMIT_ANTI = 3,         // RightAnti: probe rows with no match
  EMIT_ALL = 4,          // RightMark: every probe row (+ mark column)
  EMIT_NONE = 5          // LeftSemi / LeftAnti / LeftMark: only the visited flags matter
};

__device__ __forceinline__ uint32_t out_count_for(int mode, uint32_t cnt) {
  switch (mode) {
    case EMIT_PAIRS: return cnt;
    case EMIT_PAIRS_OUTER: return cnt ? cnt : 1u;
    case EMIT_SEMI: return cnt ? 1u : 0u;
    case EMIT_ANTI: return cnt ? 0u : 1u;
    case EMIT_ALL: return 1u;
    default: return 0u;
  }
}

// pass 1: one lookup per probe row.  Writes head[i] (first matching build row or kEmpty32),
// cnt[i] (number of matching build rows; omitted when the build side is unique) and the per-tile
// output-row total.
template <bool UNIQUE>
__global__ void __launch_bounds__(kProbeThreads) join_probe_count_kernel(KeyCols kc, int64_t n, TableRef t, int mode, int mark_visited,
                                                                      uint32_t* __restrict__ head_out, uint32_t* __restrict__ cnt_out,
                                                                      uint64_t* __restrict__ tile_sums, unsigned long long* __restrict__ hit_rows) {
  const int64_t tile_base = (int64_t)blockIdx.x * kProbeTile;
  uint32_t local_out = 0, local_hits = 0;
#pragma unroll
  for (int k = 0; k < kProbeItems; ++k) {
    int64_t i = tile_base + k * kProbeThreads + threadIdx.x;
    if (i >= n) break;
    uint64_t tag;
    bool ok = load_tag(kc, i, &tag);
    uint32_t* e = nullptr;
    if (ok) e = find_entry(t, tag);
    else if (t.null_slot) e = (uint32_t*)t.null_slot;
    uint32_t head = kEmpty32, cnt = 0;
    if (e) {
      uint2 hc = __ldcg((const uint2*)e);
      if (hc.x != kEmpty32) {
        head = hc.x;
        cnt = (hc.y & ~kVisitedBit) + 1u;
        if (mark_visited && !(hc.y & kVisitedBit)) atomicOr(e + 1, kVisitedBit);
        local_hits++;
      }
    }
    head_out[i] = head;
    if (!UNIQUE) cnt_out[i] = cnt;
    local_out += out_count_for(mode, cnt);
  }
  uint64_t tot = block_reduce_sum<kProbeThreads, uint64_t>((uint64_t)local_out);
  uint64_t hits = block_reduce_sum<kProbeThreads, uint64_t>((uint64_t)local_hits);
  if (threadIdx.x == 0) {
    tile_sums[blockIdx.x] = tot;
    if (hits) atomicAdd(hit_rows, (unsigned long long)hits);
  }
}

// pass 2: emit (build_idx, probe_idx) pairs in reference order: probe-row order, and within one
// probe row ascending build row (chain order).
template <bool UNIQUE>
__global__ void __launch_bounds__(kProbeThreads) join_emit_kernel(int64_t n, const uint32_t* __restrict__ head_in, const uint32_t* __restrict__ cnt_in,
                                                               const uint32_t* __restrict__ next, const uint64_t* __restrict__ tile_offsets, int mode,
                                                               uint32_t* __restrict__ build_idx, uint32_t* __restrict__ probe_idx) {
  const int64_t tile_base = (int64_t)blockIdx.x * kProbeTile;
  uint64_t base = tile_offsets[blockIdx.x];
#pragma unroll
  for (int k = 0; k < kProbeItems; ++k) {
    int64_t i = tile_base + k * kProbeThreads + threadIdx.x;
    uint32_t head = kEmpty32, cnt = 0;
    if (i < n) {
      head = head_in[i];
      cnt = UNIQUE ? (head != kEmpty32 ? 1u : 0u) : cnt_in[i];
    }
    uint32_t oc = i < n ? out_count_for(mode, cnt) : 0u;
    uint32_t tot;
    uint32_t ex = block_exclusive_scan<kProbeThreads, uint32_t>(oc, &tot);
    uint64_t pos = base + ex;
    if (oc) {
      if (mode == EMIT_PAIRS || (mode == EMIT_PAIRS_OUTER && cnt)) {
        uint32_t r = head;
        for (uint32_t m = 0; m < cnt; ++m) {
          build_idx[pos + m] = r;
          probe_idx[pos + m] = (uint32_t)i;
          if (!UNIQUE && m + 1 < cnt) r = next[r];
        }
      } else {
        // outer padding / semi / anti / mark: one row; build index = first match or NULL
        if (build_idx) build_idx[pos] = head;
        probe_idx[pos] = (uint32_t)i;
      }
    }
    base += tot;
  }
}

// ------------------------------------------------------------------------------------------
// fused probe + materialise (unique build side, Inner/Left): one pass, reference order.
//   tile = 256 threads x 4 consecutive probe rows; lookups -> matched (build,probe) pairs compacted in
//   shared memory -> the tile's output offset through a decoupled look-back over tile descriptors
//   (single pass, no global pair arrays, no second probe) -> coalesced writes of every output column,
//   gathering build columns by build row and probe columns by probe row.
// ------------------------------------------------------------------------------------------
constexpr int kFusedThreads = 256;
constexpr int kFusedItems = 4;
constexpr int kFusedTile = kFusedThreads * kFusedItems;
constexpr int kMaxFusedCols = 16;
struct FusedCols {
  int n;
  const void* src[kMaxFusedCols];
  void* dst[kMaxFusedCols];
  int width[kMaxFusedCols];  // 1,2,4,8,16 bytes
  int side[kMaxFusedCols];   // 0 build, 1 probe
};
__global__ void __launch_bounds__(kFusedThreads) join_probe_fused_kernel(KeyCols kc, int64_t n, TableRef t, int mark_visited, FusedCols oc,
                                                                      unsigned long long* __restrict__ tile_desc, unsigned int* __restrict__ tile_counter,
                                                                      unsigned long long* __restrict__ totals /* [out_rows, hit_rows] */) {
  __shared__ uint32_t s_b[kFusedTile], s_p[kFusedTile];
  __shared__ unsigned int s_tile;
  __shared__ unsigned long long s_base;
  if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);  // dynamic tile order = look-back never waits on an unscheduled tile
  __syncthreads();
  const int64_t tile = s_tile;
  const int64_t row0 = tile * kFusedTile + (int64_t)threadIdx.x * kFusedItems;
  uint32_t heads[kFusedItems];
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    heads[k] = kEmpty32;
    const int64_t i = row0 + k;
    if (i < n) {
      uint64_t tag;
      bool ok = load_tag(kc, i, &tag);
      uint32_t* e = nullptr;
      if (ok) e = find_entry(t, tag);
      else if (t.null_slot) e = (uint32_t*)t.null_slot;
      if (e) {
        uint2 hc = __ldcg((const uint2*)e);
        if (hc.x != kEmpty32) {
          heads[k] = hc.x;
          ++m;
          if (mark_visited && !(hc.y & kVisitedBit)) atomicOr(e + 1, kVisitedBit);
        }
      }
    }
  }
  uint32_t tot;
  uint32_t ex = block_exclusive_scan<kFusedThreads, uint32_t>(m, &tot);
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k)
    if (heads[k] != kEmpty32) { s_b[ex] = heads[k]; s_p[ex] = (uint32_t)(row0 + k - tile * kFusedTile); ++ex; }
  if (threadIdx.x < 32) {
    unsigned long long exclusive = tile_lookback(tile, tot, tile_desc);
    if (threadIdx.x == 0) {
      s_base = exclusive;
      if ((tile + 1) * (int64_t)kFusedTile >= n) totals[0] = exclusive + tot;  // last tile: total output rows
      if (tot) atomicAdd(&totals[1], (unsigned long long)tot);
    }
  }
  __syncthreads();
  const unsigned long long base = s_base;
  const int64_t prow0 = tile * kFusedTile;
  // ---- materialise: every output column, coalesced writes ----
  for (int c = 0; c < oc.n; ++c) {
    const bool build_side = oc.side[c] == 0;
    switch (oc.width[c]) {
      case 8: {
        const uint64_t* src = (const uint64_t*)oc.src[c];
        uint64_t* dst = (uint64_t*)oc.dst[c] + base;
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = build_side ? src[s_b[j]] : src[prow0 + s_p[j]];
        break;
      }
      case 4: {
        const uint32_t* src = (const uint32_t*)oc.src[c];
        uint32_t* dst = (uint32_t*)oc.dst[c] + base;
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = build_side ? src[s_b[j]] : src[prow0 + s_p[j]];
        break;
      }
      case 2: {
        const uint16_t* src = (const uint16_t*)oc.src[c];
        uint16_t* dst = (uint16_t*)oc.dst[c] + base;
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = build_side ? src[s_b[j]] : src[prow0 + s_p[j]];
        break;
      }
      case 1: {
        const uint8_t* src = (const uint8_t*)oc.src[c];
        uint8_t* dst = (uint8_t*)oc.dst[c] + base;
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = build_side ? src[s_b[j]] : src[prow0 + s_p[j]];
        break;
      }
      default: {
        const uint4* src = (const uint4*)oc.src[c];
        uint4* dst = (uint4*)oc.dst[c] + base;
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = build_side ? src[s_b[j]] : src[prow0 + s_p[j]];
        break;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// inline-payload table (unique build keys, Inner join, narrow build side): the slot IS the build row.
//   slot = {key:u64} or {key:u64, payload:u64} where payload packs every non-key build output column
//   (<= 64 bits together).  A probe is ONE random access (one 64 B DRAM fetch) instead of table + gather,
//   and build-key output columns are read from the probe key (bit-identical by the join condition).
//   Dense keys (the reference's ArrayMap rule) use direct addressing slot = key - min instead of hashing.
//   Any duplicate key or the all-ones key aborts the attempt (flag) and the generic table is built instead.
// ------------------------------------------------------------------------------------------
constexpr int kMaxPayloadCols = 8;
constexpr int kInlineSlotsPer100Rows = 250;   // hashed inline table: 250 slots per 100 build rows
struct PayloadCols { int n; const void* ptr[kMaxPayloadCols]; int width[kMaxPayloadCols]; int shift[kMaxPayloadCols]; };
struct InlineRef { void* slots; uint64_t cap; int dense; uint64_t amin; int bucket; /* probe sequences start on a 4-slot boundary (one 64 B line for 16 B slots) */
                   const unsigned long long* bloom; uint64_t bloom_blocks; /* optional membership filter over the build keys (dfgpu_hashjoin_options.membership_filter) */ };
struct InlineOut {
  int n;
  int kind[kMaxFusedCols];   // 0: gather from a probe-side column by probe row; 1: extract from the payload word
  const void* src[kMaxFusedCols];
  void* dst[kMaxFusedCols];
  int width[kMaxFusedCols];
  int shift[kMaxFusedCols];
  uint32_t* pidx_out;        // optional: matched probe row per output row (for nullable probe columns gathered afterwards)
};

__device__ __forceinline__ uint64_t load_payload(const PayloadCols& pc, int64_t row) {
  uint64_t p = 0;
#pragma unroll
  for (int c = 0; c < kMaxPayloadCols; ++c) {
    if (c >= pc.n) break;
    uint64_t v;
    switch (pc.width[c]) {
      case 1: v = ((const uint8_t*)pc.ptr[c])[row]; break;
      case 2: v = ((const uint16_t*)pc.ptr[c])[row]; break;
      case 4: v = ((const uint32_t*)pc.ptr[c])[row]; break;
      default: v = ((const uint64_t*)pc.ptr[c])[row]; break;
    }
    p |= v << pc.shift[c];
  }
  return p;
}

// membership filter over the (non-NULL) build keys: the stand-alone join's form of dynamic filter pushdown (a27; the fused pipeline
// carries the same filter in dfgpu_lookup) — a probe row whose key is not in the filter skips the table access, which is a DRAM miss
__global__ void __launch_bounds__(256) join_bloom_build_kernel(KeyCols kc, int64_t n, unsigned long long* __restrict__ bloom, uint64_t blocks) {
  for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    uint64_t tag;
    if (load_tag(kc, row, &tag)) bloom_set(bloom, blocks, tag);
  }
}

template <int W>
__global__ void __launch_bounds__(256) join_build_inline_kernel(KeyCols kc, PayloadCols pc, int64_t n, InlineRef t, unsigned long long* counters /* [valid, nulls, fail] */) {
  unsigned int valid = 0, nulls = 0, fail = 0;
  for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    uint64_t tag;
    if (!load_tag(kc, row, &tag)) { nulls++; continue; }  // NULL key: never matches under NullEqualsNothing
    valid++;
    if (tag == kEmpty64) { fail = 1; continue; }
    const uint64_t pay = W == 2 ? load_payload(pc, row) : 0ull;
    uint64_t s = t.dense ? (tag - t.amin) : (t.bucket ? (__umul64hi(hash_u64(tag, kSeedJoin), t.cap >> 2) << 2) : __umul64hi(hash_u64(tag, kSeedJoin), t.cap));
    while (true) {
      unsigned long long prev;
      if (W == 2) prev = cas128((Slot128*)t.slots + s, Slot128{kEmpty64, kEmpty64}, Slot128{tag, pay}).lo;
      else prev = atomicCAS((unsigned long long*)t.slots + s, (unsigned long long)kEmpty64, (unsigned long long)tag);
      if (prev == kEmpty64) break;
      if (prev == tag) { fail = 1; break; }  // duplicate build key
      if (++s == t.cap) s = 0;
    }
  }
  fail = __any_sync(0xffffffffu, fail) ? 1u : 0u;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { valid += __shfl_xor_sync(0xffffffffu, valid, d); nulls += __shfl_xor_sync(0xffffffffu, nulls, d); }
  if ((threadIdx.x & 31) == 0) {
    if (valid) atomicAdd(&counters[0], (unsigned long long)valid);
    if (nulls) atomicAdd(&counters[1], (unsigned long long)nulls);
    if (fail) atomicExch(&counters[2], 1ull);
  }
}

template <int W, bool BLOOM>
__global__ void __launch_bounds__(kFusedThreads) join_probe_inline_kernel(KeyCols kc, int64_t n, InlineRef t, InlineOut oc,
                                                                       unsigned long long* __restrict__ tile_desc, unsigned int* __restrict__ tile_counter,
                                                                       unsigned long long* __restrict__ totals) {
  __shared__ unsigned long long s_pay[W == 2 ? kFusedTile : 1];
  __shared__ uint32_t s_p[kFusedTile];
  __shared__ unsigned int s_tile;
  __shared__ unsigned long long s_base;
  if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);
  __syncthreads();
  const int64_t tile = s_tile;
  const int64_t row0 = tile * kFusedTile + (int64_t)threadIdx.x * kFusedItems;
  uint64_t tags[kFusedItems], slot[kFusedItems], pays[kFusedItems];
  bool live[kFusedItems], hit[kFusedItems];
  // phase 1: keys and first-slot loads for all 4 rows are issued before any is consumed (memory-level parallelism)
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    const int64_t i = row0 + k;
    live[k] = i < n && load_tag(kc, i, &tags[k]) && tags[k] != kEmpty64;
    hit[k] = false;
    pays[k] = 0;
    slot[k] = 0;
    if (live[k]) {
      if (t.dense) { slot[k] = tags[k] - t.amin; if (slot[k] >= t.cap) live[k] = false; }
      else slot[k] = t.bucket ? (__umul64hi(hash_u64(tags[k], kSeedJoin), t.cap >> 2) << 2) : __umul64hi(hash_u64(tags[k], kSeedJoin), t.cap);
    }
  }
  if (BLOOM) {   // the filter words of the 4 rows are fetched back to back (L2-resident), then the rows without a partner drop out
    unsigned long long bw[kFusedItems]; uint32_t bt[kFusedItems];
#pragma unroll
    for (int k = 0; k < kFusedItems; ++k) { bw[k] = ~0ull; bt[k] = 0; if (live[k]) { const BloomPos bp = bloom_pos(tags[k], t.bloom_blocks); bt[k] = bp.t; bw[k] = __ldg(t.bloom + bp.block); } }
#pragma unroll
    for (int k = 0; k < kFusedItems; ++k) if (live[k] && !bloom_test(bw[k], bt[k])) live[k] = false;
  }
  uint64_t cur[kFusedItems], curp[kFusedItems];
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    cur[k] = kEmpty64; curp[k] = 0;
    if (live[k]) {
      if (W == 2) { const uint4 v = __ldcg((const uint4*)t.slots + slot[k]); cur[k] = (uint64_t)v.x | ((uint64_t)v.y << 32); curp[k] = (uint64_t)v.z | ((uint64_t)v.w << 32); }
      else cur[k] = __ldcg((const unsigned long long*)t.slots + slot[k]);
    }
  }
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    if (!live[k]) continue;
    while (true) {  // linear probing continues only on a foreign key (rare at load factor 0.5; never in dense mode)
      if (cur[k] == tags[k]) { hit[k] = true; pays[k] = curp[k]; break; }
      if (cur[k] == kEmpty64 || t.dense) break;
      if (++slot[k] == t.cap) slot[k] = 0;
      if (W == 2) { const uint4 v = __ldcg((const uint4*)t.slots + slot[k]); cur[k] = (uint64_t)v.x | ((uint64_t)v.y << 32); curp[k] = (uint64_t)v.z | ((uint64_t)v.w << 32); }
      else cur[k] = __ldcg((const unsigned long long*)t.slots + slot[k]);
    }
    m += hit[k] ? 1u : 0u;
  }
  uint32_t tot;
  uint32_t ex = block_exclusive_scan<kFusedThreads, uint32_t>(m, &tot);
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k)
    if (hit[k]) { if (W == 2) s_pay[ex] = pays[k]; s_p[ex] = (uint32_t)(row0 + k - tile * kFusedTile); ++ex; }
  if (threadIdx.x < 32) {
    unsigned long long exclusive = tile_lookback(tile, tot, tile_desc);
    if (threadIdx.x == 0) {
      s_base = exclusive;
      if ((tile + 1) * (int64_t)kFusedTile >= n) totals[0] = exclusive + tot;
      if (tot) atomicAdd(&totals[1], (unsigned long long)tot);
    }
  }
  __syncthreads();
  const unsigned long long base = s_base;
  const int64_t prow0 = tile * kFusedTile;
  if (oc.pidx_out) for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) oc.pidx_out[base + j] = (uint32_t)(prow0 + s_p[j]);
  for (int c = 0; c < oc.n; ++c) {
    if (oc.kind[c] == 0) {
      switch (oc.width[c]) {
        case 8: { const uint64_t* src = (const uint64_t*)oc.src[c]; uint64_t* dst = (uint64_t*)oc.dst[c] + base;
                  for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = src[prow0 + s_p[j]]; break; }
        case 4: { const uint32_t* src = (const uint32_t*)oc.src[c]; uint32_t* dst = (uint32_t*)oc.dst[c] + base;
                  for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = src[prow0 + s_p[j]]; break; }
        case 2: { const uint16_t* src = (const uint16_t*)oc.src[c]; uint16_t* dst = (uint16_t*)oc.dst[c] + base;
                  for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = src[prow0 + s_p[j]]; break; }
        case 1: { const uint8_t* src = (const uint8_t*)oc.src[c]; uint8_t* dst = (uint8_t*)oc.dst[c] + base;
                  for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = src[prow0 + s_p[j]]; break; }
        default: { const uint4* src = (const uint4*)oc.src[c]; uint4* dst = (uint4*)oc.dst[c] + base;
                  for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = src[prow0 + s_p[j]]; break; }
      }
    } else if (oc.kind[c] == 1 && W == 2) {
      const int sh = oc.shift[c];
      switch (oc.width[c]) {
        case 8: { uint64_t* dst = (uint64_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = s_pay[j]; break; }
        case 4: { uint32_t* dst = (uint32_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint32_t)(s_pay[j] >> sh); break; }
        case 2: { uint16_t* dst = (uint16_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint16_t)(s_pay[j] >> sh); break; }
        default: { uint8_t* dst = (uint8_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint8_t)(s_pay[j] >> sh); break; }
      }
    }
  }
}

constexpr int kStageCols = 4;   // probe-side output columns staged through shared memory (8 B each per row)

// width-generic loads / stores of one value as 64 bits
__device__ __forceinline__ uint64_t load_w(const void* p, int width, int64_t i) {
  switch (width) {
    case 1: return ((const uint8_t*)p)[i];
    case 2: return ((const uint16_t*)p)[i];
    case 4: return ((const uint32_t*)p)[i];
    default: return ((const uint64_t*)p)[i];
  }
}
__device__ __forceinline__ void store_w(void* p, int width, uint64_t i, uint64_t v) {
  switch (width) {
    case 1: ((uint8_t*)p)[i] = (uint8_t)v; break;
    case 2: ((uint16_t*)p)[i] = (uint16_t)v; break;
    case 4: ((uint32_t*)p)[i] = (uint32_t)v; break;
    default: ((uint64_t*)p)[i] = v; break;
  }
}

// Tile = 256 threads x 4 rows, rows interleaved (row = tile_base + k*256 + tid) so every global load of a
// probe column is one fully coalesced 2 KB wavefront.  Matched rows are ranked in row order with warp
// ballots + one 32-entry scan, their output values (payload word + up to 4 probe-side columns, read while
// the lines are hot) are staged in shared memory, the tile's output offset comes from the decoupled
// look-back, and every output column is then written with fully coalesced stores.  The pipelined host probe
// runs it on each staged chunk.
template <int W>
__global__ void __launch_bounds__(kFusedThreads) join_probe_inline_staged_kernel(KeyCols kc, int64_t n, InlineRef t, InlineOut oc,
                                                                       unsigned long long* __restrict__ tile_desc, unsigned int* __restrict__ tile_counter,
                                                                       unsigned long long* __restrict__ totals) {
  __shared__ unsigned long long s_pay[W == 2 ? kFusedTile : 1];
  __shared__ unsigned long long s_val[kStageCols][kFusedTile];
  __shared__ uint32_t s_p[kFusedTile];
  __shared__ uint32_t s_cnt[kFusedItems * (kFusedThreads / 32) + 1];
  __shared__ unsigned int s_tile;
  __shared__ unsigned long long s_base;
  if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);
  __syncthreads();
  const int64_t tile = s_tile;
  const int64_t prow0 = tile * kFusedTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t tags[kFusedItems], slot[kFusedItems], pays[kFusedItems], cur[kFusedItems], curp[kFusedItems];
  bool live[kFusedItems], hit[kFusedItems];
  // phase 1: keys, then first-slot loads, for all 4 rows before any is consumed (memory-level parallelism)
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    const int64_t i = prow0 + k * kFusedThreads + threadIdx.x;
    live[k] = i < n && load_tag(kc, i, &tags[k]) && tags[k] != kEmpty64;
    hit[k] = false; pays[k] = 0; slot[k] = 0;
    if (live[k]) {
      if (t.dense) { slot[k] = tags[k] - t.amin; if (slot[k] >= t.cap) live[k] = false; }
      else slot[k] = __umul64hi(hash_u64(tags[k], kSeedJoin), t.cap);
    }
  }
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    cur[k] = kEmpty64; curp[k] = 0;
    if (live[k]) {
      if (W == 2) { const uint4 v = __ldcg((const uint4*)t.slots + slot[k]); cur[k] = (uint64_t)v.x | ((uint64_t)v.y << 32); curp[k] = (uint64_t)v.z | ((uint64_t)v.w << 32); }
      else cur[k] = __ldcg((const unsigned long long*)t.slots + slot[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    if (!live[k]) continue;
    while (true) {  // linear probing continues only on a foreign key (never in dense mode)
      if (cur[k] == tags[k]) { hit[k] = true; pays[k] = curp[k]; break; }
      if (cur[k] == kEmpty64 || t.dense) break;
      if (++slot[k] == t.cap) slot[k] = 0;
      if (W == 2) { const uint4 v = __ldcg((const uint4*)t.slots + slot[k]); cur[k] = (uint64_t)v.x | ((uint64_t)v.y << 32); curp[k] = (uint64_t)v.z | ((uint64_t)v.w << 32); }
      else cur[k] = __ldcg((const unsigned long long*)t.slots + slot[k]);
    }
  }
  // phase 2: rank the matches in row order: (k, warp) segments are consecutive row ranges
  uint32_t bal[kFusedItems];
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    bal[k] = __ballot_sync(0xffffffffu, hit[k]);
    if (lane == 0) s_cnt[k * (kFusedThreads / 32) + warp] = __popc(bal[k]);
  }
  __syncthreads();
  if (warp == 0) {  // exclusive scan of the 32 segment counts
    uint32_t c = s_cnt[lane], inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t nb = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += nb; }
    s_cnt[lane] = inc - c;
    if (lane == 31) s_cnt[32] = inc;
  }
  __syncthreads();
  const uint32_t tot = s_cnt[32];
  // phase 3: stage output values of the matched rows
#pragma unroll
  for (int k = 0; k < kFusedItems; ++k) {
    if (!hit[k]) continue;
    const uint32_t pos = s_cnt[k * (kFusedThreads / 32) + warp] + __popc(bal[k] & ((1u << lane) - 1u));
    const int64_t i = prow0 + k * kFusedThreads + threadIdx.x;
    if (W == 2) s_pay[pos] = pays[k];
    s_p[pos] = (uint32_t)(i - prow0);
    int sc = 0;
    for (int c = 0; c < oc.n; ++c)
      if (oc.kind[c] == 0 && oc.width[c] <= 8 && sc < kStageCols) { s_val[sc][pos] = load_w(oc.src[c], oc.width[c], i); ++sc; }
  }
  if (threadIdx.x < 32) {
    unsigned long long exclusive = tile_lookback(tile, tot, tile_desc);
    if (threadIdx.x == 0) {
      s_base = exclusive;
      if ((tile + 1) * (int64_t)kFusedTile >= n) totals[0] = exclusive + tot;
      if (tot) atomicAdd(&totals[1], (unsigned long long)tot);
    }
  }
  __syncthreads();
  const unsigned long long base = s_base;
  if (oc.pidx_out) for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) oc.pidx_out[base + j] = (uint32_t)(prow0 + s_p[j]);
  // phase 4: coalesced column writes
  int sc = 0;
  for (int c = 0; c < oc.n; ++c) {
    if (oc.kind[c] == 0) {
      if (oc.width[c] <= 8 && sc < kStageCols) {
        const unsigned long long* sv = s_val[sc++];
        switch (oc.width[c]) {
          case 8: { uint64_t* dst = (uint64_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = sv[j]; break; }
          case 4: { uint32_t* dst = (uint32_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint32_t)sv[j]; break; }
          case 2: { uint16_t* dst = (uint16_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint16_t)sv[j]; break; }
          default: { uint8_t* dst = (uint8_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint8_t)sv[j]; break; }
        }
      } else if (oc.width[c] == 16) {
        const uint4* src = (const uint4*)oc.src[c]; uint4* dst = (uint4*)oc.dst[c] + base;
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = src[prow0 + s_p[j]];
      } else {
        for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) store_w(oc.dst[c], oc.width[c], base + j, load_w(oc.src[c], oc.width[c], prow0 + s_p[j]));
      }
    } else if (oc.kind[c] == 1 && W == 2) {
      const int sh = oc.shift[c];
      switch (oc.width[c]) {
        case 8: { uint64_t* dst = (uint64_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = s_pay[j]; break; }
        case 4: { uint32_t* dst = (uint32_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint32_t)(s_pay[j] >> sh); break; }
        case 2: { uint16_t* dst = (uint16_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint16_t)(s_pay[j] >> sh); break; }
        default: { uint8_t* dst = (uint8_t*)oc.dst[c] + base; for (uint32_t j = threadIdx.x; j < tot; j += kFusedThreads) dst[j] = (uint8_t)(s_pay[j] >> sh); break; }
      }
    }
  }
}

// final pass over the build rows: which rows were matched by any probe row (the reference's
// visited_indices_bitmap, exec.rs:2712-2723) — recovered from the per-key visited flag.
__global__ void __launch_bounds__(256) join_build_flags_kernel(KeyCols kc, int64_t n, TableRef t, uint32_t* __restrict__ visited_words) {
  int64_t nw = (n + 31) / 32;
  int lane = threadIdx.x & 31;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    int64_t row = wi * 32 + lane;
    bool vis = false;
    if (row < n) {
      uint64_t tag;
      bool ok = load_tag(kc, row, &tag);
      uint32_t* e = nullptr;
      if (ok) e = find_entry(t, tag);
      else if (t.null_slot) e = (uint32_t*)t.null_slot;
      if (e) { uint2 hc = __ldcg((const uint2*)e); vis = (hc.x != kEmpty32) && (hc.y & kVisitedBit); }
    }
    uint32_t w = __ballot_sync(0xffffffffu, vis);
    if (lane == 0) visited_words[wi] = w;
  }
}

// mark column: is_not_null(indices) (utils.rs:1358-1360) as a bit-packed Boolean column
__global__ void mark_from_idx_kernel(const uint32_t* __restrict__ idx, int64_t n, uint32_t* __restrict__ out_words) {
  int64_t nw = (n + 31) / 32;
  int lane = threadIdx.x & 31;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    int64_t i = wi * 32 + lane;
    bool v = i < n && idx[i] != kEmpty32;
    uint32_t w = __ballot_sync(0xffffffffu, v);
    if (lane == 0) out_words[wi] = w;
  }
}

}  // namespace dfgpu

#include "radix_probe.cuh"

// ==========================================================================================
// operator state
// ==========================================================================================
using namespace dfgpu;

struct dfgpu_hashjoin {
  dfgpu_ctx* ctx = nullptr;
  dfgpu_hashjoin_options opt;
  std::vector<int> build_types, probe_types, on_build, on_probe, out_side, out_index;
  // build side
  std::vector<std::vector<DCol>> build_parts;  // per pushed batch
  std::vector<DCol> build_cols;                // concatenated
  int64_t nB = 0;
  bool built = false, probe_done = false;
  DevBuf slots, amap, next, null_slot, counters;
  TableRef table{};
  KeyCols build_keys{};
  bool use_array_map = false, unique = false;
  int64_t distinct = 0, valid_rows = 0, null_rows = 0;
  bool need_visited = false;
  int emit_mode = EMIT_PAIRS;
  // JoinFilter (joins/utils.rs apply_join_filter_to_indices :1248-1320): residual predicate over an intermediate batch
  bool has_filter = false;
  std::vector<int> filt_side, filt_index;
  ExprPlan filt_plan;
  DevBuf visited_rows;   // per build ROW visited bitmap (with a filter, rows of one key can differ)
  // inline-payload table (unique keys, Inner, narrow build side)
  bool inline_ok = false;
  int inline_words = 0;
  DevBuf inline_slots, bloom;
  InlineRef iref{};
  std::vector<int> out_kind, out_src, out_shift;  // per output column: kind (0 probe gather / 1 payload), probe column index, payload shift
  // output
  std::deque<BatchPtr> outq;
  // metrics (BuildProbeJoinMetrics, joins/utils.rs:1756-1778)
  int64_t m_build_rows = 0, m_build_batches = 0, m_input_rows = 0, m_input_batches = 0, m_output_rows = 0, m_output_batches = 0,
          m_array_map = 0, m_probe_hits = 0, m_radix_probes = 0, m_pipelined_probes = 0;
  // wide keys (> 64 bits together, or a 16-byte Decimal128 key): the table is keyed by a 64-bit hash of the key columns (a hidden INT64
  // column appended to both sides) and key equality becomes a conjunct of the JoinFilter — the reference's own scheme: lookup by hash,
  // then equal_rows_arr on the candidate pairs (joins/utils.rs:2191-2257, hash_join/stream.rs lookup_join_hashmap)
  bool wide = false;
  std::vector<int> wide_on_build, wide_on_probe;
  std::vector<dfgpu_expr_node> wide_expr;   // (kb0 = kp0) AND (kb1 = kp1) ... over intermediate columns 0 .. 2 n_keys - 1
  bool probe_side_non_empty = false;
  bool probe_has_null = false;   // null-aware LeftAnti: a NULL probe key was seen (JoinLeftData::probe_side_has_null)
};

namespace dfgpu {

// ---- wide keys: one 64-bit hash per row over all key columns -------------------------------------------------------------------
constexpr int kMaxWideKeys = 8;
struct WideKeyCols { int n; const void* ptr[kMaxWideKeys]; const uint8_t* valid[kMaxWideKeys]; int64_t voff[kMaxWideKeys]; int width[kMaxWideKeys], is_float[kMaxWideKeys]; };
__global__ void __launch_bounds__(256) wide_key_kernel(WideKeyCols kc, int64_t n, int null_equals_null, unsigned long long* __restrict__ out, uint32_t* __restrict__ out_valid) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (n + 31) / 32;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t row = wi * 32 + lane;
    bool ok = row < n;
    if (row < n) {
      uint64_t h = kSeedJoin;
#pragma unroll 1
      for (int c = 0; c < kc.n; ++c) {
        if (kc.valid[c] && !bit_get(kc.valid[c], kc.voff[c] + row)) {
          if (null_equals_null) { h = hash_combine(h, 0x6E756C6Cull); continue; }   // NULL joins NULL: one fixed token per NULL key
          ok = false; break;                                                          // a NULL key never matches (utils.rs:2146-2155)
        }
        uint64_t v, v2 = 0;
        switch (kc.width[c]) {
          case 0: v = bit_get((const uint8_t*)kc.ptr[c], kc.voff[c] + row) ? 1ull : 0ull; break;
          case 1: v = ((const uint8_t*)kc.ptr[c])[row]; break;
          case 2: v = ((const uint16_t*)kc.ptr[c])[row]; break;
          case 4: v = ((const uint32_t*)kc.ptr[c])[row]; if (kc.is_float[c] && (v & 0x7FFFFFFFull) == 0) v = 0; break;   // -0.0 hashes as +0.0: only the equality conjunct tells them apart
          case 16: v = ((const uint64_t*)kc.ptr[c])[2 * row]; v2 = ((const uint64_t*)kc.ptr[c])[2 * row + 1]; break;
          default: v = ((const uint64_t*)kc.ptr[c])[row]; if (kc.is_float[c] && (v << 1) == 0) v = 0; break;
        }
        h = hash_combine(h, v);
        if (kc.width[c] == 16) h = hash_combine(h, v2);
      }
      if (h == kEmpty64) h = 0x5bd1e995ull;      // the table's empty marker is not a key
      out[row] = ok ? h : 0ull;
    }
    const uint32_t b = __ballot_sync(0xffffffffu, ok);
    if (lane == 0 && out_valid) out_valid[wi] = b;
  }
}

// the hidden key column of one batch
static DCol wide_key_column(dfgpu_hashjoin* j, const std::vector<DCol>& cols, const std::vector<int>& on) {
  dfgpu_ctx* ctx = j->ctx;
  set_device(ctx);
  const int64_t n = cols.empty() ? 0 : cols[0].length;
  WideKeyCols kc;
  memset(&kc, 0, sizeof(kc));
  kc.n = (int)on.size();
  bool any_valid = false;
  for (int c = 0; c < kc.n; ++c) {
    const DCol& col = cols[on[c]];
    kc.ptr[c] = col.values; kc.valid[c] = col.validity; kc.voff[c] = col.offset; kc.width[c] = type_width(col.type); kc.is_float[c] = type_is_float(col.type) ? 1 : 0;
    any_valid = any_valid || col.validity != nullptr;
  }
  const bool nen = j->opt.null_equality == DFGPU_NULL_EQUALS_NULL;
  DCol out = alloc_col(ctx, DFGPU_INT64, n, any_valid && !nen);
  if (n > 0) {
    wide_key_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(kc, n, nen ? 1 : 0, (unsigned long long*)out.own_values->ptr,
                                                                         out.own_validity ? out.own_validity->as<uint32_t>() : nullptr);
    DF_LAUNCH_CHECK(ctx);
  }
  out.null_count = (any_valid && !nen) ? -1 : 0;
  return out;
}

static void make_keycols(const std::vector<DCol>& cols, const std::vector<int>& on, KeyCols* kc) {
  memset(kc, 0, sizeof(*kc));
  kc->n = (int)on.size();
  int shift = 0;
  for (int c = 0; c < kc->n; ++c) {
    const DCol& col = cols[on[c]];
    kc->ptr[c] = col.values;
    kc->valid[c] = col.validity;
    kc->voff[c] = col.offset;
    kc->width[c] = type_width(col.type);
    kc->sgn[c] = type_is_signed_int(col.type) ? 1 : 0;
    kc->shift[c] = shift;
    shift += 8 * kc->width[c];
  }
}

// the wide-key equality conjunct reads a float key component as the unsigned type of its width, so it compares the bits: -0.0 does not
// join +0.0 and a NaN joins a NaN with the same bits, as on the exact 64-bit tag (the reference hashes a float by its bits,
// hash_utils.rs hash_float_value, so unequal bits never reach its equality check)
static int wide_key_eq_type(int t) { return t == DFGPU_FLOAT32 ? DFGPU_UINT32 : (t == DFGPU_FLOAT64 ? DFGPU_UINT64 : t); }

static void check_join_keys(dfgpu_hashjoin* j) {
  int bits = 0;
  bool wide = false;
  DF_CHECK(!j->on_build.empty(), DFGPU_ERR_INVALID, "hash join: at least one key column");
  for (size_t c = 0; c < j->on_build.size(); ++c) {
    int bt = j->build_types[j->on_build[c]], pt = j->probe_types[j->on_probe[c]];
    DF_CHECK(type_width(bt) == type_width(pt) && type_is_float(bt) == type_is_float(pt) &&
                 type_is_signed_int(bt) == type_is_signed_int(pt),
             DFGPU_ERR_INVALID, "hash join: key types differ between build and probe side");
    if (type_is_decimal(bt)) DF_CHECK(bt == pt, DFGPU_ERR_INVALID, "hash join: Decimal128 key columns need equal precision and scale on both sides");
    int w = type_width(bt);
    DF_CHECK(w >= 0 && w <= 16, DFGPU_ERR_UNSUPPORTED, "hash join: key type must be a fixed-width type");
    if (w == 16 || w == 0) wide = true;
    bits += 8 * w;
  }
  if (bits > 64 || j->on_build.size() > (size_t)kMaxKeys) wide = true;
  if (wide) {
    // keys that do not fit the exact 64-bit tag: hash + equality conjunct (see dfgpu_hashjoin::wide)
    DF_CHECK(j->on_build.size() <= (size_t)kMaxWideKeys, DFGPU_ERR_UNSUPPORTED, "hash join: at most 8 key columns");
    DF_CHECK(!j->opt.null_aware, DFGPU_ERR_UNSUPPORTED, "hash join: null-aware anti join on a key wider than 64 bits stays on the CPU operator");
    j->wide = true;
    j->wide_on_build = j->on_build; j->wide_on_probe = j->on_probe;
    const int nk = (int)j->on_build.size();
    std::vector<int32_t> types;
    for (int c = 0; c < nk; ++c) {
      j->filt_side.push_back(0); j->filt_index.push_back(j->wide_on_build[c]); types.push_back(wide_key_eq_type(j->build_types[j->wide_on_build[c]]));
      j->filt_side.push_back(1); j->filt_index.push_back(j->wide_on_probe[c]); types.push_back(wide_key_eq_type(j->probe_types[j->wide_on_probe[c]]));
    }
    const int eq = j->opt.null_equality == DFGPU_NULL_EQUALS_NULL ? DFGPU_OP_IS_NOT_DISTINCT_FROM : DFGPU_OP_EQ;
    auto node = [](int kind, int a) { dfgpu_expr_node nd; memset(&nd, 0, sizeof(nd)); nd.kind = kind; nd.a = a; return nd; };
    for (int c = 0; c < nk; ++c) {
      j->wide_expr.push_back(node(DFGPU_EXPR_COLUMN, 2 * c));
      j->wide_expr.push_back(node(DFGPU_EXPR_COLUMN, 2 * c + 1));
      j->wide_expr.push_back(node(DFGPU_EXPR_BINARY, eq));
      if (c > 0) j->wide_expr.push_back(node(DFGPU_EXPR_BINARY, DFGPU_OP_AND));
    }
    j->filt_plan = plan_expr(types.data(), (int)types.size(), j->wide_expr.data(), (int)j->wide_expr.size());
    j->has_filter = true;
    // the hidden hash-key column goes last on both sides and becomes the only `on` column
    j->on_build.assign(1, (int)j->build_types.size()); j->on_probe.assign(1, (int)j->probe_types.size());
    j->build_types.push_back(DFGPU_INT64); j->probe_types.push_back(DFGPU_INT64);
    return;
  }
  if (j->opt.null_equality == DFGPU_NULL_EQUALS_NULL)
    DF_CHECK(j->on_build.size() == 1, DFGPU_ERR_UNSUPPORTED, "hash join: NullEqualsNull on several key columns takes the wide-key path (pass keys wider than 64 bits) or a single column");
}

static void push_build(dfgpu_hashjoin* j, std::vector<DCol>&& cols) {
  DF_CHECK(!j->built, DFGPU_ERR_STATE, "push_build after finish_build");
  if (j->wide && cols.size() + 1 == j->build_types.size()) cols.push_back(wide_key_column(j, cols, j->wide_on_build));
  DF_CHECK(cols.size() == j->build_types.size(), DFGPU_ERR_INVALID, "build batch column count mismatch");
  int64_t rows = cols.empty() ? 0 : cols[0].length;
  for (size_t c = 0; c < cols.size(); ++c) {
    DF_CHECK(cols[c].type == j->build_types[c], DFGPU_ERR_INVALID, "build batch column type mismatch");
    DF_CHECK(cols[c].length == rows, DFGPU_ERR_INVALID, "build batch ragged columns");
  }
  j->nB += rows;
  j->m_build_rows += rows;
  j->m_build_batches++;
  if (rows > 0) j->build_parts.push_back(std::move(cols));
}

static void finish_build(dfgpu_hashjoin* j) {
  DF_CHECK(!j->built, DFGPU_ERR_STATE, "finish_build called twice");
  dfgpu_ctx* ctx = j->ctx;
  set_device(ctx);
  DF_CHECK(j->nB < (int64_t)kEmpty32, DFGPU_ERR_UNSUPPORTED, "hash join: build side must have < 2^32-1 rows");
  // concat_batches (exec.rs:2705)
  j->build_cols.clear();
  for (size_t c = 0; c < j->build_types.size(); ++c) {
    std::vector<DCol> parts;
    for (auto& b : j->build_parts) parts.push_back(b[c]);
    if (parts.empty()) j->build_cols.push_back(alloc_col(ctx, j->build_types[c], 0, false));
    else j->build_cols.push_back(concat_columns(ctx, parts, j->build_types[c]));
  }
  j->build_parts.clear();
  make_keycols(j->build_cols, j->on_build, &j->build_keys);
  const int64_t n = j->nB;
  j->counters.alloc(ctx, 8 * 8);
  j->counters.zero();
  j->next.alloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4);
  j->next.fill(0xFF);
  memset(&j->table, 0, sizeof(j->table));
  j->table.next = j->next.as<uint32_t>();
  j->table.force_collisions = j->opt.force_hash_collisions;
  if (j->opt.null_equality == DFGPU_NULL_EQUALS_NULL) {
    j->null_slot.alloc(ctx, 8);
    j->null_slot.fill(0xFF);
    j->table.null_slot = j->null_slot.as<uint2>();
  }

  // ---- perfect-hash (ArrayMap) decision: try_create_array_map, exec.rs:111-191 ----
  j->use_array_map = false;
  const int kt = j->build_types[j->on_build[0]];
  bool am_type_ok = j->on_build.size() == 1 && type_is_int(kt) && kt != DFGPU_DATE32 && kt != DFGPU_DATE64 && kt != DFGPU_TIMESTAMP;
  // (ArrayMap::is_supported_type, array_map.rs:106-119: Int8..Int64, UInt8..UInt64 only)
  if (am_type_ok && n > 0) {
    bool null_block = false;
    if (j->opt.null_equality == DFGPU_NULL_EQUALS_NULL) {
      // exec.rs:124-131: any NULL build key disables the ArrayMap under NullEqualsNull
      const DCol& kcol = j->build_cols[j->on_build[0]];
      if (kcol.validity && count_set_bits(ctx, kcol.validity, kcol.offset, kcol.length) != kcol.length) null_block = true;
    }
    if (!null_block) {
      DevBuf mm(ctx, 24);
      unsigned long long init[3];
      int sgn = type_is_signed_int(kt) ? 1 : 0;
      if (sgn) { init[0] = (unsigned long long)LLONG_MAX; init[1] = (unsigned long long)LLONG_MIN; } else { init[0] = ~0ull; init[1] = 0; }
      init[2] = 0;
      DF_CUDA(cudaMemcpyAsync(mm.ptr, init, 24, cudaMemcpyHostToDevice, ctx->stream));
      join_minmax_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(j->build_keys, n, sgn, mm.as<unsigned long long>());
      DF_LAUNCH_CHECK(ctx);
      unsigned long long h[3];
      DF_CUDA(cudaMemcpyAsync(h, mm.ptr, 24, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
      if (h[2] > 0) {  // bounds exist only if some key is non-null (exec.rs:140-148)
        uint64_t minv = h[0], maxv = h[1];
        uint64_t range = maxv - minv;  // wrapping_sub, array_map.rs:154
        bool ok = (uint64_t)n < 0xFFFFFFFFull && range != ~0ull;
        if (ok) {
          double dense_ratio = (double)n / ((double)range + 1.0);
          if (range >= (uint64_t)j->opt.perfect_hash_join_small_build_threshold && dense_ratio <= j->opt.perfect_hash_join_min_key_density) ok = false;
        }
        // device memory guard (reservation.try_grow, exec.rs:181-182): at most 16 GiB for the direct array
        if (ok && (range + 1) > (1ull << 31)) ok = false;
        if (ok) {
          j->use_array_map = true;
          j->amap.alloc(ctx, (size_t)(range + 1) * 8);
          j->amap.fill(0xFF);
          j->table.amap = j->amap.as<uint2>();
          j->table.amin = minv;
          j->table.asize = range + 1;
          j->m_array_map = 1;
        }
      }
    }
  }
  // ---- inline-payload attempt ----
  j->inline_ok = false;
  if (n > 0 && !j->has_filter && j->emit_mode == EMIT_PAIRS && !j->need_visited && j->opt.null_equality == DFGPU_NULL_EQUALS_NOTHING && !j->opt.force_hash_collisions &&
      j->out_side.size() <= (size_t)kMaxFusedCols) {
    bool ok = true;
    int bits = 0;
    PayloadCols pc;
    memset(&pc, 0, sizeof(pc));
    j->out_kind.assign(j->out_side.size(), 0); j->out_src.assign(j->out_side.size(), 0); j->out_shift.assign(j->out_side.size(), 0);
    std::vector<int> pay_of_col(j->build_types.size(), -1);
    for (size_t c = 0; c < j->out_side.size() && ok; ++c) {
      const int side = j->out_side[c], ix = j->out_index[c];
      if (side == 2) { ok = false; break; }
      if (side == 1) { j->out_kind[c] = 0; j->out_src[c] = ix; if (j->probe_types[ix] == DFGPU_BOOL) ok = false; continue; }
      // build side: a key column is read from the probe key (exact-tag equality makes them bit-identical)
      int key_pos = -1;
      for (size_t k = 0; k < j->on_build.size(); ++k) if (j->on_build[k] == ix) key_pos = (int)k;
      if (key_pos >= 0 && type_width(j->build_types[ix]) == type_width(j->probe_types[j->on_probe[key_pos]])) { j->out_kind[c] = 0; j->out_src[c] = j->on_probe[key_pos]; continue; }
      const DCol& bc = j->build_cols[ix];
      const int w = type_width(bc.type);
      if (bc.type == DFGPU_BOOL || bc.validity || w < 1 || w > 8) { ok = false; break; }
      if (pay_of_col[ix] < 0) {
        if (pc.n >= kMaxPayloadCols || bits + 8 * w > 64) { ok = false; break; }
        pc.ptr[pc.n] = bc.values; pc.width[pc.n] = w; pc.shift[pc.n] = bits;
        pay_of_col[ix] = bits;
        bits += 8 * w; pc.n++;
      }
      j->out_kind[c] = 1; j->out_shift[c] = pay_of_col[ix];
    }
    if (ok) {
      const int W = pc.n ? 2 : 1;
      const uint64_t cap = j->use_array_map ? j->table.asize : ((std::max<uint64_t>(1024, (uint64_t)n * kInlineSlotsPer100Rows / 100) + 3) & ~3ull);
      j->inline_slots.alloc(ctx, (size_t)cap * 8 * W);
      j->inline_slots.fill(0xFF);
      j->iref.slots = j->inline_slots.ptr; j->iref.cap = cap; j->iref.dense = j->use_array_map ? 1 : 0; j->iref.amin = j->table.amin;
      j->iref.bucket = 0;   // bucket-aligned start slots were a round-1 experiment that only join_probe_inline_kernel honoured (ADVICE r1): retired
      DF_CUDA(cudaMemsetAsync(j->counters.ptr, 0, 64, ctx->stream));
      {
        KernelTimer kt(ctx, "join_build");
        if (W == 2) join_build_inline_kernel<2><<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(j->build_keys, pc, n, j->iref, j->counters.as<unsigned long long>());
        else join_build_inline_kernel<1><<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(j->build_keys, pc, n, j->iref, j->counters.as<unsigned long long>());
        DF_LAUNCH_CHECK(ctx);
      }
      unsigned long long hc[3];
      DF_CUDA(cudaMemcpyAsync(hc, j->counters.ptr, 24, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
      if (hc[2] == 0) {
        if (j->opt.membership_filter && !j->use_array_map && n > 0) {
          // 16 bits per build key, one 64-bit block per 4 keys; probed before the table by the ordered probe kernel
          const uint64_t blocks = std::max<uint64_t>(1024, ((uint64_t)n + 3) / 4);
          j->bloom.alloc(ctx, (size_t)blocks * 8);
          j->bloom.zero();
          KernelTimer kt(ctx, "join_build");
          join_bloom_build_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(j->build_keys, n, j->bloom.as<unsigned long long>(), blocks);
          DF_LAUNCH_CHECK(ctx);
          j->iref.bloom = j->bloom.as<unsigned long long>(); j->iref.bloom_blocks = blocks;
        }
        j->inline_ok = true; j->inline_words = W;
        j->distinct = j->valid_rows = (int64_t)hc[0]; j->null_rows = (int64_t)hc[1];
        j->unique = true;
        j->amap.release();   // the direct {head,cnt} array is not needed
        j->next.release();
        j->built = true;
        return;
      }
      j->inline_slots.release();  // duplicates (or the all-ones key): fall through to the generic chained table
      DF_CUDA(cudaMemsetAsync(j->counters.ptr, 0, 64, ctx->stream));
    }
  }
  if (!j->use_array_map) {
    uint64_t cap = std::max<uint64_t>(1024, (uint64_t)n * 2);
    j->slots.alloc(ctx, (size_t)(cap + 1) * 16);
    j->slots.fill(0xFF);
    j->table.slots = j->slots.as<uint4>();
    j->table.cap = cap;
  }
  if (n > 0) {
    KernelTimer kt(ctx, "join_build");
    join_build_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(j->build_keys, n, j->table, j->counters.as<unsigned long long>());
    DF_LAUNCH_CHECK(ctx);
  }
  unsigned long long hc[3];
  DF_CUDA(cudaMemcpyAsync(hc, j->counters.ptr, 24, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  j->distinct = (int64_t)hc[0];
  j->valid_rows = (int64_t)hc[1];
  j->null_rows = (int64_t)hc[2];
  j->unique = (j->distinct == j->valid_rows);  // map.len() == next.len() fast path, join_hash_map.rs:410-429
  if (j->has_filter && j->need_visited) { j->visited_rows.alloc(ctx, (size_t)((n + 31) / 32 + 1) * 4); j->visited_rows.zero(); }
  j->built = true;
}

static void emit_batch(dfgpu_hashjoin* j, BatchPtr b) {
  j->m_output_rows += b->rows;
  j->m_output_batches++;
  j->outq.push_back(std::move(b));
}

// build_batch_from_indices (utils.rs:1332-1387): one gather per output column
static BatchPtr materialize(dfgpu_hashjoin* j, const std::vector<DCol>* probe_cols, const uint32_t* bidx, const uint32_t* pidx, int64_t n,
                            bool bidx_nullable, bool pidx_all_null, const uint32_t* mark_src) {
  dfgpu_ctx* ctx = j->ctx;
  BatchPtr out(new dfgpu_batch());
  out->ctx = ctx; out->rows = n; out->host = false;
  for (size_t c = 0; c < j->out_side.size(); ++c) {
    int side = j->out_side[c], ix = j->out_index[c];
    if (side == 2) {
      DCol m = alloc_col(ctx, DFGPU_BOOL, n, false);
      if (n) {
        mark_from_idx_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(mark_src, n, m.own_values->as<uint32_t>());
        DF_LAUNCH_CHECK(ctx);
      }
      out->cols.push_back(std::move(m));
    } else if (side == 0) {
      if (!bidx) out->cols.push_back(null_column(ctx, j->build_types[ix], n));
      else out->cols.push_back(take_column(ctx, j->build_cols[ix], bidx, n, bidx_nullable));
    } else {
      if (pidx_all_null || !probe_cols) out->cols.push_back(null_column(ctx, j->probe_types[ix], n));
      else out->cols.push_back(take_column(ctx, (*probe_cols)[ix], pidx, n, false));
    }
  }
  return out;
}

__global__ void scatter_u32_kernel(const uint32_t* __restrict__ pos, int64_t n, uint32_t* __restrict__ dst) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[pos[i]] = 0u;
}
__global__ void mark_bits_kernel(const uint32_t* __restrict__ idx, int64_t n, uint32_t* __restrict__ words) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t r = idx[i];
    atomicOr(&words[r >> 5], 1u << (r & 31));
  }
}

static DCol idx_as_col(const uint32_t* p, int64_t n) {
  DCol d;
  d.type = DFGPU_UINT32; d.length = n; d.values = p; d.null_count = 0;
  return d;
}

// Probe with a JoinFilter: candidate pairs -> filter on the intermediate batch -> join-type handling from the
// surviving pairs (stream.rs:896-948: apply_join_filter_to_indices, then visited bitmap + adjust_indices_by_join_type).
static void push_probe_filtered(dfgpu_hashjoin* j, const std::vector<DCol>& cols, const KeyCols& pk, int64_t n) {
  dfgpu_ctx* ctx = j->ctx;
  const int jt = j->opt.join_type;
  // 1. every candidate pair (equal keys), reference order
  const int64_t ntiles = (n + kProbeTile - 1) / kProbeTile;
  DevBuf head(ctx, (size_t)n * 4), cnt(ctx, (size_t)n * 4), tiles(ctx, (size_t)(ntiles + 1) * 8), hits(ctx, 8);
  hits.zero();
  join_probe_count_kernel<false><<<(int)ntiles, kProbeThreads, 0, ctx->stream>>>(pk, n, j->table, EMIT_PAIRS, 0, head.as<uint32_t>(), cnt.as<uint32_t>(),
                                                                                 tiles.as<uint64_t>(), hits.as<unsigned long long>());
  DF_LAUNCH_CHECK(ctx);
  scan_tiles_kernel<1024><<<1, 1024, 0, ctx->stream>>>(tiles.as<uint64_t>(), ntiles, tiles.as<uint64_t>() + ntiles);
  DF_LAUNCH_CHECK(ctx);
  const int64_t total = (int64_t)read_scalar<uint64_t>(ctx, tiles.as<uint64_t>() + ntiles);
  DevBuf bidx(ctx, (size_t)std::max<int64_t>(total, 1) * 4), pidx(ctx, (size_t)std::max<int64_t>(total, 1) * 4);
  join_emit_kernel<false><<<(int)ntiles, kProbeThreads, 0, ctx->stream>>>(n, head.as<uint32_t>(), cnt.as<uint32_t>(), j->table.next, tiles.as<uint64_t>(), EMIT_PAIRS,
                                                                         bidx.as<uint32_t>(), pidx.as<uint32_t>());
  DF_LAUNCH_CHECK(ctx);
  // 2. the filter's intermediate batch (only the referenced columns are gathered) and its predicate
  DCol fb, fp;  // surviving pairs
  int64_t kept = 0;
  if (total > 0) {
    std::vector<DCol> inter;
    for (size_t c = 0; c < j->filt_side.size(); ++c) {
      inter.push_back(j->filt_side[c] == 0 ? take_column(ctx, j->build_cols[j->filt_index[c]], bidx.as<uint32_t>(), total, false)
                                           : take_column(ctx, cols[j->filt_index[c]], pidx.as<uint32_t>(), total, false));
      if (j->wide && c < 2 * j->wide_on_build.size()) inter.back().type = wide_key_eq_type(inter.back().type);   // planned by check_join_keys
    }
    EvalResult ev = evaluate_expr(ctx, j->filt_plan, inter, total, false, true);
    DevBuf sel;
    kept = compact_flag_indices(ctx, ev.select_words.as<uint32_t>(), total, 1, &sel);
    if (kept > 0) {
      fb = take_column(ctx, idx_as_col(bidx.as<uint32_t>(), total), sel.as<uint32_t>(), kept, false);
      fp = take_column(ctx, idx_as_col(pidx.as<uint32_t>(), total), sel.as<uint32_t>(), kept, false);
    }
  }
  const uint32_t* fbp = kept ? (const uint32_t*)fb.values : nullptr;
  const uint32_t* fpp = kept ? (const uint32_t*)fp.values : nullptr;
  // 3. visited build rows (Left / Full / LeftSemi / LeftAnti / LeftMark)
  if (j->need_visited && kept > 0) {
    mark_bits_kernel<<<grid_for(kept, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(fbp, kept, j->visited_rows.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
  }
  // 4. probe rows that kept at least one pair
  DevBuf pm(ctx, (size_t)((n + 31) / 32) * 4);
  pm.zero();
  if (kept > 0) {
    mark_bits_kernel<<<grid_for(kept, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(fpp, kept, pm.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
  }
  j->m_probe_hits += count_set_bits(ctx, pm.as<uint8_t>(), 0, n);
  BatchPtr out;
  switch (jt) {
    case DFGPU_JOIN_INNER: case DFGPU_JOIN_LEFT:
      if (kept) out = materialize(j, &cols, fbp, fpp, kept, false, false, nullptr);
      break;
    case DFGPU_JOIN_RIGHT: case DFGPU_JOIN_FULL: {
      // matched pairs, then the unmatched probe rows of this batch (append_right_indices, utils.rs:1509-1570)
      DevBuf un;
      const int64_t nun = compact_flag_indices(ctx, pm.as<uint32_t>(), n, 0, &un);
      const int64_t tot2 = kept + nun;
      if (tot2 == 0) break;
      DevBuf b2(ctx, (size_t)tot2 * 4), p2(ctx, (size_t)tot2 * 4);
      if (kept) {
        DF_CUDA(cudaMemcpyAsync(b2.ptr, fbp, (size_t)kept * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        DF_CUDA(cudaMemcpyAsync(p2.ptr, fpp, (size_t)kept * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      }
      if (nun) {
        DF_CUDA(cudaMemsetAsync((char*)b2.ptr + (size_t)kept * 4, 0xFF, (size_t)nun * 4, ctx->stream));  // NULL build index
        DF_CUDA(cudaMemcpyAsync((char*)p2.ptr + (size_t)kept * 4, un.ptr, (size_t)nun * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      }
      out = materialize(j, &cols, b2.as<uint32_t>(), p2.as<uint32_t>(), tot2, true, false, nullptr);
      break;
    }
    case DFGPU_JOIN_RIGHT_SEMI: case DFGPU_JOIN_RIGHT_ANTI: {
      DevBuf sel;
      const int64_t ns = compact_flag_indices(ctx, pm.as<uint32_t>(), n, jt == DFGPU_JOIN_RIGHT_SEMI ? 1 : 0, &sel);
      if (ns) out = materialize(j, &cols, nullptr, sel.as<uint32_t>(), ns, true, false, nullptr);
      break;
    }
    case DFGPU_JOIN_RIGHT_MARK: {
      DevBuf all(ctx, (size_t)n * 4), markidx(ctx, (size_t)n * 4);
      fill_iota(ctx, all.as<uint32_t>(), n);
      // mark source: an index array whose NULL marker encodes "no surviving pair"
      DF_CUDA(cudaMemsetAsync(markidx.ptr, 0xFF, (size_t)n * 4, ctx->stream));
      if (kept) {
        DevBuf msel;
        const int64_t nm = compact_flag_indices(ctx, pm.as<uint32_t>(), n, 1, &msel);
        // scatter 0 into the matched positions
        if (nm) {
          DCol zeros = alloc_col(ctx, DFGPU_UINT32, nm, false);
          zeros.own_values->zero();
          scatter_u32_kernel<<<grid_for(nm, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(msel.as<uint32_t>(), nm, markidx.as<uint32_t>());
          DF_LAUNCH_CHECK(ctx);
        }
      }
      out = materialize(j, &cols, nullptr, all.as<uint32_t>(), n, true, false, markidx.as<uint32_t>());
      break;
    }
    default: break;  // LeftSemi / LeftAnti / LeftMark: produced by finish_probe from visited_rows
  }
  if (out && out->rows > 0) emit_batch(j, std::move(out));
}

static void push_probe(dfgpu_hashjoin* j, std::vector<DCol>&& cols) {
  DF_CHECK(j->built, DFGPU_ERR_STATE, "push_probe before finish_build");
  DF_CHECK(!j->probe_done, DFGPU_ERR_STATE, "push_probe after finish_probe");
  if (j->wide && cols.size() + 1 == j->probe_types.size()) cols.push_back(wide_key_column(j, cols, j->wide_on_probe));
  DF_CHECK(cols.size() == j->probe_types.size(), DFGPU_ERR_INVALID, "probe batch column count mismatch");
  dfgpu_ctx* ctx = j->ctx;
  set_device(ctx);
  int64_t n = cols.empty() ? 0 : cols[0].length;
  for (size_t c = 0; c < cols.size(); ++c) {
    DF_CHECK(cols[c].type == j->probe_types[c], DFGPU_ERR_INVALID, "probe batch column type mismatch");
    DF_CHECK(cols[c].length == n, DFGPU_ERR_INVALID, "probe batch ragged columns");
  }
  DF_CHECK(n < (int64_t)kEmpty32, DFGPU_ERR_UNSUPPORTED, "hash join: a probe batch must have < 2^32-1 rows");
  j->m_input_rows += n;
  j->m_input_batches++;
  if (n == 0) return;
  j->probe_side_non_empty = true;
  if (j->opt.null_aware) {   // NOT IN semantics (stream.rs:755-806, 937-956)
    const DCol& kcol = cols[j->on_probe[0]];
    const bool key_has_null = kcol.validity && count_set_bits(ctx, kcol.validity, kcol.offset, n) != n;
    if (j->opt.join_type == DFGPU_JOIN_LEFT_ANTI) {
      if (key_has_null) j->probe_has_null = true;   // a NULL in the subquery: NOT IN is never TRUE, nothing is output
      if (j->probe_has_null) return;
    } else {  // RightAnti
      if (j->null_rows > 0) return;                 // build side has a NULL key: no probe row qualifies
      if (key_has_null && j->nB > 0) {              // NULL probe keys are not emitted (an empty build side emits every row)
        const int64_t nw = (n + 31) / 32;
        DevBuf bits(ctx, (size_t)(nw + 1) * 4);
        bits.zero();
        bitmap_or_copy(ctx, bits.as<uint8_t>(), 0, kcol.validity, kcol.offset, n);
        DevBuf idx;
        const int64_t keep = compact_flag_indices(ctx, bits.as<uint32_t>(), n, 1, &idx);
        j->m_input_rows -= n; j->m_input_batches--;
        if (keep == 0) { j->m_input_rows += n; j->m_input_batches++; return; }
        std::vector<DCol> kept;
        for (size_t c = 0; c < cols.size(); ++c) {
          DCol t = take_column(ctx, cols[c], idx.as<uint32_t>(), keep, false);
          if ((int)c == j->on_probe[0]) { t.validity = nullptr; t.null_count = 0; t.own_validity.reset(); }   // every kept key is valid
          kept.push_back(std::move(t));
        }
        push_probe(j, std::move(kept));
        j->m_input_rows += n - keep;
        return;
      }
    }
  }
  const int mode = j->emit_mode;
  // empty / unmatchable build side: build_batch_empty_build_side (utils.rs:1393-1430)
  KeyCols pk;
  make_keycols(cols, j->on_probe, &pk);
  // ---- inline-payload path ----
  if (j->inline_ok) {
    InlineOut oc;
    memset(&oc, 0, sizeof(oc));
    oc.n = (int)j->out_side.size();
    BatchPtr out(new dfgpu_batch());
    out->ctx = ctx; out->host = false;
    out->cols.resize(oc.n);
    bool need_pidx = false;
    for (int c = 0; c < oc.n; ++c) {
      const int otype = j->out_side[c] == 0 ? j->build_types[j->out_index[c]] : j->probe_types[j->out_index[c]];
      oc.kind[c] = j->out_kind[c]; oc.width[c] = type_width(otype); oc.shift[c] = j->out_shift[c];
      if (j->out_kind[c] == 0 && (cols[j->out_src[c]].validity || otype == DFGPU_BOOL)) { oc.kind[c] = 2; need_pidx = true; continue; }  // gathered afterwards
      DCol d = alloc_col(ctx, otype, n, false);
      oc.dst[c] = d.own_values->ptr;
      oc.src[c] = j->out_kind[c] == 0 ? cols[j->out_src[c]].values : nullptr;
      out->cols[c] = std::move(d);
    }
    // ---- radix-partitioned probe (row order not required, table several times the L2): radix_probe.cuh ----
    {
      const size_t tbytes = (size_t)j->iref.cap * 8 * j->inline_words;
      const int force_parts = getenv("DFGPU_JOIN_RADIX_PARTS") ? atoi(getenv("DFGPU_JOIN_RADIX_PARTS")) : 0;   // tests force the path on small inputs
      bool radix = !j->opt.ordered_output && !j->iref.dense && !j->iref.bucket && !need_pidx && pk.n == 1 && pk.width[0] == 8 && !pk.valid[0] &&
                   ((uintptr_t)pk.ptr[0] % 16 == 0) && ((tbytes > (size_t)40 << 20 && n >= (1ll << 22)) || force_parts >= 2);
      // every probe-side output column must be the key column or ONE other plain 8-byte column (it rides in the 16-byte record)
      int carry = -1;
      RadixOut ro;
      memset(&ro, 0, sizeof(ro));
      ro.n = oc.n;
      for (int c = 0; c < oc.n && radix; ++c) {
        ro.width[c] = oc.width[c]; ro.dst[c] = oc.dst[c]; ro.shift[c] = oc.shift[c];
        if (oc.kind[c] == 1) { ro.kind[c] = 2; continue; }
        const int src = j->out_src[c];
        if (src == j->on_probe[0]) { ro.kind[c] = 0; continue; }
        if (type_width(cols[src].type) != 8 || ((uintptr_t)cols[src].values % 16 != 0) || (carry >= 0 && carry != src)) { radix = false; break; }
        carry = src; ro.kind[c] = 1;
      }
      if (radix) {
        const unsigned long long* keys = (const unsigned long long*)pk.ptr[0];
        const unsigned long long* vals = carry >= 0 ? (const unsigned long long*)cols[carry].values : keys;
        DevBuf recs(ctx, (size_t)n * 16), meta(ctx, (size_t)(kRadixMetaWords + 2) * 8);
        meta.zero();
        unsigned long long* rtot = meta.as<unsigned long long>() + kRadixMetaWords;    // output rows
        unsigned int* rtile = (unsigned int*)(rtot + 1);
        {
          KernelTimer kt(ctx, "radix_partition");
          radix_partition(ctx, keys, vals, n, tbytes, force_parts, recs.ptr, meta.as<unsigned long long>());
        }
        {
          KernelTimer kt(ctx, "join_probe");
          bool all8 = true;
          for (int c = 0; c < ro.n; ++c) all8 = all8 && ro.width[c] == 8;
          if (j->inline_words == 2) {
            if (all8) radix_probe_kernel<2, true><<<kNumSMs * 8, 256, 0, ctx->stream>>>(recs.as<RadixRec>(), n, j->iref, ro, rtile, rtot);
            else radix_probe_kernel<2, false><<<kNumSMs * 8, 256, 0, ctx->stream>>>(recs.as<RadixRec>(), n, j->iref, ro, rtile, rtot);
          } else {
            if (all8) radix_probe_kernel<1, true><<<kNumSMs * 8, 256, 0, ctx->stream>>>(recs.as<RadixRec>(), n, j->iref, ro, rtile, rtot);
            else radix_probe_kernel<1, false><<<kNumSMs * 8, 256, 0, ctx->stream>>>(recs.as<RadixRec>(), n, j->iref, ro, rtile, rtot);
          }
          DF_LAUNCH_CHECK(ctx);
        }
        unsigned long long hrows = 0;
        DF_CUDA(cudaMemcpyAsync(&hrows, rtot, 8, cudaMemcpyDeviceToHost, ctx->stream));
        DF_CUDA(cudaStreamSynchronize(ctx->stream));
        out->rows = (int64_t)hrows;
        for (int c = 0; c < oc.n; ++c) out->cols[c].length = out->rows;
        j->m_probe_hits += (int64_t)hrows;
        j->m_radix_probes++;
        if (out->rows > 0) emit_batch(j, std::move(out));
        return;
      }
    }
    DevBuf pidx;
    if (need_pidx) { pidx.alloc(ctx, (size_t)n * 4); oc.pidx_out = pidx.as<uint32_t>(); }
    const int64_t nt = (n + kFusedTile - 1) / kFusedTile;
    DevBuf desc(ctx, (size_t)nt * 8 + 32);
    desc.zero();
    unsigned long long* totals = (unsigned long long*)((char*)desc.ptr + (size_t)nt * 8);
    unsigned int* counter = (unsigned int*)(totals + 2);
    {
      KernelTimer kt(ctx, "join_probe");
      if (j->iref.bloom) {
        if (j->inline_words == 2) join_probe_inline_kernel<2, true><<<(int)nt, kFusedThreads, 0, ctx->stream>>>(pk, n, j->iref, oc, desc.as<unsigned long long>(), counter, totals);
        else join_probe_inline_kernel<1, true><<<(int)nt, kFusedThreads, 0, ctx->stream>>>(pk, n, j->iref, oc, desc.as<unsigned long long>(), counter, totals);
      } else {
        if (j->inline_words == 2) join_probe_inline_kernel<2, false><<<(int)nt, kFusedThreads, 0, ctx->stream>>>(pk, n, j->iref, oc, desc.as<unsigned long long>(), counter, totals);
        else join_probe_inline_kernel<1, false><<<(int)nt, kFusedThreads, 0, ctx->stream>>>(pk, n, j->iref, oc, desc.as<unsigned long long>(), counter, totals);
      }
      DF_LAUNCH_CHECK(ctx);
    }
    unsigned long long h[2];
    DF_CUDA(cudaMemcpyAsync(h, totals, 16, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    out->rows = (int64_t)h[0];
    for (int c = 0; c < oc.n; ++c) {
      if (oc.kind[c] == 2) out->cols[c] = take_column(ctx, cols[j->out_src[c]], pidx.as<uint32_t>(), out->rows, false);
      else out->cols[c].length = out->rows;
    }
    j->m_probe_hits += (int64_t)h[1];
    if (out->rows > 0) emit_batch(j, std::move(out));
    return;
  }
  // ---- fused single-pass path: unique build keys, one output row per matching probe row, plain columns ----
  if (j->has_filter) { push_probe_filtered(j, cols, pk, n); return; }
  if (mode == EMIT_PAIRS && j->unique && !j->opt.force_hash_collisions && j->out_side.size() <= (size_t)kMaxFusedCols) {
    bool plain = true;
    for (size_t c = 0; c < j->out_side.size() && plain; ++c) {
      const DCol& src = j->out_side[c] == 0 ? j->build_cols[j->out_index[c]] : (j->out_side[c] == 1 ? cols[j->out_index[c]] : cols[0]);
      if (j->out_side[c] == 2 || src.type == DFGPU_BOOL || src.validity) plain = false;
    }
    if (plain) {
      FusedCols oc;
      memset(&oc, 0, sizeof(oc));
      oc.n = (int)j->out_side.size();
      BatchPtr out(new dfgpu_batch());
      out->ctx = ctx; out->host = false;
      for (int c = 0; c < oc.n; ++c) {
        const DCol& src = j->out_side[c] == 0 ? j->build_cols[j->out_index[c]] : cols[j->out_index[c]];
        DCol d = alloc_col(ctx, src.type, n, false);  // unique build: at most one output row per probe row
        oc.src[c] = src.values; oc.dst[c] = d.own_values->ptr; oc.width[c] = type_width(src.type); oc.side[c] = j->out_side[c];
        out->cols.push_back(std::move(d));
      }
      const int64_t nt = (n + kFusedTile - 1) / kFusedTile;
      DevBuf desc(ctx, (size_t)nt * 8 + 32);
      desc.zero();
      unsigned long long* totals = (unsigned long long*)((char*)desc.ptr + (size_t)nt * 8);
      unsigned int* counter = (unsigned int*)(totals + 2);
      {
        KernelTimer kt(ctx, "join_probe");
        join_probe_fused_kernel<<<(int)nt, kFusedThreads, 0, ctx->stream>>>(pk, n, j->table, j->need_visited ? 1 : 0, oc, desc.as<unsigned long long>(), counter, totals);
        DF_LAUNCH_CHECK(ctx);
      }
      unsigned long long h[2];
      DF_CUDA(cudaMemcpyAsync(h, totals, 16, cudaMemcpyDeviceToHost, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));
      out->rows = (int64_t)h[0];
      for (auto& c : out->cols) c.length = out->rows;
      j->m_probe_hits += (int64_t)h[1];
      if (out->rows > 0) emit_batch(j, std::move(out));
      return;
    }
  }
  const int64_t ntiles = (n + kProbeTile - 1) / kProbeTile;
  DevBuf head(ctx, (size_t)n * 4), cnt, tiles(ctx, (size_t)(ntiles + 1) * 8), hits(ctx, 8);
  hits.zero();
  if (!j->unique) cnt.alloc(ctx, (size_t)n * 4);
  KernelTimer* ktp = new KernelTimer(ctx, "join_probe");
  if (j->unique)
    join_probe_count_kernel<true><<<(int)ntiles, kProbeThreads, 0, ctx->stream>>>(pk, n, j->table, mode, j->need_visited ? 1 : 0, head.as<uint32_t>(), nullptr,
                                                                                  tiles.as<uint64_t>(), hits.as<unsigned long long>());
  else
    join_probe_count_kernel<false><<<(int)ntiles, kProbeThreads, 0, ctx->stream>>>(pk, n, j->table, mode, j->need_visited ? 1 : 0, head.as<uint32_t>(), cnt.as<uint32_t>(),
                                                                                   tiles.as<uint64_t>(), hits.as<unsigned long long>());
  DF_LAUNCH_CHECK(ctx);
  delete ktp;
  if (mode == EMIT_NONE) {
    j->m_probe_hits += (int64_t)read_scalar<unsigned long long>(ctx, hits.as<unsigned long long>());
    return;
  }
  scan_tiles_kernel<1024><<<1, 1024, 0, ctx->stream>>>(tiles.as<uint64_t>(), ntiles, tiles.as<uint64_t>() + ntiles);
  DF_LAUNCH_CHECK(ctx);
  uint64_t total = read_scalar<uint64_t>(ctx, tiles.as<uint64_t>() + ntiles);
  DF_CHECK(total < (uint64_t)kEmpty32 * 64ull, DFGPU_ERR_OOM, "hash join: output of one probe batch too large");
  const bool need_bidx = (mode == EMIT_PAIRS || mode == EMIT_PAIRS_OUTER || mode == EMIT_ALL);
  DevBuf bidx, pidx(ctx, (size_t)std::max<uint64_t>(total, 1) * 4);
  if (need_bidx) bidx.alloc(ctx, (size_t)std::max<uint64_t>(total, 1) * 4);
  if (j->unique)
    join_emit_kernel<true><<<(int)ntiles, kProbeThreads, 0, ctx->stream>>>(n, head.as<uint32_t>(), nullptr, j->table.next, tiles.as<uint64_t>(), mode,
                                                                          need_bidx ? bidx.as<uint32_t>() : nullptr, pidx.as<uint32_t>());
  else
    join_emit_kernel<false><<<(int)ntiles, kProbeThreads, 0, ctx->stream>>>(n, head.as<uint32_t>(), cnt.as<uint32_t>(), j->table.next, tiles.as<uint64_t>(), mode,
                                                                           need_bidx ? bidx.as<uint32_t>() : nullptr, pidx.as<uint32_t>());
  DF_LAUNCH_CHECK(ctx);
  BatchPtr out;
  if (mode == EMIT_PAIRS)
    out = materialize(j, &cols, bidx.as<uint32_t>(), pidx.as<uint32_t>(), (int64_t)total, false, false, nullptr);
  else if (mode == EMIT_PAIRS_OUTER)
    out = materialize(j, &cols, bidx.as<uint32_t>(), pidx.as<uint32_t>(), (int64_t)total, true, false, nullptr);
  else if (mode == EMIT_ALL)  // RightMark: build_batch and probe_batch swap roles (stream.rs:953-958); mark = is_not_null(match)
    out = materialize(j, &cols, nullptr, pidx.as<uint32_t>(), (int64_t)total, true, false, bidx.as<uint32_t>());
  else  // RightSemi / RightAnti: probe columns only
    out = materialize(j, &cols, nullptr, pidx.as<uint32_t>(), (int64_t)total, true, false, nullptr);
  j->m_probe_hits += (int64_t)read_scalar<unsigned long long>(ctx, hits.as<unsigned long long>());
  if (out->rows > 0) emit_batch(j, std::move(out));
}

// ------------------------------------------------------------------------------------------
// pipelined host probe (inline table): the probe batch is cut into chunks; H2D of chunk i+1, the probe kernel
// of chunk i and D2H of chunk i-1 run on three streams, so the PCIe link is busy in both directions while the
// kernels run (the host entry point is PCIe-bound: 1.6 GB in + 2.4 GB out per C2 probe side vs a few ms of kernels).
// Output rows land at consecutive offsets of ONE pinned host batch, in probe order.
// ------------------------------------------------------------------------------------------
static bool push_probe_host_pipelined(dfgpu_hashjoin* j, const dfgpu_column* hcols, int32_t n_cols) {
  if (!j->inline_ok || n_cols != (int)j->probe_types.size()) return false;
  const int64_t n = n_cols ? hcols[0].length : 0;
  constexpr int64_t kChunk = 8ll << 20;
  if (n < 2 * kChunk) return false;  // small batches: the simple path
  for (int c = 0; c < n_cols; ++c) {
    if (hcols[c].type != j->probe_types[c] || hcols[c].length != n) return false;
    if (hcols[c].validity && hcols[c].null_count != 0) return false;
    if (hcols[c].type == DFGPU_BOOL) return false;
  }
  dfgpu_ctx* ctx = j->ctx;
  set_device(ctx);
  if (!ctx->copy_in) { DF_CUDA(cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking)); DF_CUDA(cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking)); }
  const int nout = (int)j->out_side.size();
  const int64_t nchunks = (n + kChunk - 1) / kChunk;
  // which probe columns are actually needed on the device (keys + gathered outputs)
  std::vector<bool> need(n_cols, false);
  for (int c : j->on_probe) need[c] = true;
  for (int c = 0; c < nout; ++c) if (j->out_kind[c] == 0) need[j->out_src[c]] = true;
  // double-buffered device staging
  std::vector<std::vector<DevBuf>> din(2), dout(2);
  std::vector<DevBuf> desc(2);
  const int64_t nt = (kChunk + kFusedTile - 1) / kFusedTile;
  for (int b = 0; b < 2; ++b) {
    din[b].resize(n_cols); dout[b].resize(nout);
    for (int c = 0; c < n_cols; ++c) if (need[c]) din[b][c].alloc(ctx, (size_t)kChunk * type_width(j->probe_types[c]));
    for (int c = 0; c < nout; ++c) {
      const int otype = j->out_side[c] == 0 ? j->build_types[j->out_index[c]] : j->probe_types[j->out_index[c]];
      dout[b][c].alloc(ctx, (size_t)kChunk * type_width(otype));
    }
    desc[b].alloc(ctx, (size_t)nt * 8 + 32);
  }
  // the host result batch (capacity n rows: unique build keys => at most one output row per probe row)
  BatchPtr hb(new dfgpu_batch());
  hb->ctx = ctx; hb->host = true;
  std::vector<int> owidth(nout);
  for (int c = 0; c < nout; ++c) {
    const int otype = j->out_side[c] == 0 ? j->build_types[j->out_index[c]] : j->probe_types[j->out_index[c]];
    owidth[c] = type_width(otype);
    HCol h;
    h.type = otype; h.null_count = 0;
    h.values = std::make_shared<HostBuf>((size_t)std::max<int64_t>(n, 1) * owidth[c]);
    hb->hcols.push_back(std::move(h));
  }
  HostBuf totals_host((size_t)nchunks * 16);
  std::vector<cudaEvent_t> ev_in(nchunks), ev_k(nchunks), ev_out(nchunks);
  for (int64_t i = 0; i < nchunks; ++i) { DF_CUDA(cudaEventCreateWithFlags(&ev_in[i], cudaEventDisableTiming)); DF_CUDA(cudaEventCreateWithFlags(&ev_k[i], cudaEventDisableTiming)); DF_CUDA(cudaEventCreateWithFlags(&ev_out[i], cudaEventDisableTiming)); }
  cudaEvent_t ev_ready;
  DF_CUDA(cudaEventCreateWithFlags(&ev_ready, cudaEventDisableTiming));
  DF_CUDA(cudaEventRecord(ev_ready, ctx->stream));  // build finished + staging allocated
  DF_CUDA(cudaStreamWaitEvent(ctx->copy_in, ev_ready, 0));
  DF_CUDA(cudaStreamWaitEvent(ctx->copy_out, ev_ready, 0));
  auto issue_h2d = [&](int64_t i) {
    const int b = (int)(i & 1);
    const int64_t r0 = i * kChunk, len = std::min<int64_t>(kChunk, n - r0);
    if (i >= 2) DF_CUDA(cudaStreamWaitEvent(ctx->copy_in, ev_k[i - 2], 0));  // staging buffer b consumed by chunk i-2's kernel
    for (int c = 0; c < n_cols; ++c) {
      if (!need[c]) continue;
      const int w = type_width(j->probe_types[c]);
      DF_CUDA(cudaMemcpyAsync(din[b][c].ptr, (const char*)hcols[c].values + (hcols[c].offset + r0) * w, (size_t)len * w, cudaMemcpyHostToDevice, ctx->copy_in));
    }
    DF_CUDA(cudaEventRecord(ev_in[i], ctx->copy_in));
  };
  int64_t out_rows = 0, hits = 0;
  issue_h2d(0);
  for (int64_t i = 0; i < nchunks; ++i) {
    const int b = (int)(i & 1);
    const int64_t r0 = i * kChunk, len = std::min<int64_t>(kChunk, n - r0);
    if (i + 1 < nchunks) issue_h2d(i + 1);
    DF_CUDA(cudaStreamWaitEvent(ctx->stream, ev_in[i], 0));
    if (i >= 2) DF_CUDA(cudaStreamWaitEvent(ctx->stream, ev_out[i - 2], 0));  // output staging b drained by chunk i-2's D2H
    std::vector<DCol> cols(n_cols);
    for (int c = 0; c < n_cols; ++c) { cols[c].type = j->probe_types[c]; cols[c].length = len; cols[c].values = din[b][c].ptr; }
    KeyCols pk;
    make_keycols(cols, j->on_probe, &pk);
    InlineOut oc;
    memset(&oc, 0, sizeof(oc));
    oc.n = nout;
    for (int c = 0; c < nout; ++c) {
      oc.kind[c] = j->out_kind[c]; oc.width[c] = owidth[c]; oc.shift[c] = j->out_shift[c]; oc.dst[c] = dout[b][c].ptr;
      oc.src[c] = j->out_kind[c] == 0 ? din[b][j->out_src[c]].ptr : nullptr;
    }
    DF_CUDA(cudaMemsetAsync(desc[b].ptr, 0, desc[b].bytes, ctx->stream));
    const int64_t ntl = (len + kFusedTile - 1) / kFusedTile;
    unsigned long long* totals = (unsigned long long*)((char*)desc[b].ptr + (size_t)nt * 8);
    unsigned int* counter = (unsigned int*)(totals + 2);
    {
      KernelTimer kt(ctx, "join_probe");
      if (j->inline_words == 2) join_probe_inline_staged_kernel<2><<<(int)ntl, kFusedThreads, 0, ctx->stream>>>(pk, len, j->iref, oc, desc[b].as<unsigned long long>(), counter, totals);
      else join_probe_inline_staged_kernel<1><<<(int)ntl, kFusedThreads, 0, ctx->stream>>>(pk, len, j->iref, oc, desc[b].as<unsigned long long>(), counter, totals);
      DF_LAUNCH_CHECK(ctx);
    }
    DF_CUDA(cudaMemcpyAsync((char*)totals_host.ptr + i * 16, totals, 16, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaEventRecord(ev_k[i], ctx->stream));
    DF_CUDA(cudaEventSynchronize(ev_k[i]));  // the chunk's output row count decides where its rows land on the host
    const unsigned long long* th = (const unsigned long long*)((char*)totals_host.ptr + i * 16);
    const int64_t rows = (int64_t)th[0];
    hits += (int64_t)th[1];
    for (int c = 0; c < nout; ++c)
      if (rows) DF_CUDA(cudaMemcpyAsync((char*)hb->hcols[c].values->ptr + (size_t)out_rows * owidth[c], dout[b][c].ptr, (size_t)rows * owidth[c], cudaMemcpyDeviceToHost, ctx->copy_out));
    DF_CUDA(cudaEventRecord(ev_out[i], ctx->copy_out));
    out_rows += rows;
  }
  DF_CUDA(cudaStreamSynchronize(ctx->copy_out));
  DF_CUDA(cudaStreamSynchronize(ctx->copy_in));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int64_t i = 0; i < nchunks; ++i) { cudaEventDestroy(ev_in[i]); cudaEventDestroy(ev_k[i]); cudaEventDestroy(ev_out[i]); }
  cudaEventDestroy(ev_ready);
  hb->rows = out_rows;
  for (auto& h : hb->hcols) h.length = out_rows;
  j->m_input_rows += n;
  j->m_input_batches++;
  j->m_probe_hits += hits;
  j->m_pipelined_probes++;
  j->probe_side_non_empty = true;
  if (out_rows > 0) emit_batch(j, std::move(hb));
  return true;
}

static void finish_probe(dfgpu_hashjoin* j) {
  DF_CHECK(j->built, DFGPU_ERR_STATE, "finish_probe before finish_build");
  DF_CHECK(!j->probe_done, DFGPU_ERR_STATE, "finish_probe called twice");
  j->probe_done = true;
  dfgpu_ctx* ctx = j->ctx;
  set_device(ctx);
  const int jt = j->opt.join_type;
  // need_produce_result_in_final (utils.rs:1181-1190)
  if (!(jt == DFGPU_JOIN_LEFT || jt == DFGPU_JOIN_FULL || jt == DFGPU_JOIN_LEFT_SEMI || jt == DFGPU_JOIN_LEFT_ANTI || jt == DFGPU_JOIN_LEFT_MARK)) return;
  const int64_t n = j->nB;
  if (n == 0) return;
  // get_final_indices_from_bit_map (utils.rs:1210-1245)
  int64_t nw = (n + 31) / 32;
  DevBuf vis(ctx, (size_t)nw * 4);
  if (j->has_filter) {
    DF_CUDA(cudaMemcpyAsync(vis.ptr, j->visited_rows.ptr, (size_t)nw * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  } else {
    join_build_flags_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(j->build_keys, n, j->table, vis.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
  }
  if (j->opt.null_aware && jt == DFGPU_JOIN_LEFT_ANTI) {   // stream.rs:1016-1072
    if (j->probe_has_null) return;
    const DCol& k = j->build_cols[j->on_build[0]];
    if (j->probe_side_non_empty && k.validity) {   // NULL NOT IN (non-empty) is never TRUE; NULL NOT IN (empty) is
      mark_null_keys_kernel<<<grid_for(nw, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(k.validity, k.offset, n, vis.as<uint32_t>());
      DF_LAUNCH_CHECK(ctx);
    }
  }
  if (jt == DFGPU_JOIN_LEFT_MARK) {
    // all build rows + mark column (visited)
    DevBuf all(ctx, (size_t)n * 4);
    fill_iota(ctx, all.as<uint32_t>(), n);
    BatchPtr out(new dfgpu_batch());
    out->ctx = ctx; out->rows = n; out->host = false;
    for (size_t c = 0; c < j->out_side.size(); ++c) {
      int side = j->out_side[c], ix = j->out_index[c];
      if (side == 2) {
        DCol m = alloc_col(ctx, DFGPU_BOOL, n, false);
        DF_CUDA(cudaMemcpyAsync(m.own_values->ptr, vis.ptr, (size_t)nw * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        out->cols.push_back(std::move(m));
      } else if (side == 0) out->cols.push_back(take_column(ctx, j->build_cols[ix], all.as<uint32_t>(), n, false));
      else out->cols.push_back(null_column(ctx, j->probe_types[ix], n));
    }
    emit_batch(j, std::move(out));
    return;
  }
  const int want_set = (jt == DFGPU_JOIN_LEFT_SEMI) ? 1 : 0;
  DevBuf idx;
  int64_t total = compact_flag_indices(ctx, vis.as<uint32_t>(), n, want_set, &idx);
  if (total == 0) return;
  BatchPtr out = materialize(j, nullptr, idx.as<uint32_t>(), nullptr, (int64_t)total, false, true, nullptr);
  emit_batch(j, std::move(out));
}

}  // namespace dfgpu

// ==========================================================================================
// extern "C"
// ==========================================================================================

extern "C" {

void dfgpu_hashjoin_default_options(dfgpu_hashjoin_options* o) {
  memset(o, 0, sizeof(*o));
  o->join_type = DFGPU_JOIN_INNER;
  o->null_equality = DFGPU_NULL_EQUALS_NOTHING;
  o->batch_size = 8192;
  o->perfect_hash_join_small_build_threshold = 1024;  // config.rs:913
  o->perfect_hash_join_min_key_density = 0.15;        // config.rs:923
  o->force_hash_collisions = 0;
  o->ordered_output = 1;
}

int dfgpu_hashjoin_create(dfgpu_ctx* ctx, const int32_t* build_types, int32_t n_build_cols, const int32_t* probe_types, int32_t n_probe_cols,
                          const int32_t* on_build, const int32_t* on_probe, int32_t n_on, const int32_t* out_side, const int32_t* out_index,
                          int32_t n_out, const dfgpu_hashjoin_options* opts, dfgpu_hashjoin** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && out && opts, DFGPU_ERR_INVALID, "null argument");
  if (opts->null_aware) {   // HashJoinExecBuilder validation, exec.rs:429-455
    DF_CHECK(opts->join_type == DFGPU_JOIN_LEFT_ANTI || opts->join_type == DFGPU_JOIN_RIGHT_ANTI, DFGPU_ERR_INVALID,
             "null_aware can only be true for LeftAnti joins and RightAnti joins with `CollectLeft` `PartitionMode`");
    DF_CHECK(n_on == 1, DFGPU_ERR_INVALID, "null_aware anti join only supports single column join key");
  }
  std::unique_ptr<dfgpu_hashjoin> j(new dfgpu_hashjoin());
  j->ctx = ctx;
  j->opt = *opts;
  j->build_types.assign(build_types, build_types + n_build_cols);
  j->probe_types.assign(probe_types, probe_types + n_probe_cols);
  j->on_build.assign(on_build, on_build + n_on);
  j->on_probe.assign(on_probe, on_probe + n_on);
  j->out_side.assign(out_side, out_side + n_out);
  j->out_index.assign(out_index, out_index + n_out);
  for (int c = 0; c < n_on; ++c) {
    DF_CHECK(on_build[c] >= 0 && on_build[c] < n_build_cols && on_probe[c] >= 0 && on_probe[c] < n_probe_cols, DFGPU_ERR_INVALID, "join key column index out of range");
  }
  for (int c = 0; c < n_out; ++c) {
    int lim = out_side[c] == 0 ? n_build_cols : out_side[c] == 1 ? n_probe_cols : 1;
    DF_CHECK(out_side[c] >= 0 && out_side[c] <= 2 && out_index[c] >= 0 && out_index[c] < lim, DFGPU_ERR_INVALID, "output column mapping out of range");
  }
  check_join_keys(j.get());
  switch (opts->join_type) {
    case DFGPU_JOIN_INNER: j->emit_mode = EMIT_PAIRS; break;
    case DFGPU_JOIN_LEFT: j->emit_mode = EMIT_PAIRS; j->need_visited = true; break;
    case DFGPU_JOIN_RIGHT: j->emit_mode = EMIT_PAIRS_OUTER; break;
    case DFGPU_JOIN_FULL: j->emit_mode = EMIT_PAIRS_OUTER; j->need_visited = true; break;
    case DFGPU_JOIN_RIGHT_SEMI: j->emit_mode = EMIT_SEMI; break;
    case DFGPU_JOIN_RIGHT_ANTI: j->emit_mode = EMIT_ANTI; break;
    case DFGPU_JOIN_RIGHT_MARK: j->emit_mode = EMIT_ALL; break;
    case DFGPU_JOIN_LEFT_SEMI: case DFGPU_JOIN_LEFT_ANTI: case DFGPU_JOIN_LEFT_MARK: j->emit_mode = EMIT_NONE; j->need_visited = true; break;
    default: throw Error(DFGPU_ERR_INVALID, "unknown join type");
  }
  *out = j.release();
  DF_API_END
}

static std::vector<DCol> host_cols_to_device(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n) {
  set_device(ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n; ++i) v.push_back(upload_column(ctx, cols[i]));
  return v;
}
static std::vector<DCol> device_cols_copy(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n) {
  set_device(ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n; ++i) v.push_back(copy_column_device(ctx, device_view(cols[i])));
  return v;
}
static std::vector<DCol> device_cols_view(const dfgpu_column* cols, int32_t n) {
  std::vector<DCol> v;
  for (int i = 0; i < n; ++i) v.push_back(device_view(cols[i]));
  return v;
}

int dfgpu_hashjoin_set_filter(dfgpu_hashjoin* j, const int32_t* col_side, const int32_t* col_index, int32_t n_cols, const dfgpu_expr_node* expr, int32_t n_nodes) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  DF_CHECK(j && col_side && col_index && expr && n_cols >= 1, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(!j->built && j->build_parts.empty(), DFGPU_ERR_STATE, "set_filter must be called before any batch is pushed");
  DF_CHECK(!(j->opt.null_aware && j->opt.join_type == DFGPU_JOIN_RIGHT_ANTI), DFGPU_ERR_INVALID, "null_aware RightAnti join does not support a join filter");
  std::vector<int32_t> types;
  std::vector<int> fside, findex;
  std::vector<dfgpu_expr_node> nodes;
  int shift = 0;
  if (j->wide) {   // key equality stays the first conjunct; the user's column references move behind the key columns
    DF_CHECK(j->filt_side.size() == 2 * j->wide_on_build.size(), DFGPU_ERR_STATE, "set_filter called twice");
    fside = j->filt_side; findex = j->filt_index;
    for (size_t c = 0; c < fside.size(); ++c) types.push_back(wide_key_eq_type((fside[c] == 0 ? j->build_types : j->probe_types)[findex[c]]));
    nodes = j->wide_expr;
    shift = (int)fside.size();
  }
  for (int c = 0; c < n_cols; ++c) {
    DF_CHECK(col_side[c] == 0 || col_side[c] == 1, DFGPU_ERR_INVALID, "join filter column side must be 0 (build) or 1 (probe)");
    const auto& tv = col_side[c] == 0 ? j->build_types : j->probe_types;
    const int limit = (int)tv.size() - (j->wide ? 1 : 0);   // the hidden hash-key column is not addressable
    DF_CHECK(col_index[c] >= 0 && col_index[c] < limit, DFGPU_ERR_INVALID, "join filter column index out of range");
    types.push_back(tv[col_index[c]]);
    fside.push_back(col_side[c]); findex.push_back(col_index[c]);
  }
  for (int i = 0; i < n_nodes; ++i) {
    dfgpu_expr_node nd = expr[i];
    if (nd.kind == DFGPU_EXPR_COLUMN) { DF_CHECK(nd.a >= 0 && nd.a < n_cols, DFGPU_ERR_INVALID, "join filter: column index out of range"); nd.a += shift; }
    nodes.push_back(nd);
  }
  if (j->wide) { dfgpu_expr_node a; memset(&a, 0, sizeof(a)); a.kind = DFGPU_EXPR_BINARY; a.a = DFGPU_OP_AND; nodes.push_back(a); }
  {
    // the user's expression must be Boolean on its own
    ExprPlan user = plan_expr(types.data() + shift, n_cols, expr, n_nodes);
    DF_CHECK(user.root_type == DFGPU_BOOL, DFGPU_ERR_INVALID, "join filter expression must return Boolean");
  }
  j->filt_plan = plan_expr(types.data(), (int)types.size(), nodes.data(), (int)nodes.size());
  DF_CHECK(j->filt_plan.root_type == DFGPU_BOOL, DFGPU_ERR_INVALID, "join filter expression must return Boolean");
  j->filt_side = fside;
  j->filt_index = findex;
  j->has_filter = true;
  DF_API_END
}
int dfgpu_hashjoin_push_build_host(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  push_build(j, host_cols_to_device(j->ctx, cols, n_cols));
  // the caller owns the host buffers only until this call returns (dfgpu.h): pinned sources are copied asynchronously,
  // so the H2D copies must have completed before we hand the buffers back
  DF_CUDA(cudaStreamSynchronize(j->ctx->stream));
  DF_API_END
}
int dfgpu_hashjoin_push_build_device(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  // the caller owns the input only until this call returns: keep a private copy (160 MB for C2's build side)
  push_build(j, device_cols_copy(j->ctx, cols, n_cols));
  DF_API_END
}
int dfgpu_hashjoin_finish_build(dfgpu_hashjoin* j) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  finish_build(j);
  DF_API_END
}
int dfgpu_hashjoin_push_probe_host(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  DF_CHECK(j->built, DFGPU_ERR_STATE, "push_probe before finish_build");
  DF_CHECK(!j->probe_done, DFGPU_ERR_STATE, "push_probe after finish_probe");
  if (!push_probe_host_pipelined(j, cols, n_cols)) push_probe(j, host_cols_to_device(j->ctx, cols, n_cols));
  DF_API_END
}
int dfgpu_hashjoin_push_probe_device(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  push_probe(j, device_cols_view(cols, n_cols));  // consumed before returning (outputs are gathered copies)
  DF_API_END
}
int dfgpu_hashjoin_finish_probe(dfgpu_hashjoin* j) {
  DF_API_BEGIN(j ? j->ctx : nullptr)
  finish_probe(j);
  DF_API_END
}
int dfgpu_hashjoin_next(dfgpu_hashjoin* j, int host, dfgpu_batch** out) {
  dfgpu_ctx* _ctx = j ? j->ctx : nullptr;
  try {
    DF_CHECK(j && out, DFGPU_ERR_INVALID, "null argument");
    if (j->outq.empty()) { *out = nullptr; return DFGPU_END; }
    // checked before the batch leaves the queue: a refused call must not lose its rows
    DF_CHECK(host || !j->outq.front()->host, DFGPU_ERR_STATE, "this batch was produced on the host (pipelined host probe): call next(host=1)");
    BatchPtr b = std::move(j->outq.front());
    j->outq.pop_front();
    if (host && !b->host) { set_device(j->ctx); b = to_host_batch(j->ctx, *b); }
    *out = b.release();
    return DFGPU_OK;
  } catch (const dfgpu::Error& e) { if (_ctx) _ctx->last_error = e.what(); return e.code; }
  catch (const std::exception& e) { if (_ctx) _ctx->last_error = e.what(); return DFGPU_ERR_INVALID; }
}
int64_t dfgpu_hashjoin_metric(dfgpu_hashjoin* j, const char* name) {
  if (!j || !name) return -1;
  std::string s(name);
  if (s == "build_input_rows") return j->m_build_rows;
  if (s == "build_input_batches") return j->m_build_batches;
  if (s == "input_rows") return j->m_input_rows;
  if (s == "input_batches") return j->m_input_batches;
  if (s == "output_rows") return j->m_output_rows;
  if (s == "output_batches") return j->m_output_batches;
  if (s == "array_map_created_count") return j->m_array_map;
  if (s == "inline_payload_words") return j->inline_ok ? j->inline_words : 0;   // 2: the build payload rides beside the key in the table
  if (s == "probe_hits") return j->m_probe_hits;
  if (s == "radix_partitioned_probes") return j->m_radix_probes;
  if (s == "pipelined_host_probes") return j->m_pipelined_probes;   // host pushes probed by push_probe_host_pipelined
  if (s == "membership_filter_bytes") return (int64_t)j->bloom.bytes;
  if (s == "build_distinct_keys") return j->distinct;
  if (s == "build_unique") return j->unique ? 1 : 0;
  if (s == "build_null_key_rows") return j->null_rows;
  return -1;
}
void dfgpu_hashjoin_destroy(dfgpu_hashjoin* j) {
  if (!j) return;
  cudaSetDevice(j->ctx->device);
  delete j;
}

}  // extern "C"
