// radix_probe.cuh — intra-GPU radix-partitioned probe of the inline join table (included by hash_join.cu only; radix_partition, declared
// in common.cuh, also partitions the probe records of the fused pipeline's aggregate sink, and radix_partition_records the packed build
// records of its lookups, pipeline.cu).
//
// Reference analogue: PartitionMode::Partitioned — both join inputs go through BatchPartitioner::Hash
// (physical-plan/src/repartition/mod.rs:1097-1145) so that every partition's hash table is small enough to stay in
// cache while its probe batches stream by (joins/hash_join/exec.rs:1312-1325); output order is per partition.
//
// A probe of a table several times the 50 MB L2 of an H100 is bound by the number of L2 misses (random DRAM accesses cost the
// same whatever their size), not by bytes.  The inline table is addressed by fastrange
// (slot = hi64(hash * cap)), so "partition p" is simply the contiguous slot range [p cap / P, (p+1) cap / P): the BUILD
// side needs no partitioning at all.  The PROBE side is radix-partitioned once on the top log2(P) hash bits:
//   1. radix_hist_kernel      per-partition row counts (keys only, 8 B / row)
//   2. radix_scatter_tma_kernel  one pass: 2048-row tiles of the key and carried column arrive in shared memory by TMA
//        (cp.async.bulk global->shared, mbarrier completion, double buffered), are counting-sorted by partition INSIDE shared
//        memory, and every partition's run leaves as ONE bulk store (cp.async.bulk shared->global) of 16-byte {key, value} records
//   3. radix_probe_kernel     walks the partitioned records in order: all concurrently running blocks probe the same ~16 MB
//        sub-table, so every lookup is an L2 hit instead of a DRAM miss; hits leave through a warp-aggregated
//        reservation (order inside a partition = arrival order: unspecified, like a RepartitionExec consumer's).
// Applies when the caller does not need probe order (dfgpu_hashjoin_options.ordered_output == 0).
#pragma once
#include "tma.cuh"

namespace dfgpu {

constexpr int kRadixTile = 2048, kRadixThreads = 256, kRadixPerThread = kRadixTile / kRadixThreads;   // kRadixMaxParts: common.cuh

__device__ __forceinline__ int radix_part(uint64_t key, int bits) { return (int)(hash_u64(key, kSeedJoin) >> (64 - bits)); }

// The partition kernels read their rows from one of two layouts: RECS = false, a key array and a value array; RECS = true, interleaved
// 16-byte {key, value} records (row i: key at keys[2 i], value at keys[2 i + 1]; vals unused), the fused pipeline's packed build rows.
template <bool RECS>
__device__ __forceinline__ void radix_hist_body(const unsigned long long* __restrict__ keys, int64_t n, int bits, unsigned long long* __restrict__ counts) {
  __shared__ unsigned int s_cnt[kRadixMaxParts];
  if (threadIdx.x < kRadixMaxParts) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  // two rows per iteration: one 128-bit load of two keys, or two of two records
  const int64_t n2 = n / 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n2; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t a, b;
    if constexpr (RECS) {
      const int4 u = ld_stream_16(keys + 4 * i), v = ld_stream_16(keys + 4 * i + 2);
      a = (uint64_t)(uint32_t)u.x | ((uint64_t)(uint32_t)u.y << 32); b = (uint64_t)(uint32_t)v.x | ((uint64_t)(uint32_t)v.y << 32);
    } else {
      const int4 v = ld_stream_16(keys + 2 * i);
      a = (uint64_t)(uint32_t)v.x | ((uint64_t)(uint32_t)v.y << 32); b = (uint64_t)(uint32_t)v.z | ((uint64_t)(uint32_t)v.w << 32);
    }
    atomicAdd(&s_cnt[radix_part(a, bits)], 1u);
    atomicAdd(&s_cnt[radix_part(b, bits)], 1u);
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&s_cnt[radix_part(keys[RECS ? 2 * (n - 1) : n - 1], bits)], 1u);
  __syncthreads();
  if (threadIdx.x < (1 << bits) && s_cnt[threadIdx.x]) atomicAdd(&counts[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
}
__global__ void __launch_bounds__(256) radix_hist_kernel(const unsigned long long* __restrict__ keys, int64_t n, int bits, unsigned long long* __restrict__ counts) {
  radix_hist_body<false>(keys, n, bits, counts);
}
__global__ void __launch_bounds__(256) radix_hist_records_kernel(const unsigned long long* __restrict__ recs, int64_t n, int bits, unsigned long long* __restrict__ counts) {
  radix_hist_body<true>(recs, n, bits, counts);
}

// exclusive prefix of the P counts -> partition start offsets (cursor[p] = start[p], bounds[p] = start, bounds[P] = n)
__global__ void radix_prefix_kernel(const unsigned long long* __restrict__ counts, int P, unsigned long long* __restrict__ cursor, unsigned long long* __restrict__ bounds) {
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int p = 0; p < P; ++p) { cursor[p] = s; bounds[p] = s; s += counts[p]; }
    bounds[P] = s;
  }
}

struct alignas(16) RadixRec { unsigned long long key, val; };

// Dynamic shared memory: 2 stages x { keys[2048] | vals[2048] } or 2 x { records[2048] } (2 x 32 KB, one bulk copy per array); a
// stage is reused in place as the 2048 sorted 16-byte records once every thread holds its 8 rows in registers.
template <bool RECS>
__device__ __forceinline__ void radix_scatter_body(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ vals, int64_t n, int bits,
                                                   unsigned long long* __restrict__ cursor, RadixRec* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ unsigned int s_cnt[kRadixMaxParts], s_start[kRadixMaxParts + 1];
  __shared__ unsigned long long s_gbase[kRadixMaxParts];
  const int P = 1 << bits;
  const int64_t ntiles = (n + kRadixTile - 1) / kRadixTile;
  unsigned long long* stage_keys[2] = {(unsigned long long*)smem, (unsigned long long*)(smem + 2 * kRadixTile * 8)};
  if (threadIdx.x == 0) { mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  // a tile goes through TMA when it is full (bulk copies move multiples of 16 bytes); the ragged last tile uses plain loads
  auto issue = [&](int64_t tile, int s) {
    if (tile < ntiles && (tile + 1) * (int64_t)kRadixTile <= n) {
      mbar_expect_tx(&s_bar[s], 2u * kRadixTile * 8u);
      if constexpr (RECS) {
        tma_load_1d(stage_keys[s], keys + 2 * tile * kRadixTile, kRadixTile * 16u, &s_bar[s]);
      } else {
        tma_load_1d(stage_keys[s], keys + tile * kRadixTile, kRadixTile * 8u, &s_bar[s]);
        tma_load_1d(stage_keys[s] + kRadixTile, vals + tile * kRadixTile, kRadixTile * 8u, &s_bar[s]);
      }
    }
  };
  int64_t tile = blockIdx.x;
  if (threadIdx.x == 0) { issue(tile, 0); issue(tile + gridDim.x, 1); }
  uint32_t phase[2] = {0, 0};
  int s = 0;
  for (; tile < ntiles; tile += gridDim.x, s ^= 1) {
    const bool full = (tile + 1) * (int64_t)kRadixTile <= n;
    const int rows = full ? kRadixTile : (int)(n - tile * kRadixTile);
    unsigned long long k[kRadixPerThread], v[kRadixPerThread];
    if (full) {
      mbar_wait(&s_bar[s], phase[s]);
      phase[s] ^= 1;
#pragma unroll
      for (int i = 0; i < kRadixPerThread; ++i) {
        if constexpr (RECS) {   // 16-byte shared loads (addressed from smem itself: stage_keys[s] would be a generic pointer)
          const ulonglong2 r = ((const ulonglong2*)(smem + s * (2 * kRadixTile * 8)))[threadIdx.x + i * kRadixThreads];
          k[i] = r.x; v[i] = r.y;
        }
        else { k[i] = stage_keys[s][threadIdx.x + i * kRadixThreads]; v[i] = stage_keys[s][kRadixTile + threadIdx.x + i * kRadixThreads]; }
      }
    } else {
#pragma unroll
      for (int i = 0; i < kRadixPerThread; ++i) {
        const int r = threadIdx.x + i * kRadixThreads;
        if constexpr (RECS) { k[i] = r < rows ? keys[2 * (tile * kRadixTile + r)] : 0ull; v[i] = r < rows ? keys[2 * (tile * kRadixTile + r) + 1] : 0ull; }
        else { k[i] = r < rows ? keys[tile * kRadixTile + r] : 0ull; v[i] = r < rows ? vals[tile * kRadixTile + r] : 0ull; }
      }
    }
    if (threadIdx.x < P) s_cnt[threadIdx.x] = 0;
    __syncthreads();                       // every thread holds its rows: the stage may be overwritten; counters are zero
    int part[kRadixPerThread];
    unsigned int rank[kRadixPerThread];
#pragma unroll
    for (int i = 0; i < kRadixPerThread; ++i) {
      part[i] = radix_part(k[i], bits);
      rank[i] = (threadIdx.x + i * kRadixThreads < rows) ? atomicAdd(&s_cnt[part[i]], 1u) : 0u;
    }
    __syncthreads();
    if (threadIdx.x < 32) {                // exclusive scan of <= 64 counts by one warp; global reservation of every run
      unsigned int a = threadIdx.x < P ? s_cnt[threadIdx.x] : 0u, b = threadIdx.x + 32 < P ? s_cnt[threadIdx.x + 32] : 0u;
      unsigned int ia = a, ib = b;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const unsigned int t = __shfl_up_sync(0xffffffffu, ia, d); const unsigned int u = __shfl_up_sync(0xffffffffu, ib, d); if (threadIdx.x >= d) { ia += t; ib += u; } }
      const unsigned int tot_a = __shfl_sync(0xffffffffu, ia, 31);
      if (threadIdx.x < P) { s_start[threadIdx.x] = ia - a; if (a) s_gbase[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], (unsigned long long)a); }
      if (threadIdx.x + 32 < P) { s_start[threadIdx.x + 32] = tot_a + ib - b; if (b) s_gbase[threadIdx.x + 32] = atomicAdd(&cursor[threadIdx.x + 32], (unsigned long long)b); }
    }
    __syncthreads();
    RadixRec* recs = (RadixRec*)stage_keys[s];
#pragma unroll
    for (int i = 0; i < kRadixPerThread; ++i)
      if (threadIdx.x + i * kRadixThreads < rows) recs[s_start[part[i]] + rank[i]] = RadixRec{k[i], v[i]};
    fence_async_smem();                    // generic-proxy writes -> visible to the TMA (async proxy) reads below
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += kRadixThreads) {   // one bulk store per non-empty run
      const unsigned int c = s_cnt[p];
      if (c) tma_store_1d(out + s_gbase[p], recs + s_start[p], c * 16u);
    }
    tma_store_commit();
    tma_store_wait_read();                 // the stores have READ their shared-memory source
    __syncthreads();
    if (threadIdx.x == 0) issue(tile + 2 * (int64_t)gridDim.x, s);   // refill this stage two tiles ahead
  }
}
__global__ void __launch_bounds__(kRadixThreads) radix_scatter_tma_kernel(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ vals, int64_t n, int bits,
                                                                         unsigned long long* __restrict__ cursor, RadixRec* __restrict__ out) {
  radix_scatter_body<false>(keys, vals, n, bits, cursor, out);
}
__global__ void __launch_bounds__(kRadixThreads) radix_scatter_records_kernel(const unsigned long long* __restrict__ recs, int64_t n, int bits, unsigned long long* __restrict__ cursor,
                                                                             RadixRec* __restrict__ out) {
  radix_scatter_body<true>(recs, nullptr, n, bits, cursor, out);
}

// hist -> prefix -> TMA scatter of either layout (recs: keys holds interleaved {key, value} records)
static int radix_partition_impl(dfgpu_ctx* ctx, bool recs, const unsigned long long* keys, const unsigned long long* vals, int64_t n, size_t table_bytes, int force_parts,
                                void* out, unsigned long long* meta) {
  int bits = 1;
  const size_t want = force_parts >= 2 ? (size_t)force_parts : (table_bytes + ((size_t)kRadixSubTableMB << 20) - 1) / ((size_t)kRadixSubTableMB << 20);
  while ((1u << bits) < want && bits < 6) ++bits;
  unsigned long long* counts = meta;
  unsigned long long* cursor = counts + kRadixMaxParts;
  unsigned long long* bounds = cursor + kRadixMaxParts;      // [P + 1]
  // the attribute belongs to the current device: set on every call, so any device and thread may partition
  DF_CUDA(cudaFuncSetAttribute(recs ? (const void*)radix_scatter_records_kernel : (const void*)radix_scatter_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * kRadixTile * 8));
  if (recs) radix_hist_records_kernel<<<kNumSMs * 8, 256, 0, ctx->stream>>>(keys, n, bits, counts);
  else radix_hist_kernel<<<kNumSMs * 8, 256, 0, ctx->stream>>>(keys, n, bits, counts);
  DF_LAUNCH_CHECK(ctx);
  radix_prefix_kernel<<<1, 32, 0, ctx->stream>>>(counts, 1 << bits, cursor, bounds);
  DF_LAUNCH_CHECK(ctx);
  const int64_t rtiles = (n + kRadixTile - 1) / kRadixTile;
  const int grid = (int)std::min<int64_t>(rtiles, kNumSMs * 3);
  if (recs) radix_scatter_records_kernel<<<grid, kRadixThreads, 4 * kRadixTile * 8, ctx->stream>>>(keys, n, bits, cursor, (RadixRec*)out);
  else radix_scatter_tma_kernel<<<grid, kRadixThreads, 4 * kRadixTile * 8, ctx->stream>>>(keys, vals, n, bits, cursor, (RadixRec*)out);
  DF_LAUNCH_CHECK(ctx);
  return bits;
}

// declared in common.cuh: the fused pipeline's aggregate sink partitions its probe records here too
int radix_partition(dfgpu_ctx* ctx, const unsigned long long* keys, const unsigned long long* vals, int64_t n, size_t table_bytes, int force_parts,
                    void* out, unsigned long long* meta) {
  return radix_partition_impl(ctx, false, keys, vals, n, table_bytes, force_parts, out, meta);
}
int radix_partition_records(dfgpu_ctx* ctx, const void* recs, int64_t n, size_t table_bytes, int force_parts, void* out, unsigned long long* meta) {
  return radix_partition_impl(ctx, true, (const unsigned long long*)recs, nullptr, n, table_bytes, force_parts, out, meta);
}

struct RadixOut {
  int n;
  int kind[kMaxFusedCols];    // 0: record key, 1: record value (the carried probe column), 2: field of the table payload word
  int width[kMaxFusedCols], shift[kMaxFusedCols];
  void* dst[kMaxFusedCols];
};

template <int W, bool ALL8>
__global__ void __launch_bounds__(256) radix_probe_kernel(const RadixRec* __restrict__ recs, int64_t n, InlineRef t, RadixOut oc, unsigned int* __restrict__ tile_counter,
                                                         unsigned long long* __restrict__ totals /* [out rows] */) {
  constexpr int ITEMS = 4, TILE = 256 * ITEMS;
  __shared__ unsigned int s_tile;
  const int lane = threadIdx.x & 31;
  const int64_t ntiles = (n + TILE - 1) / TILE;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);   // tiles are taken in record order: the running blocks share one sub-table
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;
    unsigned long long key[ITEMS], val[ITEMS], slot[ITEMS], cur[ITEMS], curp[ITEMS], pay[ITEMS];
    bool live[ITEMS], hit[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int64_t i = tile * TILE + k * 256 + threadIdx.x;
      live[k] = i < n; hit[k] = false; pay[k] = 0; key[k] = 0; val[k] = 0;
      if (live[k]) { const int4 r = ld_stream_16(recs + i); key[k] = (uint64_t)(uint32_t)r.x | ((uint64_t)(uint32_t)r.y << 32); val[k] = (uint64_t)(uint32_t)r.z | ((uint64_t)(uint32_t)r.w << 32); }
      if (key[k] == kEmpty64) live[k] = false;
      slot[k] = __umul64hi(hash_u64(key[k], kSeedJoin), t.cap);
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      cur[k] = kEmpty64; curp[k] = 0;
      if (live[k]) {
        if (W == 2) { const uint4 x = __ldcg((const uint4*)t.slots + slot[k]); cur[k] = (uint64_t)x.x | ((uint64_t)x.y << 32); curp[k] = (uint64_t)x.z | ((uint64_t)x.w << 32); }
        else cur[k] = __ldcg((const unsigned long long*)t.slots + slot[k]);
      }
    }
    // lockstep linear probing: each round advances every unresolved row of the lane by one slot, so the (rare) second and third
    // probes of the lane's rows overlap instead of running one dependent chain after the other
    unsigned pend = 0;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) if (live[k]) pend |= 1u << k;
    while (pend) {
#pragma unroll
      for (int k = 0; k < ITEMS; ++k) {
        if (!((pend >> k) & 1u)) continue;
        if (cur[k] == key[k]) { hit[k] = true; pay[k] = curp[k]; pend &= ~(1u << k); }
        else if (cur[k] == kEmpty64) pend &= ~(1u << k);
        else {
          if (++slot[k] == t.cap) slot[k] = 0;
          if (W == 2) { const uint4 x = __ldcg((const uint4*)t.slots + slot[k]); cur[k] = (uint64_t)x.x | ((uint64_t)x.y << 32); curp[k] = (uint64_t)x.z | ((uint64_t)x.w << 32); }
          else cur[k] = __ldcg((const unsigned long long*)t.slots + slot[k]);
        }
      }
    }
    __syncwarp();
    // warp-aggregated reservation of output rows, coalesced column writes
    unsigned int tot = 0, mypos[ITEMS];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) { const unsigned m = __ballot_sync(0xffffffffu, hit[k]); mypos[k] = tot + __popc(m & ((1u << lane) - 1u)); tot += __popc(m); }
    unsigned long long obase = 0;
    if (lane == 0 && tot) obase = atomicAdd(&totals[0], (unsigned long long)tot);
    obase = __shfl_sync(0xffffffffu, obase, 0);
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      if (!hit[k]) continue;
      const unsigned long long o = obase + mypos[k];
#pragma unroll
      for (int c = 0; c < kMaxFusedCols; ++c) {
        if (c >= oc.n) break;
        const unsigned long long x = oc.kind[c] == 0 ? key[k] : (oc.kind[c] == 1 ? val[k] : (pay[k] >> oc.shift[c]));
        if (ALL8) { ((uint64_t*)oc.dst[c])[o] = x; continue; }
        switch (oc.width[c]) {
          case 8: ((uint64_t*)oc.dst[c])[o] = x; break;
          case 4: ((uint32_t*)oc.dst[c])[o] = (uint32_t)x; break;
          case 2: ((uint16_t*)oc.dst[c])[o] = (uint16_t)x; break;
          default: ((uint8_t*)oc.dst[c])[o] = (uint8_t)x; break;
        }
      }
    }
  }
}

}  // namespace dfgpu
