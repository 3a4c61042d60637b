// partition.cu — the local pass of the hash exchange: RepartitionExec / BatchPartitioner::Hash
// (reference physical-plan/src/repartition/mod.rs:618-648, 1097-1145; partition_indices :895;
// partition_grouped_take :1237).  On 8 GPUs this pass feeds one NCCL all-to-all; rows keep their
// input order inside every partition (the reference's per-partition `take` is order preserving).
//
// Three implementations, chosen per call: packed-counter kernels for <= 8 partitions (one box), warp-match kernels for 9..32,
// and a flag-bitmap + compaction + gather path for more than 32 partitions.  All three carry validity bitmaps and Boolean
// (bit-packed) columns.
#include "batch.cuh"
#include "scan.cuh"

namespace dfgpu {

constexpr int kMaxPartKeys = 4;
struct PartKeys {
  int n;
  const void* ptr[kMaxPartKeys];
  const uint8_t* valid[kMaxPartKeys];
  int64_t voff[kMaxPartKeys];
  int width[kMaxPartKeys];
};

__device__ __forceinline__ uint64_t exchange_hash(const PartKeys& k, int64_t row) {
  // create_hashes with the repartition seed (repartition/mod.rs:650, 1126-1130): first column hashed
  // with the seed, later columns re-seeded with the running hash; NULLs leave the running hash untouched.  A Decimal128 key
  // hashes its low word like a 64-bit key, then combines the high word
  uint64_t h = 0;
  bool first = true;
#pragma unroll
  for (int c = 0; c < kMaxPartKeys; ++c) {
    if (c >= k.n) break;
    if (k.valid[c] && !bit_get(k.valid[c], k.voff[c] + row)) continue;
    uint64_t v, hi = 0;
    switch (k.width[c]) {
      case 1: v = ((const uint8_t*)k.ptr[c])[row]; break;
      case 2: v = ((const uint16_t*)k.ptr[c])[row]; break;
      case 4: v = ((const uint32_t*)k.ptr[c])[row]; break;
      case 16: v = ((const uint64_t*)k.ptr[c])[2 * row]; hi = ((const uint64_t*)k.ptr[c])[2 * row + 1]; break;
      default: v = ((const uint64_t*)k.ptr[c])[row]; break;
    }
    h = first ? hash_u64(v, kSeedExchange) : hash_combine(h, v);
    if (k.width[c] == 16) h = hash_combine(h, hi);
    first = false;
  }
  return h;
}

__global__ void __launch_bounds__(256) partition_flags_kernel(PartKeys k, int64_t n, int n_parts, uint32_t* __restrict__ flag_words /* [n_parts][nw] */) {
  const int64_t nw = (n + 31) / 32;
  const int lane = threadIdx.x & 31;
  for (int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; wi < nw; wi += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    int64_t row = wi * 32 + lane;
    int pid = -1;
    if (row < n) pid = (int)__umul64hi(exchange_hash(k, row), (uint64_t)n_parts);  // hash % n (repartition/mod.rs:875-935)
    for (int p = 0; p < n_parts; ++p) {
      uint32_t w = __ballot_sync(0xffffffffu, pid == p);
      if (lane == 0) flag_words[(int64_t)p * nw + wi] = w;
    }
  }
}

// ------------------------------------------------------------------------------------------
// single-pass radix-style partition (n_parts <= 32):
//   hist kernel   : per tile (256 thr x 8 rows) and partition, the row count (warp ballots, no atomics)
//   scan          : exclusive scan of the partition-major [part][tile] count matrix (one block)
//   scatter kernel: every row's stable rank inside its tile+partition from the same ballots; rows are staged
//                   in shared memory grouped by partition and leave as contiguous runs (coalesced stores)
// Order inside a partition = input order (stable), identical to the flag/compaction path below.
// Bit-packed columns (validity bitmaps, Boolean values) take the same staged positions: one 2048-bit stage per
// column, and each partition's run leaves as whole destination words (tile_bits_out below).
// ------------------------------------------------------------------------------------------
constexpr int kPartThreads = 256;
constexpr int kPartItems = 8;
constexpr int kPartTile = kPartThreads * kPartItems;
constexpr int kPartMaxFast = 32;
constexpr int kPartMaxCols = 16;
constexpr int kPartMaxBits = 2 * kPartMaxCols;   // a validity bitmap and Boolean values per column
struct PartCols { int n; const void* src[kPartMaxCols]; void* dst[kPartMaxCols]; int width[kPartMaxCols]; };
// bit-packed columns: source bit of row r = bit src_off + r of src (nullptr src: every bit is 1 — a column without a
// validity bitmap scattered into a receiver that has one); local mode writes dst[b] from bit 0, peer mode writes
// peer_dst[p * n + b] from bit dst_row[p]
struct PartBits { int n; const uint8_t* src[kPartMaxBits]; int64_t src_off[kPartMaxBits]; uint32_t* dst[kPartMaxBits]; uint32_t* const* peer_dst; };
// peer mode: partition p's rows go to dst_table[p * n_cols + c] (a pointer into rank p's receive buffer, mapped
// through CUDA IPC: stores travel over NVLink) starting at row dst_row[p]; nullptr table = local output columns
struct PeerDst { void* const* dst_table; const long long* dst_row; };

// dynamic shared memory of the bit-packed pass, carved from the front of the column stage before the columns use it:
// the tile row staged at every position (uint16), then one 64-word stage per bit-packed column
__host__ __device__ constexpr size_t part_bits_smem(int nbits) { return (size_t)kPartTile * 2 + (size_t)nbits * (kPartTile / 32) * 4; }

// bits [q, q + 32) of a 2048-bit stage, zero outside it (q >= -31)
__device__ __forceinline__ uint32_t stage_bits32(const uint32_t* sb, int q) {
  const int wi = q >> 5;   // floor, q may be negative
  const uint32_t lo = wi >= 0 ? sb[wi] : 0u;
  const uint32_t hi = wi + 1 < kPartTile / 32 ? sb[wi + 1] : 0u;
  return __funnelshift_r(lo, hi, (uint32_t)q & 31u);
}

// one partition's run of staged bits [s, s + len) -> destination bits [d, d + len).  A word the run covers completely is
// stored; a partly covered first / last word changes only the run's own bits, with an atomic clear then an atomic set,
// because a neighbouring run (the previous tile or chunk, the next partition, another source rank's block) may be
// writing the other bits of that word at the same time.  So no destination bitmap needs zeroing first.  sys: the
// destination may be another GPU's memory, written by other GPUs too.
__device__ __forceinline__ void bits_run_out(const uint32_t* sb, uint32_t s, uint32_t len, unsigned long long d, uint32_t* dst, bool sys, int lane) {
  if (len == 0) return;
  const unsigned long long w0 = d >> 5, w1 = (d + len - 1) >> 5;
  for (unsigned long long w = w0 + lane; w <= w1; w += 32) {
    const uint32_t v = stage_bits32(sb, (int)((long long)s + (long long)(w << 5) - (long long)d));
    uint32_t mask = ~0u;
    if (w == w0) mask &= ~0u << (uint32_t)(d & 31);
    if (w == w1) mask &= ~0u >> (31u - (uint32_t)((d + len - 1) & 31));
    if (mask == ~0u) dst[w] = v;
    else if (sys) { atomicAnd_system(dst + w, ~mask); atomicOr_system(dst + w, v & mask); }
    else { atomicAnd(dst + w, ~mask); atomicOr(dst + w, v & mask); }
  }
}

// the bit-packed columns of one tile.  s_srow[j] = tile row staged at position j (j < tile_rows); partition p's run is staged
// [s_pstart[p], s_pstart[p + 1]) and goes to destination bit goff[p] + pgoff_bias * s_pstart[p] (the two kernels keep the
// run's destination differently).  The caller synchronises the block before it reuses the stage area.
__device__ __forceinline__ void tile_bits_out(const PartBits& pb, const PeerDst& peer, int64_t base, uint32_t tile_rows, int n_parts, const uint16_t* s_srow,
                                              uint32_t* s_bits, const uint32_t* s_pstart, const unsigned long long* goff, bool pgoff_bias) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kPartThreads / 32, kWords = kPartTile / 32;
  // staged word k of bit column b: lane l contributes the bit of the row staged at 32k + l
  for (int k = warp; k < kWords; k += NW) {
    const uint32_t j = (uint32_t)k * 32 + lane;
    const bool in = j < tile_rows;
    const int64_t row = base + (in ? s_srow[j] : 0);
    for (int b = 0; b < pb.n; ++b) {
      const bool bit = in && (!pb.src[b] || bit_get(pb.src[b], pb.src_off[b] + row));
      const uint32_t word = __ballot_sync(0xffffffffu, bit);
      if (lane == 0) s_bits[b * kWords + k] = word;
    }
  }
  __syncthreads();
  for (int p = warp; p < n_parts; p += NW) {
    const uint32_t s = s_pstart[p], len = s_pstart[p + 1] - s;
    const unsigned long long d = goff[p] + (pgoff_bias ? s : 0u);
    for (int b = 0; b < pb.n; ++b)
      bits_run_out(s_bits + b * kWords, s, len, d, peer.dst_table ? pb.peer_dst[p * pb.n + b] : pb.dst[b], peer.dst_table != nullptr, lane);
  }
}

__global__ void __launch_bounds__(kPartThreads) partition_hist_kernel(PartKeys k, int64_t n, int n_parts, int64_t ntiles, unsigned long long* __restrict__ hist /* [n_parts][ntiles] */) {
  __shared__ uint32_t s_cnt[kPartMaxFast];
  const int64_t base = (int64_t)blockIdx.x * kPartTile;
  if (threadIdx.x < kPartMaxFast) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int it = 0; it < kPartItems; ++it) {
    const int64_t row = base + it * kPartThreads + threadIdx.x;
    const int pid = row < n ? (int)__umul64hi(exchange_hash(k, row), (uint64_t)n_parts) : -1;
    const uint32_t m = __match_any_sync(0xffffffffu, pid);  // lanes of this warp bound for the same partition
    if (pid >= 0 && lane == __ffs(m) - 1) atomicAdd(&s_cnt[pid], __popc(m));
  }
  __syncthreads();
  if (threadIdx.x < n_parts) hist[(int64_t)threadIdx.x * ntiles + blockIdx.x] = s_cnt[threadIdx.x];
}

template <bool BITS>
__global__ void __launch_bounds__(kPartThreads, 4) partition_scatter_kernel(PartKeys k, PartCols pc, PartBits pb, int64_t n, int n_parts, int64_t ntiles,
                                                                       const unsigned long long* __restrict__ offs /* scanned [n_parts][ntiles] */, PeerDst peer,
                                                                       int64_t tile0 /* first tile of this launch (chunked peer scatter) */) {
  __shared__ uint32_t s_seg[kPartItems * (kPartThreads / 32)][kPartMaxFast + 1];  // counts per (item, warp) segment and partition (+1: bank padding)
  __shared__ uint32_t s_pstart[kPartMaxFast + 1];
  __shared__ unsigned long long s_goff[kPartMaxFast];
  __shared__ uint8_t s_pid[kPartTile];
  extern __shared__ __align__(16) unsigned char s_stage[];  // kPartTile x (widest column) bytes
  const int64_t tile = tile0 + blockIdx.x;
  const int64_t base = tile * kPartTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kPartThreads / 32;
  int pid[kPartItems];
  uint32_t rank[kPartItems];
  for (int i = threadIdx.x; i < kPartItems * NW * (kPartMaxFast + 1); i += kPartThreads) (&s_seg[0][0])[i] = 0;
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kPartItems; ++it) {
    const int64_t row = base + it * kPartThreads + threadIdx.x;
    pid[it] = row < n ? (int)__umul64hi(exchange_hash(k, row), (uint64_t)n_parts) : -1;
    const uint32_t m = __match_any_sync(0xffffffffu, pid[it]);
    rank[it] = __popc(m & ((1u << lane) - 1u));           // stable rank among the warp's rows of the same partition
    if (pid[it] >= 0 && lane == __ffs(m) - 1) s_seg[it * NW + warp][pid[it]] = __popc(m);
  }
  __syncthreads();
  // per partition: exclusive prefix over the 64 (item, warp) segments in row order — one warp per partition, 2 segments per lane
  for (int p = warp; p < n_parts; p += NW) {
    const uint32_t c0 = s_seg[2 * lane][p], c1 = s_seg[2 * lane + 1][p];
    uint32_t inc = c0 + c1;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t nb = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += nb; }
    const uint32_t ex = inc - (c0 + c1);
    s_seg[2 * lane][p] = ex;
    s_seg[2 * lane + 1][p] = ex + c0;
    if (lane == 31) { s_pstart[p] = inc; s_goff[p] = 0; }
  }
  __syncthreads();
  if (threadIdx.x < n_parts) {
    const unsigned long long o = offs[(int64_t)threadIdx.x * ntiles + tile];   // rows of this partition in earlier tiles (row-wise scan)
    // peer mode: position inside this rank's (chunk, partition) block, shifted to where that block starts at the receiver;
    // local mode: after all rows of the lower partitions (the row totals follow the [part][tile] matrix)
    unsigned long long pbase = 0;
    if (!peer.dst_table) for (int q = 0; q < (int)threadIdx.x; ++q) pbase += offs[(int64_t)n_parts * ntiles + q];
    s_goff[threadIdx.x] = peer.dst_table ? (unsigned long long)peer.dst_row[threadIdx.x] + (o - offs[(int64_t)threadIdx.x * ntiles + tile0]) : pbase + o;
  }
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int p = 0; p < n_parts; ++p) { uint32_t c = s_pstart[p]; s_pstart[p] = run; run += c; }
    s_pstart[n_parts] = run;
  }
  __syncthreads();
  uint32_t lpos[kPartItems];
#pragma unroll
  for (int it = 0; it < kPartItems; ++it) {
    lpos[it] = 0;
    if (pid[it] >= 0) {
      lpos[it] = s_pstart[pid[it]] + s_seg[it * NW + warp][pid[it]] + rank[it];
      s_pid[lpos[it]] = (uint8_t)pid[it];
      if (BITS) ((uint16_t*)s_stage)[lpos[it]] = (uint16_t)(it * kPartThreads + threadIdx.x);
    }
  }
  const uint32_t tile_rows = s_pstart[n_parts];
  if (BITS) {
    __syncthreads();
    tile_bits_out(pb, peer, base, tile_rows, n_parts, (const uint16_t*)s_stage, (uint32_t*)(s_stage + kPartTile * 2), s_pstart, s_goff, false);
  }
  for (int c = 0; c < pc.n; ++c) {
    __syncthreads();
    const int w = pc.width[c];
#pragma unroll
    for (int it = 0; it < kPartItems; ++it) {
      if (pid[it] < 0) continue;
      const int64_t row = base + it * kPartThreads + threadIdx.x;
      switch (w) {
        case 1: ((uint8_t*)s_stage)[lpos[it]] = ((const uint8_t*)pc.src[c])[row]; break;
        case 2: ((uint16_t*)s_stage)[lpos[it]] = ((const uint16_t*)pc.src[c])[row]; break;
        case 4: ((uint32_t*)s_stage)[lpos[it]] = ((const uint32_t*)pc.src[c])[row]; break;
        case 8: ((uint64_t*)s_stage)[lpos[it]] = ((const uint64_t*)pc.src[c])[row]; break;
        default: ((uint4*)s_stage)[lpos[it]] = ((const uint4*)pc.src[c])[row]; break;
      }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < tile_rows; j += kPartThreads) {
      const int p = s_pid[j];
      const unsigned long long d = s_goff[p] + (j - s_pstart[p]);
      void* dstc = peer.dst_table ? peer.dst_table[p * pc.n + c] : pc.dst[c];
      switch (w) {
        case 1: ((uint8_t*)dstc)[d] = ((const uint8_t*)s_stage)[j]; break;
        case 2: ((uint16_t*)dstc)[d] = ((const uint16_t*)s_stage)[j]; break;
        case 4: ((uint32_t*)dstc)[d] = ((const uint32_t*)s_stage)[j]; break;
        case 8: ((uint64_t*)dstc)[d] = ((const uint64_t*)s_stage)[j]; break;
        default: ((uint4*)dstc)[d] = ((const uint4*)s_stage)[j]; break;
      }
    }
  }
}


// ------------------------------------------------------------------------------------------
// <= 8 partitions (one box has at most 8 GPUs): the ranking works on packed counters instead of warp matches.
// A thread owns 8 CONSECUTIVE rows of the tile: its per-partition counts fit one 64-bit word (8 x 8 bits), the
// block-wide exclusive scan runs on two words of 4 x 16-bit lanes (a tile holds 2048 rows < 2^16), and a row's
// staged position is  tile start of its partition + rows of that partition in lower threads + rank inside the
// thread — the stable order.  Partition ids are computed with coalesced key loads and handed over through shared
// memory (1 byte per row), staged positions likewise (2 bytes per row), so every global access is coalesced.
// ------------------------------------------------------------------------------------------
template <bool SIMPLE>
__device__ __forceinline__ int part_id8(const PartKeys& k, int64_t row, int n_parts) {
  const uint64_t h = SIMPLE ? hash_u64(((const uint64_t*)k.ptr[0])[row], kSeedExchange) : exchange_hash(k, row);
  return (int)__umul64hi(h, (uint64_t)n_parts);
}
__device__ __forceinline__ uint64_t spread_bytes16(uint32_t x) {   // bytes b0..b3 -> 16-bit lanes
  uint64_t v = x;
  v = (v | (v << 16)) & 0x0000FFFF0000FFFFull;
  v = (v | (v << 8)) & 0x00FF00FF00FF00FFull;
  return v;
}

template <bool SIMPLE>
__global__ void __launch_bounds__(kPartThreads) partition_hist8_kernel(PartKeys k, int64_t n, int n_parts, int64_t ntiles, unsigned long long* __restrict__ hist) {
  __shared__ unsigned long long s_w[kPartThreads / 32][2];
  const int64_t base = (int64_t)blockIdx.x * kPartTile;
  uint64_t cnt8 = 0;
#pragma unroll
  for (int it = 0; it < kPartItems; ++it) {
    const int64_t row = base + it * kPartThreads + threadIdx.x;
    if (row < n) cnt8 += 1ull << (8 * part_id8<SIMPLE>(k, row, n_parts));
  }
  unsigned long long lo = spread_bytes16((uint32_t)cnt8), hi = spread_bytes16((uint32_t)(cnt8 >> 32));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { lo += __shfl_xor_sync(0xffffffffu, lo, d); hi += __shfl_xor_sync(0xffffffffu, hi, d); }
  if ((threadIdx.x & 31) == 0) { s_w[threadIdx.x >> 5][0] = lo; s_w[threadIdx.x >> 5][1] = hi; }
  __syncthreads();
  if (threadIdx.x < n_parts) {
    uint32_t c = 0;
#pragma unroll
    for (int w = 0; w < kPartThreads / 32; ++w) c += (uint32_t)(s_w[w][threadIdx.x >> 2] >> (16 * (threadIdx.x & 3))) & 0xFFFFu;
    hist[(int64_t)threadIdx.x * ntiles + blockIdx.x] = c;
  }
}

template <bool SIMPLE, bool BITS>
__global__ void __launch_bounds__(kPartThreads, 4) partition_scatter8_kernel(PartKeys k, PartCols pc, PartBits pb, int64_t n, int n_parts, int64_t ntiles,
                                                                         const unsigned long long* __restrict__ offs, PeerDst peer, int64_t tile0, int cols_per_round) {
  __shared__ __align__(16) uint8_t s_pidin[kPartTile];
  __shared__ __align__(16) uint16_t s_lpos[kPartTile];
  __shared__ uint8_t s_psort[kPartTile];                     // partition of every staged row
  __shared__ unsigned long long s_w[kPartThreads / 32][2];
  __shared__ uint32_t s_pstart[9];
  __shared__ unsigned long long s_goff[8];
  __shared__ void* s_dst[8 * kPartMaxCols];
  extern __shared__ __align__(16) unsigned char s_stage[];   // cols_per_round columns, each kPartTile x width bytes
  const int64_t tile = tile0 + blockIdx.x;
  const int64_t base = tile * kPartTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // 1. partition ids, coalesced
#pragma unroll
  for (int it = 0; it < kPartItems; ++it) {
    const int r = it * kPartThreads + threadIdx.x;
    const int64_t row = base + r;
    s_pidin[r] = row < n ? (uint8_t)part_id8<SIMPLE>(k, row, n_parts) : (uint8_t)0xFF;
  }
  if (threadIdx.x < n_parts) {
    const unsigned long long o = offs[(int64_t)threadIdx.x * ntiles + tile];   // rows of this partition in earlier tiles (row-wise scan)
    // peer mode: position inside this rank's (chunk, partition) block, shifted to where that block starts at the receiver;
    // local mode: after all rows of the lower partitions (the row totals follow the [part][tile] matrix)
    unsigned long long pbase = 0;
    if (!peer.dst_table) for (int q = 0; q < (int)threadIdx.x; ++q) pbase += offs[(int64_t)n_parts * ntiles + q];
    s_goff[threadIdx.x] = peer.dst_table ? (unsigned long long)peer.dst_row[threadIdx.x] + (o - offs[(int64_t)threadIdx.x * ntiles + tile0]) : pbase + o;
  }
  for (int i = threadIdx.x; i < n_parts * pc.n; i += kPartThreads) s_dst[i] = peer.dst_table ? peer.dst_table[i] : pc.dst[i % pc.n];
  __syncthreads();
  // 2. my 8 consecutive rows: packed per-thread counts -> block-wide exclusive scan -> staged positions
  const uint64_t pids8 = *(const uint64_t*)&s_pidin[threadIdx.x * 8];
  uint64_t cnt8 = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t p = (uint32_t)(pids8 >> (8 * i)) & 0xFFu;
    if (p < 8) cnt8 += 1ull << (8 * p);
  }
  const unsigned long long lo = spread_bytes16((uint32_t)cnt8), hi = spread_bytes16((uint32_t)(cnt8 >> 32));
  unsigned long long ilo = lo, ihi = hi;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long a = __shfl_up_sync(0xffffffffu, ilo, d), b = __shfl_up_sync(0xffffffffu, ihi, d);
    if (lane >= d) { ilo += a; ihi += b; }
  }
  if (lane == 31) { s_w[warp][0] = ilo; s_w[warp][1] = ihi; }
  __syncthreads();
  unsigned long long wlo = 0, whi = 0, tlo = 0, thi = 0;
#pragma unroll
  for (int w = 0; w < kPartThreads / 32; ++w) {
    const unsigned long long a = s_w[w][0], b = s_w[w][1];
    if (w < warp) { wlo += a; whi += b; }
    tlo += a; thi += b;
  }
  // tile starts of the partitions, packed like the counters (every thread computes them: 8 adds, no extra barrier)
  unsigned long long plo = 0, phi = 0;
  uint32_t tile_rows = 0;
  {
    uint32_t run = 0;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      if (p < 4) plo |= (unsigned long long)run << (16 * p); else phi |= (unsigned long long)run << (16 * (p - 4));
      if (threadIdx.x == 0) s_pstart[p] = run;
      run += (uint32_t)((p < 4 ? tlo : thi) >> (16 * (p & 3))) & 0xFFFFu;
    }
    tile_rows = run;
    if (threadIdx.x == 0) s_pstart[8] = run;
  }
  // running staged position per partition for this thread: tile start + rows in lower threads, then +1 per own row (stable)
  unsigned long long blo = plo + wlo + ilo - lo, bhi = phi + whi + ihi - hi;
  {
    uint32_t lp[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint32_t p = (uint32_t)(pids8 >> (8 * i)) & 0xFFu;
      lp[i] = 0;
      if (p < 8) {
        const int sh = 16 * (p & 3);
        if (p < 4) { lp[i] = (uint32_t)(blo >> sh) & 0xFFFFu; blo += 1ull << sh; }
        else { lp[i] = (uint32_t)(bhi >> sh) & 0xFFFFu; bhi += 1ull << sh; }
        s_psort[lp[i]] = (uint8_t)p;
        if (BITS) ((uint16_t*)s_stage)[lp[i]] = (uint16_t)(threadIdx.x * 8 + i);
      }
    }
    *(uint4*)&s_lpos[threadIdx.x * 8] = make_uint4(lp[0] | (lp[1] << 16), lp[2] | (lp[3] << 16), lp[4] | (lp[5] << 16), lp[6] | (lp[7] << 16));
  }
  __syncthreads();
  if (threadIdx.x < n_parts) s_goff[threadIdx.x] -= s_pstart[threadIdx.x];   // destination of staged row j of partition p = s_goff[p] + j
  if (BITS) tile_bits_out(pb, peer, base, tile_rows, n_parts, (const uint16_t*)s_stage, (uint32_t*)(s_stage + kPartTile * 2), s_pstart, s_goff, true);
  // 3. columns: coalesced load -> staged position -> contiguous runs out (to local or peer memory)
  for (int c0 = 0; c0 < pc.n; c0 += cols_per_round) {
    const int c1 = min(pc.n, c0 + cols_per_round);
    __syncthreads();   // s_lpos visible (first round) / previous round's stage fully drained
    size_t soff = 0;
    for (int c = c0; c < c1; ++c) {
      const int w = pc.width[c];
      unsigned char* st = s_stage + soff;
      soff += (size_t)kPartTile * w;
#pragma unroll
      for (int it = 0; it < kPartItems; ++it) {
        const int r = it * kPartThreads + threadIdx.x;
        const int64_t row = base + r;
        if (row >= n) continue;
        const uint32_t lp = s_lpos[r];
        switch (w) {
          case 1: ((uint8_t*)st)[lp] = ((const uint8_t*)pc.src[c])[row]; break;
          case 2: ((uint16_t*)st)[lp] = ((const uint16_t*)pc.src[c])[row]; break;
          case 4: ((uint32_t*)st)[lp] = ((const uint32_t*)pc.src[c])[row]; break;
          case 8: ((uint64_t*)st)[lp] = ((const uint64_t*)pc.src[c])[row]; break;
          default: ((uint4*)st)[lp] = ((const uint4*)pc.src[c])[row]; break;
        }
      }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < tile_rows; j += kPartThreads) {
      const int p = s_psort[j];
      const unsigned long long d = s_goff[p] + j;
      soff = 0;
      for (int c = c0; c < c1; ++c) {
        const int w = pc.width[c];
        const unsigned char* st = s_stage + soff;
        soff += (size_t)kPartTile * w;
        void* dstc = s_dst[p * pc.n + c];
        switch (w) {
          case 1: ((uint8_t*)dstc)[d] = ((const uint8_t*)st)[j]; break;
          case 2: ((uint16_t*)dstc)[d] = ((const uint16_t*)st)[j]; break;
          case 4: ((uint32_t*)dstc)[d] = ((const uint32_t*)st)[j]; break;
          case 8: ((uint64_t*)dstc)[d] = ((const uint64_t*)st)[j]; break;
          default: ((uint4*)dstc)[d] = ((const uint4*)st)[j]; break;
        }
      }
    }
  }
}

// launch helpers: <= 8 partitions take the packed-counter kernels, 9..32 the warp-match kernels
static inline bool simple_key(const PartKeys& k) { return k.n == 1 && k.width[0] == 8 && !k.valid[0]; }
static void launch_partition_hist(dfgpu_ctx* ctx, const PartKeys& pk, int64_t n, int n_parts, int64_t ntiles, unsigned long long* hist) {
  if (n_parts <= 8) {
    if (simple_key(pk)) partition_hist8_kernel<true><<<(int)ntiles, kPartThreads, 0, ctx->stream>>>(pk, n, n_parts, ntiles, hist);
    else partition_hist8_kernel<false><<<(int)ntiles, kPartThreads, 0, ctx->stream>>>(pk, n, n_parts, ntiles, hist);
  } else {
    partition_hist_kernel<<<(int)ntiles, kPartThreads, 0, ctx->stream>>>(pk, n, n_parts, ntiles, hist);
  }
}
// with bit-packed columns (pb.n > 0) the _BITS instantiations run; without, the kernels are what they were before those columns existed
template <bool BITS>
static void launch_partition_scatter_t(dfgpu_ctx* ctx, const PartKeys& pk, const PartCols& pc, const PartBits& pb, int64_t n, int n_parts, int64_t ntiles,
                                       const unsigned long long* offs, PeerDst peer, int64_t tile0, int64_t tiles) {
  const size_t bits_smem = BITS ? part_bits_smem(pb.n) : 0;
  int maxw = 1, sumw = 0;
  for (int i = 0; i < pc.n; ++i) { maxw = std::max(maxw, pc.width[i]); sumw += pc.width[i]; }
  if (n_parts <= 8) {
    // stage as many columns per round as fit 32 KB (4 CTAs/SM stay resident); a 16-byte column alone needs the 32 KB
    int per_round = pc.n, round_max = 0, cur_bytes = 0;
    const int budget = 32 * 1024;
    while (per_round > 1) {   // largest uniform columns-per-round whose widest window fits the budget
      round_max = 0;
      for (int c0 = 0; c0 < pc.n; c0 += per_round) { cur_bytes = 0; for (int c = c0; c < std::min(pc.n, c0 + per_round); ++c) cur_bytes += pc.width[c] * kPartTile; round_max = std::max(round_max, cur_bytes); }
      if (round_max <= budget) break;
      --per_round;
    }
    if (per_round == 1) round_max = maxw * kPartTile;
    (void)sumw;
    const size_t smem = std::max((size_t)round_max, bits_smem);
    if (simple_key(pk)) partition_scatter8_kernel<true, BITS><<<(int)tiles, kPartThreads, smem, ctx->stream>>>(pk, pc, pb, n, n_parts, ntiles, offs, peer, tile0, per_round);
    else partition_scatter8_kernel<false, BITS><<<(int)tiles, kPartThreads, smem, ctx->stream>>>(pk, pc, pb, n, n_parts, ntiles, offs, peer, tile0, per_round);
  } else {
    partition_scatter_kernel<BITS><<<(int)tiles, kPartThreads, std::max((size_t)kPartTile * maxw, bits_smem), ctx->stream>>>(pk, pc, pb, n, n_parts, ntiles, offs, peer, tile0);
  }
}
static void launch_partition_scatter(dfgpu_ctx* ctx, const PartKeys& pk, const PartCols& pc, const PartBits& pb, int64_t n, int n_parts, int64_t ntiles,
                                     const unsigned long long* offs, PeerDst peer, int64_t tile0, int64_t tiles) {
  if (pb.n > 0) launch_partition_scatter_t<true>(ctx, pk, pc, pb, n, n_parts, ntiles, offs, peer, tile0, tiles);
  else launch_partition_scatter_t<false>(ctx, pk, pc, pb, n, n_parts, ntiles, offs, peer, tile0, tiles);
}

// the columns of a single-pass scatter: fixed-width values go to PartCols, validity bitmaps and Boolean values to PartBits.
// byte_col[i] / bit_col[b] = the input column of entry i / b; bit_is_valid[b] = entry b is that column's validity.
// dst_valid[c]: column c's destination has a validity bitmap (a source column without one writes all-ones there).
struct PartLayout {
  PartCols pc;
  PartBits pb;
  std::vector<int> byte_col, bit_col;
  std::vector<bool> bit_is_valid;
};
static PartLayout part_layout(const std::vector<DCol>& v, const std::vector<bool>& dst_valid) {
  PartLayout L;
  memset(&L.pc, 0, sizeof(L.pc)); memset(&L.pb, 0, sizeof(L.pb));
  for (int i = 0; i < (int)v.size(); ++i) {
    if (v[i].type == DFGPU_BOOL) {
      L.pb.src[L.pb.n] = (const uint8_t*)v[i].values; L.pb.src_off[L.pb.n] = v[i].offset; L.pb.n++;
      L.bit_col.push_back(i); L.bit_is_valid.push_back(false);
    } else {
      L.pc.src[L.pc.n] = v[i].values; L.pc.width[L.pc.n] = type_width(v[i].type); L.pc.n++;
      L.byte_col.push_back(i);
    }
    if (dst_valid[i]) {
      L.pb.src[L.pb.n] = v[i].validity; L.pb.src_off[L.pb.n] = v[i].offset; L.pb.n++;
      L.bit_col.push_back(i); L.bit_is_valid.push_back(true);
    }
  }
  return L;
}

}  // namespace dfgpu

using namespace dfgpu;

extern "C" int dfgpu_hash_partition_device(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys,
                                           int32_t n_parts, dfgpu_batch** out, int64_t* part_offsets_host) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && cols && key_cols && out && part_offsets_host, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(n_keys >= 1 && n_keys <= kMaxPartKeys, DFGPU_ERR_UNSUPPORTED, "hash partition: 1..4 key columns");
  DF_CHECK(n_parts >= 1 && n_parts <= 1024, DFGPU_ERR_INVALID, "hash partition: 1..1024 partitions");
  set_device(ctx);
  std::vector<DCol> v;
  for (int i = 0; i < n_cols; ++i) v.push_back(device_view(cols[i]));
  const int64_t n = n_cols ? v[0].length : 0;
  DF_CHECK(n < 0xFFFFFFFFll, DFGPU_ERR_UNSUPPORTED, "hash partition: < 2^32-1 rows per call");
  PartKeys pk;
  memset(&pk, 0, sizeof(pk));
  pk.n = n_keys;
  for (int c = 0; c < n_keys; ++c) {
    DF_CHECK(key_cols[c] >= 0 && key_cols[c] < n_cols, DFGPU_ERR_INVALID, "key column out of range");
    const DCol& col = v[key_cols[c]];
    int w = type_width(col.type);
    DF_CHECK(w >= 1 && w <= 16, DFGPU_ERR_UNSUPPORTED, "hash partition: key must be a fixed-width type of <= 128 bits");
    pk.ptr[c] = col.values; pk.valid[c] = col.validity; pk.voff[c] = col.offset; pk.width[c] = w;
  }
  BatchPtr b(new dfgpu_batch());
  b->ctx = ctx; b->rows = n; b->host = false;
  for (int p = 0; p <= n_parts; ++p) part_offsets_host[p] = 0;
  const bool fast = n > 0 && n_parts <= kPartMaxFast && n_cols <= kPartMaxCols;
  if (fast) {
    const int64_t ntiles = (n + kPartTile - 1) / kPartTile;
    DevBuf hist(ctx, (size_t)(n_parts * ntiles + n_parts) * 8);   // [part][tile] counts -> row-wise exclusive scan, then n_parts row totals
    {
      KernelTimer kt(ctx, "partition");
      launch_partition_hist(ctx, pk, n, n_parts, ntiles, hist.as<unsigned long long>());
      DF_LAUNCH_CHECK(ctx);
      scan_tiles_kernel<1024><<<n_parts, 1024, 0, ctx->stream>>>((uint64_t*)hist.ptr, ntiles, (uint64_t*)hist.ptr + (int64_t)n_parts * ntiles);
      DF_LAUNCH_CHECK(ctx);
    }
    std::vector<bool> has_valid(n_cols);
    for (int i = 0; i < n_cols; ++i) has_valid[i] = v[i].validity != nullptr;
    PartLayout L = part_layout(v, has_valid);
    for (int i = 0; i < n_cols; ++i) {
      b->cols.push_back(alloc_col(ctx, v[i].type, n, has_valid[i]));   // null_count -1 (unknown) with a bitmap, as take_column leaves it
    }
    for (int i = 0; i < L.pc.n; ++i) L.pc.dst[i] = b->cols[L.byte_col[i]].own_values->ptr;
    for (int j = 0; j < L.pb.n; ++j) {
      const DCol& d = b->cols[L.bit_col[j]];
      L.pb.dst[j] = (L.bit_is_valid[j] ? d.own_validity : d.own_values)->as<uint32_t>();
    }
    {
      KernelTimer kt(ctx, "partition");
      launch_partition_scatter(ctx, pk, L.pc, L.pb, n, n_parts, ntiles, hist.as<unsigned long long>(), PeerDst{nullptr, nullptr}, 0, ntiles);
      DF_LAUNCH_CHECK(ctx);
    }
    // partition starts = running sum of the row totals
    std::vector<unsigned long long> totals(n_parts);
    DF_CUDA(cudaMemcpyAsync(totals.data(), (const unsigned long long*)hist.ptr + (int64_t)n_parts * ntiles, (size_t)n_parts * 8, cudaMemcpyDeviceToHost, ctx->stream));
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    int64_t run = 0;
    for (int p = 0; p < n_parts; ++p) { part_offsets_host[p] = run; run += (int64_t)totals[p]; }
    part_offsets_host[n_parts] = run;
    DF_CHECK(run == n, DFGPU_ERR_CUDA, "hash partition: internal row count mismatch");
  } else if (n > 0) {
    // more than 32 partitions (or more than 16 columns): one flag bitmap per partition, compaction, then a gather per column
    const int64_t nw = (n + 31) / 32;
    DevBuf flags(ctx, (size_t)n_parts * nw * 4), perm(ctx, (size_t)n * 4);
    partition_flags_kernel<<<grid_for(n, 256, kNumSMs * 8), 256, 0, ctx->stream>>>(pk, n, n_parts, flags.as<uint32_t>());
    DF_LAUNCH_CHECK(ctx);
    int64_t pos = 0;
    for (int p = 0; p < n_parts; ++p) {
      DevBuf tiles;
      const uint32_t* w = flags.as<uint32_t>() + (int64_t)p * nw;
      int64_t cnt = compact_count(ctx, w, n, 1, &tiles);
      part_offsets_host[p] = pos;
      if (cnt) compact_emit(ctx, w, n, 1, tiles, perm.as<uint32_t>() + pos);
      pos += cnt;
    }
    part_offsets_host[n_parts] = pos;
    DF_CHECK(pos == n, DFGPU_ERR_CUDA, "hash partition: internal row count mismatch");
    for (int i = 0; i < n_cols; ++i) b->cols.push_back(take_column(ctx, v[i], perm.as<uint32_t>(), n, false));
  } else {
    for (int i = 0; i < n_cols; ++i) b->cols.push_back(alloc_col(ctx, v[i].type, 0, false));
  }
  *out = b.release();
  DF_API_END
}

// ------------------------------------------------------------------------------------------
// fused partition + exchange over peer memory: phase 1 counts, phase 2 scatters straight into the peers'
// receive buffers (pointers obtained through CUDA IPC).  Between the phases the caller all-gathers the counts so
// every rank knows where its block starts in each receiver (datafusion_b200/exchange.py PeerExchange).
// ------------------------------------------------------------------------------------------
struct dfgpu_partition_plan {
  dfgpu_ctx* ctx;
  PartKeys pk;
  std::vector<DCol> cols;   // input views: the column layout of a scatter depends on which receivers keep a validity bitmap
  int64_t n, ntiles;
  int n_parts, n_chunks;
  DevBuf hist;
  std::vector<DevBuf> dst_table, dst_row;   // per chunk: the scatter of chunk c may still be in flight when c+1 is issued
  int64_t chunk_tile(int c) const { return ntiles * c / n_chunks; }
  bool has_bits() const {   // a validity bitmap or a Boolean column: only the _nullable scatter carries it
    for (const DCol& c : cols) if (c.validity || c.type == DFGPU_BOOL) return true;
    return false;
  }
};

extern "C" int dfgpu_partition_plan_create_chunked(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys,
                                                   int32_t n_parts, int32_t n_chunks, int64_t* counts_host /* [n_chunks][n_parts] */, dfgpu_partition_plan** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && cols && key_cols && out && counts_host, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(n_keys >= 1 && n_keys <= kMaxPartKeys && n_parts >= 1 && n_parts <= kPartMaxFast && n_cols >= 1 && n_cols <= kPartMaxCols, DFGPU_ERR_UNSUPPORTED,
           "peer partition: 1..4 keys, <= 32 partitions, <= 16 columns");
  DF_CHECK(n_chunks >= 1 && n_chunks <= 64, DFGPU_ERR_INVALID, "peer partition: 1..64 chunks");
  set_device(ctx);
  std::unique_ptr<dfgpu_partition_plan> pl(new dfgpu_partition_plan());
  pl->ctx = ctx; pl->n_parts = n_parts; pl->n_chunks = n_chunks;
  for (int i = 0; i < n_cols; ++i) pl->cols.push_back(device_view(cols[i]));
  const std::vector<DCol>& v = pl->cols;
  pl->n = v[0].length;
  DF_CHECK(pl->n < 0xFFFFFFFFll, DFGPU_ERR_UNSUPPORTED, "peer partition: < 2^32-1 rows per call");
  memset(&pl->pk, 0, sizeof(pl->pk));
  pl->pk.n = n_keys;
  for (int c = 0; c < n_keys; ++c) {
    DF_CHECK(key_cols[c] >= 0 && key_cols[c] < n_cols, DFGPU_ERR_INVALID, "key column out of range");
    const DCol& col = v[key_cols[c]];
    int w = type_width(col.type);
    DF_CHECK(w >= 1 && w <= 16, DFGPU_ERR_UNSUPPORTED, "peer partition: key must be a fixed-width type of <= 128 bits");
    pl->pk.ptr[c] = col.values; pl->pk.valid[c] = col.validity; pl->pk.voff[c] = col.offset; pl->pk.width[c] = w;
  }
  pl->ntiles = std::max<int64_t>(1, (pl->n + kPartTile - 1) / kPartTile);
  pl->hist.alloc(ctx, (size_t)(n_parts * pl->ntiles + n_parts) * 8);
  {
    KernelTimer kt(ctx, "partition");
    launch_partition_hist(ctx, pl->pk, pl->n, n_parts, pl->ntiles, pl->hist.as<unsigned long long>());
    DF_LAUNCH_CHECK(ctx);
    scan_tiles_kernel<1024><<<n_parts, 1024, 0, ctx->stream>>>((uint64_t*)pl->hist.ptr, pl->ntiles, (uint64_t*)pl->hist.ptr + (int64_t)n_parts * pl->ntiles);
    DF_LAUNCH_CHECK(ctx);
  }
  // rows of partition p before the first tile of every chunk: starts[c][p] (row-wise scan), and the row totals
  std::vector<unsigned long long> starts((size_t)(n_chunks + 1) * n_parts);
  for (int c = 0; c < n_chunks; ++c)
    DF_CUDA(cudaMemcpy2DAsync(starts.data() + (size_t)c * n_parts, 8, (const unsigned long long*)pl->hist.ptr + pl->chunk_tile(c), (size_t)pl->ntiles * 8, 8, (size_t)n_parts,
                              cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaMemcpyAsync(starts.data() + (size_t)n_chunks * n_parts, (const unsigned long long*)pl->hist.ptr + (int64_t)n_parts * pl->ntiles, (size_t)n_parts * 8,
                          cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int p = 0; p < n_parts; ++p)
    for (int c = 0; c < n_chunks; ++c)
      counts_host[(size_t)c * n_parts + p] = (int64_t)(starts[(size_t)(c + 1) * n_parts + p] - starts[(size_t)c * n_parts + p]);
  pl->dst_table.resize(n_chunks); pl->dst_row.resize(n_chunks);
  *out = pl.release();
  DF_API_END
}

extern "C" int dfgpu_partition_plan_create(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys,
                                           int32_t n_parts, int64_t* counts_host, dfgpu_partition_plan** out) {
  return dfgpu_partition_plan_create_chunked(ctx, cols, n_cols, key_cols, n_keys, n_parts, 1, counts_host, out);
}

extern "C" int dfgpu_partition_plan_scatter_peer_chunk_nullable(dfgpu_partition_plan* pl, int32_t chunk, void* const* dst_bases /* [n_parts * n_cols] */,
                                                                void* const* dst_validity /* [n_parts * n_cols] or NULL */,
                                                                const int64_t* dst_row_offset /* [n_parts]: where this rank's (chunk, p) block starts at receiver p */) {
  DF_API_BEGIN(pl ? pl->ctx : nullptr)
  DF_CHECK(pl, DFGPU_ERR_INVALID, "null argument");
  dfgpu_ctx* ctx = pl->ctx;
  DF_CHECK(chunk >= 0 && chunk < pl->n_chunks && dst_bases && dst_row_offset, DFGPU_ERR_INVALID, "peer scatter: bad chunk / null argument");
  set_device(ctx);
  const int P = pl->n_parts, nc = (int)pl->cols.size();
  // column c keeps a validity bitmap at the receivers when its dst_validity entries are set: all of them or none
  std::vector<bool> dst_valid(nc, false);
  for (int c = 0; c < nc; ++c) {
    dst_valid[c] = dst_validity && dst_validity[c];
    for (int p = 1; p < P; ++p)
      DF_CHECK((dst_validity && dst_validity[(size_t)p * nc + c]) == dst_valid[c], DFGPU_ERR_INVALID, "peer scatter: a column's receive bitmaps must be given for every partition or for none");
    DF_CHECK(dst_valid[c] || !pl->cols[c].validity, DFGPU_ERR_INVALID, "peer scatter: a column with NULLs needs receive bitmaps (dst_validity)");
  }
  PartLayout L = part_layout(pl->cols, dst_valid);
  // device table: the fixed-width columns' destinations [p][i], then the bit-packed columns' [p][b]
  std::vector<void*> host_table((size_t)P * (L.pc.n + L.pb.n));
  for (int p = 0; p < P; ++p) {
    for (int i = 0; i < L.pc.n; ++i) host_table[(size_t)p * L.pc.n + i] = dst_bases[(size_t)p * nc + L.byte_col[i]];
    for (int b = 0; b < L.pb.n; ++b)
      host_table[(size_t)P * L.pc.n + (size_t)p * L.pb.n + b] = (L.bit_is_valid[b] ? dst_validity : dst_bases)[(size_t)p * nc + L.bit_col[b]];
  }
  const size_t tb = host_table.size() * sizeof(void*);
  DevBuf& table = pl->dst_table[chunk];
  DevBuf& rows = pl->dst_row[chunk];
  table.alloc(ctx, tb);
  rows.alloc(ctx, (size_t)P * 8);
  DF_CUDA(cudaMemcpyAsync(table.ptr, host_table.data(), tb, cudaMemcpyHostToDevice, ctx->stream));
  DF_CUDA(cudaMemcpyAsync(rows.ptr, dst_row_offset, (size_t)P * 8, cudaMemcpyHostToDevice, ctx->stream));
  L.pb.peer_dst = (uint32_t* const*)table.as<void*>() + (size_t)P * L.pc.n;
  const int64_t t0 = pl->chunk_tile(chunk), t1 = chunk + 1 < pl->n_chunks ? pl->chunk_tile(chunk + 1) : pl->ntiles;
  if (pl->n > 0 && t1 > t0) {
    KernelTimer kt(ctx, "partition");
    launch_partition_scatter(ctx, pl->pk, L.pc, L.pb, pl->n, P, pl->ntiles, pl->hist.as<unsigned long long>(), PeerDst{(void* const*)table.ptr, (const long long*)rows.ptr}, t0, t1 - t0);
    DF_LAUNCH_CHECK(ctx);
  }
  DF_API_END
}

extern "C" int dfgpu_partition_plan_scatter_peer_chunk(dfgpu_partition_plan* pl, int32_t chunk, void* const* dst_bases, const int64_t* dst_row_offset) {
  if (pl && pl->has_bits()) {
    if (pl->ctx) pl->ctx->last_error = "peer scatter: the plan has a nullable or Boolean column, use dfgpu_partition_plan_scatter_peer_chunk_nullable";
    return DFGPU_ERR_INVALID;
  }
  return dfgpu_partition_plan_scatter_peer_chunk_nullable(pl, chunk, dst_bases, nullptr, dst_row_offset);
}

extern "C" int dfgpu_partition_plan_scatter_peer(dfgpu_partition_plan* pl, void* const* dst_bases, const int64_t* dst_row_offset) {
  if (pl && pl->n_chunks != 1) { if (pl->ctx) pl->ctx->last_error = "peer scatter: plan has several chunks, use dfgpu_partition_plan_scatter_peer_chunk"; return DFGPU_ERR_INVALID; }
  return dfgpu_partition_plan_scatter_peer_chunk(pl, 0, dst_bases, dst_row_offset);
}

extern "C" void dfgpu_partition_plan_destroy(dfgpu_partition_plan* pl) {
  if (!pl) return;
  cudaSetDevice(pl->ctx->device);
  delete pl;
}

// CUDA IPC plumbing: a rank exports its receive buffers once, peers map them and write through NVLink
extern "C" int dfgpu_ipc_export(dfgpu_ctx* ctx, void* dev_ptr, uint8_t* handle_out /* 64 bytes */) {
  DF_API_BEGIN(ctx)
  set_device(ctx);
  cudaIpcMemHandle_t h;
  DF_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &h, 64);
  DF_API_END
}
extern "C" int dfgpu_ipc_import(dfgpu_ctx* ctx, const uint8_t* handle, void** peer_ptr_out) {
  DF_API_BEGIN(ctx)
  set_device(ctx);
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  DF_CUDA(cudaIpcOpenMemHandle(peer_ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  DF_API_END
}
extern "C" int dfgpu_ipc_close(dfgpu_ctx* ctx, void* peer_ptr) {
  DF_API_BEGIN(ctx)
  set_device(ctx);
  if (peer_ptr) DF_CUDA(cudaIpcCloseMemHandle(peer_ptr));
  DF_API_END
}
