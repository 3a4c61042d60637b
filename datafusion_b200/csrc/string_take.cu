// string_take.cu — libdfgpu_strings.so: the gather (arrow-select's `take`) of Utf8, LargeUtf8 and Utf8View rows by a device id column
// (include/dfgpu_strings.h).  It materialises the string columns a plan carried as row ids through its filters and joins.
//
// Utf8 / LargeUtf8 run in two phases because the output size is only known after a pass over the ids and the library does not
// allocate.  Phase 1 (dfgpu_string_take_offsets) resolves each id once: it writes the row's length (-1 for NULL) into the caller's
// 64-bit offsets and the address of its bytes into the scratch, sums the lengths per tile, scans the tile sums and rescans each tile
// into exclusive offsets, writing the output validity on the way.  Phase 2 (dfgpu_string_take_data) reads no id and no source offset
// again: it copies bytes from the recorded addresses, character-parallel — the threads of a block stride over the output words of the
// block's 256 rows and find each byte's row by a binary search over the rows' output offsets in shared memory, so the stores are
// coalesced and the work is even whatever the row lengths.  Utf8View gathers the 16-byte views and rebases an out-of-line view's
// buffer index; no string byte moves.
//
// Source descriptors travel as a kernel parameter, kSources to a launch; more sources take more launches over the same ids, each
// settling the rows of its sources (the first one also the NULL and out-of-range ids).  No kernel reads a byte outside the rows its
// ids name, and none uses TMA: the rows are read at random, there is no tile to stage.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/dfgpu_strings.h"
#include "strings.cuh"

namespace dfgpu {
namespace take {

using like::bit;
using like::fail;
using like::g_error;
using like::launched;
using like::store_validity;

constexpr int kThreads = 256;
constexpr int kRounds = 8;                        // rows per thread of a phase-1 tile, kThreads apart
constexpr int kTileRows = kThreads * kRounds;     // rows per phase-1 tile (one tile sum)
constexpr int kCopyRows = 256;                    // rows per block of the phase-2 byte copy
constexpr int kSources = 64;                      // source arrays one launch reaches (kernel parameters)

struct Source {
  const void* index;         // offsets (int32 / int64) or views
  const uint8_t* data;       // Utf8 / LargeUtf8: the data buffer
  const uint8_t* validity;   // or NULL
  int64_t offset, length;
  int64_t buf_base;          // Utf8View: this source's first buffer in the output's buffer list
};

struct Sources {
  Source s[kSources];
  int32_t lo, count;         // this launch settles sources [lo, lo + count)
  int32_t total;             // sources of the call
};

struct Ids {
  const void* values;        // uint32 rows of source 0, or int64 source << 32 | row
  const uint8_t* validity;
  int64_t offset;
  int32_t packed;
};

enum { kNull = 0, kHere = 1, kElsewhere = 2, kBad = 3 };

// id i -> kNull, kBad (settled by the launch with lo == 0), kElsewhere, or kHere with the launch's source index k and the row
__device__ __forceinline__ int resolve(const Sources& S, const Ids& ids, int64_t i, int& k, int64_t& row) {
  const int64_t at = ids.offset + i;
  const bool first = S.lo == 0;
  if (ids.validity != nullptr && !bit(ids.validity, at)) return first ? kNull : kElsewhere;
  int64_t src;
  if (ids.packed) {
    const uint64_t v = (uint64_t)static_cast<const int64_t*>(ids.values)[at];
    src = (int64_t)(v >> 32);
    row = (int64_t)(v & 0xFFFFFFFFull);
  } else {
    src = 0;
    row = static_cast<const uint32_t*>(ids.values)[at];
  }
  if (src >= S.total) return first ? kBad : kElsewhere;
  if (src < S.lo || src >= S.lo + S.count) return kElsewhere;
  k = (int)(src - S.lo);
  if (row >= S.s[k].length) return kBad;
  return kHere;
}

template <typename T>
__device__ __forceinline__ T block_sum(T v) {
  __shared__ T red[kThreads / 32];
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T r = 0;
  if (threadIdx.x < 32) {
    r = threadIdx.x < kThreads / 32 ? red[threadIdx.x] : T(0);
    for (int d = 16; d > 0; d >>= 1) r += __shfl_xor_sync(0xffffffffu, r, d);
  }
  return r;   // valid in thread 0
}

// exclusive scan of one value per thread over the block; *total = the block's sum
__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t* total) {
  __shared__ int64_t warp_sums[kThreads / 32 + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t incl = v;
  for (int d = 1; d < 32; d <<= 1) {
    const int64_t o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  __syncthreads();
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const int64_t w = lane < kThreads / 32 ? warp_sums[lane] : 0;
    int64_t wi = w;
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t o = __shfl_up_sync(0xffffffffu, wi, d);
      if (lane >= d) wi += o;
    }
    if (lane < kThreads / 32) warp_sums[lane] = wi - w;
    if (lane == kThreads / 32 - 1) warp_sums[kThreads / 32] = wi;
  }
  __syncthreads();
  *total = warp_sums[kThreads / 32];
  return warp_sums[warp] + incl - v;
}

// phase 1a, once per source range: each row of this launch's sources -> lens[i] (-1 = NULL) and src[i]; the tile's length sum is
// added to tile_sums[tile]; out-of-range ids are counted in status[1]
template <typename Off>
__global__ void __launch_bounds__(kThreads) take_lengths_kernel(const __grid_constant__ Sources S, const Ids ids, int64_t n,
                                                                int64_t* __restrict__ lens, const uint8_t** __restrict__ src,
                                                                unsigned long long* __restrict__ tile_sums,
                                                                unsigned long long* __restrict__ status) {
  const int64_t base = (int64_t)blockIdx.x * kTileRows;
  unsigned long long sum = 0, bad = 0;
  for (int r = 0; r < kRounds; ++r) {
    const int64_t i = base + (int64_t)r * kThreads + threadIdx.x;
    if (i >= n) break;
    int k = 0;
    int64_t row = 0;
    const int how = resolve(S, ids, i, k, row);
    if (how == kElsewhere) continue;
    int64_t len = -1;
    const uint8_t* p = nullptr;
    if (how == kHere) {
      const Source& s = S.s[k];
      const int64_t at = s.offset + row;
      if (s.validity == nullptr || bit(s.validity, at)) {
        const Off* o = static_cast<const Off*>(s.index);
        const int64_t a = (int64_t)o[at];
        len = (int64_t)o[at + 1] - a;
        p = s.data + a;
        sum += (unsigned long long)len;
      }
    }
    bad += how == kBad;
    lens[i] = len;
    src[i] = p;
  }
  sum = block_sum(sum);
  __syncthreads();
  bad = block_sum(bad);
  if (threadIdx.x == 0) {
    if (sum) atomicAdd(&tile_sums[blockIdx.x], sum);
    if (bad) atomicAdd(&status[1], bad);
  }
}

// phase 1b, one block: tile_sums[0 .. n_tiles) -> their exclusive scan, in place; status[0] = the total
__global__ void __launch_bounds__(kThreads) take_scan_tiles_kernel(unsigned long long* __restrict__ tile_sums, int64_t n_tiles,
                                                                   unsigned long long* __restrict__ status) {
  int64_t carry = 0;
  for (int64_t b = 0; b < n_tiles; b += kThreads) {
    const int64_t i = b + threadIdx.x;
    const int64_t v = i < n_tiles ? (int64_t)tile_sums[i] : 0;
    int64_t tot;
    const int64_t ex = block_exclusive_scan(v, &tot);
    if (i < n_tiles) tile_sums[i] = (unsigned long long)(carry + ex);
    carry += tot;
  }
  if (threadIdx.x == 0) status[0] = (unsigned long long)carry;
}

// phase 1c: lens -> exclusive offsets in place (a NULL row takes 0 bytes), the output validity at bit 0, NULL rows counted in status[2]
__global__ void __launch_bounds__(kThreads) take_offsets_kernel(int64_t n, int64_t* __restrict__ offs,
                                                                const unsigned long long* __restrict__ tile_sums,
                                                                uint8_t* __restrict__ out_valid, unsigned long long* __restrict__ status) {
  const int64_t base = (int64_t)blockIdx.x * kTileRows;
  int64_t carry = (int64_t)tile_sums[blockIdx.x];
  unsigned long long nulls = 0;
  for (int r = 0; r < kRounds && base + (int64_t)r * kThreads < n; ++r) {   // the bound is uniform over the block
    const int64_t row0 = base + (int64_t)r * kThreads, i = row0 + threadIdx.x;
    const int64_t len = i < n ? offs[i] : 0;
    const bool valid = i < n && len >= 0;
    nulls += i < n && len < 0;
    int64_t tot;
    const int64_t ex = block_exclusive_scan(valid ? len : 0, &tot);
    if (i < n) offs[i] = carry + ex;
    store_validity(out_valid, row0 + (threadIdx.x & ~31), n, valid);
    carry += tot;
  }
  __syncthreads();
  nulls = block_sum(nulls);
  if (threadIdx.x == 0 && nulls) atomicAdd(&status[2], nulls);
}

// phase 2: block b copies the bytes of rows [b * kCopyRows, ...), aligned output words with 32-bit stores, the unaligned head and tail
// of its byte range with byte stores (a word shared with a neighbouring block gets each byte from exactly one block); the output
// offsets are written as OutOff unless out_off is NULL (LargeUtf8 output offsets are `offs` itself)
template <typename OutOff>
__global__ void __launch_bounds__(kThreads) take_copy_kernel(int64_t n, const int64_t* __restrict__ offs, const uint8_t* const* __restrict__ src,
                                                             OutOff* __restrict__ out_off, uint8_t* __restrict__ out) {
  __shared__ int64_t dst[kCopyRows + 1];
  __shared__ const uint8_t* sp[kCopyRows];
  const int64_t r0 = (int64_t)blockIdx.x * kCopyRows;
  const int rows = (int)(n - r0 < kCopyRows ? n - r0 : kCopyRows);
  const int t = threadIdx.x;
  for (int j = t; j <= rows; j += kThreads) {
    const int64_t o = offs[r0 + j];          // offs[n] is the total
    dst[j] = o;
    if (j < rows) sp[j] = src[r0 + j];
    if (out_off != nullptr && (j < rows || r0 + j == n)) out_off[r0 + j] = (OutOff)o;
  }
  __syncthreads();
  const int64_t b0 = dst[0], b1 = dst[rows];
  // the row holding output byte b: the last row whose offset is <= b (an empty row shares its offset with the next one)
  auto row_of = [&](int64_t b) {
    int lo = 0, hi = rows - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (dst[mid] <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
  };
  const int64_t w0 = (b0 + 3) & ~(int64_t)3, w1 = b1 & ~(int64_t)3;
  if (w0 >= w1) {
    for (int64_t b = b0 + t; b < b1; b += kThreads) {
      const int r = row_of(b);
      out[b] = sp[r][b - dst[r]];
    }
    return;
  }
  if (t < w0 - b0) {
    const int64_t b = b0 + t;
    const int r = row_of(b);
    out[b] = sp[r][b - dst[r]];
  }
  if (t < b1 - w1) {
    const int64_t b = w1 + t;
    const int r = row_of(b);
    out[b] = sp[r][b - dst[r]];
  }
  for (int64_t w = w0 + 4 * (int64_t)t; w < w1; w += 4 * kThreads) {
    int r = row_of(w);
    uint32_t word = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      while (dst[r + 1] <= w + j) ++r;
      word |= (uint32_t)sp[r][w + j - dst[r]] << (8 * j);
    }
    *reinterpret_cast<uint32_t*>(out + w) = word;
  }
}

// Utf8View, once per source range: the rows of this launch's sources -> their views (an out-of-line view's buffer index rebased), a
// NULL or out-of-range row -> a zero view; validity bits ORed into the zeroed out_valid words; status[0] out-of-range ids, status[1]
// NULL rows
__global__ void __launch_bounds__(kThreads) take_views_kernel(const __grid_constant__ Sources S, const Ids ids, int64_t n,
                                                              uint4* __restrict__ out, uint32_t* __restrict__ out_valid,
                                                              unsigned long long* __restrict__ status) {
  unsigned long long bad = 0, nulls = 0;
  for (int64_t base = (int64_t)blockIdx.x * kThreads; base < n; base += (int64_t)gridDim.x * kThreads) {   // uniform over the block
    const int64_t i = base + threadIdx.x;
    bool valid = false;
    if (i < n) {
      int k = 0;
      int64_t row = 0;
      const int how = resolve(S, ids, i, k, row);
      if (how != kElsewhere) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if (how == kHere) {
          const Source& s = S.s[k];
          const int64_t at = s.offset + row;
          if (s.validity == nullptr || bit(s.validity, at)) {
            v = static_cast<const uint4*>(s.index)[at];
            if (v.x > 12) v.z += (uint32_t)s.buf_base;
            valid = true;
          }
        }
        bad += how == kBad;
        nulls += !valid;
        out[i] = v;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0 && m) atomicOr(&out_valid[i >> 5], m);
  }
  bad = block_sum(bad);
  __syncthreads();
  nulls = block_sum(nulls);
  if (threadIdx.x == 0) {
    if (bad) atomicAdd(&status[0], bad);
    if (nulls) atomicAdd(&status[1], nulls);
  }
}

// ---- host ----
template <typename Kernel>
unsigned grid_cap(Kernel kernel, int64_t n, int64_t rows_per_block) {
  int dev = 0, sms = 1, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0);
  const int64_t need = (n + rows_per_block - 1) / rows_per_block, cap = (int64_t)sms * (per_sm > 0 ? per_sm : 1);
  return (unsigned)(need < cap ? need : cap);
}

int64_t n_tiles(int64_t n) { return n > 0 ? (n + kTileRows - 1) / kTileRows : 1; }

// the sources and ids of a call: DFGPU_OK or DFGPU_ERR_INVALID
int check_args(const char* what, const dfgpu_string_column* sources, int32_t n_sources, const dfgpu_column* ids, bool views) {
  const std::string w(what);
  if (sources == nullptr || n_sources < 1) return fail(DFGPU_ERR_INVALID, w + ": no source");
  if (ids == nullptr || ids->length < 0 || ids->offset < 0) return fail(DFGPU_ERR_INVALID, w + ": no id column");
  if (ids->type != DFGPU_UINT32 && ids->type != DFGPU_INT64) return fail(DFGPU_ERR_INVALID, w + ": ids are UINT32 or INT64");
  if (ids->length > 0 && ids->values == nullptr) return fail(DFGPU_ERR_INVALID, w + ": missing id values");
  for (int32_t s = 0; s < n_sources; ++s) {
    const dfgpu_string_column& c = sources[s];
    const std::string at = w + ": source " + std::to_string(s);
    if (views ? c.layout != DFGPU_STRING_UTF8_VIEW : (c.layout != DFGPU_STRING_UTF8 && c.layout != DFGPU_STRING_LARGE_UTF8))
      return fail(DFGPU_ERR_INVALID, at + (views ? ": not a Utf8View array" : ": not a Utf8 / LargeUtf8 array"));
    if (c.layout != sources[0].layout) return fail(DFGPU_ERR_INVALID, at + ": sources differ in layout");
    if (c.length < 0 || c.offset < 0 || c.length > 0xFFFFFFFFll) return fail(DFGPU_ERR_INVALID, at + ": bad length or offset");
    if (c.length == 0) continue;
    if (c.offsets_or_views == nullptr) return fail(DFGPU_ERR_INVALID, at + ": missing offsets or views");
    if (views) {
      if (reinterpret_cast<uintptr_t>(c.offsets_or_views) & 15) return fail(DFGPU_ERR_INVALID, at + ": Utf8View views must be 16-byte aligned");
      if (c.n_data_buffers < 0 || (c.n_data_buffers > 0 && c.data_buffers == nullptr)) return fail(DFGPU_ERR_INVALID, at + ": Utf8View data buffers missing");
    } else if (c.n_data_buffers != 1 || c.data_buffers == nullptr) {
      return fail(DFGPU_ERR_INVALID, at + ": a Utf8 array has one data buffer");
    }
  }
  return DFGPU_OK;
}

Ids ids_of(const dfgpu_column* ids) {
  Ids d;
  d.values = ids->values;
  d.validity = ids->validity;
  d.offset = ids->offset;
  d.packed = ids->type == DFGPU_INT64;
  return d;
}

// launch(S) once per range of kSources sources, S.lo == 0 on the first launch; buf_base: the running count of Utf8View buffers
template <typename Launch>
int for_each_source_range(const char* what, const dfgpu_string_column* sources, int32_t n_sources, Launch launch) {
  int64_t buf_base = 0;
  for (int32_t lo = 0; lo < n_sources; lo += kSources) {
    Sources S;
    memset(&S, 0, sizeof(S));
    S.lo = lo;
    S.count = n_sources - lo < kSources ? n_sources - lo : kSources;
    S.total = n_sources;
    for (int k = 0; k < S.count; ++k) {
      const dfgpu_string_column& c = sources[lo + k];
      S.s[k].index = c.offsets_or_views;
      S.s[k].data = c.layout == DFGPU_STRING_UTF8_VIEW || c.length == 0 ? nullptr : c.data_buffers[0];
      S.s[k].validity = c.validity;
      S.s[k].offset = c.offset;
      S.s[k].length = c.length;
      S.s[k].buf_base = buf_base;
      if (c.layout == DFGPU_STRING_UTF8_VIEW) buf_base += c.n_data_buffers;
    }
    launch(S);
    const int rc = launched(what);
    if (rc != DFGPU_OK) return rc;
  }
  return DFGPU_OK;
}

int cuda_ok(cudaError_t e, const char* what) {
  if (e != cudaSuccess) return fail(DFGPU_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
  return DFGPU_OK;
}

}  // namespace take
}  // namespace dfgpu

using namespace dfgpu::take;

extern "C" int64_t dfgpu_string_take_scratch_bytes(int64_t n_ids) {
  return n_tiles(n_ids) * 8 + (n_ids > 0 ? n_ids : 0) * 8;
}

extern "C" int dfgpu_string_take_offsets(void* stream, const dfgpu_string_column* sources, int32_t n_sources, const dfgpu_column* ids,
                                         void* scratch, int64_t* offsets, uint8_t* out_validity) {
  g_error.clear();
  const char* what = "dfgpu_string_take_offsets";
  int rc = check_args(what, sources, n_sources, ids, false);
  if (rc != DFGPU_OK) return rc;
  const int64_t n = ids->length;
  if (offsets == nullptr || (n > 0 && (scratch == nullptr || out_validity == nullptr)))
    return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_offsets: missing buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned long long* status = reinterpret_cast<unsigned long long*>(offsets + n);
  if ((rc = cuda_ok(cudaMemsetAsync(offsets + n, 0, 3 * sizeof(int64_t), st), what)) != DFGPU_OK) return rc;
  if (n == 0) return cuda_ok(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st), what);
  const int64_t tiles = n_tiles(n);
  unsigned long long* tile_sums = static_cast<unsigned long long*>(scratch);
  const uint8_t** src = reinterpret_cast<const uint8_t**>(tile_sums + tiles);
  if ((rc = cuda_ok(cudaMemsetAsync(tile_sums, 0, tiles * 8, st), what)) != DFGPU_OK) return rc;
  const Ids d = ids_of(ids);
  const bool large = sources[0].layout == DFGPU_STRING_LARGE_UTF8;
  rc = for_each_source_range(what, sources, n_sources, [&](const Sources& S) {
    if (large) take_lengths_kernel<int64_t><<<(unsigned)tiles, kThreads, 0, st>>>(S, d, n, offsets, src, tile_sums, status);
    else take_lengths_kernel<int32_t><<<(unsigned)tiles, kThreads, 0, st>>>(S, d, n, offsets, src, tile_sums, status);
  });
  if (rc != DFGPU_OK) return rc;
  take_scan_tiles_kernel<<<1, kThreads, 0, st>>>(tile_sums, tiles, status);
  if ((rc = launched(what)) != DFGPU_OK) return rc;
  take_offsets_kernel<<<(unsigned)tiles, kThreads, 0, st>>>(n, offsets, tile_sums, out_validity, status);
  return launched(what);
}

extern "C" int dfgpu_string_take_data(void* stream, int32_t layout, int64_t n_ids, int64_t total_bytes, const void* scratch,
                                      const int64_t* offsets, void* out_offsets, uint8_t* out_data) {
  g_error.clear();
  if (layout != DFGPU_STRING_UTF8 && layout != DFGPU_STRING_LARGE_UTF8) return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_data: not a Utf8 / LargeUtf8 layout");
  if (n_ids < 0 || total_bytes < 0) return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_data: bad size");
  if (layout == DFGPU_STRING_UTF8 && total_bytes > INT32_MAX)
    return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_data: offset overflow (" + std::to_string(total_bytes) + " bytes do not fit a Utf8 array)");
  if (offsets == nullptr || out_offsets == nullptr || (total_bytes > 0 && out_data == nullptr) || (n_ids > 0 && scratch == nullptr))
    return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_data: missing buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n_ids == 0) {
    if (out_offsets == offsets) return DFGPU_OK;
    return cuda_ok(cudaMemsetAsync(out_offsets, 0, layout == DFGPU_STRING_UTF8 ? 4 : 8, st), "dfgpu_string_take_data");
  }
  const uint8_t* const* src = reinterpret_cast<const uint8_t* const*>(static_cast<const unsigned long long*>(scratch) + n_tiles(n_ids));
  const unsigned grid = (unsigned)((n_ids + kCopyRows - 1) / kCopyRows);
  if (layout == DFGPU_STRING_UTF8)
    take_copy_kernel<int32_t><<<grid, kThreads, 0, st>>>(n_ids, offsets, src, static_cast<int32_t*>(out_offsets), out_data);
  else
    take_copy_kernel<int64_t><<<grid, kThreads, 0, st>>>(n_ids, offsets, src, out_offsets == offsets ? nullptr : static_cast<int64_t*>(out_offsets), out_data);
  return launched("dfgpu_string_take_data");
}

extern "C" int dfgpu_string_take_views(void* stream, const dfgpu_string_column* sources, int32_t n_sources, const dfgpu_column* ids,
                                       void* out_views, uint8_t* out_validity, int64_t* status) {
  g_error.clear();
  const char* what = "dfgpu_string_take_views";
  int rc = check_args(what, sources, n_sources, ids, true);
  if (rc != DFGPU_OK) return rc;
  const int64_t n = ids->length;
  if (status == nullptr || (n > 0 && (out_views == nullptr || out_validity == nullptr)))
    return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_views: missing buffer");
  if ((reinterpret_cast<uintptr_t>(out_views) & 15) || (reinterpret_cast<uintptr_t>(out_validity) & 3))
    return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_views: out_views must be 16-byte and out_validity 4-byte aligned");
  int64_t buffers = 0;
  for (int32_t s = 0; s < n_sources; ++s) buffers += sources[s].n_data_buffers;
  if (buffers > INT32_MAX) return fail(DFGPU_ERR_INVALID, "dfgpu_string_take_views: more than 2^31 - 1 data buffers");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = cuda_ok(cudaMemsetAsync(status, 0, 2 * sizeof(int64_t), st), what)) != DFGPU_OK) return rc;
  if (n == 0) return DFGPU_OK;
  if ((rc = cuda_ok(cudaMemsetAsync(out_validity, 0, (size_t)((n + 31) / 32) * 4, st), what)) != DFGPU_OK) return rc;
  const Ids d = ids_of(ids);
  const unsigned grid = grid_cap(take_views_kernel, n, kThreads);
  return for_each_source_range(what, sources, n_sources, [&](const Sources& S) {
    take_views_kernel<<<grid, kThreads, 0, st>>>(S, d, n, static_cast<uint4*>(out_views), reinterpret_cast<uint32_t*>(out_validity),
                                                 reinterpret_cast<unsigned long long*>(status));
  });
}
