// like.cu — libdfgpu_strings.so: LIKE / NOT LIKE over Utf8, LargeUtf8, Utf8View and dictionary codes (include/dfgpu_strings.h).
//
// The host compiles a pattern into an anchored prefix, middle segments and an anchored suffix (the pieces between `%`); a segment is
// literal bytes and `_` tokens.  A row matches when the prefix matches at its start, the suffix at its end (not overlapping the
// prefix), and every middle segment in order in between.  Middle segments are found leftmost-first, which is exact: a segment always
// spans the same number of code points, so its leftmost occurrence also ends leftmost and leaves the most room for the rest.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/dfgpu_strings.h"
#include "strings.cuh"
#include "tma.cuh"

namespace dfgpu {
namespace like {

constexpr uint8_t kAny = 0xFF;       // `_` in a compiled segment: 0xFF is never a byte of valid UTF-8
constexpr int kMaxSegs = DFGPU_LIKE_MAX_SEGMENTS + 2;   // prefix and suffix may be empty

struct Program {
  uint8_t bytes[DFGPU_LIKE_MAX_PATTERN_BYTES];   // the segments back to back, `_` as kAny
  uint16_t seg_off[kMaxSegs + 1];                 // segment s is bytes[seg_off[s], seg_off[s + 1])
  uint16_t seg_min[kMaxSegs];                     // fewest string bytes segment s can match
  int32_t n_mid;         // middle segments: 1 .. n_mid (prefix 0, suffix n_mid + 1)
  int32_t has_pct;       // 0: no `%`, segment 0 must match the whole string
  int32_t min_bytes;     // fewest string bytes any match needs
  int32_t negated;
  uint32_t view_prefix;  // the prefix's leading literal bytes (up to 4, before any `_`), little-endian, for a Utf8View's inline prefix
  uint32_t view_mask;
};

constexpr int kTileRows = 512;                  // rows of one Utf8 tile (one block)
constexpr int kStageBytes = 40 * 1024;          // shared-memory stage of one tile's bytes (512 TPC-H comments of up to 78 bytes fit)
constexpr int kLongRow = 512;                   // longer rows are matched by a whole warp

__device__ __forceinline__ int cp_len(uint8_t b) { return b < 0x80 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4; }

// segment [a, b) forward at s[pos], within s[0, n): end position, or -1
__device__ __forceinline__ int64_t fwd(const Program& P, int a, int b, const uint8_t* s, int64_t pos, int64_t n) {
  for (int i = a; i < b; ++i) {
    if (pos >= n) return -1;
    const uint8_t c = P.bytes[i], t = s[pos];
    if (c == kAny) pos += cp_len(t);
    else if (t != c) return -1;
    else ++pos;
  }
  return pos <= n ? pos : -1;
}

// segment [a, b) backward, ending at s[hi) and starting at or after lo (a code-point boundary): start position, or -1
__device__ __forceinline__ int64_t bwd(const Program& P, int a, int b, const uint8_t* s, int64_t lo, int64_t hi) {
  int64_t pos = hi;
  for (int i = b - 1; i >= a; --i) {
    if (pos <= lo) return -1;
    const uint8_t c = P.bytes[i];
    --pos;
    if (c == kAny) {
      while (pos > lo && (s[pos] & 0xC0) == 0x80) --pos;
    } else if (s[pos] != c) {
      return -1;
    }
  }
  return pos;
}

// can middle segment m start at s[p]?  (its first literal byte, or a code-point boundary for a leading `_`)
__device__ __forceinline__ bool may_start(uint8_t c0, uint8_t t) { return c0 == kAny ? (t & 0xC0) != 0x80 : t == c0; }

// the anchored ends: [lo, hi) is what the middle segments may use; false when an end does not match
__device__ __forceinline__ bool match_ends(const Program& P, const uint8_t* s, int64_t n, int64_t& lo, int64_t& hi) {
  if (n < P.min_bytes) return false;
  lo = fwd(P, P.seg_off[0], P.seg_off[1], s, 0, n);
  if (!P.has_pct) return lo == n;
  if (lo < 0) return false;
  const int last = P.n_mid + 1;
  hi = bwd(P, P.seg_off[last], P.seg_off[last + 1], s, lo, n);
  return hi >= 0;
}

// one thread, one row
__device__ bool match_row(const Program& P, const uint8_t* s, int64_t n) {
  int64_t lo, hi;
  if (!match_ends(P, s, n, lo, hi)) return false;
  if (!P.has_pct) return true;
  for (int m = 1; m <= P.n_mid; ++m) {
    const int a = P.seg_off[m], b = P.seg_off[m + 1];
    const uint8_t c0 = P.bytes[a];
    int64_t found = -1;
    for (int64_t p = lo; p + P.seg_min[m] <= hi; ++p) {
      if (!may_start(c0, s[p])) continue;
      found = fwd(P, a, b, s, p, hi);
      if (found >= 0) break;
    }
    if (found < 0) return false;
    lo = found;
  }
  return true;
}

// a whole (converged) warp, one row: the ends redundantly in every lane, each middle segment tried at 32 positions at a time
__device__ bool match_row_warp(const Program& P, const uint8_t* s, int64_t n) {
  const int lane = threadIdx.x & 31;
  int64_t lo, hi;
  if (!match_ends(P, s, n, lo, hi)) return false;
  if (!P.has_pct) return true;
  for (int m = 1; m <= P.n_mid; ++m) {
    const int a = P.seg_off[m], b = P.seg_off[m + 1];
    const uint8_t c0 = P.bytes[a];
    int64_t found = -1;
    for (int64_t base = lo; base + P.seg_min[m] <= hi; base += 32) {
      const int64_t p = base + lane;
      int64_t e = -1;
      if (p + P.seg_min[m] <= hi && may_start(c0, s[p])) e = fwd(P, a, b, s, p, hi);
      const unsigned hit = __ballot_sync(0xffffffffu, e >= 0);
      if (hit) {
        found = __shfl_sync(0xffffffffu, e, __ffs(hit) - 1);
        break;
      }
    }
    if (found < 0) return false;
    lo = found;
  }
  return true;
}

// Utf8 / LargeUtf8: one block per tile of kTileRows rows.  The tile's rows are contiguous in the data buffer, so its byte range
// [offsets[r0], offsets[r1]) is staged into shared memory when it fits: the 16-byte-aligned interior by one TMA bulk copy, the
// unaligned head and tail bytes by the threads.  A tile that does not fit is matched from global memory.  Thread t of the block takes
// rows t, t + 256 of the tile, so a warp's rows are 32 consecutive ones (one validity word).
template <typename Off>
__global__ void __launch_bounds__(kThreads) like_utf8_kernel(const __grid_constant__ Program prog_in, const Off* __restrict__ offsets,
                                                             const uint8_t* __restrict__ data, const uint8_t* __restrict__ validity,
                                                             int64_t in_off, int64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  extern __shared__ __align__(128) uint8_t stage[];
  __shared__ Program P;
  __shared__ Off so[kTileRows + 1];
  __shared__ __align__(8) uint64_t bar;
  const int64_t r0 = (int64_t)blockIdx.x * kTileRows;
  const int rows = (int)min((int64_t)kTileRows, n - r0);
  load_program(P, prog_in);
  for (int i = threadIdx.x; i <= rows; i += kThreads) so[i] = offsets[in_off + r0 + i];
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uintptr_t a0 = (uintptr_t)(data + so[0]), a1 = (uintptr_t)(data + so[rows]);
  const uintptr_t base = a0 & ~(uintptr_t)15;
  const bool staged = a1 - base <= (uintptr_t)kStageBytes;
  if (staged) {
    const uintptr_t ai = (a0 + 15) & ~(uintptr_t)15, ae = a1 & ~(uintptr_t)15;
    const bool bulk = ae > ai;
    if (bulk && threadIdx.x == 0) {
      mbar_expect_tx(&bar, (uint32_t)(ae - ai));
      tma_load_1d(stage + (ai - base), reinterpret_cast<const void*>(ai), (uint32_t)(ae - ai), &bar);
    }
    const uintptr_t head_end = ai < a1 ? ai : a1, tail_begin = bulk ? ae : head_end;
    for (uintptr_t a = a0 + threadIdx.x; a < head_end; a += kThreads) stage[a - base] = *reinterpret_cast<const uint8_t*>(a);
    for (uintptr_t a = tail_begin + threadIdx.x; a < a1; a += kThreads) stage[a - base] = *reinterpret_cast<const uint8_t*>(a);
    if (bulk) mbar_wait(&bar, 0);
    __syncthreads();
  }
  const uint8_t* src = staged ? stage + (a0 - base) : data + so[0];   // byte so[i] - so[0] of src is row i's first byte
  const int lane = threadIdx.x & 31, warp0 = threadIdx.x & ~31;
#pragma unroll 1
  for (int k = 0; k < kTileRows / kThreads; ++k) {
    const int i = k * kThreads + threadIdx.x;
    if (k * kThreads + warp0 >= rows) break;                          // warp-uniform
    const bool in = i < rows;
    const int64_t row = r0 + i;
    const bool valid = in && (validity == nullptr || bit(validity, in_off + row));
    const int64_t len = in ? (int64_t)(so[i + 1] - so[i]) : 0;
    bool hit = valid && len <= kLongRow && match_row(P, src + (so[i] - so[0]), len);
    unsigned longs = __ballot_sync(0xffffffffu, valid && len > kLongRow);
    while (longs) {
      const int l = __ffs(longs) - 1;
      longs &= longs - 1;
      const int j = k * kThreads + warp0 + l;
      const bool h = match_row_warp(P, src + (so[j] - so[0]), (int64_t)(so[j + 1] - so[j]));
      if (lane == l) hit = h;
    }
    if (in) out[row] = valid ? (uint8_t)(hit != (P.negated != 0)) : 0;
    if (out_valid != nullptr) store_validity(out_valid, r0 + k * kThreads + warp0, n, valid);
  }
}

// Utf8View: one thread per row.  A string of at most 12 bytes is matched from its view; a longer one first against the view's 4-byte
// prefix (an anchored-prefix mismatch is settled without reading its buffer), then from its data buffer.  With more data buffers than
// one launch's parameters hold, launch g matches the rows whose buffer is in its range; launch 0 also writes every row no buffer
// decides and the validity.
__global__ void __launch_bounds__(kThreads) like_view_kernel(const __grid_constant__ Program prog_in, const __grid_constant__ ViewBufs bufs,
                                                             const uint4* __restrict__ views, const uint8_t* __restrict__ validity,
                                                             int64_t in_off, int64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  __shared__ Program P;
  load_program(P, prog_in);
  __syncthreads();
  const int64_t row0 = (int64_t)blockIdx.x * kThreads + (threadIdx.x & ~31);
  const int64_t row = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  const int lane = threadIdx.x & 31;
  if (row0 >= n) return;                                              // warp-uniform
  const bool in = row < n;
  const bool valid = in && (validity == nullptr || bit(validity, in_off + row));
  const bool first = bufs.lo == 0;
  bool hit = false, write = false;
  const uint8_t* s = nullptr;
  int64_t len = 0;
  if (valid) {
    const uint4 v = views[in_off + row];
    len = (int64_t)v.x;
    if (len <= 12) {
      s = reinterpret_cast<const uint8_t*>(views + in_off + row) + 4;
      write = first;
    } else if ((v.y & P.view_mask) != P.view_prefix || len < P.min_bytes) {
      write = first;
    } else if ((int32_t)v.z >= bufs.lo && (int32_t)v.z < bufs.lo + bufs.count) {
      s = bufs.ptr[(int32_t)v.z - bufs.lo] + v.w;
      write = true;
    }
  } else {
    write = in && first;
  }
  if (s != nullptr && len <= kLongRow) hit = match_row(P, s, len);
  unsigned longs = __ballot_sync(0xffffffffu, s != nullptr && len > kLongRow);
  while (longs) {
    const int l = __ffs(longs) - 1;
    longs &= longs - 1;
    const uint8_t* sl = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, (unsigned long long)s, l));
    const int64_t nl = __shfl_sync(0xffffffffu, len, l);
    const bool h = match_row_warp(P, sl, nl);
    if (lane == l) hit = h;
  }
  if (write) out[row] = valid ? (uint8_t)(hit != (P.negated != 0)) : 0;
  if (first && out_valid != nullptr) store_validity(out_valid, row0, n, valid);
}

// dictionary codes: out[i] = match[codes[i]] (any predicate evaluated over the dictionary's distinct values)
__global__ void __launch_bounds__(kThreads) like_codes_kernel(const int32_t* __restrict__ codes, const uint8_t* __restrict__ validity, int64_t in_off,
                                                              int64_t n, const uint8_t* __restrict__ match, int64_t n_codes,
                                                              uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  const int64_t row0 = (int64_t)blockIdx.x * kThreads + (threadIdx.x & ~31);
  const int64_t row = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (row0 >= n) return;
  const bool in = row < n;
  const bool valid = in && (validity == nullptr || bit(validity, in_off + row));
  if (in) {
    const int32_t c = valid ? codes[in_off + row] : -1;
    out[row] = (c >= 0 && c < n_codes) ? match[c] : 0;
  }
  if (out_valid != nullptr) store_validity(out_valid, row0, n, valid);
}

// ---- host ----
int compile(const uint8_t* pat, int64_t len, int32_t flags, Program& P) {
  if (flags & ~(DFGPU_LIKE_NEGATED | DFGPU_LIKE_CASE_INSENSITIVE)) return fail(DFGPU_ERR_INVALID, "dfgpu_like: unknown flags");
  if (flags & DFGPU_LIKE_CASE_INSENSITIVE)
    return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_like: ILIKE (case-insensitive LIKE) is not supported on the GPU: it needs Unicode case folding");
  if (len < 0 || (len > 0 && pat == nullptr)) return fail(DFGPU_ERR_INVALID, "dfgpu_like: no pattern");
  const int64_t bad = utf8_invalid_at(pat, len);
  if (bad >= 0) return fail(DFGPU_ERR_INVALID, "dfgpu_like: the pattern is not valid UTF-8 (byte " + std::to_string(bad) + ")");
  if (memchr(pat, '\\', (size_t)len) != nullptr)
    return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_like: a pattern with an escape character (\\) is not supported on the GPU");
  if (len > DFGPU_LIKE_MAX_PATTERN_BYTES)
    return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_like: the pattern is longer than " + std::to_string(DFGPU_LIKE_MAX_PATTERN_BYTES) + " bytes");
  memset(&P, 0, sizeof(P));
  // pieces between `%`: [begin, end) byte ranges of the pattern
  int64_t piece_b[DFGPU_LIKE_MAX_PATTERN_BYTES + 1], piece_e[DFGPU_LIKE_MAX_PATTERN_BYTES + 1];
  int n_pieces = 0;
  int64_t b = 0;
  for (int64_t i = 0; i <= len; ++i)
    if (i == len || pat[i] == '%') { piece_b[n_pieces] = b; piece_e[n_pieces] = i; ++n_pieces; b = i + 1; }
  int nonempty = 0;
  for (int p = 0; p < n_pieces; ++p) nonempty += piece_e[p] > piece_b[p];
  if (nonempty > DFGPU_LIKE_MAX_SEGMENTS)
    return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_like: the pattern has more than " + std::to_string(DFGPU_LIKE_MAX_SEGMENTS) + " %-separated segments");
  P.has_pct = n_pieces > 1;
  int n_seg = 0, at = 0;
  auto add = [&](int p) {
    P.seg_off[n_seg] = (uint16_t)at;
    int mn = 0;
    for (int64_t i = piece_b[p]; i < piece_e[p]; ++i) {
      if (pat[i] == '_') { P.bytes[at++] = kAny; ++mn; }
      else { P.bytes[at++] = pat[i]; ++mn; }
    }
    P.seg_min[n_seg] = (uint16_t)mn;
    P.min_bytes += mn;
    ++n_seg;
  };
  add(0);                                                         // prefix (the whole pattern without `%`)
  if (P.has_pct) {
    for (int p = 1; p + 1 < n_pieces; ++p)
      if (piece_e[p] > piece_b[p]) add(p);                        // non-empty middles
    P.n_mid = n_seg - 1;
    add(n_pieces - 1);                                            // suffix
  }
  P.seg_off[n_seg] = (uint16_t)at;
  for (int i = 0; i < 4 && i < P.seg_off[1] && P.bytes[i] != kAny; ++i) {
    P.view_prefix |= (uint32_t)P.bytes[i] << (8 * i);
    P.view_mask |= 0xFFu << (8 * i);
  }
  P.negated = (flags & DFGPU_LIKE_NEGATED) != 0;
  return DFGPU_OK;
}

}  // namespace like
}  // namespace dfgpu

using namespace dfgpu::like;

extern "C" const char* dfgpu_strings_last_error(void) { return g_error.c_str(); }

extern "C" int dfgpu_like(void* stream, const dfgpu_string_column* col, const uint8_t* pattern, int64_t pattern_len, int32_t flags,
                          uint8_t* out_values, uint8_t* out_validity) {
  g_error.clear();
  Program P;
  int rc = compile(pattern, pattern_len, flags, P);
  if (rc != DFGPU_OK) return rc;
  if (col == nullptr || col->length < 0 || col->offset < 0) return fail(DFGPU_ERR_INVALID, "dfgpu_like: no column");
  if (col->length == 0) return DFGPU_OK;
  if ((rc = check_column(col, out_values, out_validity, col->validity != nullptr, "dfgpu_like")) != DFGPU_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ov = col->validity != nullptr ? out_validity : nullptr;
  const int64_t n = col->length;
  if (col->layout == DFGPU_STRING_UTF8 || col->layout == DFGPU_STRING_LARGE_UTF8) {
    const unsigned grid = (unsigned)((n + kTileRows - 1) / kTileRows);
    if (col->layout == DFGPU_STRING_UTF8)
      like_utf8_kernel<int32_t><<<grid, kThreads, kStageBytes, st>>>(P, static_cast<const int32_t*>(col->offsets_or_views), col->data_buffers[0],
                                                                     col->validity, col->offset, n, out_values, ov);
    else
      like_utf8_kernel<int64_t><<<grid, kThreads, kStageBytes, st>>>(P, static_cast<const int64_t*>(col->offsets_or_views), col->data_buffers[0],
                                                                     col->validity, col->offset, n, out_values, ov);
    return launched("dfgpu_like");
  }
  const unsigned grid = (unsigned)((n + kThreads - 1) / kThreads);
  return for_each_view_range(col, "dfgpu_like", [&](const ViewBufs& vb) {
    like_view_kernel<<<grid, kThreads, 0, st>>>(P, vb, static_cast<const uint4*>(col->offsets_or_views), col->validity, col->offset, n,
                                                out_values, ov);
  });
}

extern "C" int dfgpu_like_codes(void* stream, const dfgpu_column* codes, const uint8_t* code_match, int64_t n_codes, uint8_t* out_values,
                                uint8_t* out_validity) {
  g_error.clear();
  if (codes == nullptr || codes->type != DFGPU_INT32 || codes->length < 0 || codes->offset < 0 || n_codes < 0)
    return fail(DFGPU_ERR_INVALID, "dfgpu_like_codes: the codes must be an INT32 column");
  if (codes->length == 0) return DFGPU_OK;
  if (out_values == nullptr || codes->values == nullptr || (n_codes > 0 && code_match == nullptr) ||
      (codes->validity != nullptr && out_validity == nullptr))
    return fail(DFGPU_ERR_INVALID, "dfgpu_like_codes: missing buffer (a column with validity needs out_validity)");
  const unsigned grid = (unsigned)((codes->length + kThreads - 1) / kThreads);
  like_codes_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const int32_t*>(codes->values), codes->validity,
                                                                              codes->offset, codes->length, code_match, n_codes, out_values,
                                                                              codes->validity != nullptr ? out_validity : nullptr);
  return launched("dfgpu_like_codes");
}
