// string_compare.cu — libdfgpu_strings.so: a string column compared with a Utf8 literal (=, <>, <, <=, >, >=) and tested against a
// static IN list of Utf8 literals, over Utf8, LargeUtf8 and Utf8View (include/dfgpu_strings.h).  Dictionary codes go through
// dfgpu_like_codes (like.cu) after the predicate is evaluated over the dictionary's distinct values.
//
// Rows are settled from the cheapest bytes first.  Utf8 / LargeUtf8: the length from the row's two offsets settles `=` / `<>` against a
// literal of another length and an IN row whose length no value has; only then are string bytes read, and an ordering comparison stops
// at the first byte that differs.  Utf8View: the view's length and 4-byte prefix, and the whole string when it is inline (12 bytes or
// fewer), settle a row without its data buffer.  The bytes beyond a string's length in a view are never read as string bytes.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_set>

#include "../../include/dfgpu_strings.h"
#include "strings.cuh"

namespace dfgpu {
namespace strings {

using like::bit;
using like::fail;
using like::g_error;
using like::kThreads;
using like::load_program;
using like::store_validity;
using like::ViewBufs;

constexpr int kUnroll = 4;                                   // Utf8 rows per thread per grid pass: their offsets load together
constexpr int kInSlots = 2 * DFGPU_STRING_IN_MAX_VALUES;     // the IN list's open-addressing table (a power of two, at most half full)
constexpr int kLenWords = DFGPU_STRING_IN_MAX_BYTES / 32 + 1;

struct CmpProgram {
  uint32_t words[DFGPU_STRING_MAX_LITERAL_BYTES / 4];   // the literal's bytes, zero padded, 4 to a little-endian word
  int32_t len;
  int32_t op;
};

struct InProgram {
  uint8_t bytes[DFGPU_STRING_IN_MAX_BYTES];          // the distinct values back to back
  uint16_t off[DFGPU_STRING_IN_MAX_VALUES + 1];      // value v is bytes[off[v], off[v + 1])
  int8_t slot[kInSlots];                             // value index by hash of the bytes, -1 = empty
  uint32_t len_bits[kLenWords];                      // bit l: some value is l bytes long
  uint32_t view_bits[8];                             // bit h: some value longer than 12 bytes has prefix hash h (length, first 4 bytes)
  int32_t missing_valid;                             // 0 when the list holds a NULL: a string found nowhere gives NULL
  int32_t negated;
};

__host__ __device__ __forceinline__ uint32_t fnv_step(uint32_t h, uint32_t b) { return (h ^ b) * 16777619u; }
__host__ __device__ __forceinline__ uint32_t hash_init(uint32_t len) { return fnv_step(2166136261u, len); }
__host__ __device__ __forceinline__ uint32_t hash_slot(uint32_t h) { return (h ^ (h >> 15)) & (kInSlots - 1); }
__host__ __device__ __forceinline__ uint32_t prefix_bit(uint32_t len, uint32_t prefix) {
  const uint32_t h = fnv_step(fnv_step(hash_init(len), prefix), prefix >> 16);
  return (h ^ (h >> 13) ^ (h >> 24)) & 255;
}

__device__ __forceinline__ bool holds(int op, int c) {
  switch (op) {
    case DFGPU_STRING_EQ: return c == 0;
    case DFGPU_STRING_NE: return c != 0;
    case DFGPU_STRING_LT: return c < 0;
    case DFGPU_STRING_LE: return c <= 0;
    case DFGPU_STRING_GT: return c > 0;
    default: return c >= 0;
  }
}

__device__ __forceinline__ int sign(int64_t d) { return d < 0 ? -1 : d > 0 ? 1 : 0; }

// order of the k (0..4) leading bytes of two little-endian words: byte-swapped, the first byte is the most significant
__device__ __forceinline__ int cmp_word(uint32_t a, uint32_t b, int k) {
  if (k <= 0) return 0;
  const uint32_t mask = k >= 4 ? 0xFFFFFFFFu : ~(0xFFFFFFFFu >> (8 * k));
  const uint32_t x = __byte_perm(a, 0, 0x0123) & mask, y = __byte_perm(b, 0, 0x0123) & mask;
  return x < y ? -1 : x > y ? 1 : 0;
}

// order of s[from, m) against lit[from, m): the first differing byte decides
__device__ __forceinline__ int cmp_bytes(const uint8_t* lit, const uint8_t* s, int64_t from, int64_t m) {
  for (int64_t i = from; i < m; ++i) {
    const int d = (int)s[i] - (int)lit[i];
    if (d != 0) return d;
  }
  return 0;
}

// a string's bytes: in a data buffer, or inline in a view's last 12 bytes (kept in registers)
struct GlobalBytes {
  const uint8_t* p;
  __device__ __forceinline__ uint32_t operator[](int64_t i) const { return p[i]; }
};
struct InlineBytes {
  uint32_t w0, w1, w2;
  __device__ __forceinline__ uint32_t operator[](int64_t i) const { return ((i < 4 ? w0 : i < 8 ? w1 : w2) >> (8 * (i & 3))) & 0xFF; }
};

// is the len-byte string s one of the values?  The length bit first, then a hash of the bytes, then the values on its probe sequence.
template <typename Bytes>
__device__ __forceinline__ bool in_list(const InProgram& P, const Bytes& s, int64_t len) {
  if (len > DFGPU_STRING_IN_MAX_BYTES || !((P.len_bits[len >> 5] >> (len & 31)) & 1)) return false;
  uint32_t h = hash_init((uint32_t)len);
  for (int64_t i = 0; i < len; ++i) h = fnv_step(h, s[i]);
  for (uint32_t k = hash_slot(h);; k = (k + 1) & (kInSlots - 1)) {
    const int v = P.slot[k];
    if (v < 0) return false;
    const int a = P.off[v];
    if (P.off[v + 1] - a != len) continue;
    int64_t i = 0;
    while (i < len && s[i] == P.bytes[a + i]) ++i;
    if (i == len) return true;
  }
}

// Utf8 / LargeUtf8 `s op literal`: each thread takes kUnroll rows of a block's kUnroll * kThreads per grid pass, a warp 32 consecutive
// ones (one validity word); the grid strides over the column.
template <typename Off>
__global__ void __launch_bounds__(kThreads) cmp_utf8_kernel(const __grid_constant__ CmpProgram prog_in, const Off* __restrict__ offsets,
                                                            const uint8_t* __restrict__ data, const uint8_t* __restrict__ validity,
                                                            int64_t in_off, int64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  __shared__ CmpProgram P;
  load_program(P, prog_in);
  __syncthreads();
  const uint8_t* lit = reinterpret_cast<const uint8_t*>(P.words);
  const int64_t L = P.len;
  const int op = P.op;
  const bool eq_only = op == DFGPU_STRING_EQ || op == DFGPU_STRING_NE;
  const int warp0 = threadIdx.x & ~31;
  for (int64_t base = (int64_t)blockIdx.x * kThreads * kUnroll; base < n; base += (int64_t)gridDim.x * kThreads * kUnroll) {
    Off a[kUnroll], b[kUnroll];
    bool valid[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const int64_t row = base + k * kThreads + threadIdx.x;
      valid[k] = row < n && (validity == nullptr || bit(validity, in_off + row));
      a[k] = valid[k] ? offsets[in_off + row] : 0;
      b[k] = valid[k] ? offsets[in_off + row + 1] : 0;
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const int64_t row0 = base + k * kThreads + warp0, row = row0 + (threadIdx.x & 31);
      if (row0 >= n) break;                                             // warp-uniform
      bool r = false;
      if (valid[k]) {
        const int64_t len = (int64_t)(b[k] - a[k]);
        int c = 1;
        if (!eq_only || len == L) {
          c = cmp_bytes(lit, data + a[k], 0, len < L ? len : L);
          if (c == 0) c = sign(len - L);
        }
        r = holds(op, c);
      }
      if (row < n) out[row] = r;
      if (out_valid != nullptr) store_validity(out_valid, row0, n, valid[k]);
    }
  }
}

// Utf8View `s op literal`: one thread per row, the grid strides over the column.  Launch 0 (bufs.lo == 0) writes every row the view
// settles and the validity; launch g writes the rows left open whose data buffer is in its range.
__global__ void __launch_bounds__(kThreads) cmp_view_kernel(const __grid_constant__ CmpProgram prog_in, const __grid_constant__ ViewBufs bufs,
                                                            const uint4* __restrict__ views, const uint8_t* __restrict__ validity, int64_t in_off,
                                                            int64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  __shared__ CmpProgram P;
  load_program(P, prog_in);
  __syncthreads();
  const int64_t L = P.len;
  const int op = P.op;
  const bool eq_only = op == DFGPU_STRING_EQ || op == DFGPU_STRING_NE;
  const bool first = bufs.lo == 0;
  for (int64_t row0 = (int64_t)blockIdx.x * kThreads + (threadIdx.x & ~31); row0 < n; row0 += (int64_t)gridDim.x * kThreads) {
    const int64_t row = row0 + (threadIdx.x & 31);
    const bool in = row < n;
    const bool valid = in && (validity == nullptr || bit(validity, in_off + row));
    bool r = false, write = in && first;
    if (valid) {
      const uint4 v = views[in_off + row];
      const int64_t len = v.x;
      const int64_t m = len < L ? len : L;
      int c = 1;
      if (!eq_only || len == L) {
        c = cmp_word(v.y, P.words[0], (int)(m < 4 ? m : 4));
        if (c == 0 && m > 4) {
          if (len <= 12) {
            c = cmp_word(v.z, P.words[1], (int)(m - 4 < 4 ? m - 4 : 4));
            if (c == 0 && m > 8) c = cmp_word(v.w, P.words[2], (int)(m - 8));
          } else {                                                      // out of line, the first 4 bytes equal: the data buffer decides
            write = (int32_t)v.z >= bufs.lo && (int32_t)v.z < bufs.lo + bufs.count;
            if (write) c = cmp_bytes(reinterpret_cast<const uint8_t*>(P.words), bufs.ptr[(int32_t)v.z - bufs.lo] + v.w, 4, m);
          }
        }
        if (c == 0) c = sign(len - L);
      }
      r = holds(op, c);
    }
    if (write) out[row] = r;
    if (first && out_valid != nullptr) store_validity(out_valid, row0, n, valid);
  }
}

// Utf8 / LargeUtf8 `s [NOT] IN (list)`: rows as in cmp_utf8_kernel
template <typename Off>
__global__ void __launch_bounds__(kThreads) in_utf8_kernel(const __grid_constant__ InProgram prog_in, const Off* __restrict__ offsets,
                                                           const uint8_t* __restrict__ data, const uint8_t* __restrict__ validity,
                                                           int64_t in_off, int64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  __shared__ InProgram P;
  load_program(P, prog_in);
  __syncthreads();
  const int warp0 = threadIdx.x & ~31;
  for (int64_t base = (int64_t)blockIdx.x * kThreads * kUnroll; base < n; base += (int64_t)gridDim.x * kThreads * kUnroll) {
    Off a[kUnroll], b[kUnroll];
    bool valid[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const int64_t row = base + k * kThreads + threadIdx.x;
      valid[k] = row < n && (validity == nullptr || bit(validity, in_off + row));
      a[k] = valid[k] ? offsets[in_off + row] : 0;
      b[k] = valid[k] ? offsets[in_off + row + 1] : 0;
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const int64_t row0 = base + k * kThreads + warp0, row = row0 + (threadIdx.x & 31);
      if (row0 >= n) break;                                             // warp-uniform
      const bool found = valid[k] && in_list(P, GlobalBytes{data + a[k]}, (int64_t)(b[k] - a[k]));
      const bool ok = valid[k] && (found || P.missing_valid);
      if (row < n) out[row] = ok && (found != (P.negated != 0));
      if (out_valid != nullptr) store_validity(out_valid, row0, n, ok);
    }
  }
}

// Utf8View `s [NOT] IN (list)`: launches as in cmp_view_kernel.  An inline string is looked up from its view; a longer one only when
// some value of its length has its 4-byte prefix (view_bits), from its data buffer.
__global__ void __launch_bounds__(kThreads) in_view_kernel(const __grid_constant__ InProgram prog_in, const __grid_constant__ ViewBufs bufs,
                                                           const uint4* __restrict__ views, const uint8_t* __restrict__ validity, int64_t in_off,
                                                           int64_t n, uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  __shared__ InProgram P;
  load_program(P, prog_in);
  __syncthreads();
  const bool first = bufs.lo == 0;
  for (int64_t row0 = (int64_t)blockIdx.x * kThreads + (threadIdx.x & ~31); row0 < n; row0 += (int64_t)gridDim.x * kThreads) {
    const int64_t row = row0 + (threadIdx.x & 31);
    const bool in = row < n;
    const bool valid = in && (validity == nullptr || bit(validity, in_off + row));
    bool found = false, write = in && first;
    if (valid) {
      const uint4 v = views[in_off + row];
      if (v.x <= 12) {
        found = in_list(P, InlineBytes{v.y, v.z, v.w}, v.x);
      } else if (v.x <= DFGPU_STRING_IN_MAX_BYTES && ((P.len_bits[v.x >> 5] >> (v.x & 31)) & 1) &&
                 ((P.view_bits[prefix_bit(v.x, v.y) >> 5] >> (prefix_bit(v.x, v.y) & 31)) & 1)) {
        write = (int32_t)v.z >= bufs.lo && (int32_t)v.z < bufs.lo + bufs.count;
        if (write) found = in_list(P, GlobalBytes{bufs.ptr[(int32_t)v.z - bufs.lo] + v.w}, v.x);
      }
    }
    const bool ok = valid && (found || P.missing_valid);
    if (write) out[row] = ok && (found != (P.negated != 0));
    if (first && out_valid != nullptr) store_validity(out_valid, row0, n, ok);
  }
}

// ---- host ----
// blocks for a grid-striding kernel: enough for rows_per_block-row blocks over n rows, at most what the device holds at once
template <typename Kernel>
unsigned grid_for(Kernel kernel, int64_t n, int64_t rows_per_block) {
  int dev = 0, sms = 1, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0);
  const int64_t need = (n + rows_per_block - 1) / rows_per_block, cap = (int64_t)sms * (per_sm > 0 ? per_sm : 1);
  return (unsigned)(need < cap ? need : cap);
}

int check_utf8(const uint8_t* p, int64_t len, const std::string& what) {
  const int64_t bad = like::utf8_invalid_at(p, len);
  if (bad >= 0) return fail(DFGPU_ERR_INVALID, what + " is not valid UTF-8 (byte " + std::to_string(bad) + ")");
  return DFGPU_OK;
}

template <typename Prog, typename Utf8K32, typename Utf8K64, typename ViewK>
int launch(const char* what, void* stream, const dfgpu_string_column* col, const Prog& P, Utf8K32 k32, Utf8K64 k64, ViewK kv,
           uint8_t* out_values, uint8_t* ov) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = col->length;
  if (col->layout == DFGPU_STRING_UTF8) {
    k32<<<grid_for(k32, n, kThreads * kUnroll), kThreads, 0, st>>>(P, static_cast<const int32_t*>(col->offsets_or_views), col->data_buffers[0],
                                                                   col->validity, col->offset, n, out_values, ov);
    return like::launched(what);
  }
  if (col->layout == DFGPU_STRING_LARGE_UTF8) {
    k64<<<grid_for(k64, n, kThreads * kUnroll), kThreads, 0, st>>>(P, static_cast<const int64_t*>(col->offsets_or_views), col->data_buffers[0],
                                                                   col->validity, col->offset, n, out_values, ov);
    return like::launched(what);
  }
  const unsigned grid = grid_for(kv, n, kThreads);
  return like::for_each_view_range(col, what, [&](const ViewBufs& vb) {
    kv<<<grid, kThreads, 0, st>>>(P, vb, static_cast<const uint4*>(col->offsets_or_views), col->validity, col->offset, n, out_values, ov);
  });
}

}  // namespace strings
}  // namespace dfgpu

using namespace dfgpu::strings;

extern "C" int dfgpu_string_compare(void* stream, const dfgpu_string_column* col, int32_t op, const uint8_t* literal, int64_t literal_len,
                                    uint8_t* out_values, uint8_t* out_validity) {
  g_error.clear();
  const char* what = "dfgpu_string_compare";
  if (op < DFGPU_STRING_EQ || op > DFGPU_STRING_GE) return fail(DFGPU_ERR_INVALID, "dfgpu_string_compare: unknown op " + std::to_string(op));
  if (literal_len < 0 || (literal_len > 0 && literal == nullptr)) return fail(DFGPU_ERR_INVALID, "dfgpu_string_compare: no literal");
  int rc = check_utf8(literal, literal_len, "dfgpu_string_compare: the literal");
  if (rc != DFGPU_OK) return rc;
  if (literal_len > DFGPU_STRING_MAX_LITERAL_BYTES)
    return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_string_compare: the literal is longer than " + std::to_string(DFGPU_STRING_MAX_LITERAL_BYTES) + " bytes");
  if (col == nullptr || col->length < 0 || col->offset < 0) return fail(DFGPU_ERR_INVALID, "dfgpu_string_compare: no column");
  if (col->length == 0) return DFGPU_OK;
  if ((rc = dfgpu::like::check_column(col, out_values, out_validity, col->validity != nullptr, what)) != DFGPU_OK) return rc;
  CmpProgram P;
  memset(&P, 0, sizeof(P));
  if (literal_len > 0) memcpy(P.words, literal, (size_t)literal_len);
  P.len = (int32_t)literal_len;
  P.op = op;
  return launch(what, stream, col, P, cmp_utf8_kernel<int32_t>, cmp_utf8_kernel<int64_t>, cmp_view_kernel, out_values,
                col->validity != nullptr ? out_validity : nullptr);
}

extern "C" int dfgpu_string_in_list(void* stream, const dfgpu_string_column* col, const uint8_t* const* values, const int64_t* value_lens,
                                    int64_t n_values, int32_t list_has_null, int32_t negated, uint8_t* out_values, uint8_t* out_validity) {
  g_error.clear();
  const char* what = "dfgpu_string_in_list";
  if (n_values < 0 || (n_values > 0 && (values == nullptr || value_lens == nullptr)))
    return fail(DFGPU_ERR_INVALID, "dfgpu_string_in_list: no list");
  std::unordered_set<std::string> distinct;
  std::string list;                                                   // the distinct values in list order, back to back
  int64_t lens[DFGPU_STRING_IN_MAX_VALUES];
  int n = 0;
  for (int64_t i = 0; i < n_values; ++i) {
    if (value_lens[i] < 0 || (value_lens[i] > 0 && values[i] == nullptr))
      return fail(DFGPU_ERR_INVALID, "dfgpu_string_in_list: value " + std::to_string(i) + " missing");
    int rc = check_utf8(values[i], value_lens[i], "dfgpu_string_in_list: value " + std::to_string(i));
    if (rc != DFGPU_OK) return rc;
    std::string v(reinterpret_cast<const char*>(values[i]), (size_t)value_lens[i]);
    if (!distinct.insert(v).second) continue;
    if (n == DFGPU_STRING_IN_MAX_VALUES)
      return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_string_in_list: the list has more than " + std::to_string(DFGPU_STRING_IN_MAX_VALUES) + " distinct values");
    if ((int64_t)list.size() + value_lens[i] > DFGPU_STRING_IN_MAX_BYTES)
      return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_string_in_list: the list's values are longer than " + std::to_string(DFGPU_STRING_IN_MAX_BYTES) + " bytes together");
    lens[n++] = value_lens[i];
    list += v;
  }
  if (col == nullptr || col->length < 0 || col->offset < 0) return fail(DFGPU_ERR_INVALID, "dfgpu_string_in_list: no column");
  if (col->length == 0) return DFGPU_OK;
  const bool validity_out = col->validity != nullptr || list_has_null != 0;
  int rc = dfgpu::like::check_column(col, out_values, out_validity, validity_out, what);
  if (rc != DFGPU_OK) return rc;
  // launch 0 writes every row's validity, but with a NULL in the list a row's validity depends on the launch that reads its buffer
  if (list_has_null && col->layout == DFGPU_STRING_UTF8_VIEW && col->n_data_buffers > dfgpu::like::kViewBufs)
    return fail(DFGPU_ERR_UNSUPPORTED, "dfgpu_string_in_list: a list with a NULL over a Utf8View column of more than " +
                                           std::to_string(dfgpu::like::kViewBufs) + " data buffers");
  InProgram P;
  memset(&P, 0, sizeof(P));
  memset(P.slot, 0xFF, sizeof(P.slot));
  if (!list.empty()) memcpy(P.bytes, list.data(), list.size());
  for (int v = 0, at = 0; v < n; at += (int)lens[v], ++v) {
    const uint8_t* s = P.bytes + at;
    const uint32_t len = (uint32_t)lens[v];
    P.off[v] = (uint16_t)at;
    P.off[v + 1] = (uint16_t)(at + len);
    P.len_bits[len >> 5] |= 1u << (len & 31);
    uint32_t h = hash_init(len);
    for (uint32_t i = 0; i < len; ++i) h = fnv_step(h, s[i]);
    uint32_t k = hash_slot(h);
    while (P.slot[k] >= 0) k = (k + 1) & (kInSlots - 1);
    P.slot[k] = (int8_t)v;
    if (len > 12) {
      const uint32_t prefix = (uint32_t)s[0] | (uint32_t)s[1] << 8 | (uint32_t)s[2] << 16 | (uint32_t)s[3] << 24;
      const uint32_t b = prefix_bit(len, prefix);
      P.view_bits[b >> 5] |= 1u << (b & 31);
    }
  }
  P.missing_valid = list_has_null == 0;
  P.negated = negated != 0;
  return launch(what, stream, col, P, in_utf8_kernel<int32_t>, in_utf8_kernel<int64_t>, in_view_kernel, out_values,
                validity_out ? out_validity : nullptr);
}
