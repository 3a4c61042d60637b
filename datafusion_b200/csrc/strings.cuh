// strings.cuh — what the kernels of libdfgpu_strings.so share (like.cu, string_compare.cu): the validity helpers, the Utf8View
// data-buffer ranges one launch reaches, the argument checks of a dfgpu_string_column, UTF-8 validation and the error message.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/dfgpu_strings.h"

namespace dfgpu {
namespace like {

constexpr int kThreads = 256;
constexpr int kViewBufs = 240;                  // Utf8View data buffers one launch can reach (kernel parameters)

__device__ __forceinline__ bool bit(const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; }

// a warp's 32 consecutive rows [row0, row0 + 32) of validity -> out_valid bytes (row0 is a multiple of 32)
__device__ __forceinline__ void store_validity(uint8_t* out_valid, int64_t row0, int64_t n, bool valid) {
  const unsigned vb = __ballot_sync(0xffffffffu, valid);
  const int lane = threadIdx.x & 31;
  if (lane < 4 && row0 + lane * 8 < n) out_valid[(row0 >> 3) + lane] = (uint8_t)(vb >> (lane * 8));
}

// a kernel's parameter program -> shared memory, word by word over the block (the caller synchronises)
template <typename Prog>
__device__ __forceinline__ void load_program(Prog& dst, const Prog& src) {
  for (int i = threadIdx.x; i < (int)(sizeof(Prog) / 4); i += blockDim.x)
    reinterpret_cast<uint32_t*>(&dst)[i] = reinterpret_cast<const uint32_t*>(&src)[i];
}

struct ViewBufs {
  const uint8_t* ptr[kViewBufs];
  int32_t lo, count;   // this launch reaches buffers [lo, lo + count)
};

// ---- host ----
inline thread_local std::string g_error;

inline int fail(int code, const std::string& msg) {
  g_error = msg;
  return code;
}

// length of the UTF-8 sequence at p[0 .. n), or 0 when it is not valid UTF-8 (overlong forms, surrogates, > U+10FFFF included)
inline int utf8_seq(const uint8_t* p, int64_t n) {
  const uint8_t b = p[0];
  if (b < 0x80) return 1;
  int len;
  uint32_t cp;
  if (b >= 0xC2 && b <= 0xDF) { len = 2; cp = b & 0x1F; }
  else if (b >= 0xE0 && b <= 0xEF) { len = 3; cp = b & 0x0F; }
  else if (b >= 0xF0 && b <= 0xF4) { len = 4; cp = b & 0x07; }
  else return 0;
  if (n < len) return 0;
  for (int i = 1; i < len; ++i) {
    if ((p[i] & 0xC0) != 0x80) return 0;
    cp = (cp << 6) | (p[i] & 0x3F);
  }
  if ((len == 3 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) || (len == 4 && (cp < 0x10000 || cp > 0x10FFFF))) return 0;
  return len;
}

// the byte index of the first invalid UTF-8 sequence in p[0 .. n), or -1 when all of it is valid
inline int64_t utf8_invalid_at(const uint8_t* p, int64_t n) {
  for (int64_t i = 0; i < n;) {
    const int l = utf8_seq(p + i, n - i);
    if (l == 0) return i;
    i += l;
  }
  return -1;
}

inline int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(DFGPU_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
  return DFGPU_OK;
}

// the buffers a call needs for col (length > 0): DFGPU_OK or DFGPU_ERR_INVALID.  `validity_out`: whether out_validity is written.
inline int check_column(const dfgpu_string_column* col, const uint8_t* out_values, const uint8_t* out_validity, bool validity_out,
                        const char* what) {
  if (out_values == nullptr || col->offsets_or_views == nullptr || (validity_out && out_validity == nullptr))
    return fail(DFGPU_ERR_INVALID, std::string(what) + ": missing buffer (a column with validity needs out_validity)");
  if (col->layout == DFGPU_STRING_UTF8 || col->layout == DFGPU_STRING_LARGE_UTF8) {
    if (col->n_data_buffers != 1 || col->data_buffers == nullptr) return fail(DFGPU_ERR_INVALID, std::string(what) + ": a Utf8 column has one data buffer");
    return DFGPU_OK;
  }
  if (col->layout != DFGPU_STRING_UTF8_VIEW) return fail(DFGPU_ERR_INVALID, std::string(what) + ": unknown string layout");
  if (reinterpret_cast<uintptr_t>(col->offsets_or_views) & 15) return fail(DFGPU_ERR_INVALID, std::string(what) + ": Utf8View views must be 16-byte aligned");
  if (col->n_data_buffers < 0 || (col->n_data_buffers > 0 && col->data_buffers == nullptr))
    return fail(DFGPU_ERR_INVALID, std::string(what) + ": Utf8View data buffers missing");
  return DFGPU_OK;
}

// Utf8View: launch(vb) once per range of kViewBufs data buffers (at least once), vb.lo == 0 on the first launch
template <typename Launch>
int for_each_view_range(const dfgpu_string_column* col, const char* what, Launch launch) {
  int lo = 0;
  do {
    ViewBufs vb;
    memset(&vb, 0, sizeof(vb));
    vb.lo = lo;
    vb.count = col->n_data_buffers - lo < kViewBufs ? col->n_data_buffers - lo : kViewBufs;
    for (int i = 0; i < vb.count; ++i) vb.ptr[i] = col->data_buffers[lo + i];
    launch(vb);
    const int rc = launched(what);
    if (rc != DFGPU_OK) return rc;
    lo += kViewBufs;
  } while (lo < col->n_data_buffers);
  return DFGPU_OK;
}

}  // namespace like
}  // namespace dfgpu
