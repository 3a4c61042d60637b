// composite_key.cu — one packing pass per pipeline push for joins on 2..4 key columns (dfgpu_lookup_create_composite).
//
// Every key tuple of the push (one per composite probe stage, plus the build sink's) becomes one 8-byte column in HBM before the
// pipeline kernel runs; the stages and the build sink then read that column as an ordinary one-column key, so the pipeline kernel, its
// ring-fed phase A, the partitioned aggregate and the partitioned build insert run unchanged.  The cost is 8 bytes written and read
// again per row and key next to the component bytes read once: the pass is bound by HBM bandwidth.
//
// A thread packs 8 consecutive rows: a component of width w arrives as 8 w bytes (128-bit loads, or one 64-bit load for 1-byte
// columns) when its base is aligned, 8 packed values leave as four 16-byte stores, and a build key's 8 validity bits as one byte.
#include "common.cuh"

namespace dfgpu {

constexpr int kPackRows = 8;

__device__ __forceinline__ uint64_t widen(uint64_t raw, int width, int sgn) {
  switch (width) {
    case 1: return sgn ? (uint64_t)(int64_t)(int8_t)raw : (raw & 0xffull);
    case 2: return sgn ? (uint64_t)(int64_t)(int16_t)raw : (raw & 0xffffull);
    case 4: return sgn ? (uint64_t)(int64_t)(int32_t)raw : (raw & 0xffffffffull);
    default: return raw;
  }
}

// the m (<= 8) values of rows r0.. of one component, sign- or zero-extended to 64 bits
__device__ __forceinline__ void load_rows(const KeyPart& kp, int64_t r0, int m, uint64_t v[kPackRows]) {
  const char* base = (const char*)kp.ptr + r0 * kp.width;
  const int align = kp.width == 1 ? 8 : 16;
  if (m == kPackRows && ((uintptr_t)kp.ptr % align) == 0) {
    const ulonglong2* b2 = (const ulonglong2*)base;
    switch (kp.width) {
      case 1: {
        const uint64_t x = __ldg((const unsigned long long*)base);
#pragma unroll
        for (int j = 0; j < kPackRows; ++j) v[j] = widen(x >> (8 * j), 1, kp.sgn);
        break;
      }
      case 2: {
        const ulonglong2 x = __ldg(b2);
#pragma unroll
        for (int j = 0; j < 4; ++j) { v[j] = widen(x.x >> (16 * j), 2, kp.sgn); v[j + 4] = widen(x.y >> (16 * j), 2, kp.sgn); }
        break;
      }
      case 4: {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const ulonglong2 x = __ldg(b2 + q);
          v[4 * q] = widen(x.x, 4, kp.sgn); v[4 * q + 1] = widen(x.x >> 32, 4, kp.sgn);
          v[4 * q + 2] = widen(x.y, 4, kp.sgn); v[4 * q + 3] = widen(x.y >> 32, 4, kp.sgn);
        }
        break;
      }
      default:
#pragma unroll
        for (int q = 0; q < 4; ++q) { const ulonglong2 x = __ldg(b2 + q); v[2 * q] = x.x; v[2 * q + 1] = x.y; }
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < kPackRows; ++j) {
    uint64_t raw = 0;
    if (j < m) switch (kp.width) {
      case 1: raw = ((const uint8_t*)base)[j]; break;
      case 2: raw = ((const uint16_t*)base)[j]; break;
      case 4: raw = ((const uint32_t*)base)[j]; break;
      default: raw = ((const unsigned long long*)base)[j]; break;
    }
    v[j] = widen(raw, kp.width, kp.sgn);
  }
}

// validity bits of rows r0 .. r0 + m - 1 (bit j = row r0 + j); a full group reads the one or two bytes that hold its 8 bits
__device__ __forceinline__ uint32_t load_valid(const KeyPart& kp, int64_t r0, int m) {
  if (!kp.valid) return 0xffu;
  const int64_t b = kp.voff + r0;
  if (m == kPackRows) {
    uint32_t x = kp.valid[b >> 3];
    if (b & 7) x |= (uint32_t)kp.valid[(b >> 3) + 1] << 8;   // bit b + 7 is a row of this group, so that byte exists
    return (x >> (b & 7)) & 0xffu;
  }
  uint32_t x = 0;
  for (int j = 0; j < m; ++j) x |= (uint32_t)bit_get(kp.valid, b + j) << j;
  return x;
}

__global__ void __launch_bounds__(256) pack_keys_kernel(const __grid_constant__ PackKeysParams kp, int64_t n) {
  const int64_t groups = (n + kPackRows - 1) / kPackRows;
  unsigned long long nulls = 0, outside = 0;
  const PackedKey& pk = kp.key[blockIdx.y];   // one key per grid row
  for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r0 = g * kPackRows;
    const int m = n - r0 < kPackRows ? (int)(n - r0) : kPackRows;
    uint64_t acc[kPackRows];
#pragma unroll
    for (int j = 0; j < kPackRows; ++j) acc[j] = 0;
    uint32_t valid = (1u << m) - 1u, inside = valid;
#pragma unroll
    for (int p = 0; p < kMaxKeyParts; ++p) {
      if (p >= pk.n_parts) break;
      const KeyPart& part = pk.part[p];
      uint64_t v[kPackRows];
      load_rows(part, r0, m, v);
      valid &= load_valid(part, r0, m);
#pragma unroll
      for (int j = 0; j < kPackRows; ++j) {
        const uint64_t d = v[j] - part.kmin;   // wrapping: below kmin lands above every range (domain <= 2^63 - 1)
        if (d >= part.range) inside &= ~(1u << j);
        acc[j] += d * part.stride;
      }
    }
    const uint32_t ok = valid & inside;
    if (pk.out_valid) {
      pk.out_valid[g] = (uint8_t)ok;
      nulls += (unsigned long long)__popc(((1u << m) - 1u) & ~valid);
      outside |= valid & ~inside;
    } else {
#pragma unroll
      for (int j = 0; j < kPackRows; ++j) if (!((ok >> j) & 1u)) acc[j] = pk.domain;
    }
    if (m == kPackRows) {
#pragma unroll
      for (int q = 0; q < kPackRows / 2; ++q) ((ulonglong2*)(pk.out + r0))[q] = make_ulonglong2(acc[2 * q], acc[2 * q + 1]);
    } else {
#pragma unroll
      for (int j = 0; j < kPackRows; ++j) if (j < m) pk.out[r0 + j] = acc[j];
    }
  }
  nulls = __reduce_add_sync(0xffffffffu, (unsigned)nulls);
  outside = __reduce_or_sync(0xffffffffu, (unsigned)outside);
  if ((threadIdx.x & 31) == 0 && kp.flags) {
    if (nulls) atomicAdd(&kp.flags[1], nulls);
    if (outside) atomicOr(&kp.flags[0], 1ull);
  }
}

void pack_keys(dfgpu_ctx* ctx, const PackKeysParams& kp, int64_t n) {
  if (n == 0 || kp.n_keys == 0) return;
  const int64_t groups = (n + kPackRows - 1) / kPackRows;
  const dim3 grid(grid_for(groups, 256, kNumSMs * 8 / kp.n_keys), kp.n_keys);
  pack_keys_kernel<<<grid, 256, 0, ctx->stream>>>(kp, n);
  DF_LAUNCH_CHECK(ctx);
}

}  // namespace dfgpu
