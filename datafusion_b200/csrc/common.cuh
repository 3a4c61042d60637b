// common.cuh — shared host/device plumbing for libdfgpu (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>
#include <memory>
#include <stdexcept>
#include <map>
#include <mutex>
#include <unordered_map>
#include "../../include/dfgpu.h"

namespace dfgpu {

// ------------------------------------------------------------------------------------------
// errors: C++ exceptions inside, converted to status codes at the extern "C" boundary
// ------------------------------------------------------------------------------------------
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define DF_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      char _buf[512];                                                                         \
      snprintf(_buf, sizeof(_buf), "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e),        \
               __FILE__, __LINE__, cudaGetErrorString(_e));                                   \
      throw ::dfgpu::Error(_e == cudaErrorMemoryAllocation ? DFGPU_ERR_OOM : DFGPU_ERR_CUDA, _buf); \
    }                                                                                         \
  } while (0)

#define DF_CHECK(cond, code, msg)                                 \
  do {                                                            \
    if (!(cond)) throw ::dfgpu::Error((code), std::string(msg));  \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// ------------------------------------------------------------------------------------------
// type helpers
// ------------------------------------------------------------------------------------------
// Decimal128(p, s): the ABI's type code carries precision and scale in its upper bytes (DFGPU_DECIMAL128_TYPE)
__host__ __device__ inline bool type_is_decimal(int t) { return (t & 0xff) == DFGPU_DECIMAL128; }
__host__ __device__ inline int dec_precision(int t) { return (t >> 8) & 0xff; }
__host__ __device__ inline int dec_scale(int t) { return (int)(int8_t)((t >> 16) & 0xff); }
__host__ __device__ inline int dec_type(int p, int s) { return DFGPU_DECIMAL128 | (p << 8) | ((s & 0xff) << 16); }
// width of a primitive (non-decimal) type code: the device interpreters' fast path (a Decimal128(p, s) code never reaches them)
__host__ __device__ inline int type_width_prim(int t) {
  switch (t) {
    case DFGPU_BOOL: return 0;  // bit-packed
    case DFGPU_INT8: case DFGPU_UINT8: return 1;
    case DFGPU_INT16: case DFGPU_UINT16: return 2;
    case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_FLOAT32: case DFGPU_DATE32: return 4;
    case DFGPU_INT64: case DFGPU_UINT64: case DFGPU_FLOAT64: case DFGPU_DATE64: case DFGPU_TIMESTAMP: return 8;
    case DFGPU_DECIMAL128: return 16;
    default: return -1;
  }
}
__host__ __device__ inline int type_width(int t) {
  switch (t) {
    case DFGPU_BOOL: return 0;  // bit-packed
    case DFGPU_INT8: case DFGPU_UINT8: return 1;
    case DFGPU_INT16: case DFGPU_UINT16: return 2;
    case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_FLOAT32: case DFGPU_DATE32: return 4;
    case DFGPU_INT64: case DFGPU_UINT64: case DFGPU_FLOAT64: case DFGPU_DATE64: case DFGPU_TIMESTAMP: return 8;
    case DFGPU_DECIMAL128: return 16;
    default: return type_is_decimal(t) ? 16 : -1;   // Decimal128(p, s): precision and scale in the upper bytes
  }
}
__host__ __device__ inline bool type_is_signed_int(int t) {
  return t == DFGPU_INT8 || t == DFGPU_INT16 || t == DFGPU_INT32 || t == DFGPU_INT64 || t == DFGPU_DATE32 ||
         t == DFGPU_DATE64 || t == DFGPU_TIMESTAMP;
}
__host__ __device__ inline bool type_is_unsigned_int(int t) {
  return t == DFGPU_UINT8 || t == DFGPU_UINT16 || t == DFGPU_UINT32 || t == DFGPU_UINT64;
}
__host__ __device__ inline bool type_is_float(int t) { return t == DFGPU_FLOAT32 || t == DFGPU_FLOAT64; }
__host__ __device__ inline bool type_is_int(int t) { return type_is_signed_int(t) || type_is_unsigned_int(t); }

// the order-preserving map double -> uint64 of float MIN / MAX (IEEE totalOrder on the bits: -NaN < -inf < ... < -0.0 < +0.0 < ... <
// +inf < +NaN).  dfgpu_agg and the pipeline sinks reduce this key with unsigned min / max and map it back when they emit, so the result
// is one of the inputs bit for bit whatever the row order
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

inline size_t values_bytes(int type, int64_t rows) {
  if (type == DFGPU_BOOL) return (size_t)((rows + 7) / 8);
  return (size_t)rows * (size_t)type_width(type);
}
inline size_t bitmap_bytes(int64_t rows) { return (size_t)((rows + 7) / 8); }
// device bitmaps are allocated in whole 64-bit words so kernels may use uint64 accesses
inline size_t bitmap_alloc_bytes(int64_t rows) { return (size_t)((rows + 63) / 64) * 8; }

// ------------------------------------------------------------------------------------------
// hashing.  Hash VALUES never reach operator output (SURVEY.md §8c: join order follows probe
// order + ascending build index, group ids are not exposed, the exchange only picks a
// partition), so any 64-bit mixer is admissible; we use the splitmix64 finaliser with the
// reference's three distinct seeds so exchange / join / aggregate hashes stay decorrelated
// (hash_join/exec.rs:105, aggregates/mod.rs:236, repartition/mod.rs:650).
// ------------------------------------------------------------------------------------------
constexpr uint64_t kSeedJoin = 12210250226015887276ull;
constexpr uint64_t kSeedAgg = 15395726432021054657ull;
constexpr uint64_t kSeedExchange = 0x9E3779B97F4A7C15ull;  // reference uses seed 0; any fixed value decorrelated from the others

__host__ __device__ inline uint64_t mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27; x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return x;
}
__host__ __device__ inline uint64_t hash_u64(uint64_t v, uint64_t seed) { return mix64(v + seed); }
// multi-column: later columns re-seed with the running hash (hash_utils.rs:306-345 does the same for primitives)
__host__ __device__ inline uint64_t hash_combine(uint64_t running, uint64_t v) { return mix64(v ^ (running * 0x9E3779B97F4A7C15ull + 0x7F4A7C15ull)); }

// counter-based generator shared with the oracle (oracle/gen.h restates it)
__host__ __device__ inline uint64_t splitmix64_at(uint64_t seed, uint64_t i) {
  uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// ------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------
}  // namespace dfgpu

struct dfgpu_kernel_timing {
  std::string name;
  double total_ms = 0;
  int64_t count = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;  // recorded, not yet resolved
};

struct dfgpu_ctx {
  // per-ctx caching device allocator: every allocation and free of this library is ordered on ctx->stream,
  // so a released block can be handed out again immediately (stream order makes the reuse safe) and the
  // steady state performs no cudaMalloc / pool growth at all.
  std::multimap<size_t, void*> dev_free;
  std::unordered_map<void*, size_t> dev_sizes;
  size_t dev_free_bytes = 0;
  size_t dev_cache_limit = 24ull << 30;  // idle blocks kept for reuse; beyond it the largest idle blocks are returned to the driver
  cudaStream_t copy_in = nullptr, copy_out = nullptr;  // lazily created: H2D / D2H streams of the pipelined host entry points
  bool time_kernels = false;                    // dfgpu_set_kernel_timing
  std::vector<dfgpu_kernel_timing> timings;     // per kernel family
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string last_error;
  int64_t launches = 0;
  void* l2_scratch = nullptr;
  size_t l2_scratch_bytes = 0;
  // small pinned scratch for scalar readbacks
  void* pinned_scalar = nullptr;
};

namespace dfgpu {

inline void set_device(dfgpu_ctx* ctx) { DF_CUDA(cudaSetDevice(ctx->device)); }

inline size_t dev_bucket(size_t n) {
  if (n <= 256) return 256;
  size_t p = 256;
  while (p * 2 <= n) p <<= 1;          // largest power of two <= n
  size_t step = p >= (1u << 20) ? p / 8 : p;  // >= 1 MiB: 12.5 % granularity; small blocks: next power of two
  return ((n + step - 1) / step) * step;
}
inline void dev_cache_trim(dfgpu_ctx* ctx) {
  cudaStreamSynchronize(ctx->stream);
  for (auto& kv : ctx->dev_free) { cudaFree(kv.second); ctx->dev_sizes.erase(kv.second); }
  ctx->dev_free.clear();
  ctx->dev_free_bytes = 0;
}
inline void* dev_alloc(dfgpu_ctx* ctx, size_t n) {
  const size_t b = dev_bucket(n);
  auto it = ctx->dev_free.find(b);
  if (it != ctx->dev_free.end()) { void* p = it->second; ctx->dev_free.erase(it); ctx->dev_free_bytes -= b; return p; }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, b);
  if (e != cudaSuccess) {
    cudaGetLastError();
    dev_cache_trim(ctx);
    e = cudaMalloc(&p, b);
    if (e != cudaSuccess) { cudaGetLastError(); throw Error(DFGPU_ERR_OOM, "device allocation of " + std::to_string(b) + " bytes failed"); }
  }
  ctx->dev_sizes[p] = b;
  return p;
}
inline void dev_free(dfgpu_ctx* ctx, void* p) {
  auto it = ctx->dev_sizes.find(p);
  if (it == ctx->dev_sizes.end()) { cudaFree(p); return; }
  ctx->dev_free.emplace(it->second, p);
  ctx->dev_free_bytes += it->second;
  if (ctx->dev_free_bytes > ctx->dev_cache_limit) {
    cudaStreamSynchronize(ctx->stream);  // blocks about to be returned may still be in use by queued work
    while (ctx->dev_free_bytes > ctx->dev_cache_limit / 2 && !ctx->dev_free.empty()) {
      auto last = std::prev(ctx->dev_free.end());  // largest idle block first
      cudaFree(last->second);
      ctx->dev_free_bytes -= last->first;
      ctx->dev_sizes.erase(last->second);
      ctx->dev_free.erase(last);
    }
  }
}

// stream-ordered device buffer on the per-ctx caching allocator above (no device sync on alloc / free in steady state)
struct DevBuf {
  dfgpu_ctx* ctx = nullptr;
  void* ptr = nullptr;
  size_t bytes = 0;
  DevBuf() {}
  DevBuf(dfgpu_ctx* c, size_t n) { alloc(c, n); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); ctx = o.ctx; ptr = o.ptr; bytes = o.bytes; o.ptr = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(dfgpu_ctx* c, size_t n) {
    release();
    ctx = c;
    bytes = n;
    if (n == 0) { ptr = nullptr; return; }
    ptr = dev_alloc(c, n);
  }
  void release() {
    if (ptr) { dev_free(ctx, ptr); ptr = nullptr; bytes = 0; }
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(ptr); }
  void zero() { if (ptr) DF_CUDA(cudaMemsetAsync(ptr, 0, bytes, ctx->stream)); }
  void fill(int byte) { if (ptr) DF_CUDA(cudaMemsetAsync(ptr, byte, bytes, ctx->stream)); }
};

// process-wide pool of pinned host blocks: cudaMallocHost of GB-sized buffers costs hundreds of ms
// (page locking), so released blocks are kept and reused by size class (power-of-two buckets).
struct PinnedPool {
  std::mutex mu;
  std::multimap<size_t, void*> free_blocks;
  size_t cached_bytes = 0;
  static constexpr size_t kMaxCached = 24ull << 30;
  static PinnedPool& get() { static PinnedPool* p = new PinnedPool(); return *p; }  // leaked on purpose: outlives ctx teardown order
  static size_t bucket(size_t n) { size_t b = 4096; while (b < n) b <<= 1; return b; }
  void* acquire(size_t n, size_t* got) {
    size_t b = bucket(n);
    {
      std::lock_guard<std::mutex> g(mu);
      auto it = free_blocks.find(b);
      if (it != free_blocks.end()) { void* p = it->second; free_blocks.erase(it); cached_bytes -= b; *got = b; return p; }
    }
    void* p = nullptr;
    cudaError_t e = cudaMallocHost(&p, b);
    if (e != cudaSuccess) {
      trim();
      e = cudaMallocHost(&p, b);
      if (e != cudaSuccess) { cudaGetLastError(); throw Error(DFGPU_ERR_OOM, "pinned host allocation failed"); }
    }
    *got = b;
    return p;
  }
  void release(void* p, size_t b) {
    std::lock_guard<std::mutex> g(mu);
    if (cached_bytes + b > kMaxCached) { cudaFreeHost(p); return; }
    free_blocks.emplace(b, p);
    cached_bytes += b;
  }
  void trim() {
    std::lock_guard<std::mutex> g(mu);
    for (auto& kv : free_blocks) cudaFreeHost(kv.second);
    free_blocks.clear();
    cached_bytes = 0;
  }
};

// pinned host buffer (pooled)
struct HostBuf {
  void* ptr = nullptr;
  size_t bytes = 0;      // requested
  size_t cap = 0;        // pooled block size
  HostBuf() {}
  explicit HostBuf(size_t n) { alloc(n); }
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  HostBuf(HostBuf&& o) noexcept { ptr = o.ptr; bytes = o.bytes; cap = o.cap; o.ptr = nullptr; o.bytes = 0; o.cap = 0; }
  HostBuf& operator=(HostBuf&& o) noexcept {
    if (this != &o) { release(); ptr = o.ptr; bytes = o.bytes; cap = o.cap; o.ptr = nullptr; o.bytes = 0; o.cap = 0; }
    return *this;
  }
  ~HostBuf() { release(); }
  void alloc(size_t n) {
    release();
    bytes = n;
    if (n == 0) return;
    ptr = PinnedPool::get().acquire(n, &cap);
  }
  void release() { if (ptr) { PinnedPool::get().release(ptr, cap); ptr = nullptr; bytes = 0; cap = 0; } }
};

// A device-resident column: either a borrowed view or owning buffers.
struct DCol {
  int type = 0;
  int64_t length = 0;
  int64_t offset = 0;          // logical element offset into values/validity
  const void* values = nullptr;
  const uint8_t* validity = nullptr;  // nullptr = all valid
  int64_t null_count = -1;
  std::shared_ptr<DevBuf> own_values, own_validity;  // keep-alive when owning
};

inline DCol view_of(const dfgpu_column& c) {
  DCol d;
  d.type = c.type; d.length = c.length; d.offset = c.offset; d.values = c.values; d.validity = c.validity;
  d.null_count = c.null_count;
  if (c.null_count == 0) d.validity = nullptr;
  return d;
}

inline DCol alloc_col(dfgpu_ctx* ctx, int type, int64_t rows, bool with_validity) {
  DCol d;
  d.type = type; d.length = rows; d.offset = 0;
  d.own_values = std::make_shared<DevBuf>(ctx, type == DFGPU_BOOL ? bitmap_alloc_bytes(rows) : values_bytes(type, rows));
  d.values = d.own_values->ptr;
  if (with_validity) {
    d.own_validity = std::make_shared<DevBuf>(ctx, bitmap_alloc_bytes(rows));
    d.validity = d.own_validity->as<uint8_t>();
  } else {
    d.null_count = 0;
  }
  return d;
}

// Optional per-kernel CUDA-event timing on the launching stream (bench.py's roofline numbers).
struct KernelTimer {
  dfgpu_ctx* ctx;
  dfgpu_kernel_timing* slot = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  KernelTimer(dfgpu_ctx* c, const char* name) : ctx(c) {
    if (!c->time_kernels) return;
    for (auto& t : c->timings) if (t.name == name) { slot = &t; break; }
    if (!slot) { c->timings.emplace_back(); c->timings.back().name = name; slot = &c->timings.back(); }
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0, c->stream);
  }
  ~KernelTimer() {
    if (!slot) return;
    cudaEventRecord(e1, ctx->stream);
    slot->pending.emplace_back(e0, e1);
  }
};

#define DF_LAUNCH_CHECK(ctx)            \
  do {                                  \
    (ctx)->launches++;                  \
    DF_CUDA(cudaGetLastError());        \
  } while (0)

inline int grid_for(int64_t work_items, int per_block, int max_blocks = kNumSMs * 16) {
  int64_t b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

// read one device scalar back (stream-synchronising)
template <class T>
inline T read_scalar(dfgpu_ctx* ctx, const T* dptr) {
  T* h = reinterpret_cast<T*>(ctx->pinned_scalar);
  DF_CUDA(cudaMemcpyAsync(h, dptr, sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  return *h;
}

// Radix partition of n {key, val} rows (radix_probe.cuh, compiled once in hash_join.cu): 16-byte records grouped by the top hash bits of
// the key, so that partition p holds exactly the keys of slot range [p cap / P, (p+1) cap / P) of any fastrange-addressed table
// (slot = hi64(hash_u64(key, kSeedJoin) * cap)).  P = table_bytes / kRadixSubTableMB rounded up to a power of two in [2, kRadixMaxParts],
// or force_parts when >= 2.  keys and vals 16-byte aligned; meta: kRadixMetaWords zeroed device words.  Returns log2(P).
constexpr int kRadixSubTableMB = 16;   // table bytes per partition, a third of the 50 MB L2
constexpr int kRadixMaxParts = 64, kRadixMetaWords = 3 * kRadixMaxParts + 1;
int radix_partition(dfgpu_ctx* ctx, const unsigned long long* keys, const unsigned long long* vals, int64_t n, size_t table_bytes, int force_parts,
                    void* out, unsigned long long* meta);
// The same for n rows that are already 16-byte {key, val} records (recs 16-byte aligned): each 2048-row tile arrives by one bulk copy.
int radix_partition_records(dfgpu_ctx* ctx, const void* recs, int64_t n, size_t table_bytes, int force_parts, void* out, unsigned long long* meta);

// Composite join keys (composite_key.cu): the tuple of 2..4 integer-like components packs into sum_g (v_g - kmin_g) * stride_g, a
// bijection of the declared domain onto [0, domain).  A probe-side key (out_valid == nullptr) whose row has a NULL or out-of-domain
// component becomes `domain`, which no lookup holds.  A build-side key gets a validity bit (out_valid, bit offset 0): 0 for a NULL
// component (counted in flags[1]) and for an out-of-domain one (flags[0] set to 1, never inserted).  Values and bitmaps are read at any
// alignment and Arrow bit offset; out is 16-byte aligned.
constexpr int kMaxKeyParts = 4, kMaxPackedKeys = 4;
struct KeyPart { const void* ptr; const uint8_t* valid; int64_t voff; int width, sgn; unsigned long long kmin, range, stride; };
struct PackedKey { int n_parts, pad; KeyPart part[kMaxKeyParts]; unsigned long long* out; uint8_t* out_valid; unsigned long long domain; };
struct PackKeysParams { int n_keys, pad; PackedKey key[kMaxPackedKeys]; unsigned long long* flags /* [out-of-domain, NULL build keys] */; };
void pack_keys(dfgpu_ctx* ctx, const PackKeysParams& kp, int64_t n);

// ------------------------------------------------------------------------------------------
// device bit helpers (Arrow validity bitmaps are LSB-numbered)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool bit_get(const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; }

// 128-bit streaming load (read-once data: keep it out of L1)
__device__ __forceinline__ int4 ld_stream_16(const void* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_16(void* p, int4 v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ int64_t ld_stream_8(const int64_t* p) {
  int64_t r;
  asm volatile("ld.global.nc.L1::no_allocate.s64 %0, [%1];" : "=l"(r) : "l"(p));
  return r;
}

}  // namespace dfgpu

// extern "C" wrappers: exceptions -> status codes + ctx->last_error
#define DF_API_BEGIN(ctxptr) dfgpu_ctx* _ctx = (ctxptr); try {
#define DF_API_END                                                                   \
  return DFGPU_OK; }                                                                 \
  catch (const dfgpu::Error& e) { if (_ctx) _ctx->last_error = e.what(); return e.code; } \
  catch (const std::exception& e) { if (_ctx) _ctx->last_error = e.what(); return DFGPU_ERR_INVALID; }
