// comm.cu — multi-GPU control inside the C ABI: dfgpu_comm (rendezvous, barrier, count all-gather, buffer sharing) and
// dfgpu_exchange (RepartitionExec Hash as fused partition + peer-memory scatter), so that a Rust host — one process (or thread)
// per GPU — drives the partition exchange without NCCL or torch.distributed.
//
// Reference being replaced: RepartitionExec / BatchPartitioner::Hash + the channels between the partitions
// (physical-plan/src/repartition/mod.rs:618-648, 1097-1145, 1320-1400).  There the "communicator" is a set of in-process tokio channels;
// here the ranks are processes on one box, so the control plane is a POSIX shared-memory segment (named after a 128-byte unique id the
// application hands to every rank, like ncclUniqueId) and the data plane is CUDA IPC: every rank maps every peer's receive buffers and the
// scatter kernel stores rows straight into the owner's HBM over NVLink.  Control messages are a few hundred bytes per exchange (a
// world x world count matrix, sense-reversing barriers): host shared memory moves them in microseconds.
#include "batch.cuh"
#include <atomic>
#include <chrono>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <thread>
#include <unistd.h>

namespace dfgpu {

constexpr int kCommMaxRanks = 8, kCommGatherWords = 64, kCommMaxShared = 16;
constexpr uint32_t kCommMagic = 0xDF69C033u;

struct CommShm {
  std::atomic<uint32_t> magic;
  std::atomic<int32_t> n_ranks;
  std::atomic<int32_t> arrived;
  std::atomic<uint32_t> generation;
  std::atomic<int32_t> failed;
  int64_t gather[kCommMaxRanks][kCommGatherWords];
  uint8_t ipc[kCommMaxRanks][kCommMaxShared][64];
};

}  // namespace dfgpu

using namespace dfgpu;

struct dfgpu_comm {
  dfgpu_ctx* ctx = nullptr;
  int n_ranks = 0, rank = 0;
  std::string shm_name;
  CommShm* shm = nullptr;
  std::vector<void*> imported;   // peer mappings to close
};

struct dfgpu_exchange {
  dfgpu_comm* comm = nullptr;
  std::vector<int> types;
  int64_t cap = 0, recv_rows = 0;
  std::vector<DevBuf> bufs, vbufs;                // this rank's receive buffers and receive validity bitmaps, one per column
  std::vector<std::vector<void*>> peer, peer_valid;   // [rank][col]
  std::vector<bool> recv_valid;                   // per column: the last run's rows carry a validity bitmap (some sender had one)
};

namespace dfgpu {

static void comm_barrier(dfgpu_comm* c) {
  CommShm* s = c->shm;
  const uint32_t gen = s->generation.load(std::memory_order_acquire);
  if (s->arrived.fetch_add(1, std::memory_order_acq_rel) + 1 == c->n_ranks) {
    s->arrived.store(0, std::memory_order_relaxed);
    s->generation.fetch_add(1, std::memory_order_acq_rel);
    return;
  }
  const auto t0 = std::chrono::steady_clock::now();
  int spins = 0;
  while (s->generation.load(std::memory_order_acquire) == gen) {
    if (++spins > 2000) { std::this_thread::yield(); }
    if ((spins & 0xFFFF) == 0) {
      if (s->failed.load(std::memory_order_relaxed)) throw Error(DFGPU_ERR_STATE, "comm: another rank failed");
      if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(120)) { s->failed.store(1); throw Error(DFGPU_ERR_STATE, "comm: barrier timed out after 120 s (a rank is missing)"); }
    }
  }
}

}  // namespace dfgpu

extern "C" {

int dfgpu_comm_unique_id(uint8_t* id_out /* 128 bytes */) {
  if (!id_out) return DFGPU_ERR_INVALID;
  memset(id_out, 0, 128);
  int fd = open("/dev/urandom", O_RDONLY);
  if (fd < 0 || read(fd, id_out, 16) != 16) { if (fd >= 0) close(fd); return DFGPU_ERR_INVALID; }
  close(fd);
  return DFGPU_OK;
}

int dfgpu_comm_init(dfgpu_ctx* ctx, int32_t n_ranks, int32_t rank, const uint8_t* id /* 128 bytes */, dfgpu_comm** out) {
  DF_API_BEGIN(ctx)
  DF_CHECK(ctx && id && out, DFGPU_ERR_INVALID, "null argument");
  DF_CHECK(n_ranks >= 1 && n_ranks <= kCommMaxRanks && rank >= 0 && rank < n_ranks, DFGPU_ERR_INVALID, "comm: 1..8 ranks of one box");
  std::unique_ptr<dfgpu_comm> c(new dfgpu_comm());
  c->ctx = ctx; c->n_ranks = n_ranks; c->rank = rank;
  char name[64];
  snprintf(name, sizeof(name), "/dfgpu_%02x%02x%02x%02x%02x%02x%02x%02x%02x%02x%02x%02x", id[0], id[1], id[2], id[3], id[4], id[5], id[6], id[7], id[8], id[9], id[10], id[11]);
  c->shm_name = name;
  int fd = -1;
  if (rank == 0) {
    shm_unlink(name);
    fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
    DF_CHECK(fd >= 0, DFGPU_ERR_STATE, "comm: cannot create the shared-memory segment");
    DF_CHECK(ftruncate(fd, sizeof(CommShm)) == 0, DFGPU_ERR_STATE, "comm: ftruncate failed");
  } else {
    const auto t0 = std::chrono::steady_clock::now();
    while (true) {
      fd = shm_open(name, O_RDWR, 0600);
      if (fd >= 0) { struct stat st; if (fstat(fd, &st) == 0 && (size_t)st.st_size >= sizeof(CommShm)) break; close(fd); fd = -1; }
      DF_CHECK(std::chrono::steady_clock::now() - t0 < std::chrono::seconds(120), DFGPU_ERR_STATE, "comm: rank 0 never created the rendezvous segment");
      std::this_thread::sleep_for(std::chrono::milliseconds(2));
    }
  }
  void* p = mmap(nullptr, sizeof(CommShm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  DF_CHECK(p != MAP_FAILED, DFGPU_ERR_STATE, "comm: mmap failed");
  c->shm = (CommShm*)p;
  if (rank == 0) {
    c->shm->arrived.store(0); c->shm->generation.store(0); c->shm->failed.store(0); c->shm->n_ranks.store(n_ranks);
    c->shm->magic.store(kCommMagic, std::memory_order_release);
  } else {
    const auto t0 = std::chrono::steady_clock::now();
    while (c->shm->magic.load(std::memory_order_acquire) != kCommMagic) {
      DF_CHECK(std::chrono::steady_clock::now() - t0 < std::chrono::seconds(120), DFGPU_ERR_STATE, "comm: rendezvous segment never initialised");
      std::this_thread::sleep_for(std::chrono::milliseconds(1));
    }
    DF_CHECK(c->shm->n_ranks.load() == n_ranks, DFGPU_ERR_INVALID, "comm: ranks disagree on the world size");
  }
  comm_barrier(c.get());
  if (rank == 0) shm_unlink(name);   // everybody has it mapped: the name can go, the memory lives until the last unmap
  *out = c.release();
  DF_API_END
}

int dfgpu_comm_barrier(dfgpu_comm* c) {
  DF_API_BEGIN(c ? c->ctx : nullptr)
  DF_CHECK(c, DFGPU_ERR_INVALID, "null argument");
  set_device(c->ctx);
  DF_CUDA(cudaStreamSynchronize(c->ctx->stream));   // "every rank's queued work is done", not only "every rank got here"
  comm_barrier(c);
  DF_API_END
}

int dfgpu_comm_allgather_i64(dfgpu_comm* c, const int64_t* mine, int32_t n, int64_t* all /* [n_ranks][n] */) {
  DF_API_BEGIN(c ? c->ctx : nullptr)
  DF_CHECK(c && mine && all && n >= 1 && n <= kCommGatherWords, DFGPU_ERR_INVALID, "comm all-gather: 1..64 values per rank");
  memcpy(c->shm->gather[c->rank], mine, (size_t)n * 8);
  comm_barrier(c);
  for (int r = 0; r < c->n_ranks; ++r) memcpy(all + (size_t)r * n, c->shm->gather[r], (size_t)n * 8);
  comm_barrier(c);   // nobody overwrites its slot before everybody has read it
  DF_API_END
}

int dfgpu_comm_share(dfgpu_comm* c, void* dev_ptr, void** peer_ptrs_out /* [n_ranks] */) {
  DF_API_BEGIN(c ? c->ctx : nullptr)
  DF_CHECK(c && dev_ptr && peer_ptrs_out, DFGPU_ERR_INVALID, "null argument");
  set_device(c->ctx);
  cudaIpcMemHandle_t h;
  DF_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
  memcpy(c->shm->ipc[c->rank][0], &h, 64);
  comm_barrier(c);
  for (int r = 0; r < c->n_ranks; ++r) {
    if (r == c->rank) { peer_ptrs_out[r] = dev_ptr; continue; }
    cudaIpcMemHandle_t hr;
    memcpy(&hr, c->shm->ipc[r][0], 64);
    void* p = nullptr;
    DF_CUDA(cudaIpcOpenMemHandle(&p, hr, cudaIpcMemLazyEnablePeerAccess));
    c->imported.push_back(p);
    peer_ptrs_out[r] = p;
  }
  comm_barrier(c);
  DF_API_END
}

int32_t dfgpu_comm_rank(dfgpu_comm* c) { return c ? c->rank : -1; }
int32_t dfgpu_comm_size(dfgpu_comm* c) { return c ? c->n_ranks : -1; }

void dfgpu_comm_destroy(dfgpu_comm* c) {
  if (!c) return;
  cudaSetDevice(c->ctx->device);
  for (void* p : c->imported) cudaIpcCloseMemHandle(p);
  if (c->shm) munmap(c->shm, sizeof(CommShm));
  delete c;
}

// ---- RepartitionExec Hash over the ranks of a communicator ----
int dfgpu_exchange_create(dfgpu_comm* c, const int32_t* col_types, int32_t n_cols, int64_t cap_rows, dfgpu_exchange** out) {
  DF_API_BEGIN(c ? c->ctx : nullptr)
  DF_CHECK(c && col_types && out && n_cols >= 1 && n_cols <= 16 && cap_rows >= 1, DFGPU_ERR_INVALID, "exchange: bad arguments");
  dfgpu_ctx* ctx = c->ctx;
  set_device(ctx);
  std::unique_ptr<dfgpu_exchange> x(new dfgpu_exchange());
  x->comm = c; x->cap = cap_rows;
  x->types.assign(col_types, col_types + n_cols);
  x->peer.assign(c->n_ranks, std::vector<void*>(n_cols, nullptr));
  x->peer_valid = x->peer;
  x->recv_valid.assign(n_cols, false);
  for (int i = 0; i < n_cols; ++i) {
    const int w = type_width(col_types[i]);
    DF_CHECK(col_types[i] == DFGPU_BOOL || (w >= 1 && w <= 16), DFGPU_ERR_UNSUPPORTED, "exchange: Boolean or fixed-width columns of <= 16 bytes");
    // a Boolean column's receive buffer is a bitmap; bitmaps are whole 64-bit words (the scatter writes 32-bit words)
    x->bufs.emplace_back(ctx, col_types[i] == DFGPU_BOOL ? bitmap_alloc_bytes(cap_rows) : (size_t)cap_rows * w);
    x->vbufs.emplace_back(ctx, bitmap_alloc_bytes(cap_rows));
    std::vector<void*> ptrs(c->n_ranks), vptrs(c->n_ranks);
    int rc = dfgpu_comm_share(c, x->bufs.back().ptr, ptrs.data());
    if (rc == DFGPU_OK) rc = dfgpu_comm_share(c, x->vbufs.back().ptr, vptrs.data());
    if (rc != DFGPU_OK) throw Error(rc, ctx->last_error);
    for (int r = 0; r < c->n_ranks; ++r) { x->peer[r][i] = ptrs[r]; x->peer_valid[r][i] = vptrs[r]; }
  }
  *out = x.release();
  DF_API_END
}

// cols: this rank's device-resident rows; rows travel to rank = exchange_hash(key columns) % n_ranks and arrive grouped by
// source rank, in source order.  Collective: every rank calls it.  On return the received rows are complete in this rank's buffers.
int dfgpu_exchange_run(dfgpu_exchange* x, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys, int64_t* recv_rows_out) {
  DF_API_BEGIN(x ? x->comm->ctx : nullptr)
  DF_CHECK(x && cols && key_cols && n_cols == (int)x->types.size(), DFGPU_ERR_INVALID, "exchange: column count differs from the exchange's schema");
  dfgpu_comm* c = x->comm;
  dfgpu_ctx* ctx = c->ctx;
  set_device(ctx);
  const int W = c->n_ranks;
  for (int i = 0; i < n_cols; ++i) DF_CHECK(cols[i].type == x->types[i], DFGPU_ERR_INVALID, "exchange: column type mismatch");
  // what every rank contributes to the all-gather: its row counts per destination, then per column whether its rows carry a validity bitmap
  const int G = W + n_cols;
  int64_t counts[kCommMaxRanks] = {0}, mine[kCommMaxRanks + 16] = {0};
  dfgpu_partition_plan* plan = nullptr;
  int rc = dfgpu_partition_plan_create(ctx, cols, n_cols, key_cols, n_keys, W, counts, &plan);   // histogram on the device; syncs (counts come back)
  if (rc != DFGPU_OK) throw Error(rc, ctx->last_error);
  struct PlanGuard { dfgpu_partition_plan* p; ~PlanGuard() { dfgpu_partition_plan_destroy(p); } } guard{plan};
  // the stream is idle here (the counts were read back): consumers of the previous exchange's rows have finished on this rank, and
  // the all-gather's barrier makes that true for every rank before anybody scatters into anybody's buffers
  for (int d = 0; d < W; ++d) mine[d] = counts[d];
  for (int i = 0; i < n_cols; ++i) mine[W + i] = (cols[i].validity && cols[i].null_count != 0) ? 1 : 0;
  int64_t all[kCommMaxRanks * (kCommMaxRanks + 16)];
  rc = dfgpu_comm_allgather_i64(c, mine, G, all);   // all[src][dst], all[src][W + col]
  if (rc != DFGPU_OK) throw Error(rc, ctx->last_error);
  int64_t recv = 0, dst_row[kCommMaxRanks];
  for (int src = 0; src < W; ++src) recv += all[src * G + c->rank];
  for (int dst = 0; dst < W; ++dst) {
    int64_t tot = 0, before = 0;
    for (int src = 0; src < W; ++src) { if (src < c->rank) before += all[src * G + dst]; tot += all[src * G + dst]; }
    DF_CHECK(tot <= x->cap, DFGPU_ERR_OOM, "exchange: a receive buffer would overflow (raise cap_rows)");
    dst_row[dst] = before;   // lower ranks' blocks come first
  }
  // a column arrives with a validity bitmap when any sender has one; senders without write all-ones into their block
  std::vector<bool> any_valid(n_cols, false);
  for (int i = 0; i < n_cols; ++i) for (int src = 0; src < W; ++src) if (all[src * G + W + i]) any_valid[i] = true;
  std::vector<void*> bases((size_t)W * n_cols), vbases((size_t)W * n_cols);
  for (int p = 0; p < W; ++p)
    for (int i = 0; i < n_cols; ++i) {
      bases[(size_t)p * n_cols + i] = x->peer[p][i];
      vbases[(size_t)p * n_cols + i] = any_valid[i] ? x->peer_valid[p][i] : nullptr;
    }
  rc = dfgpu_partition_plan_scatter_peer_chunk_nullable(plan, 0, bases.data(), vbases.data(), dst_row);
  if (rc != DFGPU_OK) throw Error(rc, ctx->last_error);
  rc = dfgpu_comm_barrier(c);   // every rank's scatter kernel has completed: all rows have landed
  if (rc != DFGPU_OK) throw Error(rc, ctx->last_error);
  x->recv_rows = recv;
  x->recv_valid = any_valid;
  if (recv_rows_out) *recv_rows_out = recv;
  DF_API_END
}

int dfgpu_exchange_columns(dfgpu_exchange* x, dfgpu_column* out, int32_t n_cols) {
  if (!x || !out || n_cols != (int)x->types.size()) return DFGPU_ERR_INVALID;
  for (int i = 0; i < n_cols; ++i) {
    memset(&out[i], 0, sizeof(dfgpu_column));
    out[i].type = x->types[i]; out[i].length = x->recv_rows; out[i].values = x->bufs[i].ptr;
    out[i].validity = x->recv_valid[i] ? (const uint8_t*)x->vbufs[i].ptr : nullptr;
    out[i].null_count = x->recv_valid[i] ? -1 : 0;
  }
  return DFGPU_OK;
}

void dfgpu_exchange_destroy(dfgpu_exchange* x) {
  if (!x) return;
  cudaSetDevice(x->comm->ctx->device);
  delete x;
}

}  // extern "C"
