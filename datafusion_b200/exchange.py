"""The partition exchange between GPUs: the stand-in for RepartitionExec's channels
(reference datafusion/physical-plan/src/repartition/mod.rs:1097-1145, 2138-2225) when both join inputs
(or the partial aggregate states) must be co-partitioned across the GPUs of one box
(PartitionMode::Partitioned, hash_join/exec.rs:1312-1325).

  local pass  : libdfgpu dfgpu_hash_partition_device — rows -> n contiguous per-destination regions (CUDA)
  counts      : one tiny all-to-all of the per-destination row counts
  payload     : ONE all-to-all-v per column over NVLink (NCCL through torch.distributed)

torch is plumbing only (process group + NCCL); `backend="gloo"` with CPU tensors exercises the same
host logic in the world_size-2 CPU tests.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

from . import capi as D

_NP = {D.INT8: "|i1", D.UINT8: "|u1", D.INT16: "<i2", D.UINT16: "<u2", D.INT32: "<i4", D.UINT32: "<u4", D.INT64: "<i8", D.UINT64: "<u8",
       D.FLOAT32: "<f4", D.FLOAT64: "<f8", D.DATE32: "<i4", D.DATE64: "<i8", D.TIMESTAMP: "<i8"}


# transport dtype by value width: NCCL (through torch) has no unsigned 16/32/64-bit types, and the exchange only moves bits
_TRANSPORT = {1: "|i1", 2: "<i2", 4: "<i4", 8: "<i8"}


def _as_tensor(torch, dev, ptr, n, type_id, owner):
    """zero-copy torch view of `n` values of a libdfgpu column (an empty tensor for empty / unallocated columns)"""
    w = D.WIDTH[type_id]
    if w not in _TRANSPORT:
        raise NotImplementedError(f"exchange: columns of type {type_id} (width {w}) are not supported yet")
    if n <= 0 or not ptr:
        return torch.empty(0, dtype=torch.as_tensor(np.zeros(0, np.dtype(_TRANSPORT[w]))).dtype, device=dev)
    return torch.as_tensor(_CudaView(ptr, n, _TRANSPORT[w], owner), device=dev)


class _CudaView:
    """zero-copy __cuda_array_interface__ view of a device pointer owned by libdfgpu"""

    def __init__(self, ptr: int, n: int, typestr: str, owner):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2, "strides": None}
        self._owner = owner


def plan_all_to_all(send_counts: Sequence[int], recv_counts: Sequence[int]):
    """split sizes + offsets of one all-to-all-v (pure host logic, unit-tested on CPU)"""
    send_counts = [int(x) for x in send_counts]; recv_counts = [int(x) for x in recv_counts]
    send_offs = np.concatenate([[0], np.cumsum(send_counts)]).astype(np.int64)
    recv_offs = np.concatenate([[0], np.cumsum(recv_counts)]).astype(np.int64)
    return send_counts, recv_counts, send_offs, recv_offs


def exchange_counts(dist, send_counts, device):
    import torch
    world = dist.get_world_size()
    s = torch.tensor(list(send_counts), dtype=torch.int64, device=device)
    r = torch.empty(world, dtype=torch.int64, device=device)
    dist.all_to_all_single(r, s)
    return [int(x) for x in r.tolist()]


def all_to_all_columns(dist, send_tensors, send_counts, recv_counts):
    """one all_to_all_single (all-to-all-v) per column tensor; returns the received tensors"""
    import torch
    out = []
    total = int(sum(recv_counts))
    for t in send_tensors:
        r = torch.empty(total, dtype=t.dtype, device=t.device)
        dist.all_to_all_single(r, t, output_split_sizes=list(recv_counts), input_split_sizes=list(send_counts))
        out.append(r)
    return out


class ExchangedBatch:
    def __init__(self, ctx, tensors, types, rows, keep, validity=None):
        self.ctx, self.tensors, self.types, self.rows, self._keep = ctx, tensors, types, rows, keep
        self.validity = validity or {}      # column index -> device batch whose BOOL column 0 is the validity bitmap

    def columns(self) -> List[D.Column]:
        cols = []
        for i, (t, ty) in enumerate(zip(self.tensors, self.types)):
            c = D.Column()
            c.type, c.flags, c.length, c.offset, c.null_count = ty, 0, self.rows, 0, 0
            c.values = t.data_ptr()
            c.validity = None
            if i in self.validity:
                c.validity = self.validity[i].column(0).values
                c.null_count = -1           # unknown; the consumer reads the bitmap
            cols.append(c)
        return cols


def _plain(c: D.Column) -> D.Column:
    o = D.Column()
    o.type, o.flags, o.length, o.offset, o.null_count, o.values, o.validity = c.type, c.flags, c.length, c.offset, 0, c.values, None
    return o


def _split_validity(ctx: D.Context, cols, key_cols: Sequence[int], nullable=None):
    """Nullable payload columns travel as (values, one INT8 `is valid` column): the exchange kernels and the all-to-all
    move whole fixed-width values only, a bit-packed bitmap cannot be cut at arbitrary row offsets.  The INT8 column is
    `CAST(col IS NOT NULL AS TINYINT)` evaluated on the device; the receiver turns it back into a bitmap with `v <> 0`.
    `nullable` forces the extra column for the listed columns even when this rank's batch happens to carry no bitmap:
    every rank must exchange the same number of columns."""
    arr = D._cols(cols)
    n = arr[0].length if len(cols) else 0
    plain, extra, vmap, keep = [], [], {}, []
    keys = list(key_cols)
    for i in range(len(cols)):
        c = arr[i]
        if c.validity or (nullable is not None and i in nullable):
            b = D.evaluate_device(ctx, [c], n, [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0), (D.EXPR_IS_NOT_NULL, 0, 0, 0, 0, 0.0), (D.EXPR_CAST, 0, D.INT8, 0, 0, 0.0)])
            keep.append(b)
            vmap[i] = len(cols) + len(extra)
            extra.append(b.column(0))
            if i in key_cols:
                # a nullable partition key (NULL group / NullEqualsNull key): hash (canonical value, is-valid) so that all NULLs
                # meet on one rank whatever bits sit under them — evaluating the bare column zeroes the value of NULL rows
                canon = D.evaluate_device(ctx, [c], n, [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0)])
                keep.append(canon)
                plain.append(_plain(canon.column(0)))
                keys.append(vmap[i])
                continue
        plain.append(_plain(c))
    return plain + extra, vmap, keep, keys


def exchange_batch(ctx: D.Context, cols, key_cols: Sequence[int], dist, nullable=None) -> ExchangedBatch:
    """hash-partition `cols` (device) on `key_cols` across the process group and exchange them; nullable non-key
    columns are supported (see _split_validity; pass `nullable` when nullability is data dependent)"""
    import torch
    world = dist.get_world_size()
    n_user = len(cols)
    cols, vmap, keep_valid, key_cols = _split_validity(ctx, cols, list(key_cols), nullable)
    batch, offs = D.hash_partition_device(ctx, cols, list(key_cols), world)
    send_counts = [offs[p + 1] - offs[p] for p in range(world)]
    dev = torch.device("cuda", ctx.device)
    shared_stream = (ctx.lib.dfgpu_ctx_stream(ctx.h) or 0) == torch.cuda.current_stream().cuda_stream
    if not shared_stream:
        ctx.sync()  # partitioned buffers must be complete before NCCL (ordered on torch's stream) reads them
    recv_counts = exchange_counts(dist, send_counts, dev)
    send_tensors, types = [], []
    for i in range(batch.num_columns):
        c = batch.column(i)
        send_tensors.append(_as_tensor(torch, dev, c.values, c.length, c.type, batch))
        types.append(c.type)
    recv = all_to_all_columns(dist, send_tensors, send_counts, recv_counts)
    if not shared_stream:
        torch.cuda.current_stream().synchronize()
    rows = int(sum(recv_counts))
    validity = {}
    for i, j in vmap.items():
        v = D.Column()
        v.type, v.flags, v.length, v.offset, v.null_count, v.values, v.validity = D.INT8, 0, rows, 0, 0, recv[j].data_ptr(), None
        validity[i] = D.evaluate_device(ctx, [v], rows, [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.INT8, 0, 0, 0.0), (D.EXPR_BINARY, D.OP_NEQ, 0, 0, 0, 0.0)])
    return ExchangedBatch(ctx, recv[:n_user], types[:n_user], rows, (batch, recv, keep_valid), validity)


def all_gather_columns(ctx: D.Context, cols, dist):
    """Replicate device columns (no NULLs) on every rank, concatenated in rank order: the CollectLeft analogue
    (hash_join/exec.rs:1326-1336 — a small build side is collected once and shared by every probe partition)."""
    import torch
    world = dist.get_world_size()
    arr = D._cols(cols)
    n = int(arr[0].length)
    dev = torch.device("cuda", ctx.device)
    shared_stream = (ctx.lib.dfgpu_ctx_stream(ctx.h) or 0) == torch.cuda.current_stream().cuda_stream
    if not shared_stream:
        ctx.sync()
    cnt = torch.tensor([n], dtype=torch.int64, device=dev)
    allc = torch.empty(world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(allc, cnt)
    counts = [int(x) for x in allc.tolist()]
    mx, total = max(counts), sum(counts)
    out, types = [], []
    for i in range(len(cols)):
        c = arr[i]
        if c.validity:
            raise NotImplementedError("all_gather_columns: nullable columns are not supported yet")
        mine = _as_tensor(torch, dev, c.values, n, c.type, cols)
        padded = torch.empty(mx, dtype=mine.dtype, device=dev)
        padded[:n] = mine
        gathered = torch.empty(world * mx, dtype=mine.dtype, device=dev)
        dist.all_gather_into_tensor(gathered, padded)
        out.append(torch.cat([gathered[r * mx: r * mx + counts[r]] for r in range(world)]) if any(k != mx for k in counts) else gathered)
        types.append(c.type)
    if not shared_stream:
        torch.cuda.current_stream().synchronize()
    return ExchangedBatch(ctx, out, types, total, None)


def _bitmap_bytes(rows: int) -> int:
    return (int(rows) + 63) // 64 * 8          # whole 64-bit words: the scatter writes bitmaps in 32-bit words


def has_bitmap(arr, n_cols: int) -> List[int]:
    """per column of a dfgpu_column array: 1 when it carries a validity bitmap that may hold a NULL (pure host logic)"""
    return [1 if (arr[i].validity and arr[i].null_count != 0) else 0 for i in range(n_cols)]


class PeerExchange:
    """Fused partition + exchange over NVLink peer memory (no NCCL payload transfer).

    Every rank owns one persistent receive buffer and one receive validity bitmap per column (capacity `cap_rows`; a
    Boolean column's buffer is a bitmap too), exported once through CUDA IPC; an exchange is: count rows per destination
    (CUDA) -> all-gather the world x world count matrix and every rank's per-column "has a validity bitmap" flags (tiny
    NCCL collective, which also orders this exchange after everybody's previous use of the buffers) -> ONE scatter
    kernel that writes each row directly into its owner's buffer -> a one-element all-reduce as the completion
    barrier.  Rows arrive grouped by source rank, in source order (same layout as the all-to-all path).  A column arrives
    with a validity bitmap when any sender had one (the other senders' rows are marked valid)."""

    def __init__(self, ctx: D.Context, dist, col_types: Sequence[int], cap_rows: int):
        import torch
        self.ctx, self.dist, self.types, self.cap = ctx, dist, list(col_types), int(cap_rows)
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.dev = torch.device("cuda", ctx.device)
        self.bufs = [D.DeviceBuffer(ctx, _bitmap_bytes(self.cap) if t == D.BOOL else self.cap * D.WIDTH[t]) for t in self.types]
        self.vbufs = [D.DeviceBuffer(ctx, _bitmap_bytes(self.cap)) for _ in self.types]
        import ctypes as C
        shared = self.bufs + self.vbufs
        mine = torch.zeros(len(shared) * 64, dtype=torch.uint8)
        for i, b in enumerate(shared):
            h = C.create_string_buffer(64)
            ctx.check(ctx.lib.dfgpu_ipc_export(ctx.h, C.c_void_p(b.ptr), h))
            mine[i * 64:(i + 1) * 64] = torch.frombuffer(bytearray(h.raw), dtype=torch.uint8)
        allh = [torch.zeros_like(mine).to(self.dev) for _ in range(self.world)]
        dist.all_gather(allh, mine.to(self.dev))
        nc = len(self.types)
        self.peer_ptrs, self.peer_valid = [], []   # [rank][col]
        for r in range(self.world):
            ptrs = []
            hb = bytes(allh[r].cpu().numpy().tobytes())
            for i in range(len(shared)):
                if r == self.rank:
                    ptrs.append(shared[i].ptr)
                else:
                    out = C.c_void_p()
                    ctx.check(ctx.lib.dfgpu_ipc_import(ctx.h, hb[i * 64:(i + 1) * 64], C.byref(out)))
                    ptrs.append(out.value)
            self.peer_ptrs.append(ptrs[:nc])
            self.peer_valid.append(ptrs[nc:])
        self._flag = torch.zeros(1, dtype=torch.int32, device=self.dev)

    def scatter(self, plan, chunk: int, dst_row, recv_valid):
        """scatter one chunk of a partition plan into the receive buffers; recv_valid[c]: column c keeps a receive bitmap"""
        import ctypes as C
        ctx, world, nc = self.ctx, self.world, len(self.types)
        bases = (C.c_void_p * (world * nc))(*[self.peer_ptrs[p][c] for p in range(world) for c in range(nc)])
        vbases = (C.c_void_p * (world * nc))(*[self.peer_valid[p][c] if recv_valid[c] else None for p in range(world) for c in range(nc)])
        rows = (C.c_int64 * world)(*[int(x) for x in dst_row])
        ctx.check(ctx.lib.dfgpu_partition_plan_scatter_peer_chunk_nullable(plan, int(chunk), bases, vbases, rows))

    def columns(self, start: int, rows: int, recv_valid) -> List[D.Column]:
        """device views of receive rows [start, start + rows)"""
        cols = []
        for i, ty in enumerate(self.types):
            c = D.Column()
            c.type, c.flags, c.length, c.offset = ty, 0, int(rows), int(start)
            c.values = self.bufs[i].ptr
            c.validity = self.vbufs[i].ptr if recv_valid[i] else None
            c.null_count = -1 if recv_valid[i] else 0
            cols.append(c)
        return cols

    def exchange(self, cols, key_cols: Sequence[int]) -> "ExchangedPeerBatch":
        import ctypes as C
        import torch
        ctx, world, nc = self.ctx, self.world, len(self.types)
        arr = D._cols(cols)
        counts = (C.c_int64 * world)()
        plan = C.c_void_p()
        ctx.check(ctx.lib.dfgpu_partition_plan_create(ctx.h, arr, nc, D._i32arr(list(key_cols)), len(key_cols), world, counts, C.byref(plan)))
        try:
            mine = torch.tensor(list(counts) + has_bitmap(arr, nc), dtype=torch.int64, device=self.dev)
            allc = torch.empty(world * (world + nc), dtype=torch.int64, device=self.dev)
            self.dist.all_gather_into_tensor(allc, mine)          # [src][dst | col]; also the "buffers are free again" barrier
            g = allc.view(world, world + nc).cpu().numpy()
            m, recv_valid = g[:, :world], g[:, world:].any(axis=0).tolist()
            recv_rows = int(m[:, self.rank].sum())
            if m.sum(axis=0).max() > self.cap:
                raise RuntimeError(f"PeerExchange: a receive buffer would overflow ({int(m.sum(axis=0).max())} rows > capacity {self.cap})")
            self.scatter(plan, 0, [int(m[:self.rank, p].sum()) for p in range(world)], recv_valid)   # my block starts after lower ranks' blocks
            shared_stream = (ctx.lib.dfgpu_ctx_stream(ctx.h) or 0) == torch.cuda.current_stream().cuda_stream
            if not shared_stream:
                ctx.sync()
            self.dist.all_reduce(self._flag)                       # completion barrier: every rank's scatter has finished
            if not shared_stream:
                torch.cuda.current_stream().synchronize()
        finally:
            ctx.lib.dfgpu_partition_plan_destroy(plan)
        return ExchangedPeerBatch(self, recv_rows, recv_valid)


class ExchangedPeerBatch:
    def __init__(self, px: PeerExchange, rows: int, recv_valid):
        self.px, self.rows, self.recv_valid = px, rows, list(recv_valid)

    def columns(self) -> List[D.Column]:
        return self.px.columns(0, self.rows, self.recv_valid)


def peer_chunk_layout(m, rank: int):
    """Receive-buffer layout of a chunked peer exchange (pure host logic, unit-tested on CPU).

    m[src][chunk][dst] = rows rank `src` sends to rank `dst` from its chunk `chunk`.  Every receiver lays its buffer
    out chunk-major, then by source rank, rows in source order — so chunk c of ALL sources is one contiguous slice
    that can be handed to the consumer as soon as the c-th completion barrier has passed.
    Returns (dst_row[chunk][dst]: where `rank`'s block starts at receiver dst,
             recv_start[chunk], recv_rows[chunk]: `rank`'s own slices,
             max_rows: the fullest receive buffer in the group)."""
    m = np.asarray(m, dtype=np.int64)
    world, chunks, world2 = m.shape
    assert world == world2 and 0 <= rank < world
    per_chunk = m.sum(axis=0)                                            # [chunk][dst]
    chunk_start = np.zeros_like(per_chunk)
    chunk_start[1:] = np.cumsum(per_chunk, axis=0)[:-1]
    dst_row = chunk_start + m[:rank].sum(axis=0)                         # lower ranks' blocks come first inside a chunk
    return dst_row, chunk_start[:, rank].copy(), per_chunk[:, rank].copy(), int(per_chunk.sum(axis=0).max())


def allgather_wrapping_sum(dist, values: Sequence[int], device) -> List[int]:
    """element-wise sum mod 2^64 of one vector of unsigned 64-bit values per rank (order-independent result fingerprints: every group /
    row is owned by exactly one rank).  Exact on the host from an all-gather — NCCL / gloo reductions have no wrapping uint64 sum."""
    import torch
    m64 = (1 << 64) - 1
    t = torch.tensor([int(v) - (1 << 64) if int(v) >= (1 << 63) else int(v) for v in values], dtype=torch.int64, device=device)
    allt = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(allt, t)
    tot = [0] * len(values)
    for a in allt:
        for i, v in enumerate(a.cpu().tolist()):
            tot[i] = (tot[i] + (v & m64)) & m64
    return tot


def _check_distributed_join(join_kwargs, supported, who):
    jt = join_kwargs.get("join_type", D.JOIN_INNER)
    if jt not in supported:
        raise D.DfgpuError(-3, f"{who}: join type {jt} needs a visited bitmap shared by all probe partitions; not supported across GPUs")
    if join_kwargs.get("null_aware"):
        raise D.DfgpuError(-3, f"{who}: null-aware anti joins need global NULL flags; not supported across GPUs")


class PartitionedHashJoin:
    """PartitionMode::Partitioned hash join over the GPUs of one box (hash_join/exec.rs:1312-1325 + the two
    RepartitionExec(Hash) inputs, repartition/mod.rs:1097-1145), with the exchange fused into the pipeline:

      exchange stream : count -> all-gather the [1+chunks] x world count rows (one tiny NCCL collective for BOTH sides)
                        -> scatter build rows into the owners' HBM over NVLink -> barrier
                        -> for each probe chunk: scatter -> barrier                      (peer stores, no NCCL payload)
      join stream     : wait(build barrier) -> build table -> for each chunk: wait(chunk barrier) -> probe + emit

    so the probe of chunk c runs while chunk c+1 is still on the wire (the reference overlaps the same way: the
    repartition channels stream batches into HashJoinStream).  Output order: chunk-major, then source rank, then
    source row order — one of the interleavings RepartitionExec may produce."""

    def __init__(self, device: int, dist, build_types, probe_types, on_build, on_probe, out_side, out_index,
                 cap_build_rows: int, cap_probe_rows: int, n_chunks: int = 4, **join_kwargs):
        import torch
        # co-partitioned inputs: every key lives on exactly one rank, so every join type is rank-local — except null-aware
        # anti joins, whose probe_has_null / build-NULL flags are global and which the reference only plans as CollectLeft
        _check_distributed_join(join_kwargs, tuple(range(10)), "PartitionedHashJoin")
        self.torch, self.dist = torch, dist
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.xs, self.js = torch.cuda.Stream(device), torch.cuda.Stream(device)
        self.ctx_x, self.ctx = D.Context(device, self.xs.cuda_stream), D.Context(device, self.js.cuda_stream)
        self.n_chunks = int(n_chunks)
        self.build_types, self.probe_types = list(build_types), list(probe_types)
        self.on_build, self.on_probe, self.out_side, self.out_index, self.join_kwargs = list(on_build), list(on_probe), list(out_side), list(out_index), join_kwargs
        with torch.cuda.stream(self.xs):
            self.px_b = PeerExchange(self.ctx_x, dist, self.build_types, cap_build_rows)
            self.px_p = PeerExchange(self.ctx_x, dist, self.probe_types, cap_probe_rows)
        self._flag = torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", device))
        self.dev = torch.device("cuda", device)

    def _plan(self, cols, key_cols, n_chunks):
        import ctypes as C
        ctx = self.ctx_x
        arr = D._cols(cols)
        counts = (C.c_int64 * (self.world * n_chunks))()
        plan = C.c_void_p()
        ctx.check(ctx.lib.dfgpu_partition_plan_create_chunked(ctx.h, arr, len(cols), D._i32arr(list(key_cols)), len(key_cols), self.world, n_chunks, counts, C.byref(plan)))
        return plan, np.array(list(counts), dtype=np.int64).reshape(n_chunks, self.world), arr

    def _gather_counts(self, cnt, flags):
        """all-gather every rank's [chunks][world] counts and per-column bitmap flags: (m[src][chunk][dst], recv_valid[col])"""
        torch, world = self.torch, self.world
        chunks = cnt.shape[0]
        mine = torch.from_numpy(np.concatenate([cnt.reshape(-1), np.asarray(flags, dtype=np.int64)])).to(self.dev)
        allc = torch.empty(world * mine.numel(), dtype=torch.int64, device=self.dev)
        self.dist.all_gather_into_tensor(allc, mine)          # also: every rank has finished reading the previous step's buffers
        g = allc.view(world, -1).cpu().numpy()
        return g[:, :chunks * world].reshape(world, chunks, world), g[:, chunks * world:].any(axis=0).tolist()

    # -- streaming form: build once, then any number of probe batches (each call is collective) ----------------
    def build(self, build_cols):
        """exchange the build side and build this rank's table (collect_left_input of the partitioned join)"""
        torch = self.torch
        assert getattr(self, "_join", None) is None, "PartitionedHashJoin: build() called twice without finish()"
        plan = None
        try:
            with torch.cuda.stream(self.xs):
                plan, cnt, arr = self._plan(build_cols, self.on_build, 1)
                m, valid = self._gather_counts(cnt, has_bitmap(arr, len(self.build_types)))
                row, start, rows, mx = peer_chunk_layout(m, self.rank)
                if mx > self.px_b.cap:
                    raise RuntimeError(f"PartitionedHashJoin: build receive buffer would overflow ({mx} rows > capacity {self.px_b.cap})")
                self.px_b.scatter(plan, 0, row[0], valid)
                self.dist.all_reduce(self._flag)
                ev = torch.cuda.Event(); ev.record(self.xs)
            self._join = D.HashJoinHandle(self.ctx, self.build_types, self.probe_types, self.on_build, self.on_probe, self.out_side, self.out_index, **self.join_kwargs)
            self.js.wait_event(ev)
            self._join.push_build_device(self.px_b.columns(start[0], rows[0], valid))
            self._join.finish_build()
            self.xs.synchronize()
        finally:
            if plan is not None:
                self.ctx_x.lib.dfgpu_partition_plan_destroy(plan)

    def probe(self, probe_cols, n_chunks: int = None, keep_output: bool = True):
        """exchange one probe batch (in n_chunks pieces, scatter of piece c+1 overlapping the probe of piece c) and probe
        it; returns the device output batches.  Host-synchronous: the batch is fully consumed when the call returns."""
        torch = self.torch
        C = int(n_chunks or self.n_chunks)
        j = self._join
        plan, outs = None, []
        try:
            with torch.cuda.stream(self.xs):
                plan, cnt, arr = self._plan(probe_cols, self.on_probe, C)
                m, valid = self._gather_counts(cnt, has_bitmap(arr, len(self.probe_types)))   # also: the receive buffers are free again
                row, start, rows, mx = peer_chunk_layout(m, self.rank)
                if mx > self.px_p.cap:
                    raise RuntimeError(f"PartitionedHashJoin: probe receive buffer would overflow ({mx} rows > capacity {self.px_p.cap})")
                evs = []
                for c in range(C):
                    self.px_p.scatter(plan, c, row[c], valid)
                    self.dist.all_reduce(self._flag)
                    e = torch.cuda.Event(); e.record(self.xs); evs.append(e)
            for c in range(C):
                self.js.wait_event(evs[c])
                j.push_probe_device(self.px_p.columns(start[c], rows[c], valid))
                got = j.drain(host=False)
                if keep_output:
                    outs += got
                else:
                    for b in got:
                        b.release()
            self.xs.synchronize()
            return outs
        finally:
            if plan is not None:
                self.ctx_x.lib.dfgpu_partition_plan_destroy(plan)

    def finish(self, keep_output: bool = True):
        """ExhaustedProbeSide: final (unmatched build) rows for outer joins; closes the join.  Returns (output_rows, batches)."""
        j = self._join
        try:
            j.finish_probe()
            tail = j.drain(host=False)
            if not keep_output:
                for b in tail:
                    b.release()
                tail = []
            return j.metric("output_rows"), tail
        finally:
            j.close()
            self._join = None

    def run(self, build_cols, probe_cols, keep_output: bool = True):
        """build_cols / probe_cols: this rank's device-resident input columns (complete before the call).  One fused
        step: both sides' counts travel in ONE collective.  Returns (output_rows, [device batches])."""
        torch, C = self.torch, self.n_chunks
        plans = []
        try:
            with torch.cuda.stream(self.xs):
                plan_b, cnt_b, keep_b = self._plan(build_cols, self.on_build, 1); plans.append(plan_b)
                plan_p, cnt_p, keep_p = self._plan(probe_cols, self.on_probe, C); plans.append(plan_p)
                nb = len(self.build_types)
                m, valid = self._gather_counts(np.concatenate([cnt_b, cnt_p]), has_bitmap(keep_b, nb) + has_bitmap(keep_p, len(self.probe_types)))
                valid_b, valid_p = valid[:nb], valid[nb:]
                row_b, start_b, rows_b, max_b = peer_chunk_layout(m[:, :1, :], self.rank)
                row_p, start_p, rows_p, max_p = peer_chunk_layout(m[:, 1:, :], self.rank)
                if max_b > self.px_b.cap or max_p > self.px_p.cap:
                    raise RuntimeError(f"PartitionedHashJoin: a receive buffer would overflow (build {max_b}/{self.px_b.cap}, probe {max_p}/{self.px_p.cap} rows)")
                self.px_b.scatter(plan_b, 0, row_b[0], valid_b)
                self.dist.all_reduce(self._flag)                    # completion barrier, ordered on the exchange stream
                ev_b = torch.cuda.Event(); ev_b.record(self.xs)
                ev_p = []
                for c in range(C):
                    self.px_p.scatter(plan_p, c, row_p[c], valid_p)
                    self.dist.all_reduce(self._flag)
                    e = torch.cuda.Event(); e.record(self.xs); ev_p.append(e)
            j = D.HashJoinHandle(self.ctx, self.build_types, self.probe_types, self.on_build, self.on_probe, self.out_side, self.out_index, **self.join_kwargs)
            outs = []
            try:
                self.js.wait_event(ev_b)
                j.push_build_device(self.px_b.columns(start_b[0], rows_b[0], valid_b))
                j.finish_build()
                for c in range(C):
                    self.js.wait_event(ev_p[c])
                    j.push_probe_device(self.px_p.columns(start_p[c], rows_p[c], valid_p))
                    if keep_output:
                        outs += j.drain(host=False)
                    else:
                        for b in j.drain(host=False):
                            b.release()
                j.finish_probe()
                tail = j.drain(host=False)
                if keep_output:
                    outs += tail
                else:
                    for b in tail:
                        b.release()
                rows = j.metric("output_rows")
            finally:
                j.close()
            self.xs.synchronize()
            return rows, outs
        finally:
            for p in plans:
                self.ctx_x.lib.dfgpu_partition_plan_destroy(p)


class PartitionedAggregate:
    """GROUP BY over the GPUs of one box, the reference's two-phase plan (aggregates/mod.rs:28-48,
    core/src/physical_planner.rs:1123-1154):

      AggregateMode::Partial on every GPU (no communication)
        -> RepartitionExec(Hash(group keys)) of the partial STATES only — never raw rows
        -> AggregateMode::FinalPartitioned on the owner of each key range.

    Every rank returns the final groups it owns; the union over ranks is the global result."""

    def __init__(self, ctx: D.Context, dist, input_types, group_cols, aggs, capacity_hint: int = 0):
        self.ctx, self.dist = ctx, dist
        self.input_types, self.group_cols, self.aggs, self.capacity_hint = list(input_types), list(group_cols), list(aggs), int(capacity_hint)

    def run(self, cols):
        ctx, ng = self.ctx, len(self.group_cols)
        part = D.AggHandle(ctx, self.input_types, self.group_cols, self.aggs, D.AGG_PARTIAL, 8192, self.capacity_hint)
        fin = None
        try:
            part.push_device(cols)
            part.finish()
            states = part.drain(host=False)
            # every rank must take part in every exchange round: agree on the number of rounds and on the state schema
            # (a rank without input rows has no state batch to read the types from)
            import torch
            world = self.dist.get_world_size()
            k = ng + sum(2 if f == D.AGG_AVG else 1 for f, _, _ in self.aggs)
            mine = [len(states)] + ([states[0].column(i).type for i in range(k)] if states else [-1] * k)
            dev = torch.device("cuda", ctx.device)
            allm = torch.empty(world * (1 + k), dtype=torch.int64, device=dev)
            self.dist.all_gather_into_tensor(allm, torch.tensor(mine, dtype=torch.int64, device=dev))
            allm = allm.view(world, 1 + k).cpu().numpy()
            rounds = int(allm[:, 0].max())
            if rounds == 0:
                return []
            types = [int(t) for t in allm[int(np.argmax(allm[:, 0] > 0)), 1:]]
            empty = D.DeviceBuffer(ctx, 64)
            # SUM / MIN / MAX states are NULL for groups that saw no value (NullState): data dependent, so always shipped as nullable
            nullable, pos = set(range(ng)), ng            # group keys: the table always emits them nullable (NULL group)
            for f, _, _ in self.aggs:
                if f == D.AGG_AVG:
                    pos += 2
                else:
                    if f in (D.AGG_SUM, D.AGG_MIN, D.AGG_MAX):
                        nullable.add(pos)
                    pos += 1
            keep = []
            for r in range(rounds):                              # one exchange per emitted state batch
                if r < len(states):
                    scols = [states[r].column(i) for i in range(k)]
                else:
                    scols = []
                    for t in types:
                        c = D.Column()
                        c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = t, 0, 0, 0, 0, empty.ptr, None
                        scols.append(c)
                ex = exchange_batch(ctx, scols, list(range(ng)), self.dist, nullable)
                keep.append(ex)
                if fin is None:
                    fin = D.AggHandle(ctx, types, list(range(ng)), [(f, -1, -1) for f, _, _ in self.aggs], D.AGG_FINAL_PARTITIONED, 8192, self.capacity_hint)
                fin.push_device(ex.columns())
            fin.finish()
            out = fin.drain(host=False)
            ctx.sync()
            for st in states:
                st.release()
            return out
        finally:
            part.close()
            if fin is not None:
                fin.close()


class BroadcastHashJoin:
    """PartitionMode::CollectLeft across GPUs (hash_join/exec.rs:1326-1336): the (small) build side is replicated on
    every GPU with one all-gather per column, the probe side stays where it is — no probe-side exchange at all."""

    # join types whose output depends only on (replicated build table, local probe rows): safe with a per-rank replica.
    # Left / Full / LeftSemi / LeftAnti / LeftMark emit build rows from ONE visited bitmap shared by all probe partitions
    # (exec.rs:206/274 report_probe_completed, stream.rs:1026): a per-rank replica would emit them once per rank.
    SUPPORTED = (D.JOIN_INNER, D.JOIN_RIGHT, D.JOIN_RIGHT_SEMI, D.JOIN_RIGHT_ANTI, D.JOIN_RIGHT_MARK)

    def __init__(self, ctx: D.Context, dist, build_types, probe_types, on_build, on_probe, out_side, out_index, **join_kwargs):
        _check_distributed_join(join_kwargs, self.SUPPORTED, "BroadcastHashJoin")
        self.ctx, self.dist = ctx, dist
        self.args = (list(build_types), list(probe_types), list(on_build), list(on_probe), list(out_side), list(out_index))
        self.join_kwargs = join_kwargs

    def run(self, build_cols, probe_cols):
        g = all_gather_columns(self.ctx, build_cols, self.dist)
        j = D.HashJoinHandle(self.ctx, *self.args, **self.join_kwargs)
        try:
            j.push_build_device(g.columns())
            j.finish_build()
            j.push_probe_device(probe_cols)
            outs = j.drain(host=False)
            j.finish_probe()
            outs += j.drain(host=False)
            return j.metric("output_rows"), outs
        finally:
            j.close()
