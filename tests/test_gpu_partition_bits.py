"""Bit-packed data through the hash exchange: validity bitmaps of every column width, Boolean values, Decimal128 keys, and the
peer scatter's receive bitmaps.  The reference is a stable argsort by the restated partition id (as in test_gpu_partition.py):
rows keep their input order inside a partition, a NULL keeps its row, and every validity bit arrives exactly."""
import ctypes as C

import numpy as np
import pytest

from datafusion_b200 import capi as D

pytestmark = pytest.mark.gpu
SEED_EXCHANGE = np.uint64(0x9E3779B97F4A7C15)
ERR_INVALID = -1   # DFGPU_ERR_INVALID


def mix64(x):
    x = x.copy()
    x ^= x >> np.uint64(30); x *= np.uint64(0xBF58476D1CE4E5B9)
    x ^= x >> np.uint64(27); x *= np.uint64(0x94D049BB133111EB)
    x ^= x >> np.uint64(31)
    return x


def part_ids(h, n_parts):
    """floor(h * n_parts / 2^64) without 128-bit integers"""
    hi, lo = h >> np.uint64(32), h & np.uint64(0xFFFFFFFF)
    return ((hi * np.uint64(n_parts) + ((lo * np.uint64(n_parts)) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


def key_hash(words, valid=None):
    """exchange_hash of one key column: an 8-byte key (uint64 view) or Decimal128 words [n, 2] (low word hashed like an
    8-byte key, then the high word combined); a NULL leaves the hash at 0"""
    with np.errstate(over="ignore"):
        if words.ndim == 2:
            h = mix64(words[:, 0] + SEED_EXCHANGE)
            h = mix64(words[:, 1] ^ (h * np.uint64(0x9E3779B97F4A7C15) + np.uint64(0x7F4A7C15)))
        else:
            h = mix64(words + SEED_EXCHANGE)
    if valid is not None:
        h = np.where(valid, h, np.uint64(0))
    return h


class Src:
    """a device column built from host arrays that hold `off` leading rows before the column's first row (Arrow offset)"""

    def __init__(self, ctx, type_id, vals, valid, off):
        self.type, self.vals, self.valid, self.off = type_id, vals, valid, off
        n = len(vals) - off
        if type_id == D.BOOL:
            vbuf = D.pack_bits(vals)
        else:
            vbuf = np.ascontiguousarray(vals)
        self._v = ctx.to_device(vbuf)
        self._m = ctx.to_device(D.pack_bits(valid)) if valid is not None else None
        c = D.Column()
        c.type, c.flags, c.length, c.offset, c.null_count = type_id, 0, n, off, (-1 if valid is not None else 0)
        c.values, c.validity = self._v.ptr, (self._m.ptr if self._m is not None else None)
        self.col = c

    def values(self):
        return self.vals[self.off:]

    def validity(self):
        return None if self.valid is None else self.valid[self.off:]


def make_columns(ctx, rng, n, off):
    """key (Int64, no NULLs), nullable 1/2/4/8/16-byte columns, Boolean with and without validity"""
    m = n + off
    vm = lambda: rng.random(m) > 0.3
    specs = [(D.INT64, rng.integers(-2**62, 2**62, m).astype(np.int64), None),
             (D.INT8, rng.integers(-128, 128, m).astype(np.int8), vm()),
             (D.INT16, rng.integers(-2**15, 2**15, m).astype(np.int16), vm()),
             (D.INT32, rng.integers(-2**31, 2**31, m).astype(np.int32), vm()),
             (D.INT64, np.arange(m, dtype=np.int64), vm()),
             (D.decimal128(38, 4), rng.integers(0, 2**63, (m, 2)).astype(np.uint64), vm()),
             (D.BOOL, rng.random(m) > 0.5, vm()),
             (D.BOOL, rng.random(m) > 0.4, None)]
    return [Src(ctx, t, v, vv, off) for t, v, vv in specs]


def check_partitioned(batch, offs, srcs, pid, n_parts):
    order = np.argsort(pid, kind="stable")
    assert offs[0] == 0 and offs[-1] == len(pid)
    assert [offs[p + 1] - offs[p] for p in range(n_parts)] == np.bincount(pid, minlength=n_parts).tolist()
    for i, s in enumerate(srcs):
        got, gvalid = batch.column_numpy(i)
        exp, evalid = s.values()[order], s.validity()
        if evalid is None:
            assert gvalid is None, f"column {i}: a bitmap appeared"
            assert np.array_equal(got, exp), f"column {i}"
        else:
            evalid = evalid[order]
            assert gvalid is not None and np.array_equal(gvalid, evalid), f"column {i}: validity"
            assert np.array_equal(got[evalid], exp[evalid]), f"column {i}: values at valid rows"


@pytest.mark.parametrize("off", [0, 3, 37])
@pytest.mark.parametrize("n_parts", [1, 2, 5, 8, 13, 32, 33])
def test_nullable_and_boolean_columns_every_width(gpu_ctx, n_parts, off):
    """<= 8 partitions: packed-counter kernels, 9..32: warp-match kernels, 33: the flag / compaction path"""
    rng = np.random.default_rng(n_parts * 100 + off)
    n = 50_003
    srcs = make_columns(gpu_ctx, rng, n, off)
    batch, offs = D.hash_partition_device(gpu_ctx, [s.col for s in srcs], [0], n_parts)
    pid = part_ids(key_hash(srcs[0].values().view(np.uint64)), n_parts)
    check_partitioned(batch, offs, srcs, pid, n_parts)
    batch.release()


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("n_parts", [3, 8, 13, 33])
def test_decimal128_key(gpu_ctx, n_parts, nulls):
    rng = np.random.default_rng(7 * n_parts + nulls)
    n = 40_001
    words = rng.integers(0, 2**63, (n, 2)).astype(np.uint64)
    words[rng.integers(0, n, n // 5)] = words[rng.integers(0, n, n // 5)]   # duplicate keys: equal keys share a partition
    words[::7, 1] = 0                                     # keys that differ from an 8-byte key only by the high word
    valid = (rng.random(n) > 0.1) if nulls else None
    srcs = [Src(gpu_ctx, D.decimal128(20, 2), words, valid, 0), Src(gpu_ctx, D.INT64, np.arange(n, dtype=np.int64), None, 0)]
    batch, offs = D.hash_partition_device(gpu_ctx, [s.col for s in srcs], [0], n_parts)
    pid = part_ids(key_hash(words, valid), n_parts)
    check_partitioned(batch, offs, srcs, pid, n_parts)
    batch.release()


def test_partitioned_join_on_decimal128_key(gpu_ctx):
    """PartitionMode::Partitioned on a Decimal128 key with NULLs: partition by partition == the global join"""
    from oracle import oracle as O
    from harness import assert_cols_equal, gpu_hash_join
    rng = np.random.default_rng(12)
    t = D.decimal128(38, 4)
    universe = rng.integers(0, 2**63, (9000, 2)).astype(np.uint64)
    bw = universe[rng.permutation(6000)[:4000]]; bv = rng.random(4000) > 0.05; bp = np.arange(4000, dtype=np.int64)
    pw = universe[rng.integers(0, 9000, 30000)]; pv = rng.random(30000) > 0.05; pp = np.arange(30000, dtype=np.int64) * 3
    P = 5
    parts = []
    for w, v, pay in ((bw, bv, bp), (pw, pv, pp)):
        s = [Src(gpu_ctx, t, w, v, 0), Src(gpu_ctx, D.INT64, pay, None, 0)]
        batch, offs = D.hash_partition_device(gpu_ctx, [x.col for x in s], [0], P)
        parts.append(([batch.column_numpy(i) for i in range(2)], offs))
        batch.release()
    outs = []
    for p in range(P):
        side = []
        for cols, offs in parts:
            a, b = offs[p], offs[p + 1]
            (kw, kv), (pay, _) = cols
            side.append([(kw[a:b], kv[a:b]), (pay[a:b], None)])
        outs.append(gpu_hash_join(gpu_ctx, side[0], side[1], [0], [0], [0, 1], [1, 1], build_types=[t, D.INT64], probe_types=[t, D.INT64]))
    got = [(np.concatenate([o[c][0] for o in outs]), None) for c in range(2)]
    ob = [(bw[:, 0].view(np.int64).copy(), bv), (bw[:, 1].view(np.int64).copy(), bv), (bp, None)]
    op = [(pw[:, 0].view(np.int64).copy(), pv), (pw[:, 1].view(np.int64).copy(), pv), (pp, None)]
    exp = O.hash_join(ob, op, [0, 1], [0, 1], [0, 1], [2, 2])
    assert len(exp[0][0]) > 1000
    assert_cols_equal(got, exp, ordered=False)


# ---- the peer scatter with every receive buffer on this GPU -------------------------------------------------------------

PEER_TYPES = [D.INT64, D.INT32, D.BOOL, D.decimal128(15, 2)]
PEER_RECV_BITMAP = [True, False, True, True]     # the key has NULLs; Int32 keeps no bitmap; Decimal128 has none at the source


def peer_sources(ctx, rng, n, off):
    m = n + off
    specs = [(D.INT64, rng.integers(-2**62, 2**62, m).astype(np.int64), rng.random(m) > 0.2),
             (D.INT32, np.arange(m, dtype=np.int32), None),
             (D.BOOL, rng.random(m) > 0.5, rng.random(m) > 0.3),
             (D.decimal128(15, 2), rng.integers(0, 2**40, (m, 2)).astype(np.uint64), None)]
    return [Src(ctx, t, v, vv, off) for t, v, vv in specs]


class Receiver:
    """receive buffers of one partition (rank): values per column, and a bitmap per column that keeps one"""

    def __init__(self, ctx, rows, fill):
        self.ctx, self.rows, self.fill = ctx, rows, fill
        nb = (rows + 63) // 64 * 8
        self.vals, self.bits = [], []
        for t, keep in zip(PEER_TYPES, PEER_RECV_BITMAP):
            if t == D.BOOL:
                self.vals.append(ctx.to_device(np.full(nb, fill, np.uint8)))
            else:
                self.vals.append(D.DeviceBuffer(ctx, rows * D.WIDTH[t]))
            self.bits.append(ctx.to_device(np.full(nb, fill, np.uint8)) if keep else None)

    def read_bits(self, buf):
        return D.unpack_bits(self.ctx.to_host(buf.ptr, buf.nbytes), self.rows)

    def read_values(self, ci, start, cnt):
        t = PEER_TYPES[ci]
        if t == D.BOOL:
            return self.read_bits(self.vals[ci])[start:start + cnt]
        w = D.WIDTH[t]
        raw = self.ctx.to_host(self.vals[ci].ptr + start * w, cnt * w)
        return raw.view(np.uint64).reshape(-1, 2) if w == 16 else raw.view(np.int64 if w == 8 else np.int32)


def plan_create(ctx, srcs, n_parts, n_chunks):
    counts = (C.c_int64 * (n_parts * n_chunks))()
    plan = C.c_void_p()
    ctx.check(ctx.lib.dfgpu_partition_plan_create_chunked(ctx.h, D._cols([s.col for s in srcs]), len(srcs), D._i32arr([0]), 1, n_parts, n_chunks,
                                                          counts, C.byref(plan)))
    return plan, np.array(list(counts), dtype=np.int64).reshape(n_chunks, n_parts)


def scatter_nullable(ctx, plan, chunk, recvs, starts):
    nc = len(PEER_TYPES)
    bases = (C.c_void_p * (len(recvs) * nc))(*[r.vals[c].ptr for r in recvs for c in range(nc)])
    vbases = (C.c_void_p * (len(recvs) * nc))(*[(r.bits[c].ptr if r.bits[c] is not None else None) for r in recvs for c in range(nc)])
    rows = (C.c_int64 * len(recvs))(*[int(x) for x in starts])
    ctx.check(ctx.lib.dfgpu_partition_plan_scatter_peer_chunk_nullable(plan, chunk, bases, vbases, rows))


def chunk_bounds(n, n_chunks):
    tile = 2048
    ntiles = (n + tile - 1) // tile
    return [min(n, (ntiles * c // n_chunks) * tile) for c in range(n_chunks)] + [n]


def expected_bits(recv, blocks):
    """per bit-carrying column: the receive bitmap after every (start, source rows, Src list) block has landed"""
    out = {}
    for ci, keep in enumerate(PEER_RECV_BITMAP):
        for kind in (["valid"] if keep else []) + (["bool"] if PEER_TYPES[ci] == D.BOOL else []):
            e = np.full(recv.rows, bool(recv.fill))
            for start, sel, srcs in blocks:
                s = srcs[ci]
                if kind == "bool":
                    e[start:start + len(sel)] = s.values()[sel]
                else:
                    e[start:start + len(sel)] = True if s.validity() is None else s.validity()[sel]
            out[(ci, kind)] = e
    return out


def check_receiver(recv, blocks):
    for (ci, kind), e in expected_bits(recv, blocks).items():
        got = recv.read_bits(recv.bits[ci] if kind == "valid" else recv.vals[ci])
        if kind == "bool":          # Boolean values: exact at valid rows inside the blocks, untouched outside
            valid = expected_bits(recv, blocks)[(ci, "valid")]
            inside = np.zeros(recv.rows, bool)
            for start, sel, _ in blocks:
                inside[start:start + len(sel)] = True
            m = ~inside | valid
            assert np.array_equal(got[m], e[m]), (ci, kind)
        else:
            assert np.array_equal(got, e), (ci, kind)
    for start, sel, srcs in blocks:
        for ci, t in enumerate(PEER_TYPES):
            if t == D.BOOL:
                continue
            got = recv.read_values(ci, start, len(sel))
            exp = srcs[ci].values()[sel]
            v = srcs[ci].validity()
            keep = np.ones(len(sel), bool) if v is None else v[sel]
            assert np.array_equal(got[keep], exp[keep]), (ci, start)


@pytest.mark.parametrize("fill", [0x00, 0xFF])
@pytest.mark.parametrize("n_parts,n_chunks", [(2, 1), (8, 4), (5, 7), (12, 3)])
def test_chunked_peer_scatter_with_receive_bitmaps(gpu_ctx, n_parts, n_chunks, fill):
    """chunk c of partition p lands at the bit offset the caller passed (gaps of 5 rows: blocks start off 32-bit word boundaries),
    chunks issued in reverse order; the bits outside every block keep the prefilled value"""
    ctx = gpu_ctx
    rng = np.random.default_rng(n_parts * 10 + n_chunks + fill)
    n, off = 50_000 + n_parts, 11
    srcs = peer_sources(ctx, rng, n, off)
    plan, cnt = plan_create(ctx, srcs, n_parts, n_chunks)
    try:
        pid = part_ids(key_hash(srcs[0].values().view(np.uint64), srcs[0].validity()), n_parts)
        bounds = chunk_bounds(n, n_chunks)
        for c in range(n_chunks):
            assert cnt[c].tolist() == np.bincount(pid[bounds[c]:bounds[c + 1]], minlength=n_parts).tolist()
        gap = 5
        starts = np.zeros((n_chunks, n_parts), dtype=np.int64)
        for p in range(n_parts):
            run = 0
            for c in range(n_chunks):
                run += gap
                starts[c, p] = run
                run += cnt[c, p]
        recvs = [Receiver(ctx, int(cnt[:, p].sum()) + gap * n_chunks + 40, fill) for p in range(n_parts)]
        for c in reversed(range(n_chunks)):
            scatter_nullable(ctx, plan, c, recvs, starts[c])
        ctx.sync()
        for p in range(n_parts):
            blocks = [(int(starts[c, p]), np.nonzero(pid[bounds[c]:bounds[c + 1]] == p)[0] + bounds[c], srcs) for c in range(n_chunks)]
            check_receiver(recvs[p], blocks)
    finally:
        ctx.lib.dfgpu_partition_plan_destroy(plan)


@pytest.mark.parametrize("fill", [0x00, 0xFF])
@pytest.mark.parametrize("n_parts", [3, 8, 20])
def test_two_sources_scatter_at_once_into_adjacent_blocks(gpu_ctx, n_parts, fill):
    """two plans ("two source ranks") on two contexts, issued back to back: source 1's block starts right after source 0's, so
    the two scatters write the shared boundary word of every receive bitmap at the same time"""
    ctx0, ctx1 = gpu_ctx, D.Context(0)
    try:
        rng = np.random.default_rng(n_parts + fill)
        srcs = [peer_sources(ctx, rng, 30_000 + 7 * r, 3 + 30 * r) for r, ctx in enumerate((ctx0, ctx1))]
        plans = [plan_create(ctx, s, n_parts, 1) for ctx, s in zip((ctx0, ctx1), srcs)]
        try:
            cnt = [pc[1][0] for pc in plans]
            lead = 13
            start0 = np.full(n_parts, lead, dtype=np.int64)
            start1 = start0 + cnt[0]
            recvs = [Receiver(ctx0, int(lead + cnt[0][p] + cnt[1][p] + 40), fill) for p in range(n_parts)]
            ctx0.sync(); ctx1.sync()
            scatter_nullable(ctx0, plans[0][0], 0, recvs, start0)
            scatter_nullable(ctx1, plans[1][0], 0, recvs, start1)
            ctx0.sync(); ctx1.sync()
            for p in range(n_parts):
                blocks = []
                for r, st in enumerate((start0, start1)):
                    s = srcs[r]
                    pid = part_ids(key_hash(s[0].values().view(np.uint64), s[0].validity()), n_parts)
                    blocks.append((int(st[p]), np.nonzero(pid == p)[0], s))
                check_receiver(recvs[p], blocks)
        finally:
            for (plan, _), ctx in zip(plans, (ctx0, ctx1)):
                ctx.lib.dfgpu_partition_plan_destroy(plan)
    finally:
        ctx1.close()


def test_old_scatter_entry_points_refuse_bit_packed_columns(gpu_ctx):
    ctx = gpu_ctx
    rng = np.random.default_rng(3)
    for srcs in ([Src(ctx, D.INT64, np.arange(5000, dtype=np.int64), rng.random(5000) > 0.5, 0)],
                 [Src(ctx, D.INT64, np.arange(5000, dtype=np.int64), None, 0), Src(ctx, D.BOOL, rng.random(5000) > 0.5, None, 0)]):
        counts = (C.c_int64 * 2)()
        plan = C.c_void_p()
        ctx.check(ctx.lib.dfgpu_partition_plan_create(ctx.h, D._cols([s.col for s in srcs]), len(srcs), D._i32arr([0]), 1, 2, counts, C.byref(plan)))
        try:
            bufs = [D.DeviceBuffer(ctx, 5000 * 8) for _ in range(2 * len(srcs))]
            bases = (C.c_void_p * len(bufs))(*[b.ptr for b in bufs])
            rows = (C.c_int64 * 2)(0, 0)
            for rc in (ctx.lib.dfgpu_partition_plan_scatter_peer(plan, bases, rows), ctx.lib.dfgpu_partition_plan_scatter_peer_chunk(plan, 0, bases, rows)):
                assert rc == ERR_INVALID
                assert b"dfgpu_partition_plan_scatter_peer_chunk_nullable" in ctx.lib.dfgpu_last_error(ctx.h)
            # the new call refuses a nullable column without receive bitmaps rather than drop its NULLs
            if srcs[0].valid is not None:
                assert ctx.lib.dfgpu_partition_plan_scatter_peer_chunk_nullable(plan, 0, bases, None, rows) == ERR_INVALID
        finally:
            ctx.lib.dfgpu_partition_plan_destroy(plan)


def test_exchange_one_rank_round_trips_nullable_boolean_and_decimal(gpu_ctx):
    """dfgpu_comm + dfgpu_exchange with one rank: every row comes back in source order; a column arrives with a bitmap exactly
    when its batch carried one, and a run after a bitmap-free run still gets every bit right (no zeroing needed)"""
    ctx = gpu_ctx
    comm = D.Comm(ctx, 1, 0, D.comm_unique_id())
    types = [D.INT64, D.decimal128(15, 2), D.BOOL, D.INT64]
    x = D.Exchange(comm, types, 70_000)
    try:
        rng = np.random.default_rng(5)
        for run, with_bitmaps in enumerate((True, False, True)):
            n = 60_000 - 1000 * run
            vm = (lambda: rng.random(n) > 0.25) if with_bitmaps else (lambda: None)
            srcs = [Src(ctx, D.INT64, rng.integers(-2**62, 2**62, n).astype(np.int64), vm(), 0),
                    Src(ctx, types[1], rng.integers(0, 2**40, (n, 2)).astype(np.uint64), vm(), 0),
                    Src(ctx, D.BOOL, rng.random(n) > 0.5, vm(), 0),
                    Src(ctx, D.INT64, np.arange(n, dtype=np.int64), None, 0)]   # never a bitmap
            out = x.run([s.col for s in srcs], [3])
            assert x.rows == n
            for i, (c, s) in enumerate(zip(out, srcs)):
                assert c.length == n and c.type == types[i]
                ev = s.validity()
                if ev is None:
                    assert not c.validity and c.null_count == 0, (run, i)
                    keep = np.ones(n, bool)
                else:
                    assert c.validity and c.null_count == -1, (run, i)
                    assert np.array_equal(D.unpack_bits(ctx.to_host(c.validity, (n + 7) // 8), n), ev), (run, i)
                    keep = ev
                if types[i] == D.BOOL:
                    got = D.unpack_bits(ctx.to_host(c.values, (n + 7) // 8), n)
                else:
                    w = D.WIDTH[types[i]]
                    raw = ctx.to_host(c.values, n * w)
                    got = raw.view(np.uint64).reshape(-1, 2) if w == 16 else raw.view(np.int64)
                assert np.array_equal(got[keep], s.values()[keep]), (run, i)
    finally:
        x.close()
        comm.close()


def test_two_gpu_exchange_of_bit_packed_columns():
    """PeerExchange, dfgpu_exchange and a Left PartitionedHashJoin with NULL keys across two GPUs (scripts/verify_partition_bits.py)"""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29543",
                        os.path.join(root, "scripts", "verify_partition_bits.py")],
                       cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "partition_bits ok=True" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
