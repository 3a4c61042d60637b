"""torchrun script (N GPUs; N = 1 exercises the same calls without peer memory): nullable, Boolean and Decimal128 columns through the peer-memory exchange.
  1. PeerExchange: every rank receives exactly the rows whose restated partition id is its rank, grouped by source rank, in
     source order, every validity bit exact (the last rank's Boolean column has no bitmap: senders disagree on nullability).
  2. dfgpu_comm + dfgpu_exchange: the same rows from the C ABI's own control plane.
  3. PartitionedHashJoin, Left join with NULL keys on both sides: the union of the rank results equals the oracle's global join.
Prints "partition_bits ok=True" on every rank when all checks pass; exits non-zero otherwise."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist

from datafusion_b200 import capi as D, exchange

rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
ts = torch.cuda.Stream(); torch.cuda.set_stream(ts)
ctx = D.Context(local, ts.cuda_stream)
SEED = np.uint64(0x9E3779B97F4A7C15)
DEC = D.decimal128(15, 2)
TYPES = [D.INT64, D.BOOL, DEC, D.INT64]


def mix64(x):
    x = x.copy()
    x ^= x >> np.uint64(30); x *= np.uint64(0xBF58476D1CE4E5B9)
    x ^= x >> np.uint64(27); x *= np.uint64(0x94D049BB133111EB)
    x ^= x >> np.uint64(31)
    return x


def part_of(key, valid, n_parts):
    with np.errstate(over="ignore"):
        h = np.where(valid, mix64(key.view(np.uint64) + SEED), np.uint64(0))
    hi, lo = h >> np.uint64(32), h & np.uint64(0xFFFFFFFF)
    return ((hi * np.uint64(n_parts) + ((lo * np.uint64(n_parts)) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


def shard(r):
    """rank r's input: (values, validity or None) per column of TYPES; column 0 is the key"""
    rng = np.random.default_rng(100 + r)
    n = 150_001 + 37 * r
    return [(rng.integers(0, 40_000, n).astype(np.int64), rng.random(n) > 0.1),
            (rng.random(n) > 0.5, (rng.random(n) > 0.3) if r < world - 1 else None),
            (rng.integers(0, 2**40, (n, 2)).astype(np.uint64), rng.random(n) > 0.2),
            (np.arange(n, dtype=np.int64) + r * 10**9, None)]


def to_device(cols, types):
    keep, out = [], []
    for (v, m), t in zip(cols, types):
        hc = D.HostColumn(v, m, t)
        dc = D.DeviceColumn.from_host(ctx, hc)
        keep.append(dc); out.append(dc.c())
    return out, keep


def read(c, n):
    if c.type == D.BOOL:
        v = D.unpack_bits(ctx.to_host(c.values, (c.offset + n + 7) // 8), n, c.offset)
    else:
        w = D.WIDTH[c.type]
        raw = ctx.to_host(c.values + c.offset * w, n * w)
        v = raw.view(np.uint64).reshape(-1, 2) if w == 16 else raw.view(np.int64)
    m = D.unpack_bits(ctx.to_host(c.validity, (c.offset + n + 7) // 8), n, c.offset) if c.validity else None
    return v, m


def expected():
    """rows this rank receives, in arrival order: source rank, then source order"""
    parts = []
    for r in range(world):
        s = shard(r)
        sel = part_of(s[0][0], s[0][1], world) == rank
        parts.append([(v[sel], np.ones(int(sel.sum()), bool) if m is None else m[sel]) for v, m in s])
    return [(np.concatenate([p[c][0] for p in parts]), np.concatenate([p[c][1] for p in parts])) for c in range(len(TYPES))]


def check(what, got_cols, rows):
    exp = expected()
    ok = rows == len(exp[0][0])
    for i, c in enumerate(got_cols):
        ev, em = exp[i]
        gv, gm = read(c, rows) if ok else (None, None)
        if not ok:
            break
        ok &= (gm is not None) == any(shard(r)[i][1] is not None for r in range(world))   # a bitmap whenever some sender had one
        gm = np.ones(rows, bool) if gm is None else gm
        ok &= bool(np.array_equal(gm, em)) and bool(np.array_equal(gv[em], ev[em]))
    print(f"rank {rank} {what}: rows={rows} ok={ok}", flush=True)
    return ok


ok = True
mine, keep = to_device(shard(rank), TYPES)
cap = 2 * len(shard(rank)[0][0])
# 1. PeerExchange, twice (buffer reuse, no zeroing between runs)
px = exchange.PeerExchange(ctx, dist, TYPES, cap)
for rep in range(2):
    b = px.exchange(mine, [0])
    torch.cuda.synchronize()
    ok &= check(f"PeerExchange rep {rep}", b.columns(), b.rows)
# 2. dfgpu_comm + dfgpu_exchange
uid = [D.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
comm = D.Comm(ctx, world, rank, uid[0])
x = D.Exchange(comm, TYPES, cap)
out = x.run(mine, [0])
ok &= check("dfgpu_exchange", out, x.rows)
comm.barrier()
x.close(); comm.close()
# 3. Left PartitionedHashJoin with NULL keys on both sides: build = (key, payload), probe = (key, payload)
from harness import assert_cols_equal, batches_to_cols  # noqa: E402
from oracle import oracle as O  # noqa: E402


def join_side(r, n, seed):
    rng = np.random.default_rng(seed + r)
    return [(rng.integers(0, 30_000, n).astype(np.int64), rng.random(n) > 0.05), (np.arange(n, dtype=np.int64) + r * 10**9, rng.random(n) > 0.1)]


nb, npr = 40_003, 200_011
bcols, bkeep = to_device(join_side(rank, nb, 7), [D.INT64, D.INT64])
pcols, pkeep = to_device(join_side(rank, npr, 70), [D.INT64, D.INT64])
pj = exchange.PartitionedHashJoin(local, dist, [D.INT64, D.INT64], [D.INT64, D.INT64], [0], [0], [0, 0, 1, 1], [0, 1, 0, 1], 2 * nb, 2 * npr,
                                  n_chunks=3, join_type=D.JOIN_LEFT)
rows, outs = pj.run(bcols, pcols)
pj.ctx.sync()
loc = batches_to_cols([o for o in outs], 4)
loc = [(v, np.ones(len(v), bool) if m is None else m) for v, m in loc]
allr = [None] * world
dist.all_gather_object(allr, loc)
if rank == 0:
    got = [(np.concatenate([a[c][0] for a in allr]), np.concatenate([a[c][1] for a in allr])) for c in range(4)]
    gb = [join_side(r, nb, 7) for r in range(world)]; gp = [join_side(r, npr, 70) for r in range(world)]
    cat = lambda sides, c: (np.concatenate([s[c][0] for s in sides]), np.concatenate([s[c][1] for s in sides]))
    exp = O.hash_join([cat(gb, 0), cat(gb, 1)], [cat(gp, 0), cat(gp, 1)], [0], [0], [0, 0, 1, 1], [0, 1, 0, 1], join_type=O.J_LEFT)
    exp = [(v, np.ones(len(v), bool) if m is None else np.asarray(m, bool)) for v, m in exp]
    # compare with NULL values zeroed (a NULL's value bits are unspecified)
    norm = lambda cols: [(np.where(m, v, 0), m) for v, m in cols]
    try:
        assert_cols_equal([(v, None) for v, _ in norm(got)] + [(m.astype(np.int64), None) for _, m in got],
                          [(v, None) for v, _ in norm(exp)] + [(m.astype(np.int64), None) for _, m in exp], ordered=False, what="left join")
        jok = True
    except AssertionError as e:
        print(e, flush=True)
        jok = False
    print(f"rank 0 PartitionedHashJoin Left: rows={len(got[0][0])} oracle={len(exp[0][0])} ok={jok}", flush=True)
    ok &= jok
for o in outs:
    o.release()
flag = torch.tensor([0 if ok else 1], device="cuda"); dist.all_reduce(flag)
ok = ok and int(flag.item()) == 0
print(f"rank {rank} partition_bits ok={ok}", flush=True)
dist.barrier(); dist.destroy_process_group()
sys.exit(0 if ok else 1)
