"""The string gather on the GPU (dfgpu_string_take_*, libdfgpu_strings.so), device resident, at the shapes late materialisation gives it.

    a. build-side gather: c_name, c_address and c_comment of SF x 150,000 customers gathered for SF x 1,500,000 orders rows in orders
       order (UINT32 ids, uniform over the customers: random access into a source larger than L2), as LargeUtf8.
    b. streamed gather: l_comment of SF x 6,000,000 lineitem rows through an l_shipdate filter (Q3's cut, about 54 % kept): INT64 ids
       packed as batch << 32 | row over one source per 4M-row batch, nondecreasing, as LargeUtf8.
    c. the Utf8View versions of both (b over one view array of every batch's buffers).
    d. at SF 0.1: the twin plan customer[c_custkey, c_name, c_address, c_comment] JOIN orders[o_custkey, o_orderkey] (Inner) through
       plan_string_payloads against the same plan through DictionaryEncodeExec / DictionaryDecodeExec, a host clock around collect()
       (the dictionary route rebuilds every distinct value on the host for each output batch, so with a value per customer it does not
       finish in minutes at SF 1).
    e. a CPU reference: Arrow C++'s pyarrow.compute.take over the same strings on all host threads, over the first 10 % of each id column
       (Arrow C++, not DataFusion).

LargeUtf8 stands for the Utf8 family at these sizes: a Utf8 output beyond 2^31 - 1 bytes is refused, as arrow's take refuses it.
Inputs: seeded TPC-H-like text from scripts/like_timing.py's word generator, one 4M-row block per column repeated on the device.  Times
are CUDA events, the median of `steps` runs after a warm-up: `ms` spans both phases and the 24-byte read of the total between them (what
a caller pays), `copy_ms` the byte copy of phase 2 alone.  Every output is checked at the timed size: each output row's length against
the source row its id names, the byte sum of all output rows against theirs, and two windows of 1M rows (the first, the middle) equal to
pyarrow.compute.take (a Utf8View output: every view against the source view, its buffer index rebased).
The floor is computed, not measured: the ids read (4 B a row UINT32, 8 B INT64), the source offsets (a 32-byte sector a row for random
ids; the sectors the rows span for nondecreasing ones), the string bytes read rounded to the 32-byte sectors they span (random ids: per
row; nondecreasing: each sector once), and the offsets (8 B a row), string bytes and validity written.  Utf8View: the ids, one sector of
views a row (random) or the views spanned (nondecreasing), 16 B written a row and the validity.  Floor time = floor bytes / 3.35 TB/s
(H100 SXM data sheet).  The card's name, power limit and SM clocks are read in the same run.

usage: python scripts/string_take_timing.py [SF=100] [steps=5]"""
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from datafusion_b200 import capi as D  # noqa: E402
import like_timing as L  # noqa: E402

PEAK_GBS = 3350.0
BLOCK = L.BLOCK
SECTOR = 32
CHECK_CHUNK = 8_000_000
EXACT_ROWS = 1_000_000


# ---- host-side generation, floors and checks (tests/test_string_take_timing_checks.py runs them on tiny data) ----
def name_text(n_rows):
    """c_name: Customer#000000001 ... (18 bytes) -> (int64 offsets, uint8 data)"""
    data = np.frombuffer("".join(f"Customer#{i:09d}" for i in range(1, n_rows + 1)).encode(), np.uint8)
    return np.arange(n_rows + 1, dtype=np.int64) * 18, data.copy()


def row_sums(offsets, data):
    """per row: the sum of its bytes (uint64; 0 for an empty row)"""
    lens = np.diff(offsets)
    if len(lens) == 0:
        return np.zeros(0, np.uint64)
    cum = np.concatenate([[0], np.cumsum(data[int(offsets[0]):int(offsets[-1])], dtype=np.uint64)])
    return cum[offsets[1:] - offsets[0]] - cum[offsets[:-1] - offsets[0]]


def sector_bytes(starts, lens, distinct=False):
    """bytes of the 32-byte sectors the ranges [start, start + len) span: per range, or each sector once (ranges in nondecreasing
    order, distinct=True)"""
    starts = np.asarray(starts, np.int64)
    lens = np.asarray(lens, np.int64)
    keep = lens > 0
    s, e = starts[keep] // SECTOR, (starts[keep] + lens[keep] - 1) // SECTOR
    span = e - s + 1
    if distinct and len(s) > 1:
        last = np.maximum.accumulate(e)
        span[1:] -= np.clip(last[:-1] - s[1:] + 1, 0, span[1:])
    return int(span.sum()) * SECTOR


def floor_bytes(layout, n_ids, id_bytes, offsets_read, strings_read, out_string_bytes):
    validity = (n_ids + 7) // 8
    if layout == "utf8_view":
        return n_ids * id_bytes + offsets_read + 16 * n_ids + validity
    return n_ids * id_bytes + offsets_read + strings_read + 8 * (n_ids + 1) + out_string_bytes + validity


def check_sum(name, got_sum, exp_sum):
    assert got_sum == exp_sum, f"{name}: the output's byte sum differs from the rows the ids name"


# ---- device side ----
class Out:
    """the caller buffers of one gather of n ids, allocated once outside the timed region"""

    def __init__(self, ctx, n, view, out_bytes=0):
        lib = D.load_strings_library()
        self.ctx, self.n, self.view = ctx, n, view
        if view:
            self.views = ctx.malloc(max(n, 1) * 16)
            self.validity = ctx.malloc((n + 31) // 32 * 4 + 8)
            self.status = ctx.malloc(16)
            self.bufs = [self.views, self.validity, self.status]
        else:
            self.offsets = ctx.malloc((n + 3) * 8)
            self.scratch = ctx.malloc(lib.dfgpu_string_take_scratch_bytes(n))
            self.validity = ctx.malloc((n + 7) // 8 + 8)
            self.data = ctx.malloc(max(out_bytes, 16))
            self.bufs = [self.offsets, self.scratch, self.validity, self.data]

    def free(self):
        for b in self.bufs:
            self.ctx.free(b)


def gather(ctx, out, cols, ids_col, copy_events=None):
    lib = D.load_strings_library()
    st = ctx.lib.dfgpu_ctx_stream(ctx.h)
    arr = (D.StringColumn * len(cols))(*cols)
    n = out.n
    if out.view:
        D._strings_check(lib.dfgpu_string_take_views(st, arr, len(cols), C.byref(ids_col), C.c_void_p(out.views), C.c_void_p(out.validity),
                                                     C.c_void_p(out.status)))
        return
    D._strings_check(lib.dfgpu_string_take_offsets(st, arr, len(cols), C.byref(ids_col), C.c_void_p(out.scratch), C.c_void_p(out.offsets),
                                                   C.c_void_p(out.validity)))
    total, bad, _ = (int(x) for x in ctx.to_host(out.offsets + n * 8, 24).view(np.int64))
    assert bad == 0, "ids outside their source"
    if copy_events:
        ctx.record(copy_events[0])
    D._strings_check(lib.dfgpu_string_take_data(st, cols[0].layout, n, total, C.c_void_p(out.scratch), C.c_void_p(out.offsets),
                                                C.c_void_p(out.offsets), C.c_void_p(out.data)))
    if copy_events:
        ctx.record(copy_events[1])


def time_gather(ctx, out, cols, ids_col, steps):
    ec = (ctx.event(), ctx.event())
    copies = []

    def fn():
        gather(ctx, out, cols, ids_col, None if out.view else ec)
    ms, runs = L.time_events(ctx, fn, steps)
    if not out.view:
        for _ in range(steps):
            fn()
            ctx.sync()
            copies.append(ctx.elapsed_ms(*ec))
    return ms, runs, (float(np.median(copies)) if copies else None)


def ids_column(ptr, n, packed):
    c = D.Column()
    c.type, c.flags, c.length, c.offset, c.null_count, c.values, c.validity = (D.INT64 if packed else D.UINT32), 0, n, 0, 0, ptr, None
    return c


def upload(ctx, arr):
    p = ctx.malloc(max(arr.nbytes, 16))
    ctx.check(ctx.lib.dfgpu_memcpy_h2d(ctx.h, C.c_void_p(p), arr.ctypes.data_as(C.c_void_p), arr.nbytes))
    return p


def check_large(ctx, name, out, exp_rows, block_offsets, block_sums, exact):
    """exp_rows: the block row of every output row, in order; exact(lo, hi): pyarrow.compute.take of output rows [lo, hi)"""
    n = out.n
    got_sum = exp_sum = 0
    lens = np.diff(block_offsets)
    for s in range(0, n, CHECK_CHUNK):
        m = min(CHECK_CHUNK, n - s)
        offs = ctx.to_host(out.offsets + s * 8, (m + 1) * 8).view(np.int64)
        got_sum += int(ctx.to_host(out.data + int(offs[0]), int(offs[-1] - offs[0])).sum(dtype=np.uint64))
        rows = exp_rows[s:s + m]
        exp_sum += int(block_sums[rows].sum(dtype=np.uint64))
        assert np.array_equal(np.diff(offs), lens[rows]), f"{name}: output row lengths differ from the rows the ids name"
    check_sum(name, got_sum, exp_sum)
    for lo in sorted({0, max(0, n // 2 - EXACT_ROWS // 2)}):
        hi = min(n, lo + EXACT_ROWS)
        offs = ctx.to_host(out.offsets + lo * 8, (hi - lo + 1) * 8).view(np.int64)
        got = L.utf8_array(offs - offs[0], ctx.to_host(out.data + int(offs[0]), int(offs[-1] - offs[0])), large=True)
        assert got.equals(exact(lo, hi)), f"{name}: rows {lo}..{hi} differ from pyarrow.compute.take"
    return "every row's length and the byte sum of all rows, and two windows of 1M rows equal to pyarrow.compute.take"


def check_views(ctx, name, out, exp_rows, block_views, block_of_row):
    """every output view against the source view of its row, its buffer index rebased to its block"""
    n = out.n
    for s in range(0, n, CHECK_CHUNK):
        m = min(CHECK_CHUNK, n - s)
        got = ctx.to_host(out.views + s * 16, m * 16).view(np.uint32).reshape(m, 4)
        exp = block_views[exp_rows[s:s + m]].copy()
        out_of_line = exp[:, 0] > 12
        exp[out_of_line, 2] = block_of_row[s:s + m][out_of_line]
        assert np.array_equal(got, exp), f"{name}: output views differ from the rows the ids name"
    return "every view equal to its source row's view with the buffer index rebased"


def block_views(offsets, data):
    """the Utf8View views of one block (buffer index 0), as scripts/like_timing.py's Text lays them out"""
    r = len(offsets) - 1
    v = np.zeros((r, 4), np.uint32)
    ln = np.diff(offsets)
    v[:, 0] = ln
    inline = ln <= 12
    for j in range(12):
        has = ln > j
        byte = np.where(has & (inline | (j < 4)), data[np.minimum(offsets[:-1] + j, len(data) - 1)], 0).astype(np.uint32)
        if j >= 4:
            byte = np.where(inline, byte, 0).astype(np.uint32)
        v[:, 1 + j // 4] |= byte << np.uint32(8 * (j % 4))
    v[~inline, 3] = offsets[:-1][~inline].astype(np.uint32)
    return v


def entry(ms, runs, copy_ms, nbytes, check):
    gbs = nbytes / (ms * 1e-3) / 1e9
    out = {"ms": round(ms, 3), "runs": [round(x, 3) for x in runs], "floor_bytes": int(nbytes), "floor_ms_at_3.35TB_s": round(nbytes / PEAK_GBS / 1e6, 3),
           "GB_s_of_floor_bytes": round(gbs, 1), "share_of_3.35TB_s": round(gbs / PEAK_GBS, 3), "check": check}
    if copy_ms is not None:
        out["copy_ms"] = round(copy_ms, 3)
    return out


def host_take(src, ids, threads):
    """Arrow C++'s take of ids from src on `threads` host threads -> (ms, result of the first piece)"""
    pieces = np.array_split(ids, threads)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        res = list(ex.map(lambda p: pc.take(src, pa.array(p)), pieces))
    return (time.perf_counter() - t0) * 1e3, res


def build_side(ctx, sf, steps, threads, rng):
    n_cust, n_ord = int(150_000 * sf), int(1_500_000 * sf)
    ids = rng.integers(0, n_cust, n_ord).astype(np.uint32)
    dids = upload(ctx, ids)
    idc = ids_column(dids, n_ord, False)
    rows_a = (ids % min(BLOCK, n_cust)).astype(np.int64)
    res = {"customers": n_cust, "orders": n_ord}
    cols = {"c_name": name_text(min(BLOCK, n_cust)),
            "c_address": L.word_text(rng, min(BLOCK, n_cust), L.WORDS, L.comment_weights(), 10, 40),
            "c_comment": L.word_text(rng, min(BLOCK, n_cust), L.WORDS, L.comment_weights(), 29, 116)}
    for name, (offs, data) in cols.items():
        text = L.Text(ctx, n_cust, offs, data)
        lens = np.diff(offs)
        out_bytes = int(lens[rows_a].sum())
        src_start = offs[:-1][rows_a] + (ids // len(lens)).astype(np.int64) * int(offs[-1])   # where each id's bytes sit in the repeated data
        strings_read = sector_bytes(src_start, lens[rows_a])
        r = {"source_bytes": text.string_bytes, "output_bytes": out_bytes}
        out = Out(ctx, n_ord, False, out_bytes)
        ms, runs, copy_ms = time_gather(ctx, out, text.col_large(), idc, steps)
        src_host = pa.concat_arrays([L.utf8_array(offs, data, large=True)] * ((n_cust + len(lens) - 1) // len(lens))).slice(0, n_cust)
        check = check_large(ctx, name, out, rows_a, offs, row_sums(offs, data), lambda lo, hi: pc.take(src_host, pa.array(ids[lo:hi])))
        r["large_utf8"] = entry(ms, runs, copy_ms, floor_bytes("large_utf8", n_ord, 4, SECTOR * n_ord, strings_read, out_bytes), check)
        out.free()
        out = Out(ctx, n_ord, True)
        ms, runs, _ = time_gather(ctx, out, text.col_view(), idc, steps)
        check = check_views(ctx, name, out, rows_a, block_views(offs, data), (ids // len(lens)).astype(np.uint32))
        r["utf8_view"] = entry(ms, runs, None, floor_bytes("utf8_view", n_ord, 4, SECTOR * n_ord, 0, 0), check)
        out.free()
        k = n_ord // 10
        host_ms, _ = host_take(src_host, ids[:k], threads)
        r["cpu_arrow_cpp_take_ms_first_10pct"] = {"ids": k, "ms": round(host_ms, 1)}
        text.free()
        res[name] = r
        print(json.dumps({name: r}), flush=True)
    ctx.free(dids)
    return res


def streamed(ctx, sf, steps, threads, rng):
    n = int(6_000_000 * sf)
    offs, data = L.word_text(rng, min(BLOCK, n), L.WORDS, L.comment_weights(), 10, 43)
    text = L.Text(ctx, n, offs, data)
    cut = 9204                                                                  # 1995-03-15 as Date32
    ship = rng.integers(8036, 10562, min(BLOCK, n))
    keep_rows = np.flatnonzero(ship > cut).astype(np.int64)
    lens = np.diff(offs)
    batches = [(k, s, r) for k, (s, r) in enumerate(text.blocks)]
    packed = np.concatenate([(np.int64(k) << 32) | keep_rows[keep_rows < r] for k, _, r in batches])
    rows_b = (packed & 0xFFFFFFFF).astype(np.int64)
    block_of = (packed >> 32).astype(np.int64)
    m = len(packed)
    out_bytes = int(lens[rows_b].sum())
    glob_start = block_of * int(offs[-1]) + offs[:-1][rows_b]
    strings_read = sector_bytes(glob_start, lens[rows_b], distinct=True)
    offsets_read = sector_bytes((block_of * BLOCK + rows_b) * 8, np.full(m, 16), distinct=True)
    res = {"lineitem": n, "kept": m, "source_bytes": text.string_bytes, "output_bytes": out_bytes}
    dids = upload(ctx, packed)
    idc = ids_column(dids, m, True)
    srcs, keep_alive = [], []
    for k, s, r in batches:                                                     # one LargeUtf8 source per batch: a slice of the column
        c = D.StringColumn()
        c.layout, c.n_data_buffers, c.length, c.offset, c.null_count = D.STRING_LARGE_UTF8, 1, r, s, 0
        c.offsets_or_views = text.large
        keep_alive.append((C.c_void_p * 1)(text.data))
        c.data_buffers, c.validity = C.cast(keep_alive[-1], C.POINTER(C.c_void_p)), None
        srcs.append(c)
    out = Out(ctx, m, False, out_bytes)
    ms, runs, copy_ms = time_gather(ctx, out, srcs, idc, steps)
    block = L.utf8_array(offs, data, large=True)
    check = check_large(ctx, "l_comment", out, rows_b, offs, row_sums(offs, data), lambda lo, hi: pc.take(block, pa.array(rows_b[lo:hi])))
    res["large_utf8"] = entry(ms, runs, copy_ms, floor_bytes("large_utf8", m, 8, offsets_read, strings_read, out_bytes), check)
    out.free()
    ctx.free(dids)
    glob = (block_of * BLOCK + rows_b).astype(np.int64)                        # Utf8View: one array of every batch's buffers, source 0
    dids = upload(ctx, glob)
    idc = ids_column(dids, m, True)
    out = Out(ctx, m, True)
    ms, runs, _ = time_gather(ctx, out, text.col_view(), idc, steps)
    check = check_views(ctx, "l_comment view", out, rows_b, block_views(offs, data), block_of.astype(np.uint32))
    res["utf8_view"] = entry(ms, runs, None, floor_bytes("utf8_view", m, 8, sector_bytes(glob * 16, np.full(m, 16), distinct=True), 0, 0), check)
    out.free()
    ctx.free(dids)
    k = m // 10
    host_ms, _ = host_take(L.utf8_array(offs, data, large=True), rows_b[:k], threads)
    res["cpu_arrow_cpp_take_ms_first_10pct"] = {"ids": k, "ms": round(host_ms, 1)}
    text.free()
    return res


def twin_plan(ctx, sf, rng):
    from datafusion_b200.exec import (DictionaryDecodeExec, DictionaryEncodeExec, GpuHashJoinExec, MemoryExec, TaskContext, collect,
                                      plan_string_dictionary, plan_string_payloads)
    nc, no = int(150_000 * sf), int(1_500_000 * sf)
    addr = L.word_text(rng, nc, L.WORDS, L.comment_weights(), 10, 40)
    com = L.word_text(rng, nc, L.WORDS, L.comment_weights(), 29, 116)
    cust = pa.table({"c_custkey": pa.array(np.arange(1, nc + 1), pa.int64()), "c_name": L.utf8_array(*name_text(nc)),
                     "c_address": L.utf8_array(*addr), "c_comment": L.utf8_array(*com)})
    orders = pa.table({"o_custkey": pa.array(rng.integers(1, nc + 1, no), pa.int64()), "o_orderkey": pa.array(np.arange(no) * 4, pa.int64())})
    mem = lambda t: MemoryExec(t.to_batches(max_chunksize=8192), t.schema)  # noqa: E731
    make = lambda c, o: GpuHashJoinExec(c, o, [("c_custkey", "o_custkey")], "Inner")  # noqa: E731
    tc = TaskContext(ctx=ctx)
    d = plan_string_dictionary()
    plans = {"plan_string_payloads": plan_string_payloads(make(mem(cust), mem(orders))),
             "dictionary_route": DictionaryDecodeExec(make(DictionaryEncodeExec(mem(cust), d), mem(orders)), ["c_name", "c_address", "c_comment"], d)}
    res, tabs = {"customers": nc, "orders": no}, {}
    for name, plan in plans.items():
        t0 = time.perf_counter()
        tabs[name] = pa.Table.from_batches(collect(plan, tc), plan.schema)
        res[name + "_s"] = round(time.perf_counter() - t0, 3)
    a, b = tabs["plan_string_payloads"], tabs["dictionary_route"]
    assert a.num_rows == b.num_rows == no and all(a[c].equals(b[c]) for c in a.schema.names), "the two routes differ"
    res["check"] = "both routes give the same rows in the same order"
    return res


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100.0
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    threads = os.cpu_count() or 1
    ctx = D.Context(0)
    out = {"sf": sf, "card": L.card(), "steps": steps, "host_threads": threads}
    rng = np.random.default_rng(42)
    out["a_build_side"] = build_side(ctx, sf, steps, threads, rng)
    out["b_streamed"] = streamed(ctx, sf, steps, threads, rng)
    print(json.dumps({"b_streamed": out["b_streamed"]}), flush=True)
    out["d_twin_plan"] = twin_plan(ctx, min(sf, 0.1), rng)
    print(json.dumps({"d_twin_plan": out["d_twin_plan"]}), flush=True)
    out["card_after"] = L.card()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
