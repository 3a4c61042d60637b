"""LIKE / NOT LIKE on the GPU (libdfgpu_strings.so), device resident, with the TPC-H predicates that use it.

    1. o_comment NOT LIKE '%special%requests%' over SF x 1,500,000 orders: as Utf8 (one array per 4M-row block, int32 offsets),
       as LargeUtf8 (one array) and as Utf8View (one array, a data buffer per block).
    2. p_name LIKE '%green%' over SF x 200,000 parts (Utf8).
    3. p_type LIKE 'PROMO%' over SF x 200,000 parts as Utf8View (the view-prefix path) and through dictionary codes (dfgpu_like over
       the 150 distinct types, then dfgpu_like_codes over the INT32 codes).
    4. Q13 with the real predicate: the LIKE pass plus the fused Left plan (orders pipeline over a LEFT stage into the join-keyed sink),
       against the LIKE pass plus dfgpu_filter -> dfgpu_hashjoin(Left) -> dfgpu_agg; checked as scripts/pipe_left_join_timing.py checks.
    5. A CPU reference: Arrow C++'s pyarrow.compute.match_like over the same strings on all host threads (Arrow C++, not DataFusion).

Inputs: seeded TPC-H-like text.  o_comment is a word stream over a fixed vocabulary that includes `special` and `requests`, cut into
rows of 19..78 bytes (49 on average), so that '%special%requests%' matches about 1-2 % of rows.  One block of 4M distinct rows is
generated on the host and copied block after block to the device (outside the timed region): at SF 100 the device holds 7.4 GB of
text, 1.2 GB of int64 offsets, 0.6 GB of int32 offsets and 2.4 GB of views; the host holds one block (about 0.3 GB).
Kernel times are CUDA events around each call, the median of `steps` runs after a warm-up; Q13 times are a host clock around work that
ends in a device synchronise.  Every timed mask is checked at the timed size against pyarrow's evaluation of the same strings: the
match count and a fingerprint of the matching row numbers.  Algorithmic bytes per row are computed from the actual lengths: Utf8 reads
its offset, its string bytes and writes one byte; Utf8View reads its 16-byte view, the out-of-line bytes of the rows its prefix does
not settle, and writes one byte; codes read 4 bytes and write one.  Peak reference: 3.35 TB/s (H100 SXM data sheet).

usage: python scripts/like_timing.py [SF=100] [steps=5]"""
import ctypes as C
import json
import os
import statistics
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
import pipe_left_join_timing as T  # noqa: E402

PEAK_GBS = 3350.0
BLOCK = 4_000_000
MIX = np.uint64(0x9E3779B97F4A7C15)
WORDS = ["special", "requests", "furiously", "final", "ironic", "deposits", "packages", "accounts", "pinto", "beans", "blithely", "carefully",
         "regular", "express", "bold", "quickly", "slyly", "even", "pending", "unusual", "theodolites", "foxes", "ideas", "instructions",
         "asymptotes", "platelets", "dependencies", "excuses", "sleep", "haggle", "nag", "wake", "boost", "cajole", "detect", "integrate"]
WEIGHT_SPECIAL = 0.035     # share of `special` and of `requests` among the words
COLORS = ["almond", "antique", "aquamarine", "azure", "beige", "bisque", "black", "blanched", "blue", "blush", "brown", "burlywood", "chartreuse",
          "chiffon", "chocolate", "coral", "cornflower", "cornsilk", "cream", "cyan", "dark", "deep", "dim", "dodger", "drab", "firebrick",
          "floral", "forest", "frosted", "gainsboro", "ghost", "goldenrod", "green", "grey", "honeydew", "hot", "indian", "ivory", "khaki"]
TYPES = [f"{a} {b} {c}" for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
         for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]


# ---- host-side generation and the exact checks (tests/test_like_timing_checks.py runs them on tiny data) ----
def word_text(rng, n_rows, words, weights, lo, hi):
    """n_rows rows of lo..hi bytes cut from a stream of space-separated words -> (int64 offsets[n_rows + 1], uint8 data)"""
    lens = rng.integers(lo, hi + 1, n_rows)
    total = int(lens.sum())
    table = np.frombuffer(b"".join(w.encode() + b" " for w in words), np.uint8)
    wlen = np.array([len(w) + 1 for w in words])
    wstart = np.concatenate([[0], np.cumsum(wlen)[:-1]])
    n_words = total // int(wlen.min()) + 2
    idx = rng.choice(len(words), n_words, p=weights)
    ends = np.cumsum(wlen[idx])
    idx = idx[:int(np.searchsorted(ends, total)) + 1]
    ln = wlen[idx]
    starts = np.repeat(np.cumsum(ln) - ln, ln)
    pos = np.arange(int(ln.sum())) - starts + np.repeat(wstart[idx], ln)
    data = table[pos][:total]
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), np.ascontiguousarray(data)


def comment_weights():
    w = np.full(len(WORDS), (1 - 2 * WEIGHT_SPECIAL) / (len(WORDS) - 2))
    w[0] = w[1] = WEIGHT_SPECIAL
    return w


def utf8_array(offsets, data, large=False):
    t, w = (pa.large_string(), np.int64) if large else (pa.string(), np.int32)
    return pa.Array.from_buffers(t, len(offsets) - 1, [None, pa.py_buffer(offsets.astype(w)), pa.py_buffer(data)])


def fingerprint(rows: np.ndarray) -> int:
    """wrapping sum of row * MIX over the matching row numbers: independent of order, changed by any added, lost or moved row"""
    with np.errstate(over="ignore"):
        return int((np.asarray(rows, np.int64).view(np.uint64) * MIX).sum(dtype=np.uint64))


def mask_summary(mask: np.ndarray) -> dict:
    rows = np.flatnonzero(mask)
    return {"matches": int(len(rows)), "fingerprint": f"{fingerprint(rows):#x}"}


def check_mask(name, got: dict, exp: dict) -> dict:
    assert got == exp, f"{name}: GPU {got} != pyarrow {exp}"
    return got


def tiled_summary(block_mask: np.ndarray, n: int) -> dict:
    """the summary of block_mask repeated to n rows, without materialising it"""
    b = len(block_mask)
    rows = np.flatnonzero(block_mask).astype(np.int64)
    full, rest = divmod(n, b)
    count, fp = 0, np.uint64(0)
    with np.errstate(over="ignore"):
        base = np.uint64(fingerprint(rows))
        for t in range(full + (1 if rest else 0)):
            r = rows if t < full else rows[rows < rest]
            fp = fp + (base if t < full else np.uint64(fingerprint(r))) + np.uint64(t * b) * np.uint64(len(r)) * MIX
            count += len(r)
    return {"matches": int(count), "fingerprint": f"{int(fp):#x}"}


# ---- device side ----
def card():
    return T.card()


class Text:
    """one text column of n rows, the 4M-row host block repeated, resident as Utf8 blocks, LargeUtf8 and Utf8View"""

    def __init__(self, ctx, n, offsets, data):
        self.ctx, self.n, self.block_offsets, self.block_data = ctx, n, offsets, data
        b = len(offsets) - 1
        self.blocks = [(s, min(b, n - s)) for s in range(0, n, b)]
        nbytes = sum(int(offsets[r]) for _, r in self.blocks)
        self.data = ctx.malloc(max(nbytes, 16))
        self.large = ctx.malloc((n + 1) * 8)
        self.small = ctx.malloc(max(n + len(self.blocks), 1) * 4)
        self.views = ctx.malloc(max(n, 1) * 16)
        lib, h = ctx.lib, ctx.h
        h2d = lambda dst, arr: ctx.check(lib.dfgpu_memcpy_h2d(h, C.c_void_p(dst), arr.ctypes.data_as(C.c_void_p), arr.nbytes))  # noqa: E731
        lens = np.diff(offsets)
        self.string_bytes = 0
        at, self.block_ptrs, self.utf8_blocks = 0, [], []
        for k, (s, r) in enumerate(self.blocks):
            nb = int(offsets[r])
            h2d(self.data + at, data[:nb])
            h2d(self.large + s * 8, (offsets[:r + 1] + at).astype(np.int64) if k == len(self.blocks) - 1 else (offsets[:r] + at).astype(np.int64))
            so = offsets[:r + 1].astype(np.int32)
            h2d(self.small + (s + k) * 4, so)
            self.utf8_blocks.append((self.small + (s + k) * 4, self.data + at, r))
            v = np.zeros((r, 4), np.uint32)
            ln = lens[:r]
            v[:, 0] = ln
            inline = ln <= 12
            for j in range(12):                                           # inline bytes, and the 4-byte prefix of the others
                has = ln > j
                col = 1 + j // 4
                byte = np.where(has & (inline | (j < 4)), data[np.minimum(offsets[:r] + j, len(data) - 1)], 0).astype(np.uint32)
                if j >= 4:
                    byte = np.where(inline, byte, 0).astype(np.uint32)
                v[:, col] |= byte << np.uint32(8 * (j % 4))
            v[~inline, 2] = k
            v[~inline, 3] = offsets[:r][~inline].astype(np.uint32)
            h2d(self.views + s * 16, v)
            self.block_ptrs.append(self.data + at)
            self.string_bytes += nb
            at += nb
        self.total_bytes = at
        self.lens_block = lens
        ctx.sync()

    def col_large(self):
        c = D.StringColumn()
        c.layout, c.n_data_buffers, c.length, c.offset, c.null_count = D.STRING_LARGE_UTF8, 1, self.n, 0, 0
        c.offsets_or_views = self.large
        self._p1 = (C.c_void_p * 1)(self.data)
        c.data_buffers, c.validity = C.cast(self._p1, C.POINTER(C.c_void_p)), None
        return [c]

    def cols_utf8(self):
        out, self._pp = [], []
        for off, dat, r in self.utf8_blocks:
            c = D.StringColumn()
            c.layout, c.n_data_buffers, c.length, c.offset, c.null_count = D.STRING_UTF8, 1, r, 0, 0
            c.offsets_or_views = off
            p = (C.c_void_p * 1)(dat)
            self._pp.append(p)
            c.data_buffers, c.validity = C.cast(p, C.POINTER(C.c_void_p)), None
            out.append(c)
        return out

    def col_view(self):
        c = D.StringColumn()
        c.layout, c.n_data_buffers, c.length, c.offset, c.null_count = D.STRING_UTF8_VIEW, len(self.block_ptrs), self.n, 0, 0
        c.offsets_or_views = self.views
        self._pv = (C.c_void_p * len(self.block_ptrs))(*self.block_ptrs)
        c.data_buffers, c.validity = C.cast(self._pv, C.POINTER(C.c_void_p)), None
        return [c]

    def view_bytes(self, pattern: bytes) -> int:
        """views + the out-of-line bytes of rows whose 4-byte prefix does not settle an anchored-prefix mismatch + one output byte"""
        lead = pattern.split(b"%")[0].split(b"_")[0][:4]
        shortest = len(pattern.replace(b"%", b""))
        o, d, ln = self.block_offsets, self.block_data, self.lens_block
        read = 0
        for s, r in self.blocks:
            l = ln[:r]
            out = (l > 12) & (l >= shortest)
            if lead:
                pre = np.ones(r, bool)
                for j, ch in enumerate(lead):
                    pre &= d[np.minimum(o[:r] + j, len(d) - 1)] == ch
                out &= pre
            read += int(l[out].sum())
        return self.n * 17 + read

    def free(self):
        for p in (self.data, self.large, self.small, self.views):
            self.ctx.free(p)


def run_like(ctx, cols, pattern: bytes, negated, out, ov=None):
    lib = D.load_strings_library()
    st = ctx.lib.dfgpu_ctx_stream(ctx.h)
    at = 0
    for c in cols:
        D._strings_check(lib.dfgpu_like(st, C.byref(c), pattern, len(pattern), D.LIKE_NEGATED if negated else 0, C.c_void_p(out + at), None))
        at += c.length


def time_events(ctx, fn, steps):
    fn()
    ctx.sync()
    e0, e1 = ctx.event(), ctx.event()
    ts = []
    for _ in range(steps):
        ctx.record(e0)
        fn()
        ctx.record(e1)
        ctx.sync()
        ts.append(ctx.elapsed_ms(e0, e1))
    return statistics.median(ts), ts


def read_mask(ctx, ptr, n):
    return ctx.to_host(ptr, n).astype(bool)


def arrow_block_mask(offsets, data, pattern: str, negated: bool) -> np.ndarray:
    m = np.asarray(pc.match_like(utf8_array(offsets, data, large=True), pattern))
    return m != negated


def cpu_reference(offsets, data, n, pattern, negated, threads):
    """match_like over n rows (the block repeated) on `threads` host threads: Arrow C++"""
    b = len(offsets) - 1
    pieces = []
    step = max(1, b // threads)
    for s in range(0, b, step):
        e = min(b, s + step)
        pieces.append(utf8_array(offsets[s:e + 1] - offsets[s], data[offsets[s]:offsets[e]], large=True))
    reps = [(p, k) for k in range((n + b - 1) // b) for p in pieces]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda pk: pc.match_like(pk[0], pattern), reps))
    return (time.perf_counter() - t0) * 1e3


def kernel_entry(ms, nbytes):
    gbs = nbytes / (ms * 1e-3) / 1e9
    return {"ms": round(ms, 3), "bytes": int(nbytes), "GB_s": round(gbs, 1), "share_of_3.35TB_s": round(gbs / PEAK_GBS, 3)}


def q13_plans(ctx, sf, text, steps):
    """the LIKE pass + fused Left plan vs the LIKE pass + dfgpu_filter -> dfgpu_hashjoin(Left) -> dfgpu_agg"""
    customer, orders, keep = T.gen(ctx, sf)
    n = orders[0].length
    mask = ctx.malloc(n)
    cols = text.col_large()
    mcol = D.Column()
    mcol.type, mcol.flags, mcol.length, mcol.offset, mcol.null_count, mcol.values, mcol.validity = D.UINT8, 0, n, 0, 0, mask, None
    o3 = [orders[0], orders[1], mcol]
    types = [D.INT64, D.INT64, D.UINT8]
    pred = [T.C(2), (D.EXPR_LITERAL, 0, D.UINT8, 0, 1, 0.0), T.B(D.OP_EQ)]

    def fused():
        run_like(ctx, cols, b"%special%requests%", True, mask)
        look = T.customer_lookup(ctx, customer, 2)
        p = D.Pipeline(ctx, types, pred, [(D.STAGE_LEFT, 1, look)], name="q13_like_left")
        p.sink_aggregate([1], [(D.AGG_COUNT, [T.C(0)])], D.AGG_SINGLE_PARTITIONED)
        p.push_device(o3); p.finish()
        res = p.drain(host=False)
        p.close(); look.close()
        return res

    def unfused():
        run_like(ctx, cols, b"%special%requests%", True, mask)
        f = D.FilterHandle(ctx, types, pred, [0, 1], batch_size=0)
        f.push_device(o3); f.finish()
        fo = f.drain(host=False)
        f.close()
        j = D.HashJoinHandle(ctx, [D.INT64], [D.INT64, D.INT64], [0], [1], [0, 1], [0, 0], D.JOIN_LEFT, batch_size=1 << 28, ordered_output=False)
        j.push_build_device(customer); j.finish_build()
        agg = D.AggHandle(ctx, [D.INT64, D.INT64], [0], [(D.AGG_COUNT, 1, -1)], D.AGG_SINGLE_PARTITIONED, 1 << 30, customer[0].length)
        for b in fo:
            j.push_probe_device([b.column(0), b.column(1)])
            for jb in j.drain(host=False):
                agg.push_device([jb.column(0), jb.column(1)]); jb.release()
        j.finish_probe()
        for jb in j.drain(host=False):
            agg.push_device([jb.column(0), jb.column(1)]); jb.release()
        agg.finish()
        res = agg.drain(host=False)
        agg.close(); j.close()
        for b in fo:
            b.release()
        return res

    for fn in (fused, unfused):
        T.histogram_of(ctx, fn())
    tf, tu, summary = [], [], None
    for _ in range(steps):
        a, rf = T.timed(ctx, fused)
        rf = T.histogram_of(ctx, rf)
        b, ru = T.timed(ctx, unfused)
        ru = T.histogram_of(ctx, ru)
        summary = T.check_q13(rf, ru)
        tf.append(a); tu.append(b)
    ctx.free(mask)
    del keep
    return {"fused_ms": round(statistics.median(tf), 2), "unfused_ms": round(statistics.median(tu), 2), "fused_runs": [round(x, 2) for x in tf],
            "unfused_runs": [round(x, 2) for x in tu], "check": summary}


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100.0
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    threads = os.cpu_count() or 1
    ctx = D.Context(0)
    out = {"sf": sf, "card": card(), "steps": steps, "host_threads": threads}
    rng = np.random.default_rng(42)
    n_ord, n_part = int(1_500_000 * sf), int(200_000 * sf)

    # 1. o_comment NOT LIKE '%special%requests%'
    offs, data = word_text(rng, min(BLOCK, n_ord), WORDS, comment_weights(), 19, 78)
    text = Text(ctx, n_ord, offs, data)
    pat, neg = "%special%requests%", True
    exp = tiled_summary(arrow_block_mask(offs, data, pat, neg), n_ord)
    mask = ctx.malloc(n_ord)
    res = {"rows": n_ord, "string_bytes": text.string_bytes, "mean_len": round(text.string_bytes / n_ord, 2),
           "match_share_of_LIKE": round(1 - exp["matches"] / n_ord, 4)}
    for name, cols, nbytes in (("utf8_blocks", text.cols_utf8(), n_ord * 5 + text.string_bytes + 4 * len(text.blocks)),
                               ("large_utf8", text.col_large(), n_ord * 9 + 8 + text.string_bytes),
                               ("utf8_view", text.col_view(), text.view_bytes(pat.encode()))):
        ms, runs = time_events(ctx, lambda cols=cols: run_like(ctx, cols, pat.encode(), neg, mask), steps)
        res[name] = dict(kernel_entry(ms, nbytes), runs=[round(x, 3) for x in runs],
                         check=check_mask(name, tiled_summary_of_device(ctx, mask, n_ord), exp))
    res["floor_ms_at_3.35TB_s"] = round((n_ord * 5 + text.string_bytes) / PEAK_GBS / 1e6, 3)
    res["cpu_arrow_cpp_ms"] = round(cpu_reference(offs, data, n_ord, pat, neg, threads), 1)
    out["o_comment_not_like"] = res
    print(json.dumps({"o_comment_not_like": res}), flush=True)

    # 4. Q13 over the same o_comment text
    out["q13"] = q13_plans(ctx, sf, text, max(1, steps // 2))
    print(json.dumps({"q13": out["q13"]}), flush=True)
    ctx.free(mask)
    text.free()

    # 2. p_name LIKE '%green%'
    poffs, pdata = word_text(rng, min(BLOCK, n_part), COLORS, None, 20, 50)
    ptext = Text(ctx, n_part, poffs, pdata)
    pmask = ctx.malloc(n_part)
    exp = tiled_summary(arrow_block_mask(poffs, pdata, "%green%", False), n_part)
    ms, runs = time_events(ctx, lambda: run_like(ctx, ptext.col_large(), b"%green%", False, pmask), steps)
    out["p_name_like_green"] = dict(kernel_entry(ms, n_part * 9 + ptext.string_bytes), rows=n_part, runs=[round(x, 3) for x in runs],
                                    check=check_mask("p_name", tiled_summary_of_device(ctx, pmask, n_part), exp),
                                    cpu_arrow_cpp_ms=round(cpu_reference(poffs, pdata, n_part, "%green%", False, threads), 1))
    print(json.dumps({"p_name_like_green": out["p_name_like_green"]}), flush=True)
    ptext.free()

    # 3. p_type LIKE 'PROMO%': Utf8View (prefix path) and dictionary codes
    codes = rng.integers(0, len(TYPES), min(BLOCK, n_part)).astype(np.int32)
    tb = [t.encode() for t in TYPES]
    toffs = np.concatenate([[0], np.cumsum([len(tb[c]) for c in codes])]).astype(np.int64)
    tdata = np.frombuffer(b"".join(tb[c] for c in codes), np.uint8).copy()
    ttext = Text(ctx, n_part, toffs, tdata)
    exp = tiled_summary(arrow_block_mask(toffs, tdata, "PROMO%", False), n_part)
    ms, runs = time_events(ctx, lambda: run_like(ctx, ttext.col_view(), b"PROMO%", False, pmask), steps)
    pv = dict(kernel_entry(ms, ttext.view_bytes(b"PROMO%")), runs=[round(x, 3) for x in runs],
              check=check_mask("p_type view", tiled_summary_of_device(ctx, pmask, n_part), exp))
    ttext.free()
    dvals = pa.array(TYPES)
    dcodes = ctx.malloc(n_part * 4)
    full_codes = np.resize(codes, n_part)
    ctx.check(ctx.lib.dfgpu_memcpy_h2d(ctx.h, C.c_void_p(dcodes), full_codes.ctypes.data_as(C.c_void_p), full_codes.nbytes))
    ccol = D.Column()
    ccol.type, ccol.flags, ccol.length, ccol.offset, ccol.null_count, ccol.values, ccol.validity = D.INT32, 0, n_part, 0, 0, dcodes, None
    lib = D.load_strings_library()
    st = ctx.lib.dfgpu_ctx_stream(ctx.h)

    def via_codes():
        cm = D.like(ctx, dvals, "PROMO%")
        D._strings_check(lib.dfgpu_like_codes(st, C.byref(ccol), C.c_void_p(cm.values.ptr), len(TYPES), C.c_void_p(pmask), None))
        return cm
    dvals = D.DeviceStrings(ctx, dvals)
    ms_c, runs_c = time_events(ctx, via_codes, steps)
    pc_ = dict(kernel_entry(ms_c, n_part * 5), runs=[round(x, 3) for x in runs_c],
               check=check_mask("p_type codes", tiled_summary_of_device(ctx, pmask, n_part), exp))
    out["p_type_like_promo"] = {"rows": n_part, "utf8_view": pv, "dictionary_codes": pc_,
                                "cpu_arrow_cpp_ms": round(cpu_reference(toffs, tdata, n_part, "PROMO%", False, threads), 1)}
    print(json.dumps({"p_type_like_promo": out["p_type_like_promo"]}), flush=True)
    ctx.free(dcodes)
    ctx.free(pmask)
    out["card_after"] = card()
    out["checks"] = "every mask: match count and row-number fingerprint equal to pyarrow.compute.match_like; Q13: c_count histogram and per-customer fingerprint equal fused vs unfused"
    print(json.dumps(out, indent=1))


def tiled_summary_of_device(ctx, ptr, n):
    return mask_summary(read_mask(ctx, ptr, n))


if __name__ == "__main__":
    main()
