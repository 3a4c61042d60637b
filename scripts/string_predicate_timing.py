"""String comparisons and IN lists on the GPU (libdfgpu_strings.so), device resident, with the TPC-H predicates that use them.

    1. l_shipmode IN ('MAIL', 'SHIP') over SF x 6,000,000 lineitem rows: as Utf8 (one array per 4M-row block, int32 offsets), as
       LargeUtf8 (one array), as Utf8View (one array, every string inline) and through dictionary codes (dfgpu_string_in_list over the 7
       distinct modes, then dfgpu_like_codes over the INT32 codes).
    2. c_mktsegment = 'BUILDING' over SF x 150,000 customers (LargeUtf8 and Utf8View).
    3. p_container IN ('SM CASE', 'SM BOX', 'SM PACK', 'SM PKG') and p_brand = 'Brand#12' over SF x 200,000 parts (LargeUtf8, Utf8View).
    4. An ordering comparison: p_type < 'MEDIUM' over SF x 200,000 parts (LargeUtf8, and Utf8View with out-of-line strings).
    5. A CPU reference: Arrow C++'s pyarrow.compute (is_in, equal, less) over the same strings on all host threads (Arrow C++, not
       DataFusion).

Inputs: seeded TPC-H-like text, each row one of the column's TPC-H values.  One block of up to 4M rows is generated on the host and
copied block after block to the device outside the timed region (scripts/like_timing.py's Text), so every row has its own bytes in HBM.
Kernel times are CUDA events around each call, the median of `steps` runs after a warm-up.  Every timed mask is checked at the timed
size against pyarrow's evaluation of the same strings: the match count and a fingerprint of the matching row numbers.  The DRAM floor
of each call is computed, not measured: Utf8 reads its offsets (4 bytes a row, 8 for LargeUtf8) and its string bytes and writes one byte
a row; Utf8View reads its 16-byte views and writes one byte (out-of-line bytes not counted); codes read 4 bytes and write one.  Floor
time = floor bytes / 3.35 TB/s (H100 SXM data sheet).  The card's name, power limit and SM clocks are read in the same run.

usage: python scripts/string_predicate_timing.py [SF=100] [steps=5]"""
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
import like_timing as L  # noqa: E402

PEAK_GBS = 3350.0
BLOCK = 4_000_000
MODES = ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"]
SEGMENTS = ["AUTOMOBILE", "BUILDING", "FURNITURE", "MACHINERY", "HOUSEHOLD"]
CONTAINERS = [f"{a} {b}" for a in ("SM", "LG", "MED", "JUMBO", "WRAP") for b in ("CASE", "BOX", "BAG", "JAR", "PKG", "PACK", "CAN", "DRUM")]
BRANDS = [f"Brand#{a}{b}" for a in range(1, 6) for b in range(1, 6)]


# ---- host-side generation and the exact checks (tests/test_string_predicate_timing_checks.py runs them on tiny data) ----
def value_text(rng, n_rows, values):
    """n_rows rows, each one of `values` drawn uniformly -> (codes int32[n_rows], int64 offsets[n_rows + 1], uint8 data)"""
    enc = [v.encode() for v in values]
    codes = rng.integers(0, len(values), n_rows).astype(np.int32)
    vlen = np.array([len(b) for b in enc], np.int64)
    vstart = np.concatenate([[0], np.cumsum(vlen)[:-1]])
    table = np.frombuffer(b"".join(enc), np.uint8)
    ln = vlen[codes]
    offsets = np.concatenate([[0], np.cumsum(ln)]).astype(np.int64)
    pos = np.arange(int(offsets[-1])) - np.repeat(offsets[:-1], ln) + np.repeat(vstart[codes], ln)
    return codes, offsets, np.ascontiguousarray(table[pos])


def arrow_mask(arr, pred):
    """pyarrow's evaluation of pred = ("in", values) or (op, literal) over arr, NULL as False"""
    kind, arg = pred
    if kind == "in":
        m = pc.is_in(arr, value_set=pa.array(arg))
    else:
        m = {"=": pc.equal, "<>": pc.not_equal, "<": pc.less, "<=": pc.less_equal, ">": pc.greater, ">=": pc.greater_equal}[kind](arr, arg)
    return np.asarray(m.fill_null(False))


def chunked_summary(chunks) -> dict:
    """the mask summary (match count, row fingerprint) of a mask given as (first row, bool chunk) pieces, equal to L.mask_summary of the
    whole mask"""
    count, fp = 0, np.uint64(0)
    with np.errstate(over="ignore"):
        for start, m in chunks:
            rows = np.flatnonzero(m).astype(np.int64) + start
            count += len(rows)
            fp = fp + np.uint64(L.fingerprint(rows))
    return {"matches": int(count), "fingerprint": f"{int(fp):#x}"}


def floor_bytes(layout, n, string_bytes, n_blocks=1):
    return {"utf8_blocks": 4 * (n + n_blocks) + string_bytes + n, "large_utf8": 8 * (n + 1) + string_bytes + n, "utf8_view": 17 * n,
            "dictionary_codes": 5 * n}[layout]


# ---- device side ----
def device_summary(ctx, ptr, n):
    return chunked_summary((s, ctx.to_host(ptr + s, min(BLOCK, n - s)).astype(bool)) for s in range(0, n, BLOCK))


def run_pred(ctx, cols, pred, out):
    lib = D.load_strings_library()
    st = ctx.lib.dfgpu_ctx_stream(ctx.h)
    kind, arg = pred
    if kind == "in":
        vals = [v.encode() for v in arg]
        ptrs = (C.c_char_p * len(vals))(*vals)
        lens = (C.c_int64 * len(vals))(*[len(v) for v in vals])
    at = 0
    for c in cols:
        if kind == "in":
            rc = lib.dfgpu_string_in_list(st, C.byref(c), ptrs, lens, len(vals), 0, 0, C.c_void_p(out + at), None)
        else:
            lit = arg.encode()
            rc = lib.dfgpu_string_compare(st, C.byref(c), D.STRING_CMP_OPS[kind], lit, len(lit), C.c_void_p(out + at), None)
        D._strings_check(rc)
        at += c.length


def cpu_reference(offsets, data, n, pred, threads):
    """pred over n rows (the block repeated) on `threads` host threads: Arrow C++"""
    b = len(offsets) - 1
    step = max(1, b // threads)
    pieces = [L.utf8_array(offsets[s:min(b, s + step) + 1] - offsets[s], data[offsets[s]:offsets[min(b, s + step)]], large=True)
              for s in range(0, b, step)]
    reps = [p for _ in range((n + b - 1) // b) for p in pieces]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda p: arrow_mask(p, pred), reps))
    return (time.perf_counter() - t0) * 1e3


def entry(ms, runs, nbytes, check):
    gbs = nbytes / (ms * 1e-3) / 1e9
    return {"ms": round(ms, 3), "runs": [round(x, 3) for x in runs], "floor_bytes": int(nbytes), "floor_ms_at_3.35TB_s": round(nbytes / PEAK_GBS / 1e6, 3),
            "GB_s_of_floor_bytes": round(gbs, 1), "share_of_3.35TB_s": round(gbs / PEAK_GBS, 3), "check": check}


def measure(ctx, name, n, values, preds, layouts, steps, threads, rng, codes_too=False):
    codes, offs, data = value_text(rng, min(BLOCK, n), values)
    text = L.Text(ctx, n, offs, data)
    mask = ctx.malloc(n)
    res = {"rows": n, "string_bytes": text.string_bytes}
    block = L.utf8_array(offs, data, large=True)
    for pname, pred in preds:
        exp = L.tiled_summary(arrow_mask(block, pred), n)
        r = {"match_share": round(exp["matches"] / n, 4)}
        for layout in layouts:
            cols = {"utf8_blocks": text.cols_utf8, "large_utf8": text.col_large, "utf8_view": text.col_view}[layout]()
            ms, runs = L.time_events(ctx, lambda cols=cols: run_pred(ctx, cols, pred, mask), steps)
            r[layout] = entry(ms, runs, floor_bytes(layout, n, text.string_bytes, len(text.blocks)),
                              L.check_mask(f"{name} {pname} {layout}", device_summary(ctx, mask, n), exp))
        if codes_too:
            r["dictionary_codes"] = via_codes(ctx, n, codes, values, pred, mask, steps, exp)
        r["cpu_arrow_cpp_ms"] = round(cpu_reference(offs, data, n, pred, threads), 1)
        res[pname] = r
    ctx.free(mask)
    text.free()
    return res


def via_codes(ctx, n, codes, values, pred, mask, steps, exp):
    dcodes = ctx.malloc(n * 4)
    for s in range(0, n, len(codes)):
        m = min(len(codes), n - s)
        ctx.check(ctx.lib.dfgpu_memcpy_h2d(ctx.h, C.c_void_p(dcodes + 4 * s), codes.ctypes.data_as(C.c_void_p), m * 4))
    ccol = D.Column()
    ccol.type, ccol.flags, ccol.length, ccol.offset, ccol.null_count, ccol.values, ccol.validity = D.INT32, 0, n, 0, 0, dcodes, None
    lib = D.load_strings_library()
    st = ctx.lib.dfgpu_ctx_stream(ctx.h)
    dvals = D.DeviceStrings(ctx, pa.array(values))
    kind, arg = pred

    def fn():
        cm = D.string_in_list(ctx, dvals, arg) if kind == "in" else D.string_compare(ctx, dvals, kind, arg)
        D._strings_check(lib.dfgpu_like_codes(st, C.byref(ccol), C.c_void_p(cm.values.ptr), len(values), C.c_void_p(mask), None))
        return cm
    ms, runs = L.time_events(ctx, fn, steps)
    out = entry(ms, runs, floor_bytes("dictionary_codes", n, 0), L.check_mask("codes", device_summary(ctx, mask, n), exp))
    ctx.free(dcodes)
    return out


def main():
    sf = float(sys.argv[1]) if len(sys.argv) > 1 else 100.0
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    threads = os.cpu_count() or 1
    ctx = D.Context(0)
    out = {"sf": sf, "card": L.card(), "steps": steps, "host_threads": threads}
    rng = np.random.default_rng(42)
    n_li, n_cust, n_part = int(6_000_000 * sf), int(150_000 * sf), int(200_000 * sf)
    all3 = ["utf8_blocks", "large_utf8", "utf8_view"]
    out["l_shipmode"] = measure(ctx, "l_shipmode", n_li, MODES, [("in_mail_ship", ("in", ["MAIL", "SHIP"]))], all3, steps, threads, rng, codes_too=True)
    print(json.dumps({"l_shipmode": out["l_shipmode"]}), flush=True)
    out["c_mktsegment"] = measure(ctx, "c_mktsegment", n_cust, SEGMENTS, [("eq_building", ("=", "BUILDING"))], all3[1:], steps, threads, rng)
    print(json.dumps({"c_mktsegment": out["c_mktsegment"]}), flush=True)
    out["p_container"] = measure(ctx, "p_container", n_part, CONTAINERS, [("in_sm", ("in", ["SM CASE", "SM BOX", "SM PACK", "SM PKG"]))],
                                 all3[1:], steps, threads, rng)
    out["p_brand"] = measure(ctx, "p_brand", n_part, BRANDS, [("eq_brand12", ("=", "Brand#12"))], all3[1:], steps, threads, rng)
    out["p_type"] = measure(ctx, "p_type", n_part, L.TYPES, [("lt_medium", ("<", "MEDIUM"))], all3[1:], steps, threads, rng)
    out["card_after"] = L.card()
    out["checks"] = "every mask: match count and row-number fingerprint equal to pyarrow.compute (is_in / equal / less) over the same strings"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
