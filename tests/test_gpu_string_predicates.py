"""dfgpu_string_compare / dfgpu_string_in_list (libdfgpu_strings.so) on the GPU against the CPU restatement
(tests/string_predicate_oracle.py), mask value and validity bit for bit: every op and IN / NOT IN over Utf8, LargeUtf8 and Utf8View,
slices at non-zero offsets, with and without NULLs, empty columns, columns longer than one grid pass, Utf8View with inline and
out-of-line strings in several data buffers, dictionary codes through dfgpu_like_codes, and the refusals."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_b200 import capi as D
from string_predicate_oracle import LITERALS, OPS, compare, gen_strings, in_list

pytestmark = pytest.mark.gpu

LAYOUTS = [pa.string(), pa.large_string(), pa.string_view()]
LISTS = [["MAIL", "SHIP"], ["SM CASE", "SM BOX", "SM PACK", "SM PKG"], ["", "a", "ab"], ["abcdefghijklm", "special requests and more", "é"],
         ["MAIL", None], [None], ["zz", "é", "éa", "中😀", "\x00", "a\x00", "DELIVER IN PERSON"], LITERALS]


@pytest.fixture(scope="module")
def ctx():
    c = D.Context(0)
    yield c
    c.close()


def got(m, n):
    v, valid = D.device_column_numpy(m)
    assert len(v) == n
    if valid is None:
        valid = np.ones(n, bool)
    assert not v[~valid].any(), "NULL results must hold 0"
    assert set(np.unique(v).tolist()) <= {0, 1}
    return [bool(x) if ok else None for x, ok in zip(v.tolist(), valid.tolist())]


def check_compare(ctx, arr, op, lit):
    g, e = got(D.string_compare(ctx, arr, op, lit), len(arr)), compare(arr.to_pylist(), op, lit)
    bad = [i for i, (x, y) in enumerate(zip(g, e)) if x != y]
    assert not bad, f"{arr.type} {op} {lit!r}: row {bad[0]} {arr[bad[0]]!r}: {g[bad[0]]} != {e[bad[0]]}"


def check_in(ctx, arr, items, negated):
    g, e = got(D.string_in_list(ctx, arr, items, negated), len(arr)), in_list(arr.to_pylist(), items, negated)
    bad = [i for i, (x, y) in enumerate(zip(g, e)) if x != y]
    assert not bad, f"{arr.type} {'NOT ' if negated else ''}IN {items!r}: row {bad[0]} {arr[bad[0]]!r}: {g[bad[0]]} != {e[bad[0]]}"


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
@pytest.mark.parametrize("null_p", [0.0, 0.15])
def test_every_op_and_list(ctx, t, null_p):
    rng = np.random.default_rng(1)
    arr = pa.array(gen_strings(rng, 5000, null_p=null_p), t)
    for lit in LITERALS:
        for op in OPS:
            check_compare(ctx, arr, op, lit)
    for items in LISTS:
        for neg in (False, True):
            check_in(ctx, arr, items, neg)


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
def test_slices_and_empty_columns(ctx, t):
    rng = np.random.default_rng(2)
    base = pa.array(gen_strings(rng, 900, null_p=0.2), t)
    for off in (0, 3, 37, 64):
        for ln in (0, 1, 31, 33, 700):
            s = base.slice(off, ln)
            for op in OPS:
                check_compare(ctx, s, op, "abc")
                check_compare(ctx, s, op, "BUILDING")
            for items in (["MAIL", "SHIP"], ["ab", None]):
                check_in(ctx, s, items, False)
                check_in(ctx, s, items, True)
    empty = pa.array([], t)
    assert got(D.string_compare(ctx, empty, "=", "a"), 0) == [] and got(D.string_in_list(ctx, empty, ["a", None]), 0) == []


def views_in_buffers(rng, vals, n_bufs, valid=None):
    """a Utf8View array with inline strings and out-of-line strings spread over n_bufs data buffers in no order, padding of the inline
    views filled with 0xFF (never relied on)"""
    bufs = [bytearray(b"\x07" * k) for k in range(n_bufs)]
    views = bytearray()
    for v in vals:
        b = (v or "").encode()
        if len(b) <= 12:
            views += len(b).to_bytes(4, "little") + b + b"\xff" * (12 - len(b))
        else:
            k = int(rng.integers(n_bufs))
            views += len(b).to_bytes(4, "little") + b[:4] + k.to_bytes(4, "little") + len(bufs[k]).to_bytes(4, "little")
            bufs[k] += b
    vb = None if valid is None else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    return pa.Array.from_buffers(pa.string_view(), len(vals), [vb, pa.py_buffer(bytes(views))] + [pa.py_buffer(bytes(b)) for b in bufs],
                                 null_count=0 if valid is None else int((~valid).sum()))


@pytest.mark.parametrize("n_bufs", [1, 3, 250])
def test_utf8view_inline_and_out_of_line_in_several_buffers(ctx, n_bufs):
    """250 buffers take two launches (240 data buffers per launch)"""
    rng = np.random.default_rng(3)
    vals = gen_strings(rng, 6000)
    valid = rng.random(len(vals)) > 0.1
    arr = views_in_buffers(rng, vals, n_bufs, valid)
    assert arr.to_pylist() == [v if ok else None for v, ok in zip(vals, valid)]
    for s in (arr, arr.slice(37)):
        for lit in ("abcdefghijklm", "abcd", "abcdefghijkl", "special requests and more", "special", "é", ""):
            for op in OPS:
                check_compare(ctx, s, op, lit)
        for items in LISTS:
            if n_bufs > 240 and None in items:
                with pytest.raises(D.DfgpuError) as e:
                    D.string_in_list(ctx, s, items)
                assert e.value.code == -3 and "240 data buffers" in str(e.value)
                continue
            check_in(ctx, s, items, False)
            check_in(ctx, s, items, True)
    for items in (["abcdefghijklm", None], ["special requests and more", "ab", None]):     # out-of-line values found, a NULL in the list
        check_in(ctx, views_in_buffers(rng, vals, min(n_bufs, 240), valid), items, True)


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
def test_longer_than_one_grid_pass(ctx, t):
    """3M rows of TPC-H ship modes, more rows than one pass of a grid that fills the device, checked against pyarrow.compute"""
    n = 3_000_000
    rng = np.random.default_rng(4)
    modes = np.array(["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB", "DELIVER IN PERSON x"], object)
    vals = modes[rng.integers(0, len(modes), n)]
    valid = rng.random(n) > 0.05
    plain = pa.array(vals, pa.string(), mask=~valid)
    arr = plain.cast(t)
    for op, lit in (("=", "SHIP"), ("<>", "MAIL"), ("<", "RAIL"), (">=", "DELIVER IN PERSON"), ("<=", "FOB"), (">", "AIR")):
        exp = {"=": pc.equal, "<>": pc.not_equal, "<": pc.less, "<=": pc.less_equal, ">": pc.greater, ">=": pc.greater_equal}[op](plain, lit)
        v, vv = D.device_column_numpy(D.string_compare(ctx, arr, op, lit))
        assert np.array_equal(vv, valid) and np.array_equal(v.astype(bool), np.asarray(exp.fill_null(False))), (op, lit)
    for neg in (False, True):
        v, vv = D.device_column_numpy(D.string_in_list(ctx, arr, ["MAIL", "SHIP"], neg))
        exp = np.asarray(pc.is_in(plain, value_set=pa.array(["MAIL", "SHIP"]))) != neg
        assert np.array_equal(vv, valid) and np.array_equal(v.astype(bool), exp & valid)
        v, vv = D.device_column_numpy(D.string_in_list(ctx, arr, ["MAIL", None], neg))
        found = np.asarray(pc.equal(plain, "MAIL").fill_null(False))
        assert np.array_equal(vv, valid & found) and np.array_equal(v.astype(bool), found & valid & (not neg))


def test_dictionary_codes(ctx):
    rng = np.random.default_rng(5)
    values = pa.array(LITERALS + ["AIR", "REG AIR", "MAIL x"])
    nd = len(values)
    codes = rng.integers(0, nd, 6000).astype(np.int32)
    valid = rng.random(6000) > 0.2
    for make, exp in ((lambda: D.string_compare(ctx, values, "<", "MAIL"), compare(values.to_pylist(), "<", "MAIL")),
                      (lambda: D.string_compare(ctx, values, "=", "BUILDING"), compare(values.to_pylist(), "=", "BUILDING")),
                      (lambda: D.string_in_list(ctx, values, ["MAIL", "SHIP", "AIR"], True), in_list(values.to_pylist(), ["MAIL", "SHIP", "AIR"], True))):
        cm = make()
        for off in (0, 5):
            dc = D.DeviceColumn.from_host(ctx, D.HostColumn(codes, valid))
            c = dc.c()
            c.offset, c.length = off, 6000 - off
            v, vv = D.device_column_numpy(D.like_codes(ctx, c, cm, nd))
            assert vv.tolist() == valid[off:].tolist()
            assert [bool(x) for x, ok in zip(v, vv) if ok] == [exp[k] for k, ok in zip(codes[off:], valid[off:]) if ok]
            assert not v[~vv].any()


def test_refusals(ctx):
    arr = pa.array(["a", "b", None])
    for args, code, msg in ((("=", "x" * 257), -3, "longer than 256"), (("=", b"\xffa"), -1, "UTF-8"), (("<", b"a\xc3"), -1, "UTF-8"),
                            (("=", b"\xed\xa0\x80"), -1, "UTF-8"), ((9, "a"), -1, "unknown op"), ((-1, "a"), -1, "unknown op")):
        with pytest.raises(D.DfgpuError) as e:
            D.string_compare(ctx, arr, *args)
        assert e.value.code == code and msg in str(e.value), (args, str(e.value))
    for items, code, msg in (([f"v{i}" for i in range(65)], -3, "more than 64"), (["x" * 600, "y" * 425], -3, "1024 bytes"),
                             (["a", b"\xc0\x80"], -1, "value 1 is not valid UTF-8")):
        with pytest.raises(D.DfgpuError) as e:
            D.string_in_list(ctx, arr, items)
        assert e.value.code == code and msg in str(e.value), (items[:3], str(e.value))
    # at the caps: accepted (duplicates count once)
    check_compare(ctx, pa.array(["x" * 256, "x" * 255, None]), "=", "x" * 256)
    check_in(ctx, pa.array(["v63", "v64", None]), [f"v{i}" for i in range(64)] * 2, False)
    check_in(ctx, pa.array(["x" * 600, "y" * 424, "y"]), ["x" * 600, "y" * 424], False)
    # malformed arguments at the C ABI
    lib = D.load_strings_library()
    ds = D.DeviceStrings(ctx, arr)
    col = ds.c()
    out = D.DeviceBuffer(ctx, 3)
    st = ctx.lib.dfgpu_ctx_stream(ctx.h)
    import ctypes as C
    assert lib.dfgpu_string_compare(st, C.byref(col), 0, b"a", 1, C.c_void_p(out.ptr), None) == -1          # validity but no out_validity
    assert lib.dfgpu_string_compare(st, None, 0, b"a", 1, C.c_void_p(out.ptr), None) == -1
    assert lib.dfgpu_string_compare(st, C.byref(col), 0, None, 3, C.c_void_p(out.ptr), None) == -1
    col2 = D.DeviceStrings(ctx, pa.array(["a", "b"])).c()
    assert lib.dfgpu_string_in_list(st, C.byref(col2), None, None, 0, 1, 0, C.c_void_p(out.ptr), None) == -1   # NULL in list, no out_validity
    assert lib.dfgpu_string_in_list(st, C.byref(col2), None, None, 2, 0, 0, C.c_void_p(out.ptr), None) == -1
    col2.layout = 7
    assert lib.dfgpu_string_compare(st, C.byref(col2), 0, b"a", 1, C.c_void_p(out.ptr), None) == -1
    assert "unknown string layout" in lib.dfgpu_strings_last_error().decode()
