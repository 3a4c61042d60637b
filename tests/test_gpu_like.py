"""dfgpu_like / dfgpu_like_codes (libdfgpu_strings.so) on the GPU against the CPU restatement of LikeExpr (tests/like_oracle.py):
every layout with LIKE and NOT LIKE, slices, Utf8View data buffers, sizes that cross tiles and alignments, dictionary codes and the
refusals."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_b200 import capi as D
from like_oracle import FIXED_PATTERNS, gen_pattern, gen_strings, like

pytestmark = pytest.mark.gpu

LAYOUTS = [pa.string(), pa.large_string(), pa.string_view()]


@pytest.fixture(scope="module")
def ctx():
    c = D.Context(0)
    yield c
    c.close()


def gpu_like(ctx, arr, pattern, negated=False):
    v, valid = D.device_column_numpy(D.like(ctx, arr, pattern, negated=negated))
    if valid is None:
        assert arr.null_count == 0
        valid = np.ones(len(arr), bool)
    assert not v[~valid].any(), "NULL rows must hold 0"
    return [bool(x) if ok else None for x, ok in zip(v.tolist(), valid.tolist())]


def check(ctx, arr, pattern, negated=False):
    exp = like(arr.to_pylist(), pattern, negated)
    got = gpu_like(ctx, arr, pattern, negated)
    bad = [i for i, (g, e) in enumerate(zip(got, exp)) if g != e]
    assert not bad, f"{pattern!r} negated={negated} {arr.type}: row {bad[0]} {arr[bad[0]]!r}: {got[bad[0]]} != {exp[bad[0]]}"


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
def test_layouts_patterns_and_nulls(ctx, t):
    rng = np.random.default_rng(1)
    arr = pa.array(gen_strings(rng, 3000, null_p=0.1) + ["", "special requests", "x" * 13, "é" * 7], t)
    pats = FIXED_PATTERNS + [gen_pattern(rng) for _ in range(60)]
    for k, p in enumerate(pats):
        check(ctx, arr, p, negated=bool(k % 2))
        check(ctx, arr, p, negated=not (k % 2))


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
def test_slices_keep_their_offsets(ctx, t):
    rng = np.random.default_rng(2)
    base = pa.array(gen_strings(rng, 700, max_len=40, null_p=0.2), t)
    for off in (0, 3, 37):
        for ln in (0, 1, 33, 600):
            s = base.slice(off, ln)
            for p in ("%a%", "_%b", "%special%requests%", "é%", "%_"):
                check(ctx, s, p)
                check(ctx, s, p, negated=True)


@pytest.mark.parametrize("t", [pa.string(), pa.large_string()], ids=str)
def test_offsets_not_from_zero_at_every_alignment(ctx, t):
    """offsets starting at 0..15 bytes into the data buffer, so tiles' byte ranges start and end at every alignment modulo 16"""
    rng = np.random.default_rng(3)
    vals = gen_strings(rng, 1500, max_len=30)
    raw = [v.encode() for v in vals]
    w = np.int32 if t == pa.string() else np.int64
    for start in range(16):
        data = b"\xff" * start + b"".join(raw) + b"\xfe" * 3        # bytes outside the array's range: invalid UTF-8, never matched
        offs = (start + np.concatenate([[0], np.cumsum([len(r) for r in raw])])).astype(w)
        arr = pa.Array.from_buffers(t, len(raw), [None, pa.py_buffer(offs.tobytes()), pa.py_buffer(data)])
        for p in ("%a%b%", "_%", "%€_", "x%"):
            check(ctx, arr, p)


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 511, 512, 513])
def test_sizes(ctx, t, n):
    rng = np.random.default_rng(n)
    arr = pa.array(gen_strings(rng, n, null_p=0.3), t)
    for p in ("%", "a%", "%a", "%a%", "_"):
        check(ctx, arr, p)
        check(ctx, arr, p, negated=True)


@pytest.mark.parametrize("t", LAYOUTS, ids=str)
def test_a_string_longer_than_any_tile(ctx, t):
    rng = np.random.default_rng(4)
    big = "".join(rng.choice(list("abcdé€ ")) for _ in range(1 << 16)) * 8 + "special x requests" + "y" * 1000   # > 1 MB
    vals = gen_strings(rng, 200) + [big] + gen_strings(rng, 200) + [big[:-1000] + "z", "é" * 700]
    arr = pa.array(vals, t)
    for p in ("%special%requests%", "%special%requests%y", "ab%", "%z", "%_y", "%é€%special%", "%qq%", "%" + "é" * 120 + "%", "_" * 200, "%" + "_" * 250):
        check(ctx, arr, p)
        check(ctx, arr, p, negated=True)


def test_utf8view_buffers_out_of_order(ctx):
    """views into three data buffers, in no buffer order, inline and out-of-line strings, a prefix pattern the view prefix decides"""
    rng = np.random.default_rng(5)
    vals = [v for v in gen_strings(rng, 3000, max_len=40)]
    bufs = [bytearray(b"\x00" * 5), bytearray(), bytearray(b"\x01" * 3)]
    views = bytearray()
    for i, v in enumerate(vals):
        b = v.encode()
        if len(b) <= 12:
            views += len(b).to_bytes(4, "little") + b + b"\x00" * (12 - len(b))
        else:
            k = int(rng.integers(3))
            views += len(b).to_bytes(4, "little") + b[:4] + k.to_bytes(4, "little") + len(bufs[k]).to_bytes(4, "little")
            bufs[k] += b
    valid = rng.random(len(vals)) > 0.1
    vb = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    arr = pa.Array.from_buffers(pa.string_view(), len(vals), [vb, pa.py_buffer(bytes(views))] + [pa.py_buffer(bytes(b)) for b in bufs],
                                null_count=int((~valid).sum()))
    assert arr.to_pylist() == [v if ok else None for v, ok in zip(vals, valid)]
    for p in ("spec%", "a%", "ab_%", "é€%", "%requests", "%a%", "____________%", "%green%"):
        check(ctx, arr, p)
        check(ctx, arr, p, negated=True)
        check(ctx, arr.slice(37), p)


def test_many_rows(ctx):
    """2^25 rows of short random text, checked against Arrow C++'s match_like"""
    n = 1 << 25
    rng = np.random.default_rng(6)
    lens = rng.integers(0, 16, n).astype(np.int32)
    offs = np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).astype(np.int32)
    data = rng.choice(np.frombuffer(b"abcxy ", np.uint8), int(offs[-1]))
    arr = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs.tobytes()), pa.py_buffer(data.tobytes())])
    for p, neg in (("%ab%c%", False), ("xy%", True), ("%a_b", False)):
        v, valid = D.device_column_numpy(D.like(ctx, arr, p, negated=neg))
        exp = np.asarray(pc.match_like(arr, p))
        assert valid is None and np.array_equal(v.astype(bool), exp != neg), p


def test_dictionary_codes(ctx):
    rng = np.random.default_rng(7)
    values = pa.array(gen_strings(rng, 50) + ["special requests", "green"])
    nd = len(values)
    for p, neg in (("%special%requests%", True), ("%green%", False), ("%a%", False)):
        cm = D.like(ctx, values, p, negated=neg)
        codes = rng.integers(0, nd, 5000).astype(np.int32)
        valid = rng.random(5000) > 0.2
        for off in (0, 5):
            dc = D.DeviceColumn.from_host(ctx, D.HostColumn(codes, valid))
            c = dc.c()
            c.offset, c.length = off, 5000 - off
            v, vv = D.device_column_numpy(D.like_codes(ctx, c, cm, nd))
            exp = like(values.to_pylist(), p, neg)
            assert vv.tolist() == valid[off:].tolist()
            assert [bool(x) for x, ok in zip(v, vv) if ok] == [exp[k] for k, ok in zip(codes[off:], valid[off:]) if ok]
            assert not v[~vv].any()
    dc = D.DeviceColumn.from_host(ctx, D.HostColumn(np.arange(10, dtype=np.int32)))
    v, vv = D.device_column_numpy(D.like_codes(ctx, dc, D.like(ctx, values, "%"), nd))
    assert vv is None and v.tolist() == [1] * 10


def test_refusals(ctx):
    arr = pa.array(["a", "b", None])
    cases = [("a\\%", False, D.DfgpuError, -3, "escape"), ("a%", True, D.DfgpuError, -3, "ILIKE"),
             ("x" * 257, False, D.DfgpuError, -3, "longer than 256"), ("%a" * 17, False, D.DfgpuError, -3, "16"),
             (b"\xffa%", False, D.DfgpuError, -1, "UTF-8"), (b"a\xc3", False, D.DfgpuError, -1, "UTF-8"),
             (b"\xed\xa0\x80", False, D.DfgpuError, -1, "UTF-8")]
    for pat, ci, exc, code, msg in cases:
        with pytest.raises(exc) as e:
            D.like(ctx, arr, pat, case_insensitive=ci)
        assert e.value.code == code and msg in str(e.value), (pat, str(e.value))
    # at the limits: accepted
    for p in ("x" * 256, "%a" * 16):
        check(ctx, pa.array(["x" * 256, "a" * 16, None]), p)
