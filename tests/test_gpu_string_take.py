"""string_take (dfgpu_string_take_offsets / _data / _views, libdfgpu_strings.so) against pyarrow.compute.take, value and validity, over
Utf8, LargeUtf8 and Utf8View: slices at offsets 0, 3 and 37, NULL strings and NULL ids, empty strings, empty id columns, rows long
enough to span many output words, UINT32 ids and packed INT64 ids over several sources (more than one launch's 64 included), Utf8View
with inline and out-of-line strings in many data buffers, and the refusals: an id outside its source, a Utf8 output beyond 2^31 - 1
bytes."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_b200 import capi as D

pytestmark = pytest.mark.gpu

TYPES = {"utf8": pa.string(), "large_utf8": pa.large_string(), "utf8_view": pa.string_view()}
WORDS = ["furiously", "special", "requests", "ß", "deposits", "日本", "", "x", "packages", "quickly", "😀"]


def strings(rng, n, null_p=0.1, long_p=0.02):
    out = []
    for _ in range(n):
        r = rng.random()
        if r < null_p:
            out.append(None)
        elif r < null_p + long_p:
            out.append("".join(rng.choice(WORDS, int(rng.integers(30, 700)))))   # 300 B .. 5 KB
        else:
            out.append(" ".join(rng.choice(WORDS, int(rng.integers(0, 6)))))      # 0 .. ~50 B, many unaligned
    return out


def view_array(values, n_buffers, rng):
    """a Utf8View array whose out-of-line strings are spread over n_buffers data buffers at random"""
    bufs = [bytearray() for _ in range(n_buffers)]
    views = np.zeros((len(values), 16), np.uint8)
    valid = np.ones(len(values), bool)
    for i, s in enumerate(values):
        if s is None:
            valid[i] = False
            continue
        b = s.encode()
        views[i, :4] = np.frombuffer(np.int32(len(b)).tobytes(), np.uint8)
        if len(b) <= 12:
            views[i, 4:4 + len(b)] = np.frombuffer(b, np.uint8)
        else:
            k = int(rng.integers(0, n_buffers))
            views[i, 4:8] = np.frombuffer(b[:4], np.uint8)
            views[i, 8:12] = np.frombuffer(np.int32(k).tobytes(), np.uint8)
            views[i, 12:16] = np.frombuffer(np.int32(len(bufs[k])).tobytes(), np.uint8)
            bufs[k] += b
    validity = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    arr = pa.Array.from_buffers(pa.string_view(), len(values), [validity, pa.py_buffer(views.tobytes())] + [pa.py_buffer(bytes(b)) for b in bufs],
                                null_count=int((~valid).sum()))
    arr.validate(full=True)
    return arr


def as_utf8(a):
    return a.cast(pa.large_string()) if not pa.types.is_large_string(a.type) else a


def expect(sources, ids):
    """pyarrow's take over the concatenated sources, the packed ids turned into rows of the concatenation"""
    ids = pa.array(ids) if not isinstance(ids, pa.Array) else ids
    if pa.types.is_int64(ids.type):
        base = np.cumsum([0] + [len(s) for s in sources])
        v = np.asarray(ids.fill_null(0))
        rows = base[v >> 32] + (v & 0xFFFFFFFF)
        ids = pa.array(rows, pa.int64(), mask=np.asarray(ids.is_null()))
    cat = pa.concat_arrays([as_utf8(s) for s in sources]) if sources else None
    return pc.take(cat, ids)


def check(got, sources, ids, typ):
    a = got.to_arrow()
    a.validate(full=True)
    assert a.type == typ
    exp = expect(sources, ids)
    assert a.null_count == exp.null_count
    assert as_utf8(a).equals(exp)


@pytest.mark.parametrize("name", list(TYPES))
@pytest.mark.parametrize("offset", [0, 3, 37])
def test_uint32_ids_over_one_slice(gpu_ctx, name, offset):
    rng = np.random.default_rng(offset * 7 + len(name))
    vals = strings(rng, 5000 + offset)
    full = view_array(vals, 5, rng) if name == "utf8_view" else pa.array(vals, TYPES[name])
    src = full.slice(offset, 5000)
    ids = rng.integers(0, 5000, 30000).astype(np.uint32)
    idn = pa.array(ids, pa.uint32(), mask=rng.random(30000) < 0.05)
    check(D.string_take(gpu_ctx, [src], idn), [src], idn, TYPES[name])


@pytest.mark.parametrize("name", list(TYPES))
@pytest.mark.parametrize("n_sources", [3, 70])
def test_packed_ids_over_several_sources(gpu_ctx, name, n_sources):
    rng = np.random.default_rng(n_sources)
    sources = []
    for s in range(n_sources):
        vals = strings(rng, int(rng.integers(1, 400)))
        a = view_array(vals, int(rng.integers(0, 4)) + 1, rng) if name == "utf8_view" else pa.array(vals, TYPES[name])
        sources.append(a.slice(s % 5))
    lens = np.array([len(s) for s in sources])
    src = rng.integers(0, n_sources, 50000)
    row = (rng.random(50000) * lens[src]).astype(np.int64)
    ids = pa.array((src.astype(np.int64) << 32) | row, pa.int64(), mask=rng.random(50000) < 0.03)
    check(D.string_take(gpu_ctx, sources, ids), sources, ids, TYPES[name])


@pytest.mark.parametrize("name", list(TYPES))
def test_nondecreasing_filter_ids_and_long_rows(gpu_ctx, name):
    """the filter's shape: nondecreasing packed ids over a few batches; and rows of kilobytes, all NULL, all empty"""
    rng = np.random.default_rng(11)
    batches = [pa.array(strings(rng, 3000, null_p=0.3, long_p=0.3), TYPES[name]) for _ in range(4)]
    batches.append(pa.array([None] * 50, TYPES[name]))
    batches.append(pa.array([""] * 70, TYPES[name]))
    ids = []
    for b, a in enumerate(batches):
        keep = np.nonzero(rng.random(len(a)) < 0.6)[0]
        ids.append((np.int64(b) << 32) | keep.astype(np.int64))
    ids = pa.array(np.concatenate(ids), pa.int64())
    check(D.string_take(gpu_ctx, batches, ids), batches, ids, TYPES[name])


@pytest.mark.parametrize("name", list(TYPES))
def test_empty_ids_and_empty_strings(gpu_ctx, name):
    src = pa.array(["", None, "", "a"], TYPES[name])
    for ids in (pa.array([], pa.uint32()), pa.array([], pa.int64())):
        got = D.string_take(gpu_ctx, [src], ids).to_arrow()
        assert len(got) == 0 and got.type == TYPES[name]
    ids = pa.array([0, 2, 0, 1, None, 3], pa.uint32())
    check(D.string_take(gpu_ctx, [src], ids), [src], ids, TYPES[name])


def test_view_buffers_are_rebased_across_many_buffers(gpu_ctx):
    """300 data buffers in one source and 2 to 9 in others: out-of-line views point into the concatenated buffer list"""
    rng = np.random.default_rng(5)
    sources = [view_array(strings(rng, 4000, long_p=0.5), 300, rng)] + [view_array(strings(rng, 500, long_p=0.5), k, rng) for k in range(2, 10)]
    lens = np.array([len(s) for s in sources])
    src = rng.integers(0, len(sources), 40000)
    ids = pa.array((src.astype(np.int64) << 32) | (rng.random(40000) * lens[src]).astype(np.int64), pa.int64())
    got = D.string_take(gpu_ctx, sources, ids)
    a = got.to_arrow()
    assert len(a.buffers()) == 2 + sum(len(s.buffers()) - 2 for s in sources)
    check(got, sources, ids, pa.string_view())


@pytest.mark.parametrize("name", list(TYPES))
def test_out_of_range_ids_are_refused(gpu_ctx, name):
    srcs = [pa.array([f"s{i}" * 5 for i in range(10)], TYPES[name]) for _ in range(70)]
    for sources, ids in (([srcs[0]], pa.array([0, 10], pa.uint32())),             # row == length
                         (srcs[:3], pa.array([(3 << 32) | 0], pa.int64())),        # no such source
                         (srcs, pa.array([(69 << 32) | 10, 5], pa.int64())),       # a row past a later launch's source
                         ([srcs[0].slice(4)], pa.array([6], pa.uint32()))):        # past the end of a slice
        with pytest.raises(D.DfgpuError, match="outside their source") as e:
            D.string_take(gpu_ctx, sources, ids)
        assert e.value.code == D.ERR_INVALID


def test_utf8_offset_overflow_is_refused_from_the_total(gpu_ctx):
    """2049 copies of a 1 MiB string exceed 2^31 - 1 bytes: refused after phase 1, before any output allocation; LargeUtf8 is not"""
    big = "x" * (1 << 20)
    ids = pa.array(np.zeros(2049, np.uint32))
    with pytest.raises(D.DfgpuError, match="offset overflow") as e:
        D.string_take(gpu_ctx, [pa.array([big], pa.string())], ids)
    assert e.value.code == D.ERR_INVALID
    got = D.string_take(gpu_ctx, [pa.array([big, "y"], pa.large_string())], pa.array([1, 0, 1], pa.uint32())).to_arrow()
    assert got.to_pylist() == ["y", big, "y"]
