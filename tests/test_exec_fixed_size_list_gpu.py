"""FixedSizeList payload columns through the host operator (dfd_repartition_exec_*).

Every case is checked row by row against the input rows taken in the CPU oracle's stable destination order: the list
validity, the child values (the raw bytes under null slots included) and the child validity, in every partition stream.
The same batches go through four operators — host -> host, host -> device, device -> device and device -> host — and their
streams must carry identical buffers.  tests/test_exec_fixed_size_list_cpu_harness.py runs these bodies on the CPU harness."""
import ctypes as C
import gc
import json
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests import device_batches as DB
from tests import device_outputs as DO
from tests.test_exec_device_input_gpu import assert_same_streams

pytestmark = pytest.mark.gpu

GiB = 1 << 30

# every child type the operator accepts that pyarrow can build (Interval(YearMonth) / Interval(DayTime) children are accepted
# too, see tests/test_fixed_size_list_cpu.py, but pyarrow has no array type for them)
CHILD_TYPES = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(), pa.float16(), pa.float32(),
               pa.float64(), pa.decimal128(20, 3), pa.decimal128(38, 0), pa.date32(), pa.date64(),
               pa.time32("s"), pa.time32("ms"), pa.time64("us"), pa.time64("ns"), pa.timestamp("us"), pa.timestamp("ns", tz="UTC"),
               pa.duration("ms"), pa.month_day_nano_interval(), pa.bool_()]
if hasattr(pa, "decimal32"):
    CHILD_TYPES += [pa.decimal32(9, 2), pa.decimal64(18, 4)]
NS = [1, 2, 3, 7, 8, 9, 31, 32, 33, 768]


@pytest.fixture(scope="module")
def ctx(built):
    c = dfd.WorkerContext(0)
    DO.COPY = DO.gpu_copy(c)
    yield c
    DO.COPY = None
    c.close()


# ------------------------------------------------------------------ inputs ----

def _width(t):
    return 0 if pa.types.is_boolean(t) else t.bit_width // 8


def _bits(rng, nbits, p_null):
    if nbits > 1 << 26:  # (the limit tests: random bytes, half the bits clear, without a float per bit)
        return rng.integers(0, 256, (nbits + 7) // 8, dtype=np.uint8).tobytes()
    return np.packbits(rng.random(nbits) >= p_null, bitorder="little").tobytes()


def fsl_array(rng, t, n, rows, parent_nulls=0.0, child_nulls=0.0, child_nullable=True, child_bitmap=None, offset=0, child_offset=0,
              bitmap_null_count_zero=False):
    """A FixedSizeList<t, n> of `rows` rows at array offset `offset` over a child at its own offset `child_offset`.  Child
    values are random bytes (or bits), so every byte under a null slot is checked too.  child_bitmap=False: a nullable
    child without a bitmap; bitmap_null_count_zero: a child bitmap of all ones with null_count 0."""
    ne = (child_offset + (offset + rows) * n)
    w = _width(t)
    vals = _bits(rng, ne, 0.5) if w == 0 else rng.integers(0, 256, ne * w, dtype=np.uint8).tobytes()
    cvalid = None
    if child_nulls > 0 and child_bitmap is not False:
        cvalid = pa.py_buffer(_bits(rng, ne, child_nulls))
    elif bitmap_null_count_zero:
        cvalid = pa.py_buffer(b"\xff" * ((ne + 7) // 8))
    child = pa.Array.from_buffers(t, ne - child_offset, [cvalid, pa.py_buffer(vals)], null_count=0 if cvalid is None or bitmap_null_count_zero else -1,
                                  offset=child_offset)
    pvalid = pa.py_buffer(_bits(rng, offset + rows, parent_nulls)) if parent_nulls > 0 else None
    ft = pa.list_(pa.field("item", t, nullable=child_nullable), n)
    return pa.Array.from_buffers(ft, rows, [pvalid], null_count=-1 if pvalid is not None else 0, offset=offset, children=[child])


def fsl_rows(a):
    """(list validity [rows], child values [rows, n x w] bytes or [rows, n] bits, child validity [rows, n]) of a FixedSizeList
    array, read from its buffers at its offsets (bytes under null slots included)."""
    n, rows, t = a.type.list_size, len(a), a.type.value_type
    v = a.values
    pb, cb, vb = a.buffers()[:3]

    def bits(buf, first, cnt):
        if buf is None or cnt == 0:
            return np.ones(cnt, dtype=bool)
        return np.unpackbits(np.frombuffer(buf, dtype=np.uint8), bitorder="little")[first:first + cnt].astype(bool)

    e0 = v.offset + a.offset * n  # (a child offset counts elements)
    pv = bits(pb if a.null_count != 0 else None, a.offset, rows)
    cv = bits(cb if v.null_count != 0 else None, e0, rows * n).reshape(rows, n)
    w = _width(t)
    if w == 0:
        vals = bits(vb, e0, rows * n).reshape(rows, n)
    else:
        vals = np.frombuffer(vb, dtype=np.uint8)[e0 * w:(e0 + rows * n) * w].reshape(rows, n * w)
    return pv, vals, cv


# ------------------------------------------------------------ device sides ----

class FslDeviceBatch(DB.DeviceBatch):
    """tests/device_batches.py's DeviceBatch with FixedSizeList columns: the parent's validity and its child array."""

    def _array(self, arr):
        if not pa.types.is_fixed_size_list(arr.type):
            return super()._array(arr)
        out = nv.ArrowArrayStruct()
        child = self._array(arr.values)
        bufs = (C.c_void_p * 1)(self._copy(arr.buffers()[0]))
        kids = (C.POINTER(nv.ArrowArrayStruct) * 1)(C.pointer(child))
        out.length, out.offset, out.n_buffers, out.null_count = len(arr), arr.offset, 1, arr.null_count
        out.buffers, out.n_children, out.children = C.cast(bufs, C.c_void_p), 1, C.cast(kids, C.c_void_p)
        out.release = C.cast(DB._child_release, C.c_void_p)
        self._keep += [out, bufs, kids, child]
        return out


def _host_array(src, t, keep):
    if not pa.types.is_fixed_size_list(t):
        return DO._array(src, t, keep)
    n = src.offset + src.length
    dev = DO._pointers(src.buffers, src.n_buffers)
    kid = C.cast(src.children, C.POINTER(C.POINTER(nv.ArrowArrayStruct)))[0].contents
    child = DO._array(kid, t.value_type, keep)
    bufs = (C.c_void_p * 1)(DO._fetch(dev[0], (n + 7) // 8, keep))
    kids = (C.POINTER(nv.ArrowArrayStruct) * 1)(C.pointer(child))
    out = nv.ArrowArrayStruct()
    out.length, out.null_count, out.offset, out.n_buffers = src.length, src.null_count, src.offset, 1
    out.buffers, out.n_children, out.children = C.cast(bufs, C.c_void_p), 1, C.cast(kids, C.c_void_p)
    out.release = C.cast(DO._child_release, C.c_void_p)
    keep += [out, bufs, kids, child]
    return out


def to_host_batch(device_array, schema):
    """tests/device_outputs.py's to_host_batch with FixedSizeList columns."""
    if DO.WAIT is not None and device_array.sync_event:
        DO.WAIT(device_array.sync_event)
    src = device_array.array
    keep = []
    kids_in = C.cast(src.children, C.POINTER(C.POINTER(nv.ArrowArrayStruct)))
    cols = [_host_array(kids_in[i].contents, schema.field(i).type, keep) for i in range(len(schema))]
    kids = (C.POINTER(nv.ArrowArrayStruct) * max(len(cols), 1))(*[C.pointer(c) for c in cols])
    bufs = (C.c_void_p * 1)(None)
    top = nv.ArrowArrayStruct()
    top.length, top.null_count, top.offset, top.n_buffers, top.n_children = src.length, 0, 0, 1, len(cols)
    top.buffers, top.children = C.cast(bufs, C.c_void_p), C.cast(kids, C.c_void_p)
    top.release = C.cast(DO._release, C.c_void_p)
    top.private_data = next(DO._KEYS)
    keep += [cols, kids, bufs, top]
    DO._LIVE[top.private_data] = keep
    return pa.RecordBatch._import_from_c(C.addressof(top), schema)


MODES = ("hh", "hd", "dd", "dh")  # input side (host / device), output side


def run_mode(ctx, mode, schema, batches, keys, N, **opts):
    ex = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash(keys, N), device_output=mode[1] == "d", **opts)
    pushed = []
    try:
        for rb in batches:
            if mode[0] == "h":
                ex.push_batch(rb)
            else:
                b = FslDeviceBatch(rb)
                pushed.append(b.key)
                ex.push_device_batch(b.device_array)
        ex.finish()
        if mode[1] == "h":
            streams = [list(ex.execute(p)) for p in range(N)]
        else:
            streams = []
            for p in range(N):
                s = ex.execute_device(p)
                streams.append([to_host_batch(b, s.schema) for b in s])
        stats = ex.stats()
    finally:
        ex.close()
    assert not set(pushed) & DB.live_batches()
    return streams, stats


def expected_order(key, N):
    ids = orc.partition_ids([key], len(key), N)
    return np.argsort(ids, kind="stable"), np.concatenate([[0], np.cumsum(np.bincount(ids, minlength=N))])


def check_against_oracle(streams, batches, N, key_col=0):
    """Each partition's rows, concatenated over its batches, are the input rows in the oracle's stable order."""
    table = pa.Table.from_batches(batches, schema=batches[0].schema) if batches else None
    key = np.concatenate([b.column(key_col).to_numpy(zero_copy_only=False) for b in batches]) if batches else np.zeros(0, np.int64)
    order, starts = expected_order(key, N)
    for c, field in enumerate(batches[0].schema if batches else []):
        per_batch = [fsl_rows(b.column(c)) if pa.types.is_fixed_size_list(field.type) else None for b in batches]
        for p in range(N):
            rows = order[starts[p]:starts[p + 1]]
            got = [b.column(c) for b in streams[p]]
            assert sum(len(g) for g in got) == len(rows), (field.name, p)
            if pa.types.is_fixed_size_list(field.type):
                want = [np.concatenate([pb[k] for pb in per_batch])[rows] for k in range(3)]
                parts = [fsl_rows(g) for g in got]
                for k, what in enumerate(("list validity", "child values", "child validity")):
                    have = np.concatenate([q[k] for q in parts]) if parts else want[k][:0]
                    assert np.array_equal(have, want[k]), (field.name, p, what)
            else:
                want = table.column(c).take(pa.array(rows, type=pa.int64())).to_pylist()
                assert [v for g in got for v in g.to_pylist()] == want, (field.name, p)


def check_case(ctx, batches, keys, N, modes=MODES, **opts):
    """The batches through every mode: the first against the oracle, the others buffer for buffer against it."""
    schema = batches[0].schema
    first, stats = None, {}
    for mode in modes:
        streams, stats[mode] = run_mode(ctx, mode, schema, batches, keys, N, **opts)
        if first is None:
            first = streams
            check_against_oracle(streams, batches, N, keys[0])
        else:
            assert_same_streams(first, streams)
    return stats


def _batch(key, *cols, names=None):
    names = names or ["k"] + [f"c{i}" for i in range(len(cols))]
    return pa.RecordBatch.from_arrays([pa.array(key, type=pa.int64())] + list(cols), names=names)


def _keys(rng, n):
    return rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64)


# ------------------------------------------------------------------- cases ----

def test_every_child_type(ctx):
    """Each accepted child type at n = 3 (a gathered width) and 4 (a scattered one for 1-, 2- and 4-byte children), nullable
    parent and child, sliced."""
    rng = np.random.Generator(np.random.PCG64(1))
    for t in CHILD_TYPES:
        for n in (3, 4):
            rows = 3000
            col = fsl_array(rng, t, n, rows, parent_nulls=0.2, child_nulls=0.3, offset=5, child_offset=3)
            check_case(ctx, [_batch(_keys(rng, rows), col)], [0], 8)


def check_n(ctx, n, child="f32", **kw):
    rng = np.random.Generator(np.random.PCG64(100 + n))
    t = pa.float32() if child == "f32" else pa.bool_()
    rows = 2500 if n < 100 else 600
    batches = []
    for b in range(3):
        col = fsl_array(rng, t, n, rows, parent_nulls=0.1, child_nulls=0.2, offset=b * 7, child_offset=b)
        batches.append(_batch(_keys(rng, rows), col))
    return check_case(ctx, batches, [0], 8, **kw)


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("child", ["f32", "bool"])
def test_list_sizes(ctx, n, child):
    check_n(ctx, n, child)


def check_nulls(ctx, case):
    rng = np.random.Generator(np.random.PCG64(7))
    rows = 4000
    kw = {"parent": dict(parent_nulls=0.3), "child": dict(child_nulls=0.3), "both": dict(parent_nulls=0.3, child_nulls=0.3),
          "no_bitmap": dict(child_nulls=0.3, child_bitmap=False), "null_count_zero": dict(bitmap_null_count_zero=True),
          "non_nullable_child": dict(child_nullable=False)}[case]
    for t in (pa.int32(), pa.bool_()):
        check_case(ctx, [_batch(_keys(rng, rows), fsl_array(rng, t, 5, rows, offset=3, **kw))], [0], 8)


@pytest.mark.parametrize("case", ["parent", "child", "both", "no_bitmap", "null_count_zero", "non_nullable_child"])
def test_nulls(ctx, case):
    check_nulls(ctx, case)


def check_slicing(ctx, t):
    """Parent offsets at every residue mod 32 and nonzero child offsets, batches of one schema appended into one chunk."""
    rng = np.random.Generator(np.random.PCG64(9))
    batches = []
    for off in range(32):
        rows = 97 + off
        col = fsl_array(rng, t, 7, rows, parent_nulls=0.2, child_nulls=0.2, offset=off, child_offset=(off * 5) % 13)
        batches.append(_batch(_keys(rng, rows), col))
    check_case(ctx, batches, [0], 3)


@pytest.mark.parametrize("t", [pa.int16(), pa.bool_()], ids=["int16", "bool"])
def test_parent_offsets_at_every_residue_and_child_offsets(ctx, t):
    check_slicing(ctx, t)


def check_batching(ctx, chunk_rows):
    """1-row and empty batches, many small batches coalesced into one chunk, and chunk cuts inside batches."""
    rng = np.random.Generator(np.random.PCG64(11))
    sizes = [1, 0, 1, 5, 0, 300, 1, 1000, 2500, 1, 0, 77]
    batches = [_batch(_keys(rng, r), fsl_array(rng, pa.float32(), 9, r, parent_nulls=0.1, child_nulls=0.1),
                      fsl_array(rng, pa.bool_(), 33, r, child_nulls=0.1, offset=3)) for r in sizes]
    check_case(ctx, batches, [0], 8, chunk_rows=chunk_rows)


@pytest.mark.parametrize("chunk_rows", [0, 64, 1000])
def test_batching_and_chunk_cuts(ctx, chunk_rows):
    check_batching(ctx, chunk_rows)


def check_mixed_schema(ctx, N):
    """Together with an Int64 key, Utf8, List<Utf8> and a dictionary column."""
    rng = np.random.Generator(np.random.PCG64(13 + N))
    batches = []
    for b, rows in enumerate([1500, 700, 2000]):
        words = [None if rng.random() < 0.1 else "w" * int(rng.integers(0, 20)) for _ in range(rows)]
        tags = [None if rng.random() < 0.1 else ["t"] * int(rng.integers(0, 3)) for _ in range(rows)]
        cat = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, 3, rows), type=pa.int32()), pa.array(["red", "green", "blue"]))
        batches.append(pa.RecordBatch.from_arrays(
            [pa.array(_keys(rng, rows)), fsl_array(rng, pa.float32(), 768, rows, parent_nulls=0.1, child_nulls=0.05, offset=b),
             pa.array(words, type=pa.string()), pa.array(tags, type=pa.list_(pa.string())), cat,
             fsl_array(rng, pa.bool_(), 31, rows, parent_nulls=0.2, child_nulls=0.2, child_offset=b)],
            names=["k", "emb", "s", "tags", "cat", "bits"]))
    check_case(ctx, batches, [0], N)


@pytest.mark.parametrize("N", [1, 3, 8, 17, 256])
def test_mixed_schema_and_partition_counts(ctx, N):
    check_mixed_schema(ctx, N)


# Profiled in a process of its own (below).  A profiling session started in the test process changes what later sessions
# there record: run that way, the whole suite's later check tests/test_fixed_size_list_gpu.py::test_k_gather_rows_runs saw
# no CUDA activity at all, not even its own kernels.  The later modules must find the process as they would without this one.
_PROFILE_BIT_ROWS = """
import json, sys
import numpy as np, pyarrow as pa, torch
from torch.profiler import ProfilerActivity, profile
import datafusion_distributed_b200 as dfd
from tests import device_outputs as DO, test_exec_fixed_size_list_gpu as G
ctx = dfd.WorkerContext(0)
DO.COPY = DO.gpu_copy(ctx)
rng = np.random.Generator(np.random.PCG64(17))
out = {}
for label, t, kw in (("nullable child", pa.int32(), dict(child_nulls=0.2)), ("boolean child", pa.bool_(), {})):
    batches = [G._batch(G._keys(rng, 5000), G.fsl_array(rng, t, 3, 5000, **kw))]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for mode in ("hh", "dd"):
            G.run_mode(ctx, mode, batches[0].schema, batches, [0], 8)
        torch.cuda.synchronize()
    out[label] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
ctx.close()
print(json.dumps(out))
"""


def test_k_gather_bit_rows_runs():
    """The nullable-child and the Boolean cases go through k_gather_bit_rows (as the 3-byte rows go through k_gather_rows)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-s", "-c", _PROFILE_BIT_ROWS], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    for label, kernels in names.items():
        assert any("k_gather_bit_rows" in k for k in kernels), (label, kernels)


# --------------------------------------------------------- 32-bit limits ----

def _need_free(nbytes):
    import torch

    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB is free")


def _row_of(a, r):
    """(list valid, child values, child validity) of row r of FixedSizeList array `a`, read from its packed buffers."""
    n, t, v = a.type.list_size, a.type.value_type, a.values
    pb, cb, vb = a.buffers()[:3]
    e0 = v.offset + (a.offset + r) * n

    def bits(buf, first, cnt):
        if buf is None:
            return np.ones(cnt, dtype=bool)
        chunk = np.frombuffer(buf, dtype=np.uint8)[first // 8:(first + cnt + 7) // 8 + 1]
        return np.unpackbits(chunk, bitorder="little")[first % 8:first % 8 + cnt].astype(bool)

    w = _width(t)
    vals = bits(vb, e0, n) if w == 0 else np.frombuffer(vb, dtype=np.uint8)[e0 * w:(e0 + n) * w]
    return bool(bits(pb if a.null_count else None, a.offset + r, 1)[0]), vals, bits(cb if v.null_count else None, e0, n)


def check_sampled(streams, batches, N, samples=4000, seed=0):
    """check_against_oracle for inputs too large to unpack: the key of every row, and the FixedSizeList columns of a random
    sample of output rows plus the last 64 rows of every partition (the highest bit and byte offsets of the chunk)."""
    assert len(batches) == 1
    rb = batches[0]
    key = rb.column(0).to_numpy()
    order, starts = expected_order(key, N)
    rng = np.random.Generator(np.random.PCG64(seed))
    for p in range(N):
        got = streams[p]
        assert np.array_equal(np.concatenate([g.column(0).to_numpy() for g in got]) if got else key[:0], key[order[starts[p]:starts[p + 1]]]), p
        cnt = int(starts[p + 1] - starts[p])
        idx = sorted(set(rng.integers(0, cnt, min(cnt, samples // N)).tolist()) | set(range(max(0, cnt - 64), cnt)))
        bounds = np.cumsum([0] + [g.num_rows for g in got])
        for i in idx:
            k = int(np.searchsorted(bounds, i, side="right") - 1)
            for c in range(1, rb.num_columns):
                have = _row_of(got[k].column(c), i - int(bounds[k]))
                want = _row_of(rb.column(c), int(order[starts[p] + i]))
                assert have[0] == want[0] and np.array_equal(have[1], want[1]) and np.array_equal(have[2], want[2]), (p, i, c)


def _check_big(ctx, batches, N, chunk_rows, modes):
    import torch

    for mode in modes:
        streams, _ = run_mode(ctx, mode, batches[0].schema, batches, [0], N, chunk_rows=chunk_rows)
        check_sampled(streams, batches, N)
        del streams
        gc.collect()
    torch.cuda.empty_cache()  # (the device copies of the input batches: give the memory back to the tests that follow)


def test_more_than_2_pow_32_child_bits_in_one_chunk(ctx):
    """FixedSizeList<Boolean, 1024> with a nullable child: 4.2 M rows in one chunk are more than 2^32 bits per bit-row column."""
    rows, n = (1 << 22) + 4099, 1024
    _need_free(16 * GiB)
    rng = np.random.Generator(np.random.PCG64(19))
    col = fsl_array(rng, pa.bool_(), n, rows, child_nulls=0.3, offset=3, child_offset=5)
    batches = [_batch(_keys(rng, rows), col)]
    _check_big(ctx, batches, 17, rows + 64, ("hh", "dd"))


def test_more_than_2_pow_31_child_bytes_in_one_chunk(ctx):
    """FixedSizeList<Float32, 768> (3 KiB rows): more than 2 GiB of child values in one chunk, gathered."""
    n = 768
    rows = (1 << 31) // (4 * n) + 1001
    _need_free(10 * GiB)
    rng = np.random.Generator(np.random.PCG64(23))
    col = fsl_array(rng, pa.float32(), n, rows, parent_nulls=0.1, offset=1)
    batches = [_batch(_keys(rng, rows), col)]
    _check_big(ctx, batches, 8, rows + 64, ("hh", "dd"))


# ----------------------------------------------------------- chunk sizing ----

def first_batch_rows(ctx, batches, **opts):
    ex = dfd.RepartitionExec(ctx, batches[0].schema, dfd.Partitioning.Hash([0], 1), **opts)
    try:
        for rb in batches:
            ex.push_batch(rb)
        ex.finish()
        return [b.num_rows for b in ex.execute(0)]
    finally:
        ex.close()


def check_chunk_sizing(ctx):
    rng = np.random.Generator(np.random.PCG64(29))
    rows = 200_000
    emb = fsl_array(rng, pa.float32(), 768, rows, parent_nulls=0.1)
    got = first_batch_rows(ctx, [_batch(_keys(rng, rows), emb)])
    per_row_bits = 64 + 8 * 3072 + 1 + 768  # the key, the values, the list validity, the child validity
    budget_rows = (256 << 20) * 8 // per_row_bits // 64 * 64
    assert got[0] == budget_rows and sum(got) == rows, got
    assert budget_rows * 3072 <= 256 << 20
    assert first_batch_rows(ctx, [_batch(_keys(rng, rows), emb)], chunk_rows=1000)[:2] == [1024, 1024]  # an explicit chunk_rows stands
    big = 5 << 20
    got = first_batch_rows(ctx, [_batch(np.arange(big, dtype=np.int64))])
    assert got == [4 << 20, big - (4 << 20)], got


def test_chunk_sizing(ctx):
    check_chunk_sizing(ctx)


# ---------------------------------------------------------------- refusals ----

def _schema_struct(fmt, child_fmt=None, child_dict=False, keep=None):
    keep = keep if keep is not None else []

    def node(f, name, flags=2):
        s = nv.ArrowSchemaStruct()
        s.format, s.name, s.flags = f.encode(), name, flags
        keep.append(s)
        return s

    col = node(fmt, b"emb")
    if child_fmt is not None:
        item = node(child_fmt, b"item")
        if child_dict:
            d = node("u", b"")
            item.dictionary = C.addressof(d)
        kids = (C.POINTER(nv.ArrowSchemaStruct) * 1)(C.pointer(item))
        keep.append(kids)
        col.n_children, col.children = 1, C.cast(kids, C.c_void_p)
    key = node("l", b"id")
    top = node("+s", b"")
    kids = (C.POINTER(nv.ArrowSchemaStruct) * 2)(C.pointer(key), C.pointer(col))
    keep.append(kids)
    top.n_children, top.children = 2, C.cast(kids, C.c_void_p)
    return top, keep


# (format, child format, child is a dictionary, emb is a key) -> refused with DFD_ERR_UNSUPPORTED naming the column
REFUSED = [("+w:4", "f", False, True), ("+w:0", "f", False, False), ("+w:4", "u", False, False), ("+w:4", "z", False, False),
           ("+w:4", "vu", False, False), ("+w:4", "c", True, False), ("+w:4", "w:16", False, False), ("+w:4", "w:12", False, False),
           ("+w:4", "+l", False, False), ("+w:4", "+w:2", False, False), ("+w:4", None, False, False), ("+w:4", "n", False, False)]


def test_refusals_at_create_name_the_column(ctx):
    for fmt, child, cdict, key in REFUSED:
        top, keep = _schema_struct(fmt, child, cdict)
        h = C.c_void_p()
        opts = nv.DfdExecOptions(0, 0, 0, 0, 0)
        rc = nv.lib().dfd_repartition_exec_create(ctx.handle, C.byref(top), (C.c_int32 * 1)(1 if key else 0), 1, 8, C.byref(opts), C.byref(h))
        msg = nv.lib().dfd_last_error().decode()
        assert rc == 6 and "emb" in msg, (fmt, child, rc, msg)
        assert not h.value
