"""Every hash-key type the host operator (RepartitionExec, csrc/dfd_exec.cu) accepts, through the operator, against the C
oracle: each destination must hold exactly the oracle's rows, in input order (a row-id Int64 payload column shows any loss,
duplication or reordering).

- every accepted flat key format, alone and as the middle key of [Int64, X, Utf8] (hash combine order), nullable with nulls
  and the edge bit patterns of its type (min / max, -0.0 / +0.0, NaNs with different payloads, +-inf, Float16 subnormals,
  negative decimals), over several batches that span small chunks, one batch sliced at offset 3;
- Dictionary<K, V> keys for all eight index types K and every value type V the operator accepts, with null indices, null
  values and values sliced at an offset; UInt8 indices >= 128 and UInt16 indices >= 32768 (read zero-extended, as
  DataFusion's `key.as_usize()`); interval values hashed field by field;
- the device partitioner's `set_key_dictionary(..., unsigned_index=True)`;
- (CPU) the library accepts exactly the key formats and dictionary combinations this module has a case for.

pyarrow has no Interval(YearMonth) ("tiM") and cannot import Interval(DayTime) ("tiD"): such columns are exported as a
pyarrow type of the same layout (Int32 / Int64) and the format string in the exported ArrowSchema is rewritten.  Output is
read from the operator's ArrowArrayStream with ctypes, never imported into pyarrow.  The operator is driven through the C ABI
returned by `native()` (the CPU harness test points it at its host stand-in)."""
import ctypes as C
import random
import re

import numpy as np
import pyarrow as pa
import pytest

from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc


def native():
    """The library whose dfd_repartition_exec_* the cases drive."""
    return nv.lib()


# Arrow format of every flat key the operator accepts -> a pyarrow type of the same layout (the exported format is then
# set to the key's format, which only changes something for "tiM" / "tiD")
FIXED = {
    "c": pa.int8(), "C": pa.uint8(), "s": pa.int16(), "S": pa.uint16(), "i": pa.int32(), "I": pa.uint32(), "l": pa.int64(), "L": pa.uint64(),
    "e": pa.float16(), "f": pa.float32(), "g": pa.float64(),
    "d:9,2,32": pa.decimal32(9, 2), "d:18,3,64": pa.decimal64(18, 3), "d:38,10": pa.decimal128(38, 10),
    "tdD": pa.date32(), "tdm": pa.date64(),
    "tts": pa.time32("s"), "ttm": pa.time32("ms"), "ttu": pa.time64("us"), "ttn": pa.time64("ns"),
    "tss:": pa.timestamp("s"), "tsm:": pa.timestamp("ms"), "tsu:": pa.timestamp("us"), "tsn:": pa.timestamp("ns"),
    "tsu:UTC": pa.timestamp("us", "UTC"), "tsn:Europe/Paris": pa.timestamp("ns", "Europe/Paris"),
    "tDs": pa.duration("s"), "tDm": pa.duration("ms"), "tDu": pa.duration("us"), "tDn": pa.duration("ns"),
    "tiM": pa.int32(),  # Interval(YearMonth): months as i32, hashed as one i32
    "tiD": pa.int64(),  # Interval(DayTime): {days: i32, milliseconds: i32}, hashed field by field
    "tin": pa.month_day_nano_interval(),
}
OTHER = {"b": pa.bool_(), "u": pa.string(), "U": pa.large_string(), "z": pa.binary(), "vu": pa.string_view(), "vz": pa.binary_view()}
KEY_FORMATS = list(FIXED) + list(OTHER)
INDEX_FORMATS = {"c": "i8", "C": "u8", "s": "i16", "S": "u16", "i": "i32", "I": "u32", "l": "i64", "L": "u64"}
DICT_VALUE_FORMATS = [f for f in KEY_FORMATS if not f.startswith("v")]  # view-typed dictionary values are refused as keys
# the value types every index type also runs as the MIDDLE key of [Int64, Dictionary<K, V>, Utf8]
DICT_MIDDLE_VALUES = ["u", "U", "z", "l", "C", "g", "b", "d:38,10", "tdD", "tin", "tiD"]

# little-endian bit patterns worth hashing, per float width
F16_EDGES = [0x0000, 0x8000, 0x7C00, 0xFC00, 0x7E00, 0x7E01, 0xFE00, 0x7C01, 0x0001, 0x03FF, 0x8001, 0x83FF, 0x7BFF, 0xFBFF, 0x3C00]
F32_EDGES = [0, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001, 1, 0x807FFFFF, 0x7F7FFFFF,
             0xFF7FFFFF, 0x3F800000]
F64_EDGES = [0, 1 << 63, 0x7FF0 << 48, 0xFFF0 << 48, 0x7FF8 << 48, (0x7FF8 << 48) | 1, 0xFFF8 << 48, (0x7FF0 << 48) | 1, 1,
             0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x3FF0 << 48]
WORDS = ["", "a", "δ", "x" * 12, "y" * 13, "z" * 16, "w" * 17, "a-much-longer-string-than-sixteen-bytes", "\x00", "ünïcödé-" * 3]
BYTES = [b"", b"\x00", b"\xff", b"\x00\xff" * 6, b"q" * 13, bytes(range(40))]

_FMT_BUFS = {}


def _width(fmt):
    return FIXED[fmt].bit_width // 8


def _edges(fmt):
    if fmt in ("e", "f", "g"):
        return {"e": F16_EDGES, "f": F32_EDGES, "g": F64_EDGES}[fmt]
    bits = 8 * _width(fmt)
    mx = (1 << bits) - 1
    out = [0, 1, mx >> 1, 1 << (bits - 1), mx, mx - 98]  # 0, 1, max, min, -1, -99 (negative decimals / intervals)
    if fmt == "tiD":
        out += [0xFFFFFFFF, 0xFFFFFFFF << 32, 0x80000000]  # {-1, 0}, {0, -1}, {min, 0}
    if fmt == "tin":
        out += [0xFFFFFFFF, 0xFFFFFFFF << 32, ((1 << 64) - 1) << 64]  # months / days / nanoseconds = -1, one at a time
    return out


def values(fmt, n, rnd, nulls=True):
    """n values of key format `fmt` (its stand-in pyarrow type): rows 3, 8, 13, ... null when `nulls` (with arbitrary bytes
    under fixed-width nulls), the type's edge patterns twice over, then random values."""
    null = [nulls and i % 5 == 3 for i in range(n)]
    if fmt in OTHER:
        pool = BYTES if fmt in ("z", "vz") else WORDS
        if fmt == "b":
            py = [None if null[i] else rnd.random() < 0.5 for i in range(n)]
        else:
            py = [None if null[i] else (pool[i % len(pool)] if i < 2 * len(pool) else
                                        (rnd.choice(pool) + (bytes([rnd.getrandbits(8)]) if isinstance(pool[0], bytes) else str(rnd.getrandbits(16)))))
                  for i in range(n)]
        return pa.array(py, type=OTHER[fmt])
    w, edges = _width(fmt), _edges(fmt)
    vals, e = [], 0
    for i in range(n):
        if not null[i] and e < 2 * len(edges):
            vals.append(edges[e % len(edges)])
            e += 1
        else:
            vals.append(rnd.getrandbits(8 * w))
    raw = b"".join(v.to_bytes(w, "little") for v in vals)
    valid = ~np.array(null, dtype=bool)
    bitmap = np.packbits(valid, bitorder="little").tobytes()
    return pa.Array.from_buffers(FIXED[fmt], n, [pa.py_buffer(bitmap), pa.py_buffer(raw)], null_count=int((~valid).sum()))


def oracle_column(arr, fmt):
    """The oracle's input for one key column whose (value) format is `fmt`; dictionaries are decoded here."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    if pa.types.is_dictionary(arr.type):
        arr = arr.dictionary_decode()
    if fmt == "tiD":
        raw = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64).view(np.uint8)
        return ("interval_day_time", raw, arr.is_valid().to_numpy(zero_copy_only=False))
    if fmt == "vz":
        return arr.cast(pa.binary())
    return arr


def _c_format(fmt):
    if fmt not in _FMT_BUFS:
        _FMT_BUFS[fmt] = C.create_string_buffer(fmt.encode())
    return C.cast(_FMT_BUFS[fmt], C.c_char_p)


def _check(lib, rc):
    if rc != 0:
        raise RuntimeError(f"status {rc}: {lib.dfd_last_error().decode('utf-8', 'replace')}")


def _read_row_ids(lib, h, p, rid_col):
    """Row ids of destination p, in stream order, read from the operator's ArrowArrayStream with ctypes."""
    st = nv.ArrowArrayStreamStruct()
    _check(lib, lib.dfd_repartition_exec_execute(h, p, C.byref(st)))
    get_next = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)(st.get_next)
    out = []
    try:
        while True:
            arr = nv.ArrowArrayStruct()
            rc = get_next(C.addressof(st), C.addressof(arr))
            if rc != 0:
                msg = C.CFUNCTYPE(C.c_char_p, C.c_void_p)(st.get_last_error)(C.addressof(st))
                raise RuntimeError(f"destination {p}: get_next {rc}: {msg}")
            if not arr.release:
                break
            try:
                child = C.cast(arr.children, C.POINTER(C.POINTER(nv.ArrowArrayStruct)))[rid_col].contents
                assert child.length == arr.length and child.null_count == 0
                if child.length:
                    data = C.cast(child.buffers, C.POINTER(C.c_void_p))[1]
                    out.append(np.ctypeslib.as_array((C.c_int64 * (child.offset + child.length)).from_address(data))[child.offset:].copy())
            finally:
                C.CFUNCTYPE(None, C.c_void_p)(arr.release)(C.addressof(arr))
    finally:
        C.CFUNCTYPE(None, C.c_void_p)(st.release)(C.addressof(st))
    return np.concatenate(out) if out else np.empty(0, dtype=np.int64)


def run_operator(ctx, table, keys, N, formats, chunk_rows=64):
    """Push `table` through a RepartitionExec(Hash(keys, N)) in ragged, sliced batches; -> row ids (last column) per destination.
    formats[i] = (format, dictionary value format or None) written into the exported schema of column i."""
    lib = native()
    cs = nv.ArrowSchemaStruct()
    table.schema._export_to_c(C.addressof(cs))
    kids = C.cast(cs.children, C.POINTER(C.POINTER(nv.ArrowSchemaStruct)))
    for i, (fmt, dict_fmt) in formats.items():
        kids[i].contents.format = _c_format(fmt)
        if dict_fmt:
            C.cast(kids[i].contents.dictionary, C.POINTER(nv.ArrowSchemaStruct)).contents.format = _c_format(dict_fmt)
    h = C.c_void_p()
    opts = nv.DfdExecOptions(chunk_rows, 0, 0, 0, 0)
    try:
        _check(lib, lib.dfd_repartition_exec_create(ctx.handle, C.byref(cs), (C.c_int32 * len(keys))(*keys), len(keys), N, C.byref(opts), C.byref(h)))
    finally:
        C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))
    try:
        n = table.num_rows
        cuts = sorted({0, min(3, n), min(50, n), n // 2, n // 2 + 1, max(n - 7, 0), n})  # the second batch starts at offset 3
        for a, b in zip(cuts[:-1], cuts[1:]):
            for rb in table.slice(a, b - a).to_batches():
                ca = nv.ArrowArrayStruct()
                rb._export_to_c(C.addressof(ca))
                _check(lib, lib.dfd_repartition_exec_push(h, C.byref(ca)))
        _check(lib, lib.dfd_repartition_exec_finish(h))
        return [_read_row_ids(lib, h, p, table.num_columns - 1) for p in range(N)]
    finally:
        lib.dfd_repartition_exec_destroy(h)


def check_placement(ctx, table, keys, N, formats, key_value_formats, what, chunk_rows=64):
    got = run_operator(ctx, table, keys, N, formats, chunk_rows)
    want = orc.partition_ids([oracle_column(table.column(k), f) for k, f in zip(keys, key_value_formats)], table.num_rows, N)
    assert sum(len(g) for g in got) == table.num_rows, what
    for p in range(N):
        assert np.array_equal(got[p], np.flatnonzero(want == p)), f"{what}, N={N}: destination {p} holds rows {got[p][:12]}..., " \
                                                                   f"the oracle {np.flatnonzero(want == p)[:12]}..."


def _seed(*parts):
    return sum(ord(ch) * (i + 1) for i, ch in enumerate("|".join(parts)))


def _row_ids(n):
    return pa.array(np.arange(n, dtype=np.int64))


def _lead_and_tail(n, rnd):
    lead = pa.array([None if i % 7 == 2 else rnd.getrandbits(64) - (1 << 63) for i in range(n)], type=pa.int64())
    return lead, values("u", n, rnd)


def check_key_format(ctx, fmt, n=300):
    rnd = random.Random(_seed(fmt))
    x = values(fmt, n, rnd)
    lead, tail = _lead_and_tail(n, rnd)
    alone = pa.table([x, _row_ids(n)], names=["x", "rid"])
    middle = pa.table([lead, x, tail, _row_ids(n)], names=["lead", "x", "tail", "rid"])
    for N in (7, 48):
        check_placement(ctx, alone, [0], N, {0: (fmt, None)}, [fmt], f"key {fmt!r} alone")
        check_placement(ctx, middle, [0, 1, 2], N, {1: (fmt, None)}, ["l", fmt, "u"], f"key {fmt!r} in the middle")


def _indices(index_fmt, n, m, rnd, lo=0):
    t = FIXED[index_fmt]
    return pa.array([None if i % 6 == 4 else rnd.randrange(lo, m) for i in range(n)], type=t)


def check_dictionary_key(ctx, index_fmt, value_fmt, n=200):
    """Dictionary<K, V>: (a) null indices and null values, N = 7; (b) values sliced at offset 2 without nulls, N = 48;
    (c) for the value types of DICT_MIDDLE_VALUES, the middle key of [Int64, Dictionary<K, V>, Utf8]."""
    rnd = random.Random(_seed(index_fmt, value_fmt))
    m = 200 if index_fmt == "C" else 20  # UInt8 indices reach 128..199
    what = f"Dictionary<{index_fmt!r}, {value_fmt!r}>"
    fm = {0: (index_fmt, value_fmt)}
    d = pa.DictionaryArray.from_arrays(_indices(index_fmt, n, m, rnd), values(value_fmt, m, rnd))
    check_placement(ctx, pa.table([d, _row_ids(n)], names=["x", "rid"]), [0], 7, fm, [value_fmt], what + " with nulls")
    sliced = values(value_fmt, m + 2, rnd, nulls=False).slice(2)
    d2 = pa.DictionaryArray.from_arrays(_indices(index_fmt, n, m, rnd), sliced)
    check_placement(ctx, pa.table([d2, _row_ids(n)], names=["x", "rid"]), [0], 48, fm, [value_fmt], what + " over sliced values")
    if value_fmt in DICT_MIDDLE_VALUES:
        lead, tail = _lead_and_tail(n, rnd)
        middle = pa.table([lead, d, tail, _row_ids(n)], names=["lead", "x", "tail", "rid"])
        for N in (7, 48):
            check_placement(ctx, middle, [0, 1, 2], N, {1: (index_fmt, value_fmt)}, ["l", value_fmt, "u"], what + " in the middle")


def check_unsigned_past_signed_range(ctx, index_fmt, m, value_fmt, n=3000):
    """Dictionary<UInt8, V> of 256 values / Dictionary<UInt16, V> of 40 000 values, most rows at indices past the signed range."""
    rnd = random.Random(_seed(index_fmt, value_fmt, str(m)))
    idx = [None if i % 11 == 5 else (rnd.randrange(m // 2, m) if i % 4 else rnd.randrange(0, m)) for i in range(n)]
    idx[:2] = [m - 1, m // 2]
    d = pa.DictionaryArray.from_arrays(pa.array(idx, type=FIXED[index_fmt]), values(value_fmt, m, rnd))
    lead, tail = _lead_and_tail(n, rnd)
    table = pa.table([lead, d, tail, _row_ids(n)], names=["lead", "x", "tail", "rid"])
    what = f"Dictionary<{index_fmt!r}, {value_fmt!r}> of {m} values"
    for N in (7, 48):
        check_placement(ctx, table.select(["x", "rid"]), [0], N, {0: (index_fmt, value_fmt)}, [value_fmt], what, chunk_rows=1024)
        check_placement(ctx, table, [0, 1, 2], N, {1: (index_fmt, value_fmt)}, ["l", value_fmt, "u"], what + " in the middle", chunk_rows=1024)


BIG_DICTIONARIES = [("C", 256, "l"), ("C", 256, "u"), ("S", 40_000, "l"), ("S", 40_000, "tiD")]


def _id(fmt):
    return re.sub(r"[^A-Za-z0-9]", "_", fmt)


# ---- the cases, on the GPU -------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("fmt", KEY_FORMATS, ids=[_id(f) for f in KEY_FORMATS])
def test_every_key_format_alone_and_in_the_middle(ctx, fmt):
    check_key_format(ctx, fmt)


DICT_CASES = [(k, v) for k in INDEX_FORMATS for v in DICT_VALUE_FORMATS]


@pytest.mark.gpu
@pytest.mark.parametrize("index_fmt,value_fmt", DICT_CASES, ids=[f"{INDEX_FORMATS[k]}-{_id(v)}" for k, v in DICT_CASES])
def test_dictionary_keys(ctx, index_fmt, value_fmt):
    check_dictionary_key(ctx, index_fmt, value_fmt)


@pytest.mark.gpu
@pytest.mark.parametrize("index_fmt,m,value_fmt", BIG_DICTIONARIES, ids=[f"{INDEX_FORMATS[k]}-{m}-{_id(v)}" for k, m, v in BIG_DICTIONARIES])
def test_unsigned_indices_past_the_signed_range(ctx, index_fmt, m, value_fmt):
    check_unsigned_past_signed_range(ctx, index_fmt, m, value_fmt)


def check_sliced_values_with_nulls_are_refused(ctx):
    """Dictionary values sliced at an offset AND carrying nulls are refused (the re-based validity is not implemented)."""
    values_ = pa.array(["a", None, "b", "c", None, "d"]).slice(1)
    d = pa.DictionaryArray.from_arrays(pa.array([0, 1, 2, None, 4] * 20, type=pa.int32()), values_)
    with pytest.raises(RuntimeError, match="sliced dictionary values with nulls"):
        run_operator(ctx, pa.table([d, _row_ids(100)], names=["x", "rid"]), [0], 4, {})


@pytest.mark.gpu
def test_sliced_dictionary_values_with_nulls_are_refused(ctx):
    check_sliced_values_with_nulls_are_refused(ctx)


@pytest.mark.gpu
def test_device_partitioner_unsigned_indices_and_interval_values(ctx):
    """HashPartitioner.set_key_dictionary(..., unsigned_index=True): UInt8 / UInt16 indices past the signed range take the
    hash of the value they name; interval-typed values are refused (dfd_hash_columns_device hashes them as one integer)."""
    import datafusion_distributed_b200 as dfd

    for index_fmt, m in (("C", 256), ("S", 40_000)):
        rnd = random.Random(m)
        n = 20_000
        vals = values("u", m, rnd)
        idx = pa.array([None if i % 9 == 1 else rnd.randrange(m // 2, m) if i % 3 else rnd.randrange(m) for i in range(n)], type=FIXED[index_fmt])
        other = pa.array([rnd.getrandbits(40) for _ in range(n)], type=pa.int64())
        d = pa.DictionaryArray.from_arrays(idx, vals)
        cols = [dfd.DeviceColumn.from_arrow(ctx, idx), dfd.DeviceColumn.from_arrow(ctx, other)]
        for N in (7, 48):
            part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
            part.set_key_dictionary(0, vals, unsigned_index=True)
            assert np.array_equal(part.partition_ids(cols, n), orc.partition_ids([d], n, N)), (index_fmt, N)
            part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([1, 0], N))
            part.set_key_dictionary(1, vals, unsigned_index=True)
            dest = orc.partition_ids([other, d], n, N)
            assert np.array_equal(part.partition_ids(cols, n), dest), (index_fmt, N)
            outs, starts = part.partition(cols, n)  # the scatter with the same key
            got = outs[1].to_arrow(ctx, 0, n).to_numpy()
            for p in range(N):
                rows = np.flatnonzero(dest == p)
                assert starts[p + 1] - starts[p] == len(rows) and np.array_equal(got[starts[p]:starts[p + 1]], other.to_numpy()[rows]), (index_fmt, N, p)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    with pytest.raises(ValueError, match="interval"):
        part.set_key_dictionary(0, pa.array([pa.MonthDayNano([1, 2, 3]), None], type=pa.month_day_nano_interval()))


# ---- which formats the library accepts as keys (CPU) -----------------------------------------------------------------------

# flat formats the library refuses as keys (payload only, or not movable at all)
REFUSED_FORMATS = ["n", "Z", "w:1", "w:4", "w:16", "w:12", "d:76,0,256", "+l", "+L", "+s", "+m", "+w:4"]


def _repartition_supported(lib, fmt, dict_fmt=None):
    keep = []

    def node(f, name, dictionary=None):
        s = nv.ArrowSchemaStruct()
        s.format, s.name, s.flags = f.encode(), name, 2  # ARROW_FLAG_NULLABLE
        s.dictionary = C.addressof(dictionary) if dictionary is not None else None
        keep.append(s)
        return s

    key = node(fmt, b"x", node(dict_fmt, b"v") if dict_fmt else None)
    kids = (C.POINTER(nv.ArrowSchemaStruct) * 2)(C.pointer(key), C.pointer(node("l", b"rid")))
    top = node("+s", b"")
    top.n_children, top.children = 2, C.cast(kids, C.c_void_p)
    return lib.dfd_repartition_supported(C.byref(top), (C.c_int32 * 1)(0), 1) == 0


def test_every_key_type_the_library_accepts_has_a_case(built):
    """Ask dfd_repartition_supported about every candidate key format and Dictionary<K, V> combination: what it accepts must
    be exactly what this module runs on the GPU, so that a newly accepted key type cannot go untested."""
    lib = nv.lib()
    candidates = KEY_FORMATS + REFUSED_FORMATS
    accepted = {f for f in candidates if _repartition_supported(lib, f)}
    assert accepted == set(KEY_FORMATS), (sorted(accepted - set(KEY_FORMATS)), sorted(set(KEY_FORMATS) - accepted))
    index_candidates = list(INDEX_FORMATS) + ["b", "e", "f", "g", "u", "d:9,2,32", "tdD", "tiM"]
    accepted = {(k, v) for k in index_candidates for v in candidates if _repartition_supported(lib, k, v)}
    assert accepted == set(DICT_CASES), (sorted(accepted - set(DICT_CASES)), sorted(set(DICT_CASES) - accepted))
    assert set(DICT_MIDDLE_VALUES) <= set(DICT_VALUE_FORMATS) and {v for _, _, v in BIG_DICTIONARIES} <= set(DICT_VALUE_FORMATS)


# the bodies above, by name, for the CPU harness of the operator's host logic (tests/test_exec_cpu_harness.py)
HARNESS_CASES = ([("check_key_format", (f,)) for f in KEY_FORMATS] +
                 [("check_dictionary_key", (k, v)) for k, v in DICT_CASES] +
                 [("check_unsigned_past_signed_range", case) for case in BIG_DICTIONARIES] +
                 [("check_sliced_values_with_nulls_are_refused", ())])
