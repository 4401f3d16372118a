"""oracle/oracle.py — ctypes binding of the C CPU ORACLE (oracle/df_oracle.c).

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import this module.
PARITY STATUS: "parity unpinned" — see oracle/df_oracle.h.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libdf_oracle.so")
_SRC = os.path.join(_HERE, "df_oracle.c")

ORC_FIXED, ORC_BOOL, ORC_UTF8, ORC_LARGE_UTF8, ORC_BINARY, ORC_INTERVAL_DAY_TIME, ORC_INTERVAL_MONTH_DAY_NANO = 0, 1, 2, 3, 4, 5, 6


class OrcState(C.Structure):
    _fields_ = [("k0", C.c_uint64), ("k1", C.c_uint64), ("k2", C.c_uint64), ("k3", C.c_uint64)]


class OrcColumn(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("width", C.c_int32),
        ("values", C.c_void_p),
        ("offsets", C.c_void_p),
        ("validity", C.c_void_p),
        ("offset", C.c_int64),
    ]


def build(force: bool = False) -> str:
    """gcc-compile the C restatement (building the checker is not using it)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(
        os.path.getmtime(_SRC), os.path.getmtime(os.path.join(_HERE, "df_oracle.h"))
    ):
        subprocess.check_call(
            ["gcc", "-O2", "-fPIC", "-shared", "-pthread", _SRC, "-o", _SO], cwd=_HERE
        )
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        L = _lib
        L.orc_state_with_seeds.restype = OrcState
        L.orc_state_with_seeds.argtypes = [C.c_uint64] * 4
        L.orc_repartition_random_state.restype = OrcState
        L.orc_hash_one_u64.restype = C.c_uint64
        L.orc_hash_one_u64.argtypes = [C.POINTER(OrcState), C.c_uint64]
        L.orc_hash_one_u128.restype = C.c_uint64
        L.orc_hash_one_u128.argtypes = [C.POINTER(OrcState), C.c_uint64, C.c_uint64]
        L.orc_hash_one_str.restype = C.c_uint64
        L.orc_hash_one_str.argtypes = [C.POINTER(OrcState), C.c_char_p, C.c_size_t]
        L.orc_hash_one_bytes.restype = C.c_uint64
        L.orc_hash_one_bytes.argtypes = [C.POINTER(OrcState), C.c_char_p, C.c_size_t]
        L.orc_combine_hashes.restype = C.c_uint64
        L.orc_combine_hashes.argtypes = [C.c_uint64, C.c_uint64]
        L.orc_create_hashes.restype = None
        L.orc_create_hashes.argtypes = [C.POINTER(OrcColumn), C.c_int, C.c_int64, C.POINTER(OrcState), C.c_void_p]
        L.orc_partition_indices.restype = None
        L.orc_partition_indices.argtypes = [C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_partition_ids.restype = None
        L.orc_partition_ids.argtypes = [C.POINTER(OrcColumn), C.c_int, C.c_int64, C.c_uint32, C.c_void_p]
        L.orc_repartition_table.restype = C.c_int
        L.orc_repartition_table.argtypes = [
            C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int, C.c_int64, C.POINTER(C.c_int32), C.c_int,
            C.c_uint32, C.c_int64, C.c_int, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p,
        ]
        L.orc_pool_create.restype = C.c_void_p
        L.orc_pool_create.argtypes = [C.c_int]
        L.orc_pool_destroy.restype = None
        L.orc_pool_destroy.argtypes = [C.c_void_p]
        L.orc_repartition_stream.restype = C.c_int
        L.orc_repartition_stream.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_int, C.c_int64, C.POINTER(C.c_int32),
                                             C.c_int, C.c_uint32, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]
    return _lib


class WorkerPool:
    """Persistent CPU worker pool for the timed reference arm (`orc_repartition_stream`)."""

    def __init__(self, n_threads: int):
        self.n_threads = n_threads
        self._h = lib().orc_pool_create(n_threads)

    def close(self):
        if self._h:
            lib().orc_pool_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def repartition(self, columns, key_cols, num_partitions: int, batch_size: int = 8192, use_threads: int = 0):
        """RepartitionExec(Hash) + LimitedBatchCoalescer over the whole table; returns (counts[N], output batches)."""
        n_rows = columns[0].shape[0]
        n_cols = len(columns)
        ptrs = (C.c_void_p * n_cols)(*[c.ctypes.data for c in columns])
        widths = (C.c_int32 * n_cols)(*[c.dtype.itemsize for c in columns])
        keys = (C.c_int32 * len(key_cols))(*key_cols)
        counts = np.zeros(num_partitions, dtype=np.int64)
        batches, cs = C.c_int64(), C.c_uint64()
        rc = lib().orc_repartition_stream(self._h, ptrs, widths, n_cols, n_rows, keys, len(key_cols), num_partitions, batch_size,
                                          use_threads, counts.ctypes.data, C.byref(batches), C.byref(cs))
        if rc != 0:
            raise MemoryError("orc_repartition_stream failed")
        return counts, batches.value


def _state(seeds=(0, 0, 0, 0)) -> OrcState:
    return lib().orc_state_with_seeds(*[C.c_uint64(s) for s in seeds])


def hash_one_int(x: int, width: int = 8, seeds=(0, 0, 0, 0)) -> int:
    st = _state(seeds)
    x &= (1 << (8 * width)) - 1
    if width == 16:
        return lib().orc_hash_one_u128(C.byref(st), x & ((1 << 64) - 1), x >> 64)
    return lib().orc_hash_one_u64(C.byref(st), x)


def hash_one_str(s: bytes, seeds=(0, 0, 0, 0)) -> int:
    st = _state(seeds)
    return lib().orc_hash_one_str(C.byref(st), s, len(s))


def hash_one_bytes(s: bytes, seeds=(0, 0, 0, 0)) -> int:
    st = _state(seeds)
    return lib().orc_hash_one_bytes(C.byref(st), s, len(s))


def combine_hashes(l: int, r: int) -> int:
    return lib().orc_combine_hashes(l, r)


class _Cols:
    """Keeps the numpy/pyarrow buffers alive next to the C descriptors."""

    def __init__(self, columns):
        self.keep = []
        self.n = len(columns)
        self.arr = (OrcColumn * self.n)()
        for i, col in enumerate(columns):
            self._fill(self.arr[i], col)

    def _fill(self, d: OrcColumn, col):
        import pyarrow as pa

        if isinstance(col, tuple):
            # ("interval_day_time" | "interval_month_day_nano", raw little-endian values as a uint8 array[, valid: bool per row])
            tag, raw, *valid = col
            raw = np.ascontiguousarray(raw, dtype=np.uint8)
            self.keep.append(raw)
            d.kind = ORC_INTERVAL_DAY_TIME if tag == "interval_day_time" else ORC_INTERVAL_MONTH_DAY_NANO
            d.width = 8 if tag == "interval_day_time" else 16
            d.values, d.offsets, d.validity, d.offset = raw.ctypes.data, None, None, 0
            if valid and valid[0] is not None:
                bits = np.packbits(np.asarray(valid[0], dtype=bool), bitorder="little")
                self.keep.append(bits)
                d.validity = bits.ctypes.data
            return
        if isinstance(col, np.ndarray):
            col = np.ascontiguousarray(col)
            self.keep.append(col)
            d.kind, d.width, d.values, d.offsets, d.validity, d.offset = (
                ORC_FIXED, col.dtype.itemsize, col.ctypes.data, None, None, 0)
            return
        if isinstance(col, pa.ChunkedArray):
            col = col.combine_chunks()
        if isinstance(col, pa.DictionaryArray):
            # DataFusion hash_dictionary: a row hashes as its dictionary VALUE (null index / null value: skipped) — exactly the
            # hash of the decoded array
            col = col.dictionary_decode()
        if pa.types.is_string_view(col.type) if hasattr(pa.types, "is_string_view") else False:
            col = col.cast(pa.string())  # Utf8View hashes over the string bytes exactly like Utf8
        assert isinstance(col, pa.Array), type(col)
        self.keep.append(col)
        bufs = col.buffers()
        d.validity = bufs[0].address if (bufs[0] is not None and col.null_count > 0) else None
        d.offset = col.offset
        t = col.type
        if pa.types.is_boolean(t):
            d.kind, d.width, d.values, d.offsets = ORC_BOOL, 0, bufs[1].address, None
        elif pa.types.is_string(t) or pa.types.is_binary(t):
            d.kind = ORC_UTF8 if pa.types.is_string(t) else ORC_BINARY
            d.width, d.offsets = 0, bufs[1].address
            d.values = bufs[2].address if bufs[2] is not None else None
        elif pa.types.is_interval(t):  # month_day_nano_interval: 16 B {months: i32, days: i32, nanoseconds: i64}
            d.kind, d.width, d.values, d.offsets = ORC_INTERVAL_MONTH_DAY_NANO, 16, bufs[1].address, None
        elif pa.types.is_large_string(t):
            d.kind, d.width, d.offsets = ORC_LARGE_UTF8, 0, bufs[1].address
            d.values = bufs[2].address if bufs[2] is not None else None
        else:
            d.kind, d.width, d.values, d.offsets = ORC_FIXED, t.bit_width // 8, bufs[1].address, None


def create_hashes(columns, n_rows: int, seeds=(0, 0, 0, 0)) -> np.ndarray:
    """datafusion-common create_hashes over numpy arrays / pyarrow arrays."""
    cols = _Cols(columns)
    st = _state(seeds)
    h = np.zeros(n_rows, dtype=np.uint64)
    lib().orc_create_hashes(cols.arr, cols.n, n_rows, C.byref(st), h.ctypes.data)
    return h


def partition_ids(key_columns, n_rows: int, num_partitions: int) -> np.ndarray:
    """dest[i] = create_hashes(keys)[i] % num_partitions (REPARTITION_RANDOM_STATE)."""
    cols = _Cols(key_columns)
    dest = np.empty(n_rows, dtype=np.uint32)
    lib().orc_partition_ids(cols.arr, cols.n, n_rows, num_partitions, dest.ctypes.data)
    return dest


def partition_indices(hashes: np.ndarray, num_partitions: int):
    """BatchPartitioner Hash arm: (counts[N], indices[n] grouped by destination, starts[N+1])."""
    hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
    n = hashes.shape[0]
    counts = np.zeros(num_partitions, dtype=np.int64)
    indices = np.empty(n, dtype=np.uint32)
    starts = np.zeros(num_partitions + 1, dtype=np.int64)
    lib().orc_partition_indices(hashes.ctypes.data, n, num_partitions, counts.ctypes.data,
                                indices.ctypes.data, starts.ctypes.data)
    return counts, indices, starts


def repartition_table(columns, key_cols, num_partitions: int, batch_size: int = 8192,
                      n_threads: int = 1, materialize: bool = True):
    """RepartitionExec(Hash(keys, N)) restatement over fixed-width numpy columns.

    Returns (out_columns | None, counts[N], starts[N+1]).  With n_threads == 1
    the per-destination order is exactly the input order (invariant iii)."""
    columns = [np.ascontiguousarray(c) for c in columns]
    n_rows = columns[0].shape[0]
    n_cols = len(columns)
    ptrs = (C.c_void_p * n_cols)(*[c.ctypes.data for c in columns])
    widths = (C.c_int32 * n_cols)(*[c.dtype.itemsize for c in columns])
    keys = (C.c_int32 * len(key_cols))(*key_cols)
    counts = np.zeros(num_partitions, dtype=np.int64)
    starts = np.zeros(num_partitions + 1, dtype=np.int64)
    outs = None
    out_ptrs = None
    if materialize:
        outs = [np.empty_like(c) for c in columns]
        out_ptrs = (C.c_void_p * n_cols)(*[c.ctypes.data for c in outs])
    rc = lib().orc_repartition_table(ptrs, widths, n_cols, n_rows, keys, len(key_cols), num_partitions,
                                     batch_size, n_threads, out_ptrs, counts.ctypes.data, starts.ctypes.data)
    if rc != 0:
        raise MemoryError("orc_repartition_table failed")
    return outs, counts, starts
