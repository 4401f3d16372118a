"""ctypes binding of the C ABI declared in include/dfd_b200.h.

This is the same binding a Rust `extern "C"` block would make (INTEGRATION.md);
Python is only the test/bench host.  There is no CPU fallback: if the shared
library is missing or CUDA is unavailable every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DFD_LIB_TAG selects a tuning-sweep build (_lib/libdfd_b200_<tag>.so, see build.py); default = the product library
_TAG = os.environ.get("DFD_LIB_TAG", "")
LIB_PATH = os.path.join(_HERE, "_lib", f"libdfd_b200{('_' + _TAG) if _TAG else ''}.so")

DFD_OK = 0
STATUS = {
    0: "DFD_OK", 1: "DFD_ERR_INVALID_ARGUMENT", 2: "DFD_ERR_OOM", 3: "DFD_ERR_CUDA", 4: "DFD_ERR_NCCL",
    5: "DFD_ERR_INTERNAL", 6: "DFD_ERR_UNSUPPORTED", 7: "DFD_ERR_CAPACITY",
}

COL_FIXED, COL_BOOL, COL_UTF8, COL_LARGE_UTF8, COL_BINARY = 0, 1, 2, 3, 4
EXCHANGE_NCCL, EXCHANGE_FUSED = 0, 1
ROUTE_SHUFFLE, ROUTE_COALESCE, ROUTE_BROADCAST = 0, 1, 2
AGG_SUM_I64, AGG_SUM_F64, AGG_MIN_I64, AGG_MAX_I64, AGG_SUM_I128, AGG_MIN_F64, AGG_MAX_F64 = 0, 1, 2, 3, 4, 5, 6
KEY_HASH_PLAIN, KEY_HASH_INTERVAL_DAY_TIME, KEY_HASH_INTERVAL_MONTH_DAY_NANO = 0, 1, 2


class DfdError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"{STATUS.get(status, status)}: {message}")
        self.status = status
        self.message = message


class DfdColumn(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("width", C.c_int32),
        ("values", C.c_void_p),
        ("offsets", C.c_void_p),
        ("validity", C.c_void_p),
        ("offset", C.c_int64),
        ("values_bytes", C.c_int64),
    ]


class DfdMetrics(C.Structure):
    _fields_ = [
        ("calls", C.c_uint64),
        ("rows", C.c_uint64),
        ("bytes_in", C.c_uint64),
        ("bytes_out", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("hist_ms", C.c_double),
        ("scan_ms", C.c_double),
        ("scatter_ms", C.c_double),
        ("h2d_ms", C.c_double),
        ("d2h_ms", C.c_double),
        ("scatter_launches", C.c_uint64),
        ("onepass_reruns", C.c_uint64),
    ]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


class DfdExecOptions(C.Structure):
    _fields_ = [("chunk_rows", C.c_int64), ("pipeline_depth", C.c_int32), ("pinned_pool_chunks", C.c_int32),
                ("max_pinned_chunks", C.c_int32), ("reserved", C.c_int32)]


class DfdExecStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("rows_in", "rows_out", "bytes_h2d", "bytes_d2h", "pinned_chunks", "pinned_chunks_allocated",
                                          "pinned_chunks_reused", "ns_push", "ns_wait_d2h", "ns_wait_pool")]


class ArrowSchemaStruct(C.Structure):
    """struct ArrowSchema (Arrow C Data Interface), opaque storage for pyarrow's _export_to_c."""
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
                ("n_children", C.c_int64), ("children", C.c_void_p), ("dictionary", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArrayStruct(C.Structure):
    _fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                ("n_children", C.c_int64), ("buffers", C.c_void_p), ("children", C.c_void_p),
                ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArrayStreamStruct(C.Structure):
    _fields_ = [("get_schema", C.c_void_p), ("get_next", C.c_void_p), ("get_last_error", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowDeviceArrayStruct(C.Structure):
    _fields_ = [("array", ArrowArrayStruct), ("device_id", C.c_int64), ("device_type", C.c_int32), ("sync_event", C.c_void_p),
                ("reserved", C.c_int64 * 3)]


# name -> (restype, argtypes).  Every symbol include/dfd_b200.h declares.
_VP = C.c_void_p
SIGNATURES = {
    "dfd_abi_version": (C.c_int, []),
    "dfd_last_error": (C.c_char_p, []),
    "dfd_status_name": (C.c_char_p, [C.c_int]),
    "dfd_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "dfd_ctx_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "dfd_ctx_destroy": (None, [_VP]),
    "dfd_ctx_stream": (_VP, [_VP]),
    "dfd_ctx_synchronize": (C.c_int, [_VP]),
    "dfd_ctx_set_profiling": (C.c_int, [_VP, C.c_int]),
    "dfd_device_alloc": (C.c_int, [_VP, C.c_size_t, C.POINTER(_VP)]),
    "dfd_device_free": (C.c_int, [_VP, _VP]),
    "dfd_host_alloc": (C.c_int, [_VP, C.c_size_t, C.POINTER(_VP)]),
    "dfd_host_free": (C.c_int, [_VP, _VP]),
    "dfd_memcpy_h2d": (C.c_int, [_VP, _VP, _VP, C.c_size_t]),
    "dfd_memcpy_d2h": (C.c_int, [_VP, _VP, _VP, C.c_size_t]),
    "dfd_memset_device": (C.c_int, [_VP, _VP, C.c_int, C.c_size_t]),
    "dfd_flush_l2": (C.c_int, [_VP]),
    "dfd_timer_start": (C.c_int, [_VP]),
    "dfd_timer_stop": (C.c_int, [_VP, C.POINTER(C.c_float)]),
    "dfd_partitioner_create": (C.c_int, [_VP, C.c_uint32, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_uint64), C.POINTER(_VP)]),
    "dfd_partitioner_destroy": (None, [_VP]),
    "dfd_partitioner_num_partitions": (C.c_uint32, [_VP]),
    "dfd_partitioner_set_key_hash_mode": (C.c_int, [_VP, C.c_int, C.c_int]),
    "dfd_partitioner_set_key_dictionary": (C.c_int, [_VP, C.c_int, _VP, _VP, C.c_int]),
    "dfd_hash_columns_device": (C.c_int, [_VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.POINTER(C.c_uint64), _VP]),
    "dfd_partition_ids_device": (C.c_int, [_VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, _VP]),
    "dfd_partition_device": (C.c_int, [_VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.POINTER(DfdColumn), C.POINTER(C.c_int64)]),
    "dfd_partitioner_part_starts_device": (_VP, [_VP]),
    "dfd_partition_device_onepass": (C.c_int, [_VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.POINTER(DfdColumn), C.c_int64,
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "dfd_partitioner_collect": (C.c_int, [_VP, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "dfd_arrow_format_layout": (C.c_int, [C.c_char_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "dfd_schema_supported": (C.c_int, [C.POINTER(ArrowSchemaStruct)]),
    "dfd_repartition_supported": (C.c_int, [_VP, C.POINTER(C.c_int32), C.c_int]),
    "dfd_repartition_exec_create": (C.c_int, [_VP, C.POINTER(ArrowSchemaStruct), C.POINTER(C.c_int32), C.c_int, C.c_uint32,
                                              C.POINTER(DfdExecOptions), C.POINTER(_VP)]),
    "dfd_repartition_exec_destroy": (None, [_VP]),
    "dfd_repartition_exec_push": (C.c_int, [_VP, C.POINTER(ArrowArrayStruct)]),
    "dfd_repartition_exec_finish": (C.c_int, [_VP]),
    "dfd_repartition_exec_abort": (C.c_int, [_VP, C.c_char_p]),
    "dfd_repartition_exec_run": (C.c_int, [_VP, C.POINTER(ArrowArrayStreamStruct)]),
    "dfd_repartition_exec_execute": (C.c_int, [_VP, C.c_uint32, C.POINTER(ArrowArrayStreamStruct)]),
    "dfd_repartition_exec_stats": (C.c_int, [_VP, C.POINTER(DfdExecStats)]),
    "dfd_nccl_unique_id": (C.c_int, [_VP]),
    "dfd_exchange_create": (C.c_int, [_VP, C.c_int, C.c_int, _VP, C.POINTER(_VP)]),
    "dfd_exchange_destroy": (None, [_VP]),
    "dfd_exchange_rank": (C.c_int, [_VP]),
    "dfd_exchange_world": (C.c_int, [_VP]),
    "dfd_exchange_setup_window": (C.c_int, [_VP, C.c_size_t]),
    "dfd_exchange_plan": (C.c_int, [C.c_int, C.c_uint32, C.c_int, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_int64)]),
    "dfd_shuffle_device": (C.c_int, [_VP, _VP, C.c_int, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.c_uint32,
                                     C.POINTER(DfdColumn), C.c_int64, C.POINTER(C.c_int64)]),
    "dfd_shuffle_device_async": (C.c_int, [_VP, _VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.c_uint32, C.POINTER(DfdColumn)]),
    "dfd_exchange_wait": (C.c_int, [_VP, C.POINTER(C.c_int64)]),
    "dfd_shuffle_device_onepass": (C.c_int, [_VP, _VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.c_uint32, C.POINTER(DfdColumn)]),
    "dfd_exchange_collect": (C.c_int, [_VP, C.POINTER(DfdColumn), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "dfd_exchange_onepass_fallbacks": (C.c_uint64, [_VP]),
    "dfd_exchange_phase_ms": (C.c_int, [_VP, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "dfd_partial_reduce_device": (C.c_int, [_VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_int32), _VP,
                                            C.c_uint32, C.POINTER(DfdColumn), C.POINTER(C.c_int64), _VP]),
    "dfd_shuffle_stream_begin": (C.c_int, [_VP, _VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.c_uint32, C.POINTER(C.c_uint8), C.POINTER(_VP)]),
    "dfd_shuffle_stream_next": (C.c_int, [_VP, C.POINTER(DfdColumn), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "dfd_shuffle_stream_stats": (C.c_int, [_VP, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "dfd_shuffle_stream_end": (None, [_VP]),
    "dfd_coalesce_task_group": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "dfd_route_segment_source": (C.c_int, [C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_uint32, C.POINTER(C.c_int), C.POINTER(C.c_uint32),
                                           C.POINTER(C.c_uint32)]),
    "dfd_exchange_gather": (C.c_int, [_VP, C.c_int, C.POINTER(DfdColumn), C.c_int, C.POINTER(C.c_int64), C.c_uint32, C.c_int, C.POINTER(DfdColumn)]),
    "dfd_exchange_pending_segments": (C.c_uint32, [_VP]),
    "dfd_shuffle_host": (C.c_int, [_VP, _VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.c_uint32, C.c_int, C.POINTER(DfdColumn),
                                   C.c_int64, C.POINTER(C.c_int64)]),
    "dfd_exchange_stats": (C.c_int, [_VP, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "dfd_export_partition_device": (C.c_int, [_VP, C.POINTER(DfdColumn), C.c_int, C.c_int64, C.c_int64, C.POINTER(ArrowDeviceArrayStruct)]),
    "dfd_metrics_get": (C.c_int, [_VP, C.POINTER(DfdMetrics)]),
    "dfd_metrics_reset": (C.c_int, [_VP]),
}

_lib = None


def lib():
    """Load libdfd_b200.so (fails loudly if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback for the CUDA path)"
            )
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status: int):
    if status != DFD_OK:
        raise DfdError(status, lib().dfd_last_error().decode("utf-8", "replace"))
