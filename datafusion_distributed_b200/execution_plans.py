"""Host mirror of the reference's operator surface for the shuffle path.

`RepartitionExec` ≙ DataFusion's `RepartitionExec(Partitioning::Hash)` as the
reference builds it (src/execution_plans/network_shuffle.rs:126-134) and runs
it on every producer task (src/worker/impl_execute_task.rs:77-86):
`execute(partition)` returns the stream of that destination's record batches.
Host Arrow batches in, host Arrow batches out; the work happens on the GPU.  Batches may also be device-resident on
either side (`push_device_batch` / `run_device`, `device_output=True` + `execute_device`).
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Optional

from . import _native as nv
from .device import WorkerContext
from .partitioner import Partitioning


class PinnedTable:
    """Column buffers in pinned host memory (what an Arrow allocator plugged into
    `dfd_host_alloc` gives the upstream operator), exposed as pyarrow arrays."""

    def __init__(self, ctx: WorkerContext, n_rows: int, dtypes):
        import numpy as np

        self.ctx = ctx
        self.n_rows = n_rows
        self._ptrs = []
        self.columns = []
        ctx._adopt(self)
        for dt in dtypes:
            dt = np.dtype(dt)
            nbytes = max(n_rows * dt.itemsize, 16)
            p = C.c_void_p()
            nv.check(nv.lib().dfd_host_alloc(ctx.handle, nbytes, C.byref(p)))
            self._ptrs.append(p)
            buf = (C.c_char * nbytes).from_address(p.value)
            self.columns.append(np.frombuffer(buf, dtype=dt, count=n_rows))

    def record_batches(self, names, batch_rows: int):
        """Zero-copy pyarrow RecordBatches over the pinned buffers."""
        import pyarrow as pa

        out = []
        for lo in range(0, self.n_rows, batch_rows):
            hi = min(lo + batch_rows, self.n_rows)
            arrays = []
            for col in self.columns:
                t = pa.from_numpy_dtype(col.dtype)
                buf = pa.foreign_buffer(col.ctypes.data + lo * col.dtype.itemsize, (hi - lo) * col.dtype.itemsize, base=self)
                arrays.append(pa.Array.from_buffers(t, hi - lo, [None, buf]))
            out.append(pa.RecordBatch.from_arrays(arrays, names=list(names)))
        return out

    def close(self):
        for p in self._ptrs:
            if p and self.ctx.handle:
                nv.lib().dfd_host_free(self.ctx.handle, p)
        self._ptrs = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceBatchStream:
    """Iterator over an Arrow C Device stream (`struct ArrowDeviceArrayStream`) of one destination's batches.  Each item is an
    owned `ArrowDeviceArrayStruct`; it is released when the next one is asked for (or on `close`), so a consumer finishes
    its device reads of a batch (after waiting on its `sync_event`) before it moves on."""

    def __init__(self, stream: "nv.ArrowDeviceArrayStreamStruct"):
        self._cs = stream
        self._last = None

    @property
    def device_type(self) -> int:
        return self._cs.device_type

    @property
    def schema(self):
        import pyarrow as pa

        out = nv.ArrowSchemaStruct()
        rc = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)(self._cs.get_schema)(C.addressof(self._cs), C.addressof(out))
        if rc:
            raise OSError(rc, "get_schema failed")
        return pa.Schema._import_from_c(C.addressof(out))

    def __iter__(self):
        return self

    def _release_last(self):
        if self._last is not None and self._last.array.release:
            C.CFUNCTYPE(None, C.c_void_p)(self._last.array.release)(C.addressof(self._last.array))
        self._last = None

    def __next__(self):
        self._release_last()
        if not self._cs.release:
            raise StopIteration
        out = nv.ArrowDeviceArrayStruct()
        rc = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)(self._cs.get_next)(C.addressof(self._cs), C.addressof(out))
        if rc:
            msg = C.CFUNCTYPE(C.c_char_p, C.c_void_p)(self._cs.get_last_error)(C.addressof(self._cs))
            text = msg.decode("utf-8", "replace") if msg else "unknown"
            self.close()
            raise OSError(rc, text)
        if not out.array.release:
            self.close()
            raise StopIteration
        self._last = out
        return out

    def close(self):
        self._release_last()
        if self._cs.release:
            C.CFUNCTYPE(None, C.c_void_p)(self._cs.release)(C.addressof(self._cs))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RepartitionExec:
    """`RepartitionExec::try_new(input, Partitioning::Hash(exprs, n))` on one GPU worker."""

    def __init__(self, ctx: WorkerContext, schema, partitioning: Partitioning, chunk_rows: int = 0,
                 pipeline_depth: int = 0, pinned_pool_chunks: int = 0, max_pinned_chunks: int = 0, device_output: bool = False):
        self.ctx = ctx
        self.schema = schema
        self.partitioning = partitioning
        cs = nv.ArrowSchemaStruct()
        schema._export_to_c(C.addressof(cs))
        keys = (C.c_int32 * len(partitioning.key_cols))(*partitioning.key_cols)
        opts = nv.DfdExecOptions(chunk_rows, pipeline_depth, pinned_pool_chunks, max_pinned_chunks, 1 if device_output else 0)
        self._h = C.c_void_p()
        try:
            nv.check(nv.lib().dfd_repartition_exec_create(ctx.handle, C.byref(cs), keys, len(partitioning.key_cols),
                                                          partitioning.partition_count, C.byref(opts), C.byref(self._h)))
        finally:
            if cs.release:  # the operator only borrows the schema
                C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))
        ctx._adopt(self)

    def name(self) -> str:
        return "RepartitionExec"

    def output_partitioning(self) -> Partitioning:
        return self.partitioning

    def push_batch(self, batch):
        """Feed one input RecordBatch (≙ one item of the child plan's stream)."""
        ca = nv.ArrowArrayStruct()
        batch._export_to_c(C.addressof(ca))
        nv.check(nv.lib().dfd_repartition_exec_push(self._h, C.byref(ca)))

    def push_device_batch(self, device_array):
        """Feed one DEVICE-resident input batch: a pointer (int or ctypes) to a `struct ArrowDeviceArray` on this worker's
        GPU.  Ownership of its `array` moves to the operator (its release is called once the device work that reads it is
        done).  An operator takes either host batches (`push_batch` / `run`) or device batches, never both."""
        addr = device_array if isinstance(device_array, int) else C.addressof(device_array)
        nv.check(nv.lib().dfd_repartition_exec_push_device(self._h, C.cast(C.c_void_p(addr), C.POINTER(nv.ArrowDeviceArrayStruct))))

    def finish(self):
        nv.check(nv.lib().dfd_repartition_exec_finish(self._h))

    def abort(self, message: str):
        """The producer's input failed: every partition stream ends with an error carrying `message`
        (≙ RepartitionExec forwarding an input error to all of its output partitions)."""
        nv.check(nv.lib().dfd_repartition_exec_abort(self._h, message.encode()))

    def run(self, reader):
        """Pull a pyarrow RecordBatchReader (≙ child.execute()) to exhaustion."""
        cs = nv.ArrowArrayStreamStruct()
        reader._export_to_c(C.addressof(cs))
        nv.check(nv.lib().dfd_repartition_exec_run(self._h, C.byref(cs)))

    def execute(self, partition: int):
        """≙ ExecutionPlan::execute(partition, ctx): a RecordBatchReader of that destination."""
        import pyarrow as pa

        cs = nv.ArrowArrayStreamStruct()
        nv.check(nv.lib().dfd_repartition_exec_execute(self._h, partition, C.byref(cs)))
        return pa.RecordBatchReader._import_from_c(C.addressof(cs))

    def run_device(self, device_stream):
        """Pull an Arrow C Device stream (a pointer, int or ctypes, to a `struct ArrowDeviceArrayStream` of CUDA batches on this
        worker's GPU) to exhaustion, then finish.  The stream is released, whatever the outcome."""
        addr = device_stream if isinstance(device_stream, int) else C.addressof(device_stream)
        nv.check(nv.lib().dfd_repartition_exec_run_device(self._h, C.cast(C.c_void_p(addr), C.POINTER(nv.ArrowDeviceArrayStreamStruct))))

    def execute_device(self, partition: int) -> DeviceBatchStream:
        """`execute(partition)` of an operator created with `device_output=True`: that destination's batches as
        `ArrowDeviceArrayStruct`s whose buffers are in this worker's GPU memory."""
        cs = nv.ArrowDeviceArrayStreamStruct()
        nv.check(nv.lib().dfd_repartition_exec_execute_device(self._h, partition, C.byref(cs)))
        return DeviceBatchStream(cs)

    def stats(self) -> dict:
        st = nv.DfdExecStats()
        nv.check(nv.lib().dfd_repartition_exec_stats(self._h, C.byref(st)))
        return {k: getattr(st, k) for k, _ in st._fields_}

    def close(self):
        if self._h and self.ctx.handle:
            nv.lib().dfd_repartition_exec_destroy(self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
