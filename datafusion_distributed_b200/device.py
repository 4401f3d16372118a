"""Device-side handles for the host mirror: worker context, buffers, columns.

`WorkerContext` ≙ one reference `Worker` (src/worker/worker_service.rs:39-49)
pinned to one GPU.  Columns are described exactly like the C ABI's
`dfd_column` (Arrow buffers flattened); they can wrap torch CUDA tensors
(torch is only a device-memory provider here) or library-owned allocations
uploaded from pyarrow arrays.
"""
from __future__ import annotations

import ctypes as C
import weakref
from dataclasses import dataclass, field
from typing import Any, Optional, Sequence

import numpy as np

from . import _native as nv


class WorkerContext:
    """One GPU's streams + scratch.  No CPU fallback: raises if CUDA is absent."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        nv.check(nv.lib().dfd_ctx_create(device, C.byref(self._h)))
        self.device = device
        # native objects created on this context; they must be destroyed BEFORE the context
        self._children = weakref.WeakSet()

    def _adopt(self, child):
        self._children.add(child)

    @property
    def handle(self):
        return self._h

    def close(self):
        if self._h:
            for child in list(self._children):
                try:
                    child.close()
                except Exception:
                    pass
            nv.lib().dfd_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def synchronize(self):
        nv.check(nv.lib().dfd_ctx_synchronize(self._h))

    def set_profiling(self, on: bool):
        nv.check(nv.lib().dfd_ctx_set_profiling(self._h, 1 if on else 0))

    def flush_l2(self):
        nv.check(nv.lib().dfd_flush_l2(self._h))

    def timer_start(self):
        nv.check(nv.lib().dfd_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        nv.check(nv.lib().dfd_timer_stop(self._h, C.byref(ms)))
        return ms.value

    def metrics(self) -> dict:
        m = nv.DfdMetrics()
        nv.check(nv.lib().dfd_metrics_get(self._h, C.byref(m)))
        return m.as_dict()

    def reset_metrics(self):
        nv.check(nv.lib().dfd_metrics_reset(self._h))

    def stream_ptr(self) -> int:
        return nv.lib().dfd_ctx_stream(self._h) or 0

    # -- memory ----------------------------------------------------------
    def alloc(self, nbytes: int) -> "DeviceBuffer":
        return DeviceBuffer(self, nbytes)

    def upload(self, arr: np.ndarray) -> "DeviceBuffer":
        arr = np.ascontiguousarray(arr)
        buf = DeviceBuffer(self, max(arr.nbytes, 1))
        if arr.nbytes:
            nv.check(nv.lib().dfd_memcpy_h2d(self._h, buf.ptr, arr.ctypes.data, arr.nbytes))
        return buf

    def upload_raw(self, address: int, nbytes: int, pad_to: int = 4) -> "DeviceBuffer":
        cap = max((nbytes + pad_to - 1) // pad_to * pad_to, pad_to)
        buf = DeviceBuffer(self, cap)
        nv.check(nv.lib().dfd_memset_device(self._h, buf.ptr, 0, cap))
        if nbytes:
            nv.check(nv.lib().dfd_memcpy_h2d(self._h, buf.ptr, address, nbytes))
        return buf


class DeviceBuffer:
    def __init__(self, ctx: WorkerContext, nbytes: int):
        self.ctx = ctx
        self.nbytes = nbytes
        p = C.c_void_p()
        nv.check(nv.lib().dfd_device_alloc(ctx.handle, nbytes, C.byref(p)))
        self.ptr = p.value
        ctx._adopt(self)

    def close(self):
        if self.ptr and self.ctx.handle:
            nv.lib().dfd_device_free(self.ctx.handle, self.ptr)
        self.ptr = None

    def zero(self):
        nv.check(nv.lib().dfd_memset_device(self.ctx.handle, self.ptr, 0, self.nbytes))
        return self

    def download(self, dtype=np.uint8, count: Optional[int] = None) -> np.ndarray:
        dtype = np.dtype(dtype)
        n = self.nbytes // dtype.itemsize if count is None else count
        out = np.empty(n, dtype=dtype)
        if n:
            nv.check(nv.lib().dfd_memcpy_d2h(self.ctx.handle, out.ctypes.data, self.ptr, n * dtype.itemsize))
        return out

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class DeviceColumn:
    """One device-resident column == one `dfd_column`."""

    kind: int
    width: int
    values: int
    offsets: int = 0
    validity: int = 0
    offset: int = 0
    length: int = 0
    keep: Any = field(default=None, repr=False)  # owners of the memory
    arrow_type: Any = None
    values_bytes: int = 0  # var-width kinds: size (capacity for outputs) of `values`

    def as_c(self) -> nv.DfdColumn:
        return nv.DfdColumn(self.kind, self.width, self.values or None, self.offsets or None,
                            self.validity or None, self.offset, self.values_bytes)

    @staticmethod
    def from_torch(t, validity=None) -> "DeviceColumn":
        """Wrap a contiguous CUDA tensor (and optional uint8 bitmap tensor)."""
        assert t.is_cuda and t.is_contiguous()
        return DeviceColumn(nv.COL_FIXED, t.element_size(), t.data_ptr(), 0,
                            validity.data_ptr() if validity is not None else 0, 0, t.numel(), (t, validity))

    @staticmethod
    def from_arrow(ctx: WorkerContext, arr) -> "DeviceColumn":
        """Upload a host pyarrow Array's buffers as they are (offset preserved)."""
        import pyarrow as pa

        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        t = arr.type
        bufs = arr.buffers()
        keep = []
        validity = 0
        if bufs[0] is not None and arr.null_count > 0:
            vb = ctx.upload_raw(bufs[0].address, bufs[0].size)
            keep.append(vb)
            validity = vb.ptr
        if pa.types.is_boolean(t):
            b = ctx.upload_raw(bufs[1].address, bufs[1].size)
            keep.append(b)
            return DeviceColumn(nv.COL_BOOL, 0, b.ptr, 0, validity, arr.offset, len(arr), keep, t)
        if pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t):
            kind = nv.COL_UTF8 if pa.types.is_string(t) else (nv.COL_BINARY if pa.types.is_binary(t) else nv.COL_LARGE_UTF8)
            ob = ctx.upload_raw(bufs[1].address, bufs[1].size)
            db = ctx.upload_raw(bufs[2].address if bufs[2] is not None else 0, bufs[2].size if bufs[2] is not None else 0)
            keep += [ob, db]
            return DeviceColumn(kind, 0, db.ptr, ob.ptr, validity, arr.offset, len(arr), keep, t,
                                bufs[2].size if bufs[2] is not None else 0)
        if pa.types.is_fixed_size_list(t):
            # one FIXED column of n x (child width) bytes per row: the child's values from its first element on
            child = arr.values
            if child.null_count or not pa.types.is_primitive(child.type) or pa.types.is_boolean(child.type):
                raise ValueError(f"FixedSizeList column: the child must be a non-null fixed-width primitive, not {child.type}")
            cw = child.type.bit_width // 8
            cb = child.buffers()[1]
            b = ctx.upload_raw(cb.address + child.offset * cw, len(child) * cw)
            keep.append(b)
            return DeviceColumn(nv.COL_FIXED, t.list_size * cw, b.ptr, 0, validity, arr.offset, len(arr), keep, t)
        width = t.bit_width // 8
        b = ctx.upload_raw(bufs[1].address, bufs[1].size, pad_to=max(width, 4))
        keep.append(b)
        return DeviceColumn(nv.COL_FIXED, width, b.ptr, 0, validity, arr.offset, len(arr), keep, t)

    @staticmethod
    def empty_like(ctx: WorkerContext, col: "DeviceColumn", n_rows: int) -> "DeviceColumn":
        """Output column for dfd_partition_device (offset 0, zeroed bitmaps)."""
        keep = []
        validity = 0
        if col.validity:
            vb = ctx.alloc(max((n_rows + 31) // 32 * 4, 4)).zero()
            keep.append(vb)
            validity = vb.ptr
        if col.kind == nv.COL_BOOL:
            b = ctx.alloc(max((n_rows + 31) // 32 * 4, 4)).zero()
        elif col.kind == nv.COL_FIXED:
            b = ctx.alloc(max(n_rows * col.width, 16))
        else:  # variable width: offsets (n+1) + a byte buffer as large as the input's
            ow = 8 if col.kind == nv.COL_LARGE_UTF8 else 4
            ob = ctx.alloc((n_rows + 1) * ow)
            b = ctx.alloc(max(col.values_bytes, 16))
            keep += [ob, b]
            return DeviceColumn(col.kind, 0, b.ptr, ob.ptr, validity, 0, n_rows, keep, col.arrow_type, max(col.values_bytes, 16))
        keep.append(b)
        return DeviceColumn(col.kind, col.width, b.ptr, 0, validity, 0, n_rows, keep, col.arrow_type)

    def to_arrow(self, ctx: WorkerContext, start: int, stop: int):
        """Download rows [start, stop) of a (offset-0) column as a pyarrow Array."""
        import pyarrow as pa

        n = stop - start
        validity_buf = None
        null_count = 0
        if self.validity:
            nbytes = (self.length + 7) // 8
            vb = self.keep[0].download(np.uint8, nbytes)
            bits = np.unpackbits(vb, bitorder="little")[start:stop]
            null_count = int(n - bits.sum())
            validity_buf = pa.py_buffer(np.packbits(bits, bitorder="little").tobytes())
        if self.kind == nv.COL_BOOL:
            raw = self.keep[-1].download(np.uint8, (self.length + 7) // 8)
            bits = np.unpackbits(raw, bitorder="little")[start:stop]
            data = pa.py_buffer(np.packbits(bits, bitorder="little").tobytes())
            return pa.Array.from_buffers(pa.bool_(), n, [validity_buf, data], null_count=null_count)
        if self.kind == nv.COL_FIXED:
            raw = self.keep[-1].download(np.uint8, self.length * self.width)
            data = pa.py_buffer(raw[start * self.width: stop * self.width].tobytes())
            t = self.arrow_type
            if t is not None and pa.types.is_fixed_size_list(t):
                child = pa.Array.from_buffers(t.value_type, n * t.list_size, [None, data])
                return pa.Array.from_buffers(t, n, [validity_buf], null_count=null_count, children=[child])
            return pa.Array.from_buffers(t, n, [validity_buf, data], null_count=null_count)
        # variable width: rebase the offsets of rows [start, stop) to zero
        odt = np.int64 if self.kind == nv.COL_LARGE_UTF8 else np.int32
        off = self.keep[-2].download(odt, self.length + 1)[start:stop + 1]
        lo, hi = (int(off[0]), int(off[-1])) if n or len(off) else (0, 0)
        raw = self.keep[-1].download(np.uint8, max(hi, 1))
        data = pa.py_buffer(raw[lo:hi].tobytes())
        offs = pa.py_buffer((off - lo).astype(odt).tobytes())
        return pa.Array.from_buffers(self.arrow_type, n, [validity_buf, offs, data], null_count=null_count)


def columns_to_c(cols: Sequence[DeviceColumn]):
    arr = (nv.DfdColumn * len(cols))()
    for i, c in enumerate(cols):
        arr[i] = c.as_c()
    return arr
