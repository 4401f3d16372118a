"""Test helper: a pyarrow RecordBatch as a DEVICE-resident Arrow C Device Data Interface batch (`struct ArrowDeviceArray`).

Every buffer of the batch — of its columns, their children, dictionaries and list children — is copied into memory
obtained from `alloc` (CUDA memory through torch on the GPU; host memory for the CPU harness, whose stand-in runtime treats
host pointers as device pointers).  The ArrowArray tree itself is built in ctypes (host memory, as the interface
specifies), with a release callback that drops the copies and counts its calls."""
import ctypes as C
import itertools

import pyarrow as pa

from datafusion_distributed_b200 import _native as nv

ARROW_DEVICE_CPU, ARROW_DEVICE_CUDA = 1, 2


def torch_alloc(data, stream=None):
    """Device copy of `data` (bytes-like) -> (pointer, owner).  With `stream`, the copy is enqueued there from pinned memory
    and the caller synchronises through an event; otherwise it is complete on return."""
    import torch

    n = len(data)
    dev = torch.empty(max(n, 1) + 64, dtype=torch.uint8, device="cuda")
    if n:
        src = torch.frombuffer(bytearray(data), dtype=torch.uint8)
        if stream is None:
            dev[:n].copy_(src)
        else:
            pinned = src.pin_memory()
            with torch.cuda.stream(stream):
                dev[:n].copy_(pinned, non_blocking=True)
            return dev.data_ptr(), (dev, pinned)
    return dev.data_ptr(), dev


def host_alloc(data, stream=None):
    """The CPU harness's 'device' memory: host memory."""
    n = len(data)
    buf = C.create_string_buffer(max(n, 1) + 64)
    if n:
        C.memmove(buf, bytes(data), n)
    return C.addressof(buf), buf


ALLOC = torch_alloc  # (the CPU harness swaps in host_alloc)

_RELEASE_T = C.CFUNCTYPE(None, C.POINTER(nv.ArrowArrayStruct))
_LIVE = {}
_KEYS = itertools.count(1)
RELEASED = []  # private_data keys of the batches whose release has run, in call order


@_RELEASE_T
def _release(arr):
    key = arr.contents.private_data
    RELEASED.append(key)
    _LIVE.pop(key, None)  # (drops the device copies and the ctypes tree)
    arr.contents.release = None


class DeviceBatch:
    """Owner of one device-resident batch; `.device_array` is the ArrowDeviceArray to push, `.key` its release id."""

    def __init__(self, batch, null_count_unknown=False, alloc=None, stream=None, device_id=0, device_type=ARROW_DEVICE_CUDA):
        self._alloc = alloc or ALLOC
        self._stream = stream
        self._unknown = null_count_unknown
        self._keep = []
        self.key = next(_KEYS)
        cols = [self._array(c) for c in batch.columns]
        kids = (C.POINTER(nv.ArrowArrayStruct) * len(cols))(*[C.pointer(c) for c in cols])
        bufs = (C.c_void_p * 1)(None)
        self._keep += [cols, kids, bufs]
        self.device_array = nv.ArrowDeviceArrayStruct()
        a = self.device_array.array
        a.length, a.null_count, a.offset, a.n_buffers, a.n_children = batch.num_rows, 0, 0, 1, len(cols)
        a.buffers = C.cast(bufs, C.c_void_p)
        a.children = C.cast(kids, C.c_void_p)
        a.release = C.cast(_release, C.c_void_p)
        a.private_data = self.key
        self.device_array.device_id = device_id
        self.device_array.device_type = device_type
        self.device_array.sync_event = None
        _LIVE[self.key] = self._keep

    def _copy(self, buf, nbytes=None):
        if buf is None:
            return None
        data = memoryview(buf)[: buf.size if nbytes is None else nbytes]
        ptr, owner = self._alloc(data, self._stream) if self._stream is not None else self._alloc(data)
        self._keep.append(owner)
        return ptr

    def _array(self, arr):
        t = arr.type
        out = nv.ArrowArrayStruct()
        children, dictionary = [], None
        if pa.types.is_dictionary(t):
            own = arr.buffers()[:2]
            dictionary = self._array(arr.dictionary)
        elif pa.types.is_list(t):
            own = arr.buffers()[:2]
            children = [self._array(arr.values)]
        elif pa.types.is_string_view(t) or pa.types.is_binary_view(t):
            own = arr.buffers()
            sizes = pa.py_buffer(b"".join(b.size.to_bytes(8, "little") for b in own[2:]))
            own = own + [sizes]  # the variadic buffer sizes (also on the device, as the interface says)
        else:
            own = arr.buffers()
        ptrs = [self._copy(b) for b in own]
        bufs = (C.c_void_p * len(ptrs))(*ptrs)
        out.length, out.offset, out.n_buffers = len(arr), arr.offset, len(ptrs)
        out.null_count = -1 if (self._unknown and arr.null_count) else arr.null_count
        out.buffers = C.cast(bufs, C.c_void_p)
        if children:
            kids = (C.POINTER(nv.ArrowArrayStruct) * len(children))(*[C.pointer(c) for c in children])
            out.n_children, out.children = len(children), C.cast(kids, C.c_void_p)
            self._keep.append(kids)
        if dictionary is not None:
            out.dictionary = C.cast(C.pointer(dictionary), C.c_void_p)
        out.release = C.cast(_child_release, C.c_void_p)
        self._keep += [out, bufs, children, dictionary]
        return out


@_RELEASE_T
def _child_release(arr):
    arr.contents.release = None


def live_batches():
    """Keys of the device batches built and not yet released."""
    return set(_LIVE)
