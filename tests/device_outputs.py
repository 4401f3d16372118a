"""Test helper: a DEVICE-resident output batch (`struct ArrowDeviceArray` of dfd_repartition_exec_execute_device) as a pyarrow
RecordBatch in host memory.

Every buffer of the batch — of its columns, their dictionaries and list children — is copied to the host (after a wait on
the batch's `sync_event`), and the same ArrowArray tree, with the same offsets, lengths and null counts, is imported through
pyarrow's C data interface: exactly how the host-output stream's batches arrive, so the two can be compared buffer by buffer.
Buffer sizes follow from type, offset and length (string bytes from the last offset, view data from the variadic sizes).

`COPY` and `WAIT` are swappable: the library's D2H copy and cudaEventSynchronize on the GPU; memmove and nothing on the CPU
harness, whose stand-in runtime treats host pointers as device pointers."""
import ctypes as C
import itertools

import pyarrow as pa

from datafusion_distributed_b200 import _native as nv

ARROW_DEVICE_CUDA = 2


def gpu_copy(ctx):
    """copy(dst_address, device_pointer, nbytes) through dfd_memcpy_d2h of the worker context."""
    def copy(dst, src, n):
        nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, C.c_void_p(dst), C.c_void_p(src), n))
    return copy


def gpu_wait(sync_event):
    """Host wait (cudaEventSynchronize, through ctypes) on the cudaEvent_t that `sync_event` points to."""
    handle = C.c_void_p.from_address(sync_event).value
    for name in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = C.CDLL(name)
        except OSError:
            continue
        rt.cudaEventSynchronize.argtypes = [C.c_void_p]
        rc = rt.cudaEventSynchronize(handle)
        assert rc == 0, f"cudaEventSynchronize: {rc}"
        return
    raise OSError("no CUDA runtime library to wait on the batch's sync_event with")


def host_copy(dst, src, n):
    C.memmove(dst, src, n)


COPY, WAIT = None, gpu_wait  # (COPY is bound to a context by the test module; the CPU harness swaps in host_copy / no wait)

_RELEASE_T = C.CFUNCTYPE(None, C.POINTER(nv.ArrowArrayStruct))
_LIVE = {}
_KEYS = itertools.count(1)


@_RELEASE_T
def _release(arr):
    _LIVE.pop(arr.contents.private_data, None)
    arr.contents.release = None


@_RELEASE_T
def _child_release(arr):
    arr.contents.release = None


def _pointers(addr, n):
    return list((C.c_void_p * n).from_address(addr)) if n else []


def _fetch(ptr, nbytes, keep):
    """Host copy of nbytes at device pointer `ptr` -> its address (None for a NULL buffer)."""
    if ptr is None:
        return None
    buf = C.create_string_buffer(max(nbytes, 1) + 8)
    if nbytes:
        COPY(C.addressof(buf), ptr, nbytes)
    keep.append(buf)
    return C.addressof(buf)


def _array(src, t, keep):
    """Host copy of the device-resident ArrowArray `src` of pyarrow type `t` (same offset / length / null_count)."""
    n = src.offset + src.length
    dev = _pointers(src.buffers, src.n_buffers)
    host = [None] * len(dev)
    children, dictionary = [], None
    if len(dev) > 0:
        host[0] = _fetch(dev[0], (n + 7) // 8, keep)
    if pa.types.is_dictionary(t):
        host[1] = _fetch(dev[1], n * (t.index_type.bit_width // 8), keep)
        dictionary = _array(C.cast(src.dictionary, C.POINTER(nv.ArrowArrayStruct)).contents, t.value_type, keep)
    elif pa.types.is_list(t):
        host[1] = _fetch(dev[1], (n + 1) * 4, keep)
        kid = C.cast(src.children, C.POINTER(C.POINTER(nv.ArrowArrayStruct)))[0].contents
        children = [_array(kid, t.value_type, keep)]
    elif pa.types.is_string_view(t) or pa.types.is_binary_view(t):
        host[1] = _fetch(dev[1], n * 16, keep)
        n_data = len(dev) - 3
        host[-1] = _fetch(dev[-1], n_data * 8, keep)
        sizes = (C.c_int64 * n_data).from_address(host[-1]) if n_data else []
        for k in range(n_data):
            host[2 + k] = _fetch(dev[2 + k], sizes[k], keep)
    elif pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t) or pa.types.is_large_binary(t):
        wide = pa.types.is_large_string(t) or pa.types.is_large_binary(t)
        host[1] = _fetch(dev[1], (n + 1) * (8 if wide else 4), keep)
        last = ((C.c_int64 if wide else C.c_int32) * (n + 1)).from_address(host[1])[n]
        host[2] = _fetch(dev[2], last, keep)
    elif pa.types.is_boolean(t):
        host[1] = _fetch(dev[1], (n + 7) // 8, keep)
    else:
        host[1] = _fetch(dev[1], n * (t.bit_width // 8), keep)
    out = nv.ArrowArrayStruct()
    bufs = (C.c_void_p * max(len(host), 1))(*host)
    out.length, out.null_count, out.offset, out.n_buffers = src.length, src.null_count, src.offset, len(host)
    out.buffers = C.cast(bufs, C.c_void_p)
    if children:
        kids = (C.POINTER(nv.ArrowArrayStruct) * len(children))(*[C.pointer(c) for c in children])
        out.n_children, out.children = len(children), C.cast(kids, C.c_void_p)
        keep.append(kids)
    if dictionary is not None:
        out.dictionary = C.cast(C.pointer(dictionary), C.c_void_p)
    out.release = C.cast(_child_release, C.c_void_p)
    keep += [out, bufs, children, dictionary]
    return out


def to_host_batch(device_array, schema):
    """pyarrow RecordBatch with host copies of every buffer of `device_array` (an ArrowDeviceArrayStruct of `schema`)."""
    if WAIT is not None and device_array.sync_event:
        WAIT(device_array.sync_event)
    src = device_array.array
    assert src.n_children == len(schema) and src.offset == 0
    keep = []
    kids_in = C.cast(src.children, C.POINTER(C.POINTER(nv.ArrowArrayStruct)))
    cols = [_array(kids_in[i].contents, schema.field(i).type, keep) for i in range(len(schema))]
    kids = (C.POINTER(nv.ArrowArrayStruct) * max(len(cols), 1))(*[C.pointer(c) for c in cols])
    bufs = (C.c_void_p * 1)(None)
    top = nv.ArrowArrayStruct()
    top.length, top.null_count, top.offset, top.n_buffers, top.n_children = src.length, 0, 0, 1, len(cols)
    top.buffers, top.children = C.cast(bufs, C.c_void_p), C.cast(kids, C.c_void_p)
    top.release = C.cast(_release, C.c_void_p)
    top.private_data = next(_KEYS)
    keep += [cols, kids, bufs, top]
    _LIVE[top.private_data] = keep
    return pa.RecordBatch._import_from_c(C.addressof(top), schema)
