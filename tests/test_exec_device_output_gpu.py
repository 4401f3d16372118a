"""GPU tests of the host operator's DEVICE output (dfd_exec_options.device_output, dfd_repartition_exec_execute_device,
dfd_repartition_exec_run_device): the same record batches run host -> host (the reference), host -> device and
device -> device must give identical partition streams once every device buffer is copied to the host — the same batches,
batch boundaries, offsets, lengths, null counts, values (the bytes under null slots included), all 16 bytes of every view,
list offsets and children, dictionary values.  tests/test_exec_device_output_cpu_harness.py runs these bodies on the CPU
harness."""
import ctypes as C
import random
import threading
import time

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from tests import device_batches as DB
from tests import device_outputs as DO
from tests import test_exec_device_input_gpu as IN
from tests.test_exec_device_input_gpu import assert_same_streams, push_device
from tests.test_exec_gpu import reference_fixture_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    """A worker context of this module's own (as in the device-input module); the helper's copies go through it."""
    c = dfd.WorkerContext(0)
    DO.COPY = DO.gpu_copy(c)
    yield c
    DO.COPY = None
    c.close()


def host_streams(ex, N):
    return [list(ex.execute(p)) for p in range(N)]


def device_streams(ctx, ex, N):
    """Every partition's device stream, each batch checked and copied to the host before it is released."""
    out = []
    for p in range(N):
        stream = ex.execute_device(p)
        assert stream.device_type == DO.ARROW_DEVICE_CUDA
        schema, got = stream.schema, []
        for b in stream:
            assert b.sync_event and b.device_type == DO.ARROW_DEVICE_CUDA and b.device_id == getattr(ctx, "device", 0)
            got.append(DO.to_host_batch(b, schema))
        out.append(got)
    return out


def run_three(ctx, schema, batches, keys, N, null_count_unknown=False, **opts):
    """host -> host, host -> device, device -> device; asserts identical streams; returns the stats of the two device-output runs."""
    part = dfd.Partitioning.Hash(keys, N)
    hh = dfd.RepartitionExec(ctx, schema, part, **opts)
    for rb in batches:
        hh.push_batch(rb)
    hh.finish()
    want, hstats = host_streams(hh, N), hh.stats()
    hh.close()
    hd = dfd.RepartitionExec(ctx, schema, part, device_output=True, **opts)
    for rb in batches:
        hd.push_batch(rb)
    hd.finish()
    got, hdstats = device_streams(ctx, hd, N), hd.stats()
    hd.close()
    assert_same_streams(want, got)
    assert hdstats["bytes_d2h"] == 0 and hdstats["rows_out"] == hstats["rows_out"]
    dd = dfd.RepartitionExec(ctx, schema, part, device_output=True, **opts)
    pushed = [push_device(dd, rb, null_count_unknown=null_count_unknown) for rb in batches]
    dd.finish()
    got, ddstats = device_streams(ctx, dd, N), dd.stats()
    dd.close()
    assert_same_streams(want, got)
    assert not set(pushed) & DB.live_batches()  # every input batch released once its output batches are ...
    assert sorted(k for k in DB.RELEASED if k in set(pushed)) == sorted(pushed)  # ... exactly once
    assert ddstats["bytes_h2d"] == 0 and ddstats["rows_out"] == hstats["rows_out"] == sum(b.num_rows for b in batches)
    return hdstats, ddstats


@pytest.mark.parametrize("batch_rows,chunk_rows", [(8192, 0), (1024, 10_000), (100_000, 65_536)])
def test_fixed_width_batches_move_nothing_over_pcie(ctx, batch_rows, chunk_rows):
    """(k: Int64, v: Int64), Hash([k], 8), batches below, at and above a chunk.  Device in + device out: no byte crosses PCIe."""
    rng = np.random.Generator(np.random.PCG64(1))
    n = 300_000
    t = pa.table([pa.array(rng.integers(-2**62, 2**62, n)), pa.array(rng.integers(0, 2**40, n))], names=["k", "v"])
    hd, dd = run_three(ctx, t.schema, t.to_batches(max_chunksize=batch_rows), [0], 8, chunk_rows=chunk_rows)
    assert dd["bytes_h2d"] == 0 and dd["bytes_d2h"] == 0
    assert hd["bytes_h2d"] == n * 16


@pytest.mark.parametrize("keys", [[0], [5, 2]])
def test_nullable_bool_mixed_widths_sliced(ctx, keys):
    """Nullable columns of every width, Boolean values, sliced batches, unknown null counts; P = 17 and 3."""
    t = IN._mixed_table(20_000, 3)
    clean = pa.table([c.fill_null(False) if pa.types.is_boolean(c.type) else c.fill_null(0) for c in t.slice(0, 1_500).columns], schema=t.schema)
    batches = list(clean.to_batches(max_chunksize=700))
    cuts = [1_500, 1_503, 1_511, 4_000, 4_001, 13_333, 20_000]
    for a, b in zip(cuts[:-1], cuts[1:]):
        batches += t.slice(a, b - a).to_batches(max_chunksize=997)
    _, dd = run_three(ctx, t.schema, batches, keys, 17, chunk_rows=4_096, null_count_unknown=True)
    assert dd["bytes_d2h"] == 0
    run_three(ctx, t.schema, batches, keys, 3, chunk_rows=1_000_000)


@pytest.mark.parametrize("keys", [[0], [1], [3, 1]])
def test_strings_as_keys_and_payload(ctx, keys):
    """Utf8, LargeUtf8 and Binary; sliced batches; chunks cut early by a small chunk_rows."""
    t = IN._strings_table(12_000, 4)
    batches = []
    for a, b in [(0, 5), (5, 3_001), (3_001, 12_000)]:
        batches += t.slice(a, b - a).to_batches(max_chunksize=1_024)
    run_three(ctx, t.schema, batches, keys, 8, chunk_rows=2_048, null_count_unknown=True)
    run_three(ctx, t.schema, batches, keys, 6)


def views_table(n, seed):
    rnd = random.Random(seed)
    lengths = [0, 1, 3, 4, 5, 11, 12, 13, 16, 40]
    s = [None if rnd.random() < 0.1 else "".join(rnd.choice("abcdefgh") for _ in range(rnd.choice(lengths))) for _ in range(n)]
    return pa.table([pa.array(range(n), type=pa.int64()), pa.array(s, type=pa.string_view()),
                     pa.array([None if v is None else v.encode() for v in s], type=pa.binary_view())], names=["id", "v", "bv"])


@pytest.mark.parametrize("keys", [[0], [1], [2, 0]])
def test_views_of_every_length_class(ctx, keys):
    """Utf8View / BinaryView with strings of 0, 1, 11, 12, 13 and more bytes at every byte alignment of the chunk's data buffer,
    and nulls: the views k_emit_chunk builds are compared over all 16 bytes with those dfd::host::build_views builds."""
    t = views_table(10_000, 5)
    batches = [t.slice(0, 3).to_batches()[0]] + t.slice(3, 9_997).to_batches(max_chunksize=1_700)
    run_three(ctx, t.schema, batches, keys, 5, chunk_rows=4_096, null_count_unknown=True)
    run_three(ctx, t.schema, batches, keys, 8)


def dictionary_batches():
    n = 3_000
    rnd = random.Random(6)
    d1 = pa.array(["red", None, "blue", "green"])
    batches = []
    for k in range(8):
        vals = d1 if k % 4 != 3 else pa.array(["red", None, "blue", "GREEN"])
        if k % 2:
            vals = pa.array(vals.to_pylist())  # equal values, another object
        idx = pa.array([None if rnd.random() < 0.1 else rnd.randrange(4) for _ in range(n)], type=pa.int32())
        batches.append(pa.record_batch([pa.array(range(k * n, (k + 1) * n), type=pa.int64()), pa.DictionaryArray.from_arrays(idx, vals),
                                        pa.DictionaryArray.from_arrays(idx.cast(pa.int8()), pa.array([1.5, 2.5, None, 4.5]))], names=["id", "cat", "num"])
                       )
    return batches


@pytest.mark.parametrize("keys", [[0], [1], [1, 0]])
def test_dictionaries_as_payload_and_as_key(ctx, keys):
    """Device batches carry device-resident dictionaries: uploaded once per chunk (host input, counted in bytes_h2d) or the
    input batch's own (device input).  Equal dictionaries share a chunk, changed ones cut it."""
    batches = dictionary_batches()
    hd, _ = run_three(ctx, batches[0].schema, batches, keys, 4, chunk_rows=8_192)
    assert hd["bytes_h2d"] > sum(b.num_rows for b in batches) * 13  # the rows (8 + 4 + 1 bytes each) and the chunks' dictionaries


def test_device_input_batches_with_dictionaries_live_until_their_output_is_released(ctx):
    """Device input + device output: an output batch references its input batch's device dictionary, so that input batch is
    released with the last output batch that references it — exactly once — and not at finish()."""
    batches = dictionary_batches()[:3]
    N = 4
    ex = dfd.RepartitionExec(ctx, batches[0].schema, dfd.Partitioning.Hash([0], N), device_output=True, chunk_rows=1 << 20)
    pushed = [push_device(ex, rb) for rb in batches]
    ex.finish()
    assert pushed[-1] in DB.live_batches()  # the chunk's batches reference the dictionary of the last batch staged into it
    assert not set(pushed[:-1]) & DB.live_batches()
    rows = 0
    for p in range(N):
        for b in ex.execute_device(p):
            assert pushed[-1] in DB.live_batches()
            rows += b.array.length
    assert rows == sum(b.num_rows for b in batches)
    assert pushed[-1] not in DB.live_batches()
    ex.close()
    assert sorted(k for k in DB.RELEASED if k in set(pushed)) == sorted(pushed)


@pytest.mark.parametrize("keys,N", [([0], 8), ([0, 3], 17)])
def test_reference_fixture_schema(ctx, keys, N):
    """The reference's 9-column bench schema (List<Utf8> and Dictionary<Int32, Utf8> included) at 8192-row batches."""
    t = reference_fixture_table(40_000, 11)
    run_three(ctx, t.schema, t.to_batches(max_chunksize=8_192), keys, N, chunk_rows=16_384)


def test_lists_of_strings_binaries_and_primitives(ctx):
    for t in IN._list_tables():
        run_three(ctx, t.schema, t.to_batches(max_chunksize=300), [0], 5, chunk_rows=512)
        run_three(ctx, t.schema, t.slice(7).to_batches(max_chunksize=211), [0], 3, null_count_unknown=True)


def _two_columns(n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return pa.table([pa.array(rng.integers(0, 2**60, n)), pa.array(np.arange(n, dtype=np.int64))], names=["k", "v"])


def _consume_ids(ctx, ex, N, got, delay=0.0):
    def consume(p):
        stream = ex.execute_device(p)
        schema = stream.schema
        for b in stream:
            got[p].append(DO.to_host_batch(b, schema).column(1).to_numpy().copy())
            time.sleep(delay)

    threads = [threading.Thread(target=consume, args=(p,)) for p in range(N)]
    for th in threads:
        th.start()
    return threads


def test_bounded_pool_blocks_the_producer_until_consumers_release_device_batches(ctx):
    """max_pinned_chunks = 2 counts device chunks: the producer thread stalls until a consumer releases device batches, and
    every row still arrives exactly once."""
    N, n = 4, 200_000
    t = _two_columns(n, 10)
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N), device_output=True, chunk_rows=8_192, pipeline_depth=2,
                             pinned_pool_chunks=2, max_pinned_chunks=2)
    pushed = []

    def produce():
        for rb in t.to_batches(max_chunksize=8_192):
            ex.push_batch(rb)
            pushed.append(rb.num_rows)
        ex.finish()

    producer = threading.Thread(target=produce)
    producer.start()
    time.sleep(0.5)
    stalled_at = len(pushed)
    assert producer.is_alive() and stalled_at < 6  # (two chunks out, nothing released: the third flush waits)
    got = [[] for _ in range(N)]
    threads = _consume_ids(ctx, ex, N, got)
    producer.join()
    for th in threads:
        th.join()
    st = ex.stats()
    assert st["pinned_chunks"] <= 2 and st["ns_wait_pool"] > 0
    ex.close()
    ids = np.sort(np.concatenate([a for g in got for a in g]))
    assert np.array_equal(ids, np.arange(n))


def test_device_chunks_are_reused_once_consumers_release(ctx):
    """The number of device chunks allocated does not grow with the number of chunks pushed."""
    N, n = 4, 400_000
    t = _two_columns(n, 11)
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N), device_output=True, chunk_rows=8_192, max_pinned_chunks=4)
    got = [[] for _ in range(N)]
    threads = _consume_ids(ctx, ex, N, got)
    for rb in t.to_batches(max_chunksize=8_192):
        ex.push_batch(rb)
    ex.finish()
    for th in threads:
        th.join()
    st = ex.stats()
    assert st["pinned_chunks_allocated"] <= 4 and st["rows_out"] == n  # (49 chunks went through them)
    ex.close()
    assert sum(len(a) for g in got for a in g) == n


def test_abort_and_input_errors_reach_every_device_stream_after_the_queued_batches(ctx):
    t = _two_columns(40_000, 12)
    N = 3
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N), device_output=True, chunk_rows=8_192)
    for rb in t.to_batches(max_chunksize=8_192):
        ex.push_batch(rb)
    ex.abort("upstream failed")
    rows = 0
    for p in range(N):
        with pytest.raises(OSError, match="upstream failed"):
            for b in ex.execute_device(p):
                rows += b.array.length
    assert 0 < rows <= t.num_rows  # what was queued before the abort came first
    ex.close()
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N), device_output=True)
    with pytest.raises(dfd.DfdError, match="columns"):
        ex.push_batch(pa.record_batch([t.column(0).chunk(0)], names=["k"]))
    for p in range(N):
        with pytest.raises(OSError, match="columns"):
            for _ in ex.execute_device(p):
                pass
    ex.close()


def test_streams_of_the_wrong_kind_are_refused(ctx):
    t = _two_columns(100, 13)
    host = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], 2))
    dev = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], 2), device_output=True)
    with pytest.raises(dfd.DfdError) as ei:
        host.execute_device(0)
    assert ei.value.status == 1 and "host-output" in ei.value.message
    with pytest.raises(dfd.DfdError) as ei:
        dev.execute(0)
    assert ei.value.status == 1 and "device-output" in ei.value.message
    for ex in (host, dev):  # both still work
        ex.push_batch(t.to_batches()[0])
        ex.finish()
    assert sum(b.num_rows for p in range(2) for b in host.execute(p)) == 100
    assert sum(b.array.length for p in range(2) for b in dev.execute_device(p)) == 100
    host.close()
    dev.close()


class DeviceStream:
    """A small ArrowDeviceArrayStream over DeviceBatches (ctypes callbacks), counting its releases."""

    def __init__(self, batches, fail_at=None, device_type=DB.ARROW_DEVICE_CUDA):
        self.batches, self.fail_at, self.i, self.released = list(batches), fail_at, 0, 0
        self._msg = C.create_string_buffer(b"page 7 of the device reader is corrupt")
        self._next = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(nv.ArrowDeviceArrayStruct))(self._get_next)
        self._err = C.CFUNCTYPE(C.c_void_p, C.c_void_p)(lambda s: C.addressof(self._msg))
        self._rel = C.CFUNCTYPE(None, C.POINTER(nv.ArrowDeviceArrayStreamStruct))(self._release)
        self.struct = nv.ArrowDeviceArrayStreamStruct()
        self.struct.device_type = device_type
        self.struct.get_next = C.cast(self._next, C.c_void_p)
        self.struct.get_last_error = C.cast(self._err, C.c_void_p)
        self.struct.release = C.cast(self._rel, C.c_void_p)

    def _get_next(self, s, out):
        if self.fail_at is not None and self.i == self.fail_at:
            return 5
        if self.i >= len(self.batches):
            C.memset(out, 0, C.sizeof(nv.ArrowDeviceArrayStruct))
            return 0
        C.memmove(out, C.addressof(self.batches[self.i].device_array), C.sizeof(nv.ArrowDeviceArrayStruct))
        self.i += 1
        return 0

    def _release(self, s):
        self.released += 1
        s.contents.release = None


def test_run_device_pulls_a_device_stream(ctx):
    """run_device over a stream of device batches gives the streams that pushing them gives; a failing get_next aborts the
    operator with the stream's message; a CPU-typed stream is refused; the stream is released exactly once each time."""
    t = IN._strings_table(6_000, 14)
    batches, N = t.to_batches(max_chunksize=1_000), 5
    part = dfd.Partitioning.Hash([1], N)
    pushed = dfd.RepartitionExec(ctx, t.schema, part, device_output=True, chunk_rows=2_048)
    for rb in batches:
        push_device(pushed, rb)
    pushed.finish()
    want = device_streams(ctx, pushed, N)
    pushed.close()
    ran = dfd.RepartitionExec(ctx, t.schema, part, device_output=True, chunk_rows=2_048)
    src = DeviceStream([DB.DeviceBatch(rb) for rb in batches])
    ran.run_device(src.struct)
    assert src.released == 1 and src.i == len(batches)
    assert_same_streams(want, device_streams(ctx, ran, N))
    ran.close()

    bad = dfd.RepartitionExec(ctx, t.schema, part, device_output=True, chunk_rows=2_048)
    made = [DB.DeviceBatch(rb) for rb in batches]
    src = DeviceStream(made, fail_at=3)
    with pytest.raises(dfd.DfdError, match="page 7 of the device reader is corrupt"):
        bad.run_device(src.struct)
    assert src.released == 1
    for p in range(N):
        with pytest.raises(OSError, match="page 7"):
            for _ in bad.execute_device(p):
                pass
    bad.close()
    del made, src  # (the batches never pulled go with their owners)

    cpu = dfd.RepartitionExec(ctx, t.schema, part, device_output=True)
    src = DeviceStream([], device_type=DB.ARROW_DEVICE_CPU)
    with pytest.raises(dfd.DfdError) as ei:
        cpu.run_device(src.struct)
    assert ei.value.status == 1 and "device type" in ei.value.message and src.released == 1
    cpu.close()
