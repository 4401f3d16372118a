"""GPU tests of the host operator's DEVICE input path (dfd_repartition_exec_push_device): the same record batches pushed once
as host batches (push) and once as device-resident Arrow C Device batches must give identical partition streams — the
same batches, batch boundaries, row order, values (the bytes under null slots included), validity, offsets, view layout,
dictionary values and list children.  tests/test_exec_device_input_cpu_harness.py runs these bodies on the CPU harness."""
import ctypes as C
import random
import threading

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from tests import device_batches as DB
from tests import test_exec_keys_gpu as K
from tests.test_exec_gpu import reference_fixture_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    """A worker context of this module's own: the pinned output chunks its operators leave in the context's cache go
    with it, instead of filling the cache of the session's context that later modules test."""
    c = dfd.WorkerContext(0)
    yield c
    c.close()


def _streams(ex, N):
    return [list(ex.execute(p)) for p in range(N)]


def _assert_same_array(a, b, where):
    assert a.type == b.type and len(a) == len(b) and a.offset == b.offset, where
    assert a.null_count == b.null_count, where
    ba, bb = a.buffers(), b.buffers()
    assert len(ba) == len(bb), where
    for k, (x, y) in enumerate(zip(ba, bb)):  # (the whole imported buffers: the chunk up to the end of this slice)
        assert (x is None) == (y is None), (where, k)
        if x is not None:
            assert x.equals(y), (where, k)
    if pa.types.is_dictionary(a.type):  # (buffers() covers the indices only)
        assert _same_values(a.dictionary, b.dictionary), where


def _same_values(x, y):
    """Same values, float NaNs compared by bit pattern."""
    if x.equals(y):
        return True
    if len(x) != len(y) or x.type != y.type or not pa.types.is_floating(x.type):
        return False
    w = x.type.bit_width // 8
    raw = [np.frombuffer(v.buffers()[1], dtype=np.uint8)[v.offset * w:(v.offset + len(v)) * w] for v in (x, y)]
    valid = [v.is_valid().to_numpy(zero_copy_only=False) for v in (x, y)]
    keep = np.repeat(valid[0], w)
    return np.array_equal(valid[0], valid[1]) and np.array_equal(raw[0][keep], raw[1][keep])


def assert_same_streams(host, dev):
    assert len(host) == len(dev)
    for p, (hs, ds) in enumerate(zip(host, dev)):
        assert [b.num_rows for b in hs] == [b.num_rows for b in ds], p  # same batch boundaries
        for k, (hb, db) in enumerate(zip(hs, ds)):
            assert hb.schema.equals(db.schema), (p, k)
            for c in range(hb.num_columns):
                _assert_same_array(hb.column(c), db.column(c), (p, k, hb.schema.names[c]))


def push_device(ex, rb, **kw):
    b = DB.DeviceBatch(rb, **kw)
    ex.push_device_batch(b.device_array)
    return b.key


def run_both(ctx, schema, batches, keys, N, null_count_unknown=False, **opts):
    """Push `batches` through a host-input and a device-input operator; assert identical streams; return the device stats."""
    host = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash(keys, N), **opts)
    for rb in batches:
        host.push_batch(rb)
    host.finish()
    want, hstats = _streams(host, N), host.stats()
    host.close()
    dev = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash(keys, N), **opts)
    pushed = [push_device(dev, rb, null_count_unknown=null_count_unknown) for rb in batches]
    dev.finish()
    assert not set(pushed) & DB.live_batches()  # every batch released by finish() ...
    assert sorted(k for k in DB.RELEASED if k in set(pushed)) == sorted(pushed)  # ... exactly once
    got, dstats = _streams(dev, N), dev.stats()
    dev.close()
    assert_same_streams(want, got)
    assert dstats["bytes_h2d"] == 0 and dstats["rows_in"] == hstats["rows_in"] == sum(b.num_rows for b in batches)
    assert dstats["rows_out"] == hstats["rows_out"]
    return dstats


@pytest.mark.parametrize("batch_rows,chunk_rows", [(8192, 0), (1024, 10_000), (100_000, 65_536)])
def test_fixed_width_batches(ctx, batch_rows, chunk_rows):
    """cfg-1 shape (k: Int64, v: Int64), Hash([k], 8): batches smaller than, equal to and larger than a chunk."""
    rng = np.random.Generator(np.random.PCG64(1))
    n = 300_000
    t = pa.table([pa.array(rng.integers(-2**62, 2**62, n)), pa.array(rng.integers(0, 2**40, n))], names=["k", "v"])
    st = run_both(ctx, t.schema, t.to_batches(max_chunksize=batch_rows), [0], 8, chunk_rows=chunk_rows)
    assert st["bytes_d2h"] > 0


def _mixed_table(n, seed):
    rnd = random.Random(seed)

    def maybe(v, p=0.2):
        return None if rnd.random() < p else v

    return pa.table([pa.array([rnd.getrandbits(62) for _ in range(n)], type=pa.int64()),
                     pa.array([maybe(rnd.getrandbits(7)) for _ in range(n)], type=pa.int8()),
                     pa.array([maybe(rnd.getrandbits(15)) for _ in range(n)], type=pa.int16()),
                     pa.array([maybe(rnd.random() < 0.5) for _ in range(n)], type=pa.bool_()),
                     pa.array([rnd.random() < 0.3 for _ in range(n)], type=pa.bool_()),
                     pa.array([maybe(rnd.random()) for _ in range(n)], type=pa.float64()),
                     pa.array([maybe(rnd.getrandbits(60)) for _ in range(n)], type=pa.decimal128(38, 2)),
                     pa.array([maybe(rnd.getrandbits(30)) for _ in range(n)], type=pa.int32())],
                    names=["id", "i8", "i16", "b", "bnn", "f", "dec", "i32"])


@pytest.mark.parametrize("keys", [[0], [1, 3], [5, 2]])
def test_nullable_bool_mixed_widths_sliced(ctx, keys):
    """Nullable columns of every width, Boolean values and keys, sliced batches (non-zero child offsets at every bit
    position), null_count -1, a first batch without nulls followed by batches with them."""
    t = _mixed_table(20_000, 3)
    clean = pa.table([c.fill_null(False) if pa.types.is_boolean(c.type) else c.fill_null(0) for c in t.slice(0, 1_500).columns], schema=t.schema)
    batches = list(clean.to_batches(max_chunksize=700))
    cuts = [1_500, 1_503, 1_511, 4_000, 4_001, 13_333, 20_000]
    for a, b in zip(cuts[:-1], cuts[1:]):
        batches += t.slice(a, b - a).to_batches(max_chunksize=997)
    run_both(ctx, t.schema, batches, keys, 7, chunk_rows=4_096, null_count_unknown=True)
    run_both(ctx, t.schema, batches, keys, 3, chunk_rows=1_000_000)


def _strings_table(n, seed):
    rnd = random.Random(seed)
    words = ["", "a", "hello", "x" * 13, "ünïcödé", "a-much-longer-string-than-twelve-bytes"]
    s = [None if rnd.random() < 0.1 else rnd.choice(words) + str(rnd.getrandbits(10)) for _ in range(n)]
    return pa.table([pa.array(range(n), type=pa.int64()), pa.array(s, type=pa.string()), pa.array(s, type=pa.large_string()),
                     pa.array([None if v is None else v.encode() * (1 + len(v) % 3) for v in s], type=pa.binary())],
                    names=["id", "u", "U", "z"])


@pytest.mark.parametrize("keys", [[0], [1], [2, 0], [3, 1]])
def test_strings_as_keys_and_payload(ctx, keys):
    """Utf8, LargeUtf8 and Binary as keys and as payload; sliced batches; chunks cut early by small chunk_rows."""
    t = _strings_table(12_000, 4)
    batches = []
    for a, b in [(0, 5), (5, 3_001), (3_001, 12_000)]:
        batches += t.slice(a, b - a).to_batches(max_chunksize=1_024)
    run_both(ctx, t.schema, batches, keys, 6, chunk_rows=2_048, null_count_unknown=True)
    run_both(ctx, t.schema, batches, keys, 6)


def test_all_empty_strings(ctx):
    n = 5_000
    t = pa.table([pa.array(range(n), type=pa.int64()), pa.array([""] * n), pa.array([None if i % 3 else b"" for i in range(n)], type=pa.binary())],
                 names=["id", "s", "b"])
    run_both(ctx, t.schema, t.to_batches(max_chunksize=1_000), [1], 4, chunk_rows=2_048)
    run_both(ctx, t.schema, t.to_batches(max_chunksize=1_000), [0], 4)


def test_views_inline_and_out_of_line_over_several_buffers(ctx):
    """Utf8View / BinaryView with inline (<= 12 bytes) and out-of-line strings spread over several variadic data buffers."""
    rnd = random.Random(5)
    parts = []
    for k in range(4):
        s = [None if rnd.random() < 0.1 else ("w" * rnd.choice([0, 3, 12, 13, 40])) + str(k) + str(rnd.getrandbits(9)) for _ in range(2_500)]
        parts.append(pa.table([pa.array(range(k * 2_500, (k + 1) * 2_500), type=pa.int64()), pa.array(s, type=pa.string_view()),
                               pa.array([None if v is None else v.encode() for v in s], type=pa.binary_view())], names=["id", "v", "bv"]))
    views = pa.concat_arrays([p.column(1).combine_chunks() for p in parts])
    bviews = pa.concat_arrays([p.column(2).combine_chunks() for p in parts])
    assert len(views.buffers()) > 3  # several data buffers
    t = pa.table([pa.array(range(10_000), type=pa.int64()), views, bviews], names=["id", "v", "bv"])
    batches = [t.slice(0, 3).to_batches()[0]] + t.slice(3, 9_997).to_batches(max_chunksize=1_700)
    for keys in ([0], [1], [2, 0]):
        run_both(ctx, t.schema, batches, keys, 5, chunk_rows=4_096, null_count_unknown=True)


def test_dictionary_payload_shared_and_cut_chunks(ctx):
    """Dictionary payload: equal-valued dictionaries in different objects share a chunk, changed dictionaries cut it."""
    n = 3_000
    rnd = random.Random(6)
    d1 = pa.array(["red", None, "blue", "green"])
    batches = []
    for k in range(8):
        vals = d1 if k % 4 != 3 else pa.array(["red", None, "blue", "GREEN"])
        if k % 2:
            vals = pa.array(vals.to_pylist())  # equal values, another object
        idx = pa.array([None if rnd.random() < 0.1 else rnd.randrange(4) for _ in range(n)], type=pa.int32())
        batches.append(pa.record_batch([pa.array(range(k * n, (k + 1) * n), type=pa.int64()), pa.DictionaryArray.from_arrays(idx, vals)],
                                       names=["id", "cat"]))
    schema = batches[0].schema
    for keys in ([0], [1], [1, 0]):
        st = run_both(ctx, schema, batches, keys, 4, chunk_rows=8_192)
        assert st["bytes_d2h"] > 0


@pytest.mark.parametrize("index_fmt,value_fmt", K.DICT_CASES, ids=[f"{i}-{K._id(v)}" for i, v in K.DICT_CASES])
def test_dictionary_keys(ctx, index_fmt, value_fmt):
    """Every (index, value) pair the keys suite covers, as the hash key (hashed through the device-resident values)."""
    check_dictionary_key(ctx, index_fmt, value_fmt)


def check_dictionary_key(ctx, index_fmt, value_fmt, n=600):
    rnd = random.Random(K._seed("dk", index_fmt, value_fmt))
    m = 17
    d = pa.DictionaryArray.from_arrays(K._indices(index_fmt, n, m, rnd), K.values(value_fmt, m, rnd))
    t = pa.table([pa.array(range(n), type=pa.int64()), d], names=["rid", "x"])
    run_both(ctx, t.schema, t.to_batches(max_chunksize=250), [1], 5, chunk_rows=512)


@pytest.mark.parametrize("fmt", K.KEY_FORMATS, ids=[K._id(f) for f in K.KEY_FORMATS])
def test_every_key_format(ctx, fmt):
    check_key_format(ctx, fmt)


def check_key_format(ctx, fmt, n=700):
    rnd = random.Random(K._seed("kf", fmt))
    x = K.values(fmt, n, rnd)
    lead = pa.array([None if i % 7 == 2 else rnd.getrandbits(63) for i in range(n)], type=pa.int64())
    t = pa.table([lead, x, pa.array(range(n), type=pa.int64())], names=["lead", "x", "rid"])
    batches = [t.slice(0, 1).to_batches()[0]] + t.slice(1, n - 1).to_batches(max_chunksize=233)
    run_both(ctx, t.schema, batches, [1], 6, chunk_rows=512)
    run_both(ctx, t.schema, batches, [0, 1], 6, chunk_rows=512, null_count_unknown=True)


def _list_tables():
    ids = pa.array(range(1000), type=pa.int64())
    base = pa.array([[b"a", None, b"ccc"] if i % 3 == 0 else ([] if i % 3 == 1 else None) for i in range(1200)], type=pa.list_(pa.binary()))
    sliced = base.slice(200, 1000)
    empties = pa.array([[] for _ in range(1000)], type=pa.list_(pa.string()))
    nulls = pa.array([None] * 1000, type=pa.list_(pa.string()))
    flat = pa.array([str(i) for i in range(3000)], type=pa.string()).slice(500, 2000)
    fromchild = pa.ListArray.from_arrays(pa.array(range(0, 2001, 2), type=pa.int32()), flat)
    edges = pa.table([ids, sliced, empties, nulls, fromchild], names=["id", "b", "e", "n", "c"])
    rnd = random.Random(8)
    prims = pa.table([ids, pa.array([None if i % 9 == 4 else [rnd.getrandbits(31) for _ in range(i % 4)] for i in range(1000)], type=pa.list_(pa.int32())),
                      pa.array([[None if k == 1 else rnd.random() for k in range(i % 3)] for i in range(1000)], type=pa.list_(pa.float64())),
                      pa.array([[rnd.getrandbits(60)] * (i % 2) for i in range(1000)], type=pa.list_(pa.field("item", pa.int64(), False)))],
                     names=["id", "ints", "floats", "nn"])
    return edges, prims


def test_lists_of_strings_binaries_and_primitives(ctx):
    """List<Utf8>, List<Binary> and List<primitive> payload, with the edge shapes of the host suite: all-null lists, all-empty
    lists, a batch with no elements, a sliced list and a child with its own offset."""
    for t in _list_tables():
        run_both(ctx, t.schema, t.to_batches(max_chunksize=300), [0], 5, chunk_rows=512)
        run_both(ctx, t.schema, t.slice(7).to_batches(max_chunksize=211), [0], 3, null_count_unknown=True)


@pytest.mark.parametrize("keys", [[0], [0, 3]])
def test_reference_fixture_schema_at_8192_row_batches(ctx, keys):
    """The reference's 9-column bench schema (List<Utf8> and Dictionary<Int32, Utf8> included) at 8192-row batches."""
    t = reference_fixture_table(40_000, 11)
    run_both(ctx, t.schema, t.to_batches(max_chunksize=8_192), keys, 16, chunk_rows=16_384)


def test_large_binary_and_fixed_size_binary_payload(ctx):
    rnd = random.Random(9)
    n = 4_000
    t = pa.table([pa.array(range(n), type=pa.int64()),
                  pa.array([None if i % 11 == 0 else bytes(rnd.getrandbits(8) for _ in range(i % 23)) for i in range(n)], type=pa.large_binary()),
                  pa.array([None if i % 5 == 0 else bytes(rnd.getrandbits(8) for _ in range(16)) for i in range(n)], type=pa.binary(16)),
                  pa.array([bytes([i % 256, 7]) for i in range(n)], type=pa.binary(2))], names=["id", "lb", "uuid", "w2"])
    run_both(ctx, t.schema, t.slice(3).to_batches(max_chunksize=900), [0], 4, chunk_rows=1_024, null_count_unknown=True)


def test_back_pressure_with_concurrent_consumers(ctx):
    """max_pinned_chunks bounds the pinned pool: device pushes block until consumers release chunks; everything arrives."""
    N, n = 4, 200_000
    rng = np.random.Generator(np.random.PCG64(10))
    t = pa.table([pa.array(rng.integers(0, 2**60, n)), pa.array(rng.integers(0, 2**60, n))], names=["k", "v"])
    host = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N), chunk_rows=8_192)
    for rb in t.to_batches(max_chunksize=5_000):
        host.push_batch(rb)
    host.finish()
    want = _streams(host, N)
    host.close()
    dev = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N), chunk_rows=8_192, pinned_pool_chunks=2, max_pinned_chunks=3)
    got = [None] * N

    def consume(p):  # (copies the rows out and lets each batch go: holding them would hold the pinned chunks)
        got[p] = [(b.num_rows, [c.to_numpy().copy() for c in b.columns]) for b in dev.execute(p)]

    threads = [threading.Thread(target=consume, args=(p,)) for p in range(N)]
    for th in threads:
        th.start()
    for rb in t.to_batches(max_chunksize=5_000):
        push_device(dev, rb)
    dev.finish()
    for th in threads:
        th.join()
    assert dev.stats()["pinned_chunks"] <= 3
    dev.close()
    for p in range(N):
        assert [b.num_rows for b in want[p]] == [r for r, _ in got[p]], p
        for b, (_, cols) in zip(want[p], got[p]):
            for c, arr in zip(b.columns, cols):
                assert np.array_equal(c.to_numpy(), arr), p


def test_abort_after_device_pushes_releases_the_batches(ctx):
    t = _strings_table(6_000, 12)
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], 3), chunk_rows=2_048)
    keys = [push_device(ex, rb) for rb in t.to_batches(max_chunksize=1_000)]
    ex.abort("upstream failed")
    assert not set(keys) & DB.live_batches()  # released, each once
    assert sorted(k for k in DB.RELEASED if k in set(keys)) == sorted(keys)
    rows = 0
    for p in range(3):
        r = ex.execute(p)
        with pytest.raises(Exception, match="upstream failed"):
            for b in r:
                rows += b.num_rows
    assert rows <= t.num_rows
    ex.close()


def _expect_refusal(ex, fn, word):
    with pytest.raises(dfd.DfdError) as ei:
        fn()
    assert ei.value.status == 1 and word in ei.value.message, ei.value.message
    for p in range(ex.partitioning.partition_count):  # the operator has failed: every stream ends with the error
        with pytest.raises(Exception):
            for _ in ex.execute(p):
                pass


def test_refusals_release_the_batch_and_fail_the_operator(ctx):
    t = pa.table([pa.array(range(100), type=pa.int64()), pa.array([str(i) for i in range(100)])], names=["k", "s"])
    rb = t.to_batches()[0]
    cases = [("device type", lambda ex: push_device(ex, rb, device_type=DB.ARROW_DEVICE_CPU)),
             ("device", lambda ex: push_device(ex, rb, device_id=getattr(ctx, "device", 0) + 1)),
             ("columns", lambda ex: push_device(ex, pa.record_batch([rb.column(0)], names=["k"]))),
             ("host batches", lambda ex: (ex.push_batch(rb), push_device(ex, rb))),
             ("device batches", lambda ex: (push_device(ex, rb), ex.push_batch(rb)))]
    for word, fn in cases:
        before = set(DB.live_batches())
        ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], 2))
        _expect_refusal(ex, lambda: fn(ex), word)
        assert DB.live_batches() <= before, word  # the refused (and any accepted) batch was released
        ex.close()
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], 2))  # empty pushes decide nothing
    ex.push_batch(rb.slice(0, 0))
    push_device(ex, rb.slice(0, 0))
    push_device(ex, rb)
    ex.finish()
    assert sum(b.num_rows for p in range(2) for b in ex.execute(p)) == 100
    ex.close()


def test_sync_event_is_waited_on(ctx):
    """The batch's buffers are filled by a copy on a side stream queued behind a long independent operation there; the
    event recorded after it goes in sync_event and the batch is pushed at once.  The output must still be right."""
    import torch

    n, N = 1 << 20, 4
    rng = np.random.Generator(np.random.PCG64(13))
    t = pa.table([pa.array(rng.integers(0, 2**62, n)), pa.array(rng.integers(0, 2**62, n))], names=["k", "v"])
    rb = t.to_batches()[0]
    host = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N))
    host.push_batch(rb)
    host.finish()
    want = _streams(host, N)
    host.close()
    side = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(8):
            a = a @ a / 64.0  # (ordinary work ahead of the copies on the producer's stream)
    b = DB.DeviceBatch(rb, stream=side)
    ev = torch.cuda.Event()
    ev.record(side)
    handle = C.c_void_p(ev.cuda_event)
    b.device_array.sync_event = C.cast(C.pointer(handle), C.c_void_p)
    dev = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], N))
    dev.push_device_batch(b.device_array)
    dev.finish()
    got = _streams(dev, N)
    dev.close()
    assert_same_streams(want, got)
    torch.cuda.synchronize()
