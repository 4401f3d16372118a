"""GPU parity tests of the host operator (RepartitionExec over Arrow C Data /
C Stream): HOST record batches in, per-destination HOST record batch streams
out, compared bit-exactly (values AND order) with the CPU oracle."""
import random

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from oracle import oracle as orc
from tests.util import cfg2_columns, expected_partitions

pytestmark = pytest.mark.gpu


def collect(exec_, N):
    return [exec_.execute(p).read_all() for p in range(N)]


def batches_of(arrays, names, batch_rows):
    t = pa.table(arrays, names=names)
    return t.to_batches(max_chunksize=batch_rows)


@pytest.mark.parametrize("batch_rows,chunk_rows", [(8192, 0), (1024, 10_000), (100_000, 65_536), (1_000_000, 0)])
def test_cfg1_shape_matches_oracle_exactly(ctx, batch_rows, chunk_rows):
    """cfg-1 shape (ShuffleBench defaults): 1M rows, (k: Int64, v: Int64), Hash([k], 8)."""
    rng = np.random.Generator(np.random.PCG64(1))
    n, N = 1_000_000, 8
    k = rng.integers(0, 2**63 - 1, n, dtype=np.int64)
    v = np.arange(n, dtype=np.int64)
    ex = dfd.RepartitionExec(ctx, pa.schema([("k", pa.int64()), ("v", pa.int64())]), dfd.Partitioning.Hash([0], N),
                             chunk_rows=chunk_rows)
    for b in batches_of([k, v], ["k", "v"], batch_rows):
        ex.push_batch(b)
    ex.finish()
    outs = collect(ex, N)
    ref, counts, starts = orc.repartition_table([k, v], [0], N, 8192, 1)
    st = ex.stats()
    assert st["rows_in"] == n and st["rows_out"] == n
    for p in range(N):
        assert outs[p].num_rows == counts[p]
        assert np.array_equal(outs[p].column("k").to_numpy(), ref[0][starts[p]:starts[p + 1]])
        assert np.array_equal(outs[p].column("v").to_numpy(), ref[1][starts[p]:starts[p + 1]])
    ex.close()


def test_nullable_bool_mixed_widths_and_sliced_batches(ctx):
    rnd = random.Random(4)
    rng = np.random.Generator(np.random.PCG64(4))
    n, N = 50_000, 12
    key = pa.array([rnd.choice([None, rnd.getrandbits(40)]) for _ in range(n)], type=pa.int64())
    i32 = pa.array([rnd.choice([None, rnd.getrandbits(31)]) for _ in range(n)], type=pa.int32())
    u8 = pa.array(rng.integers(0, 255, n, dtype=np.uint8))
    f64 = pa.array(rng.standard_normal(n))
    bl = pa.array([rnd.choice([None, True, False]) for _ in range(n)])
    ts = pa.array(rng.integers(0, 2**60, n, dtype=np.int64)).cast(pa.timestamp("ns"))
    names = ["key", "i32", "u8", "f64", "bl", "ts"]
    table = pa.table([key, i32, u8, f64, bl, ts], names=names)
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0, 1], N), chunk_rows=16_384)
    # ragged, sliced batches: offsets that are not multiples of 8
    cuts = [0, 13, 1000, 1003, 20_001, 20_001, 37_777, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        for rb in table.slice(a, b - a).to_batches():
            ex.push_batch(rb)
    ex.finish()
    outs = collect(ex, N)
    dest = orc.partition_ids([key, i32], n, N)
    order, starts = expected_partitions(dest, N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].num_rows == want.num_rows
        assert outs[p].equals(want), p
    ex.close()


def test_run_from_reader_and_empty_inputs(ctx):
    cols = cfg2_columns(30_000, 3)
    names = ["a", "b", "c"]
    table = pa.table(cols, names=names)
    batches = table.to_batches(max_chunksize=7000)
    batches.insert(2, table.slice(0, 0).to_batches()[0] if table.slice(0, 0).to_batches() else pa.RecordBatch.from_arrays(
        [pa.array([], type=pa.int64())] * 3, names=names))
    reader = pa.RecordBatchReader.from_batches(table.schema, batches)
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], 3))
    ex.run(reader)
    outs = collect(ex, 3)
    ref, counts, starts = orc.repartition_table(cols, [0], 3, 8192, 1)
    for p in range(3):
        assert np.array_equal(outs[p].column("b").to_numpy(), ref[1][starts[p]:starts[p + 1]])
    ex.close()
    # no input at all: every partition stream ends immediately, schema preserved (invariants ii, iv)
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], 4))
    ex.finish()
    for p in range(4):
        t = ex.execute(p).read_all()
        assert t.num_rows == 0 and t.schema.names == names
    ex.close()


def test_single_partition_and_pinned_input(ctx):
    n = 200_000
    pt = dfd.PinnedTable(ctx, n, [np.int64, np.int64])
    rng = np.random.Generator(np.random.PCG64(9))
    pt.columns[0][:] = rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64)
    pt.columns[1][:] = np.arange(n)
    ex = dfd.RepartitionExec(ctx, pa.schema([("k", pa.int64()), ("v", pa.int64())]), dfd.Partitioning.Hash([0], 1))
    for rb in pt.record_batches(["k", "v"], 50_000):
        ex.push_batch(rb)
    ex.finish()
    out = ex.execute(0).read_all()
    assert np.array_equal(out.column("v").to_numpy(), np.arange(n))
    ex.close()


def test_operator_errors(ctx):
    with pytest.raises(dfd.DfdError) as e:  # List<Utf8> travels as payload, but is not a hash key
        dfd.RepartitionExec(ctx, pa.schema([("s", pa.list_(pa.string()))]), dfd.Partitioning.Hash([0], 4))
    assert e.value.status == 6  # DFD_ERR_UNSUPPORTED
    with pytest.raises(dfd.DfdError) as e:  # other nested types are still out of scope
        dfd.RepartitionExec(ctx, pa.schema([("k", pa.int64()), ("s", pa.list_(pa.list_(pa.int32())))]), dfd.Partitioning.Hash([0], 4))
    assert e.value.status == 6
    with pytest.raises(dfd.DfdError) as e:
        dfd.RepartitionExec(ctx, pa.schema([("k", pa.int64()), ("s", pa.struct([("a", pa.int32())]))]), dfd.Partitioning.Hash([0], 4))
    assert e.value.status == 6
    sch = pa.schema([("k", pa.int64())])
    with pytest.raises(dfd.DfdError):
        dfd.RepartitionExec(ctx, sch, dfd.Partitioning.Hash([1], 4))
    ex = dfd.RepartitionExec(ctx, sch, dfd.Partitioning.Hash([0], 4))
    ex.finish()
    with pytest.raises(dfd.DfdError):
        ex.push_batch(pa.RecordBatch.from_arrays([pa.array([1, 2, 3])], names=["k"]))
    ex.close()
    # wrong column count: the error reaches every partition stream
    ex = dfd.RepartitionExec(ctx, sch, dfd.Partitioning.Hash([0], 2))
    with pytest.raises(dfd.DfdError):
        ex.push_batch(pa.RecordBatch.from_arrays([pa.array([1]), pa.array([2])], names=["k", "x"]))
    for p in range(2):
        with pytest.raises(Exception):
            ex.execute(p).read_all()
    ex.close()
    # a List<Utf8> whose child offsets decrease over the pushed rows (list offsets 1, 1, 2 over child offsets 0, 6, 2, 8: the
    # rows' element runs from byte 6 to byte 2): refused before any of its bytes are staged, and the error reaches every
    # partition stream
    child = pa.Array.from_buffers(pa.string(), 3, [None, pa.py_buffer(np.array([0, 6, 2, 8], dtype=np.int32).tobytes()), pa.py_buffer(b"abcdefgh")])
    lst = pa.Array.from_buffers(pa.list_(pa.string()), 2, [None, pa.py_buffer(np.array([1, 1, 2], dtype=np.int32).tobytes())], children=[child])
    rb = pa.RecordBatch.from_arrays([pa.array([1, 2], type=pa.int64()), lst], names=["k", "s"])
    ex = dfd.RepartitionExec(ctx, rb.schema, dfd.Partitioning.Hash([0], 2))
    with pytest.raises(dfd.DfdError) as e:
        ex.push_batch(rb)
    assert e.value.status == 1 and "list offsets are not monotonic" in str(e.value)  # DFD_ERR_INVALID_ARGUMENT
    with pytest.raises(dfd.DfdError):
        ex.finish()
    for p in range(2):
        with pytest.raises(Exception):
            ex.execute(p).read_all()
    ex.close()


def test_abort_fails_every_partition_stream_after_the_queued_rows(ctx):
    """The producer's input failed mid-way (dfd_repartition_exec_abort): like RepartitionExec forwarding an input error to
    all of its outputs, every partition stream delivers what was already queued and then ends with the input's message."""
    n, N = 40_000, 4
    cols = cfg2_columns(n, 2)
    table = pa.table(cols, names=["k", "v"])
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=8_192)
    for rb in table.to_batches(max_chunksize=8_192):
        ex.push_batch(rb)
    ex.abort("parquet page 7 is corrupt")
    ex.abort("a second failure does not replace the first")
    for p in range(N):
        reader, rows, err = ex.execute(p), 0, None
        try:
            for rb in reader:
                rows += rb.num_rows
        except Exception as e:  # pyarrow raises from get_next's EIO with get_last_error's text
            err = str(e)
        assert err is not None and "parquet page 7 is corrupt" in err, (p, rows, err)
    with pytest.raises(dfd.DfdError):
        ex.push_batch(table.to_batches()[0])
    ex.close()
    # abort after a clean finish is a no-op: the streams end normally
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N))
    ex.push_batch(table.to_batches()[0])
    ex.finish()
    ex.abort("too late")
    assert sum(ex.execute(p).read_all().num_rows for p in range(N)) == table.to_batches()[0].num_rows
    ex.close()


def test_utf8_keys_and_payload_through_the_operator(ctx):
    """cfg-3 / cfg-5 shapes through the host operator: Utf8 keys, Utf8 / LargeUtf8 / Binary payload, nulls, slices."""
    rnd = random.Random(12)
    n, N = 40_000, 6
    words = ["", "a", "N", "O", "F", "R", "search phrase", "x" * 70, "päö"]
    uid = pa.array([rnd.getrandbits(18) for _ in range(n)], type=pa.int64())
    phrase = pa.array([rnd.choice([None] + words) if rnd.random() < 0.8 else "q%d" % rnd.getrandbits(30) for _ in range(n)], type=pa.string())
    big = pa.array([rnd.choice([None, "big" * rnd.randint(0, 20)]) for _ in range(n)], type=pa.large_string())
    binv = pa.array([rnd.choice([None, b"", bytes(rnd.getrandbits(8) for _ in range(rnd.randint(0, 12)))]) for _ in range(n)], type=pa.binary())
    val = pa.array(np.arange(n, dtype=np.int32))
    names = ["uid", "phrase", "big", "bin", "val"]
    table = pa.table([uid, phrase, big, binv, val], names=names)
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0, 1], N), chunk_rows=8192)
    cuts = [0, 5, 9000, 9003, 25_001, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        for rb in table.slice(a, b - a).to_batches(max_chunksize=7000):
            ex.push_batch(rb)
    ex.finish()
    outs = collect(ex, N)
    dest = orc.partition_ids([uid, phrase], n, N)
    order, starts = expected_partitions(dest, N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].num_rows == want.num_rows
        assert outs[p].equals(want), p
    ex.close()


def test_all_empty_strings_chunk(ctx):
    """A chunk whose string column has zero bytes still yields valid Arrow arrays."""
    n = 1000
    t = pa.table([pa.array(np.arange(n, dtype=np.int64)), pa.array([""] * n, type=pa.string())], names=["k", "s"])
    ex = dfd.RepartitionExec(ctx, t.schema, dfd.Partitioning.Hash([0], 3))
    for rb in t.to_batches():
        ex.push_batch(rb)
    ex.finish()
    total = 0
    for p in range(3):
        out = ex.execute(p).read_all()
        assert out.column("s").to_pylist() == [""] * out.num_rows
        total += out.num_rows
    assert total == n
    ex.close()


def test_utf8view_and_dictionary_columns_round_trip(ctx):
    """Utf8View columns (what DataFusion reads parquet strings as by default) and Dictionary<Int32, Utf8> columns (the
    reference's bench schema, src/execution_plans/benchmarks/fixture.rs:13-33), as keys and as payload: the output
    batches keep the input schema (views stay views, dictionaries travel by reference) and every destination equals the
    oracle's rows, in order.  The reference GC's such arrays before its network hop (impl_execute_task.rs:248-271); here
    the output views point into one compact per-chunk data buffer, which is the same effect."""
    rnd = random.Random(9)
    n, N = 40_000, 12
    words = ["", "a", "hello", "x" * 12, "y" * 13, "a-much-longer-string-than-twelve-bytes", "ünïcödé-" * 3]
    sv = pa.array([rnd.choice(words) + ("" if rnd.random() < 0.5 else str(rnd.getrandbits(20))) if rnd.random() > 0.1 else None
                   for _ in range(n)], type=pa.string()).cast(pa.string_view())
    dict_values = pa.array(["red", "green", None, "blue-" * 5, ""], type=pa.string())
    cat = pa.DictionaryArray.from_arrays(pa.array([rnd.choice([None, 0, 1, 2, 3, 4]) for _ in range(n)], type=pa.int32()), dict_values)
    idv = pa.array([rnd.getrandbits(30) for _ in range(n)], type=pa.int64())
    bv = pa.array([None if rnd.random() < 0.2 else bytes(rnd.getrandbits(8) for _ in range(rnd.randint(0, 20))) for _ in range(n)],
                  type=pa.binary()).cast(pa.binary_view())
    table = pa.table([idv, sv, cat, bv], names=["id", "label", "category", "raw"])
    # (pyarrow has no take / hash kernels for view types: the expectation is computed on the same data as Utf8 / Binary)
    plain = pa.table([idv, sv.cast(pa.string()), cat, bv.cast(pa.binary())], names=table.column_names)
    for keys in ([0], [1], [2], [2, 1, 0]):
        ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash(keys, N), chunk_rows=8_192)
        cuts = [0, 5, 5_000, 5_003, 20_001, n]
        for a, b in zip(cuts[:-1], cuts[1:]):
            for rb in table.slice(a, b - a).to_batches(max_chunksize=3_000):
                ex.push_batch(rb)
        ex.finish()
        outs = collect(ex, N)
        dest = orc.partition_ids([plain.column(k).combine_chunks() for k in keys], n, N)
        order, starts = expected_partitions(dest, N)
        for p in range(N):
            want = plain.take(pa.array(order[starts[p]:starts[p + 1]]))
            assert outs[p].schema.equals(table.schema), (keys, p, outs[p].schema)
            assert outs[p].num_rows == want.num_rows, (keys, p)
            for name in table.column_names:
                got_c, want_c = outs[p].column(name).combine_chunks(), want.column(name).combine_chunks()
                if pa.types.is_dictionary(got_c.type):
                    got_c, want_c = got_c.dictionary_decode(), want_c.dictionary_decode()
                assert got_c.cast(want_c.type).equals(want_c), (keys, p, name)
        ex.close()


def test_small_batches_of_every_shape_coalesce_into_full_chunks(ctx):
    """Batches with validity bitmaps, booleans, strings, views, dictionaries and lists are appended to the open chunk (bitmaps
    concatenated at bit granularity, string offsets re-based) like plain ones: 400 ragged batches of ~75 rows make 4 chunks of
    8192 rows, not 400 — and the rows still match the oracle in order.  Columns that gain a validity bitmap half-way through a
    chunk (first batches without nulls) and a second dictionary (cuts the chunk) are part of the input."""
    rnd = random.Random(31)
    n, N = 30_000, 6
    table = reference_fixture_table(n, 32)
    # the first 5 000 rows have no nulls at all in `label` / `flag` (no validity buffers in those batches)
    label = table.column("label").combine_chunks().to_pylist()
    flag = table.column("flag").combine_chunks().to_pylist()
    for r in range(5_000):
        label[r] = label[r] if label[r] is not None else "filled"
        flag[r] = bool(flag[r])
    table = table.set_column(3, table.schema.field("label"), pa.array(label, type=pa.string()))
    table = table.set_column(2, table.schema.field("flag"), pa.array(flag, type=pa.bool_()))
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=8_192)
    a, pushed = 0, 0
    while a < n:
        b = min(n, a + rnd.randint(1, 150))
        ex.push_batch(table.slice(a, b - a).combine_chunks().to_batches()[0])
        a, pushed = b, pushed + 1
    ex.finish()
    assert pushed > 300
    outs = [ex.execute(p).read_all() for p in range(N)]
    dest = orc.partition_ids([table.column(0).combine_chunks()], n, N)
    order, starts = expected_partitions(dest, N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].num_rows == want.num_rows
        assert len(outs[p].column(0).chunks) <= 4, len(outs[p].column(0).chunks)  # one batch per CHUNK and destination
        for name in table.column_names:
            got_c, want_c = outs[p].column(name).combine_chunks(), want.column(name).combine_chunks()
            if pa.types.is_dictionary(got_c.type):
                got_c, want_c = got_c.dictionary_decode(), want_c.dictionary_decode()
            assert got_c.equals(want_c), (p, name)
    ex.close()


def reference_fixture_table(n, seed):
    """Random rows of the reference's 9-column bench schema (src/execution_plans/benchmarks/fixture.rs:13-33)."""
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    words = ["", "a", "tag", "hello-world", "x" * 40, "ünï", "0123456789abcdef"]

    def maybe(v, p=0.1):
        return None if rnd.random() < p else v

    schema = pa.schema([pa.field("id", pa.int64(), False), pa.field("metric", pa.float64(), False), ("flag", pa.bool_()), ("label", pa.string()),
                        ("category", pa.dictionary(pa.int32(), pa.string())), pa.field("raw", pa.uint8(), False),
                        pa.field("ts", pa.timestamp("ns"), False), pa.field("count", pa.int32(), False), ("tags", pa.list_(pa.string()))])
    cat = pa.DictionaryArray.from_arrays(pa.array([maybe(rnd.randrange(4)) for _ in range(n)], type=pa.int32()),
                                         pa.array(["alpha", "beta", "", "gamma-" * 4], type=pa.string()))
    tags = pa.array([maybe([maybe(rnd.choice(words) + str(rnd.getrandbits(8)), 0.15) for _ in range(rnd.choice([0, 0, 1, 2, 3, 7]))], 0.12)
                     for _ in range(n)], type=pa.list_(pa.string()))
    cols = [pa.array(rng.integers(-2**40, 2**40, n), type=pa.int64()), pa.array(rng.standard_normal(n)),
            pa.array([maybe(rnd.random() < 0.5) for _ in range(n)], type=pa.bool_()),
            pa.array([maybe(rnd.choice(words) + str(rnd.getrandbits(12))) for _ in range(n)], type=pa.string()), cat,
            pa.array(rng.integers(0, 256, n).astype(np.uint8)), pa.array(rng.integers(0, 2**60, n), type=pa.timestamp("ns")),
            pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32)), tags]
    return pa.Table.from_arrays(cols, schema=schema)


@pytest.mark.parametrize("keys", [[0], [3], [4, 0], [7, 2]])
def test_reference_bench_fixture_schema_with_list_column(ctx, keys):
    """All nine columns of the reference's shuffle-bench schema, List<Utf8> included, through the operator: the schema
    that comes out is the one that went in and every destination holds the oracle's rows in the oracle's order — null
    lists, empty lists, null elements and sliced input batches included."""
    n, N = 30_000, 16
    table = reference_fixture_table(n, 21)
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash(keys, N), chunk_rows=8_192)
    cuts = [0, 3, 4_000, 4_003, 17_001, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        for rb in table.slice(a, b - a).to_batches(max_chunksize=2_500):
            ex.push_batch(rb)
    ex.finish()
    outs = collect(ex, N)
    dest = orc.partition_ids([table.column(k).combine_chunks() for k in keys], n, N)
    order, starts = expected_partitions(dest, N)
    total = 0
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].schema.equals(table.schema), (p, outs[p].schema)
        assert outs[p].num_rows == want.num_rows, p
        total += outs[p].num_rows
        for name in table.column_names:
            got_c, want_c = outs[p].column(name).combine_chunks(), want.column(name).combine_chunks()
            if pa.types.is_dictionary(got_c.type):
                got_c, want_c = got_c.dictionary_decode(), want_c.dictionary_decode()
            assert got_c.equals(want_c), (keys, p, name)
        for chunk in outs[p].column("tags").chunks:
            chunk.validate(full=True)
    assert total == n
    ex.close()


def test_list_column_edge_shapes(ctx):
    """List<Binary> and List<Utf8> payload: all-null lists, all-empty lists, a batch with no list elements at all, and a child
    array that is itself sliced (non-zero child offset)."""
    N = 5
    ids = pa.array(range(1000), type=pa.int64())
    base = pa.array([[b"a", None, b"ccc"] if i % 3 == 0 else ([] if i % 3 == 1 else None) for i in range(1200)], type=pa.list_(pa.binary()))
    sliced = base.slice(200, 1000)  # list offsets start inside the child
    empties = pa.array([[] for _ in range(1000)], type=pa.list_(pa.string()))
    nulls = pa.array([None] * 1000, type=pa.list_(pa.string()))
    flat = pa.array([str(i) for i in range(3000)], type=pa.string()).slice(500, 2000)  # child with its own offset
    fromchild = pa.ListArray.from_arrays(pa.array(range(0, 2001, 2), type=pa.int32()), flat)
    table = pa.table([ids, sliced, empties, nulls, fromchild], names=["id", "b", "e", "n", "c"])
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=512)
    for rb in table.to_batches(max_chunksize=300):
        ex.push_batch(rb)
    ex.finish()
    outs = collect(ex, N)
    dest = orc.partition_ids([ids], 1000, N)
    order, starts = expected_partitions(dest, N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].schema.equals(table.schema)
        for name in table.column_names:
            assert outs[p].column(name).combine_chunks().equals(want.column(name).combine_chunks()), (p, name)
    ex.close()


def test_bounded_pinned_pool_blocks_the_producer_until_consumers_release(ctx):
    """max_pinned_chunks: the producer's push() blocks (back-pressure) instead of growing pinned memory without bound;
    with concurrent consumers everything still arrives, in order."""
    import threading
    import time

    n, N = 400_000, 4
    cols = cfg2_columns(n, 2)
    table = pa.table(cols, names=["k", "v"])
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=16_384, pipeline_depth=2, pinned_pool_chunks=3,
                             max_pinned_chunks=3)
    got = [[] for _ in range(N)]

    def consume(p):
        for rb in ex.execute(p):
            time.sleep(0.0005)  # a slow consumer: holds its batch for a moment before dropping it
            got[p].append(rb.column(1).to_numpy().copy())
            del rb

    threads = [threading.Thread(target=consume, args=(p,)) for p in range(N)]
    for t in threads:
        t.start()
    for rb in table.to_batches(max_chunksize=8_192):
        ex.push_batch(rb)
    ex.finish()
    for t in threads:
        t.join()
    ref, counts, starts = orc.repartition_table(cols, [0], N, 8192, 1)
    for p in range(N):
        assert np.array_equal(np.concatenate(got[p]), ref[1][starts[p]:starts[p + 1]])
    ex.close()


def test_pinned_chunks_are_reused_by_the_next_operator_of_the_same_shape(ctx):
    """The worker context keeps the pinned output chunks of finished operators: a second operator with the same column
    layout and chunk size pins nothing new (the reference's workers get this from their caching allocator,
    benchmarks/cdk/bin/worker.rs:32), a different layout does not take them, and the results stay bit-identical."""
    n, N = 200_000, 8
    cols = cfg2_columns(n, 3)
    table = pa.table(cols, names=["k", "a", "b"])
    ref, counts, starts = orc.repartition_table(cols, [0], N, 8192, 1)

    def run(schema_table, chunk_rows):
        ex = dfd.RepartitionExec(ctx, schema_table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=chunk_rows, pinned_pool_chunks=4)
        for rb in schema_table.to_batches(max_chunksize=8_192):
            ex.push_batch(rb)
        ex.finish()
        outs = collect(ex, N)
        st = ex.stats()
        ex.close()
        return outs, st

    outs, st1 = run(table, 32_768)
    assert st1["pinned_chunks"] >= 4 and st1["pinned_chunks_allocated"] + st1["pinned_chunks_reused"] == st1["pinned_chunks"]
    for p in range(N):
        assert np.array_equal(outs[p].column("b").to_numpy(), ref[2][starts[p]:starts[p + 1]])
    del outs  # the last output batch returns its chunk; the pool dies and hands its chunks to the context
    outs, st2 = run(table, 32_768)
    assert st2["pinned_chunks_reused"] >= 4 and st2["pinned_chunks_allocated"] == 0, st2
    for p in range(N):
        assert outs[p].num_rows == counts[p]
        for c, name in enumerate(["k", "a", "b"]):
            assert np.array_equal(outs[p].column(name).to_numpy(), ref[c][starts[p]:starts[p + 1]])
    del outs
    # another chunk size / another layout: nothing is taken over
    _, st3 = run(table, 16_384)
    assert st3["pinned_chunks_reused"] == 0
    _, st4 = run(table.select(["k", "a"]), 32_768)
    assert st4["pinned_chunks_reused"] == 0
    assert st4["ns_push"] > 0


def test_large_binary_and_fixed_size_binary_travel_as_payload(ctx):
    """LargeBinary (int64 offsets + bytes) and FixedSizeBinary(16) / (4) — UUIDs — move through the operator as payload with
    their types intact; as hash KEYS they are refused when the operator is created (DataFusion hashes them as byte slices,
    which the device does not do for these layouts)."""
    rnd = random.Random(21)
    n, N = 30_000, 6
    key = pa.array([rnd.getrandbits(40) for _ in range(n)], type=pa.int64())
    uuid = pa.array([rnd.randbytes(16) for _ in range(n)], type=pa.binary(16))
    tag4 = pa.array([None if rnd.random() < 0.1 else rnd.randbytes(4) for _ in range(n)], type=pa.binary(4))
    blob = pa.array([None if rnd.random() < 0.1 else rnd.randbytes(rnd.randint(0, 40)) for _ in range(n)], type=pa.large_binary())
    table = pa.table([key, uuid, tag4, blob], names=["key", "uuid", "tag4", "blob"])
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=8_192)
    for rb in table.to_batches(max_chunksize=3_000):
        ex.push_batch(rb)
    ex.finish()
    outs = collect(ex, N)
    dest = orc.partition_ids([key], n, N)
    order, starts = expected_partitions(dest, N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].schema.equals(table.schema), p
        assert outs[p].equals(want), p
    ex.close()
    for bad_key in (1, 2, 3):
        with pytest.raises(dfd.DfdError) as e:
            dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0, bad_key], N))
        assert e.value.status == 6 and "cannot be hash keys" in str(e.value)


def test_lists_of_primitives_travel_as_payload(ctx):
    """List<Int64> / List<Float32> / List<Decimal128> (the partial states of array_agg / median) through the operator: nullable
    lists, nullable elements, empty lists, sliced batches — every destination equals the oracle's rows in order."""
    import decimal

    rnd = random.Random(33)
    n, N = 20_000, 5
    key = pa.array([rnd.getrandbits(40) for _ in range(n)], type=pa.int64())

    def lists(make, typ, null_rows, null_elems):
        rows = []
        for _ in range(n):
            if rnd.random() < null_rows:
                rows.append(None)
            else:
                rows.append([None if rnd.random() < null_elems else make() for _ in range(rnd.choice([0, 0, 1, 2, 5]))])
        return pa.array(rows, type=pa.list_(typ))

    l64 = lists(lambda: rnd.getrandbits(60) - (1 << 59), pa.int64(), 0.1, 0.15)
    f32 = lists(lambda: float(rnd.randint(-1000, 1000)) / 8, pa.float32(), 0.0, 0.0)
    dec = lists(lambda: decimal.Decimal(rnd.randint(-10**12, 10**12)).scaleb(-2), pa.decimal128(18, 2), 0.05, 0.1)
    table = pa.table([key, l64, f32, dec], names=["key", "l64", "f32", "dec"])
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=4_096)
    cuts = [0, 7, 3_000, 3_001, 11_111, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        for rb in table.slice(a, b - a).to_batches(max_chunksize=1_500):
            ex.push_batch(rb)
    ex.finish()
    outs = collect(ex, N)
    dest = orc.partition_ids([key], n, N)
    order, starts = expected_partitions(dest, N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        assert outs[p].schema.equals(table.schema), p
        outs[p].validate(full=True)
        for name in table.column_names:
            assert outs[p].column(name).combine_chunks().equals(want.column(name).combine_chunks()), (p, name)
    ex.close()
    with pytest.raises(dfd.DfdError) as e:
        dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([1], N))
    assert e.value.status == 6


def test_equal_dictionaries_of_consecutive_batches_share_a_chunk(ctx):
    """Readers re-materialise a column's dictionary for every batch: batches whose dictionaries are different OBJECTS with the same
    values are appended to the same chunk (one launch, one output batch per destination), a batch with other values still cuts it."""
    rnd = random.Random(3)
    values = ["red", "green", None, "blue-" * 4, ""]
    n_batches, rows, N = 20, 1_000, 4
    batches, all_rows = [], []
    for b in range(n_batches):
        vals = list(values) if b != 12 else ["other", "values", None, "here", "!"]   # batch 12 really has another dictionary
        dictionary = pa.array(list(vals), type=pa.string())                           # a fresh object (fresh buffers) every time
        idx = pa.array([rnd.choice([None, 0, 1, 2, 3, 4]) for _ in range(rows)], type=pa.int32())
        key = pa.array([rnd.getrandbits(40) for _ in range(rows)], type=pa.int64())
        batches.append(pa.record_batch([key, pa.DictionaryArray.from_arrays(idx, dictionary)], names=["key", "cat"]))
        all_rows.append(pa.table([key, pa.DictionaryArray.from_arrays(idx, dictionary).dictionary_decode()], names=["key", "cat"]))
    plain = pa.concat_tables(all_rows)
    for keys in ([0], [1, 0]):
        ex = dfd.RepartitionExec(ctx, batches[0].schema, dfd.Partitioning.Hash(keys, N), chunk_rows=8_192)
        for rb in batches:
            ex.push_batch(rb)
        ex.finish()
        readers = [ex.execute(p) for p in range(N)]
        outs = [[rb for rb in r] for r in readers]
        dest = orc.partition_ids([plain.column(k) for k in keys], plain.num_rows, N)
        order, starts = expected_partitions(dest, N)
        for p in range(N):
            want = plain.take(pa.array(order[starts[p]:starts[p + 1]]))
            got_key = pa.concat_arrays([rb.column(0) for rb in outs[p]])
            got_cat = pa.concat_arrays([rb.column(1).dictionary_decode() for rb in outs[p]])
            assert got_key.equals(want.column("key").combine_chunks()) and got_cat.equals(want.column("cat").combine_chunks()), (keys, p)
            # 20 000 rows in chunks of 8 192, cut once more before and after batch 12: a handful of output batches, not 20
            assert len(outs[p]) <= 6, (keys, p, len(outs[p]))
        del outs, readers
        ex.close()
