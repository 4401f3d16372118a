"""Randomised schemas and batchings through the host operator on the CPU harness (tests/test_exec_cpu_harness.py): every
supported column kind — fixed widths, nullable, boolean, Utf8 / LargeUtf8 / Binary, views, dictionaries (changing between
batches, null values, null indices), List<Utf8 / Binary> — as payload and, where allowed, as hash key; ragged and sliced
input batches against chunk sizes that cut them anywhere.  Every destination must hold the rows the oracle's partition
ids select, in input order, with the input schema.  Every case runs twice: host batches through push, and the same batches
as device batches (host stand-ins, tests/device_batches.py) through push_device on the device harness library
(tests/test_exec_device_input_cpu_harness.py), a superset of the host one."""
import random

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as orc
from tests import device_batches as DB
from tests.test_exec_device_input_cpu_harness import harness  # noqa: F401  (module-scoped fixture: builds the harness once)
from tests.util import expected_partitions


def _strings(rnd, n, null_p, maxlen=30):
    alphabet = "abcdefghijklmnopqrstuvwxyzäß0123456789 "
    return [None if rnd.random() < null_p else "".join(rnd.choice(alphabet) for _ in range(rnd.choice([0, 1, 3, 12, 13, rnd.randint(0, maxlen)])))
            for _ in range(n)]


def _column(rnd, rng, kind, n):
    """(array fed to the operator, equivalent array pyarrow can take()/compare, may be a hash key)"""
    if kind == "i64":
        a = pa.array(rng.integers(-(2**62), 2**62, n, dtype=np.int64))
        return a, a, True
    if kind == "i32?":
        a = pa.array([None if rnd.random() < 0.15 else rnd.randint(-(2**31), 2**31 - 1) for _ in range(n)], type=pa.int32())
        return a, a, True
    if kind == "u8":
        a = pa.array(rng.integers(0, 256, n).astype(np.uint8))
        return a, a, True
    if kind == "f64":
        a = pa.array(rng.standard_normal(n))
        return a, a, True
    if kind == "bool?":
        a = pa.array([rnd.choice([None, True, False]) for _ in range(n)], type=pa.bool_())
        return a, a, True
    if kind == "date32":
        a = pa.array(rng.integers(0, 20000, n).astype(np.int32)).cast(pa.date32())
        return a, a, True
    if kind == "dec128?":
        import decimal

        a = pa.array([None if rnd.random() < 0.1 else decimal.Decimal(rnd.randint(-10**15, 10**15)).scaleb(-3) for _ in range(n)], type=pa.decimal128(20, 3))
        return a, a, True
    if kind == "utf8?":
        a = pa.array(_strings(rnd, n, 0.1), type=pa.string())
        return a, a, True
    if kind == "large_utf8":
        a = pa.array(_strings(rnd, n, 0.0), type=pa.large_string())
        return a, a, True
    if kind == "binary?":
        a = pa.array([None if rnd.random() < 0.2 else rnd.randbytes(rnd.randint(0, 20)) for _ in range(n)], type=pa.binary())
        return a, a, True
    # (view arrays WITHOUT any out-of-line value have no data buffer, and pyarrow's C Data export of such an array crashes —
    # inside libarrow, before the operator sees anything: keep one long value in every view column)
    if kind == "string_view?":
        vals = _strings(rnd, n, 0.1, 40)
        vals[rnd.randrange(n)] = "a-value-longer-than-twelve-bytes"
        p = pa.array(vals, type=pa.string())
        return p.cast(pa.string_view()), p, True
    if kind == "binary_view":
        vals = [rnd.randbytes(rnd.choice([0, 5, 12, 13, 30])) for _ in range(n)]
        vals[rnd.randrange(n)] = rnd.randbytes(21)
        p = pa.array(vals, type=pa.binary())
        return p.cast(pa.binary_view()), p, False
    if kind == "large_binary?":
        a = pa.array([None if rnd.random() < 0.1 else rnd.randbytes(rnd.randint(0, 25)) for _ in range(n)], type=pa.large_binary())
        return a, a, False  # payload only: DataFusion hashes it as a byte slice
    if kind == "uuid":
        a = pa.array([rnd.randbytes(16) for _ in range(n)], type=pa.binary(16))
        return a, a, False
    if kind == "fsb4?":
        a = pa.array([None if rnd.random() < 0.1 else rnd.randbytes(4) for _ in range(n)], type=pa.binary(4))
        return a, a, False
    if kind.startswith("dict"):
        index_type = {"dict8": pa.int8(), "dict16": pa.int16(), "dict32": pa.int32()}[kind]
        # the dictionary CHANGES along the column: pieces with their own values (the operator cuts its chunk there)
        pieces, left = [], n
        while left > 0:
            m = min(left, rnd.randint(1, max(1, n // 2)))
            values = pa.array([None if rnd.random() < 0.2 else f"v{rnd.randint(0, 50)}" + "x" * rnd.randint(0, 15) for _ in range(rnd.randint(1, 20))], type=pa.string())
            idx = pa.array([None if rnd.random() < 0.1 else rnd.randrange(len(values)) for _ in range(m)], type=index_type)
            pieces.append(pa.DictionaryArray.from_arrays(idx, values))
            left -= m
        # (pyarrow cannot unify dictionaries that hold null values: the expectation works on the decoded strings, which is also
        # what DataFusion's hash_dictionary hashes)
        return pa.chunked_array(pieces), pa.chunked_array([p.dictionary_decode() for p in pieces]), True
    if kind in ("list<i64>?", "list<f32>"):
        prim = kind == "list<f32>"
        rows = []
        for _ in range(n):
            if not prim and rnd.random() < 0.1:
                rows.append(None)
            else:
                rows.append([float(rnd.randint(-99, 99)) / 4 if prim else (None if rnd.random() < 0.2 else rnd.getrandbits(50)) for _ in range(rnd.randint(0, 4))])
        a = pa.array(rows, type=pa.list_(pa.float32() if prim else pa.int64()))
        return a, a, False
    if kind in ("list<utf8>?", "list<binary>"):
        binary = kind == "list<binary>"
        rows = []
        for _ in range(n):
            if not binary and rnd.random() < 0.1:
                rows.append(None)
            else:
                k = rnd.randint(0, 4)
                rows.append([rnd.randbytes(rnd.randint(0, 9)) for _ in range(k)] if binary else _strings(rnd, k, 0.15, 12))
        a = pa.array(rows, type=pa.list_(pa.binary() if binary else pa.string()))
        return a, a, False
    raise AssertionError(kind)


KINDS = ["i64", "i32?", "u8", "f64", "bool?", "date32", "dec128?", "utf8?", "large_utf8", "binary?", "string_view?", "binary_view", "dict8", "dict16",
         "dict32", "list<utf8>?", "list<binary>", "large_binary?", "uuid", "fsb4?", "list<i64>?", "list<f32>"]


@pytest.mark.parametrize("seed", range(24))
def test_random_schema_and_batching_matches_the_oracle(harness, seed):  # noqa: F811
    ns, ctx, _ = harness
    rnd = random.Random(1000 + seed)
    rng = np.random.Generator(np.random.PCG64(1000 + seed))
    n = rnd.choice([1, 63, 1000, 5000, 20_000])
    kinds = rnd.sample(KINDS, rnd.randint(1, 7))
    if rnd.random() < 0.5 and "i64" not in kinds:
        kinds.insert(0, "i64")
    cols = [_column(rnd, rng, k, n) for k in kinds]
    names = [f"c{i}_{k}" for i, k in enumerate(kinds)]
    fed = pa.table([c[0] for c in cols], names=names)
    plain = pa.table([c[1] for c in cols], names=names)
    keyable = [i for i, c in enumerate(cols) if c[2]]
    if not keyable:
        fed = fed.append_column("k", pa.array(rng.integers(0, 1000, n, dtype=np.int64)))
        plain = plain.append_column("k", fed.column("k"))
        keyable = [fed.num_columns - 1]
    keys = rnd.sample(keyable, rnd.randint(1, min(3, len(keyable))))
    N = rnd.choice([1, 2, 3, 8, 12, 48, 257])
    chunk_rows = rnd.choice([64, 1000, 4096, 0])
    depth = rnd.choice([0, 2, 4])
    # ragged feeding: random cuts, each cut re-batched with a random maximum size (slices with odd offsets, empty batches)
    cuts = sorted({0, n} | {rnd.randint(0, n) for _ in range(rnd.randint(0, 6))})
    batches = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        batches += fed.slice(a, b - a).to_batches(max_chunksize=rnd.choice([7, 100, 8192, 100_000]))
    if rnd.random() < 0.3:
        batches.append(fed.slice(0, 0).to_batches()[0] if fed.slice(0, 0).to_batches() else pa.RecordBatch.from_pylist([], schema=fed.schema))
    dest = orc.partition_ids([plain.column(k) for k in keys], n, N)
    order, starts = expected_partitions(dest, N)
    for device in (False, True):
        ex = ns.RepartitionExec(ctx, fed.schema, ns.Partitioning.Hash(keys, N), chunk_rows=chunk_rows, pipeline_depth=depth)
        for rb in batches:
            if device:
                ex.push_device_batch(DB.DeviceBatch(rb, alloc=DB.host_alloc).device_array)
            else:
                ex.push_batch(rb)
        ex.finish()
        outs = [ex.execute(p).read_all() for p in range(N)]
        st = ex.stats()
        assert st["rows_in"] == n and st["rows_out"] == n
        for p in range(N):
            want = plain.take(pa.array(order[starts[p]:starts[p + 1]]))
            got = outs[p]
            assert got.schema.equals(fed.schema), (kinds, p, device)
            assert got.num_rows == want.num_rows, (kinds, keys, N, p, device)
            if got.num_rows:
                got.validate(full=True)
            for name in names:
                g, w = got.column(name), want.column(name).combine_chunks()
                if pa.types.is_dictionary(g.type):  # decode chunk by chunk (the chunks of a destination may carry different dictionaries)
                    g = pa.chunked_array([c.dictionary_decode() for c in g.chunks], type=g.type.value_type)
                g = g.combine_chunks()
                assert g.cast(w.type).equals(w), (kinds, keys, N, chunk_rows, p, name, device)
        ex.close()


def test_long_strings_grow_the_chunk_buffers(harness):  # noqa: F811
    """Strings of tens of kilobytes (a plain column, a view column and the elements of a list): the chunk's device byte
    buffers and the pinned landing buffers grow while batches are appended, without losing what is already staged."""
    ns, ctx, _ = harness
    rnd = random.Random(3)
    n, N = 1500, 5
    big = pa.array([None if rnd.random() < 0.05 else ("x" * rnd.choice([0, 10, 3000, 20000]) + str(i)) for i in range(n)], type=pa.string())
    key = pa.array(np.arange(n, dtype=np.int64))
    lst = pa.array([[("y" * rnd.choice([1, 500, 9000])) + str(i) for _ in range(rnd.randint(0, 3))] for i in range(n)], type=pa.list_(pa.string()))
    fed = pa.table([key, big, lst, big.cast(pa.string_view())], names=["k", "s", "l", "v"])
    plain = pa.table([key, big, lst, big], names=["k", "s", "l", "v"])
    dest = orc.partition_ids([key], n, N)
    order, starts = expected_partitions(dest, N)
    for chunk_rows in (64, 1000):
        ex = ns.RepartitionExec(ctx, fed.schema, ns.Partitioning.Hash([0], N), chunk_rows=chunk_rows)
        for rb in fed.to_batches(max_chunksize=333):
            ex.push_batch(rb)
        ex.finish()
        outs = [ex.execute(p).read_all() for p in range(N)]
        for p in range(N):
            want = plain.take(pa.array(order[starts[p]:starts[p + 1]]))
            for name in fed.column_names:
                g, w = outs[p].column(name).combine_chunks(), want.column(name).combine_chunks()
                assert g.cast(w.type).equals(w), (chunk_rows, p, name)
        ex.close()
