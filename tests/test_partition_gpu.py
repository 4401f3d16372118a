"""GPU parity tests: the CUDA path (through the C ABI) vs the CPU oracle.

Bar: bit-exact (integer / byte / index work) — identical destination ids,
identical per-destination counts, and identical per-destination row ORDER
(the kernel is stable, invariant iii), on the same seeded inputs.
"""
import random

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from oracle import oracle as orc
from tests.util import cfg2_columns, edge_sizes, expected_partitions, golden

pytestmark = pytest.mark.gpu

ALL_N = [1, 2, 3, 7, 8, 12, 16, 48, 64, 255, 256, 1000, 4096]


def dev_cols(ctx, arrays):
    return [dfd.DeviceColumn.from_arrow(ctx, a if isinstance(a, pa.Array) else pa.array(a)) for a in arrays]


def gpu_ids(ctx, arrays, key_cols, N, seeds=None):
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N), seeds)
    return part.partition_ids(dev_cols(ctx, arrays), len(arrays[0]))


# ---------------------------------------------------------------- hashing ----

def test_golden_vectors_on_gpu(ctx):
    g = golden()
    for width, typ in [(1, pa.uint8()), (2, pa.uint16()), (4, pa.uint32()), (8, pa.uint64())]:
        ents = [e for e in g["ints"] if e["width"] == width]
        arr = pa.array([int(e["value"]) for e in ents], type=typ)
        for N in (8, 12, 4096):
            ids = gpu_ids(ctx, [arr], [0], N)
            assert ids.tolist() == [int(e["hash"], 16) % N for e in ents]
    ents = [e for e in g["ints"] if e["width"] == 16]
    raw = b"".join(int(e["value"]).to_bytes(16, "little") for e in ents)
    arr = pa.Array.from_buffers(pa.decimal128(38, 0), len(ents), [None, pa.py_buffer(raw)])
    ids = gpu_ids(ctx, [arr], [0], 1000)
    assert ids.tolist() == [int(e["hash"], 16) % 1000 for e in ents]
    strs = [bytes.fromhex(e["hex"]) for e in g["strings"]]
    b = pa.array(strs, type=pa.binary())
    s = pa.Array.from_buffers(pa.string(), len(b), b.buffers())
    assert gpu_ids(ctx, [s], [0], 4096).tolist() == [int(e["str_hash"], 16) % 4096 for e in g["strings"]]
    assert gpu_ids(ctx, [b], [0], 4096).tolist() == [int(e["bytes_hash"], 16) % 4096 for e in g["strings"]]
    for e in g["seeded"]:
        ids = gpu_ids(ctx, [pa.array([int(e["value"])], type=pa.int64())], [0], 4093, e["seeds"])
        assert ids[0] == int(e["hash"], 16) % 4093
    rows = g["rows_i64_i32_utf8"]
    a = pa.array([None if r["i64"] is None else int(r["i64"]) for r in rows], type=pa.uint64())
    bb = pa.array([None if r["i32"] is None else int(r["i32"]) for r in rows], type=pa.uint32())
    cb = pa.array([None if r["utf8_hex"] is None else bytes.fromhex(r["utf8_hex"]) for r in rows], type=pa.binary())
    cs = pa.Array.from_buffers(pa.string(), len(cb), cb.buffers(), null_count=cb.null_count)
    for N in (1, 2, 3, 8, 12, 16, 48, 1000, 4096):
        ids = gpu_ids(ctx, [a, bb, cs], [0, 1, 2], N)
        assert ids.tolist() == [r["mod"][str(N)] for r in rows]


@pytest.mark.parametrize("N", ALL_N)
def test_partition_ids_i64_all_moduli(ctx, N):
    key = cfg2_columns(200_003, 1)[0]
    assert np.array_equal(gpu_ids(ctx, [key], [0], N), orc.partition_ids([key], len(key), N))


@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64, np.uint32, np.float32, np.float64])
def test_partition_ids_fixed_widths(ctx, dtype):
    rng = np.random.Generator(np.random.PCG64(3))
    n = 50_001
    if np.issubdtype(dtype, np.floating):
        v = rng.standard_normal(n).astype(dtype)
    else:
        ii = np.iinfo(dtype)
        v = rng.integers(ii.min, ii.max, n, dtype=dtype, endpoint=True)
    assert np.array_equal(gpu_ids(ctx, [v], [0], 12), orc.partition_ids([v], n, 12))


def test_partition_ids_multi_key_nulls_strings_offsets(ctx):
    rnd = random.Random(11)
    n = 20_000
    a = pa.array([rnd.choice([None, rnd.getrandbits(63)]) for _ in range(n)], type=pa.int64())
    s = pa.array([rnd.choice([None, "", "a", "x" * rnd.randint(0, 70), "päö" * rnd.randint(0, 9)]) for _ in range(n)], type=pa.string())
    bl = pa.array([rnd.choice([None, True, False]) for _ in range(n)])
    d = pa.array([rnd.choice([None, rnd.getrandbits(15)]) for _ in range(n)], type=pa.int16())
    ls = s.cast(pa.large_string())
    bn = s.cast(pa.binary())
    for keys in ([a], [a, s], [s], [bl, d], [a, s, bl, d], [ls, a], [bn], [d, bn, a]):
        for N in (8, 48, 1000):
            got = gpu_ids(ctx, keys, list(range(len(keys))), N)
            assert np.array_equal(got, orc.partition_ids(keys, n, N)), (len(keys), N)
    # sliced arrays (Arrow offset != 0, validity + offsets not byte aligned)
    sl = [a.slice(13, 9000), s.slice(13, 9000), bl.slice(13, 9000)]
    assert np.array_equal(gpu_ids(ctx, sl, [0, 1, 2], 12), orc.partition_ids(sl, 9000, 12))


def test_all_null_single_key_goes_to_partition_zero(ctx):
    a = pa.array([None] * 1000, type=pa.int64())
    assert not gpu_ids(ctx, [a], [0], 8).any()


# ---------------------------------------------------------------- scatter ----

def run_partition(ctx, arrays, key_cols, N):
    n = len(arrays[0])
    cols = dev_cols(ctx, arrays)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N))
    outs, starts = part.partition(cols, n)
    return outs, starts


@pytest.mark.parametrize("n_rows", edge_sizes())
def test_scatter_matches_oracle_ragged_sizes(ctx, n_rows):
    cols = cfg2_columns(n_rows, 3)
    outs, starts = run_partition(ctx, cols, [0], 8)
    ref_outs, ref_counts, ref_starts = orc.repartition_table(cols, [0], 8, 8192, 1)
    assert np.array_equal(starts, ref_starts)
    for c in range(3):
        got = outs[c].keep[-1].download(np.int64, n_rows)
        assert np.array_equal(got, ref_outs[c]), c


@pytest.mark.parametrize("N", ALL_N)
def test_scatter_cfg1_shape_all_moduli(ctx, N):
    """cfg-1: 1M rows, schema (k: Int64, v: Int64), v = row index."""
    rng = np.random.Generator(np.random.PCG64(1))
    n = 1_000_000
    k = rng.integers(0, 2**63 - 1, n, dtype=np.int64)
    v = np.arange(n, dtype=np.int64)
    outs, starts = run_partition(ctx, [k, v], [0], N)
    ref_outs, _, ref_starts = orc.repartition_table([k, v], [0], N, 8192, 1)
    assert np.array_equal(starts, ref_starts)
    assert np.array_equal(outs[0].keep[-1].download(np.int64, n), ref_outs[0])
    assert np.array_equal(outs[1].keep[-1].download(np.int64, n), ref_outs[1])


def test_scatter_cfg2_shape_8_cols_two_keys(ctx):
    cols = cfg2_columns(1 << 20, 8)
    for keys in ([0], [0, 1]):
        outs, starts = run_partition(ctx, cols, keys, 8)
        ref_outs, _, ref_starts = orc.repartition_table(cols, keys, 8, 8192, 1)
        assert np.array_equal(starts, ref_starts)
        for c in range(8):
            assert np.array_equal(outs[c].keep[-1].download(np.int64, 1 << 20), ref_outs[c])


def test_scatter_skew_single_hot_key(ctx):
    n = 300_000
    k = np.full(n, 12345, dtype=np.int64)
    k[::1000] = np.arange(0, n, 1000)
    v = np.arange(n, dtype=np.int64)
    outs, starts = run_partition(ctx, [k, v], [0], 16)
    ref_outs, _, ref_starts = orc.repartition_table([k, v], [0], 16, 8192, 1)
    assert np.array_equal(starts, ref_starts)
    assert np.array_equal(outs[1].keep[-1].download(np.int64, n), ref_outs[1])


def test_scatter_mixed_widths_nulls_and_bools(ctx):
    rnd = random.Random(2)
    rng = np.random.Generator(np.random.PCG64(2))
    n = 70_001
    key = pa.array([rnd.choice([None, rnd.getrandbits(40)]) for _ in range(n)], type=pa.int64())
    c8 = pa.array(rng.integers(0, 255, n, dtype=np.uint8))
    c16 = pa.array(rng.integers(-30000, 30000, n, dtype=np.int16))
    c32 = pa.array([rnd.choice([None, rnd.getrandbits(31)]) for _ in range(n)], type=pa.int32())
    f64 = pa.array(rng.standard_normal(n))
    bl = pa.array([rnd.choice([None, True, False]) for _ in range(n)])
    raw = rng.integers(0, 255, n * 16, dtype=np.uint8).tobytes()
    dec = pa.Array.from_buffers(pa.decimal128(38, 0), n, [None, pa.py_buffer(raw)])
    arrays = [key, c8, c16, c32, f64, bl, dec]
    for N in (8, 48):
        outs, starts = run_partition(ctx, arrays, [0, 3], N)
        dest = orc.partition_ids([key, c32], n, N)
        order, ref_starts = expected_partitions(dest, N)
        assert np.array_equal(starts, ref_starts)
        idx = pa.array(order)
        for c, arr in enumerate(arrays):
            want = arr.take(idx)
            got = outs[c].to_arrow(ctx, 0, n)
            assert got.equals(want), (N, c, arr.type)


def test_scatter_many_columns_multiple_launches(ctx):
    n = 10_000
    cols = cfg2_columns(n, 30)
    outs, starts = run_partition(ctx, cols, [0], 8)
    ref_outs, _, ref_starts = orc.repartition_table(cols, [0], 8, 8192, 1)
    assert np.array_equal(starts, ref_starts)
    for c in (0, 1, 23, 24, 29):
        assert np.array_equal(outs[c].keep[-1].download(np.int64, n), ref_outs[c])


def test_error_behaviour(ctx):
    with pytest.raises(dfd.DfdError) as e:
        dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 0))
    assert e.value.status == 1
    with pytest.raises(dfd.DfdError):
        dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 5000))
    with pytest.raises(dfd.DfdError):
        dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([], 8))
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([3], 8))
    with pytest.raises(dfd.DfdError) as e:
        part.partition_ids(dev_cols(ctx, [np.arange(10, dtype=np.int64)]), 10)
    assert "out of range" in str(e.value)


# ------------------------------------------------ full size (BASELINE cfg-2) ----

def test_full_size_cfg2_properties(ctx):
    """2^26 rows x 8 x i64, N=8: size-independent properties, checked on device.
    (torch is only the checker's array library here.)"""
    import torch

    n, C, N = 1 << 26, 8, 8
    g = torch.Generator(device="cuda").manual_seed(42)
    key = torch.randint(-(2**63), 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    rid = torch.arange(n, dtype=torch.int64, device="cuda")
    ins = [key] + [rid * 8 + j for j in range(1, C)]
    outs = [torch.empty_like(t) for t in ins]
    torch.cuda.synchronize()
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    _, starts = part.partition([dfd.DeviceColumn.from_torch(t) for t in ins], n,
                               [dfd.DeviceColumn.from_torch(t) for t in outs])
    # (1) counts == oracle counts on the same keys
    key_h = key.cpu().numpy()
    dest = orc.partition_ids([key_h], n, N)
    assert np.array_equal(np.diff(starts), np.bincount(dest, minlength=N))
    # (2) every output row landed in the partition its key hashes to (re-hash the OUTPUT on GPU and on CPU sample)
    ids_out = part.partition_ids([dfd.DeviceColumn.from_torch(outs[0])], n)
    for p in range(N):
        seg = ids_out[starts[p]:starts[p + 1]]
        assert (seg == p).all()
    # (3) rows are intact: col j == row_id*8 + j for the same row_id, and key matches the input key of that row
    rid_out = (outs[1] - 1) >> 3
    for j in range(2, C):
        assert torch.equal(outs[j], rid_out * 8 + j)
    assert torch.equal(key[rid_out], outs[0])
    # (4) stability: row ids strictly increase inside each destination (=> also a permutation, no dup / loss)
    for p in range(N):
        seg = rid_out[starts[p]:starts[p + 1]]
        assert bool((seg[1:] > seg[:-1]).all())
    assert int(rid_out.sum().item()) == n * (n - 1) // 2
    # (5) first 1M rows of partition 0 equal the oracle's order exactly
    want = np.nonzero(dest == 0)[0][:1_000_000]
    assert np.array_equal(rid_out[starts[0]:starts[0] + len(want)].cpu().numpy(), want)


# ------------------------------------------- variable-width payload (K4) ----

def _rand_strings(rnd, n, null_frac=0.1, empty_frac=0.3, max_len=40):
    out = []
    for _ in range(n):
        x = rnd.random()
        if x < null_frac:
            out.append(None)
        elif x < null_frac + empty_frac:
            out.append("")
        else:
            out.append("".join(rnd.choice("abcdefghijklmnopqrstuvwxyzäß0123456789 ") for _ in range(rnd.randint(1, max_len))))
    return out


@pytest.mark.parametrize("N", [1, 6, 8, 48])
def test_scatter_variable_width_payload_and_keys(ctx, N):
    """cfg-5 shape in small: Hash([UserID: Int64, SearchPhrase: Utf8], N) with Utf8/LargeUtf8/Binary payload."""
    rnd = random.Random(29)
    n = 30_011
    uid = pa.array([rnd.choice([rnd.getrandbits(20), rnd.getrandbits(62)]) for _ in range(n)], type=pa.int64())
    phrase = pa.array(_rand_strings(rnd, n, 0.05, 0.7, 60), type=pa.string())
    big = pa.array(_rand_strings(rnd, n, 0.2, 0.1, 100), type=pa.large_string())
    binv = pa.array([None if s is None else s.encode() for s in _rand_strings(rnd, n, 0.1, 0.1, 17)], type=pa.binary())
    cnt = pa.array(np.arange(n, dtype=np.int32))
    arrays = [uid, phrase, big, binv, cnt]
    outs, starts = run_partition(ctx, arrays, [0, 1], N)
    dest = orc.partition_ids([uid, phrase], n, N)
    order, ref_starts = expected_partitions(dest, N)
    assert np.array_equal(starts, ref_starts)
    for p in range(N):
        idx = pa.array(order[starts[p]:starts[p + 1]])
        for c, arr in enumerate(arrays):
            got = outs[c].to_arrow(ctx, int(starts[p]), int(starts[p + 1]))
            assert got.equals(arr.take(idx)), (N, p, c)


def _long_binary(rng, n):
    """Binary values of 0 to 3000 bytes, most of them 256 to 1100 (the byte copy's long-value branch), about 5% null.
    Lengths are random, so a long value's source and destination offsets agree mod 8 for some values and not others."""
    lens = np.where(rng.random(n) < 0.7, rng.integers(256, 1101, n), rng.integers(0, 3001, n))
    blob = rng.integers(32, 127, int(lens.sum()), dtype=np.uint8).tobytes()  # (printable ASCII: valid UTF-8 too)
    ends = np.cumsum(lens)
    null = rng.random(n) < 0.05
    return pa.array([None if null[i] else blob[ends[i] - lens[i]:ends[i]] for i in range(n)], type=pa.binary())


@pytest.mark.parametrize("N", [8, 48])
def test_scatter_long_variable_width_values_as_keys_and_payload(ctx, N):
    """Utf8 / LargeUtf8 / Binary values up to 3000 bytes, whole and sliced, as the hash keys (long-string hashing loops
    many times) and as the payload they move with."""
    rng = np.random.Generator(np.random.PCG64(N))
    n = 6_007
    bn = _long_binary(rng, n)
    s = pa.Array.from_buffers(pa.string(), n, _long_binary(rng, n).buffers(), null_count=-1)
    ls = _long_binary(rng, n).cast(pa.string()).cast(pa.large_string())
    idx_col = pa.array(np.arange(n, dtype=np.int32))
    for arrays in ([s, ls, bn, idx_col], [a.slice(7, n - 20) for a in (s, ls, bn, idx_col)]):
        m = len(arrays[0])
        outs, starts = run_partition(ctx, arrays, [0, 1, 2], N)
        order, ref_starts = expected_partitions(orc.partition_ids(arrays[:3], m, N), N)
        assert np.array_equal(starts, ref_starts)
        for p in range(N):
            idx = pa.array(order[starts[p]:starts[p + 1]])
            for c, arr in enumerate(arrays):
                got = outs[c].to_arrow(ctx, int(starts[p]), int(starts[p + 1]))
                assert got.equals(arr.take(idx)), (N, m, p, c)


def test_variable_width_sliced_input_and_empty(ctx):
    rnd = random.Random(5)
    s = pa.array(_rand_strings(rnd, 5000, 0.1, 0.2, 30), type=pa.string())
    k = pa.array(np.arange(5000, dtype=np.int64))
    sl = [k.slice(77, 3001), s.slice(77, 3001)]
    outs, starts = run_partition(ctx, sl, [0], 5)
    dest = orc.partition_ids([sl[0]], 3001, 5)
    order, ref_starts = expected_partitions(dest, 5)
    assert np.array_equal(starts, ref_starts)
    assert outs[1].to_arrow(ctx, 0, 3001).equals(sl[1].take(pa.array(order)))
    outs, starts = run_partition(ctx, [k.slice(0, 0), s.slice(0, 0)], [0], 4)
    assert not starts.any()


def test_variable_width_capacity_error(ctx):
    s = pa.array(["hello", "world", "x" * 100], type=pa.string())
    k = pa.array([1, 2, 3], type=pa.int64())
    cols = dev_cols(ctx, [k, s])
    outs = [dfd.DeviceColumn.empty_like(ctx, c, 3) for c in cols]
    outs[1].values_bytes = 8  # too small
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 2))
    with pytest.raises(dfd.DfdError) as e:
        part.partition(cols, 3, outs)
    assert e.value.status == 7


def test_context_closes_its_children_first(built):
    """Destroy order must not matter to the caller: closing the worker context first
    tears down the partitioners / buffers / operators created on it."""
    import gc

    c2 = dfd.WorkerContext(0)
    part = dfd.HashPartitioner(c2, dfd.Partitioning.Hash([0], 4))
    buf = c2.alloc(1024)
    ex = dfd.RepartitionExec(c2, pa.schema([("k", pa.int64())]), dfd.Partitioning.Hash([0], 2), chunk_rows=1024)
    c2.close()
    del part, buf, ex
    gc.collect()


def test_arrow_c_device_export_of_one_destination(ctx):
    """dfd_export_partition_device: ArrowDeviceArray (CUDA) slice of a partition result, read back through its buffers."""
    import ctypes as C

    from datafusion_distributed_b200 import _native as nv
    from datafusion_distributed_b200.device import columns_to_c

    n, N = 10_000, 4
    cols = cfg2_columns(n, 2)
    outs, starts = run_partition(ctx, cols, [0], N)
    ref, _, rs = orc.repartition_table(cols, [0], N, 8192, 1)
    p = 2
    dev = nv.ArrowDeviceArrayStruct()
    nv.check(nv.lib().dfd_export_partition_device(ctx.handle, columns_to_c(outs), 2, int(starts[p]), int(starts[p + 1] - starts[p]), C.byref(dev)))
    assert dev.device_type == 2 and dev.device_id == 0 and dev.sync_event  # ARROW_DEVICE_CUDA
    assert dev.array.length == starts[p + 1] - starts[p] and dev.array.n_children == 2
    children = C.cast(dev.array.children, C.POINTER(C.POINTER(nv.ArrowArrayStruct)))
    for c in range(2):
        ch = children[c].contents
        assert ch.offset == starts[p] and ch.length == dev.array.length and ch.n_buffers == 2
        bufs = C.cast(ch.buffers, C.POINTER(C.c_void_p))
        got = np.empty(ch.length, dtype=np.int64)
        nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, got.ctypes.data, bufs[1] + ch.offset * 8, ch.length * 8))
        assert np.array_equal(got, ref[c][rs[p]:rs[p + 1]])
    C.CFUNCTYPE(None, C.c_void_p)(dev.array.release)(C.addressof(dev.array))
    assert not dev.array.release


def test_interval_keys_hash_field_by_field_on_gpu(ctx):
    """Interval(DayTime) / Interval(MonthDayNano) KEY columns: one hasher write per struct field (arrow's derived Hash)."""
    import struct

    from datafusion_distributed_b200 import _native as nv

    rng = np.random.Generator(np.random.PCG64(99))
    n = 20_000
    days = rng.integers(-2**31, 2**31 - 1, n, dtype=np.int32)
    ms = rng.integers(-2**31, 2**31 - 1, n, dtype=np.int32)
    raw_dt = np.stack([days, ms], axis=1).copy().view(np.int64).reshape(n)  # {days: i32, milliseconds: i32}
    months = rng.integers(-2**31, 2**31 - 1, n, dtype=np.int32)
    nanos = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    raw_mdn = np.zeros(n, dtype=[("m", "<i4"), ("d", "<i4"), ("n", "<i8")])
    raw_mdn["m"], raw_mdn["d"], raw_mdn["n"] = months, days, nanos
    mdn = pa.Array.from_buffers(pa.decimal128(38, 0), n, [None, pa.py_buffer(raw_mdn.tobytes())])  # any 16-byte fixed layout
    cols = dev_cols(ctx, [raw_dt, mdn])
    for N in (8, 48, 1000):
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        part.set_key_hash_mode(0, nv.KEY_HASH_INTERVAL_DAY_TIME)
        want = orc.partition_ids([("interval_day_time", raw_dt.view(np.uint8))], n, N)
        assert np.array_equal(part.partition_ids(cols, n), want)
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([1, 0], N))
        part.set_key_hash_mode(0, nv.KEY_HASH_INTERVAL_MONTH_DAY_NANO)
        part.set_key_hash_mode(1, nv.KEY_HASH_INTERVAL_DAY_TIME)
        want = orc.partition_ids([("interval_month_day_nano", np.frombuffer(raw_mdn.tobytes(), dtype=np.uint8)),
                                  ("interval_day_time", raw_dt.view(np.uint8))], n, N)
        assert np.array_equal(part.partition_ids(cols, n), want)
    # plain hashing of the same bytes gives different placements: the mode matters
    plain = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 1000)).partition_ids(cols, n)
    assert not np.array_equal(plain, orc.partition_ids([("interval_day_time", raw_dt.view(np.uint8))], n, 1000))
    with pytest.raises(dfd.DfdError):
        dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8)).set_key_hash_mode(0, 7)


def test_dictionary_keys_hash_through_their_values(ctx):
    """Dictionary<Int32, Utf8> / Dictionary<Int8, Int64> key columns (the reference's bench schema: fixture.rs:13-33):
    placement equals hashing the decoded values; null indices and null dictionary values contribute nothing."""
    rnd = random.Random(4)
    n = 30_000
    values = pa.array(["alpha", None, "", "gamma-" * 9, "δ", "zz"], type=pa.string())
    idx = pa.array([rnd.choice([None, 0, 1, 2, 3, 4, 5]) for _ in range(n)], type=pa.int32())
    d = pa.DictionaryArray.from_arrays(idx, values)
    other = pa.array([rnd.getrandbits(20) for _ in range(n)], type=pa.int64())
    ivalues = pa.array([7, -1, None, 1 << 40], type=pa.int64())
    idx8 = pa.array([rnd.choice([None, 0, 1, 2, 3]) for _ in range(n)], type=pa.int8())
    d2 = pa.DictionaryArray.from_arrays(idx8, ivalues)
    cols = dev_cols(ctx, [idx, other, idx8])  # the INDICES travel as plain fixed-width columns
    for N in (8, 48, 1000):
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        part.set_key_dictionary(0, values)
        assert np.array_equal(part.partition_ids(cols, n), orc.partition_ids([d], n, N)), N
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([1, 0, 2], N))
        part.set_key_dictionary(1, values)
        part.set_key_dictionary(2, ivalues)
        assert np.array_equal(part.partition_ids(cols, n), orc.partition_ids([other, d, d2], n, N)), N
    # and the scatter itself (indices + payload) with a dictionary key
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 12))
    part.set_key_dictionary(0, values)
    outs, starts = part.partition(cols, n)
    dest = orc.partition_ids([d], n, 12)
    order, ref_starts = expected_partitions(dest, 12)
    assert np.array_equal(starts, ref_starts)
    assert outs[0].to_arrow(ctx, 0, n).equals(idx.take(pa.array(order)))
    assert outs[1].to_arrow(ctx, 0, n).equals(other.take(pa.array(order)))
    part.set_key_dictionary(0, None)
    assert np.array_equal(part.partition_ids([cols[1]], n), orc.partition_ids([other], n, 12))  # plain key again
