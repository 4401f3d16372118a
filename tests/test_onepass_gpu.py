"""GPU parity tests of the single-pass partition kernel (k_scatter<ONEPASS>: hash once,
decoupled look-back instead of the histogram pass, per-destination regions) vs the CPU oracle.
Bar: bit-exact per destination, including row order."""
import random

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from oracle import oracle as orc
from tests.util import cfg2_columns, edge_sizes, expected_partitions, multi_tile_rows, tile_geometry

pytestmark = pytest.mark.gpu


def dev_cols(ctx, arrays):
    return [dfd.DeviceColumn.from_arrow(ctx, a if isinstance(a, pa.Array) else pa.array(a)) for a in arrays]


def check_against_oracle(ctx, arrays, key_cols, N, region_rows=None, two_pass=False):
    """Single-pass partition (or, with two_pass, the dense partition()) of `arrays` against the oracle."""
    n = len(arrays[0])
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N))
    if two_pass:
        outs, part_starts = part.partition(dev_cols(ctx, arrays), n)
        starts, counts = part_starts[:-1], np.diff(part_starts)
    else:
        outs, starts, counts = part.partition_onepass(dev_cols(ctx, arrays), n, region_rows)
    keys = [arrays[k] for k in key_cols]
    dest = orc.partition_ids(keys, n, N)
    order, ref_starts = expected_partitions(dest, N)
    assert np.array_equal(counts, np.diff(ref_starts)), (N, counts, np.diff(ref_starts))
    total = int((starts + counts).max()) if n else 0
    got_all = [outs[c].to_arrow(ctx, 0, max(total, 0)) for c in range(len(arrays))]
    for p in range(N):
        idx = pa.array(order[ref_starts[p]:ref_starts[p + 1]])
        for c, arr in enumerate(arrays):
            arr = arr if isinstance(arr, pa.Array) else pa.array(arr)
            got = got_all[c].slice(int(starts[p]), int(counts[p]))
            assert got.equals(arr.take(idx)), (N, p, c)
    return part, starts, counts


@pytest.mark.parametrize("n_rows", edge_sizes())
def test_onepass_ragged_sizes(ctx, n_rows):
    check_against_oracle(ctx, cfg2_columns(n_rows, 3), [0], 8)


@pytest.mark.parametrize("N", [1, 2, 3, 7, 8, 9, 12, 16, 17, 48, 64, 255, 256])
def test_onepass_all_moduli_cfg1_shape(ctx, N):
    rng = np.random.Generator(np.random.PCG64(1))
    n = 1_000_000
    k = rng.integers(0, 2**63 - 1, n, dtype=np.int64)
    v = np.arange(n, dtype=np.int64)
    check_against_oracle(ctx, [k, v], [0], N)


def test_onepass_two_keys_eight_columns(ctx):
    check_against_oracle(ctx, cfg2_columns(1 << 20, 8), [0, 1], 8)


def test_onepass_large_n_falls_back_to_two_pass_dense(ctx):
    n = 200_000
    cols = cfg2_columns(n, 2)
    part, starts, counts = check_against_oracle(ctx, cols, [0], 1000)
    assert np.array_equal(starts[1:], np.cumsum(counts)[:-1])  # dense layout


def test_onepass_mixed_widths_nulls_bools(ctx):
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
        check_against_oracle(ctx, arrays, [0, 3], N)


def mixed_table(n, seed):
    """Nullable Int64 and Int32 keys, UInt8 / Int16 / Float64 / Decimal128 payload and a nullable Boolean."""
    rng = np.random.Generator(np.random.PCG64(seed))
    key = pa.array(rng.integers(0, 1 << 40, n, dtype=np.int64), mask=rng.random(n) < 0.5)
    c8 = pa.array(rng.integers(0, 255, n, dtype=np.uint8))
    c16 = pa.array(rng.integers(-30000, 30000, n, dtype=np.int16))
    c32 = pa.array(rng.integers(0, 1 << 31, n, dtype=np.int32), mask=rng.random(n) < 0.5)
    f64 = pa.array(rng.standard_normal(n))
    bl = pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.3)
    dec = pa.Array.from_buffers(pa.decimal128(38, 0), n, [None, pa.py_buffer(rng.integers(0, 255, n * 16, dtype=np.uint8).tobytes())])
    return [key, c8, c16, c32, f64, bl, dec]


def test_onepass_every_cta_handles_many_tiles_mixed_schema(ctx):
    """Generic two-column key, 1 / 2 / 4 / 8 / 16-byte columns (the 16-byte one split into row ranges), nulls and a
    boolean column (follow-up launches), with every CTA looping over several tiles."""
    check_against_oracle(ctx, mixed_table(multi_tile_rows(), 31), [0, 3], 48)


def test_onepass_every_cta_handles_many_tiles_cfg2_two_keys(ctx):
    check_against_oracle(ctx, cfg2_columns(multi_tile_rows(), 4), [0, 1], 8)


def sliced_payload(n, offset, seed):
    """Payload columns of widths 1, 2, 4, 8 and 16 and a nullable Boolean, each a slice at `offset` of a longer array:
    the source of every column tile is then off its 16-byte alignment (or, for offset 1 and width 1, its byte count)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    m = n + offset + 5
    arrays = [pa.array(rng.integers(0, 255, m, dtype=np.uint8)), pa.array(rng.integers(-30000, 30000, m, dtype=np.int16)),
              pa.array(rng.integers(-(1 << 31), 1 << 31, m, dtype=np.int32), mask=rng.random(m) < 0.2),
              pa.array(rng.integers(-(1 << 62), 1 << 62, m, dtype=np.int64)),
              pa.Array.from_buffers(pa.decimal128(38, 0), m, [None, pa.py_buffer(rng.integers(0, 255, m * 16, dtype=np.uint8).tobytes())]),
              pa.array(rng.random(m) < 0.5, mask=rng.random(m) < 0.3)]
    return [a.slice(offset, n) for a in arrays]


@pytest.mark.parametrize("offset", [1, 3, 13])
@pytest.mark.parametrize("sliced_key", [False, True])
def test_onepass_and_two_pass_sliced_inputs(ctx, offset, sliced_key):
    """Sliced payload (Arrow offset 1 / 3 / 13) under an unsliced non-null Int64 key, where the single-pass producer
    takes the fast key path and only its element-wise fallback copy changes, and under a sliced key (generic key path).
    The same inputs go through the two-pass partition()."""
    n, N = 3 * tile_geometry()[1] * 7 + 11, 12
    rng = np.random.Generator(np.random.PCG64(offset))
    key = pa.array(rng.integers(-(1 << 63), (1 << 63) - 1, n + offset, dtype=np.int64))
    key = key.slice(offset, n) if sliced_key else key.slice(0, n)
    arrays = [key] + sliced_payload(n, offset, 40 + offset)
    check_against_oracle(ctx, arrays, [0], N)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    outs, starts = part.partition(dev_cols(ctx, arrays), n)
    order, ref_starts = expected_partitions(orc.partition_ids([key], n, N), N)
    assert np.array_equal(starts, ref_starts)
    idx = pa.array(order)
    for c, arr in enumerate(arrays):
        assert outs[c].to_arrow(ctx, 0, n).equals(arr.take(idx)), (c, arr.type)


def test_onepass_region_capacity_exactly_max_count(ctx):
    """Regions of exactly the largest destination's row count fit without a re-run; one row less re-runs exactly once
    into the dense layout, bit-exact."""
    n, N = 200_003, 8
    cols = cfg2_columns(n, 3)
    c = np.bincount(orc.partition_ids([cols[0]], n, N), minlength=N)
    mx = int(c.max())
    assert (mx - 1) * N >= n  # one row less still holds every row in total: valid input
    before = ctx.metrics()["onepass_reruns"]
    _, starts, counts = check_against_oracle(ctx, cols, [0], N, region_rows=mx)
    assert ctx.metrics()["onepass_reruns"] == before
    assert np.array_equal(starts, np.arange(N) * mx)
    _, starts, counts = check_against_oracle(ctx, cols, [0], N, region_rows=mx - 1)
    assert ctx.metrics()["onepass_reruns"] == before + 1
    assert np.array_equal(starts[1:], np.cumsum(counts)[:-1]) and starts[0] == 0  # dense after the re-run


def test_onepass_many_columns_multiple_launches(ctx):
    check_against_oracle(ctx, cfg2_columns(10_000, 30), [0], 8)


def test_onepass_skew_overflows_regions_and_reruns_exactly(ctx):
    """A single hot key sends almost every row to one destination: the optimistic regions overflow,
    the counts are still exact and collection re-runs with exact (dense) regions."""
    n = 300_000
    k = np.full(n, 12345, dtype=np.int64)
    k[::1000] = np.arange(0, n, 1000)
    v = np.arange(n, dtype=np.int64)
    before = ctx.metrics()["onepass_reruns"]
    part, starts, counts = check_against_oracle(ctx, [k, v], [0], 16)
    assert ctx.metrics()["onepass_reruns"] == before + 1
    assert np.array_equal(starts[1:], np.cumsum(counts)[:-1])  # dense after the re-run
    # the same partitioner keeps working (ticket / epoch state is consistent after an overflowed launch)
    cols = cfg2_columns(50_000, 2)
    outs, s2, c2 = part.partition_onepass(dev_cols(ctx, cols), 50_000)
    assert int(c2.sum()) == 50_000


def test_onepass_async_then_collect_and_repeated_calls(ctx):
    n, N = 500_000, 8
    cols = cfg2_columns(n, 4)
    dcols = dev_cols(ctx, cols)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    rr = part.default_region_rows(n)
    outs = [dfd.DeviceColumn.empty_like(ctx, c, N * rr) for c in dcols]
    for _ in range(5):  # back-to-back launches share the look-back table: epochs must not alias
        part.partition_onepass(dcols, n, rr, outs, sync=False)
    starts, counts = part.collect()
    ref, rc, rs = orc.repartition_table(cols, [0], N, 8192, 1)
    assert np.array_equal(counts, rc)
    for c in range(4):
        got = outs[c].keep[-1].download(np.int64, N * rr)
        for p in range(N):
            assert np.array_equal(got[starts[p]:starts[p] + counts[p]], ref[c][rs[p]:rs[p + 1]])


def test_onepass_rejects_too_small_regions(ctx):
    cols = cfg2_columns(10_000, 2)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    with pytest.raises(dfd.DfdError) as e:
        part.partition_onepass(dev_cols(ctx, cols), 10_000, region_rows=100)
    assert e.value.status == 1


def test_onepass_full_size_cfg2_properties(ctx):
    """2^26 rows x 8 x i64, N=8 (BASELINE cfg-2) through the single-pass kernel: size-independent properties."""
    import torch

    n, C, N = 1 << 26, 8, 8
    g = torch.Generator(device="cuda").manual_seed(42)
    key = torch.randint(-(2**63), 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    rid = torch.arange(n, dtype=torch.int64, device="cuda")
    ins = [key] + [rid * 8 + j for j in range(1, C)]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    rr = part.default_region_rows(n)
    outs = [torch.zeros(N * rr, dtype=torch.int64, device="cuda") for _ in ins]
    torch.cuda.synchronize()
    _, starts, counts = part.partition_onepass([dfd.DeviceColumn.from_torch(t) for t in ins], n, rr,
                                               [dfd.DeviceColumn.from_torch(t) for t in outs])
    assert ctx.metrics()["onepass_reruns"] == ctx.metrics()["onepass_reruns"]  # (uniform keys: no re-run expected below)
    key_h = key.cpu().numpy()
    dest = orc.partition_ids([key_h], n, N)
    assert np.array_equal(counts, np.bincount(dest, minlength=N))
    assert np.array_equal(starts, np.arange(N) * rr)
    seen = 0
    for p in range(N):
        a, b = int(starts[p]), int(starts[p] + counts[p])
        ids = part.partition_ids([dfd.DeviceColumn.from_torch(outs[0][a:b].contiguous())], b - a)
        assert (ids == p).all()
        rid_out = (outs[1][a:b] - 1) >> 3
        for j in range(2, C):
            assert torch.equal(outs[j][a:b], rid_out * 8 + j)
        assert torch.equal(key[rid_out], outs[0][a:b])
        assert bool((rid_out[1:] > rid_out[:-1]).all())  # stable
        seen += int(rid_out.sum().item())
        if p == 0:
            want = np.nonzero(dest == 0)[0][:1_000_000]
            assert np.array_equal(rid_out[:len(want)].cpu().numpy(), want)
    assert seen == n * (n - 1) // 2
