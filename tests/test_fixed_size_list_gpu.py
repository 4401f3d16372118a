"""Fixed-width payload columns of widths no scatter instantiation moves (FixedSizeList rows such as embeddings): the two-pass
partition gathers them after the scatter with k_gather_rows.  Every case is compared byte for byte with the input rows taken
in the oracle's stable destination order; guard bytes after each output must stay untouched.  The single-pass partition,
the exchange, PartialReduce and hash keys keep refusing such columns."""
import gc
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.util import multi_tile_rows

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

WIDTHS = [3, 12, 24, 32, 64, 100, 3072]
NS = [3, 8, 17, 256]
GUARD = 64
GiB = 1 << 30


def raw_col(t, width, offset, n, mis):
    """A FIXED dfd column whose values start `mis` bytes into the uint8 tensor t (rows counted from `offset`)."""
    return dfd.DeviceColumn(nv.COL_FIXED, width, t.data_ptr() + mis, 0, 0, offset, n, (t,))


def expected_order(key, N):
    ids = orc.partition_ids([key], len(key), N)
    return np.argsort(ids, kind="stable"), np.concatenate([[0], np.cumsum(np.bincount(ids, minlength=N))])


def run_case(ctx, rng, w, N, n, offset, mis_in, mis_out):
    key = rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64)
    payload = rng.integers(0, 256, (offset + n) * w, dtype=np.uint8)
    t_in = torch.empty(mis_in + payload.size + 1, dtype=torch.uint8, device="cuda")
    t_in[mis_in:mis_in + payload.size] = torch.from_numpy(payload).cuda()
    t_out = torch.full((mis_out + n * w + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    kcol = dfd.DeviceColumn.from_arrow(ctx, pa.array(key))
    out_key = dfd.DeviceColumn.empty_like(ctx, kcol, n)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    torch.cuda.synchronize()  # (the library works on a stream of its own: torch's writes must have landed)
    _, starts = part.partition([kcol, raw_col(t_in, w, offset, n, mis_in)], n, [out_key, raw_col(t_out, w, 0, n, mis_out)])
    order, ref_starts = expected_order(key, N)
    assert np.array_equal(starts, ref_starts)
    got = t_out.cpu().numpy()
    want = payload.reshape(offset + n, w)[offset:][order].reshape(-1)
    assert np.array_equal(got[mis_out:mis_out + n * w], want), f"w={w} N={N} n={n}"
    assert (got[:mis_out] == 0xA5).all() and (got[mis_out + n * w:] == 0xA5).all(), "bytes outside the output were written"
    assert np.array_equal(out_key.keep[-1].download(np.int64, n), key[order])


@pytest.mark.parametrize("w", WIDTHS)
def test_wide_fixed_partition_matches_the_oracle(ctx, w):
    rng = np.random.Generator(np.random.PCG64(w))
    big = multi_tile_rows() if w <= 100 else 100_003
    for i, N in enumerate(NS):
        # aligned and unaligned cases alternate: a row offset and base pointers off the 16-byte grid (any width, any base)
        offset, mis_in, mis_out = (0, 0, 0) if i % 2 == 0 else (3, 1 + i, 5 + i)
        for n in (0, 1, big if i < 2 else 20_011):
            run_case(ctx, rng, w, N, n, offset, mis_in, mis_out)
        gc.collect()


def test_fixed_size_list_mirror_round_trips(ctx):
    """DeviceColumn.from_arrow / to_arrow carry a FixedSizeList<Float32, 16> (sliced, with list nulls) as one FIXED column."""
    rng = np.random.Generator(np.random.PCG64(5))
    n, d, N = 50_003, 16, 8
    key = rng.integers(-(2**63), 2**63 - 1, n + 7, dtype=np.int64)
    vals = pa.array(rng.standard_normal((n + 7) * d).astype(np.float32))
    mask = rng.random(n + 7) < 0.1
    emb = pa.FixedSizeListArray.from_arrays(vals, d, mask=pa.array(mask)).slice(7)
    keys = pa.array(key).slice(7)
    cols = [dfd.DeviceColumn.from_arrow(ctx, keys), dfd.DeviceColumn.from_arrow(ctx, emb)]
    assert cols[1].kind == nv.COL_FIXED and cols[1].width == 4 * d
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    outs, starts = part.partition(cols, n)
    order, ref_starts = expected_order(key[7:], N)
    assert np.array_equal(starts, ref_starts)
    got = outs[1].to_arrow(ctx, 0, n)
    assert got.type == emb.type
    assert got.equals(emb.take(pa.array(order)))


def test_wide_fixed_partition_counts(ctx):
    """A gather launch is a kernel launch (not a scatter launch); bytes_in / bytes_out count n x w."""
    n, w, N = 10_007, 36, 8
    rng = np.random.Generator(np.random.PCG64(11))
    t_in = torch.from_numpy(rng.integers(0, 256, n * w, dtype=np.uint8)).cuda()
    t_out = torch.empty(n * w, dtype=torch.uint8, device="cuda")
    kcol = dfd.DeviceColumn.from_arrow(ctx, pa.array(rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64)))
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    args = ([kcol, raw_col(t_in, w, 0, n, 0)], n, [dfd.DeviceColumn.empty_like(ctx, kcol, n), raw_col(t_out, w, 0, n, 0)])
    torch.cuda.synchronize()
    part.partition(*args)  # (warm-up)
    m0 = ctx.metrics()
    part.partition(*args)
    m1 = ctx.metrics()
    d = {k: m1[k] - m0[k] for k in ("kernel_launches", "scatter_launches", "bytes_in", "bytes_out", "rows", "calls")}
    # k_iota_u32, k_tile_hist, k_scan_tiles, k_scatter (widths 8 and 4: the key and the iota), k_gather_rows
    assert d == {"kernel_launches": 6, "scatter_launches": 2, "bytes_in": n * (8 + w), "bytes_out": n * (8 + w), "rows": n, "calls": 1}


def test_k_gather_rows_runs(ctx):
    from torch.profiler import ProfilerActivity, profile

    n, w = 4097, 3072
    t_in = torch.zeros(n * w, dtype=torch.uint8, device="cuda")
    t_out = torch.empty(n * w, dtype=torch.uint8, device="cuda")
    kcol = dfd.DeviceColumn.from_arrow(ctx, pa.array(np.arange(n, dtype=np.int64)))
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        part.partition([kcol, raw_col(t_in, w, 0, n, 0)], n, [dfd.DeviceColumn.empty_like(ctx, kcol, n), raw_col(t_out, w, 0, n, 0)])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("k_gather_rows" in s for s in names), sorted(set(names))


# ------------------------------------------------------------------ refusals ----

def wide_table(ctx, n, w=12):
    rng = np.random.Generator(np.random.PCG64(2))
    key = dfd.DeviceColumn.from_arrow(ctx, pa.array(rng.integers(0, 1000, n, dtype=np.int64)))
    t = torch.zeros(n * w, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    return [key, raw_col(t, w, 0, n, 0)]


def assert_refused(fn, status=6):
    with pytest.raises(nv.DfdError) as e:
        fn()
    assert e.value.status == status, e.value
    return e.value


def test_single_pass_refuses_wide_fixed_columns(ctx):
    n = 1000
    cols = wide_table(ctx, n)
    for N in (8, 1000):  # (N > 256 would take the two-pass path: refused all the same)
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        assert_refused(lambda: part.partition_onepass(cols, n))


def test_wide_fixed_key_is_refused(ctx):
    n = 1000
    cols = wide_table(ctx, n)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([1], 8))
    assert_refused(lambda: part.partition(cols, n))
    assert_refused(lambda: part.partition_ids(cols, n))


def test_zero_width_fixed_column_is_refused(ctx):
    n = 100
    cols = wide_table(ctx, n)
    cols[1] = dfd.DeviceColumn(nv.COL_FIXED, 0, cols[1].values, 0, 0, 0, n, cols[1].keep)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    assert_refused(lambda: part.partition(cols, n, [cols[0], cols[1]]))


def test_exchange_refuses_wide_fixed_columns(ctx):
    n, N = 1000, 8
    cols = wide_table(ctx, n)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(64 << 20)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], N), uuid.uuid4(), 1, 1, 1)
    assert_refused(lambda: node.shuffle(ex, cols, n))
    outs = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in cols]
    assert_refused(lambda: node.shuffle(ex, cols, n, mode=nv.EXCHANGE_NCCL, out_cols=outs, out_capacity_rows=n))
    assert_refused(lambda: node.shuffle_onepass(ex, cols, n))


def test_partial_reduce_refuses_wide_fixed_columns(ctx):
    n = 1000
    cols = wide_table(ctx, n)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    outs, _ = part.partition([cols[0]], n)
    starts = nv.lib().dfd_partitioner_part_starts_device(part._h)
    # the wide column as a group key: PartialReduce refuses a key width outside 1/2/4/8/16 with INVALID_ARGUMENT (as before)
    red = dfd.PartialReduceExec(ctx, [0, 1], [-1, -1])
    err = assert_refused(lambda: red.reduce(cols, n, starts, 8), status=1)
    assert "value width 12" in err.message, err


# ----------------------------------------------------------- past 32-bit limits ----

def test_more_than_2_pow_31_child_elements_in_one_call(ctx):
    """FixedSizeList<Float32, 768> rows (3 KiB): more than 2^31 floats, 8 GiB of values, in one partition call.  Row x width
    byte offsets pass 2^32; the check runs on the device."""
    d, N = 768, 17
    w = 4 * d
    n = (1 << 31) // d + 1001
    need = 3 * n * w + n * 64
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 * GiB:
        pytest.skip(f"needs {(need + 2 * GiB) / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB is free")
    g = torch.Generator(device="cuda").manual_seed(3)
    key = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device="cuda", generator=g)
    vals = torch.randint(-(2**31), 2**31 - 1, (n, d), dtype=torch.int32, device="cuda", generator=g)
    out = torch.empty_like(vals)
    kcol = dfd.DeviceColumn.from_torch(key)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    in_cols = [kcol, dfd.DeviceColumn(nv.COL_FIXED, w, vals.data_ptr(), 0, 0, 0, n, (vals,))]
    out_key = torch.empty_like(key)
    out_cols = [dfd.DeviceColumn.from_torch(out_key), dfd.DeviceColumn(nv.COL_FIXED, w, out.data_ptr(), 0, 0, 0, n, (out,))]
    torch.cuda.synchronize()  # (the library works on a stream of its own: the random inputs must have landed)
    _, starts = part.partition(in_cols, n, out_cols)
    assert starts[-1] == n
    # the key column rides the scatter kernels; its destination order is the order every gathered row must follow
    order = torch.from_numpy(np.argsort(orc.partition_ids([key.cpu().numpy()], n, N), kind="stable")).cuda()
    assert torch.equal(out_key, key[order])
    for lo in range(0, n, 1 << 18):
        hi = min(n, lo + (1 << 18))
        assert torch.equal(out[lo:hi], vals[order[lo:hi]]), f"rows [{lo}, {hi})"
