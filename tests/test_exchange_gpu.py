"""GPU tests of the exchange: world=1 on any box, world=T via torchrun when the
box has more than one GPU (the driver's 1-GPU tier skips that case)."""
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.util import cfg2_columns

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("mode", [nv.EXCHANGE_NCCL, nv.EXCHANGE_FUSED])
def test_single_worker_shuffle_equals_local_repartition(ctx, mode):
    check_single_worker_shuffle(ctx, mode, 8)


@pytest.mark.parametrize("P", [16, 17, 48])
def test_single_worker_fused_shuffle_past_the_aligned_cutoff(ctx, P):
    """Peer kernels write out aligned runs up to 16 partitions; past that their plain (KV == K) instantiations run."""
    check_single_worker_shuffle(ctx, nv.EXCHANGE_FUSED, P)


def check_single_worker_shuffle(ctx, mode, P):
    import pyarrow as pa

    n = 300_007
    cols = cfg2_columns(n, 4)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(n * 4 * 8 + (1 << 20))
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, pa.array(c)) for c in cols]
    out_cols = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in in_cols] if mode == nv.EXCHANGE_NCCL else None
    outs, starts = node.shuffle(ex, in_cols, n, mode, out_cols, n)
    if mode == nv.EXCHANGE_FUSED:  # the asynchronous form (two pipelined shuffles, one wait) gives the same result
        node.shuffle_async(ex, in_cols, n)
        node.shuffle_async(ex, in_cols, n)
        outs, starts = node.wait(ex)
    ref, rc, rs = orc.repartition_table(cols, [0], P, 8192, 1)
    assert np.array_equal(starts, rs)
    for q in range(P):
        _, a, b = node.execute(q, dfd.DistributedTaskContext(0, 1))
        for c in range(4):
            got = np.empty(b - a, dtype=np.int64)
            nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, got.ctypes.data, outs[c].values + a * 8, (b - a) * 8))
            assert np.array_equal(got, ref[c][rs[q]:rs[q + 1]])
    ex.close()


def test_single_worker_onepass_shuffle_segments(ctx):
    check_single_worker_onepass_shuffle(ctx, 8)


@pytest.mark.parametrize("P", [16, 17, 48, 256])
def test_single_worker_onepass_shuffle_past_the_aligned_cutoff(ctx, P):
    """The single-pass peer kernel's aligned write-out ends at 16 partitions; 256 is the single-pass maximum."""
    check_single_worker_onepass_shuffle(ctx, P)


def check_single_worker_onepass_shuffle(ctx, P):
    """Single-pass fused exchange at world=1: partition q is one segment (one producer), bit-exact and in input order;
    back-to-back shuffles reuse the window (ready/done flags)."""
    import pyarrow as pa

    n = 300_007
    cols = cfg2_columns(n, 4)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(int(n * 4 * 8 * 1.5) + (1 << 20))
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, pa.array(c)) for c in cols]
    for _ in range(3):
        node.shuffle_onepass(ex, in_cols, n)
    outs, seg_starts, seg_counts = node.collect(ex)
    ref, rc, rs = orc.repartition_table(cols, [0], P, 8192, 1)
    assert np.array_equal(seg_counts[:, 0], rc)
    for q in range(P):
        _, segs = node.execute_segments(q, dfd.DistributedTaskContext(0, 1))
        (a, cnt), = segs
        for c in range(4):
            got = np.empty(cnt, dtype=np.int64)
            nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, got.ctypes.data, outs[c].values + a * 8, cnt * 8))
            assert np.array_equal(got, ref[c][rs[q]:rs[q + 1]])
    # skew: a hot key overflows its sub-window -> exact re-run (dense layout), nothing lost
    k = np.full(n, 5, dtype=np.int64)
    k[::50] = np.arange(0, n, 50)
    hot = [dfd.DeviceColumn.from_arrow(ctx, pa.array(k)), dfd.DeviceColumn.from_arrow(ctx, pa.array(np.arange(n, dtype=np.int64)))]
    ex2 = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex2.setup_window(n * 2 * 8 + (1 << 20))
    node.shuffle_onepass(ex2, hot, n)
    outs, seg_starts, seg_counts = node.collect(ex2)
    assert nv.lib().dfd_exchange_onepass_fallbacks(ex2._h) == 1
    ref, rc, rs = orc.repartition_table([k, np.arange(n, dtype=np.int64)], [0], P, 8192, 1)
    assert np.array_equal(seg_counts[:, 0], rc)
    for q in range(P):
        a, cnt = int(seg_starts[q, 0]), int(seg_counts[q, 0])
        got = np.empty(cnt, dtype=np.int64)
        nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, got.ctypes.data, outs[1].values + a * 8, cnt * 8))
        assert np.array_equal(got, ref[1][rs[q]:rs[q + 1]])
    ex.close()
    ex2.close()


def test_single_worker_onepass_shuffle_every_cta_handles_many_tiles(ctx):
    """Single-pass peer kernel at world=1 with every CTA looping over several tiles, 4 / 8 / 16-byte columns.  They are
    fixed-width and non-null: a nullable, boolean or string column would send the shuffle to the push transport."""
    import pyarrow as pa

    from tests.util import expected_partitions, multi_tile_rows

    n, P = multi_tile_rows(), 48
    rng = np.random.Generator(np.random.PCG64(21))
    key = rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64, endpoint=True)
    raw = rng.integers(0, 255, n * 16, dtype=np.uint8).tobytes()
    arrays = [pa.array(key), pa.array(rng.integers(-(2**31), 2**31 - 1, n, dtype=np.int32)), pa.array(np.arange(n, dtype=np.int64)),
              pa.Array.from_buffers(pa.decimal128(38, 0), n, [None, pa.py_buffer(raw)])]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(int(n * 36 * 1.5) + (1 << 20))
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    node.shuffle_onepass(ex, [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays], n)
    outs, seg_starts, seg_counts = node.collect(ex)
    assert nv.lib().dfd_exchange_onepass_fallbacks(ex._h) == 0
    order, ref_starts = expected_partitions(orc.partition_ids([key], n, P), P)
    assert np.array_equal(seg_counts[:, 0], np.diff(ref_starts))
    for q in range(P):
        idx = pa.array(order[ref_starts[q]:ref_starts[q + 1]])
        for c, arr in enumerate(arrays):
            got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(seg_starts[q, 0]), int(seg_counts[q, 0]))
            assert got.equals(arr.take(idx)), (q, c)
    ex.close()


def test_fused_window_overflow_is_reported(ctx):
    import pyarrow as pa

    n = 100_000
    cols = cfg2_columns(n, 2)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(n * 8)  # half of what 2 columns need
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], 4), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, pa.array(c)) for c in cols]
    with pytest.raises(dfd.DfdError) as e:
        node.shuffle(ex, in_cols, n, nv.EXCHANGE_FUSED)
    assert e.value.status == 7  # DFD_ERR_CAPACITY
    ex.close()


def test_multi_gpu_shuffle_under_torchrun(built):
    import ctypes as C

    n = C.c_int(0)
    nv.lib().dfd_device_count(C.byref(n))
    if n.value < 2:
        pytest.skip("needs >= 2 GPUs (run tests/mgpu_shuffle_check.py under torchrun on a multi-GPU box)")
    world = min(n.value, 8)  # every GPU of the box: the driver's multi-GPU tiers run this at 2 / 4 / 8 ranks
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "mgpu_shuffle_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert "MGPU_SHUFFLE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


@pytest.mark.parametrize("n_chunks", [1, 3, 7])
def test_single_worker_host_to_host_shuffle(ctx, n_chunks):
    """dfd_shuffle_host at world=1: pinned host columns in, chunk-major host segments out."""
    n, P = 250_003, 8
    cols = cfg2_columns(n, 3)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(2 * (n * 3 * 8 + (1 << 16)))
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    pin_in = dfd.PinnedTable(ctx, n, [np.int64] * 3)
    pin_out = dfd.PinnedTable(ctx, n, [np.int64] * 3)
    for c in range(3):
        pin_in.columns[c][:] = cols[c]
    h_in = [dfd.DeviceColumn(nv.COL_FIXED, 8, a.ctypes.data, length=n) for a in pin_in.columns]
    h_out = [dfd.DeviceColumn(nv.COL_FIXED, 8, a.ctypes.data, length=n) for a in pin_out.columns]
    cps = node.shuffle_host(ex, h_in, n, n_chunks, h_out, n)
    assert cps[-1, -1] == n
    ref, rc, rs = orc.repartition_table(cols, [0], P, 8192, 1)
    for q in range(P):
        # one producer: concatenating the chunks of destination q reproduces the oracle's order exactly
        idx = np.concatenate([np.arange(cps[i, q], cps[i, q + 1]) for i in range(n_chunks)])
        for c in range(3):
            assert np.array_equal(pin_out.columns[c][idx], ref[c][rs[q]:rs[q + 1]]), (q, c)
    with pytest.raises(dfd.DfdError) as e:
        node.shuffle_host(ex, h_in, n, n_chunks, h_out, n // 2)
    assert e.value.status == 7
    ex.close()


def _mixed_table(n, seed):
    import random

    import pyarrow as pa

    rnd = random.Random(seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    key = pa.array([rnd.choice([None, rnd.getrandbits(30)]) for _ in range(n)], type=pa.int64())
    s = pa.array([rnd.choice([None, "", "N", "O", "phrase %d" % rnd.getrandbits(16), "x" * rnd.randint(0, 50)]) for _ in range(n)], type=pa.string())
    ls = pa.array([rnd.choice([None, "L" * rnd.randint(0, 9)]) for _ in range(n)], type=pa.large_string())
    bl = pa.array([rnd.choice([None, True, False]) for _ in range(n)])
    i32 = pa.array([rnd.choice([None, rnd.getrandbits(31)]) for _ in range(n)], type=pa.int32())
    f64 = pa.array(rng.standard_normal(n))
    return [key, s, ls, bl, i32, f64]


def test_single_worker_nccl_mode_moves_every_column_kind(ctx):
    """NCCL-mode exchange with nullable, boolean and string columns (keys: Int64 + Utf8) at world=1."""
    import pyarrow as pa

    from tests.util import expected_partitions

    n, P = 20_011, 6
    arrays = _mixed_table(n, 17)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], P), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    out_cols = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in in_cols]
    outs, starts = node.shuffle(ex, in_cols, n, nv.EXCHANGE_NCCL, out_cols, n)
    dest = orc.partition_ids([arrays[0], arrays[1]], n, P)
    order, ref_starts = expected_partitions(dest, P)
    assert np.array_equal(starts, ref_starts)
    idx = pa.array(order)
    for c, arr in enumerate(arrays):
        assert outs[c].to_arrow(ctx, 0, n).equals(arr.take(idx)), (c, arr.type)
    ex.close()


def test_single_worker_push_transport_moves_every_column_kind(ctx):
    """NCCL-free push transport (nullable / boolean / string columns; keys Int64 + Utf8) at world=1: every partition's
    single segment equals the oracle's rows in order, read in place from the window as Arrow buffers."""
    import pyarrow as pa

    from tests.util import expected_partitions

    n, P = 20_011, 6
    arrays = _mixed_table(n, 17)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(8 << 20)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], P), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    dest = orc.partition_ids([arrays[0], arrays[1]], n, P)
    order, ref_starts = expected_partitions(dest, P)
    for rep in range(2):
        node.shuffle_onepass(ex, in_cols, n, nullable=[True] * len(arrays))
        outs, seg_starts, seg_counts = node.collect(ex)
        assert np.array_equal(seg_counts[:, 0], np.diff(ref_starts))
        assert (seg_starts % 32 == 0).all()
        for q in range(P):
            idx = pa.array(order[ref_starts[q]:ref_starts[q + 1]])
            for c, arr in enumerate(arrays):
                got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(seg_starts[q, 0]), int(seg_counts[q, 0]))
                assert got.equals(arr.take(idx)), (rep, q, c, arr.type)
    # sliced inputs (Arrow offset != 0) and an empty worker
    sl = [a.slice(13, 9000) for a in arrays]
    node.shuffle_onepass(ex, [dfd.DeviceColumn.from_arrow(ctx, a) for a in sl], 9000, nullable=[True] * len(arrays))
    outs, seg_starts, seg_counts = node.collect(ex)
    d2 = orc.partition_ids([sl[0], sl[1]], 9000, P)
    o2, s2 = expected_partitions(d2, P)
    for q in range(P):
        for c, arr in enumerate(sl):
            got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(seg_starts[q, 0]), int(seg_counts[q, 0]))
            assert got.equals(arr.take(pa.array(o2[s2[q]:s2[q + 1]]))), (q, c)
    node.shuffle_onepass(ex, [dfd.DeviceColumn.from_arrow(ctx, a.slice(0, 0)) for a in arrays], 0, nullable=[True] * len(arrays))
    outs, seg_starts, seg_counts = node.collect(ex)
    assert not seg_counts.any()
    # window too small: reported, consistent on every worker
    ex2 = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex2.setup_window(64 << 10)
    with pytest.raises(dfd.DfdError) as e:
        node.shuffle_onepass(ex2, in_cols, n, nullable=[True] * len(arrays))
    assert e.value.status == 7
    ex.close()
    ex2.close()


def test_single_worker_coalesce_and_broadcast(ctx):
    """NetworkCoalesceExec / NetworkBroadcastExec over the push transport at world=1: the consumer sees the producer's
    partitions unchanged (every column kind), read in place from the window."""
    import pyarrow as pa

    n, P = 9_001, 4
    arrays = _mixed_table(n, 5)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(8 << 20)
    cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    starts = [0, 100, 100, 5000, n]  # one empty partition
    co = dfd.NetworkCoalesceExec.try_new(P, uuid.uuid4(), 1, 1, 1)
    outs, ss, sc = co.gather(ex, cols, starts, nullable=[True] * len(arrays))
    assert co.output_partition_count() == P and sc.tolist() == [100, 0, 4900, n - 5000]
    for p in range(P):
        _, a, cnt = co.execute(p, dfd.DistributedTaskContext(0, 1))
        for c, arr in enumerate(arrays):
            got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], a, cnt)
            assert got.equals(arr.slice(starts[p], starts[p + 1] - starts[p])), (p, c)
    bc = dfd.NetworkBroadcastExec.try_new(P, uuid.uuid4(), 2, 1, 1)
    outs, ss, sc = bc.gather(ex, cols, starts, nullable=[True] * len(arrays))
    for p in range(P):
        _, segs = bc.execute(p, dfd.DistributedTaskContext(0, 1))
        (a, cnt), = segs
        for c, arr in enumerate(arrays):
            got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], a, cnt)
            assert got.equals(arr.slice(starts[p], starts[p + 1] - starts[p])), (p, c)
    # sliced inputs (Arrow offset != 0)
    sl = [a.slice(17, 4000) for a in arrays]
    outs, ss, sc = co.gather(ex, [dfd.DeviceColumn.from_arrow(ctx, a) for a in sl], [0, 1, 2, 3000, 4000], nullable=[True] * len(arrays))
    for c, arr in enumerate(sl):
        got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(ss[2]), int(sc[2]))
        assert got.equals(arr.slice(2, 2998)), c
    ex.close()


def test_back_pressure_rounds_instead_of_capacity_error(ctx):
    """A window far smaller than the data (and a single hot key): the shuffle is delivered in rounds that shrink until they
    fit; the union of the rounds equals the oracle, per partition and in order (one producer)."""
    import pyarrow as pa

    n, P = 200_000, 4
    k = np.full(n, 42, dtype=np.int64)
    k[::7] = np.arange(0, n, 7)
    v = np.arange(n, dtype=np.int64)
    s = pa.array([("s%d" % (i % 1000)) if i % 3 else None for i in range(n)], type=pa.string())
    arrays = [pa.array(k), pa.array(v), s]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(1 << 20)  # ~ 1/6 of what one round of everything would need
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    got = [[[] for _ in arrays] for _ in range(P)]
    for outs, ss, sc in node.shuffle_rounds(ex, cols, n, nullable=[False, False, True]):
        for q in range(P):
            for c in range(len(arrays)):
                got[q][c].append(dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(ss[q, 0]), int(sc[q, 0])))
    assert node.last_stream_stats["rounds"] > 1 and node.last_stream_stats["splits"] >= 1
    dest = orc.partition_ids([k], n, P)
    for q in range(P):
        idx = pa.array(np.nonzero(dest == q)[0])
        for c, arr in enumerate(arrays):
            assert pa.concat_arrays(got[q][c]).equals(arr.take(idx)), (q, c)
    # the same data through the single-pass path (fixed-width, non-null) with a small window: overflow -> exact re-run -> rounds
    ex2 = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex2.setup_window(1 << 20)
    cols2 = cols[:2]
    rows = 0
    parts = [[] for _ in range(P)]
    for outs, ss, sc in node.shuffle_rounds(ex2, cols2, n):
        for q in range(P):
            parts[q].append(dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[1], int(ss[q, 0]), int(sc[q, 0])))
            rows += int(sc[q, 0])
    assert rows == n and node.last_stream_stats["rounds"] > 1
    for q in range(P):
        assert pa.concat_arrays(parts[q]).equals(arrays[1].take(pa.array(np.nonzero(dest == q)[0])))
    ex.close()
    ex2.close()
