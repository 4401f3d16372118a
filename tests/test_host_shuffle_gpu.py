"""dfd_shuffle_host with nullable, Boolean and string columns (the push transport, chunk by chunk) at world 1.

Every output buffer is compared with the oracle's destinations (orc.partition_ids, rows in input order per chunk and
partition), byte for byte and with guard bytes behind every capacity (tests/host_shuffle_util.py).  The multi-GPU form runs
tests/mgpu_host_shuffle_check.py under torch.distributed.run when the box has two or more GPUs."""
import ctypes as C
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests import host_shuffle_util as H

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def shuffle_host(ctx, arrays, keys, P, n_chunks, nullable=None, window=16 << 20, cap=None, byte_slack=0, ex=None, expect_status=0):
    """One world-1 dfd_shuffle_host of `arrays` (host buffers) through Hash(keys, P); checks every output buffer against the
    oracle and returns (chunk_part_starts, HostOut).  cap / byte_slack shrink the outputs (rows / string bytes) relative to
    what the data needs; with expect_status != 0 the call must fail with that status."""
    n = len(arrays[0])
    nullable = nullable if nullable is not None else [a.null_count > 0 for a in arrays]
    own = ex is None
    if own:
        ex = dfd.ShuffleExchange(ctx, 0, 1, None)
        ex.setup_window(window)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash(keys, P), uuid.uuid4(), 1, 1, 1)
    dests = orc.partition_ids([arrays[k] for k in keys], n, P) if n else np.zeros(0, np.int64)
    order, cps_want = H.expected_order(dests, n, n_chunks, P)
    total = len(order)
    nbytes = {i: H.string_bytes(a, order) + byte_slack for i, a in enumerate(arrays) if H.is_var(a.type)}
    out = H.HostOut([a.type for a in arrays], total if cap is None else cap, nullable, nbytes)
    h_in = H.in_columns(arrays, n)
    before = ex.stats()["shuffles"]
    try:
        if expect_status:
            with pytest.raises(dfd.DfdError) as e:
                node.shuffle_host(ex, h_in, n, n_chunks, out.cols, out.cap)
            assert e.value.status == expect_status, e.value
            return e.value, out
        cps = node.shuffle_host(ex, h_in, n, n_chunks, out.cols, out.cap)
        assert ex.stats()["shuffles"] - before == n_chunks  # one collective shuffle per chunk
        assert np.array_equal(cps, cps_want), (cps, cps_want)
        H.verify(out, [[(a, order)] for a in arrays], total)
        return cps, out
    finally:
        if own:
            ex.close()


def test_every_kind_alone(ctx):
    import pyarrow as pa

    n, rng = 30_011, np.random.Generator(np.random.PCG64(3))
    alone = {
        "int64 nullable": pa.array(rng.integers(0, 1000, n), mask=rng.random(n) < 0.2),
        "utf8": pa.array(["s%d" % (i % 977) * (i % 5) for i in range(n)], type=pa.string()),
        "large_utf8": pa.array(["L%d" % (i % 313) for i in range(n)], type=pa.large_string()),
        "binary": pa.array([bytes(rng.integers(0, 256, i % 23, dtype=np.uint8)) for i in range(n)], type=pa.binary()),
        "boolean": pa.array(rng.random(n) < 0.3, type=pa.bool_()),
    }
    for name, a in alone.items():
        shuffle_host(ctx, [a], [0], 6, 3)
        shuffle_host(ctx, [a], [0], 6, 7, nullable=[True])


@pytest.mark.parametrize("P", [1, 6, 64])
@pytest.mark.parametrize("n_chunks", [1, 3, 7])
def test_mixed_schema(ctx, P, n_chunks):
    arrays = H.mixed_arrays(20_011, 17)
    shuffle_host(ctx, arrays, [0, 1], P, n_chunks, nullable=[True] * len(arrays))


def test_more_chunks_than_rows_and_a_producer_with_no_rows(ctx):
    arrays = H.mixed_arrays(41, 5)
    shuffle_host(ctx, arrays, [0, 1], 6, 50, nullable=[True] * len(arrays))
    shuffle_host(ctx, H.mixed_arrays(0, 5), [0, 1], 6, 3, nullable=[True] * 6)
    shuffle_host(ctx, H.mixed_arrays(0, 5), [0, 1], 6, 1, nullable=[True] * 6)


def test_nulls_no_nulls_and_schema_nullable_without_a_bitmap(ctx):
    """Nullable with nulls; a nullable schema over rows without nulls (no input bitmap: all ones come out); the same rows
    with the columns not marked nullable (only the Boolean / string kinds send them to the push transport)."""
    with_nulls = H.mixed_arrays(9_001, 8)
    shuffle_host(ctx, with_nulls, [0, 1], 6, 3, nullable=[True] * 6)
    no_nulls = H.mixed_arrays(9_001, 8, nulls=False)
    assert all(a.null_count == 0 for a in no_nulls)
    _, out = shuffle_host(ctx, no_nulls, [0, 1], 6, 3, nullable=[True] * 6)
    total = 9_001
    vb, _ = out.bufs[(0, "validity")]
    assert np.unpackbits(vb[:(total + 31) // 32 * 4], bitorder="little")[:total].all()
    shuffle_host(ctx, no_nulls, [0, 1], 6, 3, nullable=[False] * 6)


def test_empty_strings_and_junk_under_nulls(ctx):
    """Utf8 / Binary / LargeUtf8 rows of length 0 next to NULL rows whose offsets still span bytes (junk the output keeps,
    as every transport does: a null row's bytes travel with it), and Int64 values under nulls."""
    import pyarrow as pa

    n = 12_347
    rng = np.random.Generator(np.random.PCG64(11))
    lens = rng.integers(0, 9, n)
    lens[rng.random(n) < 0.3] = 0
    null = rng.random(n) < 0.25
    validity = pa.py_buffer(np.packbits(~null, bitorder="little").tobytes())
    data = pa.py_buffer(rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes())
    off32 = pa.py_buffer(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32).tobytes())
    off64 = pa.py_buffer(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64).tobytes())
    s = pa.Array.from_buffers(pa.string(), n, [validity, off32, data])
    b = pa.Array.from_buffers(pa.binary(), n, [validity, off32, data])
    ls = pa.Array.from_buffers(pa.large_string(), n, [validity, off64, data])
    v = pa.Array.from_buffers(pa.int64(), n, [validity, pa.py_buffer(rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64).tobytes())])
    assert s.null_count > 0 and H.string_bytes(s, np.nonzero(null)[0]) > 0
    for n_chunks in (1, 5):
        shuffle_host(ctx, [v, s, b, ls], [3, 0], 7, n_chunks)


def test_exact_capacity_and_one_short(ctx):
    """Rows: exactly the rows delivered fit, one fewer is DFD_ERR_CAPACITY.  String bytes: the same, per column."""
    arrays = H.mixed_arrays(7_777, 23)
    flags = [True] * 6
    shuffle_host(ctx, arrays, [0, 1], 6, 3, nullable=flags)  # cap = exactly the rows, values_bytes = exactly the bytes
    err, out = shuffle_host(ctx, arrays, [0, 1], 6, 3, nullable=flags, cap=7_776, expect_status=7)
    assert "7776 rows" in str(err) and "7777" in str(err), err
    for b in out.bufs.values():  # (earlier chunks were delivered; nothing past any capacity was written)
        assert (b[0][b[1]:] == H.FILL).all()
    err, out = shuffle_host(ctx, arrays, [0, 1], 6, 3, nullable=flags, byte_slack=-1, expect_status=7)
    assert "string bytes" in str(err), err
    for b in out.bufs.values():
        assert (b[0][b[1]:] == H.FILL).all()


def test_window_too_small_for_a_chunk_then_a_call_that_fits(ctx):
    """A chunk that does not fit the receive window is DFD_ERR_CAPACITY (every worker agrees, nothing of it is written);
    the same exchange then takes the same rows in smaller chunks."""
    arrays = H.mixed_arrays(20_011, 29)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(512 << 10)
    err, out = shuffle_host(ctx, arrays, [0, 1], 6, 1, nullable=[True] * 6, ex=ex, expect_status=7)
    assert "receive window" in str(err), err
    for b in out.bufs.values():
        assert (b[0] == H.FILL).all()
    shuffle_host(ctx, arrays, [0, 1], 6, 4, nullable=[True] * 6, ex=ex)
    ex.close()


def test_refusals_before_any_shuffle(ctx):
    import pyarrow as pa

    n = 100
    arrays = H.mixed_arrays(n, 2)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(4 << 20)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], 4), uuid.uuid4(), 1, 1, 1)
    out = H.HostOut([a.type for a in arrays], n, [True] * 6, {1: 4096, 2: 4096})
    h_in = H.in_columns(arrays, n)
    before = ex.stats()["shuffles"]
    sliced = list(h_in)
    sliced[4] = dfd.DeviceColumn(h_in[4].kind, h_in[4].width, h_in[4].values, 0, h_in[4].validity, 1, n - 1)
    with pytest.raises(dfd.DfdError) as e:
        node.shuffle_host(ex, sliced, n - 1, 2, out.cols, n)
    assert e.value.status == 6  # DFD_ERR_UNSUPPORTED: Arrow offset != 0
    wide = list(h_in)
    raw = pa.py_buffer(np.zeros(n * 12, np.uint8).tobytes())
    wide[5] = dfd.DeviceColumn(nv.COL_FIXED, 12, raw.address, length=n, keep=raw)
    wide_out = list(out.cols)
    wide_out[5] = dfd.DeviceColumn(nv.COL_FIXED, 12, out.cols[5].values, length=n)
    with pytest.raises(dfd.DfdError) as e:
        node.shuffle_host(ex, wide, n, 2, wide_out, n)
    assert e.value.status == 6  # a 12-byte fixed column
    assert ex.stats()["shuffles"] == before
    ex.close()


def test_multi_gpu_host_shuffle_under_torchrun(built):
    n = C.c_int(0)
    nv.lib().dfd_device_count(C.byref(n))
    if n.value < 2:
        pytest.skip("needs >= 2 GPUs (run tests/mgpu_host_shuffle_check.py under torchrun on a multi-GPU box)")
    world = min(n.value, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29543", os.path.join(ROOT, "tests", "mgpu_host_shuffle_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert "MGPU_HOST_SHUFFLE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
