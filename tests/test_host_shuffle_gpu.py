"""dfd_shuffle_host with nullable, Boolean and string columns (the push transport, chunk by chunk) at world 1.

Every output buffer is compared with the oracle's destinations (orc.partition_ids, rows in input order per chunk and
partition), byte for byte and with guard bytes behind every capacity (tests/host_shuffle_util.py).  The multi-GPU form runs
tests/mgpu_host_shuffle_check.py under torch.distributed.run when the box has two or more GPUs.  Fixed-width non-null
schemas take the two-pass fused path; they run here at every width too.

The edge cases restate the compaction layout on the host (H.bit_launches, with PUSH_THREADS and BIT_WORDS_PER_CTA read
from dfd_exchange.cu) and assert the boundary each one reaches: k_place_bits runs of more than one CTA, a run ending
exactly on a CTA boundary and one bit past it at seam residues 0 / 1 / 17 / 31, dozens of multi-CTA runs in one launch,
seams on a word boundary, one host word filled by 11 chunks, empty chunks between chunks that share a word, the push
metadata cap and the growth of the compaction run table.  A child process checks with torch.profiler that k_place_bits
ran the restated launches and CTAs.  The string-offset limits of this path are in tests/test_limits_gpu.py.

On one H100 80GB HBM3 at a 700 W power limit the module takes about 40 s (about 23 s of it the profiler child), at most about
1.1 GiB of device memory and 5.1 GiB of host memory."""
import ctypes as C
import os
import re
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


def shuffle_host(ctx, arrays, keys, P, n_chunks, nullable=None, window=16 << 20, cap=None, byte_slack=0, ex=None, expect_status=0,
                 shift=0):
    """One world-1 dfd_shuffle_host of `arrays` (host buffers) through Hash(keys, P); checks every output buffer against the
    oracle and returns (chunk_part_starts, HostOut).  cap / byte_slack shrink the outputs (rows / string bytes) relative to
    what the data needs; with expect_status != 0 the call must fail with that status.  shift = 1 puts every output buffer
    at an odd address."""
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
    out = H.HostOut([a.type for a in arrays], total if cap is None else cap, nullable, nbytes, shift)
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
    # fixed widths 1, 2, 4, 8 and 16 without nulls: the two-pass fused path first, then the push transport (nullable).  (An
    # interval key needs its hash mode declared, so MonthDayNano travels as payload only, in the test below.)
    for i, t in enumerate((pa.int8(), pa.int16(), pa.float16(), pa.int32(), pa.int64(), pa.decimal128(38, 0))):
        alone[str(t)] = H.fixed_array(t, n, 30 + i)
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


# ---------------------------------------------------------------- k_place_bits past one CTA, seams and folds ----
# Each case restates its k_place_bits launches (H.bit_launches: per chunk, the runs of every bitmap lane and the fold runs)
# and asserts the boundary it is meant to reach.  Bits are checked bit for bit by verify(), zero bits past the last row too.

def bit_schema(n, seed, key=None):
    """Int64 key (nullable schema, no nulls), Boolean with nulls and Int32 with nulls: four bitmap lanes."""
    import pyarrow as pa

    rng = np.random.Generator(np.random.PCG64(seed))
    key = pa.array(rng.integers(0, 1 << 40, n) if key is None else key, type=pa.int64())
    bl = pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.3, type=pa.bool_())
    i32 = pa.array(rng.integers(0, 1 << 31, n), mask=rng.random(n) < 0.2, type=pa.int32())
    return [key, bl, i32]


BIT_LANES = 4  # key validity, Boolean values, Boolean validity, Int32 validity


def keys_to(dests, P, seed):
    """Int64 keys whose oracle destination under Hash([key], P) is dests[i] (drawn from a pool of keys per destination)."""
    import pyarrow as pa

    pool = np.arange(1 << 16, dtype=np.int64) * 7919 + 13
    pd = orc.partition_ids([pa.array(pool)], len(pool), P)
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.empty(len(dests), np.int64)
    for q in range(P):
        m = dests == q
        out[m] = rng.choice(pool[pd == q], int(m.sum()))
    return out


def cta_boundary_case(target, extra):
    """P = 2, two chunks of R rows with R % 32 == target: chunk 1 starts at host bit `target`.  Its destination-0 run has
    a = 2 * 32768 - target + extra rows, so it ends exactly on the second CTA's last word (extra 0) or one bit past it
    (extra 1).  (At P = 1 the two halves of a call are equal, which lets a run end on a CTA boundary only at residues 0 and
    16, hence two destinations.)"""
    R = 2 * H.BITS_PER_CTA + 64 + target
    a = 2 * H.BITS_PER_CTA - target + extra
    rng = np.random.Generator(np.random.PCG64(100 + target))
    d1 = np.concatenate([np.zeros(a, np.int64), np.ones(R - a, np.int64)])
    dests = np.concatenate([rng.integers(0, 2, R), rng.permutation(d1)])
    return bit_schema(2 * R, target, keys_to(dests, 2, target)), 2, 2


def place_bits_cases():
    """(case, arrays, P, n_chunks) of the multi-CTA cases; case = ("one run", None), ("seam", (residue, bits past the CTA))
    or ("segments", None)."""
    yield ("one run", None), bit_schema(3 * H.BITS_PER_CTA + 5, 1), 1, 1
    for target in (0, 1, 17, 31):
        for extra in (0, 1):
            yield ("seam", (target, extra)), *cta_boundary_case(target, extra)
    yield ("segments", None), bit_schema(8 * 50_000, 2), 8, 1


def check_place_bits_case(case, cps, P):
    what, arg = case
    launches = H.bit_launches(cps, BIT_LANES)
    multi = [(d, n) for _, _, runs in launches for d, n, _ in runs if H.run_ctas(d, n) > 1]
    if what == "one run":
        (_, _, runs), = launches
        assert [H.run_words(d, n) for d, n, _ in runs] == [3 * H.BIT_WORDS_PER_CTA + 1] * BIT_LANES
        assert [H.run_ctas(d, n) for d, n, _ in runs] == [4] * BIT_LANES  # CTAs 1-3 run at w0 > 0, reading src[t-1] across
    elif what == "seam":
        target, extra = arg
        (_, _, r0), (ch, out_row, r1) = launches
        assert ch == 1 and out_row & 31 == target
        d, n, _ = r1[0]  # destination 0 of chunk 1, first lane
        assert d == target and (d & 31) + n == 2 * H.BITS_PER_CTA + extra
        assert H.run_words(d, n) == 2 * H.BIT_WORDS_PER_CTA + extra and H.run_ctas(d, n) == 2 + extra
        assert sum(1 for _, _, fold in r1 if fold) == (BIT_LANES if target else 0)
    else:
        (_, _, runs), = launches
        assert len(runs) == P * BIT_LANES and len(multi) == P * BIT_LANES >= 24  # dozens of multi-CTA runs in one launch
        assert H.launch_ctas(runs) >= 2 * P * BIT_LANES
    return launches


def test_place_bits_past_one_cta(ctx):
    for case, arrays, P, n_chunks in place_bits_cases():
        cps, _ = shuffle_host(ctx, arrays, [0], P, n_chunks, nullable=[True] * 3)
        check_place_bits_case(case, cps, P)


PROFILE_CHILD = "DFD_TEST_HOST_SHUFFLE_PROFILE"


def test_place_bits_launches_match_the_restated_runs(ctx, tmp_path):
    """A child process (a profiler session of its own: kernel records of a long-running test process can stop) runs the
    multi-CTA cases under torch.profiler and asserts that k_place_bits ran once per delivering chunk, with the restated
    number of CTAs when the trace carries each kernel's grid."""
    if not os.environ.get(PROFILE_CHILD):
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
            "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider", "-k", "test_place_bits_launches_match_the_restated_runs"]
        r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **{PROFILE_CHILD: "1"}), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]
        return
    import json

    import torch
    from torch.profiler import ProfilerActivity, profile

    want = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case, arrays, P, n_chunks in place_bits_cases():
            cps, _ = shuffle_host(ctx, arrays, [0], P, n_chunks, nullable=[True] * 3)
            want += [H.launch_ctas(runs) for _, _, runs in check_place_bits_case(case, cps, P)]
        torch.cuda.synchronize()
    trace = str(tmp_path / "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and "k_place_bits" in e.get("name", "")]
    ev.sort(key=lambda e: e["ts"])
    assert len(ev) == len(want) == 18, (len(ev), want)  # 1 + 8 x 2 + 1 delivering chunks
    grids = [e.get("args", {}).get("grid") for e in ev]
    if all(grids):
        assert [g[0] for g in grids] == want, ([g[0] for g in grids], want)


@pytest.mark.parametrize("case", ["multiples of 32 rows", "3-row chunks", "empty chunks between"])
def test_seams_and_folds(ctx, case):
    """P = 1: chunks of 224 rows (every seam on a word boundary: no fold); 11 chunks of 3 rows (host word 0 collects the
    bits of all 11); 40 rows in 64 chunks (empty chunks between chunks that share a word, so the fold reads the output stage
    of the chunk two back, and every nonzero seam residue 1-31)."""
    n, n_chunks = {"multiples of 32 rows": (5 * 224, 5), "3-row chunks": (33, 11), "empty chunks between": (40, 64)}[case]
    cps, _ = shuffle_host(ctx, bit_schema(n, 5), [0], 1, n_chunks, nullable=[True] * 3)
    launches = H.bit_launches(cps, BIT_LANES)
    folds = [(ch, out_row) for ch, out_row, runs in launches if any(f for _, _, f in runs)]
    if case == "multiples of 32 rows":
        assert len(launches) == 5 and all(out_row % 32 == 0 for _, out_row, _ in launches) and not folds
    elif case == "3-row chunks":
        assert sum(1 for _, out_row, _ in launches if out_row >> 5 == 0) == 11 and len(folds) == 10
    else:
        chunks = [ch for ch, _, _ in launches]
        assert len(chunks) == 40 and any(b - a == 2 for a, b in zip(chunks, chunks[1:]))  # delivering, empty, delivering
        assert {out_row & 31 for _, out_row in folds} == set(range(1, 32))
        assert any(ch - prev == 2 and out_row & 31 for (prev, _, _), (ch, out_row, _) in zip(launches, launches[1:]))


# ---------------------------------------------------------------------------------- column kinds and widths ----

@pytest.mark.parametrize("n_chunks", [3, 7])
def test_every_fixed_width_beside_a_boolean(ctx, n_chunks):
    """Nullable and non-nullable columns of 1, 2, 4, 8 and 16 bytes next to a nullable Boolean, in the push transport."""
    import pyarrow as pa

    n = 12_345
    rng = np.random.Generator(np.random.PCG64(21))
    arrays = [pa.array(rng.integers(0, 1 << 40, n), type=pa.int64()),
              pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.3, type=pa.bool_())]
    for i, (t, nf) in enumerate([(pa.int8(), 0.2), (pa.int8(), 0), (pa.int16(), 0.3), (pa.float16(), 0), (pa.int32(), 0.1), (pa.int32(), 0),
                                 (pa.int64(), 0.5), (pa.decimal128(38, 0), 0.2), (pa.month_day_nano_interval(), 0)]):
        arrays.append(H.fixed_array(t, n, 40 + i, nf))
    shuffle_host(ctx, arrays, [0], 6, n_chunks)


@pytest.mark.parametrize("P", [6, 64])
def test_binary_in_the_mixed_schema(ctx, P):
    arrays = H.mixed_arrays(20_011, 19, binary=True)
    assert arrays[-1].null_count > 0
    shuffle_host(ctx, arrays, [0, 1], P, 5, nullable=[True] * len(arrays))


@pytest.mark.parametrize("width", [1, 2, 16])
def test_key_on_a_narrow_or_wide_column(ctx, width):
    """Hash keys of 1, 2 and 16 bytes (Int8, Int16, Decimal128, with nulls), alone and with an Int64 key."""
    import pyarrow as pa

    n = 15_007
    t = {1: pa.int8(), 2: pa.int16(), 16: pa.decimal128(38, 0)}[width]
    rest = H.mixed_arrays(n, 31)
    arrays = [H.fixed_array(t, n, 50 + width, 0.1)] + rest[1:4]
    shuffle_host(ctx, arrays, [0], 6, 3)
    shuffle_host(ctx, [arrays[0], rest[0], rest[3]], [1, 0], 6, 3)


@pytest.mark.parametrize("n_chunks", [1, 3, 7])
def test_fused_path_at_every_width_exact_and_one_short(ctx, n_chunks):
    """Fixed-width non-null columns of 1, 2, 4, 8 and 16 bytes take the two-pass fused path: exact capacity delivers, one row
    short is DFD_ERR_CAPACITY with nothing written past the capacity."""
    import pyarrow as pa

    n = 30_011
    arrays = [H.fixed_array(t, n, 60 + i) for i, t in enumerate((pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.decimal128(38, 0)))]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(16 << 20)
    shuffle_host(ctx, arrays, [3], 8, n_chunks, ex=ex)
    assert ex.stats()["shuffles"] == n_chunks
    err, out = shuffle_host(ctx, arrays, [3, 0], 8, n_chunks, cap=n - 1, ex=ex, expect_status=7)
    assert f"hold {n - 1} rows" in str(err), err
    for b in out.bufs.values():
        assert (b[0][b[1]:] == H.FILL).all()
    shuffle_host(ctx, arrays, [4], 8, n_chunks, ex=ex)  # the exchange is still usable
    ex.close()


# ------------------------------------------------------------------------ inputs the staging must not assume ----

def strings_from_lengths(typ, lens, base, seed, null_frac=0.0):
    """A string array whose offsets start at `base` (bytes before it are junk no row covers)."""
    import pyarrow as pa

    rng = np.random.Generator(np.random.PCG64(seed))
    off = base + np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    data = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    validity = pa.py_buffer(np.packbits(rng.random(len(lens)) >= null_frac, bitorder="little").tobytes()) if null_frac else None
    odt = np.int64 if typ == pa.large_string() else np.int32
    return pa.Array.from_buffers(typ, len(lens), [validity, pa.py_buffer(off.astype(odt).tobytes()), pa.py_buffer(data.tobytes())])


def test_string_offsets_starting_at_an_odd_value(ctx):
    """Utf8, Binary and LargeUtf8 whose offsets start at 1 000 003: the output offsets still start at 0."""
    import pyarrow as pa

    n = 9_001
    rng = np.random.Generator(np.random.PCG64(71))
    key = pa.array(rng.integers(0, 1 << 40, n), type=pa.int64())
    arrays = [key] + [strings_from_lengths(t, rng.integers(0, 30, n), 1_000_003, 72 + i, 0.2)
                      for i, t in enumerate((pa.string(), pa.binary(), pa.large_string()))]
    for a in arrays[1:]:
        assert np.frombuffer(a.buffers()[1], np.int64 if a.type == pa.large_string() else np.int32)[0] == 1_000_003
    for n_chunks in (1, 4):
        shuffle_host(ctx, arrays, [0], 6, n_chunks)
        shuffle_host(ctx, arrays, [1, 0], 6, n_chunks)


def test_chunk_seams_at_every_byte_residue(ctx):
    """16 chunks of 500 rows whose first byte offsets fall at residues 0 .. 15 mod 16 (rows of 16 bytes, the last row of each
    chunk 17), for Utf8, Binary and LargeUtf8."""
    import pyarrow as pa

    R, k = 500, 16
    n = R * k
    lens = np.full(n, 16)
    lens[R - 1::R] = 17
    rng = np.random.Generator(np.random.PCG64(81))
    arrays = [pa.array(rng.integers(0, 1 << 40, n), type=pa.int64())] + [strings_from_lengths(t, lens, 0, 82 + i, 0.1)
                                                                         for i, t in enumerate((pa.string(), pa.binary(), pa.large_string()))]
    off = np.concatenate([[0], np.cumsum(lens)])
    assert [int(off[n * i // k]) % 16 for i in range(k)] == list(range(16))
    shuffle_host(ctx, arrays, [0], 6, k)


def test_every_buffer_at_an_odd_address(ctx):
    """Every input and output buffer at an odd host address: the mixed schema with Binary (push transport) and fixed widths
    1 to 16 without nulls (fused path)."""
    import pyarrow as pa

    arrays = [H.at_odd_address(a) for a in H.mixed_arrays(10_007, 91, binary=True)]
    shuffle_host(ctx, arrays, [0, 1], 6, 5, nullable=[True] * len(arrays), shift=1)
    fixed = [H.at_odd_address(H.fixed_array(t, 10_007, 92 + i)) for i, t in enumerate((pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.decimal128(38, 0)))]
    shuffle_host(ctx, fixed, [3], 6, 5, shift=1)


# ---------------------------------------------------------------------------------------- pipeline and reuse ----

def test_2_pow_20_rows_in_64_chunks(ctx):
    """2^20 rows of the mixed schema in 64 chunks at P = 8: H2D, push, compaction and D2H overlap on 16 384-row chunks."""
    arrays = H.mixed_arrays(1 << 20, 101)
    shuffle_host(ctx, arrays, [0, 1], 8, 64, nullable=[True] * 6, window=64 << 20)


def test_one_exchange_fixed_then_mixed_then_larger_mixed_then_fixed(ctx):
    import pyarrow as pa

    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(32 << 20)
    fixed = [H.fixed_array(t, 20_003, 110 + i) for i, t in enumerate((pa.int64(), pa.int16(), pa.decimal128(38, 0)))]
    shuffle_host(ctx, fixed, [0], 6, 3, ex=ex)
    shuffle_host(ctx, H.mixed_arrays(5_003, 111), [0, 1], 6, 3, nullable=[True] * 6, ex=ex)
    shuffle_host(ctx, H.mixed_arrays(80_021, 112, binary=True), [0, 1], 6, 2, nullable=[True] * 7, ex=ex)  # larger stages
    shuffle_host(ctx, fixed, [0, 1], 6, 4, ex=ex)
    ex.close()


PUSH_RUN_BYTES, BIT_RUN_BYTES = 48, 40  # sizeof(PushRun), sizeof(BitRun) in dfd_exchange.cu


def test_run_table_grows_between_two_chunks(ctx):
    """P = 256: every key of chunk 0 goes to destination 0, chunk 1's keys cover all 256.  The compaction run table sized
    for chunk 0 (twice its need) is too small for chunk 1 and is reallocated inside the call."""
    import pyarrow as pa

    P, R = 256, 4_000
    rng = np.random.Generator(np.random.PCG64(121))
    dests = np.concatenate([np.zeros(R, np.int64), rng.permutation(np.arange(R) % P)])
    key = keys_to(dests, P, 121)
    arrays = [pa.array(key, type=pa.int64()), pa.array(rng.random(2 * R) < 0.5, type=pa.bool_())]
    cps, _ = shuffle_host(ctx, arrays, [0], P, 2, nullable=[True, False])
    need = []
    for ch in range(2):
        segs = int((np.diff(cps[ch]) > 0).sum())
        (_, _, runs), = [lch for lch in H.bit_launches(cps, 2) if lch[0] == ch]
        need.append((segs * PUSH_RUN_BYTES + 15) // 16 * 16 + len(runs) * BIT_RUN_BYTES)
    assert need[1] > 2 * need[0], need


# ------------------------------------------------------------------------------------------- metadata cap ----

def test_push_metadata_cap(ctx):
    """(1 + V) x P x T <= 2048 metadata entries: V = 2 (Utf8 + LargeUtf8) at P = 682 (2046) delivers and P = 683 (2049) is
    DFD_ERR_UNSUPPORTED with every output buffer untouched, after which the exchange takes P = 682 again; V = 0 (nullable
    Int64 alone) at P = 2048 delivers and P = 2049 is refused."""
    import pyarrow as pa

    with open(os.path.join(ROOT, "datafusion_distributed_b200", "csrc", "dfd_types.cuh")) as f:
        meta_max = int(re.search(r"XCHG_META_MAX\s*=\s*(\d+);", f.read()).group(1))
    n = 6_007
    m = H.mixed_arrays(n, 131)
    arrays = [m[0], m[1], m[2]]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(32 << 20)
    assert 3 * 682 <= meta_max < 3 * 683
    shuffle_host(ctx, arrays, [0], 682, 2, nullable=[True] * 3, ex=ex)
    err, out = shuffle_host(ctx, arrays, [0], 683, 2, nullable=[True] * 3, ex=ex, expect_status=6)
    assert "metadata entries" in str(err), err
    for b in out.bufs.values():
        assert (b[0] == H.FILL).all()
    shuffle_host(ctx, arrays, [0], 682, 2, nullable=[True] * 3, ex=ex)
    i64 = [pa.array(np.arange(n) * 31, mask=np.arange(n) % 7 == 0, type=pa.int64())]
    shuffle_host(ctx, i64, [0], 2048, 2, ex=ex)
    err, out = shuffle_host(ctx, i64, [0], 2049, 2, ex=ex, expect_status=6)
    assert "metadata entries" in str(err), err
    for b in out.bufs.values():
        assert (b[0] == H.FILL).all()
    ex.close()
