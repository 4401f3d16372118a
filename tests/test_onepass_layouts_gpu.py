"""GPU parity tests of the single-pass partition at the layouts its write-out caps and region arithmetic are sized for.

k_scatter_onepass holds a compile-time number of write-out slots per tile: KP pairs per thread in the local write-out
(T / 2 + 63 N pairs at most for N <= 16, T / 2 + N above), KV rows per thread in the aligned write-out (T + 62 N).  A
pair past the cap would be dropped: rows would go missing with no fault.  Random keys pad a destination's run by about
half the worst case, so the constructions here (tests/util.py worst_case_counts, residue_sweep_counts) build the key
column tile by tile: run starts at 63 (mod 64) and counts of 2 (mod 64), odd starts and even counts above N = 16, and
every run-start residue mod 64 for every destination.

Each construction, and random keys at N in {1, 3, 8, 17, 48, 256} and n from 0 to multi_tile_rows(), runs with regions
of exactly the largest count (odd), the largest + 1 and + 31 (not a multiple of 32), and the largest - 1 or a skewed key
(the exact dense re-run, synchronous and through collect()), under four schemas: the fast Int64 key; a generic Int16 key
with 1-16 byte columns; a two-column nullable key with nullable columns of every width and two Booleans (bit follow-up
launches); 30 mixed-width nullable columns (fixed-width follow-ups past MAX_COLS_PER_LAUNCH).

Checks are on raw buffers, not Array.equals (which ignores values under null slots; the kernel moves them anyway):
every output row's bytes, validity bit and Boolean bit are its input row's, in stable order; bits outside the
destinations' rows are 0 (the library zeroes bitmaps) and fixed-width rows outside keep the guard fill; a guard tail past
N * region_rows is untouched.  After a re-run, rows and bits in [n, N * region_rows) are unspecified: the first launch
may have written there, so nothing is asserted on them.

The peer side runs the constructions through shuffle_onepass and EXCHANGE_FUSED at world 1."""
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.test_instantiations_gpu import assert_ran, check_exchange, profiled, targets
from tests.util import (PAIR_ALIGN_MAX_N, dest_lut, domain_values, expected_partitions, keys_for_counts, multi_tile_rows,
                        region_construction, residue_sweep_counts, tile_geometry, tile_slots, worst_case_counts)

pytestmark = pytest.mark.gpu
GUARD = 0xA5  # fill of every output buffer before a call
TAIL = 64  # guard rows (and guard bitmap words) past N * region_rows
MAX_COLS_PER_LAUNCH = 24  # dfd_types.cuh


# ------------------------------------------------------------------------------------------------- schemas ----

def _col(rng, kind, n, nulls):
    mask = rng.random(n) < 0.3 if nulls else None
    if kind == "dec128":
        data = pa.py_buffer(rng.integers(0, 256, n * 16, dtype=np.uint8).tobytes())
        valid = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if nulls else None
        return pa.Array.from_buffers(pa.decimal128(38, 0), n, [valid, data], null_count=int(mask.sum()) if nulls else 0)
    if kind == "bool":
        return pa.array(rng.random(n) < 0.5, mask=mask)
    dt = {"u8": np.uint8, "i16": np.int16, "i32": np.int32, "i64": np.int64}[kind]
    info = np.iinfo(dt)
    return pa.array(rng.integers(info.min, info.max, n, dtype=dt, endpoint=True), mask=mask)


def _nullable_key_pool(N):
    """Two-column key pool (Int16 v, Int32 7) for every v, then (v, null): 2^17 entries and their destinations."""
    v = domain_values("i16")
    k0 = pa.array(np.concatenate([v, v]))
    k1 = pa.array(np.full(2 * len(v), 7, dtype=np.int32), mask=np.arange(2 * len(v)) >= len(v))
    return (k0, k1), orc.partition_ids([k0, k1], 2 * len(v), N).astype(np.int32)


SCHEMAS = ("fast", "generic", "nullable", "wide")


def pool_of(schema, N):
    """Destinations of every key pool entry of a schema (indexed like the pool)."""
    if schema in ("fast", "wide"):
        return dest_lut("i64", N)
    if schema == "generic":
        return dest_lut("i16", N)
    return _nullable_key_pool(N)[1]


def table(schema, N, idx, seed):
    """(arrays, key columns) of a schema whose key column(s) are the key pool rows `idx`."""
    n, rng = len(idx), np.random.Generator(np.random.PCG64(seed))
    if schema == "fast":
        arrays = [pa.array(domain_values("i64")[idx]), _col(rng, "i64", n, False), _col(rng, "i64", n, False)]
        return arrays, [0]
    if schema == "generic":
        arrays = [pa.array(domain_values("i16")[idx])] + [_col(rng, k, n, False) for k in ("u8", "i16", "i32", "i64", "dec128")]
        return arrays, [0]
    if schema == "nullable":
        (k0, k1), _ = _nullable_key_pool(N)
        take = pa.array(idx)
        arrays = [k0.take(take), k1.take(take)] + [_col(rng, k, n, True) for k in ("u8", "i16", "i32", "i64", "dec128", "bool")]
        return arrays + [_col(rng, "bool", n, False)], [0, 1]
    kinds = ["u8", "i16", "i32", "i64", "dec128"]
    return [pa.array(domain_values("i64")[idx])] + [_col(rng, kinds[j % 5], n, j % 2 == 0) for j in range(29)], [0]


def instantiations(schema, arrays, N):
    """The single-pass and follow-up instantiations a local call of this schema launches (dispatch of run_onepass)."""
    fixed = [a for a in arrays if not pa.types.is_boolean(a.type)]
    widths = [a.type.byte_width for a in fixed]
    ring = min(max(widths[:MAX_COLS_PER_LAUNCH]), 8)
    fast = schema in ("fast", "wide")
    want = targets(1, fast and ring == 8, [ring], False, N)
    follow = sorted(set(widths[MAX_COLS_PER_LAUNCH:]))
    if any(a.null_count for a in arrays) or any(pa.types.is_boolean(a.type) for a in arrays):
        follow.append(0)
    return want | targets(2, fast, follow, False, N) if follow else want


# ------------------------------------------------------------------------------------- peer aligned write-out ----

def exchange_starts(ctx, arrays, key_cols, P, window):
    """Segment starts of one world-1 single-pass shuffle (partition q's sub-window is segment q)."""
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    try:
        ex.setup_window(window)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash(key_cols, P), uuid.uuid4(), 1, 1, 1)
        in_cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
        node.shuffle_onepass(ex, in_cols, len(arrays[0]))
        _, seg_starts, _ = node.collect(ex)
        return seg_starts[:, 0]
    finally:
        ex.close()


# (first in the file: after the many profiled local cases, a profiler session in the same process recorded no kernels)
@pytest.mark.parametrize("fast", [pytest.param(True, id="fast_key"), pytest.param(False, id="generic_key")])
@pytest.mark.parametrize("P", [8, 16])
def test_peer_aligned_constructed_runs(ctx, P, fast):
    """Runs built to fill the aligned write-out (o = 31 mod 32, counts of 2 mod 32) against the sub-window stride of
    the exchange, learnt from a first call, through shuffle_onepass and EXCHANGE_FUSED."""
    pool = dest_lut("i64" if fast else "i16", P)
    vals = domain_values("i64" if fast else "i16")
    probe = np.random.Generator(np.random.PCG64(P)).integers(0, len(pool), 4 * T)
    schema = lambda idx: [pa.array(vals[idx]), pa.array(np.arange(len(idx), dtype=np.int32)),  # noqa: E731
                          _col(np.random.Generator(np.random.PCG64(len(idx))), "dec128", len(idx), False)]
    window = 64 << 20
    starts = exchange_starts(ctx, schema(probe), [0], P, window)
    stride = int(starts[1] - starts[0])
    assert (np.diff(starts) == stride).all() and stride % 32 == 0, starts
    cnt = worst_case_counts(P, T, 3, [(p * stride) % 32 for p in range(P)], aligned=True)
    slots = tile_slots(cnt, np.arange(P) * stride, P, aligned=True)
    assert slots.max() >= T + 62 * P - 62, slots
    assert int(cnt.sum(axis=0).max()) <= stride
    arrays = schema(keys_for_counts(cnt, pool, seed=P))
    assert np.array_equal(exchange_starts(ctx, arrays, [0], P, window), starts)  # (the same stride for these rows)
    ring = 8  # (the Decimal128 column makes the widest column 16 bytes: an 8-byte ring)
    fallbacks, ran = profiled(ctx, lambda: check_exchange(ctx, arrays, [0], P, window=window))
    assert fallbacks == 0
    assert_ran(ran, targets(1, fast, [ring], True, P))
    _, ran = profiled(ctx, lambda: check_exchange(ctx, arrays, [0], P, fused=True, window=window))
    assert_ran(ran, targets(0, fast, [8, 4, 16] if fast else [2, 4, 16], True, P))


# ------------------------------------------------------------------------------------------ raw buffer checks ----

def _bits(buf, offset, n):
    return np.unpackbits(np.frombuffer(buf, dtype=np.uint8), bitorder="little")[offset:offset + n].astype(bool)


def out_columns(ctx, dcols, rows):
    """Output columns of `rows` rows plus TAIL guard rows, every byte GUARD: [(DeviceColumn, values buffer, validity buffer)]."""
    outs = []
    words = (rows + 31) // 32 + TAIL
    for c in dcols:
        vb = ctx.upload(np.full(words * 4, GUARD, dtype=np.uint8)) if c.validity else None
        nbytes = words * 4 if c.kind == nv.COL_BOOL else (rows + TAIL) * c.width
        b = ctx.upload(np.full(nbytes, GUARD, dtype=np.uint8))
        outs.append((dfd.DeviceColumn(c.kind, c.width, b.ptr, 0, vb.ptr if vb else 0, 0, rows, [vb, b], c.arrow_type), b, vb))
    return outs


def check_raw(arrays, outs, order, ref_starts, starts, rows, n, dense):
    """Every output row / bit against its input row; outside the destinations' rows, guard fill (fixed width) or 0 (bits);
    the tail past `rows` untouched.  `dense`: after a re-run, [n, rows) is unspecified."""
    N = len(starts)
    dst = np.concatenate([np.arange(starts[p], starts[p] + ref_starts[p + 1] - ref_starts[p]) for p in range(N)]).astype(np.int64)
    src = order.astype(np.int64)
    written = np.zeros(rows, dtype=bool)
    written[dst] = True
    free = ~written
    if dense:
        free[n:] = False
    zero_to = ((rows + 31) // 32) * 32  # bits the library zeroes before the launch
    for c, (arr, (col, b, vb)) in enumerate(zip(arrays, outs)):
        bufs = arr.buffers()
        if pa.types.is_boolean(arr.type):
            got = _bits(b.download(np.uint8), 0, zero_to + TAIL * 32)
            want = _bits(bufs[1], arr.offset, n)
            assert np.array_equal(got[dst], want[src]), (c, "boolean bits")
            assert not got[:rows][free].any() and (dense or not got[rows:zero_to].any()), (c, "boolean bits outside the runs")
            assert (b.download(np.uint8)[zero_to // 8:] == GUARD).all(), (c, "boolean guard tail")
        else:
            w = arr.type.byte_width
            got = b.download(np.uint8).reshape(-1, w)
            want = np.frombuffer(bufs[1], dtype=np.uint8)[arr.offset * w:(arr.offset + n) * w].reshape(n, w)
            assert np.array_equal(got[dst], want[src]), (c, arr.type, "values")
            assert (got[:rows][free] == GUARD).all(), (c, arr.type, "rows outside the runs")
            assert (got[rows:] == GUARD).all(), (c, arr.type, "guard tail")
        if vb is not None:
            got = _bits(vb.download(np.uint8), 0, zero_to + TAIL * 32)
            want = _bits(bufs[0], arr.offset, n)
            assert np.array_equal(got[dst], want[src]), (c, "validity bits")
            assert not got[:rows][free].any() and (dense or not got[rows:zero_to].any()), (c, "validity bits outside the runs")
            assert (vb.download(np.uint8)[zero_to // 8:] == GUARD).all(), (c, "validity guard tail")


def run_local(ctx, arrays, key_cols, N, rr, rerun, sync):
    """One partition_onepass call into guarded output columns, checked raw against the oracle.  `rerun`: whether the
    regions overflow (the metrics' re-run count then grows by exactly one, and the layout is dense)."""
    n = len(arrays[0])
    dest = orc.partition_ids([arrays[k] for k in key_cols], n, N)
    order, ref_starts = expected_partitions(dest, N)
    counts_ref = np.diff(ref_starts)
    assert (int(counts_ref.max()) > rr if n else False) == rerun, "the case does not reach the layout it is built for"
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    outs = out_columns(ctx, dcols, N * rr)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N))
    before = ctx.metrics()["onepass_reruns"]
    _, starts, counts = part.partition_onepass(dcols, n, rr, [o[0] for o in outs], sync=sync)
    if not sync:
        assert starts is None
        starts, counts = part.collect()
    assert ctx.metrics()["onepass_reruns"] - before == int(rerun)
    assert np.array_equal(counts, counts_ref), (counts, counts_ref)
    want_starts = ref_starts[:-1] if rerun else np.arange(N, dtype=np.int64) * rr
    assert np.array_equal(starts, want_starts), (starts, want_starts)
    check_raw(arrays, outs, order, ref_starts, starts, N * rr, n, rerun)


# --------------------------------------------------------------------------------- constructed destination runs ----

T = tile_geometry()[1]
CONSTRUCTIONS = {  # name -> (N, builder of counts from base residues and delta, modulus of the residues)
    "worst16": (16, lambda b, d: worst_case_counts(16, T, 3, b), 64),
    "worst8": (8, lambda b, d: worst_case_counts(8, T, 3, b), 64),
    "pairs17": (17, lambda b, d: worst_case_counts(17, T, 3, b), 2),
    "pairs256": (256, lambda b, d: worst_case_counts(256, T, 3, b), 2),
    "sweep3": (3, lambda b, d: residue_sweep_counts(3, T, b, 1), 64),
    "sweep8": (8, lambda b, d: residue_sweep_counts(8, T, b, 1), 64),
}
LAYOUTS = {  # name -> (region rows - the largest count, re-run, sync)
    "exact_odd": (0, False, True), "plus1": (1, False, True), "plus31": (31, False, True),
    "minus1_sync": (-1, True, True), "minus1_collect": (-1, True, False),
}


def constructed(name, delta):
    N, make, M = CONSTRUCTIONS[name]
    cnt, rr = region_construction(lambda b: make(b, delta), N, delta, M)
    return N, cnt, rr


@pytest.mark.parametrize("schema", SCHEMAS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("name", list(CONSTRUCTIONS))
def test_local_constructed_runs(ctx, name, layout, schema):
    delta, rerun, sync = LAYOUTS[layout]
    N, cnt, rr = constructed(name, delta)
    if not rerun:  # the region layout is the one the runs were built against
        pairs = tile_slots(cnt, np.arange(N) * rr, N)
        if N <= PAIR_ALIGN_MAX_N and name.startswith("worst"):
            assert pairs.max() >= T // 2 + 63 * N - 63, pairs
        if name == "worst16" and delta == 1:
            assert pairs[-1] == cnt[-1].sum() // 2 + 63 * N, pairs  # the bound, exactly
    idx = keys_for_counts(cnt, pool_of(schema, N), seed=N * 7 + delta)
    arrays, key_cols = table(schema, N, idx, seed=N + delta)
    if layout in ("exact_odd", "minus1_sync"):
        _, ran = profiled(ctx, lambda: run_local(ctx, arrays, key_cols, N, rr, rerun, sync))
        assert_ran(ran, instantiations(schema, arrays, N))
    else:
        run_local(ctx, arrays, key_cols, N, rr, rerun, sync)


# ------------------------------------------------------------------------------------------------- random keys ----

RANDOM_N = [1, 3, 8, 17, 48, 256]
RANDOM_SIZES = ["0", "1", "31", "33", "tile-1", "tile+1", "multi_tile"]
RANDOM_LAYOUTS = ["exact_odd", "plus1", "plus31", "minus1_sync", "minus1_collect", "skew_sync", "skew_collect"]


def random_rows(size):
    return {"tile-1": T - 1, "tile+1": T + 1, "multi_tile": multi_tile_rows()}[size] if not size.isdigit() else int(size)


@pytest.mark.parametrize("layout", RANDOM_LAYOUTS)
@pytest.mark.parametrize("size", RANDOM_SIZES)
@pytest.mark.parametrize("N", RANDOM_N, ids=lambda N: f"N{N}")
def test_local_random_keys(ctx, N, size, layout):
    """Random keys; the schema rotates with the case (multi-tile sizes skip the 30-column one to bound the run time)."""
    n = random_rows(size)
    i = RANDOM_N.index(N) + RANDOM_SIZES.index(size) + RANDOM_LAYOUTS.index(layout)
    schema = SCHEMAS[i % (3 if size == "multi_tile" else 4)]
    rng = np.random.Generator(np.random.PCG64(i))
    dests = pool_of(schema, N)
    if layout.startswith("skew"):  # 90 % of the rows on one key: destination dests[k] outgrows a fair region
        idx = np.where(rng.random(n) < 0.9, 12345, rng.integers(0, len(dests), n))
    else:
        idx = rng.integers(0, len(dests), n)
    counts = np.bincount(dests[idx], minlength=N)
    mx = int(counts.max()) if n else 0
    rerun = layout.startswith(("minus1", "skew"))
    if layout.startswith("skew"):
        rr = -(-n // N) + 1
    else:
        rr = mx + {"exact_odd": 0, "plus1": 1, "plus31": 31, "minus1_sync": -1, "minus1_collect": -1}[layout]
        if layout == "exact_odd" and rr % 2 == 0:
            rr += 1  # (one more row than the largest count: still no re-run)
    if rerun and (rr < 1 or rr * N < n or mx <= rr):
        pytest.skip(f"no valid overflowing region size at n={n}, N={N} (largest count {mx})")
    rr = max(rr, 1)
    arrays, key_cols = table(schema, N, idx, seed=i)
    run_local(ctx, arrays, key_cols, N, rr, rerun, not layout.endswith("collect"))


# --------------------------------------------------------------------------------------- dense fallbacks ----

def run_dense(ctx, arrays, key_cols, N, n):
    """dfd_partition_device_onepass on a schema it sends down the dense two-pass path: starts are the prefix sums of the
    counts, and every row and bit is its input row's."""
    dest = orc.partition_ids([arrays[k] for k in key_cols], n, N)
    order, ref_starts = expected_partitions(dest, N)
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N))
    outs = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in dcols]  # (the dense layout needs n rows, whatever region_rows says)
    outs, starts, counts = part.partition_onepass(dcols, n, max(n, 1), outs)
    assert np.array_equal(counts, np.diff(ref_starts)) and np.array_equal(starts, ref_starts[:-1])
    for c, arr in enumerate(arrays):
        got = outs[c].to_arrow(ctx, 0, n)
        want = arr.take(pa.array(order))
        bufs, wb = got.buffers(), want.buffers()
        if pa.types.is_boolean(arr.type):
            assert np.array_equal(_bits(bufs[1], 0, n), _bits(arr.buffers()[1], arr.offset, n)[order]), c
        elif pa.types.is_string(arr.type):
            assert got.equals(want), c
        else:
            w = arr.type.byte_width
            src = np.frombuffer(arr.buffers()[1], dtype=np.uint8)[arr.offset * w:(arr.offset + n) * w].reshape(n, w)
            assert np.array_equal(np.frombuffer(bufs[1], dtype=np.uint8)[:n * w].reshape(n, w), src[order]), c
        if arr.null_count:
            assert np.array_equal(_bits(bufs[0], 0, n), _bits(arr.buffers()[0], arr.offset, n)[order]), (c, "validity")


@pytest.mark.parametrize("n", [0, 1, 33, T + 1, 100_003])
def test_dense_fallbacks_keep_start_count_contract(ctx, n):
    """A Boolean-only schema (no fixed-width column), a schema with a string column, and N > 256."""
    rng = np.random.Generator(np.random.PCG64(n))
    bools = [_col(rng, "bool", n, False), _col(rng, "bool", n, True), _col(rng, "bool", n, True)]
    run_dense(ctx, bools, [0], 8, n)
    strs = pa.array([None if x < 0.2 else "s" * int(x * 20) for x in rng.random(n)], type=pa.string())
    run_dense(ctx, [_col(rng, "i32", n, False), strs, _col(rng, "bool", n, True), _col(rng, "i16", n, True)], [0], 17, n)
    run_dense(ctx, [_col(rng, "i64", n, False), _col(rng, "u8", n, True), _col(rng, "bool", n, True)], [0], 300, n)

