"""GPU parity tests that launch every scatter instantiation the dispatch reaches (tests/util.py scatter_dispatch), one
group of template arguments per case: narrow single-pass rings, generic keys in peer mode, peer follow-up launches, the
two-pass fused exchange with every element width.  Each case records the kernels it launched with torch.profiler and
asserts that the instantiations it targets ran, so a case routed elsewhere (push transport, dense fallback, another ring
width) fails.
The last test checks that the cases together launched every reachable instantiation.
Bar: bit-exact against the oracle per destination or per segment, including row order."""
import sys
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.test_onepass_gpu import check_against_oracle, dev_cols
from tests.util import (WIDTH_V, edge_sizes, expected_partitions, multi_tile_rows, scatter_dispatch, scatter_inst, scatter_instances,
                        tile_geometry, use_aligned)

pytestmark = pytest.mark.gpu
LAUNCHED = set()  # the scatter instantiations the cases of this process ran

SIZES = ["multi_tile", "tile_edge"]
PS = [pytest.param(8, id="P8"), pytest.param(17, id="P17")]  # aligned / linear write-out of peer launches (ALIGNED_MAX_N = 16)


def n_rows(size):
    if size == "multi_tile":
        return multi_tile_rows()
    n = 2 * tile_geometry()[1] + 1  # two single-pass tiles and one row: a ragged two-pass tile too
    assert n in edge_sizes()
    return n


def profiled(ctx, fn):
    """fn() under torch.profiler with CUDA activities: (its result, the scatter instantiations it launched).

    A profiler session late in a long-running test process can come back without any of the kernels it ran.  The
    context's own count of scatter launches tells such a session from a call that launched no scatter kernel: when the
    library launched some and the profiler recorded none, the call is profiled again, at most twice, and fails if no
    session records them.  A call routed to other instantiations records those, so it still fails assert_ran."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        before = ctx.metrics()["scatter_launches"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        launched = ctx.metrics()["scatter_launches"] - before
        ran = scatter_instances(e.name for e in prof.events())
        if ran or not launched:
            break
    assert ran or not launched, f"{launched} scatter launches, and three profiler sessions recorded none of them"
    LAUNCHED.update(ran)
    return out, ran


def targets(mode, fast, widths, peer, N):
    """The instantiations a launch of each column width in `widths` (0 = bit columns) runs, by the dispatch restatement."""
    return {scatter_inst(mode, fast, WIDTH_V[w], peer, use_aligned(N, peer)) for w in widths}


def assert_ran(ran, want):
    assert want <= ran, f"not launched: {sorted(want - ran)}; launched: {sorted(ran)}"


def column(rng, kind, n, offset=0, nulls=False):
    """A seeded column of `kind` (u8, i16, i32, i64, dec128 or bool): rows [offset, offset + n) of a longer array."""
    m = n + offset + 5
    mask = rng.random(m) < 0.3 if nulls else None
    if kind == "dec128":
        raw = pa.py_buffer(rng.integers(0, 256, m * 16, dtype=np.uint8).tobytes())
        a = pa.Array.from_buffers(pa.decimal128(38, 0), m, [None, raw])
    elif kind == "bool":
        a = pa.array(rng.random(m) < 0.5, mask=mask)
    else:
        dt = {"u8": np.uint8, "i16": np.int16, "i32": np.int32, "i64": np.int64}[kind]
        info = np.iinfo(dt)
        a = pa.array(rng.integers(info.min, info.max, m, dtype=dt, endpoint=True), mask=mask)
    return a.slice(offset, n)


def mixed_fixed(rng, n, lead):
    """30 fixed-width columns: the key columns `lead`, filled up to the first MAX_COLS_PER_LAUNCH = 24 (the single-pass
    launch), then six of widths 8, 4, 16, 2, 1, 1: past the per-launch limit, they go to follow-up launches of every
    width.  Mostly narrow columns keep the schema at ~100 bytes a row."""
    fill = 24 - len(lead)
    kinds = (["i32", "i64", "dec128"] + ["u8", "i16"] * fill)[:fill] + ["i64", "i32", "dec128", "i16", "u8", "u8"]
    return lead + [column(rng, k, n) for k in kinds]


def sliced(rng, kind, n):
    return column(rng, kind, n, offset=7)


# ------------------------------------------------------------------------------------------- local single-pass ----

NARROW_KEYS = {  # key name -> (key columns, widest column in bytes)
    "u8": (lambda rng, n: [column(rng, "u8", n)], 1),
    "i16": (lambda rng, n: [column(rng, "i16", n)], 2),
    "i32": (lambda rng, n: [column(rng, "i32", n)], 4),
    "i16_i32": (lambda rng, n: [column(rng, "i16", n), column(rng, "i32", n)], 4),
    "sliced_i16": (lambda rng, n: [sliced(rng, "i16", n)], 2),
}


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("key", list(NARROW_KEYS))
def test_local_onepass_narrow_ring(ctx, key, size, P):
    """Schemas whose widest column is 1, 2 or 4 bytes: the single-pass kernel runs a ring of that width under a generic
    key; a nullable column and a Boolean add follow-up launches of bit columns on the single-pass tiling."""
    n, rng = n_rows(size), np.random.Generator(np.random.PCG64(len(key) * 100 + P))
    make, ring = NARROW_KEYS[key]
    keys = make(rng, n)
    narrow = {1: "u8", 2: "i16", 4: "i32"}[ring]
    arrays = keys + [column(rng, "u8", n), column(rng, narrow, n, nulls=True), column(rng, "bool", n, nulls=True)]
    _, ran = profiled(ctx, lambda: check_against_oracle(ctx, arrays, list(range(len(keys))), P))
    assert_ran(ran, targets(1, False, [ring], False, P) | targets(2, False, [0], False, P))


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("offset", [1, 3, 13])
def test_local_onepass_narrow_ring_sliced_payload(ctx, offset, size):
    """Payload sliced at an odd Arrow offset: the single-pass producer's element-wise fallback copy on a 2-byte ring."""
    n, P = n_rows(size), 8
    rng = np.random.Generator(np.random.PCG64(offset))
    arrays = [column(rng, "i16", n)] + [column(rng, k, n, offset=offset, nulls=nl) for k, nl in
                                        (("u8", False), ("i16", True), ("u8", False), ("bool", True))]
    _, ran = profiled(ctx, lambda: check_against_oracle(ctx, arrays, [0], P))
    assert_ran(ran, targets(1, False, [2], False, P) | targets(2, False, [0], False, P))


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("fast", [pytest.param(True, id="fast_key"), pytest.param(False, id="generic_key")])
def test_local_wide_schema_every_width(ctx, fast, size, P):
    """30 fixed-width columns, a nullable one and a Boolean through partition() (a two-pass launch per width, bit columns
    included) and partition_onepass() (the single-pass launch and follow-ups of every width), under the fast Int64 key
    and a generic (sliced) one."""
    n = n_rows(size)
    rng = np.random.Generator(np.random.PCG64(7 + P))
    key = column(rng, "i64", n) if fast else sliced(rng, "i64", n)
    arrays = mixed_fixed(rng, n, [key]) + [column(rng, "i32", n, nulls=True), column(rng, "bool", n, nulls=True)]
    _, ran = profiled(ctx, lambda: check_against_oracle(ctx, arrays, [0], P))
    assert_ran(ran, targets(1, fast, [8], False, P) | targets(2, fast, [8, 4, 16, 2, 1, 0], False, P))
    _, ran = profiled(ctx, lambda: check_against_oracle(ctx, arrays, [0], P, two_pass=True))
    assert_ran(ran, targets(0, fast, [8, 4, 16, 2, 1, 0], False, P))


# ---------------------------------------------------------------------------------------- exchange at world 1 ----

def check_exchange(ctx, arrays, key_cols, P, fused=False, window=None):
    """World-1 exchange of `arrays` (fixed-width, non-null): single-pass (shuffle_onepass + collect) or two-pass fused
    (EXCHANGE_FUSED).  Partition q is one segment, equal to the oracle's rows in input order.  Returns the exchange's
    count of single-pass shuffles that overflowed and re-ran through the two-pass path."""
    n = len(arrays[0])
    order, ref_starts = expected_partitions(orc.partition_ids([arrays[k] for k in key_cols], n, P), P)
    rb = sum(a.type.byte_width for a in arrays)
    if window is None:  # every (partition, producer) sub-window holds the largest partition
        window = int(rb * P * (int(np.diff(ref_starts).max()) + 64) * 1.1) + (1 << 20)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    try:
        ex.setup_window(window)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash(key_cols, P), uuid.uuid4(), 1, 1, 1)
        in_cols = dev_cols(ctx, arrays)  # (alive until collect(): an overflowed single-pass shuffle re-runs from them)
        if fused:
            outs, starts = node.shuffle(ex, in_cols, n, nv.EXCHANGE_FUSED)
            seg_starts, seg_counts = starts[:-1], np.diff(starts)
        else:
            node.shuffle_onepass(ex, in_cols, n)
            outs, seg_starts, seg_counts = node.collect(ex)
            seg_starts, seg_counts = seg_starts[:, 0], seg_counts[:, 0]
        assert np.array_equal(seg_counts, np.diff(ref_starts))
        for q in range(P):
            idx = pa.array(order[ref_starts[q]:ref_starts[q + 1]])
            for c, arr in enumerate(arrays):
                got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(seg_starts[q]), int(seg_counts[q]))
                assert got.equals(arr.take(idx)), (q, c, arr.type)
        return nv.lib().dfd_exchange_onepass_fallbacks(ex._h)
    finally:
        ex.close()


EXCHANGE_KEYS = {  # key name -> (columns, key columns, widest column up to 8 bytes, fast key)
    "u8": (lambda rng, n: [column(rng, "u8", n), column(rng, "u8", n)], [0], 1, False),
    "i16": (lambda rng, n: [column(rng, "i16", n), column(rng, "u8", n), column(rng, "i16", n)], [0], 2, False),
    "i32": (lambda rng, n: [column(rng, "i32", n), column(rng, "u8", n), column(rng, "i16", n), column(rng, "i32", n)], [0], 4, False),
    "sliced_i64": (lambda rng, n: [sliced(rng, "i64", n), column(rng, "i32", n), column(rng, "dec128", n)], [0], 8, False),
    "i64_i32": (lambda rng, n: [column(rng, "i64", n), column(rng, "i32", n), column(rng, "dec128", n)], [0, 1], 8, False),
    "i64": (lambda rng, n: [column(rng, "i64", n), column(rng, "i32", n), column(rng, "dec128", n)], [0], 8, True),
}


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("key", list(EXCHANGE_KEYS))
def test_exchange_onepass_ring_widths_and_keys(ctx, key, size, P):
    """The single-pass peer kernel with rings of 1, 2, 4 and 8 bytes under generic keys (Int32, a sliced Int64, and
    Int64 + Int32; a 1- or 2-byte ring needs a key that narrow, as the key is one of the moved columns), Decimal128
    columns, and the fast Int64 key.  No sub-window overflows, so nothing re-runs through the two-pass path."""
    n, rng = n_rows(size), np.random.Generator(np.random.PCG64(len(key) * 10 + P))
    make, key_cols, ring, fast = EXCHANGE_KEYS[key]
    arrays = make(rng, n)
    fallbacks, ran = profiled(ctx, lambda: check_exchange(ctx, arrays, key_cols, P))
    assert fallbacks == 0
    assert_ran(ran, targets(1, fast, [ring], True, P))


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("fast", [pytest.param(True, id="fast_key"), pytest.param(False, id="generic_key")])
def test_exchange_onepass_follow_ups(ctx, fast, size, P):
    """A single-pass exchange of 30 fixed-width columns: the six past the per-launch limit go to peer follow-up launches
    of every width, under the fast Int64 key and a generic Int64 + Int32 key."""
    n = n_rows(size)
    rng = np.random.Generator(np.random.PCG64(11 + P))
    arrays = mixed_fixed(rng, n, [column(rng, "i64", n), column(rng, "i32", n)])
    fallbacks, ran = profiled(ctx, lambda: check_exchange(ctx, arrays, [0] if fast else [0, 1], P))
    assert fallbacks == 0
    assert_ran(ran, targets(1, fast, [8], True, P) | targets(2, fast, [8, 4, 16, 2, 1], True, P))


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("fast", [pytest.param(True, id="fast_key"), pytest.param(False, id="generic_key")])
def test_exchange_fused_two_pass_every_width(ctx, fast, size, P):
    """EXCHANGE_FUSED: one two-pass peer launch per width (1, 2, 4, 8 and 16 bytes) under the fast and a generic key."""
    n = n_rows(size)
    rng = np.random.Generator(np.random.PCG64(13 + P))
    key = column(rng, "i64", n) if fast else sliced(rng, "i64", n)
    arrays = [key] + [column(rng, k, n) for k in ("u8", "i16", "i32", "dec128")]
    _, ran = profiled(ctx, lambda: check_exchange(ctx, arrays, [0], P, fused=True))
    assert_ran(ran, targets(0, fast, [8, 4, 16, 2, 1], True, P))


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("size", SIZES)
def test_exchange_onepass_overflow_reruns_narrow_schema(ctx, size, P):
    """A hot Int16 key overflows its single-pass sub-window (2-byte ring); the shuffle re-runs exactly once through the
    two-pass peer kernels of the narrow widths, with the same rows in the same order."""
    n = n_rows(size)
    rng = np.random.Generator(np.random.PCG64(17 + P))
    k = np.full(n, 77, dtype=np.int16)
    k[::50] = rng.integers(-(1 << 15), 1 << 15, len(k[::50]), dtype=np.int16)
    arrays = [pa.array(k), column(rng, "u8", n), column(rng, "i16", n)]
    fallbacks, ran = profiled(ctx, lambda: check_exchange(ctx, arrays, [0], P, window=int(n * 5 * 1.5) + (64 << 10)))
    assert fallbacks == 1
    assert_ran(ran, targets(1, False, [2], True, P) | targets(0, False, [2, 1], True, P))


def test_all_reachable_instantiations_ran_in_process(request):
    """The cases above launched every instantiation the dispatch reaches."""
    here = sys.modules[__name__]
    selected = {it.originalname for it in request.session.items if getattr(it, "module", None) is here}
    everything = {name for name in dir(here) if name.startswith("test_")}
    if selected != everything:
        pytest.skip("needs every test of the module in one run")
    reach = scatter_dispatch()
    missing = set(reach) - LAUNCHED
    assert not missing, "never launched:\n" + "\n".join(f"{i}: {reach[i]}" for i in sorted(missing))
