"""GPU parity tests of the two-pass partition at the edges of its kernels: K1 `k_tile_hist`, K1b `k_scan_tiles`, K2
`k_scatter`, K4 `k_var_*` and `k_gather_rows`.

- K1 histogram variants: NF = 1 / 2 / 4 / 0 packed counters for N <= 4 / <= 8 / <= 16 / above, under the fast Int64 key
  and generic keys, at both sides of every switch point (N = 4|5, 8|9, 16|17, 256|257) and at 1, T - 1, T, T + 1 and a
  ragged multi-tile row count.  A child process records the kernels with torch.profiler and asserts that all eight
  k_tile_hist<..., FAST, NF> instantiations ran.
- K2 with adversarial tiles, built from the key domain of tests/util.py (domain_values / dest_lut): every row of a tile to
  destination 0 or to N - 1, T distinct destinations per tile at N = 4096, destination = row mod N, only destinations
  0 and N - 1, and one row in the ragged last tile.
- K1b: tile counts at both sides of the points where a warp's share of tiles grows (1024|1025, 2048|2049 tiles) and
  part_starts scans of one or several rounds, full or ragged (N = 1023 ... 4096).
- Scratch reuse on one context: N and n_rows growing and shrinking, and two partitioners interleaved.
- Generic keys through every follow-up width (more than MAX_COLS_PER_LAUNCH 8-byte columns; 4, 16, 2 and 1 bytes; a
  nullable Boolean), Utf8 / LargeUtf8 (K4) and FixedSizeList<Float32, 24> (k_gather_rows), sliced, at N up to 4096.
- The fused exchange (world 1) at N = 3996 ... 4096 with Decimal128 and Interval(MonthDayNano) columns: its peer scatter
  keeps the per-destination output bases in the warp-counter region of shared memory, so it fits wherever the local
  scatter does.

Every local case is bit-exact against the C oracle: part_starts, and every output column's bytes in the oracle's
stable order.  Output buffers start filled with a guard byte; the bytes past each output stay untouched, bits past the
last row of a bitmap are zero up to the 32-bit word the library clears, and the bytes past that word keep the guard.

One H100 80GB HBM3 at 700 W: the module's 79 cases take about 35 s, 19 s of it in the child process, with at most about
1.1 GiB of device memory in use."""
import os
import re
import subprocess
import sys
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.util import _int_arg, dest_lut, domain_values, expected_partitions, tile_geometry

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 0xA5  # fill of every output buffer before a call
TAIL = 64  # guard rows (bytes for strings, 32-bit words for bitmaps) past every output
MAX_COLS_PER_LAUNCH = 24  # dfd_types.cuh
SCAN_THREADS = 1024  # k_scan_tiles<1024> (dfd_api.cu run_hist_scan)
T = tile_geometry()[0]  # two-pass tile rows
W_SCAN = SCAN_THREADS // 32
PROFILE_CHILD = "DFD_TEST_TWOPASS_PROFILE"  # set in the child process that records the K1 instantiations


def hist_nf(N):
    """Packed-counter fields of k_tile_hist (run_hist_scan): 1, 2 or 4 64-bit accumulators of four 16-bit counters."""
    return 1 if N <= 4 else 2 if N <= 8 else 4 if N <= 16 else 0


def scan_per(n_tiles):
    """Tiles each warp of k_scan_tiles scans: ceil(n_tiles / W) rounded up to a multiple of 32."""
    return (-(-n_tiles // W_SCAN) + 31) // 32 * 32


def n_tiles_of(n):
    return -(-n // T) if n else 1


# ------------------------------------------------------------------------------------------------- columns ----

def column(rng, kind, n, offset=0, nulls=False):
    """A seeded column of `kind`: rows [offset, offset + n) of a longer array (so the Arrow offset is `offset`)."""
    m = n + offset + 3
    mask = rng.random(m) < 0.25 if nulls else None
    if kind in ("dec128", "mdn"):
        raw = pa.py_buffer(rng.integers(0, 256, m * 16, dtype=np.uint8).tobytes())
        valid = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if nulls else None
        typ = pa.decimal128(38, 0) if kind == "dec128" else pa.month_day_nano_interval()
        a = pa.Array.from_buffers(typ, m, [valid, raw], null_count=int(mask.sum()) if nulls else 0)
    elif kind == "bool":
        a = pa.array(rng.random(m) < 0.5, mask=mask)
    elif kind in ("utf8", "large_utf8"):
        odt = np.int32 if kind == "utf8" else np.int64
        off = np.concatenate([[0], np.cumsum(rng.integers(0, 12, m))]).astype(odt)
        data = rng.integers(97, 123, int(off[-1]), dtype=np.uint8)
        valid = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if nulls else None
        a = pa.Array.from_buffers(pa.string() if kind == "utf8" else pa.large_string(), m,
                                  [valid, pa.py_buffer(off.tobytes()), pa.py_buffer(data.tobytes())], null_count=int(mask.sum()) if nulls else 0)
    elif kind == "fsl24":
        child = pa.array(rng.standard_normal(m * 24).astype(np.float32))
        a = pa.FixedSizeListArray.from_arrays(child, 24, mask=pa.array(mask) if nulls else None)
    else:
        dt = {"u8": np.uint8, "i16": np.int16, "i32": np.int32, "i64": np.int64}[kind]
        info = np.iinfo(dt)
        a = pa.array(rng.integers(info.min, info.max, m, dtype=dt, endpoint=True), mask=mask)
    return a.slice(offset, n)


def keys_for_dests(dests, N, seed, generic=False):
    """An Int64 key column whose row i goes to destination dests[i] (a key drawn from the seeded domain of tests/util.py,
    destinations by the C oracle).  `generic`: the column is sliced (Arrow offset 1), which takes the generic key path."""
    lut, vals = dest_lut("i64", N), domain_values("i64")
    pools = [np.nonzero(lut == p)[0] for p in range(N)]
    used = np.unique(dests)
    assert all(len(pools[p]) for p in used), "a destination no key of the domain reaches"
    rng = np.random.Generator(np.random.PCG64(seed))
    pick = rng.integers(0, 1 << 30, len(dests))
    idx = np.empty(len(dests), dtype=np.int64)
    for p in used:
        sel = dests == p
        idx[sel] = pools[p][pick[sel] % len(pools[p])]
    keys = vals[idx]
    if generic:
        return pa.array(np.concatenate([[0], keys]).astype(np.int64)).slice(1)
    return pa.array(keys)


# ------------------------------------------------------------------------------------------ guarded outputs ----

def _bits(buf, offset, n):
    return np.unpackbits(np.frombuffer(buf, dtype=np.uint8), bitorder="little")[offset:offset + n].astype(bool)


def _is_var(arr):
    return pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type)


def out_columns(ctx, arrays, dcols, n):
    """Output columns of n rows, every byte GUARD, with TAIL guard rows / bytes / words past the end."""
    outs = []
    words = (n + 31) // 32 + TAIL
    for arr, c in zip(arrays, dcols):
        vb = ctx.upload(np.full(words * 4, GUARD, dtype=np.uint8)) if c.validity else None
        if _is_var(arr):
            ow = 8 if pa.types.is_large_string(arr.type) else 4
            ob = ctx.upload(np.full((n + 1 + TAIL) * ow, GUARD, dtype=np.uint8))
            b = ctx.upload(np.full(c.values_bytes + TAIL, GUARD, dtype=np.uint8))
            col = dfd.DeviceColumn(c.kind, 0, b.ptr, ob.ptr, vb.ptr if vb else 0, 0, n, [vb, ob, b], c.arrow_type, c.values_bytes)
            outs.append((col, b, vb, ob))
            continue
        nbytes = words * 4 if c.kind == nv.COL_BOOL else (n + TAIL) * c.width
        b = ctx.upload(np.full(nbytes, GUARD, dtype=np.uint8))
        outs.append((dfd.DeviceColumn(c.kind, c.width, b.ptr, 0, vb.ptr if vb else 0, 0, n, [vb, b], c.arrow_type), b, vb, None))
    return outs


def _check_bitmap(got_buf, want_bits, order, n, what):
    zero_to = (n + 31) // 32 * 32  # the library clears whole 32-bit words
    raw = got_buf.download(np.uint8)
    got = np.unpackbits(raw, bitorder="little").astype(bool)
    assert np.array_equal(got[:n], want_bits[order]), what
    assert not got[n:zero_to].any(), (what, "bits past the last row")
    assert (raw[zero_to // 8:] == GUARD).all(), (what, "bytes past the last word")


def check_columns(arrays, outs, order, n):
    """Every output column's raw bytes (and bits) equal arr.take(order); nothing past the output was written."""
    for c, (arr, (col, b, vb, ob)) in enumerate(zip(arrays, outs)):
        bufs = arr.buffers()
        what = (c, str(arr.type))
        if pa.types.is_boolean(arr.type):
            _check_bitmap(b, _bits(bufs[1], arr.offset, n), order, n, what + ("values",))
        elif _is_var(arr):
            large = pa.types.is_large_string(arr.type)
            odt = np.int64 if large else np.int32
            in_off = np.frombuffer(bufs[1], dtype=odt)[arr.offset:arr.offset + n + 1].astype(np.int64)
            lens = np.diff(in_off)[order]
            want_off = np.concatenate([[0], np.cumsum(lens)]).astype(odt)
            got_raw = ob.download(np.uint8)
            ow = 8 if large else 4
            assert np.array_equal(got_raw[:(n + 1) * ow].view(odt), want_off), what + ("offsets",)
            assert (got_raw[(n + 1) * ow:] == GUARD).all(), what + ("bytes past the offsets",)
            data = np.frombuffer(bufs[2], dtype=np.uint8) if bufs[2] is not None else np.zeros(0, dtype=np.uint8)
            starts = in_off[:-1][order]
            want = np.concatenate([data[s:s + k] for s, k in zip(starts, lens)] + [np.zeros(0, dtype=np.uint8)])
            got = b.download(np.uint8)
            assert np.array_equal(got[:len(want)], want), what + ("bytes",)
            assert (got[len(want):] == GUARD).all(), what + ("bytes past the data",)
        else:
            if pa.types.is_fixed_size_list(arr.type):
                w = arr.type.list_size * arr.type.value_type.bit_width // 8
                child = arr.values  # (the whole child: row i of the list is child rows [i * size, (i + 1) * size))
                src = np.frombuffer(child.buffers()[1], dtype=np.uint8)[child.offset * w // arr.type.list_size:]
            else:
                w = arr.type.byte_width
                src = np.frombuffer(bufs[1], dtype=np.uint8)
            want = src[arr.offset * w:(arr.offset + n) * w].reshape(n, w)[order]
            got = b.download(np.uint8)
            assert np.array_equal(got[:n * w].reshape(n, w), want), what + ("values",)
            assert (got[n * w:] == GUARD).all(), what + ("bytes past the values",)
        if vb is not None:
            _check_bitmap(vb, _bits(bufs[0], arr.offset, n), order, n, what + ("validity",))


def run_partition(ctx, arrays, key_cols, N, part=None):
    """One dfd_partition_device call into guarded outputs, checked against the oracle.  Returns the oracle's starts."""
    n = len(arrays[0])
    dest = orc.partition_ids([arrays[k] for k in key_cols], n, N)
    order, ref_starts = expected_partitions(dest, N)
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    outs = out_columns(ctx, arrays, dcols, n)
    part = part or dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N))
    _, starts = part.partition(dcols, n, [o[0] for o in outs])
    assert np.array_equal(starts, ref_starts), f"part_starts differ at N={N}, n={n}"
    check_columns(arrays, outs, order, n)
    return dest, ref_starts


# ------------------------------------------------------------------------------------------ 1. K1 variants ----

K1_N = [1, 4, 5, 8, 9, 16, 17, 255, 256, 257]
K1_KEYS = ["fast", "nullable", "i64_utf8"]
K1_ROWS = {"1": 1, "T-1": T - 1, "T": T, "T+1": T + 1, "ragged": 5 * T + 77}


def k1_table(rng, key, n):
    """(arrays, key columns): the key(s) of `key`, then a 4-, 16- and 2-byte column and a nullable Boolean."""
    if key == "fast":
        keys = [column(rng, "i64", n)]
    elif key == "nullable":
        keys = [column(rng, "i64", n, nulls=True)]
    else:
        keys = [column(rng, "i64", n), column(rng, "utf8", n, nulls=True)]
    payload = [column(rng, "i32", n), column(rng, "dec128", n), column(rng, "i16", n, nulls=True), column(rng, "bool", n, nulls=True)]
    return keys + payload, list(range(len(keys)))


@pytest.mark.parametrize("key", K1_KEYS)
@pytest.mark.parametrize("N", K1_N, ids=lambda N: f"N{N}")
def test_k1_histogram_variants(ctx, N, key):
    nf = hist_nf(N)
    assert nf == {1: 1, 4: 1, 5: 2, 8: 2, 9: 4, 16: 4}.get(N, 0)
    for i, (name, n) in enumerate(K1_ROWS.items()):
        assert n_tiles_of(n) == {"1": 1, "T-1": 1, "T": 1, "T+1": 2, "ragged": 6}[name]
        arrays, key_cols = k1_table(np.random.Generator(np.random.PCG64(N * 100 + i)), key, n)
        run_partition(ctx, arrays, key_cols, N)


_HIST_NAME = re.compile(r"k_tile_hist<([^>]*)>")


def k1_instances(names):
    """(FAST, NF) of every k_tile_hist<THREADS, K, FAST, NF> among kernel names (demangled)."""
    out = set()
    for name in names:
        m = _HIST_NAME.search(name)
        if m:
            a = [s.strip() for s in m.group(1).split(",")]
            out.add((bool(_int_arg(a[2])), _int_arg(a[3])))
    return out


def test_k1_every_histogram_instantiation_runs(ctx):
    """A child process (a profiler session of its own: kernel records of a long-running test process can stop) runs one
    call per (key path, NF) and asserts from torch.profiler's records that all eight k_tile_hist instantiations ran."""
    if not os.environ.get(PROFILE_CHILD):
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
            "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider", "-k", "test_k1_every_histogram_instantiation_runs"]
        r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **{PROFILE_CHILD: "1"}), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]
        return
    import torch
    from torch.profiler import ProfilerActivity, profile

    want = {(fast, hist_nf(N)) for fast in (True, False) for N in (4, 8, 16, 17)}
    assert len(want) == 8
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for N in (4, 8, 16, 17):
            for key in ("fast", "nullable"):
                arrays, key_cols = k1_table(np.random.Generator(np.random.PCG64(N)), key, 2 * T + 5)
                run_partition(ctx, arrays, key_cols, N)
        torch.cuda.synchronize()
    ran = k1_instances(e.name for e in prof.events())
    assert want <= ran, f"not launched: {sorted(want - ran)}; launched: {sorted(ran)}"


# ---------------------------------------------------------------------------------------- 2. skewed tiles ----

SKEW_N = 3 * T + 1  # three full tiles and a last tile of one row


def skew_dests(kind, N, n, rng):
    if kind == "all_first":
        return np.zeros(n, dtype=np.int64)
    if kind == "all_last":
        return np.full(n, N - 1, dtype=np.int64)
    if kind == "row_mod_n":
        return np.arange(n, dtype=np.int64) % N
    if kind == "first_and_last":
        return np.where(rng.random(n) < 0.5, 0, N - 1).astype(np.int64)
    assert kind == "distinct_per_tile"
    return np.concatenate([rng.permutation(N)[:min(T, n - t)] for t in range(0, n, T)]).astype(np.int64)


SKEWS = [("all_first", 16), ("all_first", 4096), ("all_last", 16), ("all_last", 4096), ("distinct_per_tile", 4096),
         ("row_mod_n", 16), ("row_mod_n", 257), ("row_mod_n", 4096), ("first_and_last", 16), ("first_and_last", 4096)]


@pytest.mark.parametrize("generic", [pytest.param(False, id="fast_key"), pytest.param(True, id="generic_key")])
@pytest.mark.parametrize("kind,N", SKEWS, ids=[f"{k}-N{N}" for k, N in SKEWS])
def test_skewed_tiles(ctx, kind, N, generic):
    rng = np.random.Generator(np.random.PCG64(N))
    dests = skew_dests(kind, N, SKEW_N, rng)
    key = keys_for_dests(dests, N, seed=N + len(kind), generic=generic)
    tiles = [dests[t:t + T] for t in range(0, SKEW_N, T)]
    assert len(tiles) == 4 and len(tiles[-1]) == 1  # (a single row in the ragged last tile)
    if kind == "distinct_per_tile":
        assert T < N and all(len(np.unique(d)) == len(d) for d in tiles)  # T destinations per full tile, one row each
    if kind == "row_mod_n":
        assert all(len(np.unique(d)) == min(N, len(d)) for d in tiles)
    if kind in ("all_first", "all_last", "first_and_last"):
        assert set(np.unique(dests)) <= {0, N - 1} and (kind != "first_and_last" or all(len(np.unique(d)) == 2 for d in tiles[:-1]))
    arrays = [key, column(rng, "i64", SKEW_N), column(rng, "dec128", SKEW_N), column(rng, "u8", SKEW_N, nulls=True)]
    dest, _ = run_partition(ctx, arrays, [0], N)
    assert np.array_equal(dest, dests), "the key construction missed its destinations"


# ------------------------------------------------------------------------------------------------- 3. K1b ----

K1B_TILES = [1, 32, 33, 1024, 1025, 2048, 2049]


@pytest.mark.parametrize("N", [8, 4095], ids=lambda N: f"N{N}")
@pytest.mark.parametrize("n_tiles", K1B_TILES)
def test_k1b_tile_split(ctx, n_tiles, N):
    """Tile counts around the points where a warp's share of tiles grows (per = 32 / 64 / 96 at 1024 | 1025, 2048 | 2049)."""
    n = (n_tiles - 1) * T + T // 2 + 3
    assert n_tiles_of(n) == n_tiles
    per = scan_per(n_tiles)
    assert per == {1: 32, 32: 32, 33: 32, 1024: 32, 1025: 64, 2048: 64, 2049: 96}[n_tiles]
    assert (n_tiles - 1) // per < W_SCAN  # every tile is some warp's
    rng = np.random.Generator(np.random.PCG64(n_tiles + N))
    generic = n_tiles % 2 == 1
    key = column(rng, "i64", n, offset=1 if generic else 0)
    run_partition(ctx, [key, column(rng, "i32", n)], [0], N)


@pytest.mark.parametrize("N", [1023, 1024, 1025, 3001, 4095, 4096], ids=lambda N: f"N{N}")
def test_k1b_part_starts_rounds(ctx, N):
    """The last CTA of k_scan_tiles scans the N totals in rounds of 1024: one full round, or several with a ragged last."""
    rounds, last = -(-N // SCAN_THREADS), N % SCAN_THREADS
    assert (rounds, last) == {1023: (1, 1023), 1024: (1, 0), 1025: (2, 1), 3001: (3, 953), 4095: (4, 1023), 4096: (4, 0)}[N]
    n = 24 * N + 11
    rng = np.random.Generator(np.random.PCG64(N))
    _, starts = run_partition(ctx, [column(rng, "i64", n), column(rng, "i16", n)], [0], N)
    assert (np.diff(starts) > 0).sum() > 0.99 * N  # (part_starts is checked at almost every destination's own start)


# ------------------------------------------------------------------------------------------ 4. scratch reuse ----

def test_scratch_reuse_across_n_and_partitioners():
    """On one context of its own: N = 4096, 8, 4096, 1025 with the row count growing and shrinking (the K1 histogram and
    the `done` counter of K1b stay in the context's scratch), then two partitioners interleaved."""
    ctx = dfd.WorkerContext(0)
    try:
        rng = np.random.Generator(np.random.PCG64(99))
        for i, (N, n, generic) in enumerate([(4096, 50_000, False), (8, 3 * T + 1, True), (4096, 400_001, True), (1025, 1000, False),
                                             (8, 600_000, False), (4096, 7, True)]):
            key = column(rng, "i64", n, offset=2 if generic else 0)
            run_partition(ctx, [key, column(rng, "dec128", n), column(rng, "bool", n, nulls=True)], [0], N)
        a = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 4096))
        b = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
        for i, (part, N, n) in enumerate([(a, 4096, 120_000), (b, 8, 5 * T), (a, 4096, 33), (b, 8, 800_000), (a, 4096, 300_000),
                                          (b, 8, 1)]):
            key = column(rng, "i64", n, offset=i % 2)
            run_partition(ctx, [key, column(rng, "i64", n), column(rng, "utf8", n)], [0], N, part=part)
    finally:
        ctx.close()


# --------------------------------------------------------------------------------- 5. follow-up launches ----

WIDE_KINDS = ["i64"] * (MAX_COLS_PER_LAUNCH + 3) + ["i32", "dec128", "i16", "u8"]


@pytest.mark.parametrize("N", [257, 4095, 4096], ids=lambda N: f"N{N}")
def test_generic_key_every_launch_kind(ctx, N):
    """A sliced nullable Int64 key (the generic path: K1 caches the 2-byte destination of every row) and, sliced too,
    27 Int64 columns (two 8-byte launches), one each of 4, 16, 2 and 1 bytes, a nullable Boolean (bit launches), Utf8 and
    LargeUtf8 (K4 through the scattered iota) and a FixedSizeList<Float32, 24> (k_gather_rows)."""
    n = 4 * T + 333
    assert n_tiles_of(n) == 5 and n % T != 0
    assert sum(k == "i64" for k in WIDE_KINDS) + 1 > MAX_COLS_PER_LAUNCH
    rng = np.random.Generator(np.random.PCG64(N))
    arrays = [column(rng, "i64", n, offset=5, nulls=True)] + [column(rng, k, n, offset=3 + j % 4, nulls=j % 3 == 0)
                                                              for j, k in enumerate(WIDE_KINDS)]
    arrays += [column(rng, "bool", n, offset=9, nulls=True), column(rng, "utf8", n, offset=11, nulls=True),
               column(rng, "large_utf8", n, offset=1), column(rng, "fsl24", n, offset=6, nulls=True)]
    assert all(a.offset != 0 for a in arrays)
    run_partition(ctx, arrays, [0], N)


# --------------------------------------------------------------------------------------- 6. fused exchange ----

def fused_shuffle_check(ctx, ex, arrays, N):
    """One world-1 EXCHANGE_FUSED shuffle on `ex`: starts, and every column in the oracle's stable order."""
    n = len(arrays[0])
    order, ref_starts = expected_partitions(orc.partition_ids([arrays[0]], n, N), N)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], N), uuid.uuid4(), 1, 1, 1)
    outs, starts = node.shuffle(ex, [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays], n, nv.EXCHANGE_FUSED)
    assert np.array_equal(np.diff(starts), np.diff(ref_starts)), f"counts differ at N={N}"
    for c, arr in enumerate(arrays):
        got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, outs[c], int(starts[0]), n)
        assert got.equals(arr.take(pa.array(order))), (N, c, arr.type)


@pytest.mark.parametrize("N", [3996, 3997, 4095, 4096], ids=lambda N: f"N{N}")
def test_fused_exchange_16_byte_columns_at_large_n(ctx, N):
    """Int64 key, Decimal128 and Interval(MonthDayNano): the two-pass peer scatter of 16-byte values at N up to 4096, then an
    ordinary shuffle on the same exchange."""
    n = 3 * T + 1
    rng = np.random.Generator(np.random.PCG64(N))
    arrays = [column(rng, "i64", n), column(rng, "dec128", n), column(rng, "mdn", n)]
    assert [dfd.DeviceColumn.from_arrow(ctx, a).width for a in arrays] == [8, 16, 16]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    try:
        ex.setup_window(64 << 20)
        fused_shuffle_check(ctx, ex, arrays, N)
        small = [column(rng, "i64", 5000), column(rng, "dec128", 5000), column(rng, "mdn", 5000)]
        fused_shuffle_check(ctx, ex, small, 8)
    finally:
        ex.close()
