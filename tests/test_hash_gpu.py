"""GPU parity tests of the row hash every partition kernel inlines (dfd_hash.cuh: AHasher, row_hash, mod_n), bit-exact
against the C oracle's 64-bit `create_hashes` under DataFusion's default seeds and under other ahash seeds.

1. `k_row_hashes` (`dfd_hash_columns_device`) == oracle, as uint64: fixed widths 1 / 2 / 4 / 8 / 16 over full-range
   values (±0.0, ±inf and NaN payloads; 16-byte keys with both halves swapped), Booleans at Arrow offsets 0-7, 13 and 37,
   Utf8 / Binary / LargeUtf8 of every length 0-48 and around 64, 128 and 256 bytes at every start address mod 8, 2 to 8
   keys of mixed kinds, sliced, all 8 null patterns of 3 keys, and 0, 1, 255, 256, 257 and one grid pass + 1 rows.
2. Every hashing kernel sends a row to checked_hash % N: `k_partition_ids`, the two-pass partition (K1 with every
   histogram variant, K2), the single-pass partition and the world-1 exchange (single-pass, fused two-pass, push), under
   the fast Int64 key and generic keys, at N = 3 ... 4096 (mask and Barrett paths), with counts and row order equal to the
   oracle's; a child process asserts from torch.profiler that the seeded calls ran the FAST and the generic
   instantiations of k_tile_hist, k_scatter and k_scatter_onepass, local and peer.  `mod_n` at every N from 1 to 4096,
   and interval keys hashed field by field, seeded.
3. A dictionary key hashes its values with the partitioner's seeds.

One H100 80GB HBM3 at 700 W: the module's 146 cases take about 55 s, 25 s of it in the child process, with at most
about 1.1 GiB of device memory in use."""
import ctypes as C
import os
import subprocess
import sys
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from datafusion_distributed_b200.device import columns_to_c
from oracle import oracle as orc
from tests.test_twopass_gpu import k1_instances
from tests.util import expected_partitions, scatter_inst, scatter_instances, seed_tuples, tile_geometry, use_aligned

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILE_CHILD = "DFD_TEST_HASH_PROFILE"  # set in the child process that records the kernel instantiations
GUARD = 0xA5A5A5A5A5A5A5A5  # fill of the hash output past the last row
TAIL = 8

SEEDS = seed_tuples()
SEED_IDS = ["default", "golden_1_2_3_4", "golden_74_79_73_78", "k0", "k1", "k2", "k3", "distinct"]
assert len(SEED_IDS) == len(SEEDS) and SEEDS[0] == (0, 0, 0, 0)
DEFAULT, SEEDED = SEEDS[0], SEEDS[-1]
BOTH = [pytest.param(DEFAULT, id="default"), pytest.param(SEEDED, id="seeded")]
ALL = [pytest.param(s, id=i) for s, i in zip(SEEDS, SEED_IDS)]

# ------------------------------------------------------------------------------------------------- columns ----


def fixed(typ, n, raw, valid=None):
    """A fixed-width (or Boolean) Arrow array over the raw little-endian bytes `raw`, bit patterns kept as they are."""
    vb = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()) if valid is not None else None
    nulls = int(n - np.count_nonzero(valid[:n])) if valid is not None else 0
    return pa.Array.from_buffers(typ, n, [vb, pa.py_buffer(np.ascontiguousarray(raw).tobytes())], null_count=nulls)


def distinct_bytes(rng, n):
    """n random bytes, none repeated within a block of 256: a read of the wrong bytes inside a value shows."""
    return np.concatenate([rng.permutation(256) for _ in range(n // 256 + 1)])[:n].astype(np.uint8)


def var_array(typ, values):
    """A Utf8 / Binary / LargeUtf8 array of byte strings (None = null); Utf8 is not validated, so random bytes hash as
    they are."""
    lens = np.array([0 if v is None else len(v) for v in values], dtype=np.int64)
    odt = np.int64 if typ == pa.large_string() else np.int32
    off = np.concatenate([[0], np.cumsum(lens)]).astype(odt)
    valid = np.array([v is not None for v in values])
    data = b"".join(v for v in values if v is not None)
    vb = None if valid.all() else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    return pa.Array.from_buffers(typ, len(values), [vb, pa.py_buffer(off.tobytes()), pa.py_buffer(data)],
                                 null_count=int((~valid).sum()))


FIXED_TYPES = {"u8": pa.uint8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "f64": pa.float64(),
               "dec128": pa.decimal128(38, 0)}
VAR_TYPES = {"utf8": pa.string(), "binary": pa.binary(), "large_utf8": pa.large_string()}


def column(rng, kind, m, valid=None):
    """A seeded column of `kind` and m rows, null where `valid` is False."""
    if kind == "bool":
        return fixed(pa.bool_(), m, rng.integers(0, 256, (m + 7) // 8, dtype=np.uint8), valid)
    if kind in FIXED_TYPES:
        typ = FIXED_TYPES[kind]
        return fixed(typ, m, rng.integers(0, 256, m * (typ.bit_width // 8), dtype=np.uint8), valid)
    typ = VAR_TYPES[kind]
    lens = rng.integers(0, 40, m)
    odt = np.int64 if kind == "large_utf8" else np.int32
    off = np.concatenate([[0], np.cumsum(lens)]).astype(odt)
    vb = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()) if valid is not None else None
    nulls = int(m - np.count_nonzero(valid)) if valid is not None else 0
    return pa.Array.from_buffers(typ, m, [vb, pa.py_buffer(off.tobytes()), pa.py_buffer(distinct_bytes(rng, int(off[-1])).tobytes())],
                                 null_count=nulls)


def dev_cols(ctx, arrays):
    return [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]


# ------------------------------------------------------------------------------------------- 1. row hashes ----

def device_hashes(ctx, arrays, n, seeds):
    """dfd_hash_columns_device over `arrays` (the default seeds as a NULL pointer, as the partitioner passes them) into
    an output whose words past row n must keep GUARD."""
    out = ctx.upload(np.full(n + TAIL, GUARD, dtype=np.uint64))
    seeds_arr = None if seeds == DEFAULT else (C.c_uint64 * 4)(*seeds)
    cols = dev_cols(ctx, arrays)
    nv.check(nv.lib().dfd_hash_columns_device(ctx.handle, columns_to_c(cols), len(cols), n, seeds_arr, out.ptr))
    got = out.download(np.uint64)
    assert (got[n:] == GUARD).all(), "k_row_hashes wrote past the last row"
    return got[:n]


def checked_hashes(ctx, arrays, seeds, n=None):
    """The device's 64-bit row hashes of `arrays`, asserted equal to the oracle's create_hashes bit for bit."""
    n = len(arrays[0]) if n is None else n
    want = orc.create_hashes(arrays, n, seeds)
    got = device_hashes(ctx, arrays, n, seeds)
    bad = np.nonzero(got != want)[0]
    assert not len(bad), (f"{len(bad)} of {n} hashes differ ({[str(a.type) for a in arrays]}, seeds {seeds}); first rows "
                          f"{bad[:4].tolist()}: got {[hex(int(x)) for x in got[bad[:4]]]}, want {[hex(int(x)) for x in want[bad[:4]]]}")
    return got


INT_TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64()]
FLOAT_SPECIALS = {  # +0, -0, +inf, -inf, quiet NaN, NaN with payload 1, negative NaN, signalling NaN, all-ones NaN
    pa.float16(): (np.uint16, [0x0000, 0x8000, 0x7C00, 0xFC00, 0x7E00, 0x7E01, 0xFE00, 0x7C01, 0x7FFF]),
    pa.float32(): (np.uint32, [0x0, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001, 0x7FFFFFFF]),
    pa.float64(): (np.uint64, [0x0, 1 << 63, 0x7FF0 << 48, 0xFFF0 << 48, 0x7FF8 << 48, (0x7FF8 << 48) | 1, 0xFFF8 << 48,
                               (0x7FF0 << 48) | 1, (1 << 63) - 1]),
}


@pytest.mark.parametrize("seeds", ALL)
def test_fixed_width_hashes(ctx, seeds):
    """Integers of 1, 2, 4 and 8 bytes over their full range (0, all ones, the sign bit, random), nullable and not;
    Float16/32/64 bit patterns that compare equal or unordered but differ in bits; 16-byte keys (lo, hi) next to (hi, lo)."""
    rng = np.random.Generator(np.random.PCG64(11))
    n = 4096
    valid = rng.random(n) >= 0.2
    for typ in INT_TYPES:
        w = typ.bit_width // 8
        raw = rng.integers(0, 256, (n, w), dtype=np.uint8)
        raw[0], raw[1], raw[2], raw[3] = 0, 0xFF, 0, 0xFF
        raw[2, -1], raw[3, -1] = 0x80, 0x7F  # the sign bit alone, and the largest signed value
        checked_hashes(ctx, [fixed(typ, n, raw)], seeds)
        checked_hashes(ctx, [fixed(typ, n, raw, valid)], seeds)
    for typ, (udt, specials) in FLOAT_SPECIALS.items():
        bits = rng.integers(0, np.iinfo(udt).max, n, dtype=udt, endpoint=True)
        bits[:len(specials)] = np.array(specials, dtype=udt)
        h = checked_hashes(ctx, [fixed(typ, n, bits)], seeds)
        assert len(set(h[:len(specials)].tolist())) == len(specials), "distinct bit patterns must hash apart"
    lo = rng.integers(0, 1 << 64, n // 2, dtype=np.uint64, endpoint=False)
    hi = lo ^ rng.integers(1, 1 << 64, n // 2, dtype=np.uint64)  # hi != lo on every row
    pairs = np.stack([lo, hi, hi, lo], axis=1).reshape(n, 2)  # row 2i = (lo, hi), row 2i + 1 = (hi, lo)
    h = checked_hashes(ctx, [fixed(pa.decimal128(38, 0), n, pairs)], seeds)
    assert (h[0::2] != h[1::2]).all(), "swapped halves of a 16-byte key must hash apart"
    checked_hashes(ctx, [fixed(pa.decimal128(38, 0), n, pairs, valid)], seeds)


@pytest.mark.parametrize("seeds", ALL)
def test_boolean_hashes_at_every_bit_offset(ctx, seeds):
    rng = np.random.Generator(np.random.PCG64(12))
    n = 4096
    m = n + 40
    bits = rng.integers(0, 256, (m + 7) // 8, dtype=np.uint8)
    valid = rng.random(m) >= 0.25
    for base in (fixed(pa.bool_(), m, bits), fixed(pa.bool_(), m, bits, valid)):
        for off in list(range(8)) + [13, 37]:
            checked_hashes(ctx, [base.slice(off, n)], seeds)


STRING_LENGTHS = list(range(49)) + [63, 64, 65, 127, 128, 129, 255, 256, 257, 4099]


def strings_at_every_alignment(rng):
    """Byte strings: for each length of STRING_LENGTHS and each residue s in 0..7, a filler value whose length puts the
    next value's first byte at a buffer offset of s mod 8, then a value of that length.  Returns (values, the index and
    start offset of every value of the chosen lengths)."""
    values, targets, pos = [], [], 0
    for L in STRING_LENGTHS:
        for s in range(8):
            filler = (s - pos) % 8
            values.append(distinct_bytes(rng, filler).tobytes())
            pos += filler
            targets.append((len(values), L, pos))
            values.append(distinct_bytes(rng, L).tobytes())
            pos += L
    return values, targets


@pytest.mark.parametrize("seeds", ALL)
def test_string_hashes_every_length_and_alignment(ctx, seeds):
    """Utf8, Binary and LargeUtf8 hash the same bytes: Utf8 and LargeUtf8 alike (write + 0xff suffix), Binary apart
    (length prefix, no suffix).  The device buffers are 256-byte aligned, so a value's buffer offset mod 8 is its start
    address mod 8, where AHasher::rd's funnel shift of two aligned words begins."""
    rng = np.random.Generator(np.random.PCG64(13))
    values, targets = strings_at_every_alignment(rng)
    for L in STRING_LENGTHS:
        assert {p % 8 for _, l, p in targets if l == L} == set(range(8))
    h = {k: checked_hashes(ctx, [var_array(t, values)], seeds) for k, t in VAR_TYPES.items()}
    assert (h["utf8"] == h["large_utf8"]).all()
    assert (h["utf8"] != h["binary"]).all(), "Utf8 and Binary of the same bytes must hash apart"
    for k, t in VAR_TYPES.items():  # offsets[0] != 0: every value one filler later, the residues shifted
        checked_hashes(ctx, [var_array(t, values).slice(3)], seeds)
    side = [b"", None, b"", b"", None, None, b"\x00", b"", None, b"\xff", b"\x00\x00"] * 9  # empty and null side by side
    for k, t in VAR_TYPES.items():
        arr = var_array(t, side)
        h = checked_hashes(ctx, [arr], seeds)
        assert (h[[i for i, v in enumerate(side) if v is None]] == 0).all()
        assert len({int(h[i]) for i, v in enumerate(side) if v == b""}) == 1
        for off in (1, 2, 5):
            checked_hashes(ctx, [arr.slice(off)], seeds)


MIXED = ["i64", "utf8", "i32", "bool", "dec128", "binary", "u8", "large_utf8"]
OFFSETS = [0, 1, 2, 3, 4, 5, 6, 7, 13, 37]


@pytest.mark.parametrize("seeds", ALL)
@pytest.mark.parametrize("n_keys", range(2, 9))
def test_multi_key_hashes_sliced(ctx, n_keys, seeds):
    """2 to 8 nullable keys of mixed kinds (the first kind rotates with the key count), all sliced at the same Arrow
    offset, as columns of one record batch are."""
    rng = np.random.Generator(np.random.PCG64(100 + n_keys))
    kinds = [MIXED[(n_keys + j) % len(MIXED)] for j in range(n_keys)]
    n = 1000
    for off in OFFSETS:
        m = n + off + 3
        arrays = [column(rng, k, m, rng.random(m) >= 0.3).slice(off, n) for k in kinds]
        checked_hashes(ctx, arrays, seeds)


@pytest.mark.parametrize("seeds", ALL)
@pytest.mark.parametrize("kinds", [("i64", "utf8", "bool"), ("binary", "dec128", "i16")], ids=lambda k: "_".join(k))
def test_three_keys_every_null_pattern(ctx, kinds, seeds):
    """Row r has key j null when bit j of r % 8 is set: a null first key (the one that overwrites rather than combines),
    middle key and last key, alone and together."""
    rng = np.random.Generator(np.random.PCG64(14))
    n = 8 * 300
    arrays = [column(rng, k, n, (np.arange(n) >> j) % 2 == 0) for j, k in enumerate(kinds)]
    h = checked_hashes(ctx, arrays, seeds)
    assert (h[np.arange(n) % 8 == 7] == 0).all()  # every key null: the hash stays 0
    assert len(np.unique(h[np.arange(n) % 8 == 0])) == n // 8
    for off in (1, 5):
        checked_hashes(ctx, [a.slice(off) for a in arrays], seeds)


def grid_rows():
    """One full grid pass of k_row_hashes (the SM count x 32 blocks of 256 threads, as hash_columns_locked caps the
    grid) and one row more: the grid-stride loop takes a second trip."""
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256 + 1


ROW_COUNTS = [0, 1, 255, 256, 257, "grid+1"]


@pytest.mark.parametrize("seeds", BOTH)
@pytest.mark.parametrize("n", ROW_COUNTS, ids=str)
def test_row_counts(ctx, n, seeds):
    n = grid_rows() if n == "grid+1" else n
    rng = np.random.Generator(np.random.PCG64(15))
    m = max(n, 1)
    arrays = [column(rng, "i64", m, rng.random(m) >= 0.2), column(rng, "utf8", m), column(rng, "bool", m)]
    h = checked_hashes(ctx, [a.slice(0, n) for a in arrays], seeds, n)
    assert len(h) == n


# ------------------------------------------------------------------------------------- 2. hashing kernels ----

N_LOCAL = [3, 7, 8, 12, 17, 4093, 4096]  # K1 NF = 1 / 2 / 2 / 4 / 0 / 0 / 0; Barrett and mask paths
N_EXCHANGE = [7, 8, 17, 4093, 4096]
ROWS = 3 * max(tile_geometry()) + 77  # several tiles of both tilings, a ragged last one
WINDOW = 64 << 20


def kernel_table(rng, key, n):
    """(arrays, key columns).  fast: one non-null Int64 key at offset 0 (the FAST instantiations); generic: a sliced
    Int64 key and an Int32 key, non-null (generic instantiations; every single-pass route takes it); nullable: a sliced
    nullable Int64 key and a Utf8 key, with a Boolean payload (two-pass and bit launches, the push transport)."""
    def sliced(kind, valid=None):
        return column(rng, kind, n + 5, valid).slice(5)

    if key == "fast":
        keys = [column(rng, "i64", n)]
    elif key == "generic":
        keys = [sliced("i64"), sliced("i32")]
    else:
        keys = [sliced("i64", rng.random(n + 5) >= 0.2), sliced("utf8", rng.random(n + 5) >= 0.1)]
    payload = [column(rng, "i32", n), column(rng, "dec128", n)] + ([column(rng, "bool", n, rng.random(n) >= 0.3)] if key == "nullable" else [])
    return keys + payload, list(range(len(keys)))


def checked_dest(ctx, arrays, key_cols, N, seeds):
    """checked_hashes(key columns) % N."""
    return (checked_hashes(ctx, [arrays[k] for k in key_cols], seeds) % np.uint64(N)).astype(np.int64)


def assert_rows(got_cols, arrays, src_of_out, what):
    """Output row j of every column equals input row src_of_out[j]."""
    idx = pa.array(src_of_out)
    for c, (got, arr) in enumerate(zip(got_cols, arrays)):
        assert got.equals(arr.take(idx)), (what, c, str(arr.type))


def check_local(ctx, arrays, key_cols, N, seeds):
    """partition_ids, partition (two-pass) and partition_onepass of a seeded partitioner against checked hashes % N."""
    n = len(arrays[0])
    dest = checked_dest(ctx, arrays, key_cols, N, seeds)
    order, starts = expected_partitions(dest, N)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash(key_cols, N), seeds)
    dcols = dev_cols(ctx, arrays)
    assert np.array_equal(part.partition_ids(dcols, n), dest), ("partition_ids", N)
    outs, got_starts = part.partition(dcols, n)
    assert np.array_equal(got_starts, starts), ("partition starts", N)
    assert_rows([o.to_arrow(ctx, 0, n) for o in outs], arrays, order, ("partition", N))
    outs, st, cn = part.partition_onepass(dcols, n)
    assert np.array_equal(cn, np.diff(starts)), ("partition_onepass counts", N)
    pos = np.repeat(st, cn) + np.arange(n) - np.repeat(starts[:-1], cn)  # output row of the j-th row in oracle order
    for c, (o, arr) in enumerate(zip(outs, arrays)):
        got = o.to_arrow(ctx, 0, int((st + cn).max()) if n else 0).take(pa.array(pos))
        assert got.equals(arr.take(pa.array(order))), ("partition_onepass", N, c, str(arr.type))


@pytest.mark.parametrize("seeds", BOTH)
@pytest.mark.parametrize("N", N_LOCAL, ids=lambda N: f"N{N}")
def test_local_partition_follows_row_hashes(ctx, N, seeds):
    rng = np.random.Generator(np.random.PCG64(N))
    for key in ("fast", "generic", "nullable"):
        arrays, key_cols = kernel_table(rng, key, ROWS)
        check_local(ctx, arrays, key_cols, N, seeds)


def check_exchange(ctx, arrays, key_cols, N, seeds, route):
    """A world-1 exchange through a seeded partitioner: "onepass" (single-pass peer kernel), "push" (shuffle_onepass of
    nullable / string columns: the push transport) or "fused" (EXCHANGE_FUSED).  Partition q holds the rows with
    checked hash % N == q, in input order."""
    n = len(arrays[0])
    dest = checked_dest(ctx, arrays, key_cols, N, seeds)
    order, starts = expected_partitions(dest, N)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    try:
        ex.setup_window(WINDOW)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash(key_cols, N), uuid.uuid4(), 1, 1, 1)
        node._part = dfd.HashPartitioner(ctx, node.input_stage_plan(), seeds)  # the producers' partitioner, seeded
        in_cols = dev_cols(ctx, arrays)  # (alive until collect())
        if route == "fused":
            outs, st = node.shuffle(ex, in_cols, n, nv.EXCHANGE_FUSED)
            seg_starts, seg_counts = st[:-1], np.diff(st)
        else:
            node.shuffle_onepass(ex, in_cols, n)
            outs, seg_starts, seg_counts = node.collect(ex)
            seg_starts, seg_counts = seg_starts[:, 0], seg_counts[:, 0]
        assert np.array_equal(seg_counts, np.diff(starts)), (route, N, "counts")
        pos = np.repeat(seg_starts, seg_counts) + np.arange(n) - np.repeat(starts[:-1], seg_counts)
        end = int((seg_starts + seg_counts).max())
        for c, (o, arr) in enumerate(zip(outs, arrays)):
            got = dfd.NetworkShuffleExec.segment_to_arrow(ctx, o, 0, end).take(pa.array(pos))
            assert got.equals(arr.take(pa.array(order))), (route, N, c, str(arr.type))
    finally:
        ex.close()


@pytest.mark.parametrize("seeds", BOTH)
@pytest.mark.parametrize("N", N_EXCHANGE, ids=lambda N: f"N{N}")
def test_exchange_follows_row_hashes(ctx, N, seeds):
    rng = np.random.Generator(np.random.PCG64(N + 1))
    # above 256 destinations shuffle_onepass takes the push transport, which refuses N x (1 + string columns) > 2048 slice
    # entries (XCHG_META_MAX): at N = 4093 and 4096 only the fused exchange runs
    small = N <= 256
    for key, routes in (("fast", ("onepass", "fused") if small else ("fused",)), ("generic", ("onepass", "fused") if small else ("fused",)),
                        ("nullable", ("push",) if small else ())):
        arrays, key_cols = kernel_table(rng, key, ROWS)
        for route in routes:
            check_exchange(ctx, arrays, key_cols, N, seeds, route)


def test_seeded_calls_ran_fast_and_generic_instantiations(ctx):
    """A child process (a profiler session of its own: kernel records of a long-running test process can stop) runs the
    seeded local and exchange checks at N = 8 with the fast and the generic key, and asserts from torch.profiler's
    records that both the FAST and the generic instantiation ran of k_tile_hist, of k_scatter (local and peer) and of
    k_scatter_onepass (local and peer)."""
    if not os.environ.get(PROFILE_CHILD):
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
            "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider", "-k", "test_seeded_calls_ran_fast_and_generic_instantiations"]
        r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **{PROFILE_CHILD: "1"}), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]
        return
    import torch
    from torch.profiler import ProfilerActivity, profile

    N = 8
    rng = np.random.Generator(np.random.PCG64(21))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for key in ("fast", "generic"):
            arrays, key_cols = kernel_table(rng, key, ROWS)
            check_local(ctx, arrays, key_cols, N, SEEDED)
            for route in ("onepass", "fused"):
                check_exchange(ctx, arrays, key_cols, N, SEEDED, route)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    hist = k1_instances(names)
    assert {(True, 2), (False, 2)} <= hist, f"k_tile_hist launched: {sorted(hist)}"
    want = {scatter_inst(mode, fast, "u64", peer, use_aligned(N, peer)) for fast in (True, False) for mode in (0, 1) for peer in (False, True)}
    ran = scatter_instances(names)
    assert want <= ran, f"not launched: {sorted(want - ran)}; launched: {sorted(ran)}"


def test_mod_n_every_partition_count(ctx):
    """k_partition_ids at every N from 1 to 4096 over 2^16 checked hashes: powers of two take the mask, the others one
    Barrett step, whose quotient falls one short (and needs the correction) for at least about 1 in N rows."""
    rng = np.random.Generator(np.random.PCG64(22))
    n = 1 << 16
    key = pa.array(rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True))
    h = checked_hashes(ctx, [key], SEEDED)
    dcols = dev_cols(ctx, [key])
    for N in range(1, 4097):
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N), SEEDED)
        got = part.partition_ids(dcols, n)
        part.close()
        want = (h % np.uint64(N)).astype(np.uint32)
        if not np.array_equal(got, want):
            bad = np.nonzero(got != want)[0]
            raise AssertionError(f"N={N}: {len(bad)} rows differ, first {bad[:4].tolist()}: got {got[bad[:4]].tolist()}, want {want[bad[:4]].tolist()}")


@pytest.mark.parametrize("seeds", ALL)
def test_interval_keys_seeded(ctx, seeds):
    """Interval(MonthDayNano) (nullable) and Interval(DayTime) keys, hashed field by field, with an Int64 key after them:
    partition_ids and the two-pass partition against the oracle's seeded create_hashes."""
    rng = np.random.Generator(np.random.PCG64(23))
    n = 20_000
    raw_dt = rng.integers(0, 256, n * 8, dtype=np.uint8)
    raw_mdn = rng.integers(0, 256, n * 16, dtype=np.uint8)
    valid = rng.random(n) >= 0.2
    other = column(rng, "i64", n)
    arrays = [fixed(pa.decimal128(38, 0), n, raw_mdn, valid), fixed(pa.int64(), n, raw_dt), other]
    h = orc.create_hashes([("interval_month_day_nano", raw_mdn, valid), ("interval_day_time", raw_dt), other], n, seeds)
    dcols = dev_cols(ctx, arrays)
    for N in (7, 4096):
        dest = (h % np.uint64(N)).astype(np.int64)
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1, 2], N), seeds)
        part.set_key_hash_mode(0, nv.KEY_HASH_INTERVAL_MONTH_DAY_NANO)
        part.set_key_hash_mode(1, nv.KEY_HASH_INTERVAL_DAY_TIME)
        assert np.array_equal(part.partition_ids(dcols, n), dest), N
        order, starts = expected_partitions(dest, N)
        outs, got_starts = part.partition(dcols, n)
        assert np.array_equal(got_starts, starts), N
        assert_rows([o.to_arrow(ctx, 0, n) for o in outs], arrays, order, ("interval partition", N))


# ------------------------------------------------------------------------------------ 3. dictionary keys ----

def combine(l, r):
    """datafusion-common combine_hashes over uint64 arrays (wrapping)."""
    return (np.uint64(17 * 37) + l) * np.uint64(37) + r


@pytest.mark.parametrize("index_type", [pa.int8(), pa.uint8(), pa.int32(), pa.uint64()], ids=str)
def test_dictionary_key_hashes_with_partitioner_seeds(ctx, index_type):
    """A seeded partitioner with a Dictionary<index_type, Utf8> key between an Int64 and a Utf8 key: a row takes the
    seeded hash of its dictionary value, combined like a plain key; a null index or a null value leaves the hash as it
    was.  UInt8 indices reach 249, past the sign bit of a byte."""
    rng = np.random.Generator(np.random.PCG64(24))
    n = 20_000
    n_values = 100 if index_type == pa.int8() else 250
    values = var_array(pa.string(), [None if i == 5 else distinct_bytes(rng, int(rng.integers(0, 30))).tobytes() for i in range(n_values)])
    idx = rng.integers(0, n_values, n)
    idx_valid = rng.random(n) >= 0.1
    indices = pa.array(idx.astype(index_type.to_pandas_dtype()), type=index_type, mask=~idx_valid)
    if index_type == pa.uint8():
        assert (idx[idx_valid] >= 128).sum() > n // 3
    first, last = column(rng, "i64", n, rng.random(n) >= 0.1), column(rng, "utf8", n, rng.random(n) >= 0.1)
    dict_h = orc.create_hashes([values], n_values, SEEDED)
    h = orc.create_hashes([first], n, SEEDED)
    take = idx_valid & values.is_valid().to_numpy(zero_copy_only=False)[idx]
    h[take] = combine(dict_h[idx[take]], h[take])
    h_last, last_valid = orc.create_hashes([last], n, SEEDED), last.is_valid().to_numpy(zero_copy_only=False)
    h[last_valid] = combine(h_last[last_valid], h[last_valid])
    assert np.array_equal(h, orc.create_hashes([first, pa.DictionaryArray.from_arrays(indices, values), last], n, SEEDED))
    dcols = dev_cols(ctx, [first, indices, last])
    for N in (7, 4096):
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1, 2], N), SEEDED)
        part.set_key_dictionary(1, values, unsigned_index=index_type in (pa.uint8(), pa.uint64()))
        got = part.partition_ids(dcols, n)
        assert np.array_equal(got, (h % np.uint64(N)).astype(np.uint32)), (N, int((got != h % np.uint64(N)).sum()))
