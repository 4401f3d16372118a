"""GPU parity tests of the device PartialReduce with nullable group keys and nullable aggregate states, bit for bit against
the null-aware exact reference of test_reduce_nulls_cpu.py (which is itself checked against pyarrow's group_by).

Every call checks, for every output column:
- the values of every group, zero bytes under a null key or state, and the validity bit of every output row;
- the guard bytes in front of and behind the values and the output bitmap, the bitmap words past ceil(G / 32) (they
  keep their fill) and the bits at and past G in the last word (zero);
- the kernel launch count (4, or 5 when a MIN / MAX state column has an input bitmap);
- a second run on the same input gives the same bytes and bits for every group.
The bytes under null keys and states hold garbage (NaNs, the op's sentinel, INT_MIN, all ones, random bits) that must
never reach a result.  Input bitmaps sit at odd byte addresses with junk bits in front of the Arrow offset."""
import uuid
from decimal import Decimal

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from tests.test_reduce_limits_gpu import grid_threads
from tests.test_reduce_nulls_cpu import ALL_OPS, MINMAX_OPS, key_matrix, reference_reduce, sentinel
from tests.test_reduce_ops_gpu import OP_TYPE, random_values

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED = 1, 6
FILL, GUARD = 0xA5, 64


def width(col):
    return 16 if col.ndim == 2 else col.dtype.itemsize


# ------------------------------------------------------------------ inputs ----

def state_values(op, n, rng):
    """n random values of op's state column (exact float sums: SUM_F64 values are small integers)."""
    if op in OP_TYPE:
        return random_values(OP_TYPE[op], n, rng)
    if op == nv.AGG_SUM_F64:
        return rng.integers(-1000, 1000, n).astype(np.float64)
    if op == nv.AGG_SUM_I128:
        return rng.integers(-(1 << 63), (1 << 63) - 1, (n, 2), dtype=np.int64, endpoint=True)
    if op in (nv.AGG_MIN_F64, nv.AGG_MAX_F64):
        bits = rng.standard_normal(n).view(np.uint64).copy()
        special = np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000000, 0xFFF0000000000000, 0, 1 << 63,
                            0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF], dtype=np.uint64)
        pick = rng.random(n) < 0.05
        bits[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
        return bits
    v = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)  # SUM_I64, MIN / MAX_I64
    pick = rng.random(n) < 0.05
    v[pick] = np.array([-(1 << 63), (1 << 63) - 1, 0, -1], dtype=np.int64)[rng.integers(0, 4, int(pick.sum()))]
    return v


def garbage_like(col, op, rng):
    """Bytes for the rows under nulls: all ones, 0x7f.., 0x80.., zero, the op's sentinel, a NaN, or random bits."""
    n, w = len(col), width(col)
    raw = rng.integers(0, 256, (n, w), dtype=np.uint8)
    pats = [np.full(w, 0xFF, np.uint8), np.r_[np.full(w - 1, 0xFF, np.uint8), 0x7F].astype(np.uint8),
            np.r_[np.zeros(w - 1, np.uint8), 0x80].astype(np.uint8), np.zeros(w, np.uint8),
            np.r_[np.zeros(max(w - 2, 0), np.uint8), np.array([0xF8, 0x7F], np.uint8)][-w:] if w >= 2 else np.array([0x7F], np.uint8)]
    if op is not None and op in MINMAX_OPS:
        pats.append(np.ascontiguousarray(sentinel(op)).view(np.uint8).reshape(-1)[:w])
    which = rng.integers(0, len(pats) + 2, n)  # the last two choices keep the random bits
    for i, p in enumerate(pats):
        raw[which == i] = p
    out = raw.view(np.int64 if col.ndim == 2 else col.dtype)
    return out.reshape(n, 2) if col.ndim == 2 else out.reshape(n)


def with_nulls(col, valid, op, rng):
    """col with garbage under every null of `valid` (None: no bitmap)."""
    if valid is None:
        return col
    col = col.copy()
    col[~valid] = garbage_like(col, op, rng)[~valid]
    return col


# ------------------------------------------------------------- device i/o ----

def upload(col, valid, off, rng):
    """A device column holding `col` at Arrow offset `off` behind `off` rows of junk; its bitmap (if any) at an odd byte
    address, with `off` junk bits in front of row 0's bit."""
    w = width(col)
    buf = np.concatenate([rng.integers(0, 256, off * w, dtype=np.uint8), np.ascontiguousarray(col).view(np.uint8).reshape(-1)])
    if buf.size == 0:
        buf = np.zeros(w, dtype=np.uint8)
    t = torch.from_numpy(buf).cuda()
    keep, vptr = [t], 0
    if valid is not None:
        bits = rng.integers(0, 2, off + len(valid) + 8).astype(bool)
        bits[off:off + len(valid)] = valid
        vb = np.concatenate([[0x5A], np.packbits(bits, bitorder="little"), [0x5A] * 8]).astype(np.uint8)
        vt = torch.from_numpy(vb).cuda()
        vptr = vt.data_ptr() + 1
        keep.append(vt)
    return dfd.DeviceColumn(nv.COL_FIXED, w, t.data_ptr(), 0, vptr, off, len(col), keep)


def guarded_output(w, capacity, nullable, bitmap_shift=0, value_shift=0):
    """Output values of `capacity` rows (from `value_shift` bytes past a 64-byte-aligned address) and, when nullable, a
    bitmap of ceil(capacity / 32) words, both inside FILL bytes with GUARD bytes in front and behind.  -> (DeviceColumn,
    values tensor, bitmap tensor or None)"""
    t = torch.full((GUARD + value_shift + capacity * w + GUARD,), FILL, dtype=torch.uint8, device="cuda")
    vt, vptr = None, 0
    if nullable:
        words = (capacity + 31) // 32
        vt = torch.full((GUARD + words * 4 + GUARD,), FILL, dtype=torch.uint8, device="cuda")
        vptr = vt.data_ptr() + GUARD + bitmap_shift
    col = dfd.DeviceColumn(nv.COL_FIXED, w, t.data_ptr() + GUARD + value_shift, 0, vptr, 0, capacity, [t] + ([vt] if vt is not None else []))
    return col, t, vt


def read_output(t, vt, w, G, name, value_shift=0):
    """Rows [0, G) of a guarded_output: (their bytes as a (G, w) uint8 array, their bits or None), after checking that
    every byte outside them keeps its fill and that the bits at and past G in the last bitmap word are zero."""
    raw = t.cpu().numpy()
    start = GUARD + value_shift
    assert bool((raw[:start] == FILL).all()) and bool((raw[start + G * w:] == FILL).all()), f"{name}: bytes outside rows [0, {G}) written"
    vals = raw[start:start + G * w].reshape(G, w)
    if vt is None:
        return vals, None
    rb = vt.cpu().numpy()
    words = (G + 31) // 32
    assert bool((rb[:GUARD] == FILL).all()), f"{name}: a byte in front of the output bitmap was written"
    assert bool((rb[GUARD + words * 4:] == FILL).all()), f"{name}: a bitmap word past row {G} was written"
    b = np.unpackbits(rb[GUARD:GUARD + words * 4], bitorder="little").astype(bool)
    assert not b[G:].any(), f"{name}: bits at or past G = {G} are set"
    return vals, b[:G]


def expected_launches(valids, ops, n):
    if n == 0:
        return 0
    return 5 if any(v is not None and op in MINMAX_OPS for v, op in zip(valids, ops)) else 4


def run_once(ctx, cols, valids, n_keys, ops, starts_d, N, offsets, out_nullable, seed):
    """One reduce of rows already laid out partition by partition.  -> (values [G rows] per column, validity [G] per
    column (None for a non-null output), out_part_starts)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n = len(cols[0])
    dcols = [upload(c, v, off, rng) for c, v, off in zip(cols, valids, offsets)]
    outs = [guarded_output(width(c), n, nb) for c, nb in zip(cols, out_nullable)]
    torch.cuda.synchronize()
    before = ctx.metrics()["kernel_launches"]
    _, out_starts = dfd.PartialReduceExec(ctx, list(range(n_keys)), [-1] * n_keys + ops).reduce(
        dcols, n, starts_d.data_ptr(), N, [o[0] for o in outs])
    assert ctx.metrics()["kernel_launches"] - before == expected_launches(valids[n_keys:], ops, n)
    G = int(out_starts[-1])
    vals, bits = [], []
    for i, (c, (_, t, vt)) in enumerate(zip(cols, outs)):
        v, b = read_output(t, vt, width(c), G, f"column {i}")
        v = v.reshape(-1).view(np.int64 if c.ndim == 2 else c.dtype)
        vals.append(v.reshape(G, 2) if c.ndim == 2 else v)
        bits.append(b)
    return vals, bits, out_starts


def reduce_checked(ctx, keys, key_valid, states, state_valid, ops, part=None, N=1, offsets=None, out_nullable=None, seed=0):
    """Lay out, reduce twice, check both runs against the reference and against each other.  -> (G, out_starts)."""
    n = len(keys[0])
    part = np.zeros(n, dtype=np.int64) if part is None else part
    order = np.argsort(part, kind="stable")
    cols = [c[order] for c in keys + states]
    valids = [v[order] if v is not None else None for v in key_valid + state_valid]
    part = part[order]
    starts = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(np.bincount(part, minlength=N), out=starts[1:])
    starts_d = torch.from_numpy(starts).cuda()
    n_keys = len(keys)
    offsets = offsets or [0] * len(cols)
    out_nullable = out_nullable or [v is not None for v in valids]
    ref_groups, ref_states = reference_reduce([part] + cols[:n_keys], [None] + valids[:n_keys], cols[n_keys:], valids[n_keys:], ops)
    runs = []
    for rep in range(2):
        vals, bits, out_starts = run_once(ctx, cols, valids, n_keys, ops, starts_d, N, offsets, out_nullable, seed + rep)
        G = int(out_starts[-1])
        assert G == len(ref_groups), (G, len(ref_groups))
        p_of_row = np.searchsorted(out_starts, np.arange(G), side="right") - 1
        kvalid = [b if b is not None else np.ones(G, dtype=bool) for b in bits[:n_keys]]
        for j in range(n_keys):
            assert not vals[j][~kvalid[j]].any(), f"key {j}: bytes of a null key row are not zero"
        m = key_matrix([p_of_row] + vals[:n_keys], [None] + kvalid)
        o = np.lexsort(m.T[::-1])
        assert np.array_equal(m[o], ref_groups), "the output groups differ from the reference"
        for j, op in enumerate(ops):
            want_v, want_b = ref_states[j]
            got_v = vals[n_keys + j][o]
            got_b = bits[n_keys + j][o] if bits[n_keys + j] is not None else np.ones(G, dtype=bool)
            bad = np.nonzero(got_b != want_b)[0]
            assert len(bad) == 0, (j, op, "validity", int(bad[0]), int(got_b[bad[0]]), len(bad))
            assert got_v.dtype == want_v.dtype and got_v.shape == want_v.shape
            gb, wb = got_v.view(np.uint8).reshape(G, -1), want_v.view(np.uint8).reshape(G, -1)
            bad = np.nonzero((gb != wb).any(axis=1))[0]
            assert len(bad) == 0, (j, op, "value", int(bad[0]), gb[bad[0]].tolist(), wb[bad[0]].tolist(), bool(want_b[bad[0]]), len(bad))
        runs.append([v[o].tobytes() for v in vals] + [b[o].tobytes() for b in bits if b is not None])
    assert runs[0] == runs[1], "two runs on the same input differ"
    return int(len(ref_groups)), out_starts


def group_valid(rng, n, frac):
    return rng.random(n) >= frac


def key_parts(keys, kvs, N, rng):
    """A partition per row that depends on its key only (a NULL key included), as in a hash-partitioned table: the input
    the reduce is defined on."""
    _, gid = np.unique(key_matrix(keys, kvs), axis=0, return_inverse=True)
    gid = gid.reshape(-1)
    return rng.integers(0, N, int(gid.max()) + 1)[gid]


# ------------------------------------------------------------------- tests ----

@pytest.mark.parametrize("frac", [0.0, 0.3, 0.97, 1.0])
def test_every_op_at_null_fraction(ctx, frac):
    """All 27 ops in one call, every state column with a bitmap and the given share of nulls (0: a bitmap, all valid;
    0.97: most groups all null; 1.0: every state null), over 20 000 groups in 4 partitions."""
    rng = np.random.Generator(np.random.PCG64(int(frac * 100) + 1))
    n, g = 300_000, 20_000
    gid = rng.integers(0, g, n).astype(np.int64)
    valids = [group_valid(rng, n, frac) for _ in ALL_OPS]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ALL_OPS, valids)]
    reduce_checked(ctx, [gid], [None], states, valids, ALL_OPS, part=gid % 4, N=4, seed=10)


def lone_valid_states(g, size, rng):
    """g groups of `size` rows in random order, and a column of every MIN / MAX op in which, by (group + column) mod 6,
    a group's one valid row is its first, its last or a random row in input order, its valid rows (rows 3, 10, 17, ...)
    all hold the op's exact sentinel, the sentinel sits at row 5 among random valid rows and nulls, or every row is null.
    Garbage lies under every null.  -> (group id of every row, state columns, their valid arrays)"""
    gid = rng.permutation(np.repeat(np.arange(g), size)).astype(np.int64)
    n = len(gid)
    order = np.argsort(gid, kind="stable")
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.arange(n) - np.repeat(np.arange(g) * size, size)
    rpos = rng.integers(0, size, g)[gid]
    states, valids = [], []
    for j, op in enumerate(MINMAX_OPS):
        col = state_values(op, n, rng)
        mode = (gid + j) % 6
        half = rng.random(n) < 0.5
        valid = np.select([mode == 0, mode == 1, mode == 2, mode == 3, mode == 4],
                          [rank == 0, rank == size - 1, rank == rpos, rank % 7 == 3, half | (rank == 5)], False)
        put = ((mode == 3) & (rank % 7 == 3)) | ((mode == 4) & (rank == 5))
        col[put] = sentinel(op)
        states.append(with_nulls(col, valid, op, rng))
        valids.append(valid)
    return gid, states, valids


def test_min_max_extremes_and_lone_valid_rows(ctx):
    """Every MIN / MAX op: groups whose one valid row is the first, the last or a random row of the group in input order,
    groups whose valid rows all hold the op's exact sentinel (the result keeps its bits and its bit), groups where it
    sits next to other values and nulls, and all-null groups."""
    gid, states, valids = lone_valid_states(3000, 40, np.random.Generator(np.random.PCG64(2)))
    reduce_checked(ctx, [gid], [None], states, valids, MINMAX_OPS, seed=20)


KEY_DTYPES = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}
NULL_KEY_STATE_OPS = [nv.AGG_SUM_I64, nv.AGG_MIN_I32, nv.AGG_MAX_F64, nv.AGG_SUM_I128, nv.AGG_MIN_U8, nv.AGG_MAX_I64]


def key_column(w, values):
    if w == 16:
        return np.stack([values.astype(np.int64), (values * 7919).astype(np.int64)], axis=1)
    return values.astype(KEY_DTYPES[w])


@pytest.mark.parametrize("w", [1, 2, 4, 8, 16])
def test_nullable_key_of_every_width(ctx, w):
    """One nullable key of 1, 2, 4, 8 or 16 bytes (20 % nulls, garbage under them: all its null rows are one group),
    states with 30 % nulls, keys in 4 partitions at random."""
    rng = np.random.Generator(np.random.PCG64(30 + w))
    n = 200_000
    key = key_column(w, rng.integers(0, 180, n))
    kv = group_valid(rng, n, 0.2)
    key = with_nulls(key, kv, None, rng)
    valids = [group_valid(rng, n, 0.3) for _ in NULL_KEY_STATE_OPS]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(NULL_KEY_STATE_OPS, valids)]
    reduce_checked(ctx, [key], [kv], states, valids, NULL_KEY_STATE_OPS, part=key_parts([key], [kv], 4, rng), N=4, seed=31)


def test_eight_nullable_keys(ctx):
    """8 keys of widths 8, 1, 2, 4, 16, 8, 1, 2, each null in about a quarter of the rows and of few values, so that the
    same values with nulls at different positions make different groups."""
    rng = np.random.Generator(np.random.PCG64(40))
    n = 150_000
    keys, kvs = [], []
    for w in (8, 1, 2, 4, 16, 8, 1, 2):
        v = group_valid(rng, n, 0.25)
        keys.append(with_nulls(key_column(w, rng.integers(0, 3, n)), v, None, rng))
        kvs.append(v)
    ops = [nv.AGG_SUM_I64, nv.AGG_MIN_I128, nv.AGG_MAX_F32, nv.AGG_MIN_I16]
    valids = [group_valid(rng, n, 0.4) for _ in ops]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ops, valids)]
    G, _ = reduce_checked(ctx, keys, kvs, states, valids, ops, part=key_parts(keys, kvs, 2, rng), N=2, seed=41)
    assert G > 10_000  # (3 values or NULL in 8 columns: most of the 4^8 combinations per partition occur)


def test_null_key_group_of_2_20_rows(ctx):
    """2^20 rows whose key is null (each with different garbage bytes) among 100 000 rows of 5 000 other keys: one group."""
    rng = np.random.Generator(np.random.PCG64(50))
    n_null, n_other = 1 << 20, 100_000
    key = np.concatenate([rng.integers(-(1 << 63), (1 << 63) - 1, n_null, dtype=np.int64, endpoint=True), rng.integers(0, 5000, n_other)])
    kv = np.concatenate([np.zeros(n_null, bool), np.ones(n_other, bool)])
    perm = rng.permutation(len(key))
    key, kv = key[perm], kv[perm]
    ops = [nv.AGG_SUM_I64, nv.AGG_MIN_F32, nv.AGG_MAX_I128, nv.AGG_SUM_F64]
    valids = [group_valid(rng, len(key), 0.5) for _ in ops]
    states = [with_nulls(state_values(op, len(key), rng), v, op, rng) for op, v in zip(ops, valids)]
    G, _ = reduce_checked(ctx, [key], [kv], states, valids, ops, seed=51)
    assert G == 5001


def test_every_column_at_its_own_bit_offset(ctx):
    """Two nullable keys and nine nullable states, every column at its own Arrow offset (1..7, 13, 37), every input
    bitmap at an odd byte address."""
    rng = np.random.Generator(np.random.PCG64(60))
    n = 120_000
    keys = [key_column(4, rng.integers(0, 40, n)), key_column(8, rng.integers(0, 40, n))]
    kvs = [group_valid(rng, n, 0.1), group_valid(rng, n, 0.15)]
    keys = [with_nulls(k, v, None, rng) for k, v in zip(keys, kvs)]
    ops = [nv.AGG_SUM_I64, nv.AGG_MIN_I8, nv.AGG_MAX_U16, nv.AGG_MIN_F64, nv.AGG_SUM_I128, nv.AGG_MAX_I128, nv.AGG_MIN_F16,
           nv.AGG_MAX_U32, nv.AGG_SUM_F64]
    valids = [group_valid(rng, n, 0.6) for _ in ops]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ops, valids)]
    offsets = [1, 2, 3, 4, 5, 6, 7, 13, 37, 3, 1]
    reduce_checked(ctx, keys, kvs, states, valids, ops, part=key_parts(keys, kvs, 3, rng), N=3, offsets=offsets, seed=61)


@pytest.mark.parametrize("n_groups", [1, 31, 32, 33, 1000])
def test_output_bitmap_words_and_all_valid_outputs(ctx, n_groups):
    """G = 1, 31, 32, 33, 1000: the last word's bits past G are zero and the words past it keep their fill.  Output
    bitmaps for columns without an input bitmap (a key and two states) come out all ones."""
    rng = np.random.Generator(np.random.PCG64(70 + n_groups))
    n = 5000
    key = rng.integers(0, n_groups, n).astype(np.int64)
    key[:n_groups] = np.arange(n_groups)
    ops = [nv.AGG_SUM_I64, nv.AGG_MIN_I32, nv.AGG_MAX_I64, nv.AGG_MIN_U8]
    valids = [None, None, group_valid(rng, n, 0.5), group_valid(rng, n, 0.9)]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ops, valids)]
    G, _ = reduce_checked(ctx, [key], [None], states, valids, ops, out_nullable=[True] * 5, seed=71)
    assert G == n_groups


def test_misaligned_output_bitmap_is_refused_before_any_launch(ctx):
    n = 1000
    rng = np.random.Generator(np.random.PCG64(80))
    key = rng.integers(0, 10, n).astype(np.int64)
    st = rng.integers(0, 100, n).astype(np.int32)
    sv = group_valid(rng, n, 0.5)
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    for shift in (1, 2, 3):
        dcols = [upload(key, None, 0, rng), upload(st, sv, 0, rng)]
        outs = [guarded_output(8, n, True), guarded_output(4, n, True, bitmap_shift=shift)]
        torch.cuda.synchronize()
        before = ctx.metrics()["kernel_launches"]
        with pytest.raises(dfd.DfdError) as ei:
            dfd.PartialReduceExec(ctx, [0], [-1, nv.AGG_MIN_I32]).reduce(dcols, n, starts.data_ptr(), 1, [o[0] for o in outs])
        assert ei.value.status == ERR_INVALID_ARGUMENT and "aligned" in ei.value.message, ei.value.message
        assert ctx.metrics()["kernel_launches"] == before
        torch.cuda.synchronize()
        for _, t, vt in outs:
            assert bool((t == FILL).all()) and bool((vt == FILL).all())


def test_input_bitmap_without_output_bitmap_is_refused(ctx):
    n = 100
    key = torch.arange(n, dtype=torch.int64, device="cuda")
    vb = torch.full(((n + 7) // 8,), 0xFF, dtype=torch.uint8, device="cuda")
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    ko = torch.empty(n, dtype=torch.int64, device="cuda")
    for i in (0, 1):  # the key or the state has the bitmap
        ins = [dfd.DeviceColumn.from_torch(key, vb if i == 0 else None), dfd.DeviceColumn.from_torch(key, vb if i == 1 else None)]
        outs = [dfd.DeviceColumn.from_torch(ko), dfd.DeviceColumn.from_torch(ko.clone())]
        with pytest.raises(dfd.DfdError) as ei:
            dfd.PartialReduceExec(ctx, [0], [-1, nv.AGG_SUM_I64]).reduce(ins, n, starts.data_ptr(), 1, outs)
        assert ei.value.status == ERR_UNSUPPORTED and "non-null" in ei.value.message


def test_launch_counts(ctx):
    """4 launches without bitmaps, with output bitmaps only and with nullable keys and SUM states; 5 once a MIN / MAX
    state column has an input bitmap (reduce_checked asserts the count of every call)."""
    rng = np.random.Generator(np.random.PCG64(90))
    n = 10_000
    key = rng.integers(0, 300, n).astype(np.int64)
    kv = group_valid(rng, n, 0.1)
    s = state_values(nv.AGG_SUM_I64, n, rng)
    m = state_values(nv.AGG_MIN_I32, n, rng)
    sv, mv = group_valid(rng, n, 0.5), group_valid(rng, n, 0.5)
    ops = [nv.AGG_SUM_I64, nv.AGG_MIN_I32]
    for kvv, valids, nullable in ((None, [None, None], [False] * 3), (None, [None, None], [True] * 3), (kv, [sv, None], None), (kv, [sv, mv], None)):
        states = [with_nulls(s, valids[0], ops[0], rng), with_nulls(m, valids[1], ops[1], rng)]
        assert expected_launches([None] + valids, [-1] + ops, n) == (5 if valids[1] is not None else 4)
        reduce_checked(ctx, [with_nulls(key, kvv, None, rng)], [kvv], states, valids, ops, out_nullable=nullable, seed=91)


def test_rows_past_two_grid_passes(ctx):
    """2G + 7 rows (G: threads of one grid pass on this device), nullable key and states, in about n / 4 groups."""
    rng = np.random.Generator(np.random.PCG64(100))
    n = 2 * grid_threads() + 7
    key = rng.integers(0, n // 4, n).astype(np.int64)
    kv = group_valid(rng, n, 0.05)
    ops = [nv.AGG_SUM_I128, nv.AGG_MIN_I64, nv.AGG_MAX_F16, nv.AGG_MIN_U64]
    valids = [group_valid(rng, n, 0.5) for _ in ops]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ops, valids)]
    key = with_nulls(key, kv, None, rng)
    reduce_checked(ctx, [key], [kv], states, valids, ops, part=key_parts([key], [kv], 16, rng), N=16, seed=101)


def test_one_group_of_2_24_rows_half_null_every_op(ctx):
    """Every op over one group of 2^24 rows, half of every state null: all rows contend for one state and one bitmap
    word per column."""
    rng = np.random.Generator(np.random.PCG64(110))
    n = 1 << 24
    key = np.zeros(n, dtype=np.int64)
    valids = [group_valid(rng, n, 0.5) for _ in ALL_OPS]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ALL_OPS, valids)]
    reduce_checked(ctx, [key], [None], states, valids, ALL_OPS, seed=111)


def test_2_20_groups(ctx):
    rng = np.random.Generator(np.random.PCG64(120))
    n = 1 << 22
    key = rng.integers(0, 1 << 20, n).astype(np.int64)
    kv = group_valid(rng, n, 0.02)
    ops = [nv.AGG_SUM_I64, nv.AGG_SUM_F64, nv.AGG_MIN_F64, nv.AGG_MAX_I8, nv.AGG_MIN_I128, nv.AGG_MAX_U32]
    valids = [group_valid(rng, n, 0.7) for _ in ops]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ops, valids)]
    key = with_nulls(key, kv, None, rng)
    reduce_checked(ctx, [key], [kv], states, valids, ops, part=key_parts([key], [kv], 8, rng), N=8, seed=121)


def test_every_row_its_own_group_every_state_null(ctx):
    """600 000 singleton groups and every state null: every output state is zero with its bit clear."""
    rng = np.random.Generator(np.random.PCG64(130))
    n = 600_000
    key = rng.permutation(n).astype(np.int64)
    valids = [np.zeros(n, dtype=bool) for _ in ALL_OPS]
    states = [with_nulls(state_values(op, n, rng), v, op, rng) for op, v in zip(ALL_OPS, valids)]
    reduce_checked(ctx, [key], [None], states, valids, ALL_OPS, part=key % 8, N=8, seed=131)


# ------------------------------------------------------------- end to end ----

def window_to_arrow(ctx, col, arrow_type, width_b, start, count):
    """Rows [start, start + count) of an exchange window column as a pyarrow Array (segments start on 32-row bounds)."""
    data = np.empty(count * width_b, dtype=np.uint8)
    nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, data.ctypes.data, col.values + start * width_b, data.nbytes))
    assert start % 8 == 0
    vb = np.empty((count + 7) // 8, dtype=np.uint8)
    if vb.size:
        nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, vb.ctypes.data, col.validity + start // 8, vb.nbytes))
    nulls = count - int(np.unpackbits(vb, bitorder="little")[:count].sum())
    return pa.Array.from_buffers(arrow_type, count, [pa.py_buffer(vb.tobytes()), pa.py_buffer(data.tobytes())], null_count=nulls)


def test_nullable_table_through_partition_reduce_and_shuffle(ctx):
    """A nullable Arrow table (Int32 key; Int64, Decimal128, Float64, Date32 states) through HashPartitioner ->
    PartialReduceExec -> shuffle_partitioned on one worker equals pyarrow's group_by of the table: integers and decimals
    exactly, float MIN / MAX bitwise."""
    rng = np.random.Generator(np.random.PCG64(140))
    n, N = 200_000, 6
    key = rng.integers(0, 3000, n).astype(np.int32)
    kv = group_valid(rng, n, 0.05)
    s = rng.integers(-(10 ** 12), 10 ** 12, n)
    sv = group_valid(rng, n, 0.4) & (key % 97 != 0)  # every key = 0 mod 97 has only null states
    dec = rng.integers(-(10 ** 17), 10 ** 17, n)
    dv = group_valid(rng, n, 0.4) & (key % 97 != 0)
    f = rng.standard_normal(n) * 1000.0
    fv = group_valid(rng, n, 0.4) & (key % 97 != 0)
    dt = rng.integers(0, 40_000, n).astype(np.int32)
    tv = group_valid(rng, n, 0.4) & (key % 97 != 0)
    table = pa.table({
        "k": pa.array(key, mask=~kv), "s": pa.array(s, mask=~sv),
        "d": pa.array([Decimal(int(x)) for x in dec], type=pa.decimal128(38, 0), mask=~dv),
        "fmin": pa.array(f, mask=~fv), "fmax": pa.array(f, mask=~fv),
        "t": pa.array(dt, type=pa.int32(), mask=~tv).cast(pa.date32()),
    })
    ops = [-1, nv.AGG_SUM_I64, nv.AGG_SUM_I128, nv.AGG_MIN_F64, nv.AGG_MAX_F64, nv.AGG_MIN_I32]
    dcols = [dfd.DeviceColumn.from_arrow(ctx, table.column(i)) for i in range(table.num_columns)]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    pouts, _ = part.partition(dcols, n)
    nullable = [True] * len(ops)
    outs, out_starts = dfd.PartialReduceExec(ctx, [0], ops).reduce(pouts, n, part.part_starts_device_ptr(), N, nullable=nullable)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    try:
        ex.setup_window(64 << 20)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], N), uuid.uuid4(), 1, 1, 1)
        wcols, ss, sc = node.shuffle_partitioned(ex, outs, out_starts, nullable=nullable)
        assert np.array_equal(sc[:, 0], np.diff(out_starts))
        widths = [4, 8, 16, 8, 8, 4]
        pieces = [[window_to_arrow(ctx, wc, table.schema.field(i).type, widths[i], int(ss[q, 0]), int(sc[q, 0])) for q in range(N)]
                  for i, wc in enumerate(wcols)]
    finally:
        ex.close()
    got = pa.table({table.column_names[i]: pa.concat_arrays(pieces[i]) for i in range(len(ops))})
    want = table.group_by("k").aggregate([("s", "sum"), ("d", "sum"), ("fmin", "min"), ("fmax", "max"), ("t", "min")])
    assert got.num_rows == want.num_rows  # one row per key (and one for the NULL key) over all partitions
    got_rows = {r["k"]: r for r in got.to_pylist()}
    assert len(got_rows) == got.num_rows and None in got_rows
    for r in want.to_pylist():
        g = got_rows[r["k"]]
        assert (g["s"], g["d"], g["t"]) == (r["s_sum"], r["d_sum"], r["t_min"]), r["k"]
        for name, col in (("fmin", "fmin_min"), ("fmax", "fmax_max")):
            a, b = g[name], r[col]
            assert (a is None and b is None) or np.float64(a).view(np.uint64) == np.float64(b).view(np.uint64), (r["k"], name, a, b)
    assert sum(1 for r in want.to_pylist() if r["s_sum"] is None) >= 25  # the all-null state groups were there
