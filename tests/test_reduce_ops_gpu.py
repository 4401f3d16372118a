"""GPU parity tests of the PartialReduce MIN / MAX ops for 8- to 128-bit signed and unsigned integers and for Float32 /
Float16 (dfd_agg_op 7..26), bit for bit against a restatement of each merge on the host:

- Integers compare as their type: numpy's own order for up to 64 bits; 128-bit decimals as Python ints (signed high
  half, unsigned low half), or, for the large cases, by a two-step numpy reduction (highest high half, then the lowest /
  highest low half among the rows that hold it) that the edge test checks against the Python ints.
- Floats compare under IEEE 754 totalOrder (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN, NaNs by payload), so
  the result is always the bits of one input row and is compared bitwise.

Every call also checks what the reduce must leave alone: bytes in front of and behind each output column and past its
out_part_starts[N] rows keep their fill."""
import uuid

import numpy as np
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.test_reduce_limits_gpu import upload_at

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED = 1, 6
FILL, GUARD = 0xA5, 64
M64 = (1 << 64) - 1

# state type -> (MIN op, numpy dtype of the column: float states travel as their bit patterns, 128-bit ones as 2 x int64)
TYPES = {
    "i32": (nv.AGG_MIN_I32, np.int32), "i16": (nv.AGG_MIN_I16, np.int16), "i8": (nv.AGG_MIN_I8, np.int8),
    "u64": (nv.AGG_MIN_U64, np.uint64), "u32": (nv.AGG_MIN_U32, np.uint32), "u16": (nv.AGG_MIN_U16, np.uint16),
    "u8": (nv.AGG_MIN_U8, np.uint8), "i128": (nv.AGG_MIN_I128, np.int64), "f32": (nv.AGG_MIN_F32, np.uint32),
    "f16": (nv.AGG_MIN_F16, np.uint16),
}
OP_TYPE = {op: t for t, (mn, _) in TYPES.items() for op in (mn, mn + 1)}
NEW_OPS = sorted(OP_TYPE)
assert NEW_OPS == list(range(7, 27))


def is_max(op):
    return (op - nv.AGG_MIN_I32) % 2 == 1


def width(col):
    return 16 if col.ndim == 2 else col.dtype.itemsize


# ------------------------------------------------------------------ inputs ----

def float_specials(w):
    """Bit patterns of +-0, +-inf, the smallest and largest subnormals of both signs, and NaNs of both signs with
    different payloads (quiet and signalling), for a float of w bits."""
    e = {16: 5, 32: 8}[w]
    m = w - 1 - e
    sign, inf = 1 << (w - 1), ((1 << e) - 1) << m
    pos = [0, inf, 1, (1 << m) - 1, inf | (1 << (m - 1)), inf | (1 << (m - 1)) | 1, inf | 1, inf | ((1 << m) - 1)]
    return pos + [sign | b for b in pos]


def edge_values(tname):
    """Values every type must order right: its extremes, pairs that differ only in the sign bit, and (unsigned) values
    above 2^(w-1) that a signed order would put below zero.  128-bit: Python ints; floats: bit patterns."""
    if tname == "i128":
        lo_edges = [0, 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, M64 - 1, M64]
        his = [-(1 << 63), -2, -1, 0, 1, (1 << 63) - 1]
        return [(h << 64) | lo for h in his for lo in lo_edges]
    if tname in ("f32", "f16"):
        w = int(tname[1:])
        return float_specials(w) + [int(b) for b in np.array([1.0, -1.0, 2.5, -2.5, 65504.0, -65504.0],
                                                             dtype=np.float16 if w == 16 else np.float32).view(f"u{w // 8}")]
    dt = np.dtype(TYPES[tname][1])
    w = 8 * dt.itemsize
    if dt.kind == "i":
        lo, hi = -(1 << (w - 1)), (1 << (w - 1)) - 1
        return [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi, 5, 5 - (1 << (w - 1)), -5, -5 + (1 << (w - 1))]  # x and x with the sign bit flipped
    top = (1 << w) - 1
    return [0, 1, 2, (1 << (w - 1)) - 1, 1 << (w - 1), (1 << (w - 1)) + 1, top - 1, top, 5, 5 | (1 << (w - 1))]


def to_column(tname, values):
    """Python values (ints / bit patterns / 128-bit ints) -> the numpy column the device reads."""
    if tname == "i128":
        v = [x & ((1 << 128) - 1) for x in values]
        lo = np.array([x & M64 for x in v], dtype=np.uint64).view(np.int64)
        hi = np.array([x >> 64 for x in v], dtype=np.uint64).view(np.int64)
        return np.stack([lo, hi], axis=1)
    return np.array(values, dtype=TYPES[tname][1])


def random_values(tname, n, rng):
    """n values of the type, about one in eight drawn from its edge values, the rest uniform over all its bit patterns
    (128-bit: high halves mostly from a few small values, so that many rows tie on the high half and the low half
    decides)."""
    edges = edge_values(tname)
    pick = rng.random(n) < 0.125
    if tname == "i128":
        col = np.empty((n, 2), dtype=np.int64)
        col[:, 0] = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
        col[:, 1] = np.where(rng.random(n) < 0.7, rng.integers(-2, 2, n), rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True))
        e = to_column("i128", edges)
        col[pick] = e[rng.integers(0, len(edges), int(pick.sum()))]
        return col
    dt = np.dtype(TYPES[tname][1])
    u = rng.integers(0, 1 << (8 * dt.itemsize), n, dtype=np.uint64).astype(f"u{dt.itemsize}")
    col = u.view(dt).copy()
    col[pick] = to_column(tname, edges)[rng.integers(0, len(edges), int(pick.sum()))]
    return col


# --------------------------------------------------------- exact reference ----

def py_values(tname, col):
    """A column as Python ints: the value for integers, the bit pattern for floats, signed 128-bit ints."""
    if tname == "i128":
        return [(hi << 64) | lo for lo, hi in zip(col[:, 0].view(np.uint64).tolist(), col[:, 1].tolist())]
    return col.tolist()


def total_order_key(bits, w):
    s = bits - (1 << w) if bits >> (w - 1) else bits
    return s ^ ((s >> (w - 1)) & ((1 << (w - 1)) - 1))


def py_merge(tname, op, xs):
    """The merged MIN / MAX of one group's Python values, as the value or bit pattern the output must hold."""
    key = (lambda b: total_order_key(b, int(tname[1:]))) if tname in ("f32", "f16") else (lambda v: v)
    return (max if is_max(op) else min)(xs, key=key)


def np_merge(tname, op, col, order, seg):
    """Vectorised MIN / MAX of every group: `order` sorts the rows by group, `seg` = first sorted row of every group.
    -> the merged value (bit pattern for floats; an (n, 2) int64 array for 128-bit) of every group."""
    red = np.maximum if is_max(op) else np.minimum
    if tname == "i128":
        lo, hi = col[order, 0].view(np.uint64), col[order, 1]
        ghi = red.reduceat(hi, seg)
        counts = np.diff(np.append(seg, len(order)))
        on_top = hi == np.repeat(ghi, counts)
        glo = red.reduceat(np.where(on_top, lo, np.uint64(0) if is_max(op) else np.uint64(M64)), seg)
        return np.stack([glo.view(np.int64), ghi], axis=1)
    c = col[order]
    if tname in ("f32", "f16"):
        w = int(tname[1:])
        s = c.view(f"i{w // 8}")
        k = s ^ ((s >> (w - 1)) & ((1 << (w - 1)) - 1)).astype(s.dtype)
        g = red.reduceat(k, seg)
        return (g ^ ((g >> (w - 1)) & ((1 << (w - 1)) - 1)).astype(g.dtype)).view(c.dtype)
    return red.reduceat(c, seg)


# ------------------------------------------------------------- device i/o ----

def guarded_output(col, capacity, base_offset=0):
    """An output column of `capacity` rows starting `base_offset` bytes past a 256-byte-aligned address, inside a buffer
    of FILL bytes with GUARD bytes in front and GUARD behind.  -> (DeviceColumn, buffer, first byte of the column)"""
    w = width(col)
    start = GUARD + base_offset
    t = torch.full((start + capacity * w + GUARD,), FILL, dtype=torch.uint8, device="cuda")
    return dfd.DeviceColumn(nv.COL_FIXED, w, t.data_ptr() + start, length=capacity, keep=t), t, start


def reduce_and_check_fill(ctx, cols, n_keys, ops, part, N, out_offsets=None, in_offsets=None):
    """Lay the rows out partition by partition, reduce them on the device (output column i at out_offsets[i] bytes past
    an aligned address, input column i at Arrow offset in_offsets[i]), and check that only the first out_part_starts[N]
    rows of each output were written.  -> (sorted input columns, output columns as numpy arrays, out_part_starts)"""
    n = len(part)
    order = np.argsort(part, kind="stable")
    cols, part = [c[order] for c in cols], part[order]
    starts = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(np.bincount(part, minlength=N), out=starts[1:])
    dcols = upload_at(cols, in_offsets or [0] * len(cols), 3)
    outs = [guarded_output(c, n, off) for c, off in zip(cols, out_offsets or [0] * len(cols))]
    starts_d = torch.from_numpy(starts).cuda()
    torch.cuda.synchronize()
    _, out_starts = dfd.PartialReduceExec(ctx, list(range(n_keys)), ops).reduce(dcols, n, starts_d.data_ptr(), N, [o[0] for o in outs])
    total = int(out_starts[-1])
    host = []
    for i, (c, (_, t, start)) in enumerate(zip(cols, outs)):
        raw = t.cpu().numpy()
        w = width(c)
        assert bool((raw[:start] == FILL).all()), f"column {i}: a byte in front of the column was written"
        assert bool((raw[start + total * w:] == FILL).all()), f"column {i}: a byte past row {total} was written"
        v = raw[start:start + total * w].view(np.int64 if c.ndim == 2 else c.dtype)
        host.append(v.reshape(total, 2) if c.ndim == 2 else v)
    return cols, host, out_starts, part


def check_groups(host, out_starts, part, gid, cols, n_keys, ops, python_ref=False):
    """Column 0 of the output is the group id (int64); every group is in one row of its own partition, and every state
    equals the reference merge of the group's rows, bit for bit."""
    n_groups = int(gid.max()) + 1
    got_gid = host[0]
    total = int(out_starts[-1])
    present = np.unique(gid)
    assert total == len(present) and np.array_equal(np.sort(got_gid), present)
    p_of_row = np.searchsorted(out_starts, np.arange(total), side="right") - 1
    gpart = np.zeros(n_groups, dtype=np.int64)
    gpart[gid] = part
    assert np.array_equal(p_of_row, gpart[got_gid])
    order = np.argsort(gid, kind="stable")
    seg = np.searchsorted(gid[order], present)
    for j in range(n_keys, len(cols)):
        op, tname = ops[j], OP_TYPE[ops[j]]
        want = np_merge(tname, op, cols[j], order, seg)  # row i = group present[i]
        got = host[j][np.argsort(got_gid)]
        assert got.tobytes() == want.tobytes(), (j, tname, op, first_mismatch(got, want))
        if python_ref:  # the same groups through Python ints / totalOrder keys, one group at a time
            vals, gv = py_values(tname, cols[j]), gid.tolist()
            per = {}
            for r, g in enumerate(gv):
                per.setdefault(g, []).append(vals[r])
            want_py = [py_merge(tname, op, per[g]) for g in present.tolist()]
            got_py = py_values(tname, got)
            assert got_py == want_py, (j, tname, op, [(g, a, b) for g, a, b in zip(present.tolist(), got_py, want_py) if a != b][:5])


def first_mismatch(got, want):
    g, w = got.reshape(len(got), -1), want.reshape(len(want), -1)
    bad = np.nonzero((g != w).any(axis=1))[0]
    return (int(bad[0]), g[bad[0]].tolist(), w[bad[0]].tolist(), len(bad)) if len(bad) else None


def group_parts(gid, N, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return rng.integers(0, N, int(gid.max()) + 1)[gid]


# ------------------------------------------------------------------- tests ----

@pytest.mark.parametrize("tname", list(TYPES))
def test_edge_values(ctx, tname):
    """MIN and MAX of one type in one call: 3 000 groups of random values with one in eight drawn from the type's edge
    values, plus one group per edge value alone and one group of every edge value together; checked against numpy and
    against plain Python ints (128-bit signed compare, totalOrder keys)."""
    rng = np.random.Generator(np.random.PCG64(1000 + NEW_OPS.index(TYPES[tname][0])))
    n, g_rand = 60_000, 3_000
    edges = to_column(tname, edge_values(tname))
    ne = len(edges)
    gid = np.concatenate([rng.integers(0, g_rand, n), g_rand + np.arange(ne), np.full(ne * 40, g_rand + ne)])
    vals = np.concatenate([random_values(tname, n, rng), edges, np.tile(edges, (40, 1) if edges.ndim == 2 else 40)])
    perm = rng.permutation(len(gid))
    gid, vals = gid[perm], vals[perm]
    mn = TYPES[tname][0]
    cols, ops = [gid.astype(np.int64), vals, vals.copy()], [-1, mn, mn + 1]
    part = group_parts(gid, 4, 5)
    scols, host, out_starts, spart = reduce_and_check_fill(ctx, cols, 1, ops, part, 4)
    check_groups(host, out_starts, spart, scols[0], scols, 1, ops, python_ref=True)


def i128(x):
    return x & ((1 << 128) - 1)


I128_GROUPS = [  # (values, MIN, MAX): signed high halves first, then unsigned low halves
    ([(5 << 64) | ((1 << 63) - 1), (5 << 64) | (1 << 63), (5 << 64) | ((1 << 63) + 1)],
     (5 << 64) | ((1 << 63) - 1), (5 << 64) | ((1 << 63) + 1)),  # equal high halves, low halves straddling 2^63
    ([(-3 << 64) | (1 << 63), (-3 << 64) | 7, (-3 << 64) | M64], (-3 << 64) | 7, (-3 << 64) | M64),  # negative high half
    ([(1 << 64) | 42, (-1 << 64) | 42, (0 << 64) | 42], (-1 << 64) | 42, (1 << 64) | 42),  # equal low halves
    ([-1, -(10 ** 30), 10 ** 30, -12345, 0], -(10 ** 30), 10 ** 30),  # negative decimals
    ([-(1 << 127), (1 << 127) - 1, 0], -(1 << 127), (1 << 127) - 1),  # the type's extremes
    ([((1 << 63) - 1) << 64, (-(1 << 63)) << 64 | M64], (-(1 << 63)) << 64 | M64, ((1 << 63) - 1) << 64),  # sign of the high half
    ([-1, 1, (1 << 64) - 1, -(1 << 64)], -(1 << 64), (1 << 64) - 1),
]


def test_i128_compares_across_the_halves(ctx):
    """Decimal128 MIN / MAX: the high halves compare signed, and only when they tie do the low halves decide, unsigned.
    Thousands of rows of each group race on its state; the expected results are written out by hand."""
    copies = 3000
    rng = np.random.Generator(np.random.PCG64(21))
    gid = np.concatenate([np.full(len(v) * copies, g) for g, (v, _, _) in enumerate(I128_GROUPS)])
    vals = [x for v, _, _ in I128_GROUPS for x in v * copies]
    perm = rng.permutation(len(gid))
    gid, col = gid[perm], to_column("i128", vals)[perm]
    ops = [-1, nv.AGG_MIN_I128, nv.AGG_MAX_I128]
    scols, host, out_starts, _ = reduce_and_check_fill(ctx, [gid.astype(np.int64), col, col.copy()], 1, ops, gid % 2, 2)
    got_min, got_max = py_values("i128", host[1]), py_values("i128", host[2])
    for r, g in enumerate(host[0].tolist()):
        _, want_min, want_max = I128_GROUPS[g]
        assert (got_min[r], got_max[r]) == (want_min, want_max), (g, got_min[r], got_max[r])


def f_bits(xs, w):
    return [int(b) for b in np.array(xs, dtype=np.float16 if w == 16 else np.float32).view(f"u{w // 8}")]


@pytest.mark.parametrize("w", [32, 16])
def test_float_special_values_total_order(ctx, w):
    """Float32 / Float16 MIN / MAX under totalOrder: a +NaN wins MAX and a -NaN wins MIN, NaNs order by payload, -0.0 <
    +0.0, subnormals sit between the zeros and the normals, and an all-NaN group yields one of its own NaNs."""
    e = {16: 5, 32: 8}[w]
    m = w - 1 - e
    S, INF = 1 << (w - 1), ((1 << e) - 1) << m
    qnan, qnan1, snan, nan_max = INF | (1 << (m - 1)), INF | (1 << (m - 1)) | 1, INF | 1, INF | ((1 << m) - 1)
    sub, sub_max = 1, (1 << m) - 1
    one, three, five = f_bits([1.0, 3.0, 5.0], w)
    groups = [  # (bit patterns, MIN, MAX)
        ([one, qnan], one, qnan),
        ([qnan, qnan1, snan, nan_max], snan, nan_max),
        ([qnan, qnan1, S | qnan], S | qnan, qnan1),
        ([S | qnan, S | snan, S | nan_max], S | nan_max, S | snan),  # negative NaNs: the largest payload is the least
        ([S, 0], S, 0),
        ([S], S, S),
        ([INF, S | INF, three], S | INF, INF),
        ([sub, S | sub, 0, S, sub_max, one], S | sub, one),
        ([S | sub_max, S | sub, S | one], S | one, S | sub),
        ([S | qnan, five], S | qnan, five),
    ]
    copies = 3000
    rng = np.random.Generator(np.random.PCG64(22 + w))
    gid = np.concatenate([np.full(len(v) * copies, g) for g, (v, _, _) in enumerate(groups)])
    bits = np.concatenate([np.tile(np.array(v, dtype=f"u{w // 8}"), copies) for v, _, _ in groups])
    perm = rng.permutation(len(gid))
    gid, bits = gid[perm], bits[perm]
    mn = TYPES[f"f{w}"][0]
    ops = [-1, mn, mn + 1]
    for _ in range(2):
        scols, host, out_starts, spart = reduce_and_check_fill(ctx, [gid.astype(np.int64), bits, bits.copy()], 1, ops, gid % 3, 3)
        for r, g in enumerate(host[0].tolist()):
            _, want_min, want_max = groups[g]
            assert (int(host[1][r]), int(host[2][r])) == (want_min, want_max), (g, hex(int(host[1][r])), hex(int(host[2][r])))
        check_groups(host, out_starts, spart, scols[0], scols, 1, ops, python_ref=True)


# (rows, groups, partitions): one group holding every row (the CAS loops' worst contention), many groups, and every row
# its own group; all of them many grid passes (132 SMs x 8 CTAs x 256 threads = 270 336 rows per pass on an H100 SXM)
SHAPES = {"one_group_2^24_rows": (1 << 24, 1, 1), "2^20_groups": (1 << 22, 1 << 20, 16), "every_row_its_own_group": (600_000, 600_000, 8)}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_group_shapes_every_new_op(ctx, shape):
    """All 20 new ops in one call, over one huge group, many groups and singleton groups."""
    n, n_groups, N = SHAPES[shape]
    rng = np.random.Generator(np.random.PCG64(31))
    gid = rng.permutation(n) if n_groups == n else rng.integers(0, n_groups, n)
    cols, ops = [gid.astype(np.int64)], [-1]
    for op in NEW_OPS:
        cols.append(random_values(OP_TYPE[op], n, rng))
        ops.append(op)
    part = group_parts(gid, N, 6)
    scols, host, out_starts, spart = reduce_and_check_fill(ctx, cols, 1, ops, part, N)
    check_groups(host, out_starts, spart, scols[0], scols, 1, ops)


def eight_keys(gid):
    """Eight key columns of widths 8, 1, 2, 4, 16, 8, 1, 2 that together are injective on the group id (the first is the
    group id itself, which the checks read back)."""
    g = gid.astype(np.int64)
    return [g, (g % 251).astype(np.uint8), (g % 30011).astype(np.int16), (g // 7).astype(np.int32), np.stack([g // 5, g % 3], axis=1),
            g * 7, (g % 2).astype(np.uint8), (g % 65521).astype(np.uint16)]


def test_eight_keys_and_24_mixed_state_columns_deterministic(ctx):
    """8 keys and 24 state columns in one call: every new op once and four of them twice, so every width 1, 2, 4, 8, 16
    appears next to the others.  Two runs give the same bytes."""
    n, n_groups, N = 1 << 20, 50_000, 8
    rng = np.random.Generator(np.random.PCG64(41))
    gid = rng.integers(0, n_groups, n)
    state_ops = NEW_OPS + [nv.AGG_MIN_U8, nv.AGG_MAX_I16, nv.AGG_MIN_I128, nv.AGG_MAX_F16]
    assert len(state_ops) == 24
    keys = eight_keys(gid)
    cols = keys + [random_values(OP_TYPE[op], n, rng) for op in state_ops]
    ops = [-1] * 8 + state_ops
    part = group_parts(gid, N, 7)
    runs = []
    for _ in range(2):
        scols, host, out_starts, spart = reduce_and_check_fill(ctx, cols, 8, ops, part, N)
        check_groups(host, out_starts, spart, scols[0], scols, 8, ops)
        order = np.argsort(host[0])  # row order inside a partition is unspecified; the bytes of every group's row are not
        runs.append([h[order].tobytes() for h in host])
    assert runs[0] == runs[1]


@pytest.mark.parametrize("base", [1, 2, 3])
def test_narrow_states_at_unaligned_bases(ctx, base):
    """1-byte states at output addresses 1, 2 and 3 mod 4 (and 2-byte ones at 2 mod 4, the one unaligned-to-4 address
    a 2-byte value can have): adjacent output rows share a 32-bit word and belong to different groups updated at the
    same moment, and the guard bytes in front of and behind every column stay as they were.  The inputs sit at odd
    Arrow offsets."""
    n, n_groups = 1 << 20, 200_000
    rng = np.random.Generator(np.random.PCG64(50 + base))
    gid = rng.integers(0, n_groups, n)
    state_ops = [nv.AGG_MIN_I8, nv.AGG_MAX_I8, nv.AGG_MIN_U8, nv.AGG_MAX_U8, nv.AGG_MIN_I16, nv.AGG_MAX_U16, nv.AGG_MIN_F16]
    cols = [gid.astype(np.int64)] + [random_values(OP_TYPE[op], n, rng) for op in state_ops]
    ops = [-1] + state_ops
    out_offsets = [0] + [base if width(c) == 1 else 2 for c in cols[1:]]
    in_offsets = [0] + [3, 1, 2, 5, 1, 3, 7]
    scols, host, out_starts, spart = reduce_and_check_fill(ctx, cols, 1, ops, group_parts(gid, 4, 8), 4, out_offsets, in_offsets)
    check_groups(host, out_starts, spart, scols[0], scols, 1, ops)


def test_i128_input_aligned_to_8_bytes(ctx):
    """A Decimal128 input column needs only 8-byte alignment (its halves are read as two 64-bit words)."""
    n = 100_000
    rng = np.random.Generator(np.random.PCG64(60))
    gid = rng.integers(0, 1000, n)
    col = random_values("i128", n, rng)
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    t = torch.from_numpy(np.concatenate([np.zeros(8, np.uint8), col.view(np.uint8).reshape(-1)])).cuda()
    key = torch.from_numpy(gid.astype(np.int64)).cuda()
    dcols = [dfd.DeviceColumn.from_torch(key), dfd.DeviceColumn(nv.COL_FIXED, 16, t.data_ptr() + 8, length=n, keep=t)]
    outs, out_starts = dfd.PartialReduceExec(ctx, [0], [-1, nv.AGG_MAX_I128]).reduce(dcols, n, starts.data_ptr(), 1)
    total = int(out_starts[-1])
    host_g = np.empty(total, np.int64)
    host_v = np.empty((total, 2), np.int64)
    nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, host_g.ctypes.data, outs[0].values, host_g.nbytes))
    nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, host_v.ctypes.data, outs[1].values, host_v.nbytes))
    present = np.unique(gid)
    order = np.argsort(gid, kind="stable")
    want = np_merge("i128", nv.AGG_MAX_I128, col, order, np.searchsorted(gid[order], present))
    assert host_v[np.argsort(host_g)].tobytes() == want.tobytes()


def test_partition_reduce_shuffle_end_to_end(ctx):
    """Partial output -> repartition -> PartialReduce with new ops -> dfd_exchange_gather(DFD_ROUTE_SHUFFLE), all on the
    device (world = 1): partition q's segment holds exactly the merged states of destination q's groups."""
    n, N = 200_000, 6
    rng = np.random.Generator(np.random.PCG64(70))
    gid = rng.integers(0, 5_000, n)
    key = (gid * 1_000_003).astype(np.int64)
    state_ops = [nv.AGG_MIN_I128, nv.AGG_MAX_I32, nv.AGG_MIN_F32, nv.AGG_MAX_U8]
    states = [random_values(OP_TYPE[op], n, rng) for op in state_ops]
    cols = [key] + states
    dcols = upload_at(cols, [0] * len(cols), 1)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    pouts, _ = part.partition(dcols, n)
    outs, out_starts = dfd.PartialReduceExec(ctx, [0], [-1] + state_ops).reduce(pouts, n, part.part_starts_device_ptr(), N)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    try:
        ex.setup_window(64 << 20)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], N), uuid.uuid4(), 1, 1, 1)
        wcols, ss, sc = node.shuffle_partitioned(ex, outs, out_starts)
        assert np.array_equal(sc[:, 0], np.diff(out_starts))
        dest = orc.partition_ids([key], n, N)
        for q in range(N):
            rows = np.nonzero(dest == q)[0]
            a, cnt = int(ss[q, 0]), int(sc[q, 0])
            present = np.unique(gid[rows])
            assert cnt == len(present)
            got = []
            for c, wc in zip(cols, wcols):
                w = width(c)
                buf = np.empty(cnt * w, dtype=np.uint8)
                nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, buf.ctypes.data, wc.values + a * w, buf.nbytes))
                v = buf.view(np.int64 if c.ndim == 2 else c.dtype)
                got.append(v.reshape(cnt, 2) if c.ndim == 2 else v)
            got_gid = got[0] // 1_000_003
            assert np.array_equal(np.sort(got_gid), present)
            g = gid[rows]
            order = np.argsort(g, kind="stable")
            seg = np.searchsorted(g[order], present)
            for j, op in enumerate(state_ops):
                want = np_merge(OP_TYPE[op], op, states[j][rows], order, seg)
                assert got[j + 1][np.argsort(got_gid)].tobytes() == want.tobytes(), (q, op)
    finally:
        ex.close()


def test_refusals(ctx):
    """Statuses of the calls the new ops refuse, each returned before any kernel runs: a state column of the wrong width,
    an op past the enum, a 128-bit output not 16-byte aligned, a 2-byte state at an odd address, and a nullable state."""
    n = 1000
    gid = np.arange(n) % 10
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    key = torch.from_numpy(gid.astype(np.int64)).cuda()

    def call(state, op, out_shift=0, validity=None):
        t = torch.from_numpy(state).cuda()
        w = 16 if state.ndim == 2 else state.dtype.itemsize
        sc = dfd.DeviceColumn(nv.COL_FIXED, w, t.data_ptr(), length=n, keep=t, validity=validity.data_ptr() if validity is not None else 0)
        ko = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        so = torch.full((n * w + 32,), FILL, dtype=torch.uint8, device="cuda")
        outs = [dfd.DeviceColumn.from_torch(ko), dfd.DeviceColumn(nv.COL_FIXED, w, so.data_ptr() + out_shift, length=n, keep=so)]
        before = ctx.metrics()["kernel_launches"]
        with pytest.raises(dfd.DfdError) as ei:
            dfd.PartialReduceExec(ctx, [0], [-1, op]).reduce([dfd.DeviceColumn.from_torch(key), sc], n, starts.data_ptr(), 1, outs)
        assert ctx.metrics()["kernel_launches"] == before
        torch.cuda.synchronize()
        assert bool((so == FILL).all()) and bool((ko == -1).all())
        return ei.value.status, ei.value.message

    i64, i32 = np.arange(n, dtype=np.int64), np.arange(n, dtype=np.int32)
    dec = np.zeros((n, 2), dtype=np.int64)
    assert call(i64, nv.AGG_MIN_I32)[0] == ERR_INVALID_ARGUMENT  # 8-byte column, 4-byte op
    assert call(i32, nv.AGG_MIN_U64)[0] == ERR_INVALID_ARGUMENT
    assert call(np.arange(n, dtype=np.int16), nv.AGG_MAX_I8)[0] == ERR_INVALID_ARGUMENT
    assert call(i64, nv.AGG_MAX_I128)[0] == ERR_INVALID_ARGUMENT
    assert call(dec, nv.AGG_MIN_I64)[0] == ERR_INVALID_ARGUMENT
    assert call(i64, nv.AGG_SUM_I128)[0] == ERR_INVALID_ARGUMENT  # (as before this op table grew)
    for op in (27, 100):
        st, msg = call(i64, op)
        assert st == ERR_INVALID_ARGUMENT and "does not match" in msg, msg
    for shift in (8, 4, 1):
        st, msg = call(dec, nv.AGG_MIN_I128, out_shift=shift)
        assert st == ERR_INVALID_ARGUMENT and "aligned" in msg, msg
    st, msg = call(np.arange(n, dtype=np.uint16), nv.AGG_MIN_U16, out_shift=1)
    assert st == ERR_INVALID_ARGUMENT and "aligned" in msg, msg
    validity = torch.full(((n + 7) // 8,), 0xFF, dtype=torch.uint8, device="cuda")
    st, msg = call(i32, nv.AGG_MAX_I32, validity=validity)
    assert st == ERR_UNSUPPORTED and "non-null" in msg, msg
