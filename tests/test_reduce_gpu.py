"""GPU parity tests of the device-side PartialReduce (dfd_partial_reduce_device) against an exact CPU reduce of the same
partitioned rows.

- SUM / COUNT over i64 wrap mod 2^64 and SUM over 128-bit decimals wraps mod 2^128, like the device's two's-complement
  atomics (Python-int sums, wrapped).  MIN / MAX over i64 are exact.
- Float MIN / MAX follow IEEE 754 totalOrder, the order arrow-rs gives floats (f64::total_cmp): -NaN < -inf < ... < -0.0
  < +0.0 < ... < +inf < +NaN, NaNs by payload.  Results are compared bitwise.
- Float SUM adds in atomics order.  It is compared with math.fsum within the error bound of recursive summation in any
  order, |got - exact| <= gamma(m - 1) * sum|x| for a group of m rows.  Groups holding inf or NaN have one IEEE answer in
  any order (NaN if a NaN or both infinities are present, else the infinity) and are compared exactly."""
import math
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.util import keys_on_slot, reduce_slot_of_i64_key, reduce_table_slots

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
# every dfd_agg_op once (the second SUM_I64 column is a COUNT state)
STATE_OPS = [nv.AGG_SUM_I64, nv.AGG_SUM_I64, nv.AGG_MIN_I64, nv.AGG_MAX_I64, nv.AGG_SUM_F64, nv.AGG_MIN_F64, nv.AGG_MAX_F64,
             nv.AGG_SUM_I128]
OPS = [-1, -1] + STATE_OPS  # two group keys first
# quiet / signalling, positive / negative NaNs with different payloads
NAN_BITS = [0x7FF8000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF, 0xFFF8000000000000,
            0xFFF0000000000001]
SPECIAL_BITS = NAN_BITS + [0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000]  # +-0, +-inf


# ------------------------------------------------------------------ inputs ----

def group_keys(kind, gid, rng):
    """Group-key columns of the rows of group ids `gid`: equal ids <-> equal keys.  A 16-byte key is an (n, 2) int64
    array (low limb first).  Multi-key kinds use columns that are not injective on their own, so only the whole key
    tells groups apart."""
    g = gid.astype(np.int64)
    top = int(g.max()) + 1 if len(g) else 1
    if kind == "mixed":  # Int64 + Int32, the Partial aggregate's usual keys
        return [g * 1_000_003, (g % 7).astype(np.int32)]
    if kind in ("w1", "w2", "w4", "w8"):
        w = int(kind[1])
        dt = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[w]
        # distinct values spread over the whole range (for 8 bytes: distinct high 62 bits, random low 2 bits)
        u = rng.choice(1 << min(8 * w, 62), top, replace=False).astype(np.uint64)
        if w == 8:
            u = (u << np.uint64(2)) | rng.integers(0, 4, top, dtype=np.uint64)
        return [u.astype({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[w]).view(dt)[g]]
    if kind == "w16":  # pairs of groups share the low limb: the high limb must be compared too
        lo = rng.choice(1 << 62, (top + 1) // 2, replace=False).astype(np.int64) - (1 << 61)
        hi = rng.integers(I64_MIN, I64_MAX, top, dtype=np.int64, endpoint=True)
        return [np.stack([lo[g // 2], hi[g]], axis=1)]
    if kind == "multi":  # widths 1, 2, 4, 8, 16 in one key; (g // 2, g % 251) is the only injective combination
        k16 = np.stack([g // 5, (g // 5) % 3], axis=1)
        return [(g % 251).astype(np.uint8), ((g // 3) % 30011).astype(np.int16), (g // 7).astype(np.int32), (g // 2) * 7, k16]
    raise ValueError(kind)


def group_states(gid, rng):
    """The eight state columns of STATE_OPS.  i64 states near +-2^62 and at INT64_MIN / INT64_MAX make the sums wrap.
    Floats are standard normals except in some groups: 1 only NaNs, 2 only +-0.0, 3 only -0.0, 4 some -inf, 6 some
    +inf and -inf, and every eighth group sprinkled with NaNs, zeros and infinities."""
    n = len(gid)
    pick = rng.integers(0, 8, n)
    big = rng.integers(1 << 62, I64_MAX, n, dtype=np.int64, endpoint=True)
    s = np.where(pick < 3, big, np.where(pick < 6, -big, rng.integers(-1000, 1000, n, dtype=np.int64)))
    s[pick == 6] = I64_MIN
    s[pick == 7] = I64_MAX
    cnt = rng.integers(1, 100, n, dtype=np.int64)
    mn = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    mx = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    mn[rng.random(n) < 0.01] = I64_MIN
    mx[rng.random(n) < 0.01] = I64_MAX
    fb = rng.standard_normal(n).view(np.uint64)
    nan_b, spec_b = np.array(NAN_BITS, dtype=np.uint64), np.array(SPECIAL_BITS, dtype=np.uint64)
    fb = np.where(gid == 1, nan_b[rng.integers(0, len(nan_b), n)], fb)
    fb = np.where(gid == 2, spec_b[rng.integers(len(NAN_BITS), len(NAN_BITS) + 2, n)], fb)
    fb = np.where(gid == 3, np.uint64(0x8000000000000000), fb)
    fb = np.where((gid == 4) & (rng.random(n) < 0.1), np.uint64(0xFFF0000000000000), fb)  # -inf among finite values
    fb = np.where((gid == 6) & (rng.random(n) < 0.1), spec_b[rng.integers(len(spec_b) - 2, len(spec_b), n)], fb)  # +inf and -inf
    sprinkle = (gid % 8 == 5) & (rng.random(n) < 0.3)
    fb = np.where(sprinkle, spec_b[rng.integers(0, len(spec_b), n)], fb)
    f = fb.view(np.float64)
    dec = np.zeros((n, 2), dtype=np.int64)
    dec[:, 0] = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)  # every low-limb add may carry
    dec[:, 1] = np.where(rng.random(n) < 0.5, rng.integers(-5, 5, n, dtype=np.int64), s)  # high limbs that wrap too
    return [s, cnt, mn, mx, f, f.copy(), f.copy(), dec]


def make_partial_agg_table(n, n_groups, seed, key_kind="mixed", gid=None):
    """The output of a Partial aggregate: group keys of `key_kind` + the states of STATE_OPS.  -> (columns, n_keys, gid)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    if gid is None:
        gid = rng.integers(0, n_groups, n)
    keys = group_keys(key_kind, gid, rng)
    return keys + group_states(gid, rng), len(keys), gid


# --------------------------------------------------------- exact reference ----

def wrap(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def total_order_key(bits):
    """IEEE 754 totalOrder as a signed integer (the usual monotone map of the f64 bit pattern)."""
    s = wrap(bits, 64)
    return s ^ ((s >> 63) & 0x7FFF_FFFF_FFFF_FFFF)


def gamma(k):
    u = 2.0 ** -53
    return k * u / (1 - k * u)


def py_values(col):
    """A column as Python values: ints (i64 / smaller), u64 bit patterns (f64), 128-bit ints (low limb first)."""
    if col.ndim == 2:
        return [(int(hi) << 64) + int(lo) for lo, hi in zip(col[:, 0].view(np.uint64).tolist(), col[:, 1].tolist())]
    if col.dtype == np.float64:
        return col.view(np.uint64).tolist()
    return col.tolist()


def key_tuple(vals, n_keys, r):
    return tuple(vals[k][r] for k in range(n_keys))


def merge(op, xs):
    """The exact merged state of one group (xs = its rows' Python values)."""
    if op == nv.AGG_SUM_I64:
        return wrap(sum(xs), 64)
    if op == nv.AGG_SUM_I128:
        return sum(xs) % (1 << 128)
    if op == nv.AGG_MIN_I64:
        return min(xs)
    if op == nv.AGG_MAX_I64:
        return max(xs)
    if op in (nv.AGG_MIN_F64, nv.AGG_MAX_F64):
        return (min if op == nv.AGG_MIN_F64 else max)(xs, key=total_order_key)
    fs = np.array(xs, dtype=np.uint64).view(np.float64)
    nan, pinf, ninf = bool(np.isnan(fs).any()), bool((fs == np.inf).any()), bool((fs == -np.inf).any())
    if nan or (pinf and ninf):
        return ("nan",)
    if pinf or ninf:
        return ("exact", math.inf if pinf else -math.inf)
    fl = fs.tolist()
    return ("bound", math.fsum(fl), math.fsum(abs(x) for x in fl), len(fl))


def exact_reduce(cols, n_keys, ops, rows):
    """{key tuple: [merged state of every state column]} of the given rows, in plain Python."""
    vals = [py_values(c[rows]) for c in cols]
    groups = {}
    for r in range(len(rows)):
        groups.setdefault(key_tuple(vals, n_keys, r), []).append(r)
    return {k: [merge(op, [vals[c][r] for r in rs]) for c, op in enumerate(ops) if op >= 0] for k, rs in groups.items()}


def check_state(op, got, want, ctx_msg):
    if op in (nv.AGG_MIN_F64, nv.AGG_MAX_F64):  # bitwise
        assert got == want, (ctx_msg, op, hex(got), hex(want))
    elif op == nv.AGG_SUM_F64:
        g = float(np.array([got], dtype=np.uint64).view(np.float64)[0])
        if want[0] == "nan":
            assert math.isnan(g), (ctx_msg, g)
        elif want[0] == "exact":
            assert g == want[1], (ctx_msg, g, want[1])
        else:
            _, fs, sabs, m = want
            # fsum is the exact sum rounded once: allow that half ulp on top of the summation bound
            assert abs(g - fs) <= gamma(m - 1) * sabs + 0.5 * math.ulp(fs), (ctx_msg, g, fs, m)
    elif op == nv.AGG_SUM_I128:
        assert got % (1 << 128) == want, (ctx_msg, op, got, want)
    else:
        assert got == want, (ctx_msg, op, got, want)


# ------------------------------------------------------------- device i/o ----

def upload(ctx, cols, offset=0):
    """Device columns holding `cols` at Arrow offset `offset` (that many junk rows in front)."""
    import torch

    rng = np.random.Generator(np.random.PCG64(offset))
    keep, dcols = [], []
    for c in cols:
        pad = rng.integers(0, 255, (offset,) + c.shape[1:], dtype=np.uint8).astype(c.dtype) if offset else c[:0]
        full = np.concatenate([pad, c])
        if full.shape[0] == 0:  # (a zero-element torch tensor has no storage: give the descriptor a real address)
            full = np.zeros((1,) + c.shape[1:], dtype=c.dtype)
        t = torch.from_numpy(np.ascontiguousarray(full)).cuda()
        keep.append(t)
        width = 16 if c.ndim == 2 else c.dtype.itemsize
        dcols.append(dfd.DeviceColumn(nv.COL_FIXED, width, t.data_ptr(), offset=offset, length=c.shape[0], keep=t))
    torch.cuda.synchronize()
    return dcols, keep


def download(ctx, col, rows, dtype, width_elems=1):
    out = np.empty(rows * width_elems, dtype=dtype)
    if rows:
        nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, out.ctypes.data, col.values, out.nbytes))
    return out.reshape(rows, width_elems) if width_elems > 1 else out


def check_reduced(ctx, outs, out_starts, cols, n_keys, ops, part_rows):
    """Partition p of the device output == exact_reduce of the input rows part_rows[p], key for key, bit for bit."""
    total = int(out_starts[-1])
    host = [py_values(download(ctx, outs[i], total, c.dtype, 2 if c.ndim == 2 else 1)) for i, c in enumerate(cols)]
    sops = [op for op in ops if op >= 0]
    for p, rows in enumerate(part_rows):
        want = exact_reduce(cols, n_keys, ops, rows)
        a, b = int(out_starts[p]), int(out_starts[p + 1])
        assert b - a == len(want), (p, b - a, len(want))
        seen = set()
        for r in range(a, b):
            k = key_tuple(host, n_keys, r)
            assert k in want and k not in seen, (p, k)
            seen.add(k)
            for j, op in enumerate(sops):
                check_state(op, host[n_keys + j][r], want[k][j], (p, k))


def reduce_prepartitioned(ctx, cols, n_keys, ops, gid, N, seed, offset=0):
    """Lay the rows out as a partitioned table (every group in one partition, chosen at random, so some partitions may
    be empty), reduce it on the device at Arrow offset `offset`, and check it against the exact reference."""
    import torch

    n = len(gid)
    rng = np.random.Generator(np.random.PCG64(seed))
    gpart = rng.integers(0, N, int(gid.max()) + 1 if n else 1)
    dest = gpart[gid]
    order = np.argsort(dest, kind="stable")
    cols = [c[order] for c in cols]
    starts = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(np.bincount(dest, minlength=N), out=starts[1:])
    dcols, _keep = upload(ctx, cols, offset)
    starts_d = torch.from_numpy(starts).cuda()
    torch.cuda.synchronize()
    outs, out_starts = dfd.PartialReduceExec(ctx, list(range(n_keys)), ops).reduce(dcols, n, starts_d.data_ptr(), N)
    check_reduced(ctx, outs, out_starts, cols, n_keys, ops, [np.arange(starts[p], starts[p + 1]) for p in range(N)])
    return outs, out_starts


# ------------------------------------------------------------------- tests ----

@pytest.mark.parametrize("n,n_groups,N", [(0, 1, 4), (1, 1, 1), (5_000, 17, 8), (200_003, 5_000, 12), (300_000, 250_000, 48)])
def test_partial_reduce_matches_cpu_group_by(ctx, n, n_groups, N):
    """Repartition on the device, then reduce: the partitioner's part_starts drive the reduce."""
    cols, n_keys, _ = make_partial_agg_table(n, n_groups, 11)
    dcols, _keep = upload(ctx, cols)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1], N))
    pouts, starts = part.partition(dcols, n)
    red = dfd.PartialReduceExec(ctx, [0, 1], OPS)
    outs, out_starts = red.reduce(pouts, n, part.part_starts_device_ptr(), N)
    dest = orc.partition_ids([cols[0], cols[1]], n, N) if n else np.zeros(0, dtype=np.uint32)
    check_reduced(ctx, outs, out_starts, cols, n_keys, OPS, [np.nonzero(dest == p)[0] for p in range(N)])
    assert out_starts[-1] <= n


# (key kind, rows, groups, partitions, Arrow offset)
EXACT_CASES = {
    "key_w1": ("w1", 40_000, 256, 8, 0),
    "key_w2": ("w2", 60_000, 3_000, 8, 0),
    "key_w4": ("w4", 60_000, 3_000, 8, 0),
    "key_w8": ("w8", 60_000, 3_000, 8, 0),
    "key_w16": ("w16", 60_000, 3_000, 8, 0),
    "multi_key_mix": ("multi", 100_000, 20_000, 12, 0),
    "sliced_offset_1": ("mixed", 50_001, 2_000, 6, 1),
    "sliced_offset_13_multi_key": ("multi", 50_001, 2_000, 6, 13),
    "more_partitions_than_groups": ("mixed", 20_000, 5, 64, 0),
    "one_group_holds_every_row": ("w8", 100_000, 1, 4, 0),
}


@pytest.mark.parametrize("case", list(EXACT_CASES))
def test_partial_reduce_exact(ctx, case):
    """All seven aggregate ops at once, against the exact reference, over key widths 1 / 2 / 4 / 8 / 16 and a mix, wrapping
    integer sums, NaN / +-0.0 / +-inf float groups, sliced inputs, empty partitions and a single group."""
    kind, n, n_groups, N, offset = EXACT_CASES[case]
    cols, n_keys, gid = make_partial_agg_table(n, n_groups, 7, kind)
    reduce_prepartitioned(ctx, cols, n_keys, [-1] * n_keys + STATE_OPS, gid, N, 3, offset)


def test_partial_reduce_every_row_its_own_group(ctx):
    n = 100_000
    gid = np.random.Generator(np.random.PCG64(4)).permutation(n)
    cols, n_keys, gid = make_partial_agg_table(n, n, 4, "w8", gid)
    outs, out_starts = reduce_prepartitioned(ctx, cols, n_keys, [-1] + STATE_OPS, gid, 16, 4)
    assert out_starts[-1] == n


def test_partial_reduce_probe_chains_wrap_past_the_table_end(ctx):
    """Thousands of distinct keys whose hashes all land on the table's last slot: every insert walks a long chain that
    wraps to slot 0 and compares keys all along it."""
    n_keys, reps = 3000, 3
    n = n_keys * reps
    slots = reduce_table_slots(n)
    keys = keys_on_slot(n_keys, slots - 1, slots, seed=9)
    assert reduce_slot_of_i64_key(int(keys[0]), slots) == slots - 1
    gid = np.random.Generator(np.random.PCG64(5)).permutation(np.repeat(np.arange(n_keys), reps))
    states = group_states(gid, np.random.Generator(np.random.PCG64(6)))
    cols = [keys[gid]] + states
    outs, out_starts = reduce_prepartitioned(ctx, cols, 1, [-1] + STATE_OPS, gid, 1, 5)
    assert out_starts[-1] == n_keys


def test_partial_reduce_float_min_max_total_order(ctx):
    """Float MIN / MAX merge under IEEE 754 totalOrder, as arrow-rs orders floats (f64::total_cmp): a NaN takes part (a
    +NaN wins MAX, a -NaN wins MIN), an all-NaN group yields one of its own NaNs (never +-inf), -0.0 < +0.0, and the
    result's bits are the same on every run however the rows' atomics interleave."""
    qnan, nan1, snan, nan_max, neg_nan = 0x7FF8000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF, 0xFFF8000000000000
    one, two, three, five = (np.array([x], dtype=np.float64).view(np.uint64)[0].item() for x in (1.0, 2.0, 3.0, 5.0))
    pzero, nzero, pinf, ninf = 0x0, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000
    groups = [  # (values, MIN bits, MAX bits)
        ([one, qnan], one, qnan),
        ([qnan, nan1, snan, nan_max], snan, nan_max),
        ([qnan, nan1, neg_nan], neg_nan, nan1),
        ([nzero, pzero], nzero, pzero),
        ([nzero], nzero, nzero),
        ([pinf, ninf, three], ninf, pinf),
        ([neg_nan, five], neg_nan, five),
        ([two], two, two),
    ]
    copies = 4000  # many rows of each group race on the same state
    rng = np.random.Generator(np.random.PCG64(8))
    gid = np.concatenate([np.full(len(v) * copies, g) for g, (v, _, _) in enumerate(groups)])
    bits = np.concatenate([np.tile(np.array(v, dtype=np.uint64), copies) for v, _, _ in groups])
    perm = rng.permutation(len(gid))
    gid, bits = gid[perm], bits[perm]
    key = (gid * 1_000_003).astype(np.int64)
    f = bits.view(np.float64)
    ops = [-1, nv.AGG_MIN_F64, nv.AGG_MAX_F64]
    for _ in range(3):
        outs, out_starts = reduce_prepartitioned(ctx, [key, f, f.copy()], 1, ops, gid, 2, 1)
        total = int(out_starts[-1])
        got_k = download(ctx, outs[0], total, np.int64)
        got_min = download(ctx, outs[1], total, np.uint64)
        got_max = download(ctx, outs[2], total, np.uint64)
        assert total == len(groups)
        for r in range(total):
            _, want_min, want_max = groups[int(got_k[r]) // 1_000_003]
            assert int(got_min[r]) == want_min, (int(got_k[r]) // 1_000_003, hex(int(got_min[r])), hex(want_min))
            assert int(got_max[r]) == want_max, (int(got_k[r]) // 1_000_003, hex(int(got_max[r])), hex(want_max))


def test_partial_reduce_then_prepartitioned_shuffle(ctx):
    """Partial output -> repartition -> PartialReduce -> exchange, all on the device (world = 1): partition q's single
    segment holds exactly the reduced groups of destination q."""
    n, N = 120_000, 6
    cols, n_keys, _ = make_partial_agg_table(n, 3_000, 5)
    dcols, _keep = upload(ctx, cols)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1], N))
    pouts, _ = part.partition(dcols, n)
    outs, out_starts = dfd.PartialReduceExec(ctx, [0, 1], OPS).reduce(pouts, n, part.part_starts_device_ptr(), N)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(16 << 20)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], N), uuid.uuid4(), 1, 1, 1)
    wcols, ss, sc = node.shuffle_partitioned(ex, outs, out_starts)
    assert np.array_equal(sc[:, 0], np.diff(out_starts))
    dest = orc.partition_ids([cols[0], cols[1]], n, N)
    for q in (0, N - 1):
        want = exact_reduce(cols, n_keys, OPS, np.nonzero(dest == q)[0])
        a, cnt = int(ss[q, 0]), int(sc[q, 0])
        g1 = dfd.NetworkShuffleExec.segment_to_arrow(ctx, dfd.DeviceColumn(nv.COL_FIXED, 8, wcols[0].values, arrow_type=pa.int64()), a, cnt).to_numpy()
        sm = dfd.NetworkShuffleExec.segment_to_arrow(ctx, dfd.DeviceColumn(nv.COL_FIXED, 8, wcols[2].values, arrow_type=pa.int64()), a, cnt).to_numpy()
        g2 = dfd.NetworkShuffleExec.segment_to_arrow(ctx, dfd.DeviceColumn(nv.COL_FIXED, 4, wcols[1].values, arrow_type=pa.int32()), a, cnt).to_numpy()
        assert len(g1) == len(want)
        for i in range(len(g1)):
            assert want[(int(g1[i]), int(g2[i]))][0] == int(sm[i])
    ex.close()


def test_partial_reduce_argument_errors(ctx):
    cols, _, _ = make_partial_agg_table(100, 5, 1)
    dcols, _keep = upload(ctx, cols)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 4))
    pouts, _ = part.partition(dcols, 100)
    with pytest.raises(dfd.DfdError):  # a key column that carries an aggregate
        dfd.PartialReduceExec(ctx, [0, 1], [nv.AGG_SUM_I64] + OPS[1:]).reduce(pouts, 100, part.part_starts_device_ptr(), 4)
    with pytest.raises(dfd.DfdError):  # SUM_I128 on an 8-byte column
        dfd.PartialReduceExec(ctx, [0, 1], OPS[:2] + [nv.AGG_SUM_I128] + OPS[3:]).reduce(pouts, 100, part.part_starts_device_ptr(), 4)
