"""GPU parity tests of the device PartialReduce (dfd_reduce.cu: k_group_insert, k_group_count, k_group_place,
k_group_combine) past one grid pass, at its argument limits and at the group table's 2^31- and 2^32-slot sizes.

The row kernels (insert, combine) stride over the rows and the slot kernels (count, place) over the table's slots, with a
grid of CTAS_PER_SM CTAs of BLOCK threads per SM; both constants are parsed out of dfd_reduce.cu and the SM count comes
from the device, so G, the threads of one grid pass, is the launch's own.  Every case asserts the passes or the limit it
is there to reach, and compares every output row with the exact reference of test_reduce_gpu.py (integer states exact,
float MIN / MAX bitwise, float SUM within the summation bound), or bit for bit where the order of a float sum cannot
change its result.  Every call also checks what the reduce leaves alone: output bytes past out_part_starts[N] and guard
bytes past each column's capacity keep their fill, and the call counts 4 kernel launches (none when there are no rows).

The 2^31- and 2^32-slot cases build keys and states on the device from a closed form whose per-group results are
arithmetic series; each runs on its own WorkerContext and skips, naming the memory it needs and the memory that is free,
when the device has too little."""
import gc
import os
import re
from collections import Counter

import numpy as np
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from tests.test_reduce_gpu import check_state, exact_reduce, group_states, make_partial_agg_table
from tests.util import REDUCE_HASH_SEED, ROOT, keys_on_slot, reduce_slot_of_i64_key, reduce_table_slots

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

REDUCE_SRC = os.path.join(ROOT, "datafusion_distributed_b200", "csrc", "dfd_reduce.cu")
KERNELS = ("k_group_insert", "k_group_count", "k_group_place", "k_group_combine")
# the state columns of group_states, in order (the second SUM_I64 column is a COUNT state)
STATE_OPS = [nv.AGG_SUM_I64, nv.AGG_SUM_I64, nv.AGG_MIN_I64, nv.AGG_MAX_I64, nv.AGG_SUM_F64, nv.AGG_MIN_F64, nv.AGG_MAX_F64,
             nv.AGG_SUM_I128]
MAX_KEYS, MAX_REDUCE_COLS = 8, 32  # dfd_internal.h / dfd_reduce.cu
ERR_INVALID_ARGUMENT = 1
FILL, GUARD = 0xA5, 64  # every output column starts as FILL bytes, with GUARD more of them past its capacity
GiB = 1 << 30
MIX_C1, MIX_C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53  # dfd_reduce.cu mix64


def _launch_geometry():
    """(CTAs per SM, threads per CTA) of the four reduce launches, read from dfd_reduce.cu."""
    with open(REDUCE_SRC) as f:
        src = f.read()
    m = re.search(r"const\s+unsigned\s+grid\s*=\s*\(unsigned\)\s*\(\s*c->sm_count\s*\*\s*(\d+)\s*\)\s*;", src)
    assert m, "dfd_reduce.cu: the grid size `(unsigned)(c->sm_count * K)` of dfd_partial_reduce_device was not found"
    blocks = {k: re.findall(rf"\b{k}<<<\s*grid\s*,\s*(\d+)\s*,", src) for k in KERNELS}
    bounds = {k: re.findall(rf"__launch_bounds__\((\d+)\)\s*{k}\b", src) for k in KERNELS}
    assert all(len(v) == 1 for v in blocks.values()), f"dfd_reduce.cu: one <<<grid, BLOCK>>> launch per kernel expected, found {blocks}"
    assert all(len(v) == 1 for v in bounds.values()), f"dfd_reduce.cu: one __launch_bounds__ per kernel expected, found {bounds}"
    sizes = {int(v[0]) for v in blocks.values()} | {int(v[0]) for v in bounds.values()}
    assert len(sizes) == 1, f"dfd_reduce.cu: the four kernels launch with different block sizes {blocks} {bounds}"
    return int(m.group(1)), sizes.pop()


CTAS_PER_SM, BLOCK = _launch_geometry()


def grid_threads():
    """G: the threads of one grid pass of every reduce kernel on device 0."""
    return torch.cuda.get_device_properties(0).multi_processor_count * CTAS_PER_SM * BLOCK


def passes(items):
    """Grid-stride passes a kernel makes over `items` rows or slots."""
    return -(-items // grid_threads())


def report(name, n):
    slots = reduce_table_slots(n)
    print(f"\n[reduce] {name}: n = {n}, {slots} slots, G = {grid_threads()}, row passes {passes(n)}, slot passes {passes(slots)}")


# ------------------------------------------------------------------ harness ----

def width(c):
    return 16 if c.ndim == 2 else c.dtype.itemsize


def as_py(col):
    """A column as the reference's Python values: ints, u64 bit patterns of floats, 128-bit ints (low limb first)."""
    if col.ndim == 2:
        return [(int(hi) << 64) + int(lo) for lo, hi in zip(col[:, 0].view(np.uint64).tolist(), col[:, 1].tolist())]
    if col.dtype == np.float64:
        return col.view(np.uint64).tolist()
    return col.tolist()


def upload_at(cols, offsets, seed):
    """Device columns holding `cols`, column i at Arrow offset offsets[i] behind that many rows of random junk."""
    rng = np.random.Generator(np.random.PCG64(seed))
    dcols = []
    for c, off in zip(cols, offsets):
        w = width(c)
        buf = np.concatenate([rng.integers(0, 256, off * w, dtype=np.uint8), np.ascontiguousarray(c).view(np.uint8).reshape(-1)])
        if buf.size == 0:  # (a zero-element tensor has no storage: give the descriptor a real address)
            buf = np.zeros(w, dtype=np.uint8)
        t = torch.from_numpy(buf).cuda()
        dcols.append(dfd.DeviceColumn(nv.COL_FIXED, w, t.data_ptr(), offset=off, length=len(c), keep=t))
    return dcols


def guarded_outputs(cols, capacity):
    """Output columns of `capacity` rows, every byte FILL, followed by GUARD more FILL bytes."""
    outs = []
    for c in cols:
        t = torch.full((capacity * width(c) + GUARD,), FILL, dtype=torch.uint8, device="cuda")
        outs.append(dfd.DeviceColumn(nv.COL_FIXED, width(c), t.data_ptr(), length=capacity, keep=t))
    return outs


def group_parts(gid, N, seed):
    """Destination partition of every row: each group in one partition chosen at random."""
    rng = np.random.Generator(np.random.PCG64(seed))
    gpart = rng.integers(0, N, int(gid.max()) + 1 if len(gid) else 1)
    return gpart[gid]


def reduce_checked(ctx, cols, n_keys, ops, part, N, offsets=None, seed=0, check=True):
    """Lay the rows out partition by partition (part[r] = partition of row r), reduce them on the device and check:
    - 4 kernel launches (0 without rows), out_part_starts[0] = 0 and non-decreasing;
    - output bytes past row out_part_starts[N] and the guard bytes past the capacity still hold FILL;
    - with `check`, partition p of the output == exact_reduce of the input rows of partition p, one row per key.
    -> (output columns as numpy arrays of out_part_starts[N] rows, out_part_starts)."""
    n = len(part)
    order = np.argsort(part, kind="stable")
    cols, part = [c[order] for c in cols], part[order]
    starts = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(np.bincount(part, minlength=N), out=starts[1:])
    dcols = upload_at(cols, offsets or [0] * len(cols), seed)
    outs = guarded_outputs(cols, n)
    starts_d = torch.from_numpy(starts).cuda()
    torch.cuda.synchronize()
    before = ctx.metrics()["kernel_launches"]
    _, out_starts = dfd.PartialReduceExec(ctx, list(range(n_keys)), ops).reduce(dcols, n, starts_d.data_ptr(), N, outs)
    assert ctx.metrics()["kernel_launches"] - before == (4 if n else 0)
    assert len(out_starts) == N + 1 and out_starts[0] == 0 and bool((np.diff(out_starts) >= 0).all()), out_starts
    total = int(out_starts[-1])
    host = []
    for i, (c, o) in enumerate(zip(cols, outs)):
        raw = o.keep.cpu().numpy()
        w = width(c)
        assert bool((raw[total * w:] == FILL).all()), f"column {i}: bytes past row {total} or past the capacity of {n} rows were written"
        v = raw[:total * w].view(np.int64 if c.ndim == 2 else c.dtype)
        host.append(v.reshape(total, 2) if c.ndim == 2 else v)
    if check:
        check_against_reference(host, out_starts, cols, n_keys, ops, part)
    return host, out_starts


def check_against_reference(host, out_starts, cols, n_keys, ops, part):
    """Every output row is one key of its partition with that key's exact merged states; every key is in one row."""
    N, total = len(out_starts) - 1, int(out_starts[-1])
    # the partition is the leading key: one exact_reduce over all rows yields every partition's groups
    want = exact_reduce([part.astype(np.int64)] + cols, n_keys + 1, [-1] + ops, np.arange(len(part)))
    per_part = Counter(k[0] for k in want)
    assert [int(out_starts[p + 1] - out_starts[p]) for p in range(N)] == [per_part.get(p, 0) for p in range(N)]
    assert total == len(want)
    p_of_row = (np.searchsorted(out_starts, np.arange(total), side="right") - 1).tolist()
    vals = [as_py(h) for h in host]
    sops = [op for op in ops if op >= 0]
    seen = set()
    for r in range(total):
        k = (p_of_row[r],) + tuple(vals[j][r] for j in range(n_keys))
        assert k in want and k not in seen, (r, k)
        seen.add(k)
        for j, op in enumerate(sops):
            check_state(op, vals[n_keys + j][r], want[k][j], k)


def table_case(n, n_groups, seed, N, key_kind="mixed"):
    cols, n_keys, gid = make_partial_agg_table(n, n_groups, seed, key_kind)
    return cols, n_keys, [-1] * n_keys + STATE_OPS, group_parts(gid, N, seed + 1)


# ------------------------------------------------------------------ 1: launch geometry ----

def test_launch_geometry_from_the_source():
    """The constants every pass count below derives from; G is one grid pass of threads on this device."""
    assert CTAS_PER_SM >= 1 and BLOCK % 32 == 0, (CTAS_PER_SM, BLOCK)
    assert grid_threads() >= BLOCK * CTAS_PER_SM
    print(f"\n[reduce] {CTAS_PER_SM} CTAs of {BLOCK} threads per SM, G = {grid_threads()}")


# ------------------------------------------------------------------ 2: grid passes ----

def test_row_kernels_loop_three_passes(ctx):
    """2G + 7 rows in ~n/4 groups: k_group_insert and k_group_combine make three passes, the slot kernels more."""
    n = 2 * grid_threads() + 7
    assert passes(n) == 3 and passes(reduce_table_slots(n)) >= 3
    report("rows past two grid passes", n)
    cols, n_keys, ops, part = table_case(n, n // 4, 21, 16)
    reduce_checked(ctx, cols, n_keys, ops, part, 16)


def test_slot_kernels_loop_while_row_kernels_do_not(ctx):
    """n = G rows (one pass of insert / combine) in a table of >= 2G slots: k_group_count and k_group_place must loop to
    count and place the groups whose slots lie past the first pass."""
    n = grid_threads()
    slots = reduce_table_slots(n)
    assert passes(n) == 1 and passes(slots) >= 2
    report("few rows, many slots", n)
    cols, n_keys, ops, part = table_case(n, n // 2, 22, 8)
    reduce_checked(ctx, cols, n_keys, ops, part, 8)


def _pow2_above_grid():
    return 1 << grid_threads().bit_length()  # the smallest power of two above G


# row counts at the 64-slot minimum and either side of the load factor 1/2 edges (2^k: the first power of two above G)
TABLE_EDGES = ["0", "1", "31", "32", "33", "2^k", "2^k+1"]


@pytest.mark.parametrize("label", TABLE_EDGES)
def test_table_size_edges(ctx, label):
    """The table has max(64, next power of two >= 2n) slots: n = 0 launches nothing, n <= 32 uses the 64-slot minimum,
    33 doubles it to 128, and 2^k / 2^k + 1 rows for the first 2^k above G sit either side of a doubling (2^(k+1) and
    2^(k+2) slots), with two row passes."""
    k2 = _pow2_above_grid()
    n, slots = {"0": (0, 64), "1": (1, 64), "31": (31, 64), "32": (32, 64), "33": (33, 128),
                "2^k": (k2, 2 * k2), "2^k+1": (k2 + 1, 4 * k2)}[label]
    assert reduce_table_slots(n) == slots
    if n > grid_threads():
        assert passes(n) == 2 and passes(slots) >= 4
    report(f"table edge {label}", n)
    cols, n_keys, ops, part = table_case(n, max(1, n // 3), 23, 4)
    _, out_starts = reduce_checked(ctx, cols, n_keys, ops, part, 4)
    if n == 0:
        assert list(out_starts) == [0] * 5


# ------------------------------------------------------------------ 3: probe chains under contention ----

def test_probe_chains_under_contention_past_one_pass(ctx):
    """Two clusters of 2000 distinct keys, each cluster homed on one slot: the table's last slot (its chain wraps to slot
    0) and the middle one.  Every key repeats hundreds of times in random order, so many threads race the same CAS and
    walk the same chain, over more than G rows.  Each key must come out in exactly one row with exact states."""
    per_cluster = 2000
    reps = max(100, grid_threads() // (2 * per_cluster) + 1)
    n = 2 * per_cluster * reps
    slots = reduce_table_slots(n)
    assert n > grid_threads() and passes(n) >= 2
    report("probe chains under contention", n)
    keys = np.concatenate([keys_on_slot(per_cluster, slots - 1, slots, seed=31), keys_on_slot(per_cluster, slots // 2, slots, seed=32)])
    assert len(np.unique(keys)) == 2 * per_cluster
    assert {reduce_slot_of_i64_key(int(k), slots) for k in keys} == {slots - 1, slots // 2}
    rng = np.random.Generator(np.random.PCG64(33))
    gid = rng.permutation(np.repeat(np.arange(2 * per_cluster), reps))
    cols = [keys[gid]] + group_states(gid, rng)
    host, out_starts = reduce_checked(ctx, cols, 1, [-1] + STATE_OPS, group_parts(gid, 3, 34), 3)
    assert int(out_starts[-1]) == 2 * per_cluster
    assert sorted(host[0].tolist()) == sorted(keys.tolist())


# ------------------------------------------------------------------ 4: argument limits ----

KEY_WIDTHS = (1, 2, 4, 8, 16, 1, 2, 4)


def eight_keys(n_base, seed):
    """Group keys of widths KEY_WIDTHS for 9 * n_base groups: base tuples, and for each base and each key k a neighbour
    that differs from it in key k alone (for the 16-byte key, in its high limb alone).  So only all eight keys together
    tell every group apart.  -> list of 8 per-group key arrays (16 bytes: (groups, 2) int64, low limb first)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    u64 = lambda size: rng.integers(0, (1 << 64) - 1, size, dtype=np.uint64, endpoint=True)
    keys = []
    for k, w in enumerate(KEY_WIDTHS):
        mask = np.uint64((1 << min(64, 8 * w)) - 1)
        lo = np.repeat(u64(n_base) & mask, 9)
        hi = np.repeat(u64(n_base), 9)
        delta = rng.integers(1, int(mask), n_base, dtype=np.uint64, endpoint=True)  # nonzero mod 2^(8w)
        if w == 16:
            hi[k + 1::9] = hi[k + 1::9] + delta
            keys.append(np.stack([lo.view(np.int64), hi.view(np.int64)], axis=1))
        else:
            lo[k + 1::9] = (lo[k + 1::9] + delta) & mask
            keys.append(lo.astype({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[w]).view({1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}[w]))
    return keys


def np_mix64(x):
    for c in (MIX_C1, MIX_C2, None):
        x = x ^ (x >> np.uint64(33))
        if c is not None:
            x = x * np.uint64(c)
    return x


def np_key_hash(keys):
    """dfd_reduce.cu's key_hash of every row of the key columns (narrow keys are read zero-extended)."""
    h = np.full(len(keys[0]), REDUCE_HASH_SEED, dtype=np.uint64)
    for k in keys:
        if k.ndim == 2:
            h = np_mix64(np_mix64(h ^ k[:, 0].view(np.uint64)) ^ k[:, 1].view(np.uint64))
        else:
            h = np_mix64(h ^ k.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[k.dtype.itemsize]).astype(np.uint64))
    return h


def one_chain(gkeys, base, slots, count, seed):
    """`count` groups equal to group `base` in keys 0..6 whose key 7 (4 bytes) puts them on base's home slot: they all
    probe one chain, and only the last key tells them apart.  -> the 8 key arrays with these groups appended."""
    mask = np.uint64(0xFFFFFFFF & (slots - 1))
    target = np_key_hash([k[base:base + 1] for k in gkeys])[0] & mask
    h7 = np_key_hash([k[base:base + 1] for k in gkeys[:7]])[0]  # key_hash after the seven shared keys
    cand = np.random.Generator(np.random.PCG64(seed)).integers(0, 1 << 32, 1 << 23, dtype=np.uint64)
    hits = np.unique(cand[(np_mix64(h7 ^ cand) & mask) == target])
    hits = hits[hits != gkeys[7][base:base + 1].view(np.uint32).astype(np.uint64)[0]][:count]
    assert len(hits) == count, len(hits)
    out = [np.concatenate([k, np.repeat(k[base:base + 1], count, axis=0)]) for k in gkeys[:7]]
    return out + [np.concatenate([gkeys[7], hits.astype(np.uint32).view(np.int32)])]


def test_eight_keys_and_thirty_two_columns(ctx):
    """MAX_KEYS = 8 group keys of widths 1, 2, 4, 8, 16, 1, 2, 4, which no proper subset of tells the groups apart, and
    24 state columns (every op, three times, each with its own values): exactly MAX_REDUCE_COLS = 32 columns, reduced
    exactly.  Besides, 48 groups share the first seven keys and the home slot of one group, so every insert of theirs
    compares all eight keys along one probe chain.  9 keys, or 33 columns, are DFD_ERR_INVALID_ARGUMENT before any
    launch."""
    n_base, n = 600, 40_000
    slots = reduce_table_slots(n)
    gkeys = one_chain(eight_keys(n_base, 41), 0, slots, 48, 45)
    n_groups = 9 * n_base + 48
    chain = [np.concatenate([k[:1], k[-48:]]) for k in gkeys]  # group 0 and the 48 on its home slot
    assert len({int(h) & (slots - 1) for h in np_key_hash(chain) & np.uint64(0xFFFFFFFF)}) == 1
    tuples = [tuple(map(tuple, k.reshape(n_groups, -1).tolist())) for k in gkeys]
    rows_of = lambda subset: list(zip(*(tuples[k] for k in subset)))
    assert len(set(rows_of(range(MAX_KEYS)))) == n_groups
    for k in range(MAX_KEYS):  # every 7 keys (so every proper subset) merge some groups
        assert len(set(rows_of([j for j in range(MAX_KEYS) if j != k]))) < n_groups, k
    rng = np.random.Generator(np.random.PCG64(42))
    gid = rng.permutation(np.concatenate([np.arange(n_groups), rng.integers(0, n_groups, n - n_groups)]))
    keys = [k[gid] for k in gkeys]
    states = group_states(gid, rng) + group_states(gid, rng) + group_states(gid, rng)
    ops = [-1] * MAX_KEYS + STATE_OPS * 3
    cols = keys + states
    assert len(cols) == MAX_REDUCE_COLS and len(keys) == MAX_KEYS

    # refused: 9 keys in 32 columns, and 8 keys in 33 columns
    part = group_parts(gid, 5, 43)
    starts = torch.from_numpy(np.array([0, n], dtype=np.int64)).cuda()
    extra_key = np.zeros(n, dtype=np.int32)
    extra_state = np.ones(n, dtype=np.int64)
    refused = [(keys + [extra_key] + states[:-1], list(range(MAX_KEYS + 1)), [-1] * (MAX_KEYS + 1) + ops[MAX_KEYS:-1]),
               (cols + [extra_state], list(range(MAX_KEYS)), ops + [nv.AGG_SUM_I64])]
    before = ctx.metrics()["kernel_launches"]
    for rcols, key_cols, rops in refused:
        assert len(rcols) == len(rops)
        dcols = upload_at(rcols, [0] * len(rcols), 44)
        with pytest.raises(dfd.DfdError) as e:
            dfd.PartialReduceExec(ctx, key_cols, rops).reduce(dcols, n, starts.data_ptr(), 1, guarded_outputs(rcols, n))
        assert e.value.status == ERR_INVALID_ARGUMENT, (len(key_cols), len(rcols), e.value)
    assert ctx.metrics()["kernel_launches"] == before

    report("8 keys x 32 columns", n)
    _, out_starts = reduce_checked(ctx, cols, MAX_KEYS, ops, part, 5)
    assert int(out_starts[-1]) == n_groups


# ------------------------------------------------------------------ 5: per-column offsets ----

OFFSETS = {  # 13 columns of the "multi" key kind (widths 1, 2, 4, 8, 16) + the 8 states, every column at its own offset;
    # column 0 at the smallest one; the 16-byte key (column 4) and the SUM_I128 state (column 12) at odd offsets
    "col0_at_0": [0, 1, 3, 7, 13, 2, 5, 9, 11, 17, 19, 23, 29],
    "col0_at_1": [1, 30, 14, 6, 3, 21, 8, 2, 27, 12, 4, 18, 9],
}


@pytest.mark.parametrize("case", list(OFFSETS))
def test_every_column_at_its_own_offset(ctx, case):
    offsets = OFFSETS[case]
    cols, n_keys, ops, part = table_case(50_001, 2_000, 51, 6, "multi")
    assert len(offsets) == len(cols) == 13 and len(set(offsets)) == 13 and min(offsets) == offsets[0]
    assert cols[4].ndim == 2 and offsets[4] % 2 == 1 and ops[12] == nv.AGG_SUM_I128 and offsets[12] % 2 == 1
    reduce_checked(ctx, cols, n_keys, ops, part, 6, offsets=offsets, seed=52)


# ------------------------------------------------------------------ 6: partition counts ----

def test_partition_counts(ctx):
    """N = 1; N = 4096 with only partitions 0, 1, 2047, 4094 and 4095 holding groups; N = 65 537 (not a power of two, above
    the partitioner's limit: partition_of's binary search takes 17 steps) with the first and last partitions filled."""
    n, n_groups = 60_000, 20_000
    cols, n_keys, gid = make_partial_agg_table(n, n_groups, 61)
    ops = [-1] * n_keys + STATE_OPS
    rng = np.random.Generator(np.random.PCG64(62))
    cases = {
        1: np.zeros(n_groups, dtype=np.int64),
        4096: np.array([0, 1, 2047, 4094, 4095])[rng.integers(0, 5, n_groups)],
        65_537: rng.integers(0, 65_537, n_groups),
    }
    cases[65_537][gid[0]] = 0
    cases[65_537][gid[gid != gid[0]][0]] = 65_536
    for N, gpart in cases.items():
        _, out_starts = reduce_checked(ctx, cols, n_keys, ops, gpart[gid], N, seed=N)
        sizes = np.diff(out_starts)
        assert sizes[0] > 0 and sizes[-1] > 0
        if N == 4096:
            assert set(np.nonzero(sizes)[0].tolist()) == {0, 1, 2047, 4094, 4095}


# ------------------------------------------------------------------ 7: bitwise float sums ----

def f64_bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def test_float_sums_bitwise_where_order_cannot_matter(ctx):
    """SUM_F64 groups whose IEEE result is the same in every order, compared bit for bit.  The sum starts from +0.0:
    - one-row groups: the row's value, except that -0.0 gives +0.0 (+0.0 + -0.0);
    - two-row groups: (+0.0 + a) + b = a + b, rounded once, whichever row comes first;
    - groups of small integers (|x| <= 2^20, at most 2000 rows): every partial sum is exact;
    - thousands of rows of only -0.0, only +0.0, and both: +0.0."""
    rng = np.random.Generator(np.random.PCG64(71))
    vals, gids, want = [], [], {}

    def add_group(v, expect):
        g = len(want)
        want[g] = int(f64_bits(expect))
        vals.append(np.asarray(v, dtype=np.float64))
        gids.append(np.full(len(v), g))

    singles = np.concatenate([rng.standard_normal(1500) * 10.0 ** rng.integers(-300, 300, 1500),
                              [5e-324, -5e-324, 2.2e-308, -1.7976931348623157e308, np.inf, -np.inf, 0.0, -0.0, -0.0]])
    for x in singles.tolist():
        add_group([x], np.float64(0.0) + x)
    for _ in range(2000):
        a, b = rng.standard_normal(2) * 10.0 ** rng.integers(-8, 8, 2)
        add_group(rng.permutation([a, b]), (np.float64(0.0) + a) + b)
    for _ in range(300):
        v = rng.integers(-(1 << 20), 1 << 20, int(rng.integers(1, 2000)), endpoint=True)
        add_group(v.astype(np.float64), float(int(v.sum())))
    add_group(np.full(5000, -0.0), 0.0)
    add_group(np.full(5000, 0.0), 0.0)
    add_group(rng.permutation(np.repeat([-0.0, 0.0], 2500)), 0.0)
    add_group(rng.permutation(np.array([3.0, -3.0] * 2000)), 0.0)  # an exact zero from opposite signs is +0.0

    perm = rng.permutation(sum(len(v) for v in vals))
    f, gid = np.concatenate(vals)[perm], np.concatenate(gids)[perm]
    key = (gid.astype(np.int64) * 0x9E3779B97F4A7C1) ^ 0x55
    n = len(gid)
    assert n > grid_threads()
    report("bitwise float sums", n)
    host, out_starts = reduce_checked(ctx, [key, f], 1, [-1, nv.AGG_SUM_F64], group_parts(gid, 4, 72), 4, check=False)
    assert int(out_starts[-1]) == len(want)
    g_of_key = dict(zip(key.tolist(), gid.tolist()))
    for k, bits in zip(host[0].tolist(), host[1].view(np.uint64).tolist()):
        g = g_of_key[k]
        assert bits == want[g], (g, hex(bits), hex(want[g]))


def test_sum_i128_every_add_carries(ctx):
    """Every low limb is 2^64 - 1, so every 128-bit add but a group's first carries into the high limb, in one group of
    more than G rows (and a second, smaller one)."""
    big = grid_threads() + 12_345
    n = big + 5_000
    rng = np.random.Generator(np.random.PCG64(81))
    gid = rng.permutation(np.concatenate([np.zeros(big, dtype=np.int64), np.ones(n - big, dtype=np.int64)]))
    dec = np.stack([np.full(n, -1, dtype=np.int64), rng.integers(-3, 3, n, dtype=np.int64, endpoint=True)], axis=1)
    key = gid * 7 + 1
    assert passes(n) == 2
    report("SUM_I128 carries", n)
    host, _ = reduce_checked(ctx, [key, dec], 1, [-1, nv.AGG_SUM_I128], np.zeros(n, dtype=np.int64), 1)
    for k, v in zip(host[0].tolist(), as_py(host[1])):
        rows = gid == (k - 1) // 7
        want = (int(rows.sum()) * ((1 << 64) - 1) + (int(dec[rows, 1].sum()) << 64)) % (1 << 128)
        assert v % (1 << 128) == want, (k, v, want)


# ------------------------------------------------------------------ 8: what the call leaves alone ----

def test_large_small_large_on_one_context(built):
    """One context reduces a large, a small, an empty and another large table: its scratch (table, slot_out, row_slot)
    is reused, and nothing of an earlier call leaks into a later one.  reduce_checked checks the launches (4 per call
    with rows, 0 without) and the FILL bytes past each result."""
    c = dfd.WorkerContext(0)
    try:
        n_large = 2 * grid_threads() + 7
        for n, n_groups, seed in ((n_large, n_large // 3, 91), (1_000, 50, 92), (0, 1, 93), (n_large, n_large // 50, 94)):
            cols, n_keys, ops, part = table_case(n, n_groups, seed, 7, "w8")
            reduce_checked(c, cols, n_keys, ops, part, 7)
    finally:
        c.close()


# ------------------------------------------------------------------ 9: the big tables ----

SEED_I64 = REDUCE_HASH_SEED - (1 << 64)  # key_hash's seed and mix64's multipliers as int64 bit patterns
C1_I64, C2_I64 = MIX_C1 - (1 << 64), MIX_C2 - (1 << 64)
LOW31 = (1 << 31) - 1
GROUP_BITS = 20
A_MULT = 0x2545F491  # row i is in group (i * A_MULT) mod 2^20 (A odd: a bijection of the low 20 bits)
CHUNK = 1 << 27


def home_slots(u, mask):
    """dfd_reduce.cu's home slot of 4-byte keys (an int64 tensor of their uint32 values): mix64(seed ^ key) & mask."""
    x = u ^ SEED_I64
    x = x ^ ((x >> 33) & LOW31)  # (logical shifts of the 64-bit pattern)
    x = x * C1_I64
    x = x ^ ((x >> 33) & LOW31)
    x = x * C2_I64
    x = x ^ ((x >> 33) & LOW31)
    return x & mask


def tail_keys(slots, tail):
    """Every 4-byte key whose home is one of the table's last `tail` slots (a search of all 2^32 keys on the device)."""
    found = []
    for a in range(0, 1 << 32, CHUNK):
        u = torch.arange(a, a + CHUNK, dtype=torch.int64, device="cuda")
        found.append(u[home_slots(u, slots - 1) >= slots - tail])
        del u
    return torch.cat(found).cpu().numpy()


def wrapped_keys(homes, slots):
    """How many keys linear probing stores past the table's last slot (so, wrapped to slot 0 on): the same for every
    insertion order, since the set of occupied slots is.  Key i in home order ends at i + max_(j<=i)(home_j - j)."""
    h = np.sort(homes)
    i = np.arange(len(h), dtype=np.int64)
    return int((i + np.maximum.accumulate(h - i) >= slots).sum())


@pytest.mark.parametrize("n", [(1 << 29) + 1, (1 << 30) + 1], ids=["2^31_slots", "2^32_slots"])
def test_big_tables(built, n):
    """n = 2^29 + 1 rows hash into 2^31 slots (slot indices up to INT32_MAX), n = 2^30 + 1 into 2^32 slots (the mask is
    all 32 bits and (s + 1) & mask wraps at 2^32).  One Int32 key, SUM / COUNT / MIN / MAX i64 states: row i is in group
    g = (i * A) mod 2^20 and its state is i, so group g holds rows r_g + 2^20 t (r_g = g / A mod 2^20) and its states are
    arithmetic series.  The key of g comes from a table of 2^20 distinct keys that holds every key homed in the table's
    last slots, enough that some probe chains wrap to slot 0.  Partitions 0 and 2 of 3 are empty."""
    slots = reduce_table_slots(n)
    assert slots == 4 * (n - 1) and slots in (1 << 31, 1 << 32)
    G_ = 1 << GROUP_BITS
    need = (20 * n + 2 * 4 * slots + 4 * n) / GiB + 1  # inputs (key, i, ones), table + slot_out + row_slot, outputs and temporaries
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < (need + 2) * GiB:
        pytest.skip(f"{slots}-slot table: needs {need + 2:.0f} GiB of free device memory, {free / GiB:.1f} GiB is free")
    print(f"\n[reduce] big table: n = {n}, {slots} slots, {free / GiB:.1f} GiB free, row passes {passes(n)}, slot passes {passes(slots)}")

    # 2^20 distinct keys: every key homed in the last slots, then a bijective image of 0, 1, 2, ... for the rest
    tail = tail_keys(slots, 4096 if slots == 1 << 32 else 2048)
    torch.cuda.empty_cache()
    rest = (np.arange(G_ + len(tail), dtype=np.uint64) * np.uint64(0x9E3779B1) ^ np.uint64(0x7F4A7C15)) & np.uint64(0xFFFFFFFF)
    rest = rest[~np.isin(rest, tail.astype(np.uint64))][:G_ - len(tail)]
    lut = np.random.Generator(np.random.PCG64(101)).permutation(np.concatenate([tail.astype(np.uint64), rest]))
    assert len(lut) == G_ and len(np.unique(lut)) == G_
    homes = home_slots(torch.from_numpy(lut.astype(np.int64)).cuda(), slots - 1).cpu().numpy()
    for u in lut[:64].tolist() + tail[:16].tolist():  # the device restatement agrees with tests/util.py's
        assert reduce_slot_of_i64_key(u, slots) == int(homes[np.nonzero(lut == u)[0][0]])
    wrapped = wrapped_keys(homes, slots)
    assert wrapped >= 1
    if slots == 1 << 32:
        assert bool((homes > 0x7FFFFFFF).any())  # slot indices past INT32_MAX
    print(f"[reduce] {len(tail)} keys homed in the last slots, {wrapped} of them wrap past slot {slots - 1}")

    c = dfd.WorkerContext(0)
    try:
        lut_d = torch.from_numpy(lut.astype(np.uint32).view(np.int32)).cuda()
        idx = torch.arange(n, dtype=torch.int64, device="cuda")  # the state of row i is i
        key = torch.empty(n, dtype=torch.int32, device="cuda")
        for a in range(0, n, CHUNK):
            key[a:a + CHUNK] = lut_d[(idx[a:a + CHUNK] * A_MULT) & (G_ - 1)]
        ones = torch.ones(n, dtype=torch.int64, device="cuda")
        torch.cuda.empty_cache()  # (the generation temporaries: the reduce allocates its scratch outside torch)
        cols = [dfd.DeviceColumn.from_torch(t) for t in (key, idx, ones, idx, idx)]
        ops = [-1, nv.AGG_SUM_I64, nv.AGG_SUM_I64, nv.AGG_MIN_I64, nv.AGG_MAX_I64]
        # outputs of G_ rows and one guard row: the reduce writes rows [0, groups) only
        outs = [torch.full((G_ + 1,), -0x5A5A5A5A5A5A5A5B if w == 8 else -0x5A5A5A5B, dtype=torch.int64 if w == 8 else torch.int32, device="cuda")
                for w in (4, 8, 8, 8, 8)]
        starts = torch.tensor([0, 0, n, n], dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        _, out_starts = dfd.PartialReduceExec(c, [0], ops).reduce(cols, n, starts.data_ptr(), 3, [dfd.DeviceColumn.from_torch(t) for t in outs])
        assert list(out_starts) == [0, 0, G_, G_]
        got = [t.cpu().numpy() for t in outs]
        del cols, key, idx, ones, outs, starts, lut_d
    finally:
        c.close()
        gc.collect()
        torch.cuda.empty_cache()

    assert got[0][G_] == np.int32(-0x5A5A5A5B) and all(g[G_] == -0x5A5A5A5A5A5A5A5B for g in got[1:])
    order = np.argsort(lut)
    pos = np.searchsorted(lut[order], got[0][:G_].view(np.uint32).astype(np.uint64))
    g = order[np.minimum(pos, G_ - 1)]
    assert np.array_equal(lut[g], got[0][:G_].view(np.uint32).astype(np.uint64)), "an output key is no input key"
    assert len(np.unique(g)) == G_
    r = (g.astype(np.int64) * pow(A_MULT, -1, G_)) % G_  # first row of group g
    t = (n - 1 - r) // G_ + 1                             # its rows: r, r + 2^20, ..., r + 2^20 (t - 1)
    assert np.array_equal(got[2][:G_], t), "COUNT"
    assert np.array_equal(got[1][:G_], t * r + G_ * (t * (t - 1) // 2)), "SUM"
    assert np.array_equal(got[3][:G_], r), "MIN"
    assert np.array_equal(got[4][:G_], r + G_ * (t - 1)), "MAX"
