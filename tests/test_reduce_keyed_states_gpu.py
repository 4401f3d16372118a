"""GPU parity tests of the device PartialReduce's keyed kernels with every aggregate op and nullable states.

A call with a Boolean, Utf8, LargeUtf8 or Binary key runs k_insert_keys, k_count_keys and k_place_keys: template
instantiations over KeyParams with their own fixed-width key hash (mix_fixed), their own null-key compare and their own
copy of the state seeds, MIN / MAX sentinels and output bits of k_place_nullable.  The other PartialReduce modules run
every op, nullable state and fixed key width through the fixed-key kernels only; this one runs them through the keyed
kernels:
- all 27 ops under each keyed kind, nullable or not, at null fractions 0, 0.3, 0.97 and 1 (and with no input bitmap
  but nullable outputs), garbage under every null (all ones, the op's sentinel, a NaN, random bits);
- MIN / MAX groups whose one valid row is the first, the last or a random row, that hold the sentinel itself, or that
  have no valid row (k_place_keys seeds the sentinel for a null representative, k_group_clear zeroes what is left);
- fixed keys of 1, 2, 4, 8 and 16 bytes beside a Utf8 or a Boolean key, in families that differ only in the last
  byte (16 bytes: only in the second half, or by swapped halves), and the same rows reduced by the fixed keys alone
  (the fixed-key kernels) and with a constant Boolean key added (the keyed kernels): the results must be equal;
- KeyParams at its largest (8 keys of every kind, 24 states, every column at its own Arrow offset), run twice;
- 1- and 2-byte MIN / MAX outputs at every base address mod 4 beside a Utf8 key;
- more rows than one grid pass (read from the device), at N = 1, 7 and 64, as singleton groups and as one hot group.

The reference is plain Python: keys as bytes / bool / int / None, integer and Decimal128 states as exact ints, float
MIN / MAX by totalOrder over bit patterns, float SUM over small integers as their exact sum (every partial sum is exact
in any order).  Every call checks states and bitmaps bit for bit (zero bytes under every null key and state), the guard
bytes in front of and behind every output buffer, the bitmap words past G, out_part_starts and the launch count (4, +1
for k_group_clear, +4 per var-width key).  A child process asserts from torch.profiler that the module's cases
launched k_insert_keys, k_count_keys, k_place_keys, k_group_combine, k_combine_nullable and k_group_clear.

One H100 80GB HBM3 at 700 W: the module's 84 cases take about 75 s, 21 s of it in the child process, with at most about
1.3 GiB of device memory in use."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from tests.test_reduce_gpu import check_state, merge, py_values
from tests.test_reduce_keys_gpu import call_reduce, layout, random_strings, read_column, upload_key
from tests.test_reduce_keys_gpu import guarded_output as key_output
from tests.test_reduce_limits_gpu import grid_threads
from tests.test_reduce_nulls_cpu import ALL_OPS, MINMAX_OPS
from tests.test_reduce_nulls_gpu import group_valid, guarded_output, lone_valid_states, read_output, state_values, upload, width, with_nulls
from tests.test_reduce_ops_gpu import OP_TYPE, py_merge
from tests.test_reduce_ops_gpu import py_values as typed_py_values

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
VAR_KINDS = ("utf8", "large", "binary")
KEYED_KINDS = ("bool",) + VAR_KINDS
PROFILE_CHILD = "DFD_TEST_KEYED_STATES_PROFILE"  # set in the child process that records the kernels


# ------------------------------------------------------------------ reference ----

def state_py(op, col):
    """A state column as the reference's Python values (ints; float bit patterns; signed 128-bit ints; SUM_F64: the
    floats, which state_values makes small integers)."""
    if op == nv.AGG_SUM_F64:
        return col.tolist()
    return typed_py_values(OP_TYPE[op], col) if op in OP_TYPE else py_values(col)


def merge_state(op, xs):
    if op == nv.AGG_SUM_F64:  # exact: the sum of integers below 2^53, from +0.0
        return float(sum(int(x) for x in xs)) + 0.0
    return py_merge(OP_TYPE[op], op, xs) if op in OP_TYPE else merge(op, xs)


def check_merged(op, got, want, where):
    if op == nv.AGG_SUM_F64:
        assert got.hex() == want.hex(), (where, op, got, want)  # (bitwise: +0.0 and -0.0 differ)
    elif op in OP_TYPE:
        assert got == want, (where, op, got, want)
    else:
        check_state(op, got, want, where)


# ------------------------------------------------------------------ columns ----

def fixed_key_column(w, values, rng):
    """Python ints (None: null) as the column of a w-byte key (their little-endian bytes; 16 bytes: (n, 2) int64), with
    garbage under the nulls.  -> (column, valid)"""
    raw = np.frombuffer(b"".join((v or 0).to_bytes(w, "little") for v in values), dtype=np.uint8).reshape(len(values), w)
    col = raw.view(np.int64) if w == 16 else raw.view(f"u{w}").reshape(-1)
    valid = np.array([v is not None for v in values], dtype=bool)
    return with_nulls(col.copy(), valid, None, rng), valid


def expected_launches(n, kinds, ops, valids):
    if n == 0:
        return 0
    clear = any(v is not None and op in MINMAX_OPS for op, v in zip(ops, valids))
    return 4 + clear + 4 * sum(k in VAR_KINDS for k in kinds)


def reduce_keyed(ctx, keys, states, ops, N=1, seed=0, key_offsets=None, state_offsets=None, value_shifts=None, out_nullable=None):
    """Reduce rows whose key columns are `keys` and whose state columns are `states` and check every output.

    keys: [(kind, Python values, nullable)], kind "bool", "utf8", "large", "binary" or the width of a fixed key;
    states: [(column, valid or None)], merged by `ops`.  Rows with equal key tuples are one group, each group in one
    random partition.  Input column i sits at its Arrow offset (var-width keys also behind a nonzero first offset, their
    bytes at an address that varies with it), output state j at value_shifts[j] bytes past an aligned address.
    -> (out_part_starts, {(partition,) + key tuple: ((bit, bytes) of every state)})"""
    rng = np.random.Generator(np.random.PCG64(seed))
    n = len(keys[0][1])
    ids = {}
    gid = np.array([ids.setdefault(t, len(ids)) for t in zip(*(k[1] for k in keys))], dtype=np.int64)
    order, starts = layout(None, gid, N, rng)
    keys = [(kind, [vals[i] for i in order], nl) for kind, vals, nl in keys]
    states = [(c[order], v[order] if v is not None else None) for c, v in states]
    part = np.repeat(np.arange(N), np.diff(starts))
    key_offsets = key_offsets or [0] * len(keys)
    state_offsets = state_offsets or [0] * len(states)
    value_shifts = value_shifts or [0] * len(states)
    out_nullable = [v is not None for _, v in states] if out_nullable is None else out_nullable

    ins, outs = [], []
    for (kind, vals, nl), off in zip(keys, key_offsets):
        assert nl or None not in vals
        if isinstance(kind, str):
            ins.append(upload_key(kind, vals, rng, arrow_off=off, first_off=3 * off % 11, addr=off % 8, validity=nl))
            outs.append(key_output(ins[-1], n, nullable=nl))
        else:
            col, valid = fixed_key_column(kind, vals, rng)
            ins.append(upload(col, valid if nl else None, off, rng))
            outs.append(guarded_output(kind, n, nl))
    for (c, v), off, shift, nl in zip(states, state_offsets, value_shifts, out_nullable):
        ins.append(upload(c, v, off, rng))
        outs.append(guarded_output(width(c), n, nl, value_shift=shift))
    dev_outs = [o if isinstance(o, dfd.DeviceColumn) else o[0] for o in outs]
    rc, out_starts, launches = call_reduce(ctx, ins, dev_outs, len(keys), N, starts, [-1] * len(keys) + list(ops))
    assert rc == 0, nv.lib().dfd_last_error()
    assert launches == expected_launches(n, [k[0] for k in keys], ops, [v for _, v in states]), launches
    assert out_starts[0] == 0 and bool((np.diff(out_starts) >= 0).all()), out_starts
    G = int(out_starts[N])

    got_keys = []
    for (kind, _, _), o in zip(keys, outs[:len(keys)]):
        if isinstance(kind, str):
            got_keys.append(read_column(o, n, G))
            continue
        vals, bits = read_output(o[1], o[2], kind, G, f"{kind}-byte key")
        bits = np.ones(G, dtype=bool) if bits is None else bits
        assert not vals[~bits].any(), "a null key's bytes are not zero"
        b, bits = vals.tobytes(), bits.tolist()
        got_keys.append([int.from_bytes(b[r * kind:(r + 1) * kind], "little") if bits[r] else None for r in range(G)])
    got = []
    for j, (op, (c, _), o, shift) in enumerate(zip(ops, states, outs[len(keys):], value_shifts)):
        vals, bits = read_output(o[1], o[2], width(c), G, f"state {j} (op {op})", shift)
        bits = np.ones(G, dtype=bool) if bits is None else bits
        assert not vals[~bits].any(), (j, op, "a null state's bytes are not zero")
        col = vals.copy().reshape(-1).view(c.dtype)
        got.append((state_py(op, col.reshape(G, 2) if c.ndim == 2 else col), bits.tolist(), vals.tobytes(), width(c)))

    rows_of = {}
    for r, t in enumerate(zip(part.tolist(), *(k[1] for k in keys))):  # (the reference's groups)
        rows_of.setdefault(t, []).append(r)
    assert G == len(rows_of), (G, len(rows_of))
    in_vals = [state_py(op, c) for op, (c, _) in zip(ops, states)]
    in_valid = [v.tolist() if v is not None else [True] * n for _, v in states]
    p_of_row = (np.searchsorted(out_starts, np.arange(G), side="right") - 1).tolist()
    result = {}
    for r in range(G):
        key = (p_of_row[r],) + tuple(k[r] for k in got_keys)
        assert key in rows_of and key not in result, ("a group is missing from the input or appears twice", key)
        for j, op in enumerate(ops):
            xs = [in_vals[j][i] for i in rows_of[key] if in_valid[j][i]]
            assert got[j][1][r] == bool(xs), (key, j, op, "validity")
            if xs:
                check_merged(op, got[j][0][r], merge_state(op, xs), (key, j))
        result[key] = tuple((bits[r], b[r * w:(r + 1) * w]) for _, bits, b, w in got)
    return out_starts, result


def nullable_states(ops, n, rng, frac):
    """A column of each op with garbage under its nulls (`frac` of the rows at random; None: no bitmap)."""
    valids = [group_valid(rng, n, frac) if frac is not None else None for _ in ops]
    return [(with_nulls(state_values(op, n, rng), v, op, rng), v) for op, v in zip(ops, valids)]


def keyed_values(kind, gid, rng, null_every=0):
    """Key values of a keyed kind for group ids `gid`: Booleans (gid odd), or a distinct string per id (the id and ':'
    before 0-37 random bytes).  Every group id = 3 mod null_every has a null key."""
    top = int(gid.max()) + 1
    if kind == "bool":
        pool = [bool(g % 2) for g in range(top)]
    else:
        pool = [b"%d:" % g + s for g, s in enumerate(random_strings(rng, top, list(range(0, 38))))]
    if null_every:
        pool = [None if g % null_every == 3 else v for g, v in enumerate(pool)]
    return [pool[g] for g in gid.tolist()]


# ------------------------------------------------------------------- tests ----

@pytest.mark.parametrize("frac", [None, 0.0, 0.3, 0.97, 1.0], ids=["no_bitmap", "0", "0.3", "0.97", "1"])
@pytest.mark.parametrize("nullable", [False, True], ids=["keys", "null_keys"])
@pytest.mark.parametrize("kind", KEYED_KINDS)
def test_every_op_under_every_keyed_kind(ctx, kind, nullable, frac):
    """All 27 ops in one call under one Boolean or var-width key (with null keys or without), over 4 000 rows in 4
    partitions: every state column with a bitmap and the given share of nulls, or (no_bitmap) none, with outputs that
    are nullable all the same, so every output bit comes from k_place_keys.  The keys of `bool` make 2-3 groups of
    ~1 300 rows, the others ~400 groups of ~10."""
    seed = 1000 * KEYED_KINDS.index(kind) + 100 * nullable + int((frac if frac is not None else 2.0) * 100)
    rng = np.random.Generator(np.random.PCG64(seed))
    n = 4000
    gid = rng.integers(0, 400, n)
    keys = [(kind, keyed_values(kind, gid, rng, 7 if nullable else 0), nullable)]
    reduce_keyed(ctx, keys, nullable_states(ALL_OPS, n, rng, frac), ALL_OPS, N=4, seed=seed, out_nullable=[True] * len(ALL_OPS))


@pytest.mark.parametrize("kind", ["utf8", "binary"])
def test_lone_valid_rows_and_sentinels_under_a_string_key(ctx, kind):
    """Every MIN / MAX op, F16 / F32 / F64 specials among the values (+-0, +-inf, NaNs of both signs and several
    payloads): in 1 500 groups of 40 rows, one valid row that is the first, the last or a random row of its group (so
    the representative is mostly null and k_place_keys seeds the sentinel), valid rows that all hold the op's sentinel,
    the sentinel among other values, or no valid row (k_group_clear zeroes the state and leaves its bit clear).  Every
    50th group has a null key (those groups are one)."""
    rng = np.random.Generator(np.random.PCG64(20 + len(kind)))
    gid, states, valids = lone_valid_states(1500, 40, rng)
    keys = [(kind, keyed_values(kind, gid, rng, 50), True)]
    reduce_keyed(ctx, keys, list(zip(states, valids)), MINMAX_OPS, N=3, seed=21)


def fixed_families(w, n_base, rng):
    """Distinct w-byte key values (Python ints, little-endian) in families that are equal in every byte but the last;
    16 bytes: equal in the first 8-byte half and different in the second, plus each base with its halves swapped."""
    out = set()
    while len(out) < n_base * 4:
        base = int(rng.integers(0, 1 << 63)) | int(rng.integers(0, 2)) << 63
        if w == 16:
            lo, hi = base, int(rng.integers(0, 1 << 63)) | 1 << 63
            out |= {lo | hi << 64, lo | ((hi + 1) & M64) << 64, lo | (hi ^ 1 << 40) << 64, hi | lo << 64}
        else:
            base &= (1 << 8 * (w - 1)) - 1
            out |= {base | int(v) << 8 * (w - 1) for v in rng.choice(256, 4, replace=False)}
    return sorted(out)


FIXED_KEY_OPS = [nv.AGG_SUM_I64, nv.AGG_MIN_I32, nv.AGG_MAX_F64, nv.AGG_SUM_I128, nv.AGG_MIN_U8, nv.AGG_MAX_I16, nv.AGG_MIN_F16]


def fixed_key_rows(w, nullable, rng, n=6000):
    """n rows of a w-byte key from fixed_families (10 % null when nullable) and states of FIXED_KEY_OPS, 30 % null."""
    vals = fixed_families(w, 16, rng)
    fixed = [vals[i] for i in rng.integers(0, len(vals), n)]
    if nullable:
        fixed = [None if rng.random() < 0.1 else v for v in fixed]
    return fixed, nullable_states(FIXED_KEY_OPS, n, rng, 0.3)


@pytest.mark.parametrize("nullable", [False, True], ids=["keys", "null_keys"])
@pytest.mark.parametrize("companion", ["utf8", "bool"])
@pytest.mark.parametrize("w", [1, 2, 4, 8, 16])
def test_fixed_key_of_every_width_beside_a_keyed_one(ctx, w, companion, nullable):
    """A 1-, 2-, 4-, 8- or 16-byte key whose values differ only in the last byte (16 bytes: in the second half alone, or
    by swapped halves) beside a Utf8 key of 4 values (after it) or a Boolean key (before it), both nullable or not."""
    rng = np.random.Generator(np.random.PCG64(300 + 10 * w + 2 * nullable + (companion == "bool")))
    fixed, states = fixed_key_rows(w, nullable, rng)
    n = len(fixed)
    pool = [b"", b"a", b"a\x00", b"longer than eight bytes"] + ([None] if nullable else [])
    other = [pool[i] for i in rng.integers(0, len(pool), n)] if companion == "utf8" else \
        [None if nullable and i == 2 else bool(i) for i in rng.integers(0, 3 if nullable else 2, n)]
    keys = [(w, fixed, nullable), ("utf8", other, nullable)] if companion == "utf8" else [("bool", other, nullable), (w, fixed, nullable)]
    reduce_keyed(ctx, keys, states, FIXED_KEY_OPS, N=5, seed=301, key_offsets=[3, 5])


@pytest.mark.parametrize("nullable", [False, True], ids=["keys", "null_keys"])
@pytest.mark.parametrize("w", [1, 2, 4, 8, 16])
def test_fixed_keys_alone_and_with_a_constant_boolean_key_agree(ctx, w, nullable):
    """The same rows reduced by a w-byte key and an 8-byte key (the fixed-key kernels), and by the same keys and a
    constant non-null Boolean key (the keyed kernels): both match the reference and hold the same (key, states) rows in
    every partition, bit for bit."""
    rng = np.random.Generator(np.random.PCG64(400 + 10 * w + nullable))
    fixed, states = fixed_key_rows(w, nullable, rng)
    n = len(fixed)
    second = [int(x) << 56 for x in rng.integers(0, 2, n)]
    keys = [(w, fixed, nullable), (8, second, False)]
    _, alone = reduce_keyed(ctx, keys, states, FIXED_KEY_OPS, N=5, seed=401)
    _, keyed = reduce_keyed(ctx, keys + [("bool", [True] * n, False)], states, FIXED_KEY_OPS, N=5, seed=401)
    assert {k + (True,): v for k, v in alone.items()} == keyed


# 24 states: every op but MAX_I16, MAX_U64 and MIN_U8, so every family (SUM, MIN / MAX of every width, signed, unsigned,
# float and Decimal128) is there
LARGEST_OPS = [op for op in ALL_OPS if op not in (nv.AGG_MAX_I16, nv.AGG_MAX_U64, nv.AGG_MIN_U8)]


def test_eight_keys_of_every_kind_and_twenty_four_states(ctx):
    """KeyParams at its largest: 8 keys (Utf8, LargeUtf8, Binary, Boolean and fixed keys of 1, 2, 8 and 16 bytes, five
    of them nullable) and 24 states, every third without a bitmap: 32 columns, each at its own Arrow offset.  Two runs
    on the same input give the same bytes and bits in every group."""
    assert len(LARGEST_OPS) == 24
    rng = np.random.Generator(np.random.PCG64(50))
    n, g = 30_000, 3_000
    gid = rng.integers(0, g, n)
    spec = [("utf8", True), ("large", False), ("binary", True), ("bool", True), (1, False), (2, True), (8, False), (16, True)]
    keys = []
    for kind, nl in spec:  # few values per key, drawn per group: only all eight keys tell most groups apart
        if kind == "bool":
            pool = [False, True]
        elif isinstance(kind, str):
            pool = random_strings(rng, 3, [0, 1, 7, 8, 9, 30])
        else:
            pool = fixed_families(kind, 1, rng)[:3]
        per_group = [pool[i] for i in rng.integers(0, len(pool), g)]
        if nl:
            per_group = [None if rng.random() < 0.15 else v for v in per_group]
        keys.append((kind, [per_group[i] for i in gid.tolist()], nl))
    states = nullable_states(LARGEST_OPS, n, rng, 0.35)
    states = [(c, None if j % 3 == 2 else v) for j, (c, v) in enumerate(states)]
    offsets = rng.permutation(np.arange(1, 40))[:32].tolist()
    runs = [reduce_keyed(ctx, keys, states, LARGEST_OPS, N=5, seed=51, key_offsets=offsets[:8], state_offsets=offsets[8:])[1] for _ in range(2)]
    assert len(runs[0]) > g // 2
    assert runs[0] == runs[1], "two runs on the same input differ"


NARROW_OPS = [nv.AGG_MIN_I8, nv.AGG_MAX_I8, nv.AGG_MIN_U8, nv.AGG_MAX_U8, nv.AGG_MIN_I16, nv.AGG_MAX_I16, nv.AGG_MIN_U16,
              nv.AGG_MAX_U16, nv.AGG_MIN_F16, nv.AGG_MAX_F16]


@pytest.mark.parametrize("base", [0, 1, 2, 3])
def test_narrow_states_at_every_base_beside_a_string_key(ctx, base):
    """1-byte MIN / MAX outputs at address `base` mod 4 and 2-byte ones at base & 2 (all a 2-byte value can have),
    beside a Utf8 key: 20 000 groups, so the neighbouring bytes of a word are other groups' states updated at the same
    moment; half the columns nullable.  The guard bytes around every column keep their fill."""
    rng = np.random.Generator(np.random.PCG64(60 + base))
    n = 60_000
    gid = rng.integers(0, 20_000, n)
    keys = [("utf8", keyed_values("utf8", gid, rng, 97), True)]
    states = nullable_states(NARROW_OPS, n, rng, 0.4)
    states = [(c, v if j % 2 else None) for j, (c, v) in enumerate(states)]
    shifts = [base if width(c) == 1 else base & 2 for c, _ in states]
    reduce_keyed(ctx, keys, states, NARROW_OPS, N=4, seed=61, state_offsets=[1, 3, 2, 5, 1, 3, 7, 2, 6, 4], value_shifts=shifts)


GRID_OPS = [nv.AGG_SUM_I64, nv.AGG_SUM_F64, nv.AGG_MIN_I8, nv.AGG_MAX_F16, nv.AGG_MIN_I128, nv.AGG_MAX_F64, nv.AGG_MAX_U32, nv.AGG_SUM_I128]


@pytest.mark.parametrize("N", [1, 7, 64])
@pytest.mark.parametrize("shape", ["every_row_its_own_group", "one_hot_group"])
def test_past_one_grid_pass(ctx, shape, N):
    """G + 4 099 rows (G: the threads of one grid pass, sm_count x 8 x 256 with sm_count read from the device), each its
    own group under a LargeUtf8 key, or all in one group under one Utf8 key (every row's insert compares bytes with one
    representative and every state's CAS loop contends on one address); states half null, one without a bitmap."""
    n = grid_threads() + 4099
    need = n * 400 + (256 << 20)  # inputs, guarded outputs and the reduce's scratch, generously
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB is free")
    rng = np.random.Generator(np.random.PCG64(70 + N))
    if shape == "one_hot_group":
        keys = [("utf8", [b"the one hot key of every row"] * n, False)]
    else:
        keys = [("large", [b"%d/" % r + bytes([r % 251]) * (r % 13) for r in rng.permutation(n).tolist()], False)]
    states = nullable_states(GRID_OPS, n, rng, 0.5)
    states[0] = (states[0][0], None)
    _, result = reduce_keyed(ctx, keys, states, GRID_OPS, N=N, seed=71)
    assert len(result) == (1 if shape == "one_hot_group" else n)


KERNELS = ("k_insert_keys", "k_count_keys", "k_place_keys", "k_group_combine", "k_combine_nullable", "k_group_clear")


def test_the_keyed_kernels_ran(ctx):
    """A child process (a profiler session of its own: kernel records of a long-running test process can stop) runs
    cases of this module with and without state bitmaps and asserts from torch.profiler's records that they launched
    each of KERNELS."""
    if not os.environ.get(PROFILE_CHILD):
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
            "-m", "pytest", os.path.abspath(__file__), "-q", "-p", "no:cacheprovider", "-k", "test_the_keyed_kernels_ran"]
        r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **{PROFILE_CHILD: "1"}), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]
        return
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        test_every_op_under_every_keyed_kind(ctx, "utf8", True, 0.3)  # k_combine_nullable, k_group_clear
        test_every_op_under_every_keyed_kind(ctx, "bool", False, None)  # k_group_combine
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    ran = {k for k in KERNELS if any(re.search(rf"\b{k}\b", name) for name in names)}
    assert ran == set(KERNELS), f"not launched: {sorted(set(KERNELS) - ran)}"
