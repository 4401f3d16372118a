"""GPU tests of the device PartialReduce (dfd_partial_reduce_device) with Boolean, Utf8, LargeUtf8 and Binary group keys,
compared bit for bit with the exact Python group-by of test_reduce_keys_cpu.py.

Output row order inside a partition is unspecified, so each partition is compared as a set of keys, each with its merged
states (COUNT, SUM, MIN and MAX over Int64).  Every output buffer starts as FILL bytes with GUARD more in front of it and
past its capacity, and every call checks what the reduce must leave alone: the bytes in front of every buffer, offsets
past entry G, string bytes past the total, value and validity words past row G (and bits at and past G inside the last
word, which must be zero), fixed-width bytes past row G.  Null keys must come out empty, with their bit clear, whatever
lies under them in the input."""
import ctypes as C
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from datafusion_distributed_b200.device import columns_to_c
from tests.test_reduce_keys_cpu import home_slot, reference_group_by
from tests.util import reduce_table_slots

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

FILL, GUARD = 0xA5, 64
ERR_INVALID, ERR_UNSUPPORTED, ERR_CAPACITY = 1, 6, 7
KIND = {"utf8": nv.COL_UTF8, "large": nv.COL_LARGE_UTF8, "binary": nv.COL_BINARY, "bool": nv.COL_BOOL, "i32": nv.COL_FIXED}
ARROW = {"utf8": pa.string(), "large": pa.large_string(), "binary": pa.binary(), "bool": pa.bool_(), "i32": pa.int32()}
STATE_OPS = [nv.AGG_SUM_I64, nv.AGG_SUM_I64, nv.AGG_MIN_I64, nv.AGG_MAX_I64]
STATE_KINDS = ["count", "sum", "min", "max"]


# ------------------------------------------------------------------ device i/o ----

def cuda_bytes(b: bytes, size=None):
    a = np.full(max(size if size is not None else len(b), 1), FILL, dtype=np.uint8)
    a[:len(b)] = np.frombuffer(b, dtype=np.uint8)
    return torch.from_numpy(a).cuda()


def packbits(bits):
    return np.packbits(np.asarray(bits, dtype=np.uint8), bitorder="little").tobytes() if len(bits) else b""


def upload_key(kind, values, rng, arrow_off=0, first_off=0, addr=0, validity=None):
    """A device input column of `values` (None = null) at Arrow offset `arrow_off` behind that many junk rows.  Var-width:
    the first offset is `first_off` (junk bytes before it) and the bytes start at `addr` mod 8; every null row holds 1-5
    junk bytes, a null Boolean or Int32 a random value.  `validity`: give a bitmap (default: only when a value is None)."""
    n = len(values)
    has_null = any(v is None for v in values)
    use_valid = has_null if validity is None else validity
    valid = [bool(rng.integers(0, 2)) for _ in range(arrow_off)] + [v is not None for v in values]
    keep = []
    vptr = 0
    if use_valid:
        vt = cuda_bytes(packbits(valid) + b"\0" * 8)
        keep.append(vt)
        vptr = vt.data_ptr()
    if kind in ("utf8", "large", "binary"):
        rows = [bytes(rng.integers(0, 256, int(rng.integers(0, 6)), dtype=np.uint8)) for _ in range(arrow_off)]
        rows += [v if v is not None else bytes(rng.integers(0, 256, int(rng.integers(1, 6)), dtype=np.uint8)) for v in values]
        offs = np.zeros(len(rows) + 1, dtype=np.int64 if kind == "large" else np.int32)
        offs[0] = first_off
        offs[1:] = first_off + np.cumsum([len(r) for r in rows])
        data = bytes(rng.integers(0, 256, addr + first_off, dtype=np.uint8)) + b"".join(rows)
        dt = cuda_bytes(data + b"\0" * 16)
        ot = torch.from_numpy(offs).cuda()
        keep += [ot, dt]
        return dfd.DeviceColumn(KIND[kind], 0, dt.data_ptr() + addr, ot.data_ptr(), vptr, arrow_off, n, keep, ARROW[kind], len(data) - addr)
    if kind == "bool":
        bits = [bool(rng.integers(0, 2)) for _ in range(arrow_off)] + [bool(v) if v is not None else bool(rng.integers(0, 2)) for v in values]
        bt = cuda_bytes(packbits(bits) + b"\0" * 8)
        keep.append(bt)
        return dfd.DeviceColumn(nv.COL_BOOL, 0, bt.data_ptr(), 0, vptr, arrow_off, n, keep, pa.bool_())
    a = rng.integers(-(1 << 31), 1 << 31, arrow_off + n, dtype=np.int64).astype(np.int32)
    a[arrow_off:] = [v if v is not None else a[arrow_off + i] for i, v in enumerate(values)]
    t = torch.from_numpy(a).cuda()
    keep.append(t)
    return dfd.DeviceColumn(nv.COL_FIXED, 4, t.data_ptr(), 0, vptr, arrow_off, n, keep, pa.int32())


def upload_state(v):
    t = torch.from_numpy(np.ascontiguousarray(v, dtype=np.int64)).cuda()
    return dfd.DeviceColumn(nv.COL_FIXED, 8, t.data_ptr(), 0, 0, 0, len(v), [t], pa.int64())


def guarded_output(col, n, cap=None, nullable=False):
    """Output column for `col` with n rows of capacity (var-width: `cap` bytes, default the input's), every byte FILL,
    each buffer with GUARD more FILL bytes in front of it and behind it (keep holds the whole buffers)."""
    keep, vptr = [], 0
    words = (n + 31) // 32 * 4

    def buf(size):
        t = cuda_bytes(b"", GUARD + size + GUARD)
        keep.append(t)
        return t.data_ptr() + GUARD

    if nullable:
        vptr = buf(words)
    if col.kind in (nv.COL_UTF8, nv.COL_LARGE_UTF8, nv.COL_BINARY):
        ow = 8 if col.kind == nv.COL_LARGE_UTF8 else 4
        cap = col.values_bytes if cap is None else cap
        optr = buf((n + 1) * ow)
        return dfd.DeviceColumn(col.kind, 0, buf(cap), optr, vptr, 0, n, keep, col.arrow_type, cap)
    vals = buf(words if col.kind == nv.COL_BOOL else n * col.width)
    return dfd.DeviceColumn(col.kind, col.width, vals, 0, vptr, 0, n, keep, col.arrow_type)


def raw(t):
    return t.cpu().numpy()


def past_front_guard(t):
    """The bytes of a guarded_output buffer from its column's first byte on, after checking the guard in front."""
    b = raw(t)
    assert (b[:GUARD] == FILL).all(), "a byte in front of an output buffer was written"
    return b[GUARD:]


def read_bits(t, n, G):
    """Bits of rows [0, G) of a guarded bit-packed output; the rest of the buffer must be as the reduce found it."""
    b = past_front_guard(t)
    words = (G + 31) // 32 * 4
    assert (b[words:] == FILL).all(), "a word past row G was written"
    bits = np.unpackbits(b[:words], bitorder="little")
    assert not bits[G:].any(), "a bit at or past G is set"
    return bits[:G].astype(bool)


def read_column(col, n, G):
    """Python values of output rows [0, G) (None for a null), after checking the guard bytes."""
    valid = read_bits(col.keep[0], n, G) if col.validity else np.ones(G, dtype=bool)
    if col.kind in (nv.COL_UTF8, nv.COL_LARGE_UTF8, nv.COL_BINARY):
        ow = 8 if col.kind == nv.COL_LARGE_UTF8 else 4
        ob, db = past_front_guard(col.keep[-2]), past_front_guard(col.keep[-1])
        assert (ob[(G + 1) * ow:] == FILL).all(), "an offset past entry G was written"
        off = ob[:(G + 1) * ow].view(np.int64 if ow == 8 else np.int32).astype(np.int64)
        assert off[0] == 0 and (np.diff(off) >= 0).all()
        total = int(off[G])
        assert (db[total:] == FILL).all(), "a byte past the total was written"
        out = []
        for r in range(G):
            s = db[off[r]:off[r + 1]].tobytes()
            if not valid[r]:
                assert s == b"", "a null key's row is not empty"
            out.append(s if valid[r] else None)
        return out
    if col.kind == nv.COL_BOOL:
        bits = read_bits(col.keep[-1], n, G)
        assert not (bits & ~valid).any(), "a null Boolean key has its value bit set"
        return [bool(b) if v else None for b, v in zip(bits, valid)]
    b = past_front_guard(col.keep[-1])
    assert (b[G * col.width:] == FILL).all(), "a value past row G was written"
    vals = b[:G * col.width].view(np.int32 if col.width == 4 else np.int64).tolist()
    return [v if ok else None for v, ok in zip(vals, valid)]


def call_reduce(ctx, ins, outs, n_keys, N, starts, ops=None):
    """dfd_partial_reduce_device over prepartitioned inputs (keys first) -> (status, out_part_starts, launches)."""
    ops = [-1] * n_keys + STATE_OPS[:len(ins) - n_keys] if ops is None else ops
    sd = torch.from_numpy(np.asarray(starts, dtype=np.int64)).cuda()
    out_starts = (C.c_int64 * (N + 1))(*([-7] * (N + 1)))
    torch.cuda.synchronize()
    before = ctx.metrics()["kernel_launches"]
    rc = nv.lib().dfd_partial_reduce_device(ctx.handle, columns_to_c(ins), len(ins), int(starts[-1]), (C.c_int32 * n_keys)(*range(n_keys)),
                                            n_keys, (C.c_int32 * len(ops))(*ops), sd.data_ptr(), N, columns_to_c(outs), out_starts, None)
    return rc, np.array(out_starts, dtype=np.int64), ctx.metrics()["kernel_launches"] - before


# ------------------------------------------------------------------ harness ----

def layout(keys, gid, N, rng):
    """Rows of groups `gid` laid out partition by partition (each group in one random partition): (order, starts)."""
    gpart = rng.integers(0, N, int(gid.max()) + 1)
    dest = gpart[gid]
    order = np.argsort(dest, kind="stable")
    starts = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(np.bincount(dest, minlength=N), out=starts[1:])
    return order, starts


def run_case(ctx, kinds, keys, N, seed, arrow_off=0, first_off=0, addr=0, validity=None, gid=None):
    """Reduce rows whose key columns are keys[k] (kind kinds[k], Python values) with the four Int64 states, each group in
    one partition, and compare every partition with the reference.  -> (G, launches)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n = len(keys[0])
    if gid is None:  # rows with equal key tuples are one group
        ids = {}
        gid = np.array([ids.setdefault(tuple(k[r] for k in keys), len(ids)) for r in range(n)], dtype=np.int64)
    order, starts = layout(keys, gid, N, rng)
    keys = [[k[i] for i in order] for k in keys]
    states = [np.ones(n, dtype=np.int64)] + [rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64) for _ in range(3)]
    ins = [upload_key(kd, k, rng, arrow_off, first_off, addr, validity) for kd, k in zip(kinds, keys)] + [upload_state(s) for s in states]
    outs = [guarded_output(c, n, nullable=bool(c.validity)) for c in ins]
    rc, out_starts, launches = call_reduce(ctx, ins, outs, len(kinds), N, starts)
    assert rc == 0, nv.lib().dfd_last_error()
    G = int(out_starts[N])
    got_keys = [read_column(o, n, G) for o in outs[:len(kinds)]]
    got_states = [read_column(o, n, G) for o in outs[len(kinds):]]
    for p in range(N):
        want = reference_group_by(keys, states, STATE_KINDS, range(int(starts[p]), int(starts[p + 1])))
        a, b = int(out_starts[p]), int(out_starts[p + 1])
        got = {tuple(k[r] for k in got_keys): [s[r] for s in got_states] for r in range(a, b)}
        assert b - a == len(got), f"partition {p}: a key appears twice"
        assert got == want, f"partition {p}"
    n_var = sum(k in ("utf8", "large", "binary") for k in kinds)
    assert launches == (4 + 4 * n_var if n else 0), launches
    return G, launches


def random_strings(rng, count, lengths):
    return [bytes(rng.integers(0, 256, int(rng.choice(lengths)), dtype=np.uint8)) for _ in range(count)]


SHORT = list(range(0, 49))
MIXED_LENGTHS = SHORT + [63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 1000]


# ------------------------------------------------------------------- tests ----

@pytest.mark.parametrize("kind", ["utf8", "large", "binary"])
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("position", ["alone", "middle"])
def test_key_kinds(ctx, kind, nullable, position):
    """A var-width key alone, or between an Int32 and a Boolean key, with and without nulls."""
    rng = np.random.Generator(np.random.PCG64(11))
    n, groups = 20_000, 2_500
    pool = random_strings(rng, groups, MIXED_LENGTHS)
    if nullable:
        pool = [None if i % 10 == 3 else s for i, s in enumerate(pool)]
    g = rng.integers(0, groups, n)
    var = [pool[i] for i in g]
    if position == "alone":
        run_case(ctx, [kind], [var], 5, 1)
    else:
        i32 = [int(i % 7) if not (nullable and i % 13 == 5) else None for i in g]
        bl = [bool(i % 2) if not (nullable and i % 11 == 4) else None for i in g]
        run_case(ctx, ["i32", kind, "bool"], [i32, var, bl], 5, 2)


@pytest.mark.parametrize("addr", range(8))
def test_lengths_at_every_address_and_slice(ctx, addr):
    """Every length 0-48, lengths around 64, 128 and 256 and past 256, with the bytes starting at every address mod 8,
    behind an Arrow offset and a nonzero first offset; copies of a long string both co-aligned and not."""
    rng = np.random.Generator(np.random.PCG64(100 + addr))
    lengths = SHORT + list(range(60, 69)) + list(range(120, 137)) + list(range(250, 263)) + [300, 511, 1000, 4099]
    pool = [bytes(rng.integers(0, 256, L, dtype=np.uint8)) for L in lengths]
    g = rng.permutation(np.repeat(np.arange(len(pool)), 3))
    kind = ["utf8", "binary", "large"][addr % 3]
    keys = [pool[i] if j % 17 else None for j, i in enumerate(g)]
    run_case(ctx, [kind], [keys], 3, 7, arrow_off=3 + addr, first_off=5 + 3 * addr, addr=addr)


def test_tricky_values(ctx):
    """"" against null, strings that are prefixes of one another or differ only by a trailing NUL, keys equal in column 1
    that differ in column 2, and non-empty bytes under every null (upload_key puts them there)."""
    vals = [b"", None, b"a", b"a\x00", b"ab", b"abc", b"abcdefgh", b"abcdefghi", b"abcdefgh\x00", b"\x00", b"\x00" * 8,
            b"\x00" * 9, b"x" * 16, b"x" * 17, b"x" * 15]
    rng = np.random.Generator(np.random.PCG64(3))
    g = rng.integers(0, len(vals), 4_000)
    k1 = [vals[i] for i in g]
    k2 = [vals[(i * 7 + j) % len(vals)] if j % 3 else vals[i] for j, i in enumerate(g)]
    for N in (1, 3):
        run_case(ctx, ["utf8"], [k1], N, 4)
        run_case(ctx, ["binary", "large"], [k1, k2], N, 5)
        run_case(ctx, ["utf8", "bool"], [[b"same"] * len(g), [bool(i % 2) if i % 5 else None for i in g]], N, 6)


@pytest.mark.parametrize("bit", range(8))
@pytest.mark.parametrize("nulls", [False, True])
def test_boolean_keys_at_every_bit_offset(ctx, bit, nulls):
    rng = np.random.Generator(np.random.PCG64(bit))
    n = 3_001
    keys = [bool(rng.integers(0, 2)) if not (nulls and rng.random() < 0.2) else None for _ in range(n)]
    G, _ = run_case(ctx, ["bool"], [keys], 1, 8, arrow_off=bit)
    assert G == len(set(keys))
    # two Boolean keys: at most 9 groups over up to 9 partitions, some empty
    keys2 = [bool(rng.integers(0, 2)) if not (nulls and rng.random() < 0.2) else None for _ in range(n)]
    run_case(ctx, ["bool", "bool"], [keys, keys2], 9, 9, arrow_off=bit)


def test_one_group_holds_every_row(ctx):
    G, _ = run_case(ctx, ["utf8"], [[b"the same key for every row"] * 100_000], 4, 10)
    assert G == 1


def test_every_row_its_own_group(ctx):
    rng = np.random.Generator(np.random.PCG64(12))
    n = 60_000
    keys = [int(r).to_bytes(4, "little") + bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8)) for r in range(n)]
    G, _ = run_case(ctx, ["large"], [keys], 16, 11)
    assert G == n


def test_more_partitions_than_groups(ctx):
    keys = [[b"alpha", b"beta", b"", None, b"gamma"][i % 5] for i in range(20_000)]
    G, _ = run_case(ctx, ["utf8"], [keys], 64, 12)
    assert G == 5


def test_probe_chain_of_string_keys_on_one_home_slot(ctx):
    """Distinct strings that differ only in their last byte or their length, all with the same home slot (found with the
    restated hash): every insert walks the chain comparing bytes."""
    reps = 3
    want_keys = 40
    slots = reduce_table_slots(want_keys * reps)
    base = b"probe-chain-key-of-some-length-"
    cands = [base[:L] + bytes([b]) for L in range(8, len(base) + 1) for b in range(256)]
    cands += [base + b"\x00" * L for L in range(1, 64)]
    by_slot = {}
    for s in cands:
        by_slot.setdefault(home_slot([s], slots), []).append(s)
    slot, chain = max(by_slot.items(), key=lambda kv: len(kv[1]))
    chain = chain[:want_keys]
    assert len(chain) >= 20, len(chain)
    rng = np.random.Generator(np.random.PCG64(13))
    g = rng.permutation(np.repeat(np.arange(len(chain)), reps))
    G, _ = run_case(ctx, ["utf8"], [[chain[i] for i in g]], 1, 14)
    assert G == len(chain)


def _capacity_inputs(rng, n=5_000):
    pool = random_strings(rng, 300, MIXED_LENGTHS) + [None]
    g = rng.integers(0, len(pool), n)
    keys = [[pool[i] for i in g], [bool(i % 2) for i in g]]
    ins = [upload_key("utf8", keys[0], rng), upload_key("bool", keys[1], rng)] + [upload_state(np.arange(n))]
    need = sum(len(s) for s in set(keys[0]) if s is not None)
    return ins, need, n


def test_exact_capacity_and_one_byte_short(ctx):
    rng = np.random.Generator(np.random.PCG64(15))
    ins, need, n = _capacity_inputs(rng)
    starts = [0, n]
    outs = [guarded_output(ins[0], n, cap=need, nullable=True), guarded_output(ins[1], n), guarded_output(ins[2], n)]
    rc, out_starts, launches = call_reduce(ctx, ins, outs, 2, 1, starts)
    assert rc == 0 and launches == 8
    G = int(out_starts[1])
    assert sum(len(s) for s in read_column(outs[0], n, G) if s) == need
    outs = [guarded_output(ins[0], n, cap=need - 1, nullable=True), guarded_output(ins[1], n), guarded_output(ins[2], n)]
    rc, out_starts, launches = call_reduce(ctx, ins, outs, 2, 1, starts)
    assert rc == ERR_CAPACITY and str(need) in nv.lib().dfd_last_error().decode()
    assert launches == 2, "a place or copy launch was counted"
    assert (out_starts == -7).all()
    for o in outs:
        for t in o.keep:
            assert (raw(t) == FILL).all(), "an output was written before the capacity refusal"


@pytest.mark.parametrize("kinds,clear,want", [
    (["bool"], False, 4), (["utf8"], False, 8), (["i32", "utf8", "bool"], False, 8), (["utf8", "large"], False, 12),
    (["binary", "utf8", "large"], True, 17), (["bool", "i32"], True, 5)])
def test_launch_counts(ctx, kinds, clear, want):
    """4 (+1 with k_group_clear) + 4 per var-width key, per the header."""
    rng = np.random.Generator(np.random.PCG64(16))
    n = 2_000
    vals = {"utf8": [b"k%d" % (i % 37) for i in range(n)], "large": [b"L" * (i % 5) for i in range(n)],
            "binary": [bytes([i % 3]) for i in range(n)], "bool": [bool(i % 2) for i in range(n)], "i32": [i % 4 for i in range(n)]}
    ins = [upload_key(k, vals[k], rng) for k in kinds]
    st = upload_state(rng.integers(0, 100, n))
    ins.append(st)
    ops = [-1] * len(kinds) + [nv.AGG_MIN_I64]
    if clear:
        vt = cuda_bytes(b"\xff" * ((n + 7) // 8) + b"\0" * 8)
        st.validity, st.keep = vt.data_ptr(), st.keep + [vt]
    outs = [guarded_output(c, n, nullable=bool(c.validity)) for c in ins]
    rc, _, launches = call_reduce(ctx, ins, outs, len(kinds), 1, [0, n], ops)
    assert rc == 0 and launches == want


def test_argument_refusals_launch_nothing(ctx):
    rng = np.random.Generator(np.random.PCG64(17))
    n = 100
    s = upload_key("utf8", [b"a", b"bb"] * 50, rng)
    b = upload_key("bool", [True, False] * 50, rng)
    k = upload_key("i32", list(range(n)), rng)
    st = upload_state(np.arange(n))

    def refused(ins, outs, n_keys, ops, status):
        rc, out_starts, launches = call_reduce(ctx, ins, outs, n_keys, 1, [0, n], ops)
        assert rc == status, (rc, nv.lib().dfd_last_error())
        assert launches == 0 and (out_starts == -7).all()
        for o in outs:
            for t in o.keep:
                assert (raw(t) == FILL).all()

    # a var-width or Boolean STATE column
    refused([k, s], [guarded_output(k, n), guarded_output(s, n)], 1, [-1, nv.AGG_SUM_I64], ERR_UNSUPPORTED)
    refused([k, b], [guarded_output(k, n), guarded_output(b, n)], 1, [-1, nv.AGG_MAX_I64], ERR_UNSUPPORTED)
    # an output of another kind than its key's
    for other in (guarded_output(b, n), guarded_output(k, n), guarded_output(upload_key("large", [b"a"] * n, rng), n)):
        refused([s, st], [other, guarded_output(st, n)], 1, [-1, nv.AGG_SUM_I64], ERR_INVALID)
    refused([b, st], [guarded_output(s, n), guarded_output(st, n)], 1, [-1, nv.AGG_SUM_I64], ERR_INVALID)
    # NULL offsets, input or output
    o = guarded_output(s, n)
    refused([s, st], [dfd.DeviceColumn(o.kind, 0, o.values, 0, 0, 0, n, o.keep, o.arrow_type, o.values_bytes), guarded_output(st, n)], 1,
            [-1, nv.AGG_SUM_I64], ERR_INVALID)
    refused([dfd.DeviceColumn(s.kind, 0, s.values, 0, 0, 0, n, s.keep, s.arrow_type, s.values_bytes), st], [guarded_output(s, n), guarded_output(st, n)], 1,
            [-1, nv.AGG_SUM_I64], ERR_INVALID)
    # a Boolean output not 4-byte aligned
    ob = guarded_output(b, n)
    refused([b, st], [dfd.DeviceColumn(nv.COL_BOOL, 0, ob.values + 2, 0, 0, 0, n, ob.keep, pa.bool_()), guarded_output(st, n)], 1,
            [-1, nv.AGG_SUM_I64], ERR_INVALID)


def test_partition_reduce_shuffle_on_string_keys(ctx):
    """Partition on (Utf8, Boolean) keys -> reduce -> shuffle_partitioned at world 1: segment q holds exactly the reduced
    groups of destination q."""
    rng = np.random.Generator(np.random.PCG64(18))
    n, N = 50_000, 6
    pool = random_strings(rng, 400, MIXED_LENGTHS)
    g = rng.integers(0, len(pool), n)
    k1 = pa.array([pool[i].hex() if i % 9 else None for i in g], type=pa.string())
    k2 = pa.array([bool(i % 2) for i in g])
    cnt = pa.array(np.ones(n, dtype=np.int64))
    sm = pa.array(rng.integers(-1000, 1000, n, dtype=np.int64))
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in (k1, k2, cnt, sm)]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1], N))
    pouts, pstarts = part.partition(dcols, n)
    outs, out_starts = dfd.PartialReduceExec(ctx, [0, 1], [-1, -1, nv.AGG_SUM_I64, nv.AGG_SUM_I64]).reduce(
        pouts, n, part.part_starts_device_ptr(), N)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(64 << 20)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], N), uuid.uuid4(), 1, 1, 1)
    wcols, ss, sc = node.shuffle_partitioned(ex, outs, out_starts)
    assert np.array_equal(sc[:, 0], np.diff(out_starts))
    seen = set()
    for q in range(N):
        a, b = int(pstarts[q]), int(pstarts[q + 1])
        rows = [pouts[i].to_arrow(ctx, a, b).to_pylist() for i in range(4)]
        want = reference_group_by(rows[:2], [np.array(rows[2]), np.array(rows[3])], ["sum", "sum"], range(b - a))
        seg = [dfd.NetworkShuffleExec.segment_to_arrow(ctx, wcols[i], int(ss[q, 0]), int(sc[q, 0])).to_pylist() for i in range(4)]
        got = {(seg[0][r], seg[1][r]): [seg[2][r], seg[3][r]] for r in range(len(seg[0]))}
        assert len(got) == len(seg[0]) and got == want, q
        assert not (seen & set(got)), "a key reached two destinations"
        seen |= set(got)
    ex.close()


def test_q1_partial_states_reduce_to_four_groups(ctx):
    """cfg-3's q1 partial states of 8 producers, partitioned on (l_returnflag, l_linestatus) and reduced: the 4 groups,
    with exact Decimal128 and Int64 sums and Float64 sums within test_reduce_gpu.py's bound."""
    from bench_workloads import cfg3_columns
    from tests.test_reduce_gpu import check_state, merge, py_values

    parts = [cfg3_columns(r) for r in range(8)]
    cols = [pa.concat_arrays([p[i] for p in parts]) for i in range(len(parts[0]))]
    n, N = len(cols[0]), 4
    ops = [-1, -1] + [nv.AGG_SUM_I128] * 4 + [nv.AGG_SUM_I64] * 4 + [nv.AGG_SUM_F64] * 2
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in cols]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1], N))
    pouts, _ = part.partition(dcols, n)
    outs, out_starts = dfd.PartialReduceExec(ctx, [0, 1], ops).reduce(pouts, n, part.part_starts_device_ptr(), N)
    G = int(out_starts[N])
    assert G == 4
    flags, status = outs[0].to_arrow(ctx, 0, G).to_pylist(), outs[1].to_arrow(ctx, 0, G).to_pylist()
    key_of = list(zip(cols[0].to_pylist(), cols[1].to_pylist()))
    assert set(zip(flags, status)) == {("A", "F"), ("N", "F"), ("N", "O"), ("R", "F")}
    for c in range(2, len(cols)):
        wide = ops[c] == nv.AGG_SUM_I128
        host_in = np.frombuffer(cols[c].buffers()[1], dtype=np.int64 if ops[c] != nv.AGG_SUM_F64 else np.float64)
        host_out = outs[c].keep[-1].download(host_in.dtype, G * (2 if wide else 1))
        vin = py_values(host_in.reshape(-1, 2) if wide else host_in)
        vout = py_values(host_out.reshape(-1, 2) if wide else host_out)
        for r in range(G):
            want = merge(ops[c], [vin[i] for i, k in enumerate(key_of) if k == (flags[r], status[r])])
            check_state(ops[c], vout[r], want, (flags[r], status[r], c))


def test_large_utf8_output_offsets_pass_4_gib(ctx):
    """2^20 distinct LargeUtf8 keys of 4 100 bytes, each twice: the groups' bytes (4.3 GB) put the output offsets past
    2^32.  Every group's length and tag bytes are checked, and the full bytes of groups on both sides of 2^32."""
    n_keys, L = 1 << 20, 4100
    total = n_keys * L
    need = 4 * total + (1 << 30)  # input twice over, output, one comparison temporary, scratch
    free, _ = torch.cuda.mem_get_info()
    if free < need + (2 << 30):
        pytest.skip(f"needs {(need + (2 << 30)) / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB is free")
    n = 2 * n_keys
    ids = torch.arange(n_keys, dtype=torch.int64, device="cuda").repeat(2)  # row r holds key r mod n_keys
    data = torch.full((n, L), 0x5C, dtype=torch.uint8, device="cuda")
    tag = ids.view(-1, 1).view(torch.uint8).view(n, 8)
    data[:, :8] = tag
    data[:, L - 8:] = tag
    data[:, 8] = (ids % 251).to(torch.uint8)
    data = data.view(-1)
    offs = torch.arange(n + 1, dtype=torch.int64, device="cuda") * L
    cnt = torch.ones(n, dtype=torch.int64, device="cuda")
    ins = [dfd.DeviceColumn(nv.COL_LARGE_UTF8, 0, data.data_ptr(), offs.data_ptr(), 0, 0, n, [data, offs], pa.large_string(), n * L),
           dfd.DeviceColumn(nv.COL_FIXED, 8, cnt.data_ptr(), 0, 0, 0, n, [cnt], pa.int64())]
    out_data = torch.empty(total, dtype=torch.uint8, device="cuda")
    out_off = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda")
    out_cnt = torch.empty(n, dtype=torch.int64, device="cuda")
    outs = [dfd.DeviceColumn(nv.COL_LARGE_UTF8, 0, out_data.data_ptr(), out_off.data_ptr(), 0, 0, n, [out_off, out_data], pa.large_string(), total),
            dfd.DeviceColumn(nv.COL_FIXED, 8, out_cnt.data_ptr(), 0, 0, 0, n, [out_cnt], pa.int64())]
    rc, out_starts, launches = call_reduce(ctx, ins, outs, 1, 1, [0, n], [-1, nv.AGG_SUM_I64])
    assert rc == 0, nv.lib().dfd_last_error()
    assert int(out_starts[1]) == n_keys and launches == 8
    off = out_off[:n_keys + 1]
    assert int(off[0]) == 0 and int(off[-1]) == total and total > (1 << 32)
    assert bool((off[1:] - off[:-1] == L).all())
    assert int(out_off[n_keys + 1]) == -1 and bool((out_off[n_keys + 1:] == -1).all())
    assert bool((out_cnt[:n_keys] == 2).all())
    grp = out_data.view(n_keys, L)
    got_ids = grp[:, :8].contiguous().view(torch.int64).view(-1)
    assert bool((grp[:, L - 8:].contiguous().view(torch.int64).view(-1) == got_ids).all())
    assert bool((grp[:, 8] == (got_ids % 251).to(torch.uint8)).all())
    assert bool((torch.sort(got_ids).values == torch.arange(n_keys, device="cuda")).all())
    assert bool((grp[:, 9:L - 8] == 0x5C).all())
    cross = (1 << 32) // L
    for o in (0, cross - 1, cross, cross + 1, n_keys - 1):
        i = int(got_ids[o])
        assert torch.equal(grp[o], data[i * L:(i + 1) * L]), o
