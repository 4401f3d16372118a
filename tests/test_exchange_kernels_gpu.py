"""GPU parity tests of the exchange's own kernels at world = 1: k_push_runs (csrc/dfd_exchange.cu), the push transport of
shuffle_onepass, coalesce, broadcast and shuffle_partitioned, past one CTA and at every alignment it distinguishes; the
NCCL-mode lane kernels k_bits_to_bytes, k_bytes_to_bits, k_offsets_to_lengths and k_var_dest_bytes (csrc/dfd_kernels.cuh)
past one grid pass; and the int32 limit of Utf8 / Binary offsets in a push-transport segment.

The reference is pyarrow on the host: every segment must equal `arr.take(rows)` or `arr.slice(...)` of its source.  String
offsets are compared raw, as int64, with the values the segment layout implies before any Arrow array is built from them, so
a wrapped or misplaced offset fails as an assertion and never sizes a download.

Sizes come from the sources: PUSH_CHUNK and PUSH_THREADS from dfd_exchange.cu, the grid cap and block of the lane launches
from dfd_api.cu.  Every case asserts the threshold it is meant to reach, computed on the host from the same run layout
push_slices_locked builds."""
import gc
import os
import re
import time
import uuid

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.util import ROOT, dest_lut, expected_partitions

pytestmark = pytest.mark.gpu

CSRC = os.path.join(ROOT, "datafusion_distributed_b200", "csrc")
GiB = 1 << 30
INT32_MAX = (1 << 31) - 1


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _push_constant(name):
    m = re.search(rf"constexpr\s+(?:int|long long)\s+{name}\s*=\s*([0-9 *]+);", _source("dfd_exchange.cu"))
    assert m, name
    v = 1
    for f in m.group(1).split("*"):
        v *= int(f)
    return v


def _lane_launch(fn):
    """(grid cap, block threads) of dfd::launch_<fn> in dfd_api.cu."""
    body = re.search(rf"int dfd::{fn}\(.*?\n}}\n", _source("dfd_api.cu"), re.S).group(0)
    cap = re.search(r">\s*(\d+)\s*\?\s*(\d+)\s*:", body)
    threads = re.search(r"<<<[^,]+,\s*(\d+)\s*,", body)
    assert cap and cap.group(1) == cap.group(2) and threads, fn
    return int(cap.group(1)), int(threads.group(1))


PUSH_CHUNK = _push_constant("PUSH_CHUNK")      # output bytes one k_push_runs CTA copies
PUSH_THREADS = _push_constant("PUSH_THREADS")
BITS_PER_CTA = PUSH_CHUNK * 8                  # RUN_BITS / RUN_ONES rows per CTA
OFF32_PER_CTA, OFF64_PER_CTA = PUSH_CHUNK // 4, PUSH_CHUNK // 8
_LANES = {fn: _lane_launch(fn) for fn in ("launch_bits_to_bytes", "launch_bytes_to_bits", "launch_offsets_to_lengths")}
assert len(set(_LANES.values())) == 1, _LANES
LANE_GRID_CAP, LANE_BLOCK = next(iter(_LANES.values()))
LANE_ONE_PASS = LANE_GRID_CAP * LANE_BLOCK     # rows one grid pass of the lane kernels covers


@pytest.fixture(scope="module")
def ctx(built):
    c = dfd.WorkerContext(0)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------ host reference ----

def ctas(out_bytes):
    return -(-out_bytes // PUSH_CHUNK)


def is_var(t):
    return pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t)


_LENGTHS = {}


def lengths(arr):
    """Byte length of every row of a string array, from its raw offsets (null rows included)."""
    key = (arr.buffers()[1].address, arr.offset, len(arr))
    if key not in _LENGTHS:
        if len(_LENGTHS) > 64:
            _LENGTHS.clear()
        odt = np.int64 if pa.types.is_large_string(arr.type) else np.int32
        off = np.frombuffer(arr.buffers()[1], dtype=odt)[arr.offset:arr.offset + len(arr) + 1].astype(np.int64)
        _LENGTHS[key] = (np.diff(off), arr)  # (the array keeps its buffer, so the address is not reused)
    return _LENGTHS[key][0]


def first_offset(arr, row):
    odt = np.int64 if pa.types.is_large_string(arr.type) else np.int32
    return int(np.frombuffer(arr.buffers()[1], dtype=odt)[arr.offset + row])


def layout(seg_rows, seg_bytes=None):
    """push_slices_locked's consumer layout: segment starts in rows (32-row aligned, >= 1 spare row) and, for a string
    column, in bytes (16-byte aligned)."""
    rs, bs, r, b = [], [], 0, 0
    for i, n in enumerate(seg_rows):
        rs.append(r)
        r = (r + n + 1 + 31) // 32 * 32
        if seg_bytes is not None:
            bs.append(b)
            b = (b + seg_bytes[i] + 15) // 16 * 16
    return rs, bs


def max_offset(seg_rows, seg_bytes):
    """The largest string offset a consumer's segments hold: the end of the last segment with rows."""
    _, bs = layout(seg_rows, seg_bytes)
    ends = [b + n for b, n, r in zip(bs, seg_bytes, seg_rows) if r > 0]
    return max(ends) if ends else 0


def grab(ctx, ptr, nbytes):
    buf = np.empty(max(nbytes, 1), dtype=np.uint8)
    assert 0 <= nbytes < 8 * GiB, nbytes
    if nbytes:
        nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, buf.ctypes.data, ptr, nbytes))
    return buf[:nbytes]


def seg_bits(ctx, ptr, start, count):
    assert start % 32 == 0
    return np.unpackbits(grab(ctx, ptr + start // 8, (count + 7) // 8), bitorder="little")[:count]


def check_segment(ctx, col, start, count, src, rows, bseg=None, what=""):
    """Rows [start, start + count) of a window column against src.take(rows).  A string segment's raw offsets must be
    bseg + the running byte lengths of its source rows; they are checked before the bytes are read."""
    want = src.take(pa.array(rows, type=pa.int64())) if len(rows) else src.slice(0, 0)
    assert count == len(rows), what
    if count == 0:
        return
    t = src.type
    vbuf, nulls = None, 0
    if col.validity:
        vb = seg_bits(ctx, col.validity, start, count)
        nulls = int(count - vb.sum())
        vbuf = pa.py_buffer(np.packbits(vb, bitorder="little").tobytes())
    else:
        assert src.null_count == 0, what
    if pa.types.is_boolean(t):
        got = pa.Array.from_buffers(t, count, [vbuf, pa.py_buffer(np.packbits(seg_bits(ctx, col.values, start, count), bitorder="little").tobytes())],
                                    null_count=nulls)
    elif not is_var(t):
        w = col.width
        got = pa.Array.from_buffers(t, count, [vbuf, pa.py_buffer(grab(ctx, col.values + start * w, count * w).tobytes())], null_count=nulls)
    else:
        ow = 8 if pa.types.is_large_string(t) else 4
        off = grab(ctx, col.offsets + start * ow, (count + 1) * ow).view(np.int64 if ow == 8 else np.int32).astype(np.int64)
        want_off = np.zeros(count + 1, dtype=np.int64)
        np.cumsum(lengths(src)[np.asarray(rows)], out=want_off[1:])
        if bseg is not None:
            want_off += bseg
        else:
            want_off += off[0]
        bad = np.nonzero(off != want_off)[0]
        assert not len(bad), f"{what}: raw offsets differ at {len(bad)} of {count + 1} entries, first at {bad[0]}: got {off[bad[0]]}, want {want_off[bad[0]]}"
        data = grab(ctx, col.values + int(off[0]), int(off[-1] - off[0]))
        got = pa.Array.from_buffers(t, count, [vbuf, pa.py_buffer((off - off[0]).astype(np.int64 if ow == 8 else np.int32).tobytes()),
                                               pa.py_buffer(data.tobytes())], null_count=nulls)
    assert got.equals(want), what


def bitmap_array(values, valid, offset=0):
    """A Boolean array over exactly-sized bitmaps (offset rows of padding in front)."""
    n = len(values)
    bits = np.concatenate([np.zeros(offset, bool), values])
    vb = None
    if valid is not None:
        vb = pa.py_buffer(np.packbits(np.concatenate([np.ones(offset, bool), valid]), bitorder="little").tobytes())
    return pa.Array.from_buffers(pa.bool_(), n, [vb, pa.py_buffer(np.packbits(bits, bitorder="little").tobytes())], offset=offset)


def strings(rng, n, max_len, typ, null_frac=0.0, lens=None):
    """Random printable strings; null rows have length 0."""
    valid = rng.random(n) >= null_frac if null_frac else np.ones(n, bool)
    if lens is None:
        lens = rng.integers(0, max_len + 1, n)
    lens = np.where(valid, lens, 0).astype(np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    data = rng.integers(32, 127, int(off[-1]), dtype=np.uint8)
    odt = np.int64 if typ == pa.large_string() else np.int32
    vb = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()) if null_frac else None
    return pa.Array.from_buffers(typ, n, [vb, pa.py_buffer(off.astype(odt).tobytes()), pa.py_buffer(data.tobytes())],
                                 null_count=int(n - valid.sum()))


def mixed_table(n, seed):
    """Every column kind the push transport moves: nullable Int64 key, Utf8, LargeUtf8, Binary (nullable in the schema,
    no nulls: RUN_ONES), Boolean, Int32, and a non-null Float64."""
    rng = np.random.Generator(np.random.PCG64(seed))
    key = pa.array(rng.integers(0, 1 << 40, n), mask=rng.random(n) < 0.05)
    s = strings(rng, n, 40, pa.string(), 0.1)
    ls = strings(rng, n, 12, pa.large_string(), 0.2)
    b = strings(rng, n, 20, pa.binary())
    bl = pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1)
    i32 = pa.array(rng.integers(-(1 << 31), 1 << 31, n).astype(np.int32), mask=rng.random(n) < 0.1)
    f64 = pa.array(rng.standard_normal(n))
    return [key, s, ls, b, bl, i32, f64]


def gather(ctx, ex, arrays, starts, nullable):
    co = dfd.NetworkCoalesceExec.try_new(len(starts) - 1, uuid.uuid4(), 1, 1, 1)
    cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    outs, ss, sc = co.gather(ex, cols, starts, nullable=nullable)
    return cols, outs, ss, sc


def check_gather(ctx, arrays, starts, outs, ss, sc):
    """Coalesce at world = 1: segment j is slice j of the producer, at the layout push_slices_locked computes."""
    seg_rows = np.diff(starts).tolist()
    rs, _ = layout(seg_rows)
    assert ss.tolist() == rs and sc.tolist() == seg_rows
    for c, arr in enumerate(arrays):
        bs = layout(seg_rows, [int(lengths(arr)[a:b].sum()) for a, b in zip(starts[:-1], starts[1:])])[1] if is_var(arr.type) else [None] * len(seg_rows)
        for j in range(len(seg_rows)):
            check_segment(ctx, outs[c], int(ss[j]), int(sc[j]), arr, np.arange(starts[j], starts[j + 1]), bs[j], f"column {c} ({arr.type}) slice {j}")


# ------------------------------------------------------------------------------------------- RUN_BYTES, fixed width ----

FIXED_TYPES = {1: pa.int8(), 2: pa.int16(), 4: pa.int32(), 8: pa.int64(), 16: pa.decimal128(38, 0)}


def byte_lengths():
    """RUN_BYTES run lengths in bytes: empty, short, around one CTA's chunk, past two chunks, several MiB."""
    return [0] + list(range(1, 18)) + [31, 32, 33, PUSH_CHUNK - 1, PUSH_CHUNK, PUSH_CHUNK + 1, 2 * PUSH_CHUNK + 7, (5 << 20) + 3]


def place(classes_and_lengths, addr_of, unit):
    """Slice boundaries (rows) that start each wanted slice at its address class mod 16, with filler slices between:
    addr_of(row) is the source address of a row, `unit` rows' bytes per row."""
    starts, wanted, row = [0], [], 0
    for cls, n in classes_and_lengths:
        pad = 0
        while (addr_of(row + pad) & 15) != cls:
            pad += 1
            assert pad < 16
        if pad:
            row += pad
            starts.append(row)
        wanted.append(len(starts) - 1)
        row += n
        starts.append(row)
    return starts, wanted


@pytest.mark.parametrize("width", [1, 2, 4, 8, 16])
def test_run_bytes_fixed_width_every_alignment_class(ctx, width):
    """Fixed-width non-null columns through coalesce: every (src ^ dst) & 15 class the width reaches (the 16 / 8 / 4 /
    1-byte bodies of RUN_BYTES), each with runs of 0 to 33 bytes, one CTA's chunk +- 1 byte, two chunks + 7 and 5 MiB."""
    offset = 3
    classes = sorted({(k * width) & 15 for k in range(16)})
    runs = [(cls, max(n // width, 0) if n >= PUSH_CHUNK else n) for cls in classes for n in byte_lengths()]
    if width > 1:  # short runs in rows; around the chunk: rows whose bytes straddle it
        runs = [(cls, n) for cls, n in runs if n < 64] + [(cls, r) for cls in classes
                                                         for r in (PUSH_CHUNK // width - 1, PUSH_CHUNK // width, PUSH_CHUNK // width + 1,
                                                                   (2 * PUSH_CHUNK + 7) // width + 1, ((5 << 20) + 3) // width)]
    rng = np.random.Generator(np.random.PCG64(width))
    total = sum(n for _, n in runs) + 16 * len(runs) + offset
    raw = rng.integers(0, 256, total * width, dtype=np.uint8)
    arr = pa.Array.from_buffers(FIXED_TYPES[width], total, [None, pa.py_buffer(raw.tobytes())]).slice(offset)
    col = dfd.DeviceColumn.from_arrow(ctx, arr)
    starts, wanted = place(runs, lambda r: col.values + (offset + r) * width, width)
    if starts[-1] != len(arr):
        starts.append(len(arr))
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(total * width + 32 * len(starts) * width + (16 << 20))
    _, outs, ss, sc = gather(ctx, ex, [arr], starts, [False])
    # the thresholds: every class with every length class, destinations 16-byte aligned, multi-CTA runs
    dst = [outs[0].values + int(ss[j]) * width for j in range(len(ss))]
    src = [col.values + (offset + starts[j]) * width for j in range(len(ss))]
    assert all(d % 16 == 0 for d in dst)
    got_classes = {((src[j] ^ dst[j]) & 15, (starts[j + 1] - starts[j]) * width) for j in wanted}
    assert {c for c, _ in got_classes} == set(classes)
    for cls in classes:
        lens = {n for c, n in got_classes if c == cls}
        assert {1, 17, 33} <= lens or width > 1
        assert max(lens) >= 5 << 20 and any(ctas(n) >= 3 for n in lens) and any(n % PUSH_CHUNK not in (0,) and ctas(n) == 2 for n in lens)
        assert any(n % 16 for n in lens if n >= 64) or width == 16
    check_gather(ctx, [arr], starts, outs, ss, sc)
    ex.close()


# ---------------------------------------------------------------------------------- RUN_BYTES / RUN_OFF*, strings ----

@pytest.mark.parametrize("typ", [pa.string(), pa.binary(), pa.large_string()], ids=["utf8", "binary", "large_utf8"])
def test_string_runs_every_byte_residue_and_offsets_past_one_cta(ctx, typ):
    """String columns through coalesce: each slice's first byte at every residue mod 16 with byte runs of 0-33 bytes, one
    chunk +- 1, two chunks + 7 and several MiB; all-empty-string slices (offsets, no byte run) and empty slices; rebased
    offsets (first != 0) in runs past one CTA of RUN_OFF32 / RUN_OFF64; a nullable variant carries the validity bitmap."""
    rng = np.random.Generator(np.random.PCG64(7))
    per_cta = OFF64_PER_CTA if typ == pa.large_string() else OFF32_PER_CTA
    plan = []  # (first byte residue, rows, bytes per row or None for random short strings)
    for res in range(16):
        for nb in [0, 1, 2, 3, 5, 8, 13, 15, 16, 17, 31, 32, 33, PUSH_CHUNK - 1, PUSH_CHUNK, PUSH_CHUNK + 1, 2 * PUSH_CHUNK + 7]:
            plan.append((res, 1, nb))  # one row holding the whole byte run
    plan += [(5, 3 * per_cta + 17, 0), (9, 0, 0), (3, 2 * per_cta + 1, None), (11, 1, (6 << 20) + 5), (0, 40, 0)]
    prefix = np.array([3, 0, 4, 1, 2, 0, 4, 3, 2])  # 9 rows cut off by the slice: first != 0 for every slice
    lens, starts, wanted = [], [0], []
    row, pos = 0, int(prefix.sum())
    for res, nrows, nb in plan:
        if pos % 16 != res:  # a filler slice of one-byte rows moves the next slice's first byte
            k = (res - pos) % 16
            lens += [1] * k
            pos += k
            row += k
            starts.append(row)
        rl = rng.integers(0, 9, nrows) if nb is None else np.full(nrows, nb)
        if nrows > 1 and nb is None:
            rl[0] = 1
        lens.extend(rl.tolist())
        pos += int(rl.sum())
        row += nrows
        wanted.append(len(starts) - 1)
        starts.append(row)
    assert (1 + 2) * (len(starts) - 1) <= 2048  # XCHG_META_MAX entries: (1 + string columns) x slices
    n = row
    all_lens = np.concatenate([prefix, np.array(lens)])
    arr = strings(rng, n + 9, 0, typ, 0.0, lens=all_lens).slice(9)
    assert first_offset(arr, 0) > 0
    nullable = strings(rng, n + 9, 0, typ, 0.3, lens=all_lens).slice(9)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(2 * int(all_lens.sum()) + 64 * len(starts) * 8 + (32 << 20))
    cols, outs, ss, sc = gather(ctx, ex, [arr, nullable], starts, [False, True])
    # thresholds: every residue of the source's first byte, with every byte-length class; offsets runs past one CTA
    lens_a = lengths(arr)
    src_first = {j: (cols[0].values + first_offset(arr, starts[j])) & 15 for j in wanted}
    nbytes = {j: int(lens_a[starts[j]:starts[j + 1]].sum()) for j in wanted}
    assert set(src_first.values()) == set(range(16))
    for res in range(16):
        got = {nbytes[j] for j in wanted if src_first[j] == res and starts[j + 1] - starts[j] == 1}
        assert {0, 1, 17, 33, PUSH_CHUNK - 1, PUSH_CHUNK + 1} <= got and any(ctas(b) >= 3 for b in got)
    assert any(ctas((starts[j + 1] - starts[j] + 1) * (8 if typ == pa.large_string() else 4)) >= 3 for j in wanted)
    assert any(starts[j + 1] - starts[j] > 1 and nbytes[j] == 0 for j in wanted)  # an all-empty-string slice
    assert any(starts[j + 1] == starts[j] for j in wanted)  # an empty slice
    check_gather(ctx, [arr, nullable], starts, outs, ss, sc)
    ex.close()


# ------------------------------------------------------------------------------------------ RUN_BITS / RUN_ONES ----

def bit_runs():
    return list(range(1, 34)) + [63, 64, 65] + [32 * k + d for k in (3, 10, 100) for d in (-1, 1)]


SHORT_BIT_RUNS = [1, 2, 31, 32, 33, 63, 64, 65, 32 * 10 - 1, 32 * 10 + 1]  # at every residue; bit_runs() at two of them


@pytest.mark.parametrize("lane", ["boolean_values", "validity"])
def test_run_bits_every_source_residue(ctx, lane):
    """Boolean values (a Boolean column) or a validity bitmap (a nullable Int32 column) through coalesce: the source bit
    (Arrow offset + slice start) at every residue mod 32 with runs of 1-33, 63-65 and 32k +- 1 rows; a run past one CTA's
    PUSH_CHUNK * 8 rows; and a last run that ends on the bitmap's last bit, where no word after it is read."""
    rng = np.random.Generator(np.random.PCG64(11))
    offset = 5
    plan = [(res, n) for res in range(32) for n in SHORT_BIT_RUNS] + [(res, n) for res in (3, 29) for n in bit_runs()]
    plan += [(7, BITS_PER_CTA + 4099), (19, 2 * BITS_PER_CTA + 33)]
    starts, wanted, row = [0], [], 0
    for res, n in plan + [(13, 64 * 32 + 17)]:  # the last run ends on the bitmap's last bit, at a residue != 0
        if (offset + row) % 32 != res:
            row += (res - offset - row) % 32
            starts.append(row)
        wanted.append(len(starts) - 1)
        row += n
        starts.append(row)
    n = row
    assert len(starts) - 1 <= 2048 and (offset + n) % 32 != 0
    values = rng.random(n) < 0.5
    valid = rng.random(n) < 0.7
    if lane == "boolean_values":
        arr = bitmap_array(values, None, offset)
    else:
        data = np.concatenate([np.zeros(offset, np.int32), rng.integers(-1000, 1000, n).astype(np.int32)])
        vb = np.packbits(np.concatenate([np.zeros(offset, bool), valid]), bitorder="little")
        vb = np.concatenate([vb, np.zeros((-len(vb)) % 4, np.uint8)])  # whole words: the last run's last word is the bitmap's last
        arr = pa.Array.from_buffers(pa.int32(), n, [pa.py_buffer(vb.tobytes()), pa.py_buffer(data.tobytes())], offset=offset)
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(16 * n + (16 << 20))
    cols, outs, ss, sc = gather(ctx, ex, [arr], starts, [lane == "validity"])
    src_bit = {j: offset + starts[j] for j in wanted}
    assert {b % 32 for b in src_bit.values()} == set(range(32))
    run_len = {res: {starts[j + 1] - starts[j] for j in wanted if src_bit[j] % 32 == res} for res in range(32)}
    assert all(run_len[res] >= set(SHORT_BIT_RUNS) for res in range(32)) and run_len[3] >= set(bit_runs()) <= run_len[29]
    assert any(starts[j + 1] - starts[j] > BITS_PER_CTA for j in wanted)
    last = len(starts) - 2
    bitmap_words = (arr.buffers()[0 if lane == "validity" else 1].size + 3) // 4
    assert (offset + starts[last + 1] - 1) // 32 == bitmap_words - 1 and (offset + starts[last]) % 32 != 0
    check_gather(ctx, [arr], starts, outs, ss, sc)
    ex.close()


def test_run_ones_past_one_cta(ctx):
    """A column nullable in the schema whose input has no bitmap: RUN_ONES writes an all-valid bitmap, here in runs past
    one CTA's PUSH_CHUNK * 8 rows and in short runs."""
    n = 2 * BITS_PER_CTA + 12_345
    arr = pa.array(np.arange(n, dtype=np.int64))
    starts = [0, 1, 33, 33 + BITS_PER_CTA + 5, n - 7, n]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(10 * n + (16 << 20))
    cols, outs, ss, sc = gather(ctx, ex, [arr], starts, [True])
    assert not cols[0].validity and outs[0].validity and max(np.diff(starts)) > BITS_PER_CTA
    for j in range(len(starts) - 1):
        assert seg_bits(ctx, outs[0].validity, int(ss[j]), int(sc[j])).all(), j
    check_gather(ctx, [arr], starts, outs, ss, sc)
    ex.close()


# --------------------------------------------------------------------------------------- through the real paths ----

N_PUSH = 3_600_007  # at P = 6 every partition's bit runs pass one CTA (BITS_PER_CTA rows)


@pytest.fixture(scope="module")
def big_table():
    full = mixed_table(N_PUSH + 23, 31)
    return [a.slice(23) for a in full]  # sliced: Arrow offset 23 on every column


@pytest.mark.parametrize("P", [6, 48])
def test_push_shuffle_and_rounds_every_column_kind(ctx, big_table, P):
    """shuffle_onepass (push transport) of every column kind at 3.6 M rows of a sliced input, then shuffle_rounds on the
    same data with a window that forces several rounds; every segment against the oracle's destinations."""
    arrays, n = big_table, N_PUSH
    dest = orc.partition_ids([arrays[0]], n, P)
    order, ref = expected_partitions(dest, P)
    counts = np.diff(ref)
    rows_of = [order[ref[q]:ref[q + 1]] for q in range(P)]
    # thresholds from the hash-chosen layout: string byte runs and bit runs past one CTA, many source bit residues
    s_bytes = [int(lengths(arrays[1])[r].sum()) for r in rows_of]
    assert max(s_bytes) > 2 * PUSH_CHUNK and max(counts) > OFF32_PER_CTA
    assert len({int(s) % 32 for s in ref[:-1]}) >= (2 if P == 6 else 16)
    if P == 6:
        assert min(counts) > BITS_PER_CTA
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    nullable = [True] * 6 + [False]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(512 << 20)
    node.shuffle_onepass(ex, cols, n, nullable=nullable)
    outs, ss, sc = node.collect(ex)
    assert np.array_equal(sc[:, 0], counts)
    rs, _ = layout(counts.tolist())
    assert ss[:, 0].tolist() == rs
    for c, arr in enumerate(arrays):
        bs = layout(counts.tolist(), [int(lengths(arr)[r].sum()) for r in rows_of])[1] if is_var(arr.type) else [None] * P
        for q in range(P):
            check_segment(ctx, outs[c], int(ss[q, 0]), int(sc[q, 0]), arr, rows_of[q], bs[q], f"shuffle column {c} partition {q}")
    ex.close()
    # back-pressured rounds: a window of ~1/5 of the data
    ex2 = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex2.setup_window(48 << 20)
    cursor = [0] * P
    for outs, ss, sc in node.shuffle_rounds(ex2, cols, n, nullable=nullable):
        cnt = sc[:, 0].tolist()
        part = [rows_of[q][cursor[q]:cursor[q] + cnt[q]] for q in range(P)]
        for c, arr in enumerate(arrays):
            bs = layout(cnt, [int(lengths(arr)[r].sum()) for r in part])[1] if is_var(arr.type) else [None] * P
            for q in range(P):
                check_segment(ctx, outs[c], int(ss[q, 0]), cnt[q], arr, part[q], bs[q], f"round column {c} partition {q}")
        cursor = [a + b for a, b in zip(cursor, cnt)]
    assert cursor == counts.tolist() and node.last_stream_stats["rounds"] >= 2
    ex2.close()


# ------------------------------------------------------------------------------------------------ NCCL-mode lanes ----

@pytest.mark.parametrize("offset", [0, 37], ids=["whole", "sliced"])
def test_nccl_mode_lanes_past_one_grid_pass(ctx, offset):
    """dfd_shuffle_device(EXCHANGE_NCCL) at n > LANE_GRID_CAP * LANE_BLOCK rows, n % 32 != 0: k_bits_to_bytes,
    k_bytes_to_bits and k_offsets_to_lengths loop a second time over their grid and k_bytes_to_bits writes a partial
    last word.  Keys from a 20-value domain leave partitions of 48 empty: k_var_dest_bytes on empty runs."""
    n, P = LANE_ONE_PASS + 251_459, 48
    assert n > LANE_ONE_PASS and n % 32
    rng = np.random.Generator(np.random.PCG64(13))
    m = n + offset
    key = pa.array(rng.choice(rng.integers(0, 1 << 40, 20), m), mask=rng.random(m) < 0.03)
    arrays = [key, pa.array(rng.random(m) < 0.5, mask=rng.random(m) < 0.2), strings(rng, m, 30, pa.string(), 0.1),
              strings(rng, m, 10, pa.large_string(), 0.15), strings(rng, m, 17, pa.binary(), 0.05)]
    arrays = [a.slice(offset) for a in arrays]
    dest = orc.partition_ids([arrays[0]], n, P)
    order, ref = expected_partitions(dest, P)
    assert (np.diff(ref) == 0).any() and (np.diff(ref) > 0).sum() >= 2
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    assert all(c.validity for c in in_cols) and all(c.offset == offset for c in in_cols)
    out_cols = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in in_cols]
    outs, starts = node.shuffle(ex, in_cols, n, nv.EXCHANGE_NCCL, out_cols, n)
    assert np.array_equal(starts, ref)
    idx = pa.array(order)
    for c, arr in enumerate(arrays):
        if is_var(arr.type):  # raw offsets before anything is built from them
            ow = 8 if pa.types.is_large_string(arr.type) else 4
            off = grab(ctx, outs[c].offsets, (n + 1) * ow).view(np.int64 if ow == 8 else np.int32).astype(np.int64)
            want = np.zeros(n + 1, dtype=np.int64)
            np.cumsum(lengths(arr)[order], out=want[1:])
            assert np.array_equal(off, want), (c, arr.type)
        assert outs[c].to_arrow(ctx, 0, n).equals(arr.take(idx)), (c, arr.type)
    ex.close()


# ------------------------------------------------------------------------------- the int32 limit of Utf8 offsets ----

class Budget:
    """Skip unless `gib` + 2 GiB of device memory is free; report wall time and the drop in free memory."""

    def __init__(self, name, gib):
        self.name, self.gib = name, gib

    def __enter__(self):
        import torch

        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        if free < (self.gib + 2) * GiB:
            pytest.skip(f"{self.name} needs {self.gib + 2} GiB of free device memory, {free / GiB:.1f} GiB is free")
        self.free0, self.low, self.t0 = free, free, time.perf_counter()
        return self

    def sample(self):
        import torch

        torch.cuda.synchronize()
        self.low = min(self.low, torch.cuda.mem_get_info()[0])

    def __exit__(self, *exc):
        import torch

        self.sample()
        gc.collect()
        torch.cuda.empty_cache()
        print(f"\n[exchange limits] {self.name}: {time.perf_counter() - self.t0:.1f} s, peak {(self.free0 - self.low) / GiB:.2f} GiB")
        return False


def big_string_column(lens, kind):
    """A device string column of the given row lengths; byte p of its data is p % 251 (a shifted byte shows)."""
    import torch

    off = torch.zeros(len(lens) + 1, dtype=torch.int64)
    torch.cumsum(torch.from_numpy(lens), 0, out=off[1:])
    total = int(off[-1])
    data = torch.arange(251, dtype=torch.uint8, device="cuda").repeat(total // 251 + 1)[:total].contiguous()
    odt = torch.int64 if kind == nv.COL_LARGE_UTF8 else torch.int32
    d_off = off.to(odt).cuda()
    typ = {nv.COL_UTF8: pa.string(), nv.COL_BINARY: pa.binary(), nv.COL_LARGE_UTF8: pa.large_string()}[kind]
    return dfd.DeviceColumn(kind, 0, data.data_ptr(), d_off.data_ptr(), 0, 0, len(lens), (data, d_off), typ, total), off.numpy()


def check_big_segments(ctx, col, seg_starts, seg_rows, in_off, ow):
    """Segments of a big string column: raw offsets first (as int64 against the layout), then every byte, chunk by chunk."""
    seg_bytes = [int(in_off[r[-1] + 1] - in_off[r[0]]) if len(r) else 0 for r in seg_rows]
    _, bs = layout([len(r) for r in seg_rows], seg_bytes)
    for j, rows in enumerate(seg_rows):
        if not len(rows):
            continue
        k = len(rows)
        off = grab(ctx, col.offsets + int(seg_starts[j]) * ow, (k + 1) * ow).view(np.int64 if ow == 8 else np.int32).astype(np.int64)
        want = in_off[rows[0]:rows[-1] + 2] - in_off[rows[0]] + bs[j]  # (a segment's rows are consecutive here)
        bad = np.nonzero(off != want)[0]
        assert not len(bad), f"segment {j}: raw offsets differ at {len(bad)} of {k + 1} entries, first at {bad[0]}: got {off[bad[0]]}, want {want[bad[0]]}"
        step = 1 << 28
        for a in range(0, seg_bytes[j], step):
            b = min(seg_bytes[j], a + step)
            got = grab(ctx, col.values + bs[j] + a, b - a)
            exp = ((np.arange(a, b, dtype=np.int64) + int(in_off[rows[0]])) % 251).astype(np.uint8)
            assert np.array_equal(got, exp), f"segment {j}: bytes [{a}, {b})"


def gather_big(ctx, col, starts, window):
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(window)
    co = dfd.NetworkCoalesceExec.try_new(len(starts) - 1, uuid.uuid4(), 1, 1, 1)
    try:
        return ex, co.gather(ex, [col], starts, nullable=[False])
    except dfd.DfdError:
        ex.close()
        raise


P_LIMIT = 64
ROWS_PER_SLICE = 1024


def limit_lengths(total_bytes):
    """P_LIMIT slices of ROWS_PER_SLICE rows whose byte counts are == 1 mod 16 (15 bytes of padding after each of the
    first P_LIMIT - 1) and add up to total_bytes."""
    per = total_bytes // P_LIMIT
    seg = [per - (per % 16) + 1] * (P_LIMIT - 1)
    seg.append(total_bytes - sum(seg))
    lens = np.empty(P_LIMIT * ROWS_PER_SLICE, dtype=np.int64)
    for j, b in enumerate(seg):
        q, r = divmod(b, ROWS_PER_SLICE)
        lens[j * ROWS_PER_SLICE:(j + 1) * ROWS_PER_SLICE] = q
        lens[j * ROWS_PER_SLICE:j * ROWS_PER_SLICE + r] += 1
    assert all(b % 16 == 1 for b in seg[:-1]) and int(lens.sum()) == total_bytes
    return lens, seg


@pytest.mark.parametrize("kind", [nv.COL_UTF8, nv.COL_BINARY], ids=["utf8", "binary"])
def test_gather_refuses_int32_offsets_past_int32_max(ctx, kind):
    """64 slices whose bytes plus 15 bytes of padding between them end at INT32_MAX + 445: DFD_ERR_CAPACITY.  Accepting
    it would leave the last segments' int32 offsets wrapped negative."""
    total = INT32_MAX - 500
    with Budget(f"gather of {total} {'Utf8' if kind == nv.COL_UTF8 else 'Binary'} bytes", 7) as bud:
        lens, seg = limit_lengths(total)
        starts = list(range(0, len(lens) + 1, ROWS_PER_SLICE))
        assert max_offset([ROWS_PER_SLICE] * P_LIMIT, seg) == total + 15 * (P_LIMIT - 1) > INT32_MAX
        col, in_off = big_string_column(lens, kind)
        try:
            ex, (outs, ss, sc) = gather_big(ctx, col, starts, total + (64 << 20))
        except dfd.DfdError as e:
            assert e.status == 7 and "int32" in e.message, e
        else:  # accepted: the offsets must still be right (they cannot be: this fails on the wrapped values)
            bud.sample()
            check_big_segments(ctx, outs[0], ss, [np.arange(a, a + ROWS_PER_SLICE) for a in starts[:-1]], in_off, 4)
            ex.close()
            pytest.fail("a Utf8 / Binary segment layout past INT32_MAX was accepted")
        bud.sample()
        del col


def test_gather_accepts_offsets_ending_at_exactly_int32_max(ctx):
    """Bytes plus padding end at exactly INT32_MAX: accepted, and the last offset is INT32_MAX."""
    total = INT32_MAX - 15 * (P_LIMIT - 1)
    with Budget("gather ending at INT32_MAX", 7) as bud:
        lens, seg = limit_lengths(total)
        starts = list(range(0, len(lens) + 1, ROWS_PER_SLICE))
        assert max_offset([ROWS_PER_SLICE] * P_LIMIT, seg) == INT32_MAX
        col, in_off = big_string_column(lens, nv.COL_UTF8)
        ex, (outs, ss, sc) = gather_big(ctx, col, starts, total + (64 << 20))
        bud.sample()
        last = grab(ctx, outs[0].offsets + (int(ss[-1]) + ROWS_PER_SLICE) * 4, 4).view(np.int32)[0]
        assert int(last) == INT32_MAX
        check_big_segments(ctx, outs[0], ss, [np.arange(a, a + ROWS_PER_SLICE) for a in starts[:-1]], in_off, 4)
        ex.close()
        del col


def test_gather_large_utf8_past_int32_max(ctx):
    """LargeUtf8 at the size Utf8 refuses: int64 offsets, accepted, offsets past INT32_MAX."""
    total = INT32_MAX - 500
    with Budget("gather of LargeUtf8 past INT32_MAX", 8) as bud:
        lens, seg = limit_lengths(total)
        starts = list(range(0, len(lens) + 1, ROWS_PER_SLICE))
        col, in_off = big_string_column(lens, nv.COL_LARGE_UTF8)
        ex, (outs, ss, sc) = gather_big(ctx, col, starts, total + (64 << 20))
        bud.sample()
        check_big_segments(ctx, outs[0], ss, [np.arange(a, a + ROWS_PER_SLICE) for a in starts[:-1]], in_off, 8)
        last = grab(ctx, outs[0].offsets + (int(ss[-1]) + ROWS_PER_SLICE) * 8, 8).view(np.int64)[0]
        assert int(last) > INT32_MAX
        ex.close()
        del col


def test_shuffle_of_int32_max_utf8_bytes_refused_then_delivered_in_rounds(ctx):
    """A Utf8 column of INT32_MAX - 100 bytes over 64 partitions: shuffle_onepass refuses it (the padding of the hashed
    partitions' byte counts takes the offsets past INT32_MAX), and shuffle_rounds delivers it byte for byte in >= 2
    rounds."""
    import torch

    total, n = INT32_MAX - 100, 1 << 21
    with Budget("shuffle of INT32_MAX - 100 Utf8 bytes", 12) as bud:
        rng = np.random.Generator(np.random.PCG64(99))
        lens = rng.integers(900, 1148, n).astype(np.int64)
        lens += (total - int(lens.sum())) // n
        lens[:total - int(lens.sum())] += 1
        assert int(lens.sum()) == total
        key_np = rng.integers(-(1 << 15), 1 << 15, n).astype(np.int16)
        dest = dest_lut("i16", P_LIMIT)[key_np.view(np.uint16)]
        order, ref = expected_partitions(dest, P_LIMIT)
        rows_of = [order[ref[q]:ref[q + 1]] for q in range(P_LIMIT)]
        seg_bytes = [int(lens[r].sum()) for r in rows_of]
        assert max_offset(np.diff(ref).tolist(), seg_bytes) > INT32_MAX
        col, in_off = big_string_column(lens, nv.COL_UTF8)
        key = torch.from_numpy(key_np).cuda()
        cols = [dfd.DeviceColumn.from_torch(key), col]
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P_LIMIT), uuid.uuid4(), 1, 1, 1)
        ex = dfd.ShuffleExchange(ctx, 0, 1, None)
        ex.setup_window(total + (256 << 20))
        refused = False
        try:
            node.shuffle_onepass(ex, cols, n, nullable=[False, False])
            outs, ss, sc = node.collect(ex)
        except dfd.DfdError as e:
            assert e.status == 7 and "int32" in e.message, e
            refused = True
        bud.sample()
        if not refused:  # accepted: the raw offsets must still be right (they cannot be)
            check_rows_and_bytes(ctx, outs[1], ss[:, 0], [r.tolist() for r in rows_of], lens, in_off)
            pytest.fail("a Utf8 segment layout past INT32_MAX was accepted")
        cursor = [0] * P_LIMIT
        for outs, ss, sc in node.shuffle_rounds(ex, cols, n, nullable=[False, False]):
            cnt = sc[:, 0].tolist()
            part = [rows_of[q][cursor[q]:cursor[q] + cnt[q]] for q in range(P_LIMIT)]
            got_key = grab(ctx, outs[0].values, 2 * (int(ss[-1, 0]) + cnt[-1])).view(np.int16)
            for q in range(P_LIMIT):
                assert np.array_equal(got_key[int(ss[q, 0]):int(ss[q, 0]) + cnt[q]], key_np[part[q]]), q
            check_rows_and_bytes(ctx, outs[1], ss[:, 0], part, lens, in_off)
            cursor = [a + b for a, b in zip(cursor, cnt)]
            bud.sample()
        assert cursor == np.diff(ref).tolist() and node.last_stream_stats["rounds"] >= 2
        ex.close()
        del col, key, cols


def check_rows_and_bytes(ctx, col, seg_starts, seg_rows, lens, in_off):
    """Utf8 segments of arbitrary source rows: raw offsets against the layout, then every row's bytes (p % 251 pattern)."""
    seg_bytes = [int(lens[r].sum()) for r in seg_rows]
    _, bs = layout([len(r) for r in seg_rows], seg_bytes)
    for j, rows in enumerate(seg_rows):
        k = len(rows)
        if not k:
            continue
        off = grab(ctx, col.offsets + int(seg_starts[j]) * 4, (k + 1) * 4).view(np.int32).astype(np.int64)
        want = np.zeros(k + 1, dtype=np.int64)
        np.cumsum(lens[rows], out=want[1:])
        want += bs[j]
        bad = np.nonzero(off != want)[0]
        assert not len(bad), f"segment {j}: raw offsets differ at {len(bad)} of {k + 1} entries, first at {bad[0]}: got {off[bad[0]]}, want {want[bad[0]]}"
        got = grab(ctx, col.values + bs[j], seg_bytes[j])
        src = np.repeat(in_off[rows] - want[:-1], lens[rows])  # input position - output position, per output byte
        exp = ((np.arange(bs[j], bs[j] + seg_bytes[j], dtype=np.int64) + src) % 251).astype(np.uint8)
        assert np.array_equal(got, exp), f"segment {j}: bytes"
