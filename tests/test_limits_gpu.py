"""GPU parity tests at the 32-bit limits of the C ABI: up to 2^32 - 1 rows per dense call, single-pass regions up to
N * region_rows = 2^32 - 2 output rows, string offset scans of more than one round (> 2 097 152 rows), LargeUtf8 byte
offsets past 2^32 and a Utf8 column of exactly 2^31 - 1 bytes, the same two through dfd_shuffle_host, whose string offsets
continue across chunks; and the argument checks just past each limit.

A row-by-row oracle does not scale to 4 G rows, so the large cases draw keys from a small domain (tests.util
domain_values) whose destinations the C oracle computes once; on the GPU a row's destination is then LUT[key].
Destination p must hold the input rows with dest == p, in input order; the check runs chunk by chunk of input rows,
keeping a cursor per destination, over every column, validity bit and string byte.  Where equal keys could be
swapped unseen, a payload derived from the row id shows a stability error.

Each large case first reads the free device memory and skips, naming the amount, if its budget plus 2 GiB is not free;
it runs on its own WorkerContext, whose scratch is released with it, and frees its tensors before returning.  The
dfd_shuffle_host cases also skip, naming the amount, when the host has too little available memory for their host
buffers.  On one H100 80GB HBM3 at a 700 W power limit the module takes about 30 s, at most about 44 GiB of device
memory and 14 GiB of host memory."""
import gc
import time

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from oracle import oracle as orc
from tests.util import PARTITION_MAX_ROWS, REDUCE_MAX_ROWS, dest_lut, domain_values, expected_partitions, onepass_regions_accepted

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

GiB = 1 << 30
CHUNK = 1 << 27  # input rows per verification step (temporaries stay under ~1 GiB)
SCAN_ROUND = 1024 * 2048  # rows one pass of k_var_scan_block_sums covers (1024 blocks of 2048 rows)


# ------------------------------------------------------------------ harness ----

class Budget:
    """Skip unless `gib` + 2 GiB of device memory is free; report wall time and the drop in free memory."""

    def __init__(self, name, gib):
        self.name, self.gib = name, gib

    def __enter__(self):
        gc.collect()  # (buffers of the previous case, so that their release does not hide this case's use)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        if free < (self.gib + 2) * GiB:
            pytest.skip(f"{self.name} needs {self.gib + 2} GiB of free device memory, {free / GiB:.1f} GiB is free")
        self.free0, self.low, self.t0 = free, free, time.perf_counter()
        return self

    def sample(self):
        torch.cuda.synchronize()
        self.low = min(self.low, torch.cuda.mem_get_info()[0])

    def __exit__(self, *exc):
        self.sample()
        torch.cuda.empty_cache()
        print(f"\n[limits] {self.name}: {time.perf_counter() - self.t0:.1f} s, peak {(self.free0 - self.low) / GiB:.2f} GiB")
        return False


def lut_of(kind, N):
    return torch.from_numpy(dest_lut(kind, N)).cuda()


def key_index(key):
    """LUT index of a key tensor chunk (domain_values order)."""
    return key.to(torch.int32) & 0xFFFF if key.dtype in (torch.int16,) else key.to(torch.int32)


_SHIFTS = None


def bits(bm, a, b):
    """Rows [a, b) of an LSB-first bitmap (uint8 tensor) as a bool tensor."""
    global _SHIFTS
    if _SHIFTS is None:
        _SHIFTS = torch.arange(8, dtype=torch.uint8, device="cuda")
    lo = a >> 3
    by = bm[lo:(b + 7) >> 3]
    return ((by.unsqueeze(1) >> _SHIFTS) & 1).flatten()[a - 8 * lo:b - 8 * lo].bool()


def bitmap_bytes(rows):
    return max((rows + 31) // 32 * 4, 4)


def fixed_col(t):
    return dfd.DeviceColumn.from_torch(t)


def bit_col(kind, values, validity, n):
    """A COL_BOOL column (values = bitmap) or a nullable fixed column (values = tensor, validity = bitmap)."""
    if kind == nv.COL_BOOL:
        return dfd.DeviceColumn(nv.COL_BOOL, 0, values.data_ptr(), 0, validity.data_ptr() if validity is not None else 0, 0, n, (values, validity))
    return dfd.DeviceColumn(nv.COL_FIXED, values.element_size(), values.data_ptr(), 0, validity.data_ptr(), 0, n, (values, validity))


def check_scatter(n, N, starts, counts, dest_of, cols, budget=None):
    """Destination p is rows [starts[p], starts[p] + counts[p]) of every output; it must hold, in input order, the input
    rows r with dest_of(r) == p.  dest_of(a, b) -> int32 tensor of rows [a, b); cols = [(input(a, b), output(a, b))]
    of row ranges (values, or bool tensors for bits)."""
    cursor = [int(s) for s in starts]
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        d = dest_of(a, b)
        ins = [get_in(a, b) for get_in, _ in cols]
        for p in range(N):
            m = d == p
            k = int(m.sum())
            if k == 0:
                continue
            o = cursor[p]
            for c, ((_, get_out), x) in enumerate(zip(cols, ins)):
                assert torch.equal(x[m], get_out(o, o + k)), f"destination {p}, column {c}, input rows [{a}, {b})"
            cursor[p] += k
        del d, ins
        if budget is not None and a == 0:
            budget.sample()
    assert [c - int(s) for c, s in zip(cursor, starts)] == [int(c) for c in counts]
    assert sum(int(c) for c in counts) == n


def dense(starts, counts):
    return int(starts[0]) == 0 and all(int(starts[p + 1]) == int(starts[p] + counts[p]) for p in range(len(counts) - 1))


def fill_chunks(t, fn):
    """t[a:b] = fn(a, b) chunk by chunk (generation temporaries stay small)."""
    for a in range(0, t.numel(), CHUNK):
        b = min(t.numel(), a + CHUNK)
        t[a:b] = fn(a, b)


def rows(a, b):
    return torch.arange(a, b, dtype=torch.int64, device="cuda")


def row_payload(a, b):
    """int8 payload derived from the row id: a reordering of equal keys changes it."""
    return (rows(a, b) % 251).to(torch.int8)


# ------------------------------------------------- case 8: the limits ----

def small_col(ctx):
    return dfd.DeviceColumn.from_arrow(ctx, pa.array(np.arange(64, dtype=np.int64)))


def test_partition_refuses_2_pow_32_rows_before_touching_memory(ctx):
    """n = 2^32 is one row past the dense cap: DFD_ERR_UNSUPPORTED from the argument check, with 64-row buffers that the
    call would overrun if it read or launched anything."""
    col = small_col(ctx)
    out = dfd.DeviceColumn.empty_like(ctx, col, 64)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    before = ctx.metrics()["kernel_launches"]
    with pytest.raises(dfd.DfdError) as e:
        part.partition([col], PARTITION_MAX_ROWS + 1, [out])
    assert e.value.status == 6, e.value
    with pytest.raises(dfd.DfdError) as e:
        part.partition_onepass([col], PARTITION_MAX_ROWS + 1, 1 << 29, [out])  # 2^29 * 8 = 2^32 rows of regions
    assert e.value.status == 6, e.value
    assert ctx.metrics()["kernel_launches"] == before
    _, starts = part.partition([col], 64, [out])  # the partitioner still works
    assert int(starts[-1]) == 64


@pytest.mark.parametrize("region_rows,N", [((1 << 32) - 1, 1), (1_431_655_765, 3), (1 << 31, 2)])
def test_onepass_refuses_regions_of_2_pow_32_minus_1_rows(ctx, region_rows, N):
    """N * region_rows = 2^32 - 1 (0xffffffff, the kernel's empty-slot value; 1 x (2^32 - 1) and 3 x 1 431 655 765) and
    2^32 (2 x 2^31): DFD_ERR_UNSUPPORTED before any launch.  One region row less is accepted (the large cases below)."""
    assert not onepass_regions_accepted(region_rows, N, 64) and region_rows * N >= (1 << 32) - 1
    col = small_col(ctx)
    out = dfd.DeviceColumn.empty_like(ctx, col, 64)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    before = ctx.metrics()["kernel_launches"]
    with pytest.raises(dfd.DfdError) as e:
        part.partition_onepass([col], 64, region_rows, [out])
    assert e.value.status == 6, e.value
    assert ctx.metrics()["kernel_launches"] == before


def test_partial_reduce_refuses_more_than_2_pow_31_rows(ctx):
    """n = 2^31 + 1 would need a 2^33-slot group table behind a 32-bit slot mask: DFD_ERR_UNSUPPORTED before anything is
    allocated (64-row buffers; a launch would overrun them).  2^32 - 1 rows and more stay DFD_ERR_INVALID_ARGUMENT."""
    keys = dfd.DeviceColumn.from_torch(torch.arange(64, dtype=torch.int64, device="cuda"))
    vals = dfd.DeviceColumn.from_torch(torch.ones(64, dtype=torch.int64, device="cuda"))
    outs = [dfd.DeviceColumn.from_torch(torch.zeros(64, dtype=torch.int64, device="cuda")) for _ in range(2)]
    starts = torch.tensor([0, 64], dtype=torch.int64, device="cuda")
    red = dfd.PartialReduceExec(ctx, [0], [-1, nv.AGG_SUM_I64])
    torch.cuda.synchronize()
    before = ctx.metrics()["kernel_launches"]
    for n, status in ((REDUCE_MAX_ROWS + 1, 6), ((1 << 32) - 2, 6), ((1 << 32) - 1, 1)):
        with pytest.raises(dfd.DfdError) as e:
            red.reduce([keys, vals], n, starts.data_ptr(), 1, outs)
        assert e.value.status == status, (n, e.value)
    assert ctx.metrics()["kernel_launches"] == before
    _, st = red.reduce([keys, vals], 64, starts.data_ptr(), 1, outs)  # still usable, and right
    assert list(st) == [0, 64]
    got = outs[1].keep[0].cpu()
    assert bool((got == 1).all())


# ------------------------------------------ case 5: multi-round offset scans ----

N_SCAN = SCAN_ROUND + (1 << 20) + 7  # 1537 scan blocks: the carry loop runs a second round


def ascii_strings(rng, n, max_len, typ, null_frac=0.0):
    lens = rng.integers(0, max_len + 1, n).astype(np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    data = rng.integers(97, 123, int(off[-1]), dtype=np.uint8)
    odt = np.int64 if typ == pa.large_string() else np.int32
    validity = None
    if null_frac:
        validity = pa.py_buffer(np.packbits(rng.random(n) >= null_frac, bitorder="little").tobytes())
    arr = pa.Array.from_buffers(typ, n, [validity, pa.py_buffer(off.astype(odt).tobytes()), pa.py_buffer(data.tobytes())])
    arr.validate(full=True)
    return arr


def scan_table():
    rng = np.random.Generator(np.random.PCG64(55))
    key = ascii_strings(rng, N_SCAN, 6, pa.string(), null_frac=0.1)  # nullable Utf8 key (about 300k distinct values)
    binp = ascii_strings(rng, N_SCAN, 9, pa.binary())
    large = ascii_strings(rng, N_SCAN, 5, pa.large_string(), null_frac=0.2)
    return [key, binp, large]


def check_arrow_partitions(ctx, arrays, outs, starts, counts, N):
    n = len(arrays[0])
    order, ref_starts = expected_partitions(orc.partition_ids([arrays[0]], n, N), N)
    assert np.array_equal(np.asarray(counts), np.diff(ref_starts)), (counts, np.diff(ref_starts))
    assert dense(starts, counts)
    idx = pa.array(order)
    for c, arr in enumerate(arrays):
        got = outs[c].to_arrow(ctx, 0, n)
        got.validate(full=True)
        assert got.equals(arr.take(idx)), (c, arr.type)


def test_multi_round_scan_two_pass_and_onepass_fallback(ctx):
    """3 145 735 rows of a nullable Utf8 key, a Binary and a nullable LargeUtf8 payload: the output offsets of every
    string column are a 1537-block scan (two rounds of k_var_scan_block_sums).  Through dfd_partition_device and through
    dfd_partition_device_onepass, which takes the two-pass path for string columns."""
    arrays = scan_table()
    N = 7
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    outs, ps = part.partition(dcols, N_SCAN)
    check_arrow_partitions(ctx, arrays, outs, ps[:-1], np.diff(ps), N)
    outs1, st1, cn1 = part.partition_onepass(dcols, N_SCAN)
    check_arrow_partitions(ctx, arrays, outs1, st1, cn1, N)


def test_multi_round_scan_nccl_mode_exchange(ctx):
    """The same columns through a world-1 NCCL-mode exchange, whose receiver rebuilds string offsets from lengths with
    k_len_write_offsets (1537 blocks)."""
    import uuid

    arrays = scan_table()
    N = 6
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], N), uuid.uuid4(), 1, 1, 1)
    in_cols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in arrays]
    out_cols = [dfd.DeviceColumn.empty_like(ctx, c, N_SCAN) for c in in_cols]
    outs, starts = node.shuffle(ex, in_cols, N_SCAN, nv.EXCHANGE_NCCL, out_cols, N_SCAN)
    check_arrow_partitions(ctx, arrays, outs, starts[:-1], np.diff(starts), N)
    ex.close()


def test_multi_round_scan_host_operator_list_column(ctx):
    """Host operator, one chunk of 1 200 000 rows whose List<Utf8> column holds about 2.4 M child strings: the list
    offsets and the child offsets are both scans of more than 1024 blocks."""
    rng = np.random.Generator(np.random.PCG64(56))
    n, N = 1_200_000, 5
    n_items = rng.integers(0, 5, n)
    loff = np.zeros(n + 1, dtype=np.int32)
    np.cumsum(n_items, out=loff[1:])
    n_child = int(loff[-1])
    assert n_child > SCAN_ROUND
    child = ascii_strings(rng, n_child, 7, pa.string(), null_frac=0.05)
    tags = pa.ListArray.from_arrays(pa.array(loff), child, mask=pa.array(rng.random(n) < 0.1))
    ids = pa.array(rng.integers(-(1 << 40), 1 << 40, n), type=pa.int64())
    table = pa.table([ids, tags], names=["id", "tags"])
    ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), chunk_rows=1 << 21)
    for rb in table.to_batches(max_chunksize=1 << 18):
        ex.push_batch(rb)
    ex.finish()
    outs = [ex.execute(p).read_all() for p in range(N)]
    assert ex.stats()["rows_out"] == n
    order, starts = expected_partitions(orc.partition_ids([ids], n, N), N)
    for p in range(N):
        want = table.take(pa.array(order[starts[p]:starts[p + 1]]))
        for name in table.column_names:
            got = outs[p].column(name).combine_chunks()
            got.validate(full=True)
            assert got.equals(want.column(name).combine_chunks()), (p, name)
    ex.close()


# ------------------------------------------------ cases 1-4: rows past 2^31 ----

def test_two_pass_generic_key_at_the_row_cap():
    """n = 2^32 - 1 rows (the cap), nullable uint8 key + Boolean payload, N = 7: output rows and bitmap words past 2^31,
    the generic-key dest_cache, Barrett mod 7 and k_tile_hist's 2-word flag path."""
    n, N = PARTITION_MAX_ROWS, 7
    with Budget("two-pass generic key, 2^32 - 1 rows", 21) as bud:
        ctx = dfd.WorkerContext(0)
        g = torch.Generator(device="cuda").manual_seed(1)
        key = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
        kval = torch.randint(0, 256, (bitmap_bytes(n),), dtype=torch.uint8, device="cuda", generator=g)
        kval[:4] = 0x0F  # (rows 0-3 valid, 4-7 null, ...)
        flag = torch.randint(0, 256, (bitmap_bytes(n),), dtype=torch.uint8, device="cuda", generator=g)
        out_key = torch.empty(n, dtype=torch.uint8, device="cuda")
        out_kval = torch.empty(bitmap_bytes(n), dtype=torch.uint8, device="cuda")
        out_flag = torch.empty(bitmap_bytes(n), dtype=torch.uint8, device="cuda")
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        torch.cuda.synchronize()
        _, ps = part.partition([bit_col(nv.COL_FIXED, key, kval, n), bit_col(nv.COL_BOOL, flag, None, n)], n,
                               [bit_col(nv.COL_FIXED, out_key, out_kval, n), bit_col(nv.COL_BOOL, out_flag, None, n)])
        bud.sample()
        ctx.close()
        lut = lut_of("u8", N)
        starts, counts = ps[:-1], np.diff(ps)
        assert int(ps[-1]) == n and dense(starts, counts)
        check_scatter(n, N, starts, counts,
                      lambda a, b: torch.where(bits(kval, a, b), lut[key_index(key[a:b])], 0),
                      [(lambda a, b: torch.where(bits(kval, a, b), key[a:b], 0),
                        lambda a, b: torch.where(bits(out_kval, a, b), out_key[a:b], 0)),
                       (lambda a, b: bits(kval, a, b), lambda a, b: bits(out_kval, a, b)),
                       (lambda a, b: bits(flag, a, b), lambda a, b: bits(out_flag, a, b))], bud)
        del key, kval, flag, out_key, out_kval, out_flag


def test_two_pass_fast_i64_key_past_int32_max():
    """n = 2^31 + 12 345 rows of a non-null Int64 key (the FAST_I64 instantiation) + an int8 row-id payload, N = 8."""
    n, N = (1 << 31) + 12_345, 8
    with Budget("two-pass FAST_I64, 2^31 + 12 345 rows", 44) as bud:
        ctx = dfd.WorkerContext(0)
        g = torch.Generator(device="cuda").manual_seed(2)
        table = torch.from_numpy(domain_values("i64")).cuda()
        idx = torch.randint(-(1 << 15), 1 << 15, (n,), dtype=torch.int16, device="cuda", generator=g)
        key = torch.empty(n, dtype=torch.int64, device="cuda")
        fill_chunks(key, lambda a, b: table[key_index(idx[a:b])])
        pay = torch.empty(n, dtype=torch.int8, device="cuda")
        fill_chunks(pay, row_payload)
        out_key = torch.empty(n, dtype=torch.int64, device="cuda")
        out_pay = torch.empty(n, dtype=torch.int8, device="cuda")
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        torch.cuda.synchronize()
        _, ps = part.partition([fixed_col(key), fixed_col(pay)], n, [fixed_col(out_key), fixed_col(out_pay)])
        bud.sample()
        ctx.close()
        lut = lut_of("i64", N)
        starts, counts = ps[:-1], np.diff(ps)
        assert int(ps[-1]) == n and dense(starts, counts)
        check_scatter(n, N, starts, counts, lambda a, b: lut[key_index(idx[a:b])],
                      [(lambda a, b: key[a:b], lambda a, b: out_key[a:b]), (lambda a, b: pay[a:b], lambda a, b: out_pay[a:b])], bud)
        del idx, key, pay, out_key, out_pay


def onepass_case(name, gib, n, N, region_rows, kind, make_key, seed, expect_rerun):
    """Single-pass partition of (key, int8 row-id payload) into N regions of region_rows rows; checked with the LUT."""
    assert onepass_regions_accepted(region_rows, N, n)
    with Budget(name, gib) as bud:
        ctx = dfd.WorkerContext(0)
        g = torch.Generator(device="cuda").manual_seed(seed)
        key = make_key(n, g)
        pay = torch.empty(n, dtype=torch.int8, device="cuda")
        fill_chunks(pay, row_payload)
        cap = N * region_rows
        out_key = torch.empty(cap, dtype=key.dtype, device="cuda")
        out_pay = torch.empty(cap, dtype=torch.int8, device="cuda")
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        torch.cuda.synchronize()
        reruns = ctx.metrics()["onepass_reruns"]
        _, starts, counts = part.partition_onepass([fixed_col(key), fixed_col(pay)], n, region_rows, [fixed_col(out_key), fixed_col(out_pay)])
        assert ctx.metrics()["onepass_reruns"] == reruns + (1 if expect_rerun else 0)
        bud.sample()
        ctx.close()
        if expect_rerun:
            assert dense(starts, counts) and int(counts.max()) > region_rows
        else:
            assert list(starts) == [p * region_rows for p in range(N)]
        assert int((starts + counts).max()) > 1 << 31  # the output rows cross INT32_MAX
        lut = lut_of(kind, N)
        check_scatter(n, N, starts, counts, lambda a, b: lut[key_index(key[a:b])],
                      [(lambda a, b: key[a:b], lambda a, b: out_key[a:b]), (lambda a, b: pay[a:b], lambda a, b: out_pay[a:b])], bud)
        del key, pay, out_key, out_pay


def test_onepass_regions_spanning_2_pow_32_minus_4_rows():
    """N = 3 regions of 1 431 655 764 rows (3 * 1 431 655 764 = 2^32 - 4), 3.9e9 rows of an int16 key: output rows past
    2^31 in the single-pass write-out, int16 and int8 columns in one launch each."""
    region_rows = 1_431_655_764
    assert 3 * region_rows == (1 << 32) - 4
    onepass_case("single-pass regions, 3.9e9 rows", 26, 3_900_000_000, 3, region_rows, "i16",
                 lambda n, g: torch.randint(-(1 << 15), 1 << 15, (n,), dtype=torch.int16, device="cuda", generator=g), 3, False)


def test_onepass_overflow_reruns_dense_past_2_pow_31():
    """N = 2 regions of 2^31 - 1 rows (2^32 - 2, the largest accepted product), n = 2^32 - 3 rows of which about 60 % go
    to destination 0: that region overflows, and the exact dense re-run writes destination 1 from row ~2.58e9 on."""
    lut = dest_lut("u8", 2)
    dom = domain_values("u8")
    pick = np.concatenate([np.resize(dom[lut == 0], 600), np.resize(dom[lut == 1], 400)])  # 60 % of draws -> destination 0
    pick_t = torch.from_numpy(pick).cuda()

    def make_key(n, g):
        key = torch.empty(n, dtype=torch.uint8, device="cuda")
        fill_chunks(key, lambda a, b: pick_t[torch.randint(0, len(pick), (b - a,), dtype=torch.int32, device="cuda", generator=g)])
        return key

    onepass_case("single-pass overflow + dense re-run, 2^32 - 3 rows", 19, (1 << 32) - 3, 2, (1 << 31) - 1, "u8", make_key, 4, True)


# ------------------------------------- cases 6-7: string bytes past 2^31 / 2^32 ----

def row_bytes(r, j):
    """Byte j of the string of row r: its 8-byte little-endian row id, then bytes derived from (r, j)."""
    head = (r >> (8 * j.clamp(max=7))) & 0xFF
    return torch.where(j < 8, head, (r * 131 + j * 29 + (r >> 11)) & 0xFF).to(torch.uint8)


def string_bytes(src_rows, lens):
    """The bytes of the strings of rows src_rows (int64 tensor), back to back."""
    r = torch.repeat_interleave(src_rows, lens)
    first = torch.cumsum(lens, 0) - lens
    j = torch.arange(r.numel(), dtype=torch.int64, device="cuda") - torch.repeat_interleave(first, lens)
    return row_bytes(r, j)


def string_case(name, gib, n, N, typ, lens, seed):
    """A String column (lengths `lens`, bytes row_bytes) as payload under an int16 key.  Expected output in (destination,
    row) order by a gather; the output offsets, bytes and key are compared with it."""
    kind = nv.COL_LARGE_UTF8 if typ == "large" else nv.COL_UTF8
    odt = torch.int64 if typ == "large" else torch.int32
    with Budget(name, gib) as bud:
        ctx = dfd.WorkerContext(0)
        g = torch.Generator(device="cuda").manual_seed(seed)
        key = torch.randint(-(1 << 15), 1 << 15, (n,), dtype=torch.int16, device="cuda", generator=g)
        off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(lens, 0, out=off[1:])
        total = int(off[-1])
        data = torch.empty(total, dtype=torch.uint8, device="cuda")
        step = 1 << 15
        for a in range(0, n, step):
            b = min(n, a + step)
            data[int(off[a]):int(off[b])] = string_bytes(rows(a, b), lens[a:b])
        in_off = off.to(odt)
        del off
        out_key = torch.empty(n, dtype=torch.int16, device="cuda")
        out_off = torch.empty(n + 1, dtype=odt, device="cuda")
        out_data = torch.empty(total, dtype=torch.uint8, device="cuda")
        part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        scol = dfd.DeviceColumn(kind, 0, data.data_ptr(), in_off.data_ptr(), 0, 0, n, (data, in_off), None, total)
        ocol = dfd.DeviceColumn(kind, 0, out_data.data_ptr(), out_off.data_ptr(), 0, 0, n, (out_data, out_off), None, total)
        torch.cuda.synchronize()
        _, ps = part.partition([fixed_col(key), scol], n, [fixed_col(out_key), ocol])
        bud.sample()
        ctx.close()
        lut = lut_of("i16", N)
        dest = lut[key_index(key)].long()
        order = torch.sort(dest, stable=True).indices  # input row of every output row
        assert np.array_equal(ps, np.concatenate([[0], np.cumsum(torch.bincount(dest, minlength=N).cpu().numpy())]))
        assert torch.equal(out_key, key[order])
        want_off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(lens[order], 0, out=want_off[1:])
        assert torch.equal(out_off, want_off.to(odt)), "output offsets"
        assert int(out_off[-1]) == total
        for a in range(0, n, step):
            b = min(n, a + step)
            lo, hi = int(want_off[a]), int(want_off[b])
            assert torch.equal(out_data[lo:hi], string_bytes(order[a:b], lens[order[a:b]])), f"bytes of output rows [{a}, {b})"
        del key, data, in_off, out_key, out_off, out_data, dest, order, want_off, scol, ocol


def test_large_utf8_payload_past_4_gib():
    """n = 2^22 + 3 rows of LargeUtf8 strings of 1000-1400 bytes (about 5 GB): int64 offsets and u64 block sums past 2^32,
    string starts at every alignment, so k_var_copy_bytes takes both its co-aligned 8-byte and its byte-wise branch."""
    n = (1 << 22) + 3
    g = torch.Generator(device="cuda").manual_seed(6)
    lens = torch.randint(1000, 1401, (n,), dtype=torch.int64, device="cuda", generator=g)
    assert int(lens.sum()) > 1 << 32
    string_case("LargeUtf8 payload past 4 GiB", 10, n, 5, "large", lens, 6)


def test_utf8_payload_of_exactly_int32_max_bytes():
    """A Utf8 payload of exactly 2^31 - 1 bytes: the last int32 output offset is INT32_MAX."""
    n = 1 << 21
    g = torch.Generator(device="cuda").manual_seed(7)
    lens = torch.randint(950, 1050, (n,), dtype=torch.int64, device="cuda", generator=g)
    deficit = (1 << 31) - 1 - int(lens.sum())
    assert deficit >= 0
    lens += deficit // n
    lens[:deficit % n] += 1
    assert int(lens.sum()) == (1 << 31) - 1
    string_case("Utf8 payload of 2^31 - 1 bytes", 5, n, 4, "utf8", lens, 7)


# ------------------------------- dfd_shuffle_host: string offsets continued across chunks ----

def host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def host_shuffle_string_case(name, gib, host_gib, typ, total, n, n_chunks, seed):
    """dfd_shuffle_host at world 1 of (int16 key, String of `total` bytes in rows of about 1000 bytes) through
    Hash([0], 4), in n_chunks chunks through a 448 MiB receive window.  The expected output is the rows of each chunk in
    (destination, row) order, destination = LUT[key]; offsets, bytes and keys are compared with it on the device."""
    import uuid

    from tests import host_shuffle_util as H

    if host_available() < host_gib * GiB:
        pytest.skip(f"{name} needs {host_gib} GiB of available host memory, {host_available() / GiB:.1f} GiB is available")
    P = 4
    odt, kind = (np.int64, pa.large_string()) if typ == "large" else (np.int32, pa.string())
    with Budget(name, gib) as bud:
        ctx = dfd.WorkerContext(0)
        g = torch.Generator(device="cuda").manual_seed(seed)
        key = torch.randint(-(1 << 15), 1 << 15, (n,), dtype=torch.int16, device="cuda", generator=g)
        lens = torch.randint(950, 1050, (n,), dtype=torch.int64, device="cuda", generator=g)
        deficit = total - int(lens.sum())
        lens += deficit // n
        lens[:deficit % n] += 1
        assert int(lens.sum()) == total and int(lens.min()) > 0
        off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(lens, 0, out=off[1:])
        data = np.empty(total, dtype=np.uint8)
        host_data = torch.from_numpy(data)
        step = 1 << 15
        for a in range(0, n, step):
            b = min(n, a + step)
            host_data[int(off[a]):int(off[b])].copy_(string_bytes(rows(a, b), lens[a:b]))
        key_h = key.cpu().numpy()
        arrays = [pa.array(key_h), pa.Array.from_buffers(kind, n, [None, pa.py_buffer(off.cpu().numpy().astype(odt)), pa.py_buffer(data)])]
        out = H.HostOut([a.type for a in arrays], n, [False, False], {1: total})
        ex = dfd.ShuffleExchange(ctx, 0, 1, None)
        ex.setup_window(448 << 20)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], P), uuid.uuid4(), 1, 1, 1)
        cps = node.shuffle_host(ex, H.in_columns(arrays, n), n, n_chunks, out.cols, n)
        bud.sample()
        ex.close()
        ctx.close()
        del arrays, host_data, data
        # expected: chunk by chunk, rows by destination in input order
        lut = lut_of("i16", P)
        dest = lut[key_index(key)].long()
        chunk = torch.zeros(n, dtype=torch.int64, device="cuda")
        for i in range(1, n_chunks):
            chunk[n * i // n_chunks:] += 1
        order = torch.sort(chunk * P + dest, stable=True).indices
        w = torch.searchsorted((chunk * P + dest)[order], torch.arange(n_chunks * P + 1, device="cuda")).cpu().numpy()
        assert np.array_equal(cps, np.stack([w[ch * P:ch * P + P + 1] for ch in range(n_chunks)]))
        kb, _ = out.bufs[(0, "values")]
        assert torch.equal(torch.from_numpy(kb[:2 * n].view(np.int16)).cuda(), key[order])
        want_off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(lens[order], 0, out=want_off[1:])
        ob, _ = out.bufs[(1, "offsets")]
        got_off = torch.from_numpy(ob[:(n + 1) * np.dtype(odt).itemsize].view(odt)).cuda().to(torch.int64)
        assert torch.equal(got_off, want_off), "output offsets"
        assert int(got_off[-1]) == total
        vb, _ = out.bufs[(1, "values")]
        for a in range(0, n, step):
            b = min(n, a + step)
            lo, hi = int(want_off[a]), int(want_off[b])
            assert torch.equal(torch.from_numpy(vb[lo:hi]).cuda(), string_bytes(order[a:b], lens[order[a:b]])), f"bytes of output rows [{a}, {b})"
        for b, cap in out.bufs.values():
            assert (b[cap:] == H.FILL).all()
        del key, lens, off, dest, chunk, order, want_off, got_off, out
    return cps


def test_host_shuffle_utf8_of_exactly_int32_max_bytes():
    """A Utf8 output of exactly 2^31 - 1 bytes delivered in 8 chunks: the int32 offsets continue across chunks up to a
    last offset of INT32_MAX, which the per-chunk check (need > INT32_MAX) accepts.  (At world 1 a Utf8 input cannot
    hold more, so the refusal one byte past needs two producers.)"""
    host_shuffle_string_case("dfd_shuffle_host, Utf8 of 2^31 - 1 bytes", 3, 6, "utf8", (1 << 31) - 1, 1 << 21, 8, 8)


def test_host_shuffle_large_utf8_past_4_gib():
    """A LargeUtf8 output of 2^32 + 2^28 bytes in 16 chunks: the int64 offsets, re-based chunk by chunk, pass 2^32."""
    host_shuffle_string_case("dfd_shuffle_host, LargeUtf8 past 4 GiB", 3, 12, "large", (1 << 32) + (1 << 28), (1 << 22) + 4_099, 16, 9)
