"""GPU tests of the host operator's device-path job-table kernels past one launch, one grid pass and one bitmap word:
k_stage_batch and k_stage_sizes (csrc/dfd_stage.cu), which assemble a chunk from device-resident input batches, and
k_emit_chunk (csrc/dfd_emit.cu), which finishes the views and list offsets of a device-resident output chunk.

Every case runs its batches host -> host, device -> host and device -> device and asserts identical streams, buffer for
buffer (the host path's staging is dfd_host_staging.h, checked against pyarrow by test_host_staging.py), and checks the
host stream's values against pyarrow: per destination, the inputs concatenated and taken in the stable order of the C
oracle's destinations.  The sizes that make a launcher split its job table or a kernel loop over its grid are derived from
the launch constants parsed out of the sources, and every case asserts the threshold, launch count or residue set it is
there to reach."""
import json
import math
import os
import re
import resource
import subprocess
import sys
from collections import Counter

import numpy as np
import pyarrow as pa
import pytest

import datafusion_distributed_b200 as dfd
from oracle import oracle as orc
from tests import device_outputs as DO
from tests.test_exec_device_input_gpu import assert_same_streams, push_device
from tests.test_exec_device_output_gpu import device_streams, host_streams
from tests.util import ROOT, expected_partitions

pytestmark = pytest.mark.gpu

CSRC = os.path.join(ROOT, "datafusion_distributed_b200", "csrc")


def _constant(source, name):
    with open(os.path.join(CSRC, source)) as f:
        m = re.search(rf"constexpr\s+int\s+{name}\s*=\s*(\d+)\s*;", f.read())
    assert m, (source, name)
    return int(m.group(1))


STAGE_BLOCK = _constant("dfd_stage.cu", "STAGE_BLOCK")
STAGE_MAX_GRID_X = _constant("dfd_stage.cu", "STAGE_MAX_GRID_X")
STAGE_MAX_JOBS = _constant("dfd_internal.h", "STAGE_MAX_JOBS")
EMIT_BLOCK = _constant("dfd_emit.cu", "EMIT_BLOCK")
EMIT_MAX_GRID_X = _constant("dfd_emit.cu", "EMIT_MAX_GRID_X")
EMIT_MAX_JOBS = _constant("dfd_emit.cu", "EMIT_MAX_JOBS")
STAGE_THREADS = STAGE_BLOCK * STAGE_MAX_GRID_X  # the most threads one k_stage_batch / k_stage_sizes launch runs
EMIT_THREADS = EMIT_BLOCK * EMIT_MAX_GRID_X     # ... and one k_emit_chunk launch
DEFAULT_CHUNK_ROWS = 4 << 20                    # dfd_repartition_exec_create's chunk_rows when none is given
KERNELS = ("k_stage_batch", "k_stage_sizes", "k_emit_chunk")


@pytest.fixture(scope="module")
def ctx(built):
    """A worker context of this module's own (as in the device-input and device-output modules); the device-output helper's
    copies go through it."""
    c = dfd.WorkerContext(0)
    DO.COPY = DO.gpu_copy(c)
    yield c
    DO.COPY = None
    c.close()


# ----------------------------------------------------------------------------------- restatement of the job tables ----

def _is_var(t):
    return pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t) or pa.types.is_large_binary(t)


def _is_view(t):
    return pa.types.is_string_view(t) or pa.types.is_binary_view(t)


def stage_jobs(field, validity):
    """Jobs stage_rows_device (dfd_exec.cu) appends for one field of one staged slice: a fixed-width or Boolean column one
    (its values), Utf8 / Binary and their Large forms two (offsets, bytes), a view column two (offsets, view bytes), a
    list four (lengths' offsets, lengths, bytes' offsets, bytes) plus two (offsets, element validity bytes) when its child
    field is nullable; plus one validity job (`validity`)."""
    t = field.type
    if pa.types.is_list(t):
        n = 4 + (2 if t.value_field.nullable else 0)
    elif _is_var(t) or _is_view(t):
        n = 2
    else:
        n = 1
    return n + (1 if validity else 0)


def size_jobs(schema):
    """measure_device (dfd_exec.cu): one k_stage_sizes job per list, view or variable-width field."""
    return sum(1 for f in schema if pa.types.is_list(f.type) or _is_view(f.type) or _is_var(f.type))


def emit_jobs(schema):
    """The emit loop of the device-output flush (dfd_exec.cu): one k_emit_chunk job per view or list field."""
    return sum(1 for f in schema if pa.types.is_list(f.type) or _is_view(f.type))


def launches(jobs, per_launch):
    return math.ceil(jobs / per_launch)


def chunk_rows_of(chunk_rows):
    """dfd_repartition_exec_create: the default, rounded up to a multiple of 64 rows."""
    r = chunk_rows or DEFAULT_CHUNK_ROWS
    return (r + 63) // 64 * 64


class Staged:
    """Restatement of the push loop (push in dfd_exec.cu) for inputs whose string bytes never cut a chunk early.
    `calls`: one entry per stage_rows_device call — (batch index, first row, rows, chunk rows before it, staging jobs,
    bitmap jobs).  A bitmap job is (field, a, b, c, n, has source): STAGE_BITS of validity or Boolean values, source bits
    [a, a + n) to chunk bits [b, b + n), chunk bits [c, b) set to one.  `chunks`: the row count of every chunk."""

    def __init__(self, schema, batches, chunk_rows):
        cap = chunk_rows_of(chunk_rows)
        self.calls, self.chunks = [], []
        rows, has_valid = 0, [False] * len(schema)
        for k, rb in enumerate(batches):
            done = 0
            while done < rb.num_rows:
                n = min(rb.num_rows - done, cap - rows)
                jobs, bits = 0, []
                for i, f in enumerate(schema):
                    col = rb.column(i)
                    valid = f.nullable and col.null_count != 0  # validity_of: the batch column's null count
                    lo = col.offset + done
                    if valid or has_valid[i]:
                        bits.append((i, lo, rows, rows if has_valid[i] else 0, n, valid))
                    if pa.types.is_boolean(f.type):
                        bits.append((i, lo, rows, rows, n, True))
                    jobs += stage_jobs(f, valid or has_valid[i])
                    has_valid[i] = has_valid[i] or valid
                self.calls.append((k, done, n, rows, jobs, bits))
                rows += n
                done += n
                if rows == cap:
                    self.chunks.append(rows)
                    rows, has_valid = 0, [False] * len(schema)
        if rows:
            self.chunks.append(rows)

    def expected_launches(self, schema, device_output):
        want = {"k_stage_batch": sum(launches(c[4], STAGE_MAX_JOBS) for c in self.calls),
                "k_stage_sizes": len(self.calls) * launches(size_jobs(schema), STAGE_MAX_JOBS)}
        want["k_emit_chunk"] = len(self.chunks) * launches(emit_jobs(schema), EMIT_MAX_JOBS) if device_output else 0
        return want


def launch_counts(fn):
    """fn() under torch.profiler with CUDA activities: (its result, launches of each of KERNELS)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return out, {k: sum(c for name, c in names.items() if k in name) for k in KERNELS}


# ------------------------------------------------------------------------------------------------ the two references ----

def device_device(ctx, schema, batches, keys, N, **opts):
    """The device -> device run: (its streams copied to the host, its stats)."""
    dd = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash(keys, N), device_output=True, **opts)
    for rb in batches:
        push_device(dd, rb)
    dd.finish()
    out = device_streams(ctx, dd, N), dd.stats()
    dd.close()
    return out


def run_all(ctx, schema, batches, keys, N, **opts):
    """host -> host, device -> host and device -> device over the same batches; asserts identical streams.  Returns the
    host -> host streams and {run: stats} of the two device-input runs."""
    part = dfd.Partitioning.Hash(keys, N)
    hh = dfd.RepartitionExec(ctx, schema, part, **opts)
    for rb in batches:
        hh.push_batch(rb)
    hh.finish()
    want = host_streams(hh, N)
    hh.close()
    dh = dfd.RepartitionExec(ctx, schema, part, **opts)
    for rb in batches:
        push_device(dh, rb)
    dh.finish()
    got, stats = host_streams(dh, N), {"device_host": dh.stats()}
    dh.close()
    assert_same_streams(want, got)
    del got
    got, stats["device_device"] = device_device(ctx, schema, batches, keys, N, **opts)
    assert_same_streams(want, got)
    for st in stats.values():
        assert st["bytes_h2d"] == 0 and st["rows_out"] == sum(b.num_rows for b in batches)
    return want, stats


def _plain(a):
    """pyarrow has no take kernel for views: compare them as their (64-bit offset) Utf8 / Binary twins."""
    if pa.types.is_string_view(a.type):
        return a.cast(pa.large_string())
    if pa.types.is_binary_view(a.type):
        return a.cast(pa.large_binary())
    return a


def check_values(schema, batches, keys, N, streams):
    """Per destination, every column of the concatenated stream equals the inputs concatenated and taken in the stable
    order of the oracle's destinations."""
    cols = [pa.concat_arrays([rb.column(i) for rb in batches]) for i in range(len(schema))]
    n = len(cols[0])
    order, starts = expected_partitions(orc.partition_ids([cols[k] for k in keys], n, N).astype(np.int64), N)
    for p in range(N):
        idx = pa.array(order[starts[p]:starts[p + 1]])
        assert sum(b.num_rows for b in streams[p]) == len(idx), p
        if not len(idx):
            continue
        for i, f in enumerate(schema):
            got = pa.concat_arrays([b.column(i) for b in streams[p]])
            assert _plain(got).equals(_plain(cols[i]).take(idx)), (p, f.name)


def check(ctx, schema, batches, keys, N, **opts):
    want, stats = run_all(ctx, schema, batches, keys, N, **opts)
    check_values(schema, batches, keys, N, want)
    return stats


# ----------------------------------------------------------------------------------------------- numpy-built inputs ----

def _bitmap(bits):
    return pa.py_buffer(np.packbits(bits, bitorder="little"))


def _nulls(rng, n, p_null):
    """(validity buffer or None, boolean valid mask)."""
    valid = rng.random(n) >= p_null if p_null else np.ones(n, dtype=bool)
    return (_bitmap(valid) if p_null else None), valid


def fixed(rng, t, n, p_null=0.0):
    """Fixed-width values of type `t` from random bytes (Decimal128: sign-extended Int64, a valid 38-digit decimal)."""
    buf, valid = _nulls(rng, n, p_null)
    if pa.types.is_decimal(t):
        lo = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
        raw = np.stack([lo, lo >> 63], axis=1)
    else:
        raw = rng.integers(0, 256, n * (t.bit_width // 8), dtype=np.uint8)
    return pa.Array.from_buffers(t, n, [buf, pa.py_buffer(raw)], null_count=int(n - valid.sum()))


def booleans(rng, n, p_null=0.0):
    buf, valid = _nulls(rng, n, p_null)
    return pa.Array.from_buffers(pa.bool_(), n, [buf, _bitmap(rng.random(n) < 0.5)], null_count=int(n - valid.sum()))


def strings(rng, t, lengths, p_null=0.0, data=None):
    """Utf8 / Binary / Large* (or, through Utf8 / Binary, a view type) with these lengths (0 under nulls) over lowercase
    ASCII bytes from one random buffer (or `data`)."""
    if _is_view(t):
        return strings(rng, pa.string() if pa.types.is_string_view(t) else pa.binary(), lengths, p_null, data).cast(t)
    n = len(lengths)
    buf, valid = _nulls(rng, n, p_null)
    lengths = np.where(valid, lengths, 0)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lengths, out=off[1:])
    if data is None:
        data = rng.integers(97, 123, int(off[-1]), dtype=np.uint8)
    wide = pa.types.is_large_string(t) or pa.types.is_large_binary(t)
    return pa.Array.from_buffers(t, n, [buf, pa.py_buffer(off.astype(np.int64 if wide else np.int32)), pa.py_buffer(data)],
                                 null_count=int(n - valid.sum()))


def lists(rng, child_type, n, max_elems, p_null=0.2, p_child_null=0.2):
    """List<child_type> (child field nullable) with 0..max_elems elements a row, nulls in the lists and in the child."""
    _, valid = _nulls(rng, n, p_null)
    counts = np.where(valid, rng.integers(0, max_elems + 1, n), 0)
    off = np.zeros(n + 1, dtype=np.int32)
    np.cumsum(counts, out=off[1:])
    ne = int(off[-1])
    child = strings(rng, child_type, rng.integers(0, 9, ne), p_child_null) if _is_var(child_type) else fixed(rng, child_type, ne, p_child_null)
    return pa.ListArray.from_arrays(pa.array(off), child, mask=pa.array(~valid))


def key_column(rng, n):
    return pa.array(rng.integers(-(1 << 62), 1 << 62, n))


def column(rng, t, n, p_null=0.2):
    if pa.types.is_list(t):
        return lists(rng, t.value_type, n, 4, p_null)
    if pa.types.is_boolean(t):
        return booleans(rng, n, p_null)
    if _is_var(t) or _is_view(t):
        return strings(rng, t, rng.integers(0, 30, n), p_null)
    return fixed(rng, t, n, p_null)


def table(rng, fields, n):
    """Int64 key `k` (non-null) and `fields` [(type, nullable)] as columns c1, c2, ...; nullable ones with nulls."""
    cols = [key_column(rng, n)] + [column(rng, t, n, 0.2 if nullable else 0.0) for t, nullable in fields]
    schema = pa.schema([pa.field("k", pa.int64(), False)] + [pa.field(f"c{i + 1}", t, nullable) for i, (t, nullable) in enumerate(fields)])
    return pa.Table.from_arrays(cols, schema=schema)


def slices(t, cuts):
    return [t.slice(a, b - a).to_batches()[0] for a, b in zip(cuts[:-1], cuts[1:])]


# ------------------------------------------------------------------------------------------------------ split tables ----

MIX = [(pa.int8(), True), (pa.int64(), True), (pa.decimal128(38, 2), True), (pa.bool_(), True), (pa.string(), True),
       (pa.large_binary(), True), (pa.string_view(), True), (pa.list_(pa.string()), True)]


def fields_for_stage_jobs(target):
    """MIX (24 jobs a slice with nulls in every column) and the key (1), then nullable Int64 columns (2 each) and at most one
    non-null Int8 (1) up to exactly `target` staging jobs."""
    rest = target - 1 - sum(stage_jobs(pa.field("x", t, n), n) for t, n in MIX)
    assert rest >= 0
    return MIX + [(pa.int64(), True)] * (rest // 2) + [(pa.int8(), False)] * (rest % 2)


VAR_KINDS = [pa.string(), pa.large_binary(), pa.string_view(), pa.list_(pa.string())]
SPLIT_CASES = {
    "small-mix": (MIX, None),
    **{f"stage-{j}-jobs": (fields_for_stage_jobs(j), j) for j in (STAGE_MAX_JOBS, STAGE_MAX_JOBS + 1, 2 * STAGE_MAX_JOBS, 2 * STAGE_MAX_JOBS + 1)},
    **{f"sizes-{j}-fields": ([(VAR_KINDS[i % 4], True) for i in range(j)], None) for j in (STAGE_MAX_JOBS + 1, 2 * STAGE_MAX_JOBS + 1)},
    f"emit-{EMIT_MAX_JOBS + 1}-fields": ([([pa.string_view(), pa.list_(pa.string())][i % 2], True) for i in range(EMIT_MAX_JOBS + 1)], None),
}


SPLIT_N, SPLIT_CHUNK_ROWS = 5, 1 << 16


def split_case_batches(case):
    fields, _ = SPLIT_CASES[case]
    rng = np.random.Generator(np.random.PCG64(sum(map(ord, case))))
    t = table(rng, fields, 2_600)
    return t.schema, slices(t, [3, 704, 1_705, 2_600])  # (sliced: non-zero column offsets)


def profile_split_cases():
    """{case: launches of KERNELS} in the device -> device run of every SPLIT_CASES case, on a context of its own."""
    c = dfd.WorkerContext(0)
    DO.COPY = DO.gpu_copy(c)
    out = {}
    for case in SPLIT_CASES:
        schema, batches = split_case_batches(case)
        _, out[case] = launch_counts(lambda: device_device(c, schema, batches, [0], SPLIT_N, chunk_rows=SPLIT_CHUNK_ROWS))
    c.close()
    return out


@pytest.fixture(scope="module")
def split_launches(built):
    """profile_split_cases() in a child process: a profiler session leaves CUPTI state behind in its process, after which
    a later module's profiler session there can come back without the kernels it ran."""
    code = "import json; from tests import test_exec_device_kernels_gpu as K; print('LAUNCHES', json.dumps(K.profile_split_cases()))"
    out = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("LAUNCHES ")][-1].split(" ", 1)[1])


@pytest.mark.parametrize("case", list(SPLIT_CASES))
def test_split_job_tables(ctx, split_launches, case):
    """Pushes whose staging, size or emit job tables fill one launch exactly, or spill into a second or third one.  A
    profiler counts the launches of every kernel in the device -> device run: ceil(jobs / table size) per push (per chunk
    for k_emit_chunk), which is more than one launch a push exactly where the table is split."""
    _, target = SPLIT_CASES[case]
    schema, batches = split_case_batches(case)
    st = Staged(schema, batches, SPLIT_CHUNK_ROWS)
    assert len(st.chunks) == 1 and len(st.calls) == 3  # every push stages once, into one chunk
    if target is not None:
        assert [c[4] for c in st.calls] == [target] * 3
    check(ctx, schema, batches, [0], SPLIT_N, chunk_rows=SPLIT_CHUNK_ROWS)
    counts = split_launches[case]
    want = st.expected_launches(schema, device_output=True)
    assert counts == want, (counts, want)
    if case.startswith("stage-") and target > STAGE_MAX_JOBS:
        assert counts["k_stage_batch"] > len(st.calls)
    if case.startswith("sizes-"):
        assert size_jobs(schema) > STAGE_MAX_JOBS and counts["k_stage_sizes"] > len(st.calls)
    if case.startswith("emit-"):
        assert emit_jobs(schema) > EMIT_MAX_JOBS and counts["k_emit_chunk"] > len(st.chunks)


# ------------------------------------------------------------------------------------------------ grid-stride passes ----

def _bits_one_push():
    rng = np.random.Generator(np.random.PCG64(21))
    n = 5_000_000
    t = table(rng, [(pa.int32(), True), (pa.bool_(), True)], n)
    return t.schema, t.to_batches(), [0], n, {"STAGE_BITS": (n + 31) // 32}


def _bits_late_bitmap():
    """A first batch without a validity bitmap, then one with nulls: its validity job sets chunk bits [0, b) to one first."""
    rng = np.random.Generator(np.random.PCG64(22))
    n0, n1 = 4_500_000, 500_000
    clean = table(rng, [(pa.int32(), False), (pa.bool_(), False)], n0)
    schema = pa.schema([clean.schema.field(0)] + [clean.schema.field(i).with_nullable(True) for i in (1, 2)])
    late = table(rng, [(pa.int32(), True), (pa.bool_(), True)], n1)
    batches = [pa.RecordBatch.from_arrays([c.combine_chunks() for c in tab.columns], schema=schema) for tab in (clean, late)]
    return schema, batches, [0], n0 + n1, {"STAGE_BITS": (n0 + n1 + 31) // 32}


def _one_column(t, n, seed, **kw):
    rng = np.random.Generator(np.random.PCG64(seed))
    tab = table(rng, [(t, True)], n)
    return tab.schema, [pa.RecordBatch.from_arrays([c.combine_chunks() for c in tab.columns], schema=tab.schema)], kw


def _strings_300k(t):
    def make():
        schema, batches, _ = _one_column(t, 300_000, 23)
        return schema, batches, [0], None, {"STAGE_OFFSETS": 300_000 + 1}
    return make


def _list_push(child):
    def make():
        rng = np.random.Generator(np.random.PCG64(24))
        n = 200_000
        lst = lists(rng, child, n, 4)
        schema = pa.schema([pa.field("k", pa.int64(), False), pa.field("l", lst.type)])
        rb = pa.RecordBatch.from_arrays([key_column(rng, n), lst], schema=schema)
        ne = len(lst.values)
        kinds = {"STAGE_LIST_OFFSETS" if _is_var(child) else "STAGE_OFFSETS": n + 1,
                 "STAGE_DIFF32" if _is_var(child) else "STAGE_FILL32": ne, "STAGE_BIT_BYTES": ne}
        return schema, [rb], [0], None, kinds
    return make


def _views_300k():
    schema, batches, _ = _one_column(pa.string_view(), 300_000, 25)
    return schema, batches, [0], None, {"STAGE_VIEW_BYTES": 300_000, "STAGE_SIZE_VIEW": 300_000}


def _emit_300k_chunks():
    rng = np.random.Generator(np.random.PCG64(26))
    t = table(rng, [(pa.string_view(), True), (pa.list_(pa.string()), True)], 600_000)
    return t.schema, t.to_batches(max_chunksize=150_000), [0], 300_000, {}


GRID_CASES = {
    "STAGE_BITS-5M-rows-one-push": _bits_one_push,
    "STAGE_BITS-5M-rows-late-bitmap": _bits_late_bitmap,
    "STAGE_OFFSETS-utf8-300k": _strings_300k(pa.string()),
    "STAGE_OFFSETS-large-utf8-300k": _strings_300k(pa.large_string()),
    "DIFF32-LIST_OFFSETS-BIT_BYTES-list-utf8": _list_push(pa.string()),
    "FILL32-OFFSETS-list-int32": _list_push(pa.int32()),
    "VIEW_BYTES-SIZE_VIEW-utf8view-300k": _views_300k,
    "EMIT-300k-row-chunks": _emit_300k_chunks,
}


@pytest.mark.parametrize("case", list(GRID_CASES))
def test_grid_stride_passes(ctx, case):
    """One case per job kind with more units than one launch has threads, so its grid-stride loop takes a second pass."""
    schema, batches, keys, chunk_rows, units = GRID_CASES[case]()
    st = Staged(schema, batches, chunk_rows or 0)
    for kind, u in units.items():  # units of work of one job of this kind, over the threads of one staging launch
        assert u > STAGE_THREADS, (kind, u, STAGE_THREADS)
    if case.startswith("STAGE_BITS"):
        assert len(st.chunks) == 1 and st.calls[-1][3] + st.calls[-1][2] > 32 * STAGE_THREADS
        if "late" in case:  # the late validity job: c = 0, b = the first batch's rows, past one pass of words
            late = [j for j in st.calls[1][5] if j[0] == 1]
            assert late and late[0][3] == 0 and late[0][2] > 32 * STAGE_THREADS and late[0][5]
    if case.startswith("EMIT"):  # EMIT_VIEWS (n views) and EMIT_LIST_OFFSETS (n + 1 offsets) of every chunk
        assert len(st.chunks) == 2 and min(st.chunks) > EMIT_THREADS
    check(ctx, schema, batches, keys, 4, chunk_rows=chunk_rows or 0)


# --------------------------------------------------------------------------------------------- every bit alignment ----

def _bit_alignment_batches(seed):
    """Slices of nullable Int16 and Boolean columns pushed one after another into one chunk, each at an Arrow offset picked
    so that its (source bit a, chunk bit b) pair mod 32 is one not reached yet; lengths cycle through 0, 1, 31, 32, 33,
    more than two words and others."""
    rng = np.random.Generator(np.random.PCG64(seed))
    m = 4_096
    t = table(rng, [(pa.int16(), True), (pa.bool_(), True)], m)
    t = pa.Table.from_arrays([c.combine_chunks() for c in t.columns], schema=t.schema)
    lengths = [0, 1, 31, 32, 33, 65, 97, 130, 7, 200, 18, 45, 3, 64, 29, 90, 12, 250]
    seen, batches, rows, k = set(), [], 0, 0
    while len(seen) < 1024 and k < 4_000:
        n = lengths[k % len(lengths)]
        k += 1
        b = rows % 32
        missing = [a for a in range(32) if (a, b) not in seen]
        a = missing[0] if missing and n else int(rng.integers(0, 32))
        off = a + 32 * int(rng.integers(0, (m - n - 32) // 32))
        rb = t.slice(off, n).to_batches()
        rb = rb[0] if rb else pa.RecordBatch.from_arrays([c.combine_chunks().slice(off, 0) for c in t.columns], schema=t.schema)
        if n and rb.column(1).null_count:  # (a validity job reads its source only when the slice has nulls)
            seen.add((a, b))
        batches.append(rb)
        rows += n
    return t.schema, batches


def _late_bitmap_batches(seed, chunk_rows):
    """For every b mod 32: a chunk whose first slice has no validity bitmap (b rows, b = 32 j + r) and whose second slice,
    at varying Arrow offsets, has nulls and fills the chunk."""
    rng = np.random.Generator(np.random.PCG64(seed))
    m = 2 * chunk_rows
    t = table(rng, [(pa.int16(), True), (pa.bool_(), True)], m)
    cols = [c.combine_chunks() for c in t.columns]
    clean = [cols[0], cols[1].fill_null(0), cols[2].fill_null(False)]
    clean = [pa.Array.from_buffers(c.type, len(c), [None] + c.buffers()[1:]) for c in clean]  # (no validity buffer at all)
    batches = []
    for r in range(32):
        b = 32 * int(rng.integers(1, chunk_rows // 64)) + r
        o0, o1 = int(rng.integers(0, m - chunk_rows)), int(rng.integers(0, m - chunk_rows))
        batches.append(pa.RecordBatch.from_arrays([c.slice(o0, b) for c in clean], schema=t.schema))
        batches.append(pa.RecordBatch.from_arrays([c.slice(o1, chunk_rows - b) for c in cols], schema=t.schema))
    return t.schema, batches


def test_every_bit_alignment(ctx):
    """STAGE_BITS merges three ranges into each chunk word: bits below c kept, [c, b) set, [b, b + n) shifted in from source
    bit a.  Every (a mod 32, b mod 32) pair is reached by a validity job and by a Boolean values job, and the late bitmap
    (c = 0 < b) at every b mod 32."""
    schema, batches = _bit_alignment_batches(31)
    st = Staged(schema, batches, 1 << 20)
    assert len(st.chunks) == 1
    for field in (1, 2):  # Int16 validity, Boolean values (and validity)
        pairs = {(a % 32, b % 32) for c in st.calls for (i, a, b, _, n, src) in c[5] if i == field and src and n}
        assert len(pairs) == 1024, (field, len(pairs))
    assert {n for _, _, n, *_ in st.calls} >= {1, 31, 32, 33} and max(n for _, _, n, *_ in st.calls) > 64
    assert any(rb.num_rows == 0 for rb in batches)
    check(ctx, schema, batches, [0], 3, chunk_rows=1 << 20)

    chunk_rows = 4_096
    schema, batches = _late_bitmap_batches(32, chunk_rows)
    st = Staged(schema, batches, chunk_rows)
    assert st.chunks == [chunk_rows] * 32
    for field in (1, 2):
        late = {b % 32 for c in st.calls for (i, a, b, c0, n, src) in c[5] if i == field and c0 == 0 < b and src}
        assert late == set(range(32)), (field, sorted(late))
    check(ctx, schema, batches, [0], 3, chunk_rows=chunk_rows)


# -------------------------------------------------------------------------------------------- every byte alignment ----

def _byte_alignment_batches(t, seed):
    """Slices of one Utf8 / Binary column (strings of 0 or 1 bytes, so any byte range is a row range) chosen so that every
    (first source byte mod 16, chunk byte fill mod 16) pair occurs with copies of 0-17 and 31-33 bytes, then two copies of
    more than 2 MiB from a tail of long strings."""
    rng = np.random.Generator(np.random.PCG64(seed))
    small, big = 8_192, 600
    lengths = np.concatenate([rng.choice([0, 1, 1, 1], small), np.full(big, 4_099)])
    col = strings(rng, t, lengths)
    key = key_column(rng, len(lengths))
    schema = pa.schema([pa.field("k", pa.int64(), False), pa.field("s", t)])
    off = np.concatenate([[0], np.cumsum(lengths)])
    first_row = {}
    for r in range(small, -1, -1):  # the first row whose offset is v
        first_row[int(off[r])] = r
    copies = list(range(18)) + [31, 32, 33]
    seen, batches, fill, k = set(), [], 0, 0

    def push(r0, r1):
        batches.append(pa.RecordBatch.from_arrays([key.slice(r0, r1 - r0), col.slice(r0, r1 - r0)], schema=schema))

    while (len(seen) < 256 or k < len(copies)) and k < 4_000:
        nbytes = copies[k % len(copies)]
        k += 1
        d = fill % 16
        missing = [a for a in range(16) if (a, d) not in seen]
        a = missing[0] if missing else int(rng.integers(0, 16))
        if nbytes:
            v = a + 16 * int(rng.integers(0, (int(off[small]) - 64) // 16))
            r0, r1 = first_row[v], first_row[v + nbytes]
        else:  # one empty string: a push that copies nothing
            empty = np.flatnonzero((lengths[:small] == 0) & (off[:small] % 16 == a))
            r0 = int(empty[rng.integers(0, len(empty))])
            v, r1 = int(off[r0]), r0 + 1
        push(r0, r1)
        if nbytes:
            seen.add((v % 16, d))
        fill += nbytes
    for r0, rows in ((small + 3, 520), (small + 1, 531)):  # > 2 MiB each, at two more residues
        push(r0, r0 + rows)
    return schema, batches


def test_every_byte_alignment_of_string_copies(ctx):
    """STAGE_COPY picks a 16, 8, 4 or 1-byte body by (src ^ dst) mod 16 and copies a head and a tail around it: Utf8 and
    Binary slices cover all 16 x 16 (source, chunk) byte residues, with copy lengths 0-17, 31-33 and above 2 MiB."""
    for t, seed in ((pa.string(), 41), (pa.binary(), 42)):
        schema, batches = _byte_alignment_batches(t, seed)
        st = Staged(schema, batches, 1 << 20)
        assert len(st.chunks) == 1
        pairs, sizes, fill = set(), set(), 0
        for rb in batches:  # prep.first = the slice's first offset, data_bytes = the chunk's bytes so far
            col = rb.column(1)
            offs = np.frombuffer(col.buffers()[1], dtype=np.int32)
            first, nbytes = int(offs[col.offset]), int(offs[col.offset + len(col)] - offs[col.offset])
            if nbytes:
                pairs.add((first % 16, fill % 16))
            sizes.add(nbytes)
            fill += nbytes
        assert len(pairs) == 256, (t, len(pairs))
        assert sizes >= set(range(18)) | {31, 32, 33} and sum(s > 2 << 20 for s in sizes) >= 2, sorted(sizes)
        check(ctx, schema, batches, [0], 4, chunk_rows=1 << 20)


def test_fixed_width_copies_at_every_arrow_offset(ctx):
    """STAGE_COPY of fixed-width values 1, 2, 4, 8 and 16 bytes wide (FixedSizeBinary(16) and Decimal128) from slices at Arrow
    offsets 0-15, into chunk fills that move by odd row counts."""
    rng = np.random.Generator(np.random.PCG64(43))
    types = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.binary(16), pa.decimal128(38, 2)]
    t = table(rng, [(ty, True) for ty in types], 4_096)
    t = pa.Table.from_arrays([c.combine_chunks() for c in t.columns], schema=t.schema)
    lengths = [1, 7, 16, 33, 100, 1_000, 3]
    batches = [t.slice(off, lengths[(off + k) % len(lengths)]).to_batches()[0] for k in range(3) for off in range(16)]
    assert {rb.column(1).offset for rb in batches} == set(range(16))
    check(ctx, t.schema, batches, [0], 4, chunk_rows=1 << 20)


def _emit_alignment_table(seed, n, N):
    """Utf8View strings of 0-20 bytes and nulls, all in one device-output chunk.  The row laid out last in the chunk (the
    last row of the last destination) gets 5 bytes and starts at a byte offset that is not a multiple of 4, so its string
    ends at the last byte of the chunk's buffer."""
    rng = np.random.Generator(np.random.PCG64(seed))
    key = key_column(rng, n)
    order, _ = expected_partitions(orc.partition_ids([key], n, N).astype(np.int64), N)
    _, valid = _nulls(rng, n, 0.1)
    lengths = np.where(valid, rng.integers(0, 21, n), 0)
    last = int(order[-1])
    valid[last], lengths[last] = True, 5
    if (int(lengths.sum()) - 5) % 4 == 0:
        r = int(np.flatnonzero(valid & (lengths < 20) & (np.arange(n) != last))[0])
        lengths[r] += 1
    s = strings(rng, pa.string(), lengths).cast(pa.string_view())
    s = pa.Array.from_buffers(s.type, n, [_bitmap(valid)] + s.buffers()[1:], null_count=int(n - valid.sum()))
    schema = pa.schema([pa.field("k", pa.int64(), False), pa.field("v", pa.string_view())])
    return pa.Table.from_arrays([key, s], schema=schema), np.where(valid, lengths, 0), order


def test_emit_views_at_every_byte_offset_and_length_class(ctx):
    """k_emit_chunk builds each view from up to four aligned words by o mod 4 and the string's length class (0-12 inline,
    above 12 a prefix): all 4 x 14 (o mod 4, min(len, 13)) pairs occur in the device-output chunk, and its last string ends
    at the last byte of the buffer at o mod 4 != 0."""
    n, N = 20_000, 4
    t, lengths, order = _emit_alignment_table(51, n, N)
    laid = lengths[order]  # the chunk's bytes: destination by destination, rows in stable order
    o = np.concatenate([[0], np.cumsum(laid)[:-1]])
    pairs = set(zip((o % 4).tolist(), np.minimum(laid, 13).tolist()))
    assert len(pairs) == 4 * 14, sorted(pairs)
    assert laid[-1] > 0 and o[-1] % 4 != 0 and o[-1] + laid[-1] == laid.sum()
    batches = t.slice(0, 9_000).to_batches() + t.slice(9_000).to_batches()
    assert Staged(t.schema, batches, 1 << 16).chunks == [n]
    check(ctx, t.schema, batches, [0], N, chunk_rows=1 << 16)


# ----------------------------------------------------------------------------------------- null views with garbage ----

def _views_with_null_garbage(seed, n, garbage):
    """Utf8View rows of 0-30 bytes (inline and out of line), 30% null.  With `garbage`, every null slot holds a view of
    1-12 bytes with non-zero inline bytes (never a pointer: a kernel ignoring validity copies wrong bytes, but in bounds);
    without, null slots are all zero."""
    rng = np.random.Generator(np.random.PCG64(seed))
    _, valid = _nulls(rng, n, 0.3)
    s = strings(rng, pa.string(), np.where(valid, rng.integers(0, 31, n), 0)).cast(pa.string_view())
    views = np.frombuffer(s.buffers()[1], dtype=np.uint8)[s.offset * 16:(s.offset + n) * 16].reshape(n, 16).copy()
    null = ~valid
    views[null] = 0
    if garbage:
        g = rng.integers(1, 13, int(null.sum()))
        inline = rng.integers(1, 256, (int(null.sum()), 12), dtype=np.uint8)
        inline[np.arange(12)[None, :] >= g[:, None]] = 0
        views[null, 0:4] = g.astype("<i4").view(np.uint8).reshape(-1, 4)
        views[null, 4:16] = inline
    return pa.Array.from_buffers(pa.string_view(), n, [_bitmap(valid), pa.py_buffer(views)] + s.buffers()[2:], null_count=int(null.sum()))


@pytest.mark.parametrize("keys", [[0], [1]], ids=["payload", "key"])
def test_null_views_with_garbage_lengths(ctx, keys):
    """k_stage_sizes turns a null view's length into 0 before the offsets scan: a batch whose null slots hold views with
    lengths 1-12 gives the streams and bytes_* stats of the same batch with zeroed null slots."""
    n = 6_000
    rng = np.random.Generator(np.random.PCG64(61))
    key = key_column(rng, n)
    schema = pa.schema([pa.field("k", pa.int64(), False), pa.field("v", pa.string_view())])
    runs = []
    for garbage in (True, False):
        v = _views_with_null_garbage(62, n, garbage)
        t = pa.Table.from_arrays([key, v], schema=schema)
        batches = slices(t, [1, 2_000, 2_003, 3_507, 5_999])
        if garbage:
            lens = np.frombuffer(v.buffers()[1], dtype=np.int32)[::4][~v.is_valid().to_numpy(zero_copy_only=False)]
            assert len(lens) and (lens > 0).all() and (lens <= 12).all()
        want, stats = run_all(ctx, schema, batches, keys, 5, chunk_rows=4_096)
        check_values(schema, batches, keys, 5, want)
        runs.append((want, stats))
    assert_same_streams(runs[0][0], runs[1][0])
    for run in ("device_host", "device_device"):
        for k in runs[0][1][run]:
            if k.startswith("bytes_"):
                assert runs[0][1][run][k] == runs[1][1][run][k], (run, k)


# --------------------------------------------------------------------------------------------------- the 32-bit cut ----

def _byte_span(a):
    """String bytes of a Utf8 array slice."""
    off = np.frombuffer(a.buffers()[1], dtype=np.int32)
    return int(off[a.offset + len(a)]) - int(off[a.offset])


def _device_used():
    import torch

    free, total = torch.cuda.mem_get_info()
    return total - free


def test_utf8_chunk_cut_at_2_gib_from_device_batches(ctx, record_property):
    """Device batches of Utf8 payload grow the chunk's byte buffer past its 1 GiB sizing cap and fill the chunk to exactly
    2^31 - 1 bytes; the next batch's first row adds one byte, so that batch starts a new chunk.  Checked one destination
    at a time against the host path and pyarrow; the peak host and device memory are recorded."""
    N, limit = 4, (1 << 31) - 1
    rng = np.random.Generator(np.random.PCG64(71))
    lengths = rng.integers(0, 2_048, 2_200_000)
    m = int(np.searchsorted(np.cumsum(lengths), limit))  # rows before the one that reaches the limit
    lengths = lengths[:m + 1]
    lengths[m] = limit - int(lengths[:m].sum())
    data = np.frombuffer(bytearray(rng.bytes(limit)), dtype=np.uint8)
    data &= 0x3F
    data |= 0x40  # (ASCII)
    big = strings(rng, pa.string(), lengths, data=data)
    assert _byte_span(big) == limit
    rows1 = len(big)
    assert rows1 < chunk_rows_of(0)  # the chunk is cut by its bytes, not its rows
    tail_len = rng.integers(0, 40, 1_000)
    tail_len[0] = 1
    tail = strings(rng, pa.string(), tail_len)
    keys = key_column(rng, rows1 + len(tail))
    schema = pa.schema([pa.field("k", pa.int64(), False), pa.field("s", pa.string())])
    off = np.frombuffer(big.buffers()[1], dtype=np.int32)
    cuts = np.linspace(0, rows1, 9).astype(np.int64)
    batches = []
    for r0, r1 in zip(cuts[:-1], cuts[1:]):  # 8 batches of ~256 MiB, each with buffers of its own (a device copy of just them)
        o = off[r0:r1 + 1]
        s = pa.Array.from_buffers(pa.string(), int(r1 - r0), [None, pa.py_buffer(o - o[0]), pa.py_buffer(data[o[0]:o[-1]])])
        batches.append(pa.RecordBatch.from_arrays([keys.slice(r0, r1 - r0), s], schema=schema))
    batches.append(pa.RecordBatch.from_arrays([keys.slice(rows1), tail], schema=schema))
    dest = orc.partition_ids([keys], len(keys), N).astype(np.int64)
    order, starts = expected_partitions(dest, N)
    base = _device_used()
    peak = [0]

    def sample():
        peak[0] = max(peak[0], _device_used() - base)

    part = dfd.Partitioning.Hash([0], N)
    hh = dfd.RepartitionExec(ctx, schema, part)
    for rb in batches:
        hh.push_batch(rb)
    hh.finish()
    sample()
    dh = dfd.RepartitionExec(ctx, schema, part)
    for rb in batches:
        push_device(dh, rb)
        sample()
    dh.finish()
    sample()
    want = []
    for p in range(N):
        hs, ds = list(hh.execute(p)), list(dh.execute(p))
        assert_same_streams([hs], [ds])
        idx = order[starts[p]:starts[p + 1]]
        first, second = idx[idx < rows1], idx[idx >= rows1] - rows1
        assert [b.num_rows for b in hs] == [len(first), len(second)], p  # the cut: the last batch opens the second chunk
        assert hs[0].column(1).equals(big.take(pa.array(first))), p
        assert hs[1].column(1).equals(tail.take(pa.array(second))), p
        assert hs[0].column(0).equals(keys.take(pa.array(first))) and hs[1].column(0).equals(keys.take(pa.array(idx[idx >= rows1]))), p
        want.append(hs)
        del ds
    assert sum(_byte_span(hs[0].column(1)) for hs in want) == limit  # the first chunk holds exactly 2^31 - 1 bytes
    dh.close()
    dd = dfd.RepartitionExec(ctx, schema, part, device_output=True)
    for rb in batches:
        push_device(dd, rb)
    dd.finish()
    sample()
    for p in range(N):
        stream = dd.execute_device(p)
        got = [DO.to_host_batch(b, stream.schema) for b in stream]
        assert_same_streams([want[p]], [got])
        del got
    dd.close()
    hh.close()
    host_peak = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / (1 << 20)
    record_property("peak_device_gib", round(peak[0] / (1 << 30), 2))
    record_property("peak_host_rss_gib", round(host_peak, 2))
    print(f"2 GiB cut: device memory in use at most {peak[0] / (1 << 30):.2f} GiB above the start (sampled), "
          f"process peak RSS {host_peak:.2f} GiB")
