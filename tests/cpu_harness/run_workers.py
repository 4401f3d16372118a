"""Sub-process body of tests/test_exchange_cpu_harness.py: T worker THREADS drive the product's exchange code (the object
nvcc built from csrc/dfd_exchange.cu, linked against the stand-in CUDA runtime / NCCL and the CPU oracle) through its
push transport and compare every (partition, producer) segment with the single-node oracle — values and order.

    python run_workers.py <harness.so> <world> <scenario> [seed]

scenario: shuffle | stream | coalesce | broadcast | mismatch | onepass | onepass_overflow | host | peer_missing | mixed | nccl | nccl_int32 | fused |
          stale"""
import ctypes as C
import os
import sys
import threading
import traceback

import numpy as np
import pyarrow as pa

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from datafusion_distributed_b200 import _native as nv  # noqa: E402  (ctypes struct definitions only; the product library is not loaded)
from oracle import oracle as orc  # noqa: E402

VP = C.c_void_p
COL = nv.DfdColumn


def bind(lib):
    sig = {
        "dfd_last_error": (C.c_char_p, []),
        "harness_ctx_create": (VP, []),
        "harness_ctx_destroy": (None, [VP]),
        "dfd_nccl_unique_id": (C.c_int, [VP]),
        "dfd_exchange_create": (C.c_int, [VP, C.c_int, C.c_int, VP, C.POINTER(VP)]),
        "dfd_exchange_destroy": (None, [VP]),
        "dfd_exchange_setup_window": (C.c_int, [VP, C.c_size_t]),
        "dfd_partitioner_create": (C.c_int, [VP, C.c_uint32, C.POINTER(C.c_int32), C.c_int, VP, C.POINTER(VP)]),
        "dfd_partitioner_destroy": (None, [VP]),
        "dfd_shuffle_device_onepass": (C.c_int, [VP, VP, C.POINTER(COL), C.c_int, C.c_int64, C.c_uint32, C.POINTER(COL)]),
        "dfd_exchange_collect": (C.c_int, [VP, C.POINTER(COL), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
        "dfd_exchange_gather": (C.c_int, [VP, C.c_int, C.POINTER(COL), C.c_int, C.POINTER(C.c_int64), C.c_uint32, C.c_int, C.POINTER(COL)]),
        "dfd_exchange_pending_segments": (C.c_uint32, [VP]),
        "dfd_shuffle_stream_begin": (C.c_int, [VP, VP, C.POINTER(COL), C.c_int, C.c_int64, C.c_uint32, C.POINTER(C.c_uint8), C.POINTER(VP)]),
        "dfd_shuffle_stream_next": (C.c_int, [VP, C.POINTER(COL), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
        "dfd_shuffle_stream_end": (None, [VP]),
        "dfd_shuffle_stream_stats": (C.c_int, [VP, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
        "dfd_exchange_onepass_fallbacks": (C.c_uint64, [VP]),
        "dfd_shuffle_device": (C.c_int, [VP, VP, C.c_int, C.POINTER(COL), C.c_int, C.c_int64, C.c_uint32, C.POINTER(COL), C.c_int64, C.POINTER(C.c_int64)]),
        "dfd_shuffle_host": (C.c_int, [VP, VP, C.POINTER(COL), C.c_int, C.c_int64, C.c_uint32, C.c_int, C.POINTER(COL), C.c_int64, C.POINTER(C.c_int64)]),
    }
    for name, (res, args) in sig.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args


class Failed(Exception):
    pass


def check(lib, rc, what):
    if rc != 0:
        raise Failed(f"{what}: status {rc}: {lib.dfd_last_error().decode('utf-8', 'replace')}")


def local_table(rank, n, seed):
    """Producer `rank`'s rows: Int64 key (nullable), Int32, Boolean (nullable), Utf8 (nullable), Float64."""
    rng = np.random.Generator(np.random.PCG64(seed * 100 + rank))
    key = pa.array(rng.integers(0, 1 << 40, n, dtype=np.int64), mask=rng.random(n) < 0.05)
    i32 = pa.array(rng.integers(-(2**31), 2**31 - 1, n).astype(np.int32))
    flag = pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1)
    words = np.array(["", "a", "hello", "x" * 13, "a-much-longer-string-than-twelve-bytes", "ünï"], dtype=object)
    s = pa.array([None if rng.random() < 0.1 else str(words[rng.integers(0, len(words))]) + str(int(rng.integers(0, 1000))) for _ in range(n)], type=pa.string())
    f64 = pa.array(rng.standard_normal(n))
    return pa.table([key, i32, flag, s, f64], names=["key", "i32", "flag", "s", "f64"])


def fixed_table(rank, n, seed, skew):
    """Producer `rank`'s rows for the single-pass exchange: fixed-width, non-null (key Int64, Int32, Float64, Int64)."""
    rng = np.random.Generator(np.random.PCG64(seed * 1000 + rank))
    key = rng.integers(0, 1 << 50, n, dtype=np.int64)
    if skew:
        key[rng.random(n) < 0.7] = 424242  # one hot key: its (partition, producer) sub-window overflows
    return pa.table([pa.array(key), pa.array(rng.integers(-(2**31), 2**31 - 1, n).astype(np.int32)), pa.array(rng.standard_normal(n)),
                     pa.array(np.arange(n, dtype=np.int64) * 8 + rank)], names=["key", "i32", "f64", "rid"])


def to_columns(table, keep):
    """pyarrow columns -> dfd_column descriptors over their (host == 'device') buffers."""
    cols = (COL * table.num_columns)()
    for i, name in enumerate(table.column_names):
        a = table.column(name).combine_chunks()
        keep.append(a)
        b = a.buffers()
        c = cols[i]
        c.offset = a.offset
        c.validity = b[0].address if (b[0] is not None and a.null_count > 0) else None
        t = a.type
        if pa.types.is_boolean(t):
            c.kind, c.width, c.values = nv.COL_BOOL, 0, b[1].address
        elif pa.types.is_string(t):
            c.kind, c.width, c.offsets = nv.COL_UTF8, 0, b[1].address
            c.values = b[2].address if b[2] is not None else None
            c.values_bytes = b[2].size if b[2] is not None else 0
        else:
            c.kind, c.width, c.values = nv.COL_FIXED, t.bit_width // 8, b[1].address
    return cols


def segment_to_arrow(col, field, start, count):
    """rows [start, start + count) of an output column in the receive window -> a pyarrow array (zero copy)."""
    t = field.type
    if count == 0:
        return pa.array([], type=t)  # (an empty segment owns no offsets)
    validity = None
    if col.validity:
        validity = pa.foreign_buffer(col.validity, (start + count + 7) // 8 + 8)
    if pa.types.is_boolean(t):
        return pa.Array.from_buffers(t, count, [validity, pa.foreign_buffer(col.values, (start + count + 7) // 8 + 8)], offset=start)
    if pa.types.is_string(t):
        offs = np.ctypeslib.as_array(C.cast(col.offsets, C.POINTER(C.c_int32)), shape=(start + count + 1,))
        nbytes = int(offs[start + count]) if count else 0
        return pa.Array.from_buffers(t, count, [validity, pa.foreign_buffer(col.offsets, 4 * (start + count + 1)), pa.foreign_buffer(col.values, max(nbytes, 1))],
                                     offset=start)
    return pa.Array.from_buffers(t, count, [validity, pa.foreign_buffer(col.values, (start + count) * (t.bit_width // 8) + 8)], offset=start)


def nullable_outs(table):
    outs = (COL * table.num_columns)()
    for i, f in enumerate(table.schema):
        outs[i].validity = 1 if f.nullable and table.column(i).null_count >= 0 and f.name in ("key", "flag", "s") else None  # the schema's flags
    return outs


def worker(lib, rank, world, uid, scenario, seed, errors, barrier):
    try:
        ctx = VP(lib.harness_ctx_create())
        ex = VP()
        check(lib, lib.dfd_exchange_create(ctx, rank, world, uid, C.byref(ex)), "dfd_exchange_create")
        window = (24 << 10) if scenario == "stream" else (8 << 20)
        if scenario == "onepass_overflow":
            window = 6000 * 28  # capacity 6000 rows of 28 bytes: sub-windows of 992 rows at 2 workers x 3 partitions
        if scenario == "mismatch" and rank == world - 1:
            window += 4096
        rc = lib.dfd_exchange_setup_window(ex, window)
        if scenario == "mismatch":
            # every worker sees that the windows differ (the sizes travel with the IPC handles) and refuses
            assert rc == 1 and b"same size" in lib.dfd_last_error(), (rc, lib.dfd_last_error())
            lib.dfd_exchange_destroy(ex)
            lib.harness_ctx_destroy(ctx)
            return
        check(lib, rc, "dfd_exchange_setup_window")
        P = 3
        N = P * world
        n = [0, 1, 700, 1500, 333, 1000, 64, 2000][rank % 8] if scenario != "stream" else 1200 + 100 * rank
        tables = [local_table(r, ([0, 1, 700, 1500, 333, 1000, 64, 2000][r % 8] if scenario != "stream" else 1200 + 100 * r), seed) for r in range(world)]
        mine = tables[rank]
        keep = []
        in_cols = to_columns(mine, keep)
        keys = (C.c_int32 * 2)(0, 3)  # Hash([key, s], N): an Int64 and a Utf8 key
        part = VP()
        check(lib, lib.dfd_partitioner_create(ctx, N, keys, 2, None, C.byref(part)), "dfd_partitioner_create")
        fields = list(mine.schema)
        dests = [orc.partition_ids([t.column("key"), t.column("s")], t.num_rows, N) for t in tables]

        def verify(outs, starts, counts, n_seg, source, rows_of):
            for sgm in range(n_seg):
                r, rows = source(sgm)
                cnt = int(counts[sgm])
                want = tables[r].take(pa.array(rows)) if r >= 0 else mine.slice(0, 0)
                assert cnt == want.num_rows, (scenario, rank, sgm, cnt, want.num_rows)
                for c, f in enumerate(fields):
                    got = segment_to_arrow(outs[c], f, int(starts[sgm]), cnt)
                    got.validate(full=True)
                    assert got.equals(want.column(c).combine_chunks()), (scenario, rank, sgm, f.name)
                rows_of[0] += cnt

        total = [0]

        def one_single_pass(data_seed):
            tabs = [fixed_table(r, 900 + 11 * r, data_seed, False) for r in range(world)]
            kp = []
            cols_ = to_columns(tabs[rank], kp)
            k1 = (C.c_int32 * 1)(0)
            p1 = VP()
            check(lib, lib.dfd_partitioner_create(ctx, N, k1, 1, None, C.byref(p1)), "dfd_partitioner_create")
            d_ = [orc.partition_ids([t.column("key")], t.num_rows, N) for t in tabs]
            o_ = (COL * tabs[rank].num_columns)()
            check(lib, lib.dfd_shuffle_device_onepass(ex, p1, cols_, tabs[rank].num_columns, tabs[rank].num_rows, P, o_), "dfd_shuffle_device_onepass")
            st_, ct_ = (C.c_int64 * (P * world))(), (C.c_int64 * (P * world))()
            check(lib, lib.dfd_exchange_collect(ex, o_, st_, ct_), "dfd_exchange_collect")
            for sgm in range(P * world):
                r, q = sgm % world, sgm // world
                want = tabs[r].take(pa.array(np.nonzero(d_[r] == rank * P + q)[0]))
                assert int(ct_[sgm]) == want.num_rows
                for c, f in enumerate(tabs[rank].schema):
                    assert segment_to_arrow(o_[c], f, int(st_[sgm]), int(ct_[sgm])).equals(want.column(c).combine_chunks()), ("single pass", rank, sgm, f.name)
            barrier.wait()
            lib.dfd_partitioner_destroy(p1)

        def one_push(data_seed):
            tabs = [local_table(r, 400 + 13 * r, data_seed) for r in range(world)]
            kp = []
            cols_ = to_columns(tabs[rank], kp)
            d_ = [orc.partition_ids([t.column("key"), t.column("s")], t.num_rows, N) for t in tabs]
            o_ = nullable_outs(tabs[rank])
            check(lib, lib.dfd_shuffle_device_onepass(ex, part, cols_, tabs[rank].num_columns, tabs[rank].num_rows, P, o_), "dfd_shuffle_device_onepass")
            st_, ct_ = (C.c_int64 * (P * world))(), (C.c_int64 * (P * world))()
            check(lib, lib.dfd_exchange_collect(ex, o_, st_, ct_), "dfd_exchange_collect")
            for sgm in range(P * world):
                r, q = sgm % world, sgm // world
                want = tabs[r].take(pa.array(np.nonzero(d_[r] == rank * P + q)[0]))
                assert int(ct_[sgm]) == want.num_rows
                for c, f in enumerate(tabs[rank].schema):
                    assert segment_to_arrow(o_[c], f, int(st_[sgm]), int(ct_[sgm])).equals(want.column(c).combine_chunks()), ("push", rank, sgm, f.name)
            barrier.wait()

        if scenario in ("nccl", "fused"):
            # dfd_shuffle_device: the dense layout (per partition, producers contiguous in task order) through the NCCL-mode
            # transport (every column kind; grouped ncclSend / ncclRecv of values, u8 images of bitmaps, string lengths + bytes) or
            # the two-pass fused transport (all-gathered counts -> plan -> peer stores; fixed-width non-null)
            for rep in range(2):
                if scenario == "nccl":
                    tabs = [local_table(r, [0, 1, 700, 1500, 333, 1000, 64, 2000][(r + rep) % 8], seed + rep) for r in range(world)]
                    kcols, pt = ["key", "s"], part
                else:
                    tabs = [fixed_table(r, 800 + 5 * r, seed + rep, False) for r in range(world)]
                    kcols = ["key"]
                    pt = VP()
                    check(lib, lib.dfd_partitioner_create(ctx, N, (C.c_int32 * 1)(0), 1, None, C.byref(pt)), "dfd_partitioner_create")
                t_me = tabs[rank]
                flds = list(t_me.schema)
                kp = []
                cols_ = to_columns(t_me, kp)
                d_ = [orc.partition_ids([t.column(k) for k in kcols], t.num_rows, N) for t in tabs]
                cap = sum(t.num_rows for t in tabs) + 8
                o_ = (COL * len(flds))()
                bufs = []
                for i, f in enumerate(flds):
                    o_[i].kind, o_[i].width = cols_[i].kind, cols_[i].width
                    if scenario == "fused":
                        continue  # (the fused transport hands out window pointers)
                    if pa.types.is_string(f.type):
                        nbytes = sum(t.column(i).combine_chunks().buffers()[2].size if t.column(i).combine_chunks().buffers()[2] is not None else 0 for t in tabs) + 64
                        ob, vb = np.zeros(cap + 1, dtype=np.int32), np.zeros(nbytes, dtype=np.uint8)
                        o_[i].offsets, o_[i].values, o_[i].values_bytes = ob.ctypes.data, vb.ctypes.data, nbytes
                        bufs += [ob, vb]
                    else:
                        vb = np.zeros(cap * max(1, f.type.bit_width // 8) + 64, dtype=np.uint8)
                        o_[i].values = vb.ctypes.data
                        bufs.append(vb)
                    if f.name in ("key", "flag", "s"):  # the schema's nullable columns: a validity buffer on EVERY worker
                        nb_ = np.zeros(cap // 8 + 64, dtype=np.uint8)
                        o_[i].validity = nb_.ctypes.data
                        bufs.append(nb_)
                ps = (C.c_int64 * (P + 1))()
                check(lib, lib.dfd_shuffle_device(ex, pt, 0 if scenario == "nccl" else 1, cols_, len(flds), t_me.num_rows, P, o_, cap, ps), "dfd_shuffle_device")
                for q in range(P):
                    want = pa.concat_tables([tabs[r].take(pa.array(np.nonzero(d_[r] == rank * P + q)[0])) for r in range(world)])
                    assert ps[q + 1] - ps[q] == want.num_rows, (scenario, rank, q)
                    for c, f in enumerate(flds):
                        got = segment_to_arrow(o_[c], f, int(ps[q]), int(ps[q + 1] - ps[q]))
                        got.validate(full=True)
                        assert got.equals(want.column(c).combine_chunks()), (scenario, rank, q, f.name)
                barrier.wait()
                if scenario == "fused":
                    lib.dfd_partitioner_destroy(pt)
        elif scenario == "mixed":
            # the transports share one window, one epoch counter and the done flags: alternate them on the same exchange
            one_single_pass(seed)
            one_push(seed + 1)
            one_push(seed + 2)
            one_single_pass(seed + 3)
            one_single_pass(seed + 4)
            one_push(seed + 5)
        elif scenario == "nccl_int32":
            # NCCL mode, one key value: every row of both producers goes to one consumer, which would receive more than INT32_MAX
            # bytes of a Utf8 column.  EVERY worker refuses before any send, the one that would receive nothing included.
            rows, row_bytes = 1100, 1 << 20
            assert world * rows * row_bytes > 2**31 - 1 >= rows * row_bytes
            off = (np.arange(rows + 1, dtype=np.int64) * row_bytes).astype(np.int32)
            s_big = pa.Array.from_buffers(pa.string(), rows, [None, pa.py_buffer(off.tobytes()), pa.py_buffer(np.full(rows * row_bytes, 97, np.uint8))])
            t_big = pa.table([pa.array(np.full(rows, 7, np.int64)), s_big], names=["key", "s"])
            kp = []
            cols_ = to_columns(t_big, kp)
            pt = VP()
            check(lib, lib.dfd_partitioner_create(ctx, N, (C.c_int32 * 1)(0), 1, None, C.byref(pt)), "dfd_partitioner_create")
            o_ = (COL * 2)()
            small = [np.zeros(64, np.uint8) for _ in range(3)]
            o_[0].kind, o_[0].width, o_[0].values = nv.COL_FIXED, 8, small[0].ctypes.data
            o_[1].kind, o_[1].offsets, o_[1].values, o_[1].values_bytes = nv.COL_UTF8, small[1].ctypes.data, small[2].ctypes.data, 64
            ps = (C.c_int64 * (P + 1))()
            rc = lib.dfd_shuffle_device(ex, pt, 0, cols_, 2, rows, P, o_, 8, ps)
            err = lib.dfd_last_error()
            assert rc == 7 and b"int32" in err, (rank, rc, err)
            barrier.wait()
            lib.dfd_partitioner_destroy(pt)
        elif scenario == "stale":
            # collect reports the LAST shuffle only: a push result is dropped as soon as another shuffle starts, an asynchronous
            # two-pass shuffle is completed by collect in its dense layout, and after an NCCL-mode shuffle (complete inside the
            # call) nothing is pending
            tabs = [fixed_table(r, 800 + 5 * r, seed, False) for r in range(world)]
            kp = []
            cols_ = to_columns(tabs[rank], kp)
            n_c, n_r = tabs[rank].num_columns, tabs[rank].num_rows
            p1 = VP()
            check(lib, lib.dfd_partitioner_create(ctx, N, (C.c_int32 * 1)(0), 1, None, C.byref(p1)), "dfd_partitioner_create")
            d_ = [orc.partition_ids([t.column("key")], t.num_rows, N) for t in tabs]
            one_push(seed + 1)
            o_ = (COL * n_c)()
            check(lib, lib.dfd_shuffle_device_async(ex, p1, cols_, n_c, n_r, P, o_), "dfd_shuffle_device_async")
            assert lib.dfd_exchange_pending_segments(ex) == 0
            st_, ct_ = (C.c_int64 * (P * world))(), (C.c_int64 * (P * world))()
            check(lib, lib.dfd_exchange_collect(ex, o_, st_, ct_), "dfd_exchange_collect")
            for sgm in range(P * world):
                r, q = sgm % world, sgm // world
                want = tabs[r].take(pa.array(np.nonzero(d_[r] == rank * P + q)[0]))
                assert int(ct_[sgm]) == want.num_rows, ("stale", rank, sgm, int(ct_[sgm]), want.num_rows)
                if sgm + 1 < P * world:  # dense: every segment starts where the one before it ends
                    assert st_[sgm + 1] == st_[sgm] + ct_[sgm], ("stale", rank, sgm)
                for c, f in enumerate(tabs[rank].schema):
                    assert segment_to_arrow(o_[c], f, int(st_[sgm]), int(ct_[sgm])).equals(want.column(c).combine_chunks()), ("stale", rank, sgm, f.name)
            barrier.wait()
            one_push(seed + 2)
            cap = sum(t.num_rows for t in tabs) + 8
            bufs = [np.zeros(cap * 8 + 64, dtype=np.uint8) for _ in range(n_c)]
            o_ = (COL * n_c)()
            for i, b in enumerate(bufs):
                o_[i].kind, o_[i].width, o_[i].values = cols_[i].kind, cols_[i].width, b.ctypes.data
            ps = (C.c_int64 * (P + 1))()
            check(lib, lib.dfd_shuffle_device(ex, p1, 0, cols_, n_c, n_r, P, o_, cap, ps), "dfd_shuffle_device(NCCL)")
            assert lib.dfd_exchange_pending_segments(ex) == 0
            rc = lib.dfd_exchange_collect(ex, o_, st_, ct_)
            assert rc == 1 and b"no shuffle is pending" in lib.dfd_last_error(), (rc, lib.dfd_last_error())
            barrier.wait()
            lib.dfd_partitioner_destroy(p1)
        elif scenario == "peer_missing":
            # the last worker fails before the exchange (it never enters the collective): the others must come back with an error
            # after the bounded flag wait — never hang (the coordinator then cancels the stage, impl_execute_task.rs:138-155)
            if rank != world - 1:
                outs = nullable_outs(mine)
                rc = lib.dfd_shuffle_device_onepass(ex, part, in_cols, len(fields), mine.num_rows, P, outs)
                assert rc == 5 and b"never published" in lib.dfd_last_error(), (rc, lib.dfd_last_error())  # DFD_ERR_INTERNAL
        elif scenario in ("onepass", "onepass_overflow"):
            # the single-pass exchange (fixed-width non-null schema): peer stores into (partition, producer) sub-windows, counts
            # and completion as peer-memory flags; a sub-window that overflows on ANY worker makes every worker re-run exactly
            for rep in range(2):
                tables = [fixed_table(r, 2000 + 10 * r, seed + rep, scenario == "onepass_overflow") for r in range(world)]
                mine = tables[rank]
                fields = list(mine.schema)
                keep.clear()
                in_cols = to_columns(mine, keep)
                k1 = (C.c_int32 * 1)(0)
                part1 = VP()
                check(lib, lib.dfd_partitioner_create(ctx, N, k1, 1, None, C.byref(part1)), "dfd_partitioner_create")
                dests = [orc.partition_ids([t.column("key")], t.num_rows, N) for t in tables]
                outs = (COL * len(fields))()
                check(lib, lib.dfd_shuffle_device_onepass(ex, part1, in_cols, len(fields), mine.num_rows, P, outs), "dfd_shuffle_device_onepass")
                starts, counts = (C.c_int64 * (P * world))(), (C.c_int64 * (P * world))()
                check(lib, lib.dfd_exchange_collect(ex, outs, starts, counts), "dfd_exchange_collect")
                total[0] = 0
                verify(outs, starts, counts, P * world, lambda s: (s % world, np.nonzero(dests[s % world] == rank * P + s // world)[0]), total)
                assert total[0] == sum(int((d // P == rank).sum()) for d in dests)
                fb = lib.dfd_exchange_onepass_fallbacks(ex)
                assert fb == (rep + 1 if scenario == "onepass_overflow" else 0), fb
                barrier.wait()
                lib.dfd_partitioner_destroy(part1)
        elif scenario == "host":
            # dfd_shuffle_host: HOST columns in, HOST columns out, the rows cut into chunks that pipeline H2D | fused shuffle | D2H
            # through the two halves of the receive window; output is chunk-major, producers contiguous per (chunk, partition)
            for n_chunks in (1, 3, 4):
                tables = [fixed_table(r, 1500 + 7 * r, seed + n_chunks, False) for r in range(world)]
                mine = tables[rank]
                fields = list(mine.schema)
                keep.clear()
                in_cols = to_columns(mine, keep)
                k1 = (C.c_int32 * 1)(0)
                part1 = VP()
                check(lib, lib.dfd_partitioner_create(ctx, N, k1, 1, None, C.byref(part1)), "dfd_partitioner_create")
                dests = [orc.partition_ids([t.column("key")], t.num_rows, N) for t in tables]
                cap = sum(t.num_rows for t in tables)
                bufs = [np.zeros(cap * (f.type.bit_width // 8) + 64, dtype=np.uint8) for f in fields]
                outs = (COL * len(fields))()
                for i, f in enumerate(fields):
                    outs[i].kind, outs[i].width, outs[i].values = nv.COL_FIXED, f.type.bit_width // 8, bufs[i].ctypes.data
                cps = (C.c_int64 * (n_chunks * (P + 1)))()
                check(lib, lib.dfd_shuffle_host(ex, part1, in_cols, len(fields), mine.num_rows, P, n_chunks, outs, cap, cps), "dfd_shuffle_host")
                for ch in range(n_chunks):
                    for q in range(P):
                        a, b = cps[ch * (P + 1) + q], cps[ch * (P + 1) + q + 1]
                        want_rows = []
                        for r in range(world):  # producers in task order, each with the rows of ITS chunk `ch`
                            nr = tables[r].num_rows
                            lo, hi = nr * ch // n_chunks, nr * (ch + 1) // n_chunks
                            want_rows.append(tables[r].slice(lo, hi - lo).take(pa.array(np.nonzero(dests[r][lo:hi] == rank * P + q)[0])))
                        want = pa.concat_tables(want_rows)
                        assert b - a == want.num_rows, (n_chunks, ch, q, a, b, want.num_rows)
                        for i, f in enumerate(fields):
                            w = f.type.bit_width // 8
                            got = pa.Array.from_buffers(f.type, b - a, [None, pa.py_buffer(bufs[i][a * w:b * w].tobytes())])
                            assert got.equals(want.column(i).combine_chunks()), (n_chunks, ch, q, f.name)
                barrier.wait()
                lib.dfd_partitioner_destroy(part1)
        elif scenario == "shuffle":
            # three shuffles in a row over the same windows (the epoch flags tell the rounds apart; a consumer's window is only
            # overwritten after it has announced the next shuffle), the last one through the pre-partitioned route
            for rep in range(3):
                if rep:
                    tables = [local_table(r, [5, 0, 900, 64, 1, 1300, 700, 33][(r + rep) % 8], seed + 17 * rep) for r in range(world)]
                    mine = tables[rank]
                    keep.clear()
                    in_cols = to_columns(mine, keep)
                    dests = [orc.partition_ids([t.column("key"), t.column("s")], t.num_rows, N) for t in tables]
                outs = nullable_outs(mine)
                if rep < 2:
                    check(lib, lib.dfd_shuffle_device_onepass(ex, part, in_cols, len(fields), mine.num_rows, P, outs), "dfd_shuffle_device_onepass")
                else:
                    # DFD_ROUTE_SHUFFLE: the rows are ALREADY grouped by global partition (what dfd_partition_device [+ PartialReduce]
                    # leaves behind); only the exchange half runs
                    order = np.argsort(dests[rank], kind="stable")
                    sorted_mine = mine.take(pa.array(order))
                    keep.clear()
                    in_cols = to_columns(sorted_mine, keep)
                    cnt = np.bincount(dests[rank], minlength=N)
                    slice_starts = (C.c_int64 * (N + 1))(0, *np.cumsum(cnt).tolist())
                    check(lib, lib.dfd_exchange_gather(ex, 0, in_cols, len(fields), slice_starts, P, world, outs), "dfd_exchange_gather(shuffle)")
                starts, counts = (C.c_int64 * (P * world))(), (C.c_int64 * (P * world))()
                check(lib, lib.dfd_exchange_collect(ex, outs, starts, counts), "dfd_exchange_collect")
                # NetworkShuffleExec::execute: partition q of consumer `rank` = global partition rank * P + q from every producer
                total[0] = 0
                verify(outs, starts, counts, P * world, lambda s: (s % world, np.nonzero(dests[s % world] == rank * P + s // world)[0]), total)
                assert total[0] == sum(int((d // P == rank).sum()) for d in dests)
                barrier.wait()  # (the test reads the window from Python: finish before the next shuffle may overwrite it)
        elif scenario == "stream":
            nullable = (C.c_uint8 * len(fields))(1, 0, 1, 1, 0)
            st = VP()
            check(lib, lib.dfd_shuffle_stream_begin(ex, part, in_cols, len(fields), mine.num_rows, P, nullable, C.byref(st)), "dfd_shuffle_stream_begin")
            got = {(q, r): [] for q in range(P) for r in range(world)}
            while True:
                outs = (COL * len(fields))()
                starts, counts, done = (C.c_int64 * (P * world))(), (C.c_int64 * (P * world))(), C.c_int(0)
                check(lib, lib.dfd_shuffle_stream_next(st, outs, starts, counts, C.byref(done)), "dfd_shuffle_stream_next")
                if done.value:
                    break
                for sgm in range(P * world):  # drain the window before the next round overwrites it
                    cnt = int(counts[sgm])
                    if cnt:
                        got[(sgm // world, sgm % world)].append(pa.table([segment_to_arrow(outs[c], f, int(starts[sgm]), cnt) for c, f in enumerate(fields)],
                                                                         names=mine.column_names).combine_chunks().to_pydict())
                barrier.wait()  # (a real consumer would hand the rows on; all workers enter the next round together anyway)
            rounds, splits = C.c_uint64(0), C.c_uint64(0)
            lib.dfd_shuffle_stream_stats(st, C.byref(rounds), C.byref(splits))
            assert rounds.value > 1 and splits.value >= 1, (rounds.value, splits.value)  # the window is too small for one round
            lib.dfd_shuffle_stream_end(st)
            for (q, r), pieces in got.items():
                want = tables[r].take(pa.array(np.nonzero(dests[r] == rank * P + q)[0])).to_pydict()
                have = {k: [v for p in pieces for v in p[k]] for k in mine.column_names}
                assert have == want or (not pieces and all(len(v) == 0 for v in want.values())), (rank, q, r)
        else:
            route = {"coalesce": 1, "broadcast": 2}[scenario]
            consumers = max(1, world - 1) if scenario == "coalesce" else world
            # this producer's P partitions = P row slices of its table (no repartition)
            cuts = sorted({0, mine.num_rows} | {int(x) for x in np.random.Generator(np.random.PCG64(seed + rank)).integers(0, mine.num_rows + 1, P - 1)})
            while len(cuts) < P + 1:
                cuts.append(mine.num_rows)
            all_cuts = []
            for r in range(world):
                nr = tables[r].num_rows
                c_ = sorted({0, nr} | {int(x) for x in np.random.Generator(np.random.PCG64(seed + r)).integers(0, nr + 1, P - 1)})
                while len(c_) < P + 1:
                    c_.append(nr)
                all_cuts.append(c_)
            slice_starts = (C.c_int64 * (P + 1))(*all_cuts[rank])
            outs = nullable_outs(mine)
            check(lib, lib.dfd_exchange_gather(ex, route, in_cols, len(fields), slice_starts, P, consumers, outs), "dfd_exchange_gather")
            nseg = lib.dfd_exchange_pending_segments(ex)
            starts, counts = (C.c_int64 * max(nseg, 1))(), (C.c_int64 * max(nseg, 1))()
            check(lib, lib.dfd_exchange_collect(ex, outs, starts, counts), "dfd_exchange_collect")
            if scenario == "broadcast":
                assert nseg == P * world
                src = lambda s: (s % world, np.arange(all_cuts[s % world][s // world], all_cuts[s % world][s // world + 1]))  # noqa: E731
            else:
                base, extra = divmod(world, consumers)
                if rank >= consumers:
                    assert nseg == 0
                    src = None
                else:
                    length, start = base + (1 if rank < extra else 0), rank * base + min(rank, extra)
                    assert nseg == (base + (1 if extra else 0)) * P

                    def src(s):
                        off, g = divmod(s, P)
                        if off >= length:
                            return -1, np.arange(0)
                        r = start + off
                        return r, np.arange(all_cuts[r][g], all_cuts[r][g + 1])
            if src:
                verify(outs, starts, counts, nseg, src, total)
        barrier.wait()  # nobody tears its window down while a peer may still read flags in it
        lib.dfd_partitioner_destroy(part)
        lib.dfd_exchange_destroy(ex)
        lib.harness_ctx_destroy(ctx)
    except BaseException:  # noqa: BLE001
        errors.append(f"rank {rank}: " + traceback.format_exc())
        try:
            barrier.abort()
        except Exception:  # noqa: BLE001
            pass


def main():
    so, world, scenario = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    seed = int(sys.argv[4]) if len(sys.argv) > 4 else 1
    lib = C.CDLL(so)
    bind(lib)
    uid = (C.c_uint8 * 128)()
    if world > 1:
        rc = lib.dfd_nccl_unique_id(uid)
        assert rc == 0, lib.dfd_last_error()
    errors, barrier = [], threading.Barrier(world)
    threads = [threading.Thread(target=worker, args=(lib, r, world, uid, scenario, seed, errors, barrier)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=120)
    if errors or any(t.is_alive() for t in threads):
        print("\n".join(errors) or "a worker thread hung", file=sys.stderr)
        os._exit(1)
    print(f"WORKERS_OK world={world} scenario={scenario}")


if __name__ == "__main__":
    main()
