"""Sub-process body of tests/test_host_shuffle_cpu_harness.py: T worker THREADS run dfd_shuffle_host (the product's exchange
object, linked against the stand-in CUDA runtime / NCCL, the CPU oracle and the CPU emulations of the push transport's and
the compaction's kernels) with nullable, Boolean and string columns, and compare every (chunk, partition) of the dense host
output with the single-node oracle.

    python run_host_shuffle_workers.py <harness.so> <world> <scenario> [seed]

scenario: mixed  — n_chunks 1 / 3 / 7 and more chunks than rows, on one exchange;
          short  — the last worker's string output is one byte short at a chunk before the last: it gets DFD_ERR_CAPACITY
                   with the chunks before that one delivered, and every other worker comes back with an error."""
import ctypes as C
import os
import sys
import threading
import traceback

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import run_workers as RW  # noqa: E402  (bindings, struct definitions, the oracle)

nv, orc, COL, VP = RW.nv, RW.orc, RW.COL, RW.VP
P = 3
ROWS = [0, 1, 700, 1500, 333, 1000, 64, 2000]
FILL = 0xAB


def mixed_table(n, seed):
    """The mixed schema of tests/test_exchange_gpu.py: Int64 (nullable), Utf8, LargeUtf8, Boolean, Int32 (nullable), Float64."""
    import random

    rnd = random.Random(seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    key = pa.array([rnd.choice([None, rnd.getrandbits(30)]) for _ in range(n)], type=pa.int64())
    s = pa.array([rnd.choice([None, "", "N", "O", "phrase %d" % rnd.getrandbits(16), "x" * rnd.randint(0, 50)]) for _ in range(n)], type=pa.string())
    ls = pa.array([rnd.choice([None, "L" * rnd.randint(0, 9)]) for _ in range(n)], type=pa.large_string())
    bl = pa.array([rnd.choice([None, True, False]) for _ in range(n)], type=pa.bool_())
    i32 = pa.array([rnd.choice([None, rnd.getrandbits(31)]) for _ in range(n)], type=pa.int32())
    f64 = pa.array(rng.standard_normal(n))
    return pa.table([key, s, ls, bl, i32, f64], names=["key", "s", "ls", "bl", "i32", "f64"])


def in_columns(table, keep):
    cols = (COL * table.num_columns)()
    for i in range(table.num_columns):
        a = table.column(i).combine_chunks()
        keep.append(a)
        b = a.buffers()
        c, t = cols[i], a.type
        assert a.offset == 0
        c.validity = b[0].address if (b[0] is not None and a.null_count > 0) else None
        if pa.types.is_boolean(t):
            c.kind, c.values = nv.COL_BOOL, b[1].address
        elif pa.types.is_string(t) or pa.types.is_large_string(t):
            c.kind, c.offsets = (nv.COL_UTF8 if pa.types.is_string(t) else nv.COL_LARGE_UTF8), b[1].address
            c.values = b[2].address if b[2] is not None else None
            c.values_bytes = b[2].size if b[2] is not None else 0
        else:
            c.kind, c.width, c.values = nv.COL_FIXED, t.bit_width // 8, b[1].address
    return cols


class HostOut:
    """Host output buffers of `cap` rows (bitmaps in whole words) with FILL guard bytes behind every capacity."""

    def __init__(self, schema, cap, nbytes):
        self.schema, self.cap, self.bufs = schema, cap, {}
        self.cols = (COL * len(schema))()
        words = (cap + 31) // 32 * 4
        for i, f in enumerate(schema):
            c, t = self.cols[i], f.type
            if pa.types.is_boolean(t):
                c.kind, c.values = nv.COL_BOOL, self._buf(i, "values", words)
            elif pa.types.is_string(t) or pa.types.is_large_string(t):
                ow = 4 if pa.types.is_string(t) else 8
                c.kind = nv.COL_UTF8 if ow == 4 else nv.COL_LARGE_UTF8
                c.offsets = self._buf(i, "offsets", (cap + 1) * ow)
                c.values, c.values_bytes = self._buf(i, "values", nbytes[i]), nbytes[i]
            else:
                c.kind, c.width = nv.COL_FIXED, t.bit_width // 8
                c.values = self._buf(i, "values", cap * c.width)
            c.validity = self._buf(i, "validity", words)  # every column nullable in the schema

    def _buf(self, i, what, n):
        b = np.full(n + 64, FILL, dtype=np.uint8)
        self.bufs[(i, what)] = (b, n)
        return b.ctypes.data

    def guards_intact(self):
        return all((b[n:] == FILL).all() for b, n in self.bufs.values())

    def column(self, i, a, b, total):
        """rows [a, b) of out column i as a pyarrow array; also checks that the bitmap bits of rows [total, word end) are 0."""
        t = self.schema[i].type
        vb, _ = self.bufs[(i, "validity")]
        bitmaps = [vb] + ([self.bufs[(i, "values")][0]] if pa.types.is_boolean(t) else [])
        for bm in bitmaps:
            bits = np.unpackbits(bm[:(total + 31) // 32 * 4], bitorder="little")
            assert not bits[total:].any(), (i, total)
        validity = pa.py_buffer(vb.tobytes())
        if pa.types.is_boolean(t):
            bufs = [validity, pa.py_buffer(self.bufs[(i, "values")][0].tobytes())]
        elif pa.types.is_string(t) or pa.types.is_large_string(t):
            bufs = [validity, pa.py_buffer(self.bufs[(i, "offsets")][0].tobytes()), pa.py_buffer(self.bufs[(i, "values")][0].tobytes())]
        else:
            bufs = [validity, pa.py_buffer(self.bufs[(i, "values")][0].tobytes())]
        return pa.Array.from_buffers(t, b - a, bufs, offset=a)

    def offsets_start_at_zero(self):
        for (i, what), (b, _) in self.bufs.items():
            if what == "offsets":
                ow = 4 if pa.types.is_string(self.schema[i].type) else 8
                assert int(b[:ow].view(np.int32 if ow == 4 else np.int64)[0]) == 0, i


def expected(tables, dests, rank, n_chunks, ch, q):
    pieces = []
    for r, t in enumerate(tables):  # producers in task order, each with the rows of ITS chunk `ch`
        nr = t.num_rows
        lo, hi = nr * ch // n_chunks, nr * (ch + 1) // n_chunks
        pieces.append(t.slice(lo, hi - lo).take(pa.array(np.nonzero(dests[r][lo:hi] == rank * P + q)[0], type=pa.int64())))
    return pa.concat_tables(pieces)


def worker(lib, rank, world, uid, scenario, seed, errors, barrier):
    try:
        ctx = VP(lib.harness_ctx_create())
        ex = VP()
        RW.check(lib, lib.dfd_exchange_create(ctx, rank, world, uid, C.byref(ex)), "dfd_exchange_create")
        RW.check(lib, lib.dfd_exchange_setup_window(ex, 8 << 20), "dfd_exchange_setup_window")
        N = P * world
        part = VP()
        RW.check(lib, lib.dfd_partitioner_create(ctx, N, (C.c_int32 * 2)(0, 1), 2, None, C.byref(part)), "dfd_partitioner_create")
        few = [0, 37, 5, 1, 40, 12, 3, 29]  # more chunks than rows: most chunks are empty on some producer
        runs = [(1, 0, ROWS), (3, 1, ROWS), (7, 2, ROWS)] + ([(50, 3, few)] if scenario == "mixed" else [])
        for n_chunks, rep, rows in runs:
            tables = [mixed_table(rows[(r + rep) % 8], seed * 100 + 10 * rep + r) for r in range(world)]
            mine = tables[rank]
            keep = []
            in_cols = in_columns(mine, keep)
            dests = [orc.partition_ids([t.column(0), t.column(1)], t.num_rows, N) for t in tables]
            want = [[expected(tables, dests, rank, n_chunks, ch, q) for q in range(P)] for ch in range(n_chunks)]
            total = sum(w.num_rows for per in want for w in per)
            nbytes = {}
            chunk_bytes = []  # bytes of column "s" this worker receives per chunk
            for i, f in enumerate(mine.schema):
                if pa.types.is_string(f.type) or pa.types.is_large_string(f.type):
                    per = [sum(len((x or "").encode()) for w in per_ch for x in w.column(i).to_pylist()) for per_ch in want]
                    nbytes[i] = sum(per)
                    if i == 1:
                        chunk_bytes = per
            victim = scenario == "short" and rank == world - 1 and n_chunks > 1
            fail_at = None
            if victim:
                fail_at = next(ch for ch in range(n_chunks - 1) if chunk_bytes[ch] > 0)
                nbytes[1] = sum(chunk_bytes[:fail_at + 1]) - 1  # one byte short of what chunks 0..fail_at need
            out = HostOut(mine.schema, total, nbytes)
            cps = (C.c_int64 * (n_chunks * (P + 1)))()
            rc = lib.dfd_shuffle_host(ex, part, in_cols, mine.num_columns, mine.num_rows, P, n_chunks, out.cols, total, cps)
            err = lib.dfd_last_error()
            if scenario == "short" and n_chunks > 1:
                if victim:
                    assert rc == 7 and b"need %d string bytes" % (nbytes[1] + 1) in err, (rc, err)
                else:
                    assert rc != 0, (rank, "a peer of the refusing worker returned success")
                checked = range(fail_at) if victim else range(0)
            else:
                RW.check(lib, rc, "dfd_shuffle_host")
                checked = range(n_chunks)
                assert cps[n_chunks * (P + 1) - 1] == total
            assert lib.dfd_exchange_pending_segments(ex) == 0
            delivered = total if not victim else (cps[(fail_at - 1) * (P + 1) + P] if fail_at else 0)
            for ch in checked:
                for q in range(P):
                    a, b = cps[ch * (P + 1) + q], cps[ch * (P + 1) + q + 1]
                    w = want[ch][q]
                    assert b - a == w.num_rows, (n_chunks, ch, q, a, b, w.num_rows)
                    for i in range(mine.num_columns):
                        got = out.column(i, a, b, delivered)
                        got.validate(full=True)
                        assert got.equals(w.column(i).combine_chunks()), (n_chunks, ch, q, mine.schema[i].name)
            assert out.guards_intact(), (rank, n_chunks)
            if not victim:
                out.offsets_start_at_zero()
            barrier.wait()
            if scenario == "short" and n_chunks > 1:
                break  # (the workers that timed out have left the exchange's epochs behind)
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
    RW.bind(lib)
    uid = (C.c_uint8 * 128)()
    if world > 1:
        assert lib.dfd_nccl_unique_id(uid) == 0, lib.dfd_last_error()
    errors, barrier = [], threading.Barrier(world)
    threads = [threading.Thread(target=worker, args=(lib, r, world, uid, scenario, seed, errors, barrier)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=240)
    if errors or any(t.is_alive() for t in threads):
        print("\n".join(errors) or "a worker thread hung", file=sys.stderr)
        os._exit(1)
    print(f"WORKERS_OK world={world} scenario={scenario}")


if __name__ == "__main__":
    main()
