"""dfd_shuffle_host throughput on the GPU: today's fixed-width path against the push path of nullable / Boolean / string schemas.

    python scripts/host_shuffle_profile.py [--out FILE] [--reps 3] [--rows 16777216,67108864] [--chunks 1,4,16]
    python -m torch.distributed.run --nproc-per-node T scripts/host_shuffle_profile.py ...   (world T, one rank per GPU)

Schemas, pinned host columns in and out:
  fixed8   8 x Int64, non-null: the two-pass fused path (two window slots)
  mixed    Int64 (nullable), Utf8 of 0-16 bytes, LargeUtf8 of 0-9 bytes, Boolean, Int32 (nullable), Float64, 10 % nulls;
           keys Int64 + Utf8: the push path (the whole window per chunk, then the compaction)
Per (schema, rows, n_chunks): the median wall time of --reps synchronous calls after one warm-up call, as rows/s and as
host bytes/s (input bytes + output bytes over the wall time), next to the pinned H2D, D2H and duplex (both directions at
once) copy rates measured in the same run with 1 GiB copies.  A separate torch.profiler run of one mixed call per n_chunks at
the smallest size gives the compaction's device time per call (the k_push_runs launch that follows the push transport's
done barrier, plus k_place_bits) and the push transport's own k_push_runs time.

Prints one JSON line (GPU name and power limit included) and writes it to --out when given.  Fails without a GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import datafusion_distributed_b200 as dfd  # noqa: E402
from datafusion_distributed_b200 import _native as nv  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    return name, power


class Pinned:
    """One pinned host buffer (dfd_host_alloc) as a numpy uint8 array."""

    def __init__(self, ctx, nbytes):
        self.ctx, p = ctx, C.c_void_p()
        nv.check(nv.lib().dfd_host_alloc(ctx.handle, max(nbytes, 16), C.byref(p)))
        self.p = p
        self.a = np.frombuffer((C.c_char * max(nbytes, 16)).from_address(p.value), dtype=np.uint8)[:nbytes]
        self.addr = p.value

    def close(self):
        nv.lib().dfd_host_free(self.ctx.handle, self.p)


def pinned_from(ctx, arr, keep):
    b = Pinned(ctx, arr.nbytes)
    b.a[:] = arr.view(np.uint8).reshape(-1)
    keep.append(b)
    return b.addr


def bitmap(rng, n, p_null):
    return np.packbits(rng.random(n) >= p_null, bitorder="little")


def make_table(ctx, schema, n, seed, keep):
    """(host input columns, host output columns, input bytes, keys) of `schema` at n rows, every buffer pinned."""
    rng = np.random.Generator(np.random.PCG64(seed))
    ins, outs, nbytes = [], [], 0
    words = (n + 31) // 32 * 4
    if schema == "fixed8":
        for c in range(8):
            v = rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64, endpoint=True) if c == 0 else np.arange(n, dtype=np.int64) * 8 + c
            ins.append(dfd.DeviceColumn(nv.COL_FIXED, 8, pinned_from(ctx, v, keep), length=n))
            keep.append(Pinned(ctx, n * 8))
            outs.append(dfd.DeviceColumn(nv.COL_FIXED, 8, keep[-1].addr, length=n))
            nbytes += n * 8
        return ins, outs, nbytes, [0]

    def fixed(v, nullable):
        nonlocal nbytes
        val = pinned_from(ctx, bitmap(rng, n, 0.1), keep) if nullable else 0
        ins.append(dfd.DeviceColumn(nv.COL_FIXED, v.itemsize, pinned_from(ctx, v, keep), 0, val, 0, n))
        outs.append(dfd.DeviceColumn(nv.COL_FIXED, v.itemsize, pinned_from(ctx, np.zeros(n * v.itemsize, np.uint8), keep), 0,
                                     pinned_from(ctx, np.zeros(words, np.uint8), keep), 0, n))
        nbytes += n * v.itemsize + (n + 7) // 8 * nullable

    def string(kind, max_len, dt):
        nonlocal nbytes
        lens = rng.integers(0, max_len + 1, n)
        off = np.zeros(n + 1, dtype=dt)
        np.cumsum(lens, out=off[1:])
        data = rng.integers(32, 127, int(off[-1]), dtype=np.uint8)
        ins.append(dfd.DeviceColumn(kind, 0, pinned_from(ctx, data, keep), pinned_from(ctx, off, keep), pinned_from(ctx, bitmap(rng, n, 0.1), keep),
                                    0, n, None, None, int(off[-1])))
        outs.append(dfd.DeviceColumn(kind, 0, pinned_from(ctx, np.zeros(int(off[-1]), np.uint8), keep), pinned_from(ctx, np.zeros(n + 1, dt), keep),
                                     pinned_from(ctx, np.zeros(words, np.uint8), keep), 0, n, None, None, int(off[-1])))
        nbytes += int(off[-1]) + off.nbytes + (n + 7) // 8

    fixed(rng.integers(0, 1 << 40, n, dtype=np.int64), True)
    string(nv.COL_UTF8, 16, np.int32)
    string(nv.COL_LARGE_UTF8, 9, np.int64)
    ins.append(dfd.DeviceColumn(nv.COL_BOOL, 0, pinned_from(ctx, bitmap(rng, n, 0.5), keep), 0, 0, 0, n))
    outs.append(dfd.DeviceColumn(nv.COL_BOOL, 0, pinned_from(ctx, np.zeros(words, np.uint8), keep), 0, pinned_from(ctx, np.zeros(words, np.uint8), keep), 0, n))
    nbytes += (n + 7) // 8
    fixed(rng.integers(0, 1 << 31, n, dtype=np.int64).astype(np.int32), True)
    fixed(rng.standard_normal(n), False)
    return ins, outs, nbytes, [0, 1]


def window_bytes(schema, n, world):
    per = n // world
    return int(per * (8 * 8 * 2 if schema == "fixed8" else 60) * 1.3) + (64 << 20)


def copy_rates(torch):
    """Pinned H2D, D2H and duplex GB/s with 1 GiB copies (median of 5)."""
    nb = 1 << 30
    h1, h2 = torch.empty(nb, dtype=torch.uint8, pin_memory=True), torch.empty(nb, dtype=torch.uint8, pin_memory=True)
    d1, d2 = torch.empty(nb, dtype=torch.uint8, device="cuda"), torch.empty(nb, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def timed(fn):
        ts = []
        for _ in range(6):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts[1:]))

    def duplex():
        with torch.cuda.stream(s1):
            d1.copy_(h1, non_blocking=True)
        with torch.cuda.stream(s2):
            h2.copy_(d2, non_blocking=True)

    return {"h2d_GBps": nb / timed(lambda: d1.copy_(h1, non_blocking=True)) / 1e9, "d2h_GBps": nb / timed(lambda: h2.copy_(d2, non_blocking=True)) / 1e9,
            "duplex_GBps": 2 * nb / timed(duplex) / 1e9}


def compaction_ms(torch, node, ex, ins, outs, n, n_chunks):
    """Device ms per call of the compaction (k_push_runs after k_xchg_done_barrier, and k_place_bits) and of the push
    transport's own k_push_runs, from one torch.profiler session over one call."""
    from torch.profiler import ProfilerActivity, profile

    node.shuffle_host(ex, ins, n, n_chunks, outs, n)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        node.shuffle_host(ex, ins, n, n_chunks, outs, n)
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    comp = push = 0.0
    after_barrier = False
    for e in kernels:
        name = e.name
        if "k_xchg_done_barrier" in name:
            after_barrier = True
        elif "k_push_runs" in name:
            if after_barrier:
                comp += e.device_time / 1e3
            else:
                push += e.device_time / 1e3
            after_barrier = False
        elif "k_place_bits" in name:
            comp += e.device_time / 1e3
        elif "k_xchg_allgather_meta" in name:
            after_barrier = False
    return {"compaction_ms": comp, "push_runs_ms": push}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rows", default="16777216,67108864")
    ap.add_argument("--chunks", default="1,4,16")
    args = ap.parse_args()
    import torch

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    uid = None
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        box = [dfd.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        uid = box[0]
    name, power = gpu_info()
    ctx = dfd.WorkerContext(local)
    rates = copy_rates(torch)
    results, profiles = [], {}
    sizes = [int(s) for s in args.rows.split(",")]
    for schema in ("fixed8", "mixed"):
        for n in sizes:
            keep = []
            per = n // world
            ins, outs, in_bytes, keys = make_table(ctx, schema, per, 7 + rank, keep)
            ex = dfd.ShuffleExchange(ctx, rank, world, uid)
            ex.setup_window(window_bytes(schema, n, world))
            node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash(keys, 8), uuid.uuid4(), 1, world, world)
            for n_chunks in [int(c) for c in args.chunks.split(",")]:
                cap = per * 2 if world > 1 else per
                node.shuffle_host(ex, ins, per, n_chunks, outs, cap)  # warm-up (stages, streams, run buffers)
                ts = []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    cps = node.shuffle_host(ex, ins, per, n_chunks, outs, cap)
                    ts.append(time.perf_counter() - t0)
                if world == 1:
                    assert cps[-1, -1] == per
                t = float(np.median(ts))
                rec = {"schema": schema, "rows": n, "n_chunks": n_chunks, "world": world, "ms": t * 1e3, "rows_per_s": per / t,
                       "host_GBps": 2 * in_bytes / t / 1e9}
                if schema == "mixed" and n == sizes[0]:
                    rec.update(compaction_ms(torch, node, ex, ins, outs, per, n_chunks))
                results.append(rec)
                print(json.dumps(rec), file=sys.stderr, flush=True)
            ex.close()
            for b in keep:
                if isinstance(b, Pinned):
                    b.close()
    line = {"profile": "host_shuffle", "gpu": name, "power_limit": power, "world": world, "reps": args.reps, "copy_rates": rates,
            "unit": "ms: median wall ms per synchronous dfd_shuffle_host call; host_GBps: (input + output host bytes) / ms; "
                    "compaction_ms / push_runs_ms: device ms per call from a torch.profiler trace", "results": results}
    s = json.dumps(line)
    if rank == 0:
        print(s)
        if args.out:
            with open(args.out, "w") as f:
                f.write(s + "\n")
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
