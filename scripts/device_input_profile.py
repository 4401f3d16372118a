"""Device-resident input of the host operator (dfd_repartition_exec_push_device) against host input, on the GPU.

    python scripts/device_input_profile.py [--out FILE] [--reps 3]

1. cfg-2 (2^26 rows x 8 Int64, Hash([0], 8)): the same rows pushed as device batches and as pinned host batches, rows/s
   end to end (first push -> every partition stream drained), and the D2H copy rate alone measured in the same run: a
   device batch moves no input over PCIe, so its bound is the D2H of the output alone.
2. The reference's 9-column bench schema at 8192-row batches: producer time per batch (ns_push / batches) and rows/s for
   device against host input.

Prints one JSON line (GPU name and power limit included) and writes it to --out when given."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench_workloads as W  # noqa: E402
import datafusion_distributed_b200 as dfd  # noqa: E402
from datafusion_distributed_b200 import _native as nv  # noqa: E402
from datafusion_distributed_b200.execution_plans import PinnedTable  # noqa: E402
from tests import device_batches as DB  # noqa: E402

_NOOP = C.CFUNCTYPE(None, C.POINTER(nv.ArrowArrayStruct))(lambda a: setattr(a.contents, "release", None))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    return name, power


def drain(ex, N):
    """Consumers of every partition stream, concurrently (batches dropped as they come); returns the threads."""
    threads = [threading.Thread(target=lambda p=p: [None for _ in ex.execute(p)]) for p in range(N)]
    for t in threads:
        t.start()
    return threads


def timed_run(ctx, schema, N, push_all, **opts):
    ex = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash([0], N), **opts)
    threads = drain(ex, N)
    t0 = time.perf_counter()
    push_all(ex)
    ex.finish()
    for t in threads:
        t.join()
    wall = time.perf_counter() - t0
    st = ex.stats()
    ex.close()
    return wall, st


class TorchDeviceBatch:
    """Zero-copy ArrowDeviceArray over rows [lo, lo + n) of device-resident int64 columns (torch tensors)."""

    def __init__(self, cols, lo, n):
        self.kids = [nv.ArrowArrayStruct() for _ in cols]
        self.bufs = [(C.c_void_p * 2)(None, c.data_ptr()) for c in cols]
        for k, b in zip(self.kids, self.bufs):
            k.length, k.null_count, k.offset, k.n_buffers = n, 0, lo, 2
            k.buffers, k.release = C.cast(b, C.c_void_p), C.cast(_NOOP, C.c_void_p)
        self.ptrs = (C.POINTER(nv.ArrowArrayStruct) * len(cols))(*[C.pointer(k) for k in self.kids])
        self.top_bufs = (C.c_void_p * 1)(None)
        self.dev = nv.ArrowDeviceArrayStruct()
        a = self.dev.array
        a.length, a.n_buffers, a.n_children = n, 1, len(cols)
        a.buffers, a.children, a.release = C.cast(self.top_bufs, C.c_void_p), C.cast(self.ptrs, C.c_void_p), C.cast(_NOOP, C.c_void_p)
        self.dev.device_type, self.dev.device_id = DB.ARROW_DEVICE_CUDA, 0

    def fresh(self):  # (a push takes ownership and clears `release`: set it again to push the same rows once more)
        self.dev.array.release = C.cast(_NOOP, C.c_void_p)
        return self.dev


def d2h_rate(torch, nbytes=1 << 30, reps=5):
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    best = 0.0
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src, non_blocking=True)
        b.record()
        b.synchronize()
        best = max(best, nbytes / (a.elapsed_time(b) / 1e3))
    return best


def cfg2(torch, ctx, reps):
    n, ncol, N, batch = 1 << 26, 8, 8, 1 << 22
    rng = np.random.Generator(np.random.PCG64(2))
    host = PinnedTable(ctx, n, [np.int64] * ncol)
    for c in host.columns:
        c[:] = rng.integers(-(2**62), 2**62, n, dtype=np.int64)
    names = [f"c{i}" for i in range(ncol)]
    host_batches = host.record_batches(names, batch)
    schema = host_batches[0].schema
    dev_cols = [torch.from_numpy(c).to("cuda") for c in host.columns]
    torch.cuda.synchronize()
    dev_batches = [TorchDeviceBatch(dev_cols, lo, min(batch, n - lo)) for lo in range(0, n, batch)]
    out = {"rows": n, "columns": ncol, "partitions": N, "batch_rows": batch}
    walls = {"device": [], "host": []}
    for _ in range(reps):
        w, st = timed_run(ctx, schema, N, lambda ex: [ex.push_device_batch(b.fresh()) for b in dev_batches])
        walls["device"].append(w)
        assert st["bytes_h2d"] == 0 and st["rows_out"] == n
        w, st = timed_run(ctx, schema, N, lambda ex: [ex.push_batch(b) for b in host_batches])
        walls["host"].append(w)
        assert st["rows_out"] == n
    for k, v in walls.items():
        out[f"{k}_rows_per_s"] = n / min(v)
        out[f"{k}_wall_s"] = sorted(v)
    rate = d2h_rate(torch)
    out["d2h_bytes_per_s"] = rate
    out["d2h_bound_rows_per_s"] = rate / (8 * ncol)  # (every output byte crosses PCIe once, D2H)
    del dev_batches, dev_cols
    host.close()
    return out


def fixture(torch, ctx, reps):
    n, N = 1 << 20, 8
    table = W.fixture_table(n)
    batches = table.to_batches(max_chunksize=8192)
    out = {"rows": n, "batch_rows": 8192, "batches": len(batches), "partitions": N}
    res = {"device": [], "host": []}
    for _ in range(reps):
        dev = [DB.DeviceBatch(b) for b in batches]  # (a new set per run: a pushed batch belongs to the operator; copies not timed)
        torch.cuda.synchronize()
        w, st = timed_run(ctx, table.schema, N, lambda ex: [ex.push_device_batch(b.device_array) for b in dev], chunk_rows=1 << 20)
        res["device"].append((w, st["ns_push"] / len(batches), st["bytes_d2h"], st["bytes_h2d"]))
        w, st = timed_run(ctx, table.schema, N, lambda ex: [ex.push_batch(b) for b in batches], chunk_rows=1 << 20)
        res["host"].append((w, st["ns_push"] / len(batches), st["bytes_d2h"], st["bytes_h2d"]))
    for k, v in res.items():
        best = min(v)
        out[f"{k}_rows_per_s"] = n / best[0]
        out[f"{k}_ns_push_per_batch"] = min(x[1] for x in v)
        out[f"{k}_bytes_h2d"] = best[3]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures the GPU path only")
    name, power = gpu_info()
    ctx = dfd.WorkerContext(0)
    line = {"profile": "device_input", "gpu": name, "power_limit": power, "cfg2": cfg2(torch, ctx, args.reps), "fixture": fixture(torch, ctx, args.reps)}
    ctx.close()
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
