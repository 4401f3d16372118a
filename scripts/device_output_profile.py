"""Device-resident OUTPUT of the host operator (device_output / execute_device) against host output, on the GPU.

    python scripts/device_output_profile.py [--out FILE] [--reps 3]

1. cfg-2-shaped chunks (2^26 rows x 8 Int64, Hash([0], 8)) and
2. the reference's 9-column bench schema at 8192-row batches,
each through a host -> host, a device -> host and a device -> device operator, alternated, after one warm-up round: rows/s
from a host clock around first push -> every partition stream drained -> device synchronise.  For device -> device the
algorithmic bytes per row are stated too (staging copy + partition, each a read and a write: 4 * C * w), and the rate they
imply.  A consumer of a device stream here releases each batch as it comes (it reads nothing).
3. In a separate process, a torch.profiler pass over a device -> device run of the 9-column schema: launches of
k_emit_chunk, and the largest device-to-host copy seen (part_starts and size read-backs only: no payload).

Prints one JSON line (GPU name and power limit included) and writes it to --out when given.  Fails without a GPU."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench_workloads as W  # noqa: E402
import datafusion_distributed_b200 as dfd  # noqa: E402
import device_input_profile as DIP  # noqa: E402
from datafusion_distributed_b200.execution_plans import PinnedTable  # noqa: E402
from tests import device_batches as DB  # noqa: E402

MODES = ("host_to_host", "device_to_host", "device_to_device")


def drain_device(ex, N):
    """Consumers of every device stream, concurrently; a batch is released when the next is asked for."""
    threads = [threading.Thread(target=lambda p=p: [None for _ in ex.execute_device(p)]) for p in range(N)]
    for t in threads:
        t.start()
    return threads


def timed_run(torch, ctx, schema, N, mode, push_host, push_device, **opts):
    device_out = mode == "device_to_device"
    ex = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash([0], N), device_output=device_out, **opts)
    threads = drain_device(ex, N) if device_out else DIP.drain(ex, N)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    (push_host if mode == "host_to_host" else push_device)(ex)
    ex.finish()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = ex.stats()
    ex.close()
    return wall, st


def measure(torch, ctx, schema, N, n_rows, reps, push_host, push_device, **opts):
    walls, stats = {m: [] for m in MODES}, {}
    for rep in range(reps + 1):  # (round 0 warms every shape up and is not recorded)
        for m in MODES:
            w, st = timed_run(torch, ctx, schema, N, m, push_host, push_device, **opts)
            assert st["rows_out"] == n_rows, (m, st)
            if rep:
                walls[m].append(w)
                stats[m] = st
    out = {}
    for m in MODES:
        out[m] = {"rows_per_s": n_rows / min(walls[m]), "wall_s": sorted(walls[m]), "bytes_h2d": stats[m]["bytes_h2d"], "bytes_d2h": stats[m]["bytes_d2h"],
                  "ns_push": stats[m]["ns_push"], "ns_wait_pool": stats[m]["ns_wait_pool"]}
    return out


def cfg2(torch, ctx, reps):
    n, ncol, N, batch = 1 << 26, 8, 8, 1 << 22
    rng = np.random.Generator(np.random.PCG64(2))
    host = PinnedTable(ctx, n, [np.int64] * ncol)
    for c in host.columns:
        c[:] = rng.integers(-(2**62), 2**62, n, dtype=np.int64)
    host_batches = host.record_batches([f"c{i}" for i in range(ncol)], batch)
    dev_cols = [torch.from_numpy(c).to("cuda") for c in host.columns]
    torch.cuda.synchronize()
    dev_batches = [DIP.TorchDeviceBatch(dev_cols, lo, min(batch, n - lo)) for lo in range(0, n, batch)]
    out = {"rows": n, "columns": ncol, "partitions": N, "batch_rows": batch}
    out.update(measure(torch, ctx, host_batches[0].schema, N, n, reps, lambda ex: [ex.push_batch(b) for b in host_batches],
                       lambda ex: [ex.push_device_batch(b.fresh()) for b in dev_batches]))
    dd = out["device_to_device"]
    assert dd["bytes_h2d"] == 0 and dd["bytes_d2h"] == 0
    dd["algorithmic_bytes_per_row"] = 4 * ncol * 8  # staging copy + partition: read + write of C columns of w bytes, twice
    dd["algorithmic_bytes_per_s"] = dd["rows_per_s"] * dd["algorithmic_bytes_per_row"]
    del dev_batches, dev_cols
    host.close()
    return out


def compact(batch):
    """The batch with buffers of its own (a slice of a table shares the table's: a device copy of it would copy them whole)."""
    import pyarrow as pa

    sink = pa.BufferOutputStream()
    with pa.ipc.new_stream(sink, batch.schema) as w:
        w.write_batch(batch)
    return pa.ipc.open_stream(sink.getvalue()).read_next_batch()


def fixture(torch, ctx, reps):
    n, N = 1 << 20, 8
    table = W.fixture_table(n)
    batches = [compact(b) for b in table.to_batches(max_chunksize=8192)]

    def push_device(ex):  # (a new set per run: a pushed batch belongs to the operator; the copies are made before the clock starts)
        for b in push_device.ready.pop():
            ex.push_device_batch(b.device_array)

    push_device.ready = [[DB.DeviceBatch(b) for b in batches] for _ in range(2 * (reps + 1))]
    torch.cuda.synchronize()
    out = {"rows": n, "batch_rows": 8192, "batches": len(batches), "partitions": N}
    out.update(measure(torch, ctx, table.schema, N, n, reps, lambda ex: [ex.push_batch(b) for b in batches], push_device, chunk_rows=1 << 20))
    return out


def trace_pass(path):
    """The profiler run (its own process): device -> device over the 9-column schema; what the trace shows goes to `path`."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    ctx = dfd.WorkerContext(0)
    n, N = 1 << 18, 8
    table = W.fixture_table(n)
    batches = [DB.DeviceBatch(compact(b)) for b in table.to_batches(max_chunksize=8192)]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        ex = dfd.RepartitionExec(ctx, table.schema, dfd.Partitioning.Hash([0], N), device_output=True, chunk_rows=1 << 16)
        threads = drain_device(ex, N)
        for b in batches:
            ex.push_device_batch(b.device_array)
        ex.finish()
        for t in threads:
            t.join()
        torch.cuda.synchronize()
        st = ex.stats()
        ex.close()
    trace = os.path.join(os.path.dirname(path), "device_output.pt.trace.json")
    prof.export_chrome_trace(trace)
    events = [e for e in json.load(open(trace))["traceEvents"] if isinstance(e, dict) and e.get("cat") in ("kernel", "gpu_memcpy")]
    d2h = [int(e.get("args", {}).get("bytes", 0)) for e in events if e["cat"] == "gpu_memcpy" and "DtoH" in e["name"]]
    kernels = sorted({e["name"].split("(")[0] for e in events if e["cat"] == "kernel"})
    out = {"rows": n, "chunk_rows": 1 << 16, "k_emit_chunk_launches": sum(1 for e in events if e["cat"] == "kernel" and "k_emit_chunk" in e["name"]),
           "memcpy_dtoh_count": len(d2h), "memcpy_dtoh_max_bytes": max(d2h, default=0), "operator_bytes_d2h": st["bytes_d2h"],
           "payload_bytes_per_chunk_at_least": (1 << 16) * 8, "kernels": kernels}
    ctx.close()
    with open(path, "w") as f:
        json.dump(out, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trace-to", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures the GPU path only")
    if args.trace_to:
        return trace_pass(args.trace_to)
    name, power = DIP.gpu_info()
    ctx = dfd.WorkerContext(0)
    line = {"profile": "device_output", "gpu": name, "power_limit": power, "cfg2": cfg2(torch, ctx, args.reps), "fixture": fixture(torch, ctx, args.reps)}
    ctx.close()
    with tempfile.TemporaryDirectory() as tmp:  # the profiler pass: a process of its own, so that tracing slows nothing timed above
        part = os.path.join(tmp, "trace.json")
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--trace-to", part])
        line["profiler"] = json.load(open(part))
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
