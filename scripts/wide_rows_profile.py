"""k_gather_rows against a device copy of the same bytes, on the GPU.

    python scripts/wide_rows_profile.py [--out FILE] [--reps 5]

A two-pass partition (dfd_partition_device, Hash([0], 8)) of an Int64 key and one FixedSizeList<Float32, n> column, moved as
one fixed-width column of w = 4n bytes, for n in {3, 16, 64, 768} (12 B to 3 KiB per row): 2^24 rows, except 2^21 rows for
n = 768 (2^24 rows of 3 KiB would need 103 GB for the input and output alone).  After one warm-up call per shape, in one
torch.profiler session, the calls alternate with a device-to-device copy_ of the column's n_rows x w bytes; the trace
gives each k_gather_rows launch and each copy its device time.  Reported per n: best and spread of the --reps gather and
copy times, the achieved rate over the 2 w algorithmic bytes a gathered row needs (one read, one write; the 4-byte input
row index per row is not counted), and its fraction of the copy's rate over the same bytes.  The whole partition call
(K1, K1b, K2 and the gather) is timed apart with CUDA events, profiler off.

Prints one JSON line (GPU name and power limit included) and writes it to --out when given.  Fails without a GPU."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import datafusion_distributed_b200 as dfd  # noqa: E402
import device_input_profile as DIP  # noqa: E402
from datafusion_distributed_b200 import _native as nv  # noqa: E402

SHAPES = [(3, 1 << 24), (16, 1 << 24), (64, 1 << 24), (768, 1 << 21)]
N = 8


def fixed(t, w, n):
    return dfd.DeviceColumn(nv.COL_FIXED, w, t.data_ptr(), 0, 0, 0, n, (t,))


def spread(v):
    return {"best": min(v), "median": float(np.median(v)), "worst": max(v)}


def shape_case(torch, ctx, d, n, reps):
    w = 4 * d
    g = torch.Generator(device="cuda").manual_seed(d)
    key = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device="cuda", generator=g)
    vals = torch.rand((n, d), dtype=torch.float32, device="cuda", generator=g)
    out, copy_dst, out_key = torch.empty_like(vals), torch.empty_like(vals), torch.empty_like(key)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    ins = [dfd.DeviceColumn.from_torch(key), fixed(vals, w, n)]
    outs = [dfd.DeviceColumn.from_torch(out_key), fixed(out, w, n)]

    def call():
        part.partition(ins, n, outs, sync=False)

    torch.cuda.synchronize()  # (the library works on a stream of its own: the random inputs must have landed)
    call()
    copy_dst.copy_(vals)
    torch.cuda.synchronize()
    # whole partition calls, profiler off
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    s = torch.cuda.current_stream()
    for a, b in ev:
        ctx.synchronize()
        a.record(s)
        call()
        ctx.synchronize()  # (the library's own stream: the end event follows it)
        b.record(s)
    torch.cuda.synchronize()
    call_ms = [a.elapsed_time(b) for a, b in ev]
    # kernel times from the trace: gather and copy alternated
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
            ctx.synchronize()
            copy_dst.copy_(vals)
            torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = [e for e in json.load(open(path))["traceEvents"] if isinstance(e, dict) and e.get("cat") in ("kernel", "gpu_memcpy")]
    gather_us = [e["dur"] for e in events if e["cat"] == "kernel" and "k_gather_rows" in e["name"]]
    copy_us = [e["dur"] for e in events if e["cat"] == "gpu_memcpy" and "DtoD" in e["name"]]
    if len(gather_us) != reps or len(copy_us) != reps:
        raise SystemExit(f"n={d}: expected {reps} gathers and copies in the trace, found {len(gather_us)} and {len(copy_us)}")
    byts = 2 * n * w
    gb, cb = min(gather_us), min(copy_us)
    del key, vals, out, copy_dst, out_key, ins, outs
    torch.cuda.empty_cache()
    return {"n": d, "row_bytes": w, "rows": n, "gather_us": spread(gather_us), "copy_us": spread(copy_us),
            "gather_tb_s": byts / gb / 1e6, "copy_tb_s": byts / cb / 1e6, "fraction_of_copy": cb / gb, "partition_call_ms": spread(call_ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures the GPU path only")
    name, power = DIP.gpu_info()
    ctx = dfd.WorkerContext(0)
    line = {"profile": "wide_rows", "gpu": name, "power_limit": power, "N": N, "reps": args.reps,
            "raw_partition": [shape_case(torch, ctx, d, n, args.reps) for d, n in SHAPES]}
    ctx.close()
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
