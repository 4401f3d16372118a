"""FixedSizeList payload through the host operator on one GPU: writes profiles/h100_fixed_size_list.json (or --out).

Measures, in one call, beside the card's name and power limit:
- the operator end to end (push, finish, every partition stream drained) for an Int64 key plus FixedSizeList<Float32, 768>
  or <Float32, 128>, with and without child nulls, host -> host, host -> device and device -> device, as rows/s and as input
  bytes/s next to the pinned duplex and device-to-device copy rates of the same run;
- k_gather_bit_rows device time (torch.profiler) in a partition of FixedSizeList<Boolean, n>, n = 1, 7, 8, 33, 768, next to
  k_gather_rows on FixedSizeList<UInt8, n / 8> rows where that width is gathered (n / 8 outside 1/2/4/8/16 bytes);
- host -> host end to end of the 768 schema with chunks sized to 64, 256 and 1024 MiB of fixed-width bytes.

Usage: python scripts/fixed_size_list_profile.py [--reps 3] [--out path]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import pyarrow as pa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import datafusion_distributed_b200 as dfd  # noqa: E402
from host_shuffle_profile import copy_rates, gpu_info  # noqa: E402
from tests import test_exec_fixed_size_list_gpu as G  # noqa: E402  (batch builders and device-batch helper)

N_PART = 8
BATCH = 65_536


def batches_of(rng, n_rows, t, n, child_nulls):
    out = []
    for lo in range(0, n_rows, BATCH):
        rows = min(BATCH, n_rows - lo)
        out.append(G._batch(G._keys(rng, rows), G.fsl_array(rng, t, n, rows, parent_nulls=0.01 if child_nulls else 0.0, child_nulls=child_nulls)))
    return out


def run_once(torch, ctx, mode, batches, **opts):
    """Seconds from the first push to the last partition batch received (device output: and its device work done)."""
    schema = batches[0].schema
    dev_in = [G.FslDeviceBatch(rb) for rb in batches] if mode[0] == "d" else None
    torch.cuda.synchronize()
    ex = dfd.RepartitionExec(ctx, schema, dfd.Partitioning.Hash([0], N_PART), device_output=mode[1] == "d", **opts)
    t0 = time.perf_counter()
    for k, rb in enumerate(batches):
        if dev_in is None:
            ex.push_batch(rb)
        else:
            ex.push_device_batch(dev_in[k].device_array)
    ex.finish()
    rows = 0
    for p in range(N_PART):
        if mode[1] == "h":
            rows += sum(b.num_rows for b in ex.execute(p))
        else:
            for b in ex.execute_device(p):
                rows += b.array.length
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    ex.close()
    assert rows == sum(b.num_rows for b in batches)
    return dt


def input_bytes(batches):
    return sum(sum(buf.size for buf in c.buffers() if buf is not None) for b in batches for c in b.columns)


def kernel_us(torch, ctx, batches, name):
    from torch.profiler import ProfilerActivity, profile

    run_once(torch, ctx, "hh", batches)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_once(torch, ctx, "hh", batches)
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and name in e.name]
    return {"launches": len(ts), "us_total": float(sum(ts)), "us_per_launch": float(np.mean(ts)) if ts else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fixed_size_list.json"))
    args = ap.parse_args()
    import torch

    name, power = gpu_info()
    ctx = dfd.WorkerContext(0)
    rates = copy_rates(torch)
    nb = 1 << 30
    a, b = torch.empty(nb, dtype=torch.uint8, device="cuda"), torch.empty(nb, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(6):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b.copy_(a)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    rates["device_copy_GBps"] = 2 * nb / float(np.median(ts[1:])) / 1e9  # (read + write)
    del a, b
    rec = {"gpu": name, "power_limit": power, "partitions": N_PART, "batch_rows": BATCH, "copy_rates": rates, "end_to_end": [], "kernels": [], "chunk_budget": []}
    rng = np.random.Generator(np.random.PCG64(1))
    for n, n_rows in ((768, 1 << 18), (128, 1 << 20)):
        for child_nulls in (0.0, 0.1):
            batches = batches_of(rng, n_rows, pa.float32(), n, child_nulls)
            nbytes = input_bytes(batches)
            for mode in ("hh", "hd", "dd"):
                run_once(torch, ctx, mode, batches)  # (warm-up: pinned and device chunks, module loads)
                dts = [run_once(torch, ctx, mode, batches) for _ in range(args.reps)]
                dt = float(np.median(dts))
                rec["end_to_end"].append({"n": n, "rows": n_rows, "child_nulls": child_nulls, "mode": mode, "s": dt, "rows_per_s": n_rows / dt,
                                          "input_GBps": nbytes / dt / 1e9, "input_bytes": nbytes})
                print(rec["end_to_end"][-1], flush=True)
            del batches
    for n in (1, 7, 8, 33, 768):
        n_rows = (1 << 24) // max(n // 8, 1) if n < 768 else 1 << 20
        batches = batches_of(rng, n_rows, pa.bool_(), n, 0.0)
        k = {"n": n, "rows": n_rows, "k_gather_bit_rows": kernel_us(torch, ctx, batches, "k_gather_bit_rows")}
        w = n // 8
        if n % 8 == 0 and w not in (1, 2, 4, 8, 16):
            k["k_gather_rows_at_n_over_8_bytes"] = kernel_us(torch, ctx, batches_of(rng, n_rows, pa.uint8(), w, 0.0), "k_gather_rows")
        else:
            k["k_gather_rows_at_n_over_8_bytes"] = "not measured: n / 8 bytes is not a whole width, or a width the scatter moves"
        rec["kernels"].append(k)
        print(k, flush=True)
        del batches
    batches = batches_of(rng, 1 << 18, pa.float32(), 768, 0.1)
    bits_per_row = 64 + 8 * 3072 + 1 + 768
    for mib in (64, 256, 1024):
        chunk_rows = (mib << 20) * 8 // bits_per_row // 64 * 64
        run_once(torch, ctx, "hh", batches, chunk_rows=chunk_rows)
        dt = float(np.median([run_once(torch, ctx, "hh", batches, chunk_rows=chunk_rows) for _ in range(args.reps)]))
        rec["chunk_budget"].append({"budget_MiB": mib, "chunk_rows": chunk_rows, "s": dt, "rows_per_s": (1 << 18) / dt, "input_GBps": input_bytes(batches) / dt / 1e9})
        print(rec["chunk_budget"][-1], flush=True)
    ctx.close()
    with open(args.out, "w") as f:
        json.dump(rec, f)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
