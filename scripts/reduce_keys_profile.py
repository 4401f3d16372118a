"""PartialReduce device time per kernel for Boolean and string group keys, and cfg-3 (TPC-H q1) end to end, on the GPU.

    python scripts/reduce_keys_profile.py [--out FILE] [--reps 5] [--rows 67108864]

Key cases, each with one COUNT state (SUM_I64), all rows in one partition, group ids drawn uniformly at random:
  i64            one Int64 key (the fixed-key kernels: the baseline)
  utf8_1         one Utf8 key of 1 byte (q1's l_returnflag-like; at most 256 groups)
  utf8_8_16      one Utf8 key of 8-16 bytes
  large_32_64    one key of 32-64 bytes (SearchPhrase-like).  LargeUtf8: at 2^26 rows its ~3.2 GB of bytes pass the
                 2^31 - 1 that Utf8's int32 offsets can address
  i64_utf8       an Int64 key and a Utf8 key of 8-16 bytes (cfg-5's key shape)
  utf8_utf8      two Utf8 keys of 1 and 8-16 bytes
  bool           one Boolean key (at most 2 groups without nulls)
at 4, 2^10, 2^20 and 2^25 groups where the key admits them (utf8_1: 4 and 256; bool: 2).  A string's length is a function
of its group, and its first 8 bytes are the group id, so keys are distinct exactly when their groups are.  After one
warm-up call per case, --reps calls run in one torch.profiler session; every kernel's device time is summed per call
(a key kind's launches: k_insert_keys ... k_copy_key_bytes) and the median over the calls is reported, with the median
wall time of --reps synchronous calls outside the profiler.

q1: cfg3_columns(0) rows (24 rows, and the same schema at 2^20 rows) through partition (N = 4) -> reduce ->
shuffle_partitioned at world 1, µs per step (median of 50 steps after 5 warm-up steps).

Prints one JSON line (GPU name and power limit included) and writes it to --out when given.  Fails without a GPU."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import device_input_profile as DIP  # noqa: E402
import datafusion_distributed_b200 as dfd  # noqa: E402
from datafusion_distributed_b200 import _native as nv  # noqa: E402

CASES = {  # name -> key columns: ("i64",) / ("bool",) / (kind, min length, max length)
    "i64": [("i64",)], "utf8_1": [("utf8", 1, 1)], "utf8_8_16": [("utf8", 8, 16)], "large_32_64": [("large", 32, 64)],
    "i64_utf8": [("i64",), ("utf8", 8, 16)], "utf8_utf8": [("utf8", 1, 1), ("utf8", 8, 16)], "bool": [("bool",)],
}
ALL = [4, 1 << 10, 1 << 20, 1 << 25]
GROUPS = {"i64": ALL, "utf8_1": [4, 256], "utf8_8_16": ALL, "large_32_64": ALL, "i64_utf8": ALL, "utf8_utf8": ALL, "bool": [2]}
KERNELS = ["k_group_insert", "k_insert_keys", "k_group_count", "k_count_keys", "k_group_place", "k_place_keys", "k_group_combine",
           "k_len_block_sums", "k_var_scan_block_sums", "k_len_write_offsets", "k_copy_key_bytes"]


def key_column(torch, spec, gid, first):
    """(input DfdColumn, output DfdColumn, tensors to keep) of one key over group ids `gid`."""
    n = gid.numel()
    if spec[0] == "i64":
        v = gid * 0x9E3779B1 + 17
        out = torch.empty_like(v)
        return nv.DfdColumn(nv.COL_FIXED, 8, v.data_ptr(), None, None, 0, 0), nv.DfdColumn(nv.COL_FIXED, 8, out.data_ptr(), None, None, 0, 0), [v, out]
    if spec[0] == "bool":
        w = (2 ** torch.arange(8, device="cuda")).to(torch.int64)
        bits = ((gid & 1).view(-1, 8) * w).sum(dim=1).to(torch.uint8)
        out = torch.empty((n + 31) // 32 * 4, dtype=torch.uint8, device="cuda")
        return nv.DfdColumn(nv.COL_BOOL, 0, bits.data_ptr(), None, None, 0, 0), nv.DfdColumn(nv.COL_BOOL, 0, out.data_ptr(), None, None, 0, 0), [bits, out]
    kind, lo, hi = spec
    g = gid if not first else gid % 256  # a 1-byte first key holds the group id's low byte
    lens = lo + (g * 0x2545F491) % (hi - lo + 1)
    odt = torch.int64 if kind == "large" else torch.int32
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    total = int(offs[-1])
    data = torch.empty(total, dtype=torch.uint8, device="cuda")
    ch = 1 << 21
    for c0 in range(0, n, ch):  # byte j of a key: byte j of its group id for j < 8, then a filler of (group, j)
        c1 = min(n, c0 + ch)
        rows = torch.repeat_interleave(torch.arange(c1 - c0, device="cuda"), lens[c0:c1])
        j = torch.arange(rows.numel(), device="cuda") - (offs[c0:c1] - offs[c0])[rows]
        gg = g[c0:c1][rows]
        b = torch.where(j < 8, (gg >> (8 * j.clamp(max=7))) & 255, (gg * 31 + j * 7) & 255)
        data[int(offs[c0]):int(offs[c1])] = b.to(torch.uint8)
        del rows, j, gg, b
    offs = offs.to(odt)
    out_off = torch.empty(n + 1, dtype=odt, device="cuda")
    out_data = torch.empty(total, dtype=torch.uint8, device="cuda")
    k = nv.COL_LARGE_UTF8 if kind == "large" else nv.COL_UTF8
    return (nv.DfdColumn(k, 0, data.data_ptr(), offs.data_ptr(), None, 0, total),
            nv.DfdColumn(k, 0, out_data.data_ptr(), out_off.data_ptr(), None, 0, total), [data, offs, out_off, out_data])


def trace_kernels(torch, calls):
    """Run `calls` in one torch.profiler session -> per call, {kernel name: summed device ms}."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for call in calls:
            call()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = [e for e in json.load(open(path))["traceEvents"] if isinstance(e, dict) and e.get("cat") == "kernel"]
    events.sort(key=lambda e: e["ts"])
    per_call = []
    for e in events:
        name = next((k for k in KERNELS if k in e.get("name", "")), None)
        if name is None:
            continue
        if name in ("k_group_insert", "k_insert_keys"):
            per_call.append({})
        per_call[-1][name] = per_call[-1].get(name, 0.0) + e["dur"] / 1e3
    if len(per_call) != len(calls):
        raise SystemExit(f"expected {len(calls)} reduce calls in the trace, found {len(per_call)}")
    return per_call


def q1_step_us(torch, ctx, input_partitions, steps=50, warmup=5):
    from bench_workloads import cfg3_columns

    cols = cfg3_columns(0, input_partitions)
    n, N = len(cols[0]), 4
    ops = [-1, -1] + [nv.AGG_SUM_I128] * 4 + [nv.AGG_SUM_I64] * 4 + [nv.AGG_SUM_F64] * 2
    dcols = [dfd.DeviceColumn.from_arrow(ctx, a) for a in cols]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0, 1], N))
    pouts = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in dcols]
    red = dfd.PartialReduceExec(ctx, [0, 1], ops)
    routs = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in dcols]
    ex = dfd.ShuffleExchange(ctx, 0, 1, None)
    ex.setup_window(256 << 20)
    node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], N), uuid.uuid4(), 1, 1, 1)
    times, groups = [], 0
    for s in range(warmup + steps):
        t0 = time.perf_counter()
        part.partition(dcols, n, pouts)
        outs, out_starts = red.reduce(pouts, n, part.part_starts_device_ptr(), N, routs)
        node.shuffle_partitioned(ex, outs, out_starts)
        ctx.synchronize()
        if s >= warmup:
            times.append((time.perf_counter() - t0) * 1e6)
        groups = int(out_starts[-1])
    ex.close()
    return {"rows": n, "groups": groups, "partitions": N, "us_per_step": {"best": min(times), "median": float(np.median(times)), "worst": max(times)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rows", type=int, default=1 << 26)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures the GPU path only")
    name, power = DIP.gpu_info()
    n = args.rows
    assert n % 32 == 0
    ctx = dfd.WorkerContext(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    ones = torch.ones(n, dtype=torch.int64, device="cuda")
    cnt_out = torch.empty(n, dtype=torch.int64, device="cuda")
    results = {}
    for case, specs in CASES.items():
        results[case] = {}
        for G in GROUPS[case]:
            gname = f"2^{G.bit_length() - 1}" if G > 256 else str(G)
            gid = torch.randint(0, G, (n,), dtype=torch.int64, device="cuda", generator=g)
            built = [key_column(torch, s, gid, i == 0 and len(specs) > 1) for i, s in enumerate(specs)]
            del gid
            k = len(specs)
            ins = (nv.DfdColumn * (k + 1))(*[b[0] for b in built], nv.DfdColumn(nv.COL_FIXED, 8, ones.data_ptr(), None, None, 0, 0))
            outs = (nv.DfdColumn * (k + 1))(*[b[1] for b in built], nv.DfdColumn(nv.COL_FIXED, 8, cnt_out.data_ptr(), None, None, 0, 0))
            keys = (C.c_int32 * k)(*range(k))
            ops = (C.c_int32 * (k + 1))(*([-1] * k + [nv.AGG_SUM_I64]))
            out_starts = (C.c_int64 * 2)()
            torch.cuda.synchronize()

            def call():
                nv.check(nv.lib().dfd_partial_reduce_device(ctx.handle, ins, k + 1, n, keys, k, ops, starts.data_ptr(), 1, outs, out_starts, None))

            call()  # warm-up
            groups = int(out_starts[1])
            wall = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                call()
                wall.append((time.perf_counter() - t0) * 1e3)
            per_call = trace_kernels(torch, [call] * args.reps)
            names = sorted({kn for pc in per_call for kn in pc}, key=KERNELS.index)
            med = {kn: float(np.median([pc.get(kn, 0.0) for pc in per_call])) for kn in names}
            results[case][gname] = {"groups_out": groups, "kernel_ms": med, "device_ms": float(np.median([sum(pc.values()) for pc in per_call])),
                                    "wall_ms": float(np.median(wall))}
            print(case, gname, json.dumps(results[case][gname]), file=sys.stderr, flush=True)
            del built, ins, outs
            torch.cuda.empty_cache()
    q1 = {"cfg3_24_rows": q1_step_us(torch, ctx, 6), "cfg3_2^20_rows": q1_step_us(torch, ctx, 1 << 18)}
    ctx.close()
    line = {"profile": "reduce_keys", "gpu": name, "power_limit": power, "rows": n, "reps": args.reps, "state": "one COUNT (SUM_I64)",
            "unit": "kernel_ms / device_ms: median ms of device time per call from a torch.profiler trace; wall_ms: median host ms per synchronous call",
            "groups": GROUPS, "cases": results, "q1_world1_partition_reduce_shuffle": q1}
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
