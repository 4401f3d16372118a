#!/usr/bin/env python
"""Where the single-pass kernel's time goes: per-phase clock64() shares of k_scatter_onepass at the cfg-2 shape
(2^26 rows x 8 Int64, Hash([col0], 8), the bench.py workload), next to the card's achievable copy rate.

Builds (unless it exists) a tagged library with -DDFD_ONEPASS_CLOCKS plus the given geometry defines, runs the partition
a few times and prints one JSON line.  The default library is not touched and has no clocks.

  python scripts/onepass_clocks.py --tag clk --defs "-DDFD_ONEPASS_SPLIT=4 -DDFD_ONEPASS_NB=8"

Cycles are summed over all CTAs as seen by consumer thread 0 and by the producer's lane 0 (every CTA is persistent, so
each total is the CTA's whole life); a share is a phase's sum over the matching total.  Copy rate: a 4 GiB device-to-device
torch copy_ timed with CUDA events — the same 128 B per cfg-2 row of HBM traffic the kernel needs."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["wait_header", "wait_keycol", "wait_col", "phase1", "lookback", "scatter", "producer_wait_empty",
          "consumer_total", "producer_total", "tiles"]  # OnePassClock order (csrc/dfd_kernels.cuh)


def copy_rate(torch, reps: int = 10) -> dict:
    n = 1 << 29  # 4 GiB of int64 read + 4 GiB written = 128 B per cfg-2 row
    src = torch.ones(n, dtype=torch.int64, device="cuda")
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dst.copy_(src)
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / reps
    del src, dst
    return {"bytes": 2 * 8 * n, "ms": ms, "GBps": 2 * 8 * n / (ms / 1e3) / 1e9}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tag", default="clk")
    ap.add_argument("--defs", default="", help="extra -D options for the single-pass sources (geometry)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rows", type=int, default=1 << 26)
    ap.add_argument("--no-copy", action="store_true")
    args = ap.parse_args()

    env = dict(os.environ, DFD_LIB_TAG=args.tag, DFD_NVCC_DEFS_ONEPASS=f"-DDFD_ONEPASS_CLOCKS {args.defs}".strip())
    lib_path = os.path.join(ROOT, "datafusion_distributed_b200", "_lib", f"libdfd_b200_{args.tag}.so")
    if not os.path.exists(lib_path):
        subprocess.check_call([sys.executable, os.path.join(ROOT, "datafusion_distributed_b200", "build.py")], env=env)
    os.environ["DFD_LIB_TAG"] = args.tag
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import datafusion_distributed_b200 as dfd
    from datafusion_distributed_b200 import _native as nv

    lib = nv.lib()
    if not hasattr(lib, "dfd_onepass_clocks"):
        raise SystemExit(f"{nv.LIB_PATH} was not built with -DDFD_ONEPASS_CLOCKS")
    lib.dfd_onepass_clocks.argtypes = [C.c_void_p, C.c_int]
    clk = np.zeros(len(PHASES) + 6, dtype=np.uint64)  # (room beyond CLK_COUNT)

    def read(reset: bool) -> np.ndarray:
        rc = lib.dfd_onepass_clocks(clk.ctypes.data, 1 if reset else 0)
        if rc:
            raise RuntimeError(f"dfd_onepass_clocks: CUDA error {rc}")
        return clk[:len(PHASES)].astype(np.float64)

    torch.cuda.set_device(0)
    n = args.rows
    g = torch.Generator(device="cuda").manual_seed(42)
    key = torch.randint(-(2**63), 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    rid = torch.arange(n, dtype=torch.int64, device="cuda")
    ins = [key] + [rid * 8 + j for j in range(1, 8)]
    del rid
    ctx = dfd.WorkerContext(0)
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], 8))
    region_rows = part.default_region_rows(n)
    outs = [torch.empty(8 * region_rows, dtype=torch.int64, device="cuda") for _ in ins]
    in_cols = [dfd.DeviceColumn.from_torch(t) for t in ins]
    out_cols = [dfd.DeviceColumn.from_torch(t) for t in outs]
    for _ in range(3):
        part.partition_onepass(in_cols, n, region_rows, out_cols, sync=False)
    ctx.synchronize()
    read(True)
    ctx.reset_metrics()
    ctx.set_profiling(True)
    for _ in range(args.steps):
        part.partition_onepass(in_cols, n, region_rows, out_cols, sync=False)
    ctx.synchronize()
    m = ctx.metrics()
    v = dict(zip(PHASES, read(True)))
    ct, pt = v["consumer_total"], v["producer_total"]
    shares = {k: v[k] / ct for k in ("wait_header", "wait_keycol", "wait_col", "phase1", "lookback", "scatter")}
    shares["scatter_issue"] = (v["scatter"] - v["wait_keycol"] - v["wait_col"]) / ct
    shares["producer_wait_empty"] = v["producer_wait_empty"] / pt
    n_payload_items = 8  # columns of the cfg-2 table; column 0 is the key
    out = {
        "tag": args.tag, "defs": args.defs, "rows": n, "steps": args.steps,
        "kernel_ms": m["scatter_ms"] / max(m["scatter_launches"], 1),
        "consumer_share": shares,
        "cycles_per_tile": {k: v[k] / max(v["tiles"], 1) for k in PHASES if k != "tiles"},
        "wait_per_column_keycol_vs_other": [v["wait_keycol"] / max(v["tiles"], 1),
                                          v["wait_col"] / max(v["tiles"], 1) / (n_payload_items - 1)],
        "tiles": v["tiles"] / args.steps,
        "device": torch.cuda.get_device_name(0),
    }
    try:
        out["power_limit_w"] = float(subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                                     capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001 — identity only
        out["power_limit_w"] = None
    if not args.no_copy:
        del outs, out_cols, ins, in_cols
        torch.cuda.empty_cache()
        out["copy_rate"] = copy_rate(torch)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
