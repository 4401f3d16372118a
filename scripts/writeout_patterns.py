#!/usr/bin/env python
"""Store patterns for the write side of the cfg-2 single-pass scatter (2^26 rows x 8 Int64, 8 destinations), next to the
card's device-to-device copy rate.  Only the stores differ between the patterns (scripts/writeout_patterns.cu):

  a        torch copy_ of the same 4 GiB: the ceiling
  b        8-byte lanes, runs at their own row alignment (what k_scatter_onepass does)
  c        8-byte lanes, warps aligned to 256 B (virtual runs, as DFD_ALIGNED_WRITEOUT=1)
  d        16-byte pairs on even output rows; odd head / tail rows of a run are one 8-byte store each
  e        d with warps aligned to 512 B
  b_wb/d_wb  b and d with default-policy stores instead of st.global.cs

Runs are per (2560-row tile, destination, column); their lengths are a seeded multinomial(2560, 1/8 each) per tile and
their output rows exact prefixes in regions of default_region_rows rows.  Every pattern is checked to write what b
writes, then timed with CUDA events over --reps launches after warm-up, at each resident-CTA count of --ctas-per-sm
(persistent grid of that many 256-thread CTAs per SM; the single-pass kernel runs 2 consumer CTAs per SM today).

  python scripts/writeout_patterns.py            # one JSON line
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "scripts", "writeout_patterns.cu")
PATTERNS = {"b": (0, 1), "c": (1, 1), "d": (2, 1), "e": (3, 1), "b_wb": (0, 0), "d_wb": (2, 0)}  # (PAT, cs)
T, D, COLS = 2560, 8, 8


def build(out_dir: str) -> str:
    lib = os.path.join(out_dir, "libwriteout_patterns.so")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.check_call([nvcc, "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-o", lib, SRC])
    return lib


def region_rows(n_rows: int, slack: float = 0.25) -> int:  # HashPartitioner.default_region_rows
    fair = -(-max(n_rows, 1) // D)
    return (int(fair * (1.0 + slack)) + 32 + 31) // 32 * 32


def runs(np, n_rows: int, seed: int):
    """(cnt, orow) [n_tiles][D] uint32: seeded multinomial run lengths per tile and each run's first output row."""
    n_tiles = -(-n_rows // T)
    rows = np.full(n_tiles, T, dtype=np.int64)
    rows[-1] = n_rows - (n_tiles - 1) * T
    rng = np.random.default_rng(seed)
    cnt = np.stack([rng.multinomial(r, [1.0 / D] * D) for r in rows]).astype(np.int64)
    rr = region_rows(n_rows)
    prefix = np.cumsum(cnt, axis=0) - cnt  # exclusive over the lower tiles
    assert int((prefix[-1] + cnt[-1]).max()) <= rr
    orow = prefix + np.arange(D, dtype=np.int64)[None, :] * rr
    assert int(orow.max()) + T < 2**32
    return cnt.astype(np.uint32), orow.astype(np.uint32), rr


def smi(query: str):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001 — identity only
        return None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 26)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3, help="timed windows per pattern, interleaved; the median is reported")
    ap.add_argument("--ctas-per-sm", default="2,3")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--lib", default=None, help="a built libwriteout_patterns.so (default: build one in a temporary directory)")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("writeout_patterns: no CUDA device")
    tmp = tempfile.TemporaryDirectory()
    lib = C.CDLL(args.lib or build(tmp.name))
    lib.writeout_launch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_longlong,
                                    C.c_int, C.c_int, C.c_void_p]
    lib.writeout_occupancy.argtypes = [C.c_int, C.POINTER(C.c_int)]

    n = args.rows
    cnt_h, orow_h, rr = runs(np, n, args.seed)
    n_tiles = cnt_h.shape[0]
    dev = torch.device("cuda", 0)
    cnt = torch.from_numpy(cnt_h.reshape(-1).copy()).to(dev)
    orow = torch.from_numpy(orow_h.reshape(-1).copy()).to(dev)
    rid = torch.arange(n, dtype=torch.int64, device=dev)
    ins = [rid * 8 + j for j in range(COLS)]
    del rid
    outs = [torch.zeros(D * rr, dtype=torch.int64, device=dev) for _ in range(COLS)]
    in_p = (C.c_void_p * COLS)(*[t.data_ptr() for t in ins])
    out_p = (C.c_void_p * COLS)(*[t.data_ptr() for t in outs])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.current_stream().cuda_stream

    def launch(name: str, per_sm: int) -> None:
        pat, cs = PATTERNS[name]
        rc = lib.writeout_launch(pat, cs, in_p, out_p, COLS, cnt.data_ptr(), orow.data_ptr(), n, n_tiles, per_sm * sms, stream)
        if rc:
            raise RuntimeError(f"writeout_launch({name}): CUDA error {rc}")

    ctas = [int(x) for x in args.ctas_per_sm.split(",")]
    for name, (pat, _) in PATTERNS.items():
        occ = C.c_int(0)
        if lib.writeout_occupancy(pat, C.byref(occ)) or occ.value < max(ctas):
            raise SystemExit(f"pattern {name}: only {occ.value} CTAs per SM fit")

    # every pattern writes what b writes (the rows between the runs stay zero)
    launch("b", ctas[0])
    ref = [t.clone() for t in outs]
    parity = {}
    for name in PATTERNS:
        for t in outs:
            t.zero_()
        launch(name, ctas[0])
        parity[name] = all(torch.equal(a, b) for a, b in zip(outs, ref))
    del ref
    if not all(parity.values()):
        raise SystemExit(f"writeout_patterns: outputs differ from pattern b: {parity}")

    bytes_moved = 2 * 8 * COLS * n
    clocks = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0", "-lms", "200"],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    ms = {f"{name}@{k}": [] for k in ctas for name in PATTERNS}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    try:
        for _ in range(args.rounds):
            for key in ms:
                name, k = key.split("@")
                for _ in range(3):
                    launch(name, int(k))
                a.record()
                for _ in range(args.reps):
                    launch(name, int(k))
                b.record()
                b.synchronize()
                ms[key].append(a.elapsed_time(b) / args.reps)
    finally:
        clocks.terminate()
        sm_clk = [int(x) for x in clocks.communicate(timeout=30)[0].split() if x.strip().isdigit()]
    del outs, ins
    torch.cuda.empty_cache()

    src = torch.ones(COLS * n, dtype=torch.int64, device=dev)  # 4 GiB read + 4 GiB written, as the patterns
    dst = torch.empty_like(src)
    copy_ms = []
    for _ in range(args.rounds):
        for _ in range(3):
            dst.copy_(src)
        a.record()
        for _ in range(args.reps):
            dst.copy_(src)
        b.record()
        b.synchronize()
        copy_ms.append(a.elapsed_time(b) / args.reps)

    def rec(v):
        m = float(np.median(v))
        return {"ms": round(m, 4), "TBps": round(bytes_moved / (m / 1e3) / 1e12, 3), "ms_all": [round(x, 4) for x in v]}

    out = {
        "rows": n, "region_rows": rr, "tiles": n_tiles, "reps": args.reps, "rounds": args.rounds, "seed": args.seed,
        "bytes_per_launch": bytes_moved,
        "a_copy": rec(copy_ms),
        "patterns": {k: rec(v) for k, v in ms.items()},
        "device": torch.cuda.get_device_name(0),
        "power_limit_w": smi("power.limit"),
        "sm_clock_mhz_median": float(np.median(sm_clk)) if sm_clk else None,
        "sm_clock_mhz_max": smi("clocks.max.sm"),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
