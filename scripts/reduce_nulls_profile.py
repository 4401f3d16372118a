"""PartialReduce device time per dfd_agg_op with nullable states, on the GPU.

    python scripts/reduce_nulls_profile.py [--out FILE] [--reps 3] [--rows 67108864] [--baseline-lib PATH]

The shapes of reduce_ops_profile.py (an Int64 key and one state column of the op's type, 2^26 rows in one partition, 1,
1 024, 2^20 and n/2 groups) along a null axis of the state column:
  none  no bitmap (k_group_combine, 4 launches)
  0     an input bitmap with every row valid (k_combine_nullable, and k_group_clear for MIN / MAX)
  0.5   half of the rows null, at random
  1.0   every row null (the states all end null)
Every call gets an output bitmap for the state exactly when its input has one.  After one warm-up call per case, the
--reps timed calls of every case run in one torch.profiler session, and the trace gives each call's combine launch
(k_group_combine or k_combine_nullable) and, for a nullable MIN / MAX, its k_group_clear launch their device time.

--baseline-lib: a libdfd_b200.so built from another commit.  Then every op's "none" case also runs on it, alternating
call by call with this tree's library in the same session, so a change of the non-null speed shows against the
run-to-run spread.

Prints one JSON line (GPU name and power limit included) and writes it to --out when given.  Fails without a GPU."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import device_input_profile as DIP  # noqa: E402
import reduce_ops_profile as ROP  # noqa: E402
from datafusion_distributed_b200 import _native as nv  # noqa: E402

AXES = ["none", "0", "0.5", "1.0"]
COMBINE = ("k_group_combine", "k_combine_nullable")


def reduce(lib, key, state, key_out, state_out, op, n, starts, in_valid=None, out_valid=None):
    def col(t, w, v):
        return nv.DfdColumn(nv.COL_FIXED, w, t.data_ptr(), None, v.data_ptr() if v is not None else None, 0, 0)

    w = state.element_size() * (state.shape[1] if state.dim() == 2 else 1)
    ins = (nv.DfdColumn * 2)(col(key, 8, None), col(state, w, in_valid))
    outs = (nv.DfdColumn * 2)(col(key_out, 8, None), col(state_out, w, out_valid))
    out_starts = (C.c_int64 * 2)()
    lib.check(lib.L.dfd_partial_reduce_device(lib.h, ins, 2, n, (C.c_int32 * 1)(0), 1, (C.c_int32 * 2)(-1, op), starts.data_ptr(), 1,
                                              outs, out_starts, None))


def trace_times(torch, calls, clears):
    """Run `calls` in one torch.profiler session -> (combine ms, k_group_clear ms or None) of each; clears[i] says whether
    call i launches k_group_clear."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for call in calls:
            call()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = [e for e in json.load(open(path))["traceEvents"] if isinstance(e, dict) and e.get("cat") == "kernel"]
    comb = sorted((e for e in events if any(k in e.get("name", "") for k in COMBINE)), key=lambda e: e["ts"])
    clr = sorted((e for e in events if "k_group_clear" in e.get("name", "")), key=lambda e: e["ts"])
    if len(comb) != len(calls) or len(clr) != sum(clears):
        raise SystemExit(f"expected {len(calls)} combine and {sum(clears)} clear launches in the trace, found {len(comb)} and {len(clr)}")
    it = iter(clr)
    return [(c["dur"] / 1e3, next(it)["dur"] / 1e3 if k else None) for c, k in zip(comb, clears)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rows", type=int, default=1 << 26)
    ap.add_argument("--baseline-lib", default="")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures the GPU path only")
    name, power = DIP.gpu_info()
    n = args.rows
    assert n % 32 == 0
    libs = {"this": ROP.Lib(nv.LIB_PATH)}
    if args.baseline_lib:
        libs["baseline"] = ROP.Lib(args.baseline_lib)
    g = torch.Generator(device="cuda").manual_seed(1)
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    key_out = torch.empty(n, dtype=torch.int64, device="cuda")
    out_valid = torch.empty(n // 8, dtype=torch.uint8, device="cuda")
    weights = (2 ** torch.arange(8, device="cuda")).to(torch.int32)
    bitmaps = {}
    for ax in AXES[1:]:
        valid = (torch.rand(n, device="cuda", generator=g) >= float(ax)).view(-1, 8).to(torch.int32)
        bitmaps[ax] = (valid * weights).sum(dim=1).to(torch.uint8)
        del valid
    groups = {"1": 1, "1024": 1024, "2^20": 1 << 20, "n/2": n // 2}
    kinds = sorted({ROP.OPS[op].split("_", 1)[1] for op in ROP.OPS})
    combine = {ROP.OPS[op]: {ax: {} for ax in AXES} for op in sorted(ROP.OPS)}
    clear = {ROP.OPS[op]: {ax: {} for ax in AXES[1:]} for op in sorted(ROP.OPS) if not ROP.OPS[op].startswith("SUM")}
    ab = {ROP.OPS[op]: {} for op in sorted(ROP.OPS)} if args.baseline_lib else "not measured"
    for gname, G in groups.items():
        key = torch.randint(0, G, (n,), dtype=torch.int64, device="cuda", generator=g)
        for kind in kinds:
            state = ROP.state_column(torch, kind, n, g)
            state_out = torch.empty_like(state)
            torch.cuda.synchronize()
            ops = [op for op in sorted(ROP.OPS) if ROP.OPS[op].endswith("_" + kind)]
            calls, clears, labels = [], [], []
            for op in ops:
                minmax = not ROP.OPS[op].startswith("SUM")
                for ax in AXES:
                    iv = bitmaps.get(ax)
                    ov = out_valid if iv is not None else None
                    tags = ["this", "baseline"] if (ax == "none" and "baseline" in libs) else ["this"]
                    for tag in tags:  # warm-up of every case on every library that runs it
                        reduce(libs[tag], key, state, key_out, state_out, op, n, starts, iv, ov)
                    for rep in range(args.reps):
                        for tag in (tags if rep % 2 == 0 else tags[::-1]):  # which build goes first alternates too
                            calls.append(lambda L=libs[tag], op=op, iv=iv, ov=ov: reduce(L, key, state, key_out, state_out, op, n, starts, iv, ov))
                            clears.append(minmax and iv is not None)
                            labels.append((op, ax, tag))
            ms = trace_times(torch, calls, clears)
            for op in ops:
                for ax in AXES:
                    mine = [t for (o, a, tag), t in zip(labels, ms) if o == op and a == ax and tag == "this"]
                    combine[ROP.OPS[op]][ax][gname] = ROP.spread([t[0] for t in mine])
                    if mine[0][1] is not None:
                        clear[ROP.OPS[op]][ax][gname] = ROP.spread([t[1] for t in mine])
                if "baseline" in libs:
                    base = [t[0] for (o, a, tag), t in zip(labels, ms) if o == op and a == "none" and tag == "baseline"]
                    ab[ROP.OPS[op]][gname] = {"this": combine[ROP.OPS[op]]["none"][gname], "baseline": ROP.spread(base)}
            del state, state_out
        del key
        torch.cuda.empty_cache()
    for lib in libs.values():
        lib.close()
    line = {"profile": "reduce_nulls", "gpu": name, "power_limit": power, "rows": n, "reps": args.reps,
            "unit": "ms of device time per launch", "groups": groups, "null_axis": AXES,
            "combine_ms": combine, "clear_ms": clear, "this_vs_baseline_combine_ms_no_bitmap": ab}
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
