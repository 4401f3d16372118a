"""k_group_combine's device time for every dfd_agg_op, on the GPU.

    python scripts/reduce_ops_profile.py [--out FILE] [--reps 3] [--rows 67108864] [--baseline-lib PATH]

One dfd_partial_reduce_device call per (op, group count): an Int64 key and one state column of the op's type, 2^26 rows in
one partition, with 1, 1 024, 2^20 and n/2 groups (uniform random group ids; one group is the CAS loops' worst case, as
every row then targets the same state).  State values: uniform random bits for the integer types, standard normals for
the floats, and for the 128-bit ops random Int64 values sign-extended, as Decimal128 columns of everyday magnitudes hold
(their high halves are all 0 or -1, so rows tie on the high half and the CAS decides: the slow path of MIN / MAX_I128).
After one warm-up call per shape, the --reps timed calls of every case run in one torch.profiler session, and the trace
gives each k_group_combine launch its device time.

--baseline-lib: a libdfd_b200.so built from another commit.  Then MIN_I64, MAX_I64 and SUM_I64, the ops a cfg of bench.py
uses, are also timed on it, alternating call by call with this tree's library in the same session, so a change of their
speed shows against the run-to-run spread.  Both libraries are driven through the same C ABI, each on a context of its own.

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
from datafusion_distributed_b200 import _native as nv  # noqa: E402

# op value -> its name without the AGG_ prefix; bytes of a state of each value kind
OPS = {getattr(nv, k): k[4:] for k in dir(nv) if k.startswith("AGG_")}
WIDTH = {"I64": 8, "F64": 8, "I128": 16, "I32": 4, "I16": 2, "I8": 1, "U64": 8, "U32": 4, "U16": 2, "U8": 1, "F32": 4, "F16": 2}
AB_OPS = [nv.AGG_MIN_I64, nv.AGG_MAX_I64, nv.AGG_SUM_I64]


def spread(v):
    return {"best": min(v), "median": float(np.median(v)), "worst": max(v)}


class Lib:
    """One build of the library: its handle and a context of its own."""

    def __init__(self, path):
        self.L = C.CDLL(path)
        for name, (res, args) in nv.SIGNATURES.items():
            fn = getattr(self.L, name)
            fn.restype, fn.argtypes = res, args
        self.h = C.c_void_p()
        self.check(self.L.dfd_ctx_create(0, C.byref(self.h)))

    def check(self, st):
        if st != nv.DFD_OK:
            raise SystemExit(f"{nv.STATUS.get(st, st)}: {self.L.dfd_last_error().decode()}")

    def reduce(self, key, state, key_out, state_out, op, n, starts):
        def col(t, w):
            return nv.DfdColumn(nv.COL_FIXED, w, t.data_ptr(), None, None, 0, 0)

        w = state.element_size() * (state.shape[1] if state.dim() == 2 else 1)
        ins, outs = (nv.DfdColumn * 2)(col(key, 8), col(state, w)), (nv.DfdColumn * 2)(col(key_out, 8), col(state_out, w))
        out_starts = (C.c_int64 * 2)()
        self.check(self.L.dfd_partial_reduce_device(self.h, ins, 2, n, (C.c_int32 * 1)(0), 1, (C.c_int32 * 2)(-1, op), starts.data_ptr(), 1,
                                                    outs, out_starts, None))

    def close(self):
        self.L.dfd_ctx_destroy(self.h)


def state_column(torch, kind, n, g):
    if kind in ("F64", "F32", "F16"):
        return torch.randn(n, dtype={"F64": torch.float64, "F32": torch.float32, "F16": torch.float16}[kind], device="cuda", generator=g)
    if kind == "I128":
        lo = torch.randint(-(2**63), 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
        return torch.stack([lo, lo >> 63], dim=1).contiguous()
    w = WIDTH[kind]
    dt = {8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.int8}[w]
    return torch.randint(-(2 ** (8 * w - 1)), 2 ** (8 * w - 1) - 1, (n,), dtype=dt, device="cuda", generator=g)


def combine_times(torch, prof_calls):
    """Run `prof_calls` (a list of thunks) in one torch.profiler session -> k_group_combine device time (ms) of each."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for call in prof_calls:
            call()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = [e for e in json.load(open(path))["traceEvents"] if isinstance(e, dict) and e.get("cat") == "kernel"
                  and "k_group_combine" in e.get("name", "")]
    events.sort(key=lambda e: e["ts"])
    if len(events) != len(prof_calls):
        raise SystemExit(f"expected {len(prof_calls)} k_group_combine launches in the trace, found {len(events)}")
    return [e["dur"] / 1e3 for e in events]


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
    libs = {"this": Lib(nv.LIB_PATH)}
    if args.baseline_lib:
        libs["baseline"] = Lib(args.baseline_lib)
    g = torch.Generator(device="cuda").manual_seed(1)
    starts = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    key_out = torch.empty(n, dtype=torch.int64, device="cuda")
    groups = {"1": 1, "1024": 1024, "2^20": 1 << 20, "n/2": n // 2}
    kinds = sorted({OPS[op].split("_", 1)[1] for op in OPS})
    per_op = {OPS[op]: {} for op in sorted(OPS)}
    ab = {OPS[op]: {} for op in AB_OPS} if args.baseline_lib else "not measured"
    for gname, G in groups.items():
        key = torch.randint(0, G, (n,), dtype=torch.int64, device="cuda", generator=g)
        for kind in kinds:
            state = state_column(torch, kind, n, g)
            state_out = torch.empty_like(state)
            torch.cuda.synchronize()
            ops = [op for op in sorted(OPS) if OPS[op].endswith("_" + kind)]
            calls, labels = [], []
            for op in ops:
                tags = ["this", "baseline"] if (op in AB_OPS and "baseline" in libs) else ["this"]
                for tag in tags:  # warm-up of every shape on every library that runs it
                    libs[tag].reduce(key, state, key_out, state_out, op, n, starts)
                for rep in range(args.reps):
                    for tag in (tags if rep % 2 == 0 else tags[::-1]):  # which build goes first alternates too
                        calls.append(lambda L=libs[tag], op=op: L.reduce(key, state, key_out, state_out, op, n, starts))
                        labels.append((op, tag))
            ms = combine_times(torch, calls)
            for op in ops:
                mine = [t for (o, tag), t in zip(labels, ms) if o == op and tag == "this"]
                per_op[OPS[op]][gname] = spread(mine)
                if op in AB_OPS and "baseline" in libs:
                    ab[OPS[op]][gname] = {"this": spread(mine), "baseline": spread([t for (o, tag), t in zip(labels, ms) if o == op and tag == "baseline"])}
            del state, state_out
        del key
        torch.cuda.empty_cache()
    for lib in libs.values():
        lib.close()
    line = {"profile": "reduce_ops", "gpu": name, "power_limit": power, "rows": n, "reps": args.reps, "kernel": "k_group_combine",
            "unit": "ms of device time per launch", "groups": groups, "combine_ms": per_op, "this_vs_baseline_ms": ab}
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
