"""Multi-GPU check of dfd_shuffle_host with nullable, Boolean and string columns, run as one process per GPU:
  python -m torch.distributed.run --nnodes=1 --nproc-per-node T --master-addr 127.0.0.1 --master-port P tests/mgpu_host_shuffle_check.py
Every rank is producer task `rank` (its own mixed-schema host table, of a different length on every rank, one of them
empty) and consumer task `rank`; every output buffer is compared byte for byte with what the oracle's destinations imply:
chunk-major, partitions in order, producers in task order (tests/host_shuffle_util.py).  torch.distributed is only
plumbing (rendezvous + shipping the NCCL id)."""
import os
import sys
import traceback
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist

    import datafusion_distributed_b200 as dfd
    from oracle import oracle as orc
    from tests import host_shuffle_util as H

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    uid = [dfd.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx = dfd.WorkerContext(local_rank)
    ex = dfd.ShuffleExchange(ctx, rank, world, uid[0])
    ex.setup_window(64 << 20)
    rows = [0 if r == world - 1 else 30_011 + 7_919 * r for r in range(world)]
    failures = 0
    for P, n_chunks in ((3, 1), (3, 4), (16, 7)):
        N = P * world
        tables = [H.mixed_arrays(rows[r], 1000 * P + 10 * n_chunks + r) for r in range(world)]
        dests = [orc.partition_ids([t[0], t[1]], len(t[0]), N) if len(t[0]) else np.zeros(0, np.int64) for t in tables]
        sources = [[] for _ in tables[rank]]
        cps_want = np.zeros((n_chunks, P + 1), dtype=np.int64)
        at = 0
        for ch in range(n_chunks):
            for q in range(P):
                cps_want[ch, q] = at
                for r, t in enumerate(tables):  # producers in task order, each with the rows of ITS chunk `ch`
                    lo, hi = rows[r] * ch // n_chunks, rows[r] * (ch + 1) // n_chunks
                    idx = lo + np.nonzero(dests[r][lo:hi] == rank * P + q)[0]
                    at += len(idx)
                    for c, a in enumerate(t):
                        sources[c].append((a, idx))
            cps_want[ch, P] = at
        total = at
        nbytes = {c: sum(H.string_bytes(arr, idx) for arr, idx in sources[c]) for c, a in enumerate(tables[rank]) if H.is_var(a.type)}
        out = H.HostOut([a.type for a in tables[rank]], total, [True] * len(tables[rank]), nbytes)
        node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0, 1], P), uuid.uuid4(), 1, world, world)
        try:
            cps = node.shuffle_host(ex, H.in_columns(tables[rank], rows[rank]), rows[rank], n_chunks, out.cols, total)
            assert np.array_equal(cps, cps_want), (cps, cps_want)
            H.verify(out, sources, total)
        except Exception:  # noqa: BLE001
            failures += 1
            print(f"rank {rank}: MISMATCH shuffle_host P={P} n_chunks={n_chunks}\n{traceback.format_exc()}", flush=True)
        dist.barrier()
    f = torch.tensor([failures], device="cuda")
    dist.all_reduce(f)
    if rank == 0:
        print(("MGPU_HOST_SHUFFLE_OK" if f.item() == 0 else "MGPU_HOST_SHUFFLE_FAILED"), "world", world, "stats", ex.stats(), flush=True)
    ex.close()
    dist.destroy_process_group()
    sys.exit(0 if f.item() == 0 else 1)


if __name__ == "__main__":
    main()
