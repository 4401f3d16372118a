"""GPU tests of the single-pass kernel's local write-out, which stores two consecutive output rows of a run at once where
a pair starts on an even output row: regions of an odd row count (so destinations start on both parities), sizes with
one-row and empty runs, 8-byte and narrower columns, and output columns whose base is not aligned to two values (every
row stored on its own).  Bar: bit-exact rows per destination, in order, and no write outside the destinations' rows."""
import numpy as np
import pytest
import torch

import datafusion_distributed_b200 as dfd
from oracle import oracle as orc
from tests.util import expected_partitions

pytestmark = pytest.mark.gpu

FILL = {torch.int64: -7, torch.int32: -7, torch.int16: -7, torch.uint8: 0xA5}


def table(kind: str, n: int):
    rng = np.random.Generator(np.random.PCG64(11))
    if kind == "i64":  # the Int64 fast key path, 8-byte ring
        return [rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64, endpoint=True),
                np.arange(n, dtype=np.int64) * 8 + 1, rng.integers(-(2**63), 2**63 - 1, n, dtype=np.int64, endpoint=True)]
    # Int32 key: generic key path, 4-byte ring moving 4-, 2- and 1-byte columns
    return [rng.integers(-(2**31), 2**31 - 1, n, dtype=np.int32, endpoint=True), np.arange(n, dtype=np.int32),
            rng.integers(-(2**15), 2**15 - 1, n, dtype=np.int16), rng.integers(0, 255, n, dtype=np.uint8)]


@pytest.mark.parametrize("kind", ["i64", "narrow"])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("n", [1, 2, 5, 37, 2561, 40_000])
@pytest.mark.parametrize("N", [3, 8, 17, 256])
def test_onepass_pairs_odd_regions(ctx, N, n, offset, kind):
    cols = table(kind, n)
    dest = orc.partition_ids([cols[0]], n, N)
    order, ref = expected_partitions(dest, N)
    rr = int(np.diff(ref).max()) | 1  # odd, and the fullest destination fills its region exactly when its count is odd
    ins = [torch.from_numpy(c).cuda() for c in cols]
    # output column base `offset` values past an allocation: offset 1 is not aligned to two values
    backing = [torch.full((N * rr + 2,), FILL[t.dtype], dtype=t.dtype, device="cuda") for t in ins]
    outs = [b[offset:offset + N * rr] for b in backing]
    part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
    _, starts, counts = part.partition_onepass([dfd.DeviceColumn.from_torch(t) for t in ins], n, rr,
                                               [dfd.DeviceColumn.from_torch(t) for t in outs])
    assert np.array_equal(counts, np.diff(ref))
    assert np.array_equal(starts, np.arange(N) * rr)
    written = np.zeros(N * rr + 2, dtype=bool)
    for p in range(N):
        written[offset + starts[p]:offset + starts[p] + counts[p]] = True
    for c, col in enumerate(cols):
        got = backing[c].cpu().numpy()
        for p in range(N):
            s = offset + int(starts[p])
            assert np.array_equal(got[s:s + counts[p]], col[order[ref[p]:ref[p + 1]]]), (p, c)
        assert np.all(got[~written] == np.asarray(FILL[ins[c].dtype]).astype(col.dtype)), c
