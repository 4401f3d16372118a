"""What the partition entry points count and time: the exact dfd_metrics deltas (kernel and scatter launches, calls, rows,
bytes) of a two-pass partition, a single-pass partition with follow-up launches and a world-1 single-pass shuffle, and the
profiling event rings behind dfd_metrics hist/scan/scatter_ms and dfd_exchange_phase_ms, driven past their 64 calls so
they are summed when full as well as when read."""
import ctypes as C
import uuid

import numpy as np
import pytest

import datafusion_distributed_b200 as dfd
from datafusion_distributed_b200 import _native as nv
from tests.test_instantiations_gpu import column, mixed_fixed
from tests.test_onepass_gpu import dev_cols

pytestmark = pytest.mark.gpu

N = 8  # destinations (world 1: partitions per task)
ROWS = 100_003
COUNTERS = ("kernel_launches", "scatter_launches", "calls", "rows", "bytes_in")
RING_CALLS = 70  # > the 64 calls an event ring holds


@pytest.fixture(scope="module")
def wctx(built):
    """A context of its own: its counters and profiling mode are not shared with other modules."""
    c = dfd.WorkerContext(0)
    yield c
    c.close()


def two_pass_table(rng, n):
    """Widths 8 (the Int64 key), 4 (nullable: a validity bitmap too) and 16."""
    return [column(rng, "i64", n), column(rng, "i32", n, nulls=True), column(rng, "dec128", n)]


def exchange_table(rng, n):
    return [column(rng, "i64", n), column(rng, "i32", n), column(rng, "dec128", n)]


class Partitions:
    """Device inputs and preallocated outputs of the three calls, so repeated calls allocate nothing."""

    def __init__(self, ctx, n, seed):
        rng = np.random.Generator(np.random.PCG64(seed))
        self.ctx, self.n = ctx, n
        self.two_pass_in = dev_cols(ctx, two_pass_table(rng, n))
        self.two_pass_out = [dfd.DeviceColumn.empty_like(ctx, c, n) for c in self.two_pass_in]
        self.two_pass_part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        self.onepass_in = dev_cols(ctx, mixed_fixed(rng, n, [column(rng, "i64", n)]))
        self.onepass_out = [dfd.DeviceColumn.empty_like(ctx, c, N * n) for c in self.onepass_in]  # regions of n rows: never overflow
        self.onepass_part = dfd.HashPartitioner(ctx, dfd.Partitioning.Hash([0], N))
        self.exchange_in = dev_cols(ctx, exchange_table(rng, n))
        self.ex = dfd.ShuffleExchange(ctx, 0, 1, None)
        self.ex.setup_window(int(28 * N * (n + 64) * 1.1) + (1 << 20))  # every sub-window holds every row
        self.node = dfd.NetworkShuffleExec.try_new(dfd.Partitioning.Hash([0], N), uuid.uuid4(), 1, 1, 1)

    def two_pass(self):
        self.two_pass_part.partition(self.two_pass_in, self.n, self.two_pass_out)

    def onepass(self):
        _, _, counts = self.onepass_part.partition_onepass(self.onepass_in, self.n, self.n, self.onepass_out)
        assert counts.sum() == self.n

    def shuffle(self):
        self.node.shuffle_onepass(self.ex, self.exchange_in, self.n)
        _, _, counts = self.node.collect(self.ex)
        assert counts.sum() == self.n
        assert nv.lib().dfd_exchange_onepass_fallbacks(self.ex._h) == 0

    def phase_ms(self):
        out3, n = (C.c_double * 3)(), C.c_uint64()
        nv.check(nv.lib().dfd_exchange_phase_ms(self.ex._h, out3, C.byref(n)))
        return list(out3), n.value

    def close(self):
        self.ex.close()


@pytest.fixture(scope="module")
def calls(wctx):
    p = Partitions(wctx, ROWS, 2024)
    yield p
    p.close()


def deltas(ctx, fn):
    before = ctx.metrics()
    fn()
    after = ctx.metrics()
    return {k: after[k] - before[k] for k in COUNTERS}


def test_two_pass_partition_counts_one_launch_per_width_group(wctx, calls):
    """K1 + K1b, then one k_scatter per width group: 8, 4, 16 and the validity bitmap."""
    n = ROWS
    assert deltas(wctx, calls.two_pass) == {"kernel_launches": 6, "scatter_launches": 4, "calls": 1, "rows": n,
                                            "bytes_in": 8 * n + 4 * n + (n + 7) // 8 + 16 * n}


def test_onepass_partition_counts_the_single_pass_launch_and_its_follow_ups(wctx, calls):
    """30 fixed-width columns (98 bytes a row): one k_scatter_onepass moves the first 24, follow-up launches the widths
    8, 4, 16, 2 and 1 (two columns) of the last six.  No K1 / K1b."""
    n = ROWS
    assert deltas(wctx, calls.onepass) == {"kernel_launches": 6, "scatter_launches": 6, "calls": 1, "rows": n, "bytes_in": 98 * n}


def test_world1_onepass_shuffle_counts_the_scatter_and_the_flag_kernels(wctx, calls):
    """One single-pass peer launch for the three columns, plus k_xchg_signal_ready and k_xchg_publish_wait."""
    n = ROWS
    assert deltas(wctx, calls.shuffle) == {"kernel_launches": 3, "scatter_launches": 1, "calls": 1, "rows": n, "bytes_in": 28 * n}


def test_profiling_event_rings_sum_every_call_when_full_and_when_read(wctx):
    p = Partitions(wctx, 20_000, 7)
    try:
        wctx.reset_metrics()
        p.phase_ms()  # (clears the exchange's sums)
        wctx.set_profiling(True)
        try:
            for _ in range(RING_CALLS):
                p.two_pass()
                p.onepass()
                p.shuffle()
        finally:
            wctx.set_profiling(False)
        m = wctx.metrics()
        assert m["calls"] == 3 * RING_CALLS
        assert m["hist_ms"] >= 0 and m["scan_ms"] >= 0 and m["scatter_ms"] > 0, m
        means, n_shuffles = p.phase_ms()
        assert n_shuffles == RING_CALLS
        assert min(means) >= 0 and means[1] > 0, means
        assert p.phase_ms() == ([0.0, 0.0, 0.0], 0)  # read once, then reset
        wctx.reset_metrics()
        m = wctx.metrics()
        assert m["calls"] == 0 and m["hist_ms"] == 0 and m["scan_ms"] == 0 and m["scatter_ms"] == 0
    finally:
        p.close()
