"""Host mirror of the consumer half: Stage / DistributedTaskContext /
NetworkShuffleExec over the NVLink exchange.

Reference surface being mirrored:
  Stage, ExecutionTask, DistributedTaskContext      src/stage.rs:71-106
  NetworkShuffleExec::try_new / execute             src/execution_plans/network_shuffle.rs:115-157, 213-238
The data plane (gRPC + Arrow Flight in the reference) is `dfd_shuffle_device`:
one worker per GPU, NCCL send/recv or fused peer stores over NVLink.
"""
from __future__ import annotations

import ctypes as C
import uuid
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import _native as nv
from .device import DeviceColumn, WorkerContext, columns_to_c
from .partitioner import HashPartitioner, Partitioning, scale_partitioning


@dataclass
class ExecutionTask:
    """src/stage.rs:85-89 — here the "url" of a worker is its rank on the NVSwitch box."""
    url: Optional[int] = None


@dataclass
class Stage:
    """src/stage.rs:71-82"""
    query_id: uuid.UUID
    num: int
    plan: Optional[Partitioning]
    tasks: List[ExecutionTask] = field(default_factory=list)


@dataclass(frozen=True)
class DistributedTaskContext:
    """src/stage.rs:92-106 — which shard of the stage this worker is."""
    task_index: int = 0
    task_count: int = 1


def exchange_plan(counts: np.ndarray, partitions_per_task: int, rank: int):
    """`dfd_exchange_plan` (pure host arithmetic): counts[T][N] -> dict of offset arrays."""
    counts = np.ascontiguousarray(counts, dtype=np.int64)
    T, N = counts.shape
    P = partitions_per_task
    send_start = np.zeros(N, np.int64)
    recv_start = np.zeros(P * T, np.int64)
    part_starts = np.zeros(P + 1, np.int64)
    dest_base = np.zeros(N, np.int64)
    recv_rows = C.c_int64()
    nv.check(nv.lib().dfd_exchange_plan(T, P, rank, counts.ctypes.data, send_start.ctypes.data, recv_start.ctypes.data,
                                        part_starts.ctypes.data, dest_base.ctypes.data, C.byref(recv_rows)))
    return {"send_start": send_start, "recv_start": recv_start.reshape(P, T), "part_starts": part_starts,
            "dest_base": dest_base, "recv_rows": recv_rows.value}


def nccl_unique_id() -> bytes:
    buf = (C.c_char * 128)()
    nv.check(nv.lib().dfd_nccl_unique_id(buf))
    return bytes(buf)


def _nullable_outs(in_cols: Sequence[DeviceColumn], nullable: Optional[Sequence[bool]]):
    """Output descriptors that carry the schema's nullable flag of every column (`nullable[i]`; default: the columns of
    this worker that have a validity bitmap), as the segment exchanges expect them on entry."""
    c_out = (nv.DfdColumn * len(in_cols))()
    for i, c in enumerate(in_cols):
        if (nullable[i] if nullable is not None else bool(c.validity)):
            c_out[i].validity = 1  # (flag only: the library replaces it with the bitmap's address)
    return c_out


def _window_columns(c_out, types, exchange: "ShuffleExchange", length: int = 0) -> List[DeviceColumn]:
    """DeviceColumns over the buffers the library set in `c_out` (they live in `exchange`'s receive window)."""
    return [DeviceColumn(c.kind, c.width, c.values or 0, c.offsets or 0, c.validity or 0, 0, length, exchange, t) for c, t in zip(c_out, types)]


class ShuffleExchange:
    """One worker's endpoint of the exchange (≙ WorkerConnectionPool + the worker's
    ExecuteTask server, src/worker/worker_connection_pool.rs:60-113)."""

    def __init__(self, ctx: WorkerContext, rank: int, world: int, unique_id: Optional[bytes]):
        self.ctx, self.rank, self.world = ctx, rank, world
        self._h = C.c_void_p()
        uid = (C.c_char * 128).from_buffer_copy(unique_id) if unique_id is not None else None
        nv.check(nv.lib().dfd_exchange_create(ctx.handle, rank, world, uid, C.byref(self._h)))
        ctx._adopt(self)

    def setup_window(self, nbytes: int):
        nv.check(nv.lib().dfd_exchange_setup_window(self._h, nbytes))

    def stats(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        nv.check(nv.lib().dfd_exchange_stats(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return {"bytes_sent": a.value, "bytes_received": b.value, "shuffles": c.value}

    def close(self):
        if self._h and self.ctx.handle:
            nv.lib().dfd_exchange_destroy(self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class NetworkShuffleExec:
    """Consumer side of the shuffle for device-resident columns.

    `try_new(input_partitioning=Hash(keys, P), ..., task_count, input_task_count)` rescales the
    producer's RepartitionExec to Hash(keys, P * task_count) (network_shuffle.rs:126-134) while
    this node keeps advertising Hash(keys, P) (properties cloned before scaling, :155).
    """

    def __init__(self, properties: Partitioning, input_stage: Stage, task_count: int):
        self.properties = properties
        self.input_stage = input_stage
        self.task_count = task_count
        self._part: Optional[HashPartitioner] = None
        self._out: Optional[List[DeviceColumn]] = None
        self._starts: Optional[np.ndarray] = None

    @staticmethod
    def try_new(input_partitioning: Partitioning, query_id: uuid.UUID, num: int, task_count: int,
                input_task_count: int) -> "NetworkShuffleExec":
        if not input_partitioning.key_cols:
            raise ValueError("NetworkShuffleExec input must be hash partitioned")
        scaled = scale_partitioning(input_partitioning, lambda p: p * task_count)
        stage = Stage(query_id, num, scaled, [ExecutionTask(None) for _ in range(input_task_count)])
        return NetworkShuffleExec(input_partitioning, stage, task_count)

    def name(self) -> str:
        return "NetworkShuffleExec"

    def output_partitioning(self) -> Partitioning:
        return self.properties

    def input_stage_plan(self) -> Partitioning:
        return self.input_stage.plan

    # -- data plane --------------------------------------------------------------
    def _partitioner(self, exchange: ShuffleExchange):
        """Handle of the producers' Hash(keys, P x task_count) partitioner, created on first use."""
        if self._part is None:
            self._part = HashPartitioner(exchange.ctx, self.input_stage.plan)
        return self._part._h

    def shuffle(self, exchange: ShuffleExchange, in_cols: Sequence[DeviceColumn], n_rows: int, mode: int = nv.EXCHANGE_FUSED,
                out_cols: Optional[List[DeviceColumn]] = None, out_capacity_rows: int = 0):
        """Run the collective for this worker: as producer task `rank` it contributes `in_cols`,
        as consumer task `rank` it receives its P partitions."""
        if len(self.input_stage.tasks) != exchange.world or self.task_count != exchange.world:
            raise ValueError("this exchange runs one producer and one consumer task per GPU worker")
        P = self.properties.partition_count
        c_in = columns_to_c(in_cols)
        if mode == nv.EXCHANGE_NCCL:
            if out_cols is None:
                raise ValueError("NCCL mode needs caller-provided output columns")
            c_out = columns_to_c(out_cols)
        else:
            c_out = (nv.DfdColumn * len(in_cols))()
        starts = (C.c_int64 * (P + 1))()
        nv.check(nv.lib().dfd_shuffle_device(exchange._h, self._partitioner(exchange), mode, c_in, len(in_cols), n_rows, P, c_out,
                                             out_capacity_rows, starts))
        if mode == nv.EXCHANGE_FUSED:
            out_cols = _window_columns(c_out, [c.arrow_type for c in in_cols], exchange, int(starts[P]))
        self._out = list(out_cols)
        self._starts = np.frombuffer(starts, dtype=np.int64).copy()
        return self._out, self._starts

    def shuffle_async(self, exchange: ShuffleExchange, in_cols: Sequence[DeviceColumn], n_rows: int):
        """Fused shuffle enqueued on the worker's stream without a host sync (`dfd_shuffle_device_async`)."""
        P = self.properties.partition_count
        c_out = (nv.DfdColumn * len(in_cols))()
        nv.check(nv.lib().dfd_shuffle_device_async(exchange._h, self._partitioner(exchange), columns_to_c(in_cols), len(in_cols), n_rows, P, c_out))
        self._pending = (c_out, [c.arrow_type for c in in_cols], exchange)

    def wait(self, exchange: ShuffleExchange):
        """Complete the last `shuffle_async`: returns (out columns, part_starts[P+1])."""
        P = self.properties.partition_count
        starts = (C.c_int64 * (P + 1))()
        nv.check(nv.lib().dfd_exchange_wait(exchange._h, starts))
        c_out, types, _ = self._pending
        self._out = _window_columns(c_out, types, exchange, int(starts[P]))
        self._starts = np.frombuffer(starts, dtype=np.int64).copy()
        return self._out, self._starts

    # -- single-pass fused shuffle (segments) -------------------------------------------------
    def shuffle_onepass(self, exchange: ShuffleExchange, in_cols: Sequence[DeviceColumn], n_rows: int,
                        nullable: Optional[Sequence[bool]] = None):
        """`dfd_shuffle_device_onepass`: the NCCL-free fused shuffle.  Fixed-width non-null columns take the single-pass
        kernel (asynchronous); nullable / boolean / string columns take the push transport.  `nullable[i]` is the
        SCHEMA's nullable flag of column i (every worker must pass the same; default: this worker's columns that
        carry a validity bitmap).  Complete it with `collect()`; `in_cols` must stay allocated until then, because a
        shuffle whose sub-window overflowed re-runs from them inside `collect()`."""
        if len(self.input_stage.tasks) != exchange.world or self.task_count != exchange.world:
            raise ValueError("this exchange runs one producer and one consumer task per GPU worker")
        P = self.properties.partition_count
        c_out = _nullable_outs(in_cols, nullable)
        nv.check(nv.lib().dfd_shuffle_device_onepass(exchange._h, self._partitioner(exchange), columns_to_c(in_cols), len(in_cols), n_rows, P, c_out))
        self._pending = (c_out, [c.arrow_type for c in in_cols], exchange)

    @staticmethod
    def segment_to_arrow(ctx: WorkerContext, col: DeviceColumn, start: int, count: int):
        """Download rows [start, start+count) of a window-resident output column as a pyarrow Array (test / debug helper)."""
        import pyarrow as pa

        def grab(ptr, nbytes):
            buf = np.empty(max(nbytes, 1), dtype=np.uint8)
            if nbytes:
                nv.check(nv.lib().dfd_memcpy_d2h(ctx.handle, buf.ctypes.data, ptr, nbytes))
            return buf[:nbytes]

        def bits(ptr):  # bitmap rows [start, start+count) re-based to bit 0
            lo = start // 8
            raw = grab(ptr + lo, (start % 8 + count + 7) // 8)
            b = np.unpackbits(raw, bitorder="little")[start % 8: start % 8 + count]
            return b

        validity_buf, null_count = None, 0
        if col.validity:
            vb = bits(col.validity)
            null_count = int(count - vb.sum())
            validity_buf = pa.py_buffer(np.packbits(vb, bitorder="little").tobytes())
        if col.kind == nv.COL_BOOL:
            data = pa.py_buffer(np.packbits(bits(col.values), bitorder="little").tobytes())
            return pa.Array.from_buffers(pa.bool_(), count, [validity_buf, data], null_count=null_count)
        if col.kind == nv.COL_FIXED:
            data = pa.py_buffer(grab(col.values + start * col.width, count * col.width).tobytes())
            return pa.Array.from_buffers(col.arrow_type, count, [validity_buf, data], null_count=null_count)
        ow = 8 if col.kind == nv.COL_LARGE_UTF8 else 4
        if count == 0:
            return pa.array([], type=col.arrow_type)
        off = grab(col.offsets + start * ow, (count + 1) * ow).view(np.int64 if ow == 8 else np.int32)
        lo, hi = int(off[0]), int(off[-1])
        data = pa.py_buffer(grab(col.values + lo, hi - lo).tobytes())
        offs = pa.py_buffer((off - lo).astype(off.dtype).tobytes())
        return pa.Array.from_buffers(col.arrow_type, count, [validity_buf, offs, data], null_count=null_count)

    def collect(self, exchange: ShuffleExchange):
        """Complete `shuffle_onepass`: returns (out columns, seg_starts[P][T], seg_counts[P][T]) — partition q is the
        merge of its T per-producer segments (rows [seg_starts[q][r], +seg_counts[q][r]) of every column)."""
        P, T = self.properties.partition_count, exchange.world
        starts, counts = (C.c_int64 * (P * T))(), (C.c_int64 * (P * T))()
        c_out, types, _ = self._pending
        nv.check(nv.lib().dfd_exchange_collect(exchange._h, c_out, starts, counts))
        self._seg_starts = np.frombuffer(starts, dtype=np.int64).reshape(P, T).copy()
        self._seg_counts = np.frombuffer(counts, dtype=np.int64).reshape(P, T).copy()
        self._out = _window_columns(c_out, types, exchange)
        self._starts = None
        return self._out, self._seg_starts, self._seg_counts

    def execute_segments(self, partition: int, task_ctx: DistributedTaskContext):
        """≙ NetworkShuffleExec::execute(partition, ctx) after `collect()`: the partition's per-producer streams as
        (columns, [(first_row, n_rows) per producer task])."""
        if self._out is None or getattr(self, "_seg_starts", None) is None:
            raise RuntimeError("shuffle_onepass()/collect() has not run")
        P = self.properties.partition_count
        if not 0 <= partition < P:
            raise IndexError(partition)
        return self._out, [(int(a), int(n)) for a, n in zip(self._seg_starts[partition], self._seg_counts[partition])]

    def shuffle_partitioned(self, exchange: ShuffleExchange, in_cols: Sequence[DeviceColumn], part_starts: Sequence[int],
                            nullable: Optional[Sequence[bool]] = None):
        """The exchange half alone, for rows that are ALREADY hash-partitioned on this worker into P x T global partitions
        (`dfd_partition_device` [+ `PartialReduceExec`]): `dfd_exchange_gather(DFD_ROUTE_SHUFFLE)`.  Returns
        (out columns, seg_starts[P][T], seg_counts[P][T])."""
        P, T = self.properties.partition_count, exchange.world
        starts = (C.c_int64 * (P * T + 1))(*[int(v) for v in part_starts])
        c_out = _nullable_outs(in_cols, nullable)
        nv.check(nv.lib().dfd_exchange_gather(exchange._h, nv.ROUTE_SHUFFLE, columns_to_c(in_cols), len(in_cols), starts, P, T, c_out))
        self._pending = (c_out, [c.arrow_type for c in in_cols], exchange)
        return self.collect(exchange)

    def shuffle_rounds(self, exchange: ShuffleExchange, in_cols: Sequence[DeviceColumn], n_rows: int,
                       nullable: Optional[Sequence[bool]] = None):
        """Back-pressured shuffle (`dfd_shuffle_stream_*`): a generator of rounds (out columns, seg_starts[P][T],
        seg_counts[P][T]); a round's buffers are valid until the next one is requested.  Rounds shrink automatically
        when a consumer's receive window cannot hold one (skew / small windows) instead of failing."""
        P, T = self.properties.partition_count, exchange.world
        h = C.c_void_p()
        nl = (C.c_uint8 * len(in_cols))(*[1 if (nullable[i] if nullable is not None else bool(c.validity)) else 0 for i, c in enumerate(in_cols)])
        nv.check(nv.lib().dfd_shuffle_stream_begin(exchange._h, self._partitioner(exchange), columns_to_c(in_cols), len(in_cols), n_rows, P, nl, C.byref(h)))
        try:
            while True:
                c_out = (nv.DfdColumn * len(in_cols))()
                starts, counts, done = (C.c_int64 * (P * T))(), (C.c_int64 * (P * T))(), C.c_int(0)
                nv.check(nv.lib().dfd_shuffle_stream_next(h, c_out, starts, counts, C.byref(done)))
                if done.value:
                    break
                outs = _window_columns(c_out, [c.arrow_type for c in in_cols], exchange)
                yield outs, np.frombuffer(starts, dtype=np.int64).reshape(P, T).copy(), np.frombuffer(counts, dtype=np.int64).reshape(P, T).copy()
            r, sp = C.c_uint64(), C.c_uint64()
            nv.lib().dfd_shuffle_stream_stats(h, C.byref(r), C.byref(sp))
            self.last_stream_stats = {"rounds": r.value, "splits": sp.value}
        finally:
            nv.lib().dfd_shuffle_stream_end(h)

    def shuffle_host(self, exchange: ShuffleExchange, host_in: Sequence[DeviceColumn], n_rows: int, n_chunks: int,
                     host_out: Sequence[DeviceColumn], out_capacity_rows: int) -> np.ndarray:
        """Host-to-host pipelined shuffle (`dfd_shuffle_host`): `host_in` / `host_out` describe HOST (pinned)
        column buffers.  Returns chunk_part_starts[n_chunks][P+1] (absolute row offsets into host_out)."""
        P = self.properties.partition_count
        starts = (C.c_int64 * (n_chunks * (P + 1)))()
        nv.check(nv.lib().dfd_shuffle_host(exchange._h, self._partitioner(exchange), columns_to_c(host_in), len(host_in), n_rows, P, n_chunks,
                                           columns_to_c(host_out), out_capacity_rows, starts))
        return np.frombuffer(starts, dtype=np.int64).reshape(n_chunks, P + 1).copy()

    def execute(self, partition: int, task_ctx: DistributedTaskContext):
        """≙ NetworkShuffleExec::execute(partition, ctx): rows with
        hash % (P*T) == P*task_index + partition, as (columns, first_row, end_row)."""
        if self._out is None:
            raise RuntimeError("shuffle() has not run")
        P = self.properties.partition_count
        if not 0 <= partition < P:
            raise IndexError(partition)
        return self._out, int(self._starts[partition]), int(self._starts[partition + 1])


# ---------------------------------------------------------------------------------------------
# Sibling exchanges over the same transport: NetworkCoalesceExec / NetworkBroadcastExec
# ---------------------------------------------------------------------------------------------

def task_group(input_task_count: int, task_index: int, task_count: int):
    """src/execution_plans/network_coalesce.rs:264-289 — the contiguous group of input tasks consumer `task_index` reads:
    (start_task, len, max_len)."""
    a, b, c = C.c_int(), C.c_int(), C.c_int()
    nv.check(nv.lib().dfd_coalesce_task_group(input_task_count, task_index, task_count, C.byref(a), C.byref(b), C.byref(c)))
    return a.value, b.value, c.value


class _GatherExec:
    ROUTE = None

    def __init__(self, partitions: int, input_stage: Stage, task_count: int):
        self.partitions = partitions          # P: partitions of every producer task
        self.input_stage = input_stage
        self.task_count = task_count          # consumer tasks
        self._out = None
        self._starts = self._counts = None

    def gather(self, exchange: ShuffleExchange, in_cols: Sequence[DeviceColumn], slice_starts: Sequence[int],
               nullable: Optional[Sequence[bool]] = None):
        """Collective: this worker (producer task `rank`) contributes its P partitions = row slices of `in_cols`."""
        if len(self.input_stage.tasks) != exchange.world:
            raise ValueError("one producer task per GPU worker")
        P = self.partitions
        starts = (C.c_int64 * (P + 1))(*[int(v) for v in slice_starts])
        c_out = _nullable_outs(in_cols, nullable)
        nv.check(nv.lib().dfd_exchange_gather(exchange._h, self.ROUTE, columns_to_c(in_cols), len(in_cols), starts, P, self.task_count, c_out))
        n = nv.lib().dfd_exchange_pending_segments(exchange._h)
        ss, sc = (C.c_int64 * max(n, 1))(), (C.c_int64 * max(n, 1))()
        nv.check(nv.lib().dfd_exchange_collect(exchange._h, c_out, ss, sc))
        self._starts = np.frombuffer(ss, dtype=np.int64)[:n].copy()
        self._counts = np.frombuffer(sc, dtype=np.int64)[:n].copy()
        self._out = _window_columns(c_out, [c.arrow_type for c in in_cols], exchange)
        return self._out, self._starts, self._counts


class NetworkCoalesceExec(_GatherExec):
    """src/execution_plans/network_coalesce.rs — coalesce the partitions of T_in tasks into task_count tasks without
    repartitioning.  Output partitions per consumer task = P x max group size; partition i reads partition i % P of
    input task group.start + i / P (empty when the group is shorter than the longest one)."""
    ROUTE = nv.ROUTE_COALESCE

    @staticmethod
    def try_new(input_partitions: int, query_id: uuid.UUID, num: int, task_count: int, input_task_count: int) -> "NetworkCoalesceExec":
        if task_count == 0:
            raise ValueError("NetworkCoalesceExec cannot be executed with task_count=0")
        return NetworkCoalesceExec(input_partitions, Stage(query_id, num, None, [ExecutionTask(None) for _ in range(input_task_count)]), task_count)

    def name(self) -> str:
        return "NetworkCoalesceExec"

    def output_partition_count(self) -> int:
        return self.partitions * max(-(-len(self.input_stage.tasks) // self.task_count), 1)

    def execute(self, partition: int, task_ctx: DistributedTaskContext):
        """-> (columns, first_row, n_rows) of output `partition` on consumer task task_ctx.task_index (n_rows 0: padding)."""
        if task_ctx.task_index >= task_ctx.task_count:
            raise ValueError(f"NetworkCoalesceExec invalid task context: task_index={task_ctx.task_index} >= task_count={task_ctx.task_count}")
        if not 0 <= partition < self.output_partition_count():
            raise IndexError(partition)
        if self._out is None:
            raise RuntimeError("gather() has not run")
        start, length, _ = task_group(len(self.input_stage.tasks), task_ctx.task_index, task_ctx.task_count)
        if partition // self.partitions >= length:
            return self._out, 0, 0
        return self._out, int(self._starts[partition]), int(self._counts[partition])


class NetworkBroadcastExec(_GatherExec):
    """src/execution_plans/network_broadcast.rs — every consumer task reads all P partitions of every input task;
    output partition p is the merge of one stream per input task."""
    ROUTE = nv.ROUTE_BROADCAST

    @staticmethod
    def try_new(input_partitions: int, query_id: uuid.UUID, num: int, task_count: int, input_task_count: int) -> "NetworkBroadcastExec":
        return NetworkBroadcastExec(input_partitions, Stage(query_id, num, None, [ExecutionTask(None) for _ in range(input_task_count)]), task_count)

    def name(self) -> str:
        return "NetworkBroadcastExec"

    def execute(self, partition: int, task_ctx: DistributedTaskContext):
        """-> (columns, [(first_row, n_rows) per input task]) of output `partition`."""
        if not 0 <= partition < self.partitions:
            raise IndexError(partition)
        if self._out is None:
            raise RuntimeError("gather() has not run")
        T = len(self.input_stage.tasks)
        return self._out, [(int(self._starts[partition * T + r]), int(self._counts[partition * T + r])) for r in range(T)]
