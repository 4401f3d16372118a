"""GPU-native (H100) hash-repartition shuffle for datafusion-distributed.

Host mirror of the reference's operator surface for ONE path
(RepartitionExec(Hash) -> exchange -> NetworkShuffleExec); all compute is in
hand-written sm_90a CUDA behind the C ABI in include/dfd_b200.h.  The package
has no CPU fallback: importing is cheap, but every compute call requires the
built `_lib/libdfd_b200.so` and a CUDA device.
"""
from . import _native
from ._native import DfdError, LIB_PATH
from .device import DeviceBuffer, DeviceColumn, WorkerContext
from .execution_plans import PinnedTable, RepartitionExec
from .network_shuffle import (DistributedTaskContext, ExecutionTask, NetworkBroadcastExec, NetworkCoalesceExec, NetworkShuffleExec,
                              ShuffleExchange, Stage, exchange_plan, nccl_unique_id, task_group)
from .partitioner import HashPartitioner, PartialReduceExec, Partitioning, agg_op, scale_partitioning

__all__ = [
    "DfdError", "LIB_PATH", "DeviceBuffer", "DeviceColumn", "WorkerContext",
    "HashPartitioner", "PartialReduceExec", "Partitioning", "agg_op", "scale_partitioning", "RepartitionExec", "PinnedTable",
    "DistributedTaskContext", "ExecutionTask", "NetworkShuffleExec", "ShuffleExchange", "Stage", "exchange_plan", "nccl_unique_id",
    "NetworkCoalesceExec", "NetworkBroadcastExec", "task_group",
]
