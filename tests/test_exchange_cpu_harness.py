"""The exchange's HOST logic with N > 1 workers on the CPU.

The object nvcc built from `csrc/dfd_exchange.cu` for the product is linked — under pytest's temporary directory, for this test
only — against the stand-in CUDA runtime (tests/cpu_harness/fake_cudart.cpp: IPC handles are pointers, kernel launches are
dispatched to CPU emulations by name), a thread-rendezvous stand-in of NCCL (fake_nccl.cpp, loaded through the library's own
dlopen("libnccl.so.2")) and the CPU oracle in place of the partition kernels.  T worker THREADS of one sub-process then run the
push transport exactly as T GPU workers would: window set-up with size agreement, the flag all-gather of row / byte counts,
every worker deriving every consumer's layout, `k_push_runs`-shaped copies into the owners' windows, the done barrier —
for the shuffle (NetworkShuffleExec), the back-pressured rounds, NetworkCoalesceExec and NetworkBroadcastExec routes, with
nullable / boolean / string columns, and compare every (partition, producer) segment with the single-node oracle.  The
single-pass exchange (fixed-width non-null schemas: ready flags, peer stores into (partition, producer) sub-windows, publish /
wait, and the overflow -> exact two-pass re-run that every worker must take together) runs the same way, its scatter kernels
replaced by row loops, and so do the two-pass fused transport and the NCCL-mode transport (grouped ncclSend / ncclRecv through
mailboxes of the stand-in NCCL)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "cpu_harness")
CSRC = os.path.join(ROOT, "datafusion_distributed_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-Xcompiler", "-fPIC"]


@pytest.fixture(scope="module")
def exchange_harness(built, tmp_path_factory):
    from datafusion_distributed_b200 import build as b
    from oracle import oracle as orc

    tmp = str(tmp_path_factory.mktemp("exchange_harness"))
    b.build()
    oracle_so = orc.build()
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC, "-I", os.path.join(ROOT, "oracle")]
    newest = max(os.path.getmtime(os.path.join(d, f)) for d in (CSRC, os.path.join(ROOT, "include")) for f in os.listdir(d))
    xobj = b.object_path("dfd_exchange.cu")  # the product's own object
    if not os.path.exists(xobj) or os.path.getmtime(xobj) < newest:
        xobj = os.path.join(tmp, "dfd_exchange.o")
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(CSRC, "dfd_exchange.cu"), "-o", xobj])
    objs = [xobj]
    for src in ("harness_dfd.cu", "harness_exchange.cu"):
        o = os.path.join(tmp, src.replace(".cu", ".o"))
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(HARNESS, src), "-o", o])
        objs.append(o)
    rt = os.path.join(tmp, "fake_cudart.o")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-c", os.path.join(HARNESS, "fake_cudart.cpp"), "-o", rt])
    so = os.path.join(tmp, "libdfd_exchange_harness.so")
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", so] + objs + [rt, oracle_so, f"-Wl,-rpath,{os.path.dirname(oracle_so)}", "-lpthread", "-ldl"])
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-shared", os.path.join(HARNESS, "fake_nccl.cpp"), "-o", os.path.join(tmp, "libnccl.so.2"),
                           "-lpthread"])
    return so, tmp


def run(exchange_harness, world, scenario, seed=1, **extra_env):
    so, tmp = exchange_harness
    env = dict(os.environ, LD_LIBRARY_PATH=tmp + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""), **extra_env)
    out = subprocess.run([sys.executable, os.path.join(HARNESS, "run_workers.py"), so, str(world), scenario, str(seed)], env=env, capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0 and f"WORKERS_OK world={world} scenario={scenario}" in out.stdout, out.stdout[-2000:] + out.stderr[-6000:]


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_push_shuffle_segments_match_the_oracle(exchange_harness, world):
    run(exchange_harness, world, "shuffle")


@pytest.mark.parametrize("world", [2, 4])
def test_back_pressured_rounds_deliver_every_row_once(exchange_harness, world):
    run(exchange_harness, world, "stream")


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_coalesce_route_with_uneven_groups(exchange_harness, world):
    run(exchange_harness, world, "coalesce")


@pytest.mark.parametrize("world", [2, 4])
def test_broadcast_route(exchange_harness, world):
    run(exchange_harness, world, "broadcast")


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_single_pass_exchange_sub_windows_and_flags(exchange_harness, world):
    run(exchange_harness, world, "onepass")


@pytest.mark.parametrize("world", [2, 3])
def test_single_pass_overflow_makes_every_worker_rerun_exactly(exchange_harness, world):
    run(exchange_harness, world, "onepass_overflow")


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_nccl_mode_moves_every_column_kind(exchange_harness, world):
    run(exchange_harness, world, "nccl")


def test_nccl_mode_refuses_int32_offsets_past_int32_max_on_every_worker(exchange_harness):
    """Two producers of 1.1 GiB of Utf8 each, all for one consumer: DFD_ERR_CAPACITY on both workers before any send."""
    run(exchange_harness, 2, "nccl_int32")


@pytest.mark.parametrize("world", [1, 2, 4])
def test_two_pass_fused_transport_dense_layout(exchange_harness, world):
    run(exchange_harness, world, "fused")


@pytest.mark.parametrize("world", [1, 2, 3])
def test_host_to_host_shuffle_in_chunks(exchange_harness, world):
    run(exchange_harness, world, "host")


@pytest.mark.parametrize("world", [2, 4])
def test_transports_alternate_on_one_window(exchange_harness, world):
    run(exchange_harness, world, "mixed")


@pytest.mark.parametrize("world", [1, 2])
def test_collect_reports_only_the_last_shuffle(exchange_harness, world):
    run(exchange_harness, world, "stale")


def test_a_missing_peer_is_an_error_after_a_bounded_wait_not_a_hang(exchange_harness):
    run(exchange_harness, 3, "peer_missing", HARNESS_FLAG_TIMEOUT_MS="400")


def test_workers_refuse_windows_of_different_sizes(exchange_harness):
    run(exchange_harness, 3, "mismatch")
