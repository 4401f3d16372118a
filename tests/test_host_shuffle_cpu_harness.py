"""dfd_shuffle_host with nullable, Boolean and string columns, on the CPU with N worker threads.

The product's `dfd_exchange` object is linked — under pytest's temporary directory, for this test only — with the stand-in
CUDA runtime and NCCL, the CPU oracle in place of the partition kernels (tests/cpu_harness/harness_dfd.cu), the CPU
emulations of the push transport's kernels (harness_exchange.cu) and of the compaction's bit kernel k_place_bits
(harness_host_bits.cu).  tests/cpu_harness/run_host_shuffle_workers.py then runs T worker THREADS through the whole
host-to-host path: staging of chunk rows at their bit offset, the push transport, the compaction of the window segments
into one dense chunk (values, re-based string offsets continued across chunks, bitmaps at any host bit with the word two
chunks share), the host capacity checks, and compares every (chunk, partition) with the single-node oracle."""
import os
import subprocess
import sys

import pytest

from tests.test_exchange_cpu_harness import CSRC, HARNESS, NVCC, NVCC_FLAGS, ROOT


@pytest.fixture(scope="module")
def host_shuffle_harness(built, tmp_path_factory):
    from datafusion_distributed_b200 import build as b
    from oracle import oracle as orc

    tmp = str(tmp_path_factory.mktemp("host_shuffle_harness"))
    b.build()
    oracle_so = orc.build()
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC, "-I", os.path.join(ROOT, "oracle")]
    newest = max(os.path.getmtime(os.path.join(d, f)) for d in (CSRC, os.path.join(ROOT, "include")) for f in os.listdir(d))
    xobj = b.object_path("dfd_exchange.cu")  # the product's own object
    if not os.path.exists(xobj) or os.path.getmtime(xobj) < newest:
        xobj = os.path.join(tmp, "dfd_exchange.o")
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(CSRC, "dfd_exchange.cu"), "-o", xobj])
    objs = [xobj]
    for src in ("harness_dfd.cu", "harness_exchange.cu", "harness_host_bits.cu"):
        o = os.path.join(tmp, src.replace(".cu", ".o"))
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(HARNESS, src), "-o", o])
        objs.append(o)
    rt = os.path.join(tmp, "fake_cudart.o")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-c", os.path.join(HARNESS, "fake_cudart.cpp"), "-o", rt])
    so = os.path.join(tmp, "libdfd_host_shuffle_harness.so")
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", so] + objs + [rt, oracle_so, f"-Wl,-rpath,{os.path.dirname(oracle_so)}", "-lpthread", "-ldl"])
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-shared", os.path.join(HARNESS, "fake_nccl.cpp"), "-o", os.path.join(tmp, "libnccl.so.2"),
                           "-lpthread"])
    return so, tmp


def run(harness, world, scenario, seed=1, **extra_env):
    so, tmp = harness
    env = dict(os.environ, LD_LIBRARY_PATH=tmp + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""), **extra_env)
    out = subprocess.run([sys.executable, os.path.join(HARNESS, "run_host_shuffle_workers.py"), so, str(world), scenario, str(seed)], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and f"WORKERS_OK world={world} scenario={scenario}" in out.stdout, out.stdout[-2000:] + out.stderr[-6000:]


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_host_shuffle_of_the_mixed_schema_matches_the_oracle(host_shuffle_harness, world):
    """Keys Int64 + Utf8 over Int64 / Utf8 / LargeUtf8 / Boolean / Int32 / Float64, nullable, with a producer of 0 rows:
    n_chunks 1, 3, 7 and 50 (more chunks than rows) on one exchange; every (chunk, partition) equals the oracle's rows,
    producers in task order, bitmap bits past the last row are 0 and nothing is written past any capacity."""
    run(host_shuffle_harness, world, "mixed")


@pytest.mark.parametrize("world", [2, 3])
def test_a_worker_one_string_byte_short_refuses_and_its_peers_fail_too(host_shuffle_harness, world):
    """The last worker's Utf8 output is one byte short of what the chunks up to one before the last need: it returns
    DFD_ERR_CAPACITY naming the bytes needed, with the chunks before that one delivered; every other worker returns an
    error after the bounded flag wait of the next chunk, none hangs."""
    run(host_shuffle_harness, world, "short", HARNESS_FLAG_TIMEOUT_MS="400")
