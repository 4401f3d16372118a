"""Shared memory of every scatter launch against the 227 KiB a CTA can have on sm_90, on the CPU.

A host-only program, compiled with nvcc under pytest's tmp directory against csrc/dfd_kernels.cuh and dfd_launch.cuh (the
same headers and tile-geometry defines the library is built with), prints the dynamic shared memory of every launch
launch_scatter_kv can make for each N in [1, DFD_MAX_PARTITIONS]:
- two-pass k_scatter: staged widths 1, 2, 4, 8 and 16 bytes, and bit columns (staged one byte per row), local and peer
  (no bit columns in peer mode);
- follow-up k_scatter on the single-pass tiling, and k_scatter_onepass (rings of 1-8 bytes), where single-pass calls
  exist (N <= ONEPASS_MAX_N);
- each also with the aligned write-out, which only peer launches take, where use_aligned turns it on (N <= ALIGNED_MAX_N).
Every launch must fit, since dfd_partitioner_create accepts every such N and a launch that does not fit fails only after
the histogram pass (and, in the exchange, after the counts were all-gathered).  The admission check (scatter_smem_worst)
must be the largest of them."""
import os
import re
import subprocess

import pytest

from tests.util import _launch_defines

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "datafusion_distributed_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SMEM_LIMIT = 227 * 1024  # dynamic shared memory one CTA can opt into on sm_90

PROGRAM = r"""
#include <cstdio>
#include "dfd_launch.cuh"
using namespace dfd;

int main() {
    std::printf("max_n %u onepass_max_n %u aligned_max_n %u\n", (unsigned)DFD_MAX_PARTITIONS, ONEPASS_MAX_N, ALIGNED_MAX_N);
    for (uint32_t N = 1; N <= DFD_MAX_PARTITIONS; ++N) {
        std::printf("N %u worst %zu\n", N, scatter_smem_worst(N));
        for (const int aligned : {0, 1}) {
            for (const int peer : {0, 1}) {
                // width 0: a bit column, staged one byte per row (launch_width_groups sets stage_width = 1)
                for (const int width : {0, 1, 2, 4, 8, 16}) {
                    const int stage = width ? width : 1;
                    std::printf("L twopass %d %d %d %zu\n", width, peer, aligned,
                                scatter_smem_bytes<TILE_THREADS, TILE_K>(N, stage, peer, aligned));
                    std::printf("L follow %d %d %d %zu\n", width, peer, aligned,
                                scatter_smem_bytes<TILE_THREADS, ONEPASS_K>(N, stage, peer, aligned));
                    if (width >= 1 && width <= 8)
                        std::printf("L onepass %d %d %d %zu\n", width, peer, aligned,
                                    onepass_smem_bytes<TILE_THREADS, ONEPASS_K, ONEPASS_NB, ONEPASS_SPLIT>(N, width, peer, aligned));
                }
            }
        }
    }
    return 0;
}
"""


def launch_reachable(kind, width, peer, aligned, N, onepass_max_n, aligned_max_n):
    """Whether the library can make this launch for a partitioner with N destinations (the dispatch of dfd_api.cu and
    dfd_launch.cuh, as tests/util.py scatter_dispatch restates it)."""
    if aligned and (not peer or N > aligned_max_n):  # use_aligned
        return False
    if peer and width == 0:  # bit columns exist only in local calls
        return False
    if kind in ("follow", "onepass") and N > onepass_max_n:
        return False
    return True


@pytest.fixture(scope="module")
def table(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("smem")
    src, exe = tmp / "smem_table.cu", tmp / "smem_table"
    src.write_text(PROGRAM)
    defs = os.environ.get("DFD_NVCC_DEFS", "").split() + os.environ.get("DFD_NVCC_DEFS_ONEPASS", "").split()
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", CSRC] + defs + [str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    head = out[0].split()
    limits = {"max_n": int(head[1]), "onepass_max_n": int(head[3]), "aligned_max_n": int(head[5])}
    worst, launches, N = {}, {}, None
    for line in out[1:]:
        f = line.split()
        if f[0] == "N":
            N = int(f[1])
            worst[N] = int(f[3])
        else:
            launches[(N, f[1], int(f[2]), bool(int(f[3])), bool(int(f[4])))] = int(f[5])
    return limits, worst, launches


def test_table_covers_every_n_width_and_mode(table):
    limits, worst, launches = table
    assert limits["max_n"] == 4096
    assert limits["aligned_max_n"] == _launch_defines(os.environ)["ALIGNED_MAX_N"]
    assert sorted(worst) == list(range(1, limits["max_n"] + 1))
    assert len(launches) == limits["max_n"] * 2 * 2 * (6 + 6 + 4)


def test_every_reachable_scatter_launch_fits_one_cta(table):
    limits, _, launches = table
    too_big = sorted((key, b) for key, b in launches.items() if b > SMEM_LIMIT and launch_reachable(*key[1:], key[0], limits["onepass_max_n"], limits["aligned_max_n"]))
    assert not too_big, f"{len(too_big)} launches need more than {SMEM_LIMIT} B, first: {too_big[:4]}"


def test_peer_launch_of_16_byte_values_fits_at_every_n(table):
    """The fused exchange's two-pass peer scatter at the largest N: 16-byte values (Decimal128, Interval(MonthDayNano),
    FixedSizeBinary(16)) need no more shared memory than the local launch, whose size dfd_partitioner_create admits."""
    limits, _, launches = table
    for N in range(1, limits["max_n"] + 1):
        local, peer = launches[(N, "twopass", 16, False, False)], launches[(N, "twopass", 16, True, False)]
        assert peer == local and peer <= SMEM_LIMIT, (N, local, peer)


def test_admission_check_is_the_largest_launch(table):
    """scatter_smem_worst, which dfd_partitioner_create compares with 227 KiB, is the largest reachable launch at every N."""
    limits, worst, launches = table
    want = {}
    for (N, *launch), b in launches.items():
        if launch_reachable(*launch, N, limits["onepass_max_n"], limits["aligned_max_n"]):
            want[N] = max(want.get(N, 0), b)
    for N in range(1, limits["max_n"] + 1):
        assert worst[N] == want[N], (N, worst[N], want[N])
    assert max(worst.values()) <= SMEM_LIMIT
    with open(os.path.join(CSRC, "dfd_api.cu")) as f:
        create = re.search(r"int dfd_partitioner_create\(.*?\n}\n", f.read(), re.S).group(0)
    assert re.search(r"scatter_smem_worst\(num_partitions\)\s*>\s*227 \* 1024", create), "dfd_partitioner_create no longer admits by scatter_smem_worst"
