"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import json
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hash_vectors.json")
LAUNCH_HEADER = os.path.join(ROOT, "datafusion_distributed_b200", "csrc", "dfd_launch.cuh")


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def cfg2_columns(n_rows: int, n_cols: int = 8, seed: int = 42):
    """SURVEY.md §8(d) cfg-2 shape: col0 = uniform i64 key, cols j>=1 = row_id*8+j."""
    rng = np.random.Generator(np.random.PCG64(seed))
    key = rng.integers(-(2**63), 2**63 - 1, n_rows, dtype=np.int64, endpoint=True)
    return [key] + [np.arange(n_rows, dtype=np.int64) * 8 + j for j in range(1, n_cols)]


def expected_partitions(dest: np.ndarray, num_partitions: int):
    """Stable per-destination row index lists from destination ids."""
    order = np.argsort(dest, kind="stable")
    counts = np.bincount(dest, minlength=num_partitions).astype(np.int64)
    starts = np.zeros(num_partitions + 1, dtype=np.int64)
    np.cumsum(counts, out=starts[1:])
    return order, starts


# ------------------------------------------------------------ tile geometry ----

def tile_geometry(env=None):
    """(two-pass tile rows, single-pass tile rows) of the library as build.py compiles it: the defaults of
    csrc/dfd_launch.cuh, overridden by the -DNAME=VALUE options of DFD_NVCC_DEFS (and, for the single-pass K, of
    DFD_NVCC_DEFS_ONEPASS), which build.py passes to nvcc.  The tile-sweep scripts rebuild with other geometries; the
    edge sizes of the scatter tests follow them through this."""
    env = os.environ if env is None else env
    with open(LAUNCH_HEADER) as f:
        src = f.read()
    vals = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DFD_\w+)\s+(\d+)", src)}
    for var in ("DFD_NVCC_DEFS", "DFD_NVCC_DEFS_ONEPASS"):
        for m in re.finditer(r"-D(DFD_\w+)=(\d+)", env.get(var, "")):
            if var == "DFD_NVCC_DEFS" or m.group(1) == "DFD_ONEPASS_K":
                vals[m.group(1)] = int(m.group(2))
    threads = vals["DFD_TILE_THREADS"]
    return threads * vals["DFD_TILE_K"], threads * vals["DFD_ONEPASS_K"]


def edge_sizes(env=None):
    """Row counts for the ragged-size scatter tests, the same for the two-pass and the single-pass kernel: for each of
    their tilings (tile_geometry), one tile and one row either side, exactly two tiles (full last tile, exact ticket
    count) and one row more.  An edge of one tiling is a ragged interior size of the other.  Plus sizes that are no
    tile edge: empty, one row, around a warp, around 2^11 and a many-tile ragged size."""
    sizes = {0, 1, 31, 32, 33, 2047, 2048, 2049, 100_003}
    for t in tile_geometry(env):
        sizes |= {t - 1, t, t + 1, 2 * t, 2 * t + 1}
    return sorted(sizes)


def multi_tile_rows():
    """A row count at which every CTA of the persistent single-pass grid handles several tiles: at least 4 tiles for
    each of the 7 CTAs of 288 threads an SM can hold at most (the grid never exceeds that).  Then a CTA ranks tile t+1
    into its second buffer while tile t scatters, with the ring parity carried from tile to tile."""
    import torch

    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    return 4 * 7 * sm_count * tile_geometry()[1] + 777  # (ragged last tile)


# ------------------------------------------------ 32-bit limits of the ABI ----
# Restatements of the row-count checks in dfd_api.cu / dfd_reduce.cu, so the limit tests name the boundary they cross.

PARTITION_MAX_ROWS = (1 << 32) - 1  # dfd_partition_device / PartitionJob::prepare: n_rows <= 2^32 - 1
REDUCE_MAX_ROWS = 1 << 31           # dfd_partial_reduce_device: the group table's slots must fit a u32 mask


def onepass_regions_accepted(region_rows: int, N: int, n_rows: int) -> bool:
    """dfd_partition_device_onepass's region check: every row fits, and N * region_rows < 2^32 - 1 (32-bit output rows,
    0xffffffff is the kernel's empty-slot sentinel)."""
    return region_rows >= 1 and region_rows * N >= n_rows and region_rows * N < (1 << 32) - 1


# Small key domains for the limit tests: the destination of every possible key is computed once by the C oracle, and the
# GPU then derives a row's destination as LUT[key] — exact at any row count, and independent of the kernels under test.

def domain_values(kind: str) -> np.ndarray:
    """Every key of a domain, at its LUT index: "u8" = all 256 uint8 values, "i16" = all 65 536 int16 values (index =
    the value's bits as uint16), "i64" = 65 536 seeded int64 values (index = an int16 row's bits as uint16)."""
    if kind == "u8":
        return np.arange(256, dtype=np.uint8)
    if kind == "i16":
        return np.arange(1 << 16, dtype=np.uint16).view(np.int16)
    if kind == "i64":
        return np.random.Generator(np.random.PCG64(2024)).integers(-(1 << 63), (1 << 63) - 1, 1 << 16, dtype=np.int64, endpoint=True)
    raise ValueError(kind)


def dest_lut(kind: str, N: int) -> np.ndarray:
    """Destination (create_hashes % N, the C oracle) of every key of domain `kind`, as int32 indexed like domain_values.
    A null key hashes to 0 and goes to destination 0."""
    from oracle import oracle as orc

    v = domain_values(kind)
    return orc.partition_ids([v], len(v), N).astype(np.int32)


# ---------------------------------------------- PartialReduce group hashing ----
# Restatement of dfd_reduce.cu's key_hash for one 8-byte key, and its inverse, to craft keys that land on a chosen slot.

M64 = (1 << 64) - 1
REDUCE_HASH_SEED = 0x9E3779B97F4A7C15
_MIX_C1, _MIX_C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53


def mix64(x: int) -> int:
    """The murmur3 64-bit finaliser (dfd_reduce.cu mix64)."""
    x ^= x >> 33
    x = (x * _MIX_C1) & M64
    x ^= x >> 33
    x = (x * _MIX_C2) & M64
    x ^= x >> 33
    return x


def unmix64(h: int) -> int:
    """Inverse of mix64: x ^= x >> 33 undoes itself (33 >= 32) and the odd multipliers are invertible mod 2^64."""
    h ^= h >> 33
    h = (h * pow(_MIX_C2, -1, 1 << 64)) & M64
    h ^= h >> 33
    h = (h * pow(_MIX_C1, -1, 1 << 64)) & M64
    h ^= h >> 33
    return h


def reduce_table_slots(n_rows: int) -> int:
    """Open-addressing table size of dfd_partial_reduce_device: the smallest power of two >= max(64, 2 * n_rows)."""
    slots = 64
    while slots < 2 * n_rows:
        slots <<= 1
    return slots


def reduce_slot_of_i64_key(k: int, slots: int) -> int:
    """Home slot of a single 8-byte group key: key_hash = mix64(seed ^ k), truncated to 32 bits, masked."""
    return mix64(REDUCE_HASH_SEED ^ (k & M64)) & 0xFFFFFFFF & (slots - 1)


def keys_on_slot(n_keys: int, slot: int, slots: int, seed: int = 0) -> np.ndarray:
    """`n_keys` distinct int64 group keys whose home slot is `slot` of a `slots`-slot table."""
    rng = np.random.Generator(np.random.PCG64(seed))
    shift = slots.bit_length() - 1
    highs = rng.choice(1 << 40, n_keys, replace=False)  # distinct hashes -> distinct keys (mix64 is a bijection)
    keys = [unmix64((int(hi) << shift) | slot) ^ REDUCE_HASH_SEED for hi in highs]
    return np.array([k - (1 << 64) if k >> 63 else k for k in keys], dtype=np.int64)
