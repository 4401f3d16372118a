"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import json
import os
import re
import subprocess
from typing import NamedTuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hash_vectors.json")
LAUNCH_HEADER = os.path.join(ROOT, "datafusion_distributed_b200", "csrc", "dfd_launch.cuh")


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def seed_tuples():
    """ahash seed tuples for the seeded hash tests: DataFusion's default (0, 0, 0, 0), the golden seeded states, each of
    the four words set alone (a word swapped into another hasher field changes the hash), and four distinct words with
    their high bits set."""
    h = 0x9E3779B97F4A7C15
    golden_seeds = sorted({tuple(e["seeds"]) for e in golden()["seeded"]})
    return ([(0, 0, 0, 0)] + golden_seeds + [tuple(h if i == j else 0 for i in range(4)) for j in range(4)] +
            [(0xF0E1D2C3B4A59687, 0x8899AABBCCDDEEFF, 0xC001D00DFEEDFACE, 0xDEADBEEF8BADF00D)])


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

def _launch_defines(env):
    """The tile-geometry macros of csrc/dfd_launch.cuh as build.py compiles them (see tile_geometry)."""
    with open(LAUNCH_HEADER) as f:
        src = f.read()
    vals = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(DFD_\w+)\s+(\d+)", src)}
    for var in ("DFD_NVCC_DEFS", "DFD_NVCC_DEFS_ONEPASS"):
        for m in re.finditer(r"-D(DFD_\w+)=(\d+)", env.get(var, "")):
            if var == "DFD_NVCC_DEFS" or m.group(1) == "DFD_ONEPASS_K":
                vals[m.group(1)] = int(m.group(2))
    vals["ALIGNED_MAX_N"] = int(re.search(r"ALIGNED_MAX_N\s*=\s*(\d+)", src).group(1))
    return vals


def tile_geometry(env=None):
    """(two-pass tile rows, single-pass tile rows) of the library as build.py compiles it: the defaults of
    csrc/dfd_launch.cuh, overridden by the -DNAME=VALUE options of DFD_NVCC_DEFS (and, for the single-pass K, of
    DFD_NVCC_DEFS_ONEPASS), which build.py passes to nvcc.  The tile-sweep scripts rebuild with other geometries; the
    edge sizes of the scatter tests follow them through this."""
    vals = _launch_defines(os.environ if env is None else env)
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


# ------------------------------------------------------ scatter instantiations ----
# The scatter kernels are templates, and launch_scatter_kv (csrc/dfd_launch.cuh) picks one instantiation per launch from
# KIND (ScatterKind: two-pass, single-pass, follow-up), FAST (Int64 key path), V (element type), PEER and ALIGNED.  An instantiation is
# named by the template arguments that tell them apart: K (rows per thread of the tiling: two-pass or single-pass), KV
# (KV > K: the aligned write-out), FAST, V and PEER.  The same parser reads the library's symbol table and the kernel
# names a profiler records, so a test can check which instantiations exist and which ones an input ran.

class ScatterInst(NamedTuple):
    kernel: str  # "k_scatter" (two-pass and follow-up launches) or "k_scatter_onepass"
    K: int
    KV: int
    fast: bool
    V: str  # one of WIDTH_V's values
    peer: bool

    @property
    def aligned(self) -> bool:
        return self.KV > self.K


WIDTH_V = {8: "u64", 4: "u32", 16: "uint4", 2: "u16", 1: "u8", 0: "bit"}  # launch_scatter_w: column width -> V (0: bit column)
_CXX_V = {"unsigned char": "u8", "unsigned short": "u16", "unsigned int": "u32", "unsigned long": "u64", "unsigned long long": "u64",
          "uint4": "uint4", "dfd::BitColumn": "bit"}
_SCATTER_NAME = re.compile(r"\bdfd::(k_scatter(?:_onepass)?)<(.*)>\s*\((?:const\s+)?dfd::ScatterParams\)")


def _cuda_tool(name: str) -> str:
    """A CUDA toolkit binary next to the nvcc that build.py uses."""
    path = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), name)
    return path if os.path.exists(path) else name


def _int_arg(a: str) -> int:
    a = re.sub(r"^\((?:int|bool|unsigned int)\)", "", a.strip())  # cu++filt writes (int)256 / (bool)1, the GNU demangler 256 / true
    return {"true": 1, "false": 0}[a] if a in ("true", "false") else int(a.rstrip("u"))


def parse_scatter_name(name: str):
    """ScatterInst of a demangled scatter kernel name such as `void dfd::k_scatter_onepass<(int)256, (int)10, (int)14,
    (int)3, (int)1, (int)3, (bool)1, unsigned int, (bool)1>(dfd::ScatterParams)`; None for any other kernel.
    k_scatter<THREADS, K, KV, MIN_CTAS, FAST, V, PEER>, k_scatter_onepass<THREADS, K, KV, NB, SPLIT, MIN_CTAS, FAST, V, PEER>."""
    m = _SCATTER_NAME.search(name)
    if not m:
        return None
    a = [s.strip() for s in m.group(2).split(",")]
    return ScatterInst(m.group(1), _int_arg(a[1]), _int_arg(a[2]), bool(_int_arg(a[-3])), _CXX_V[a[-2]], bool(_int_arg(a[-1])))


def scatter_instances(names) -> set:
    """The scatter instantiations among kernel names, demangled or mangled (those are demangled by cu++filt)."""
    names = list(names)
    mangled = [n for n in names if n.startswith("_Z")]
    if mangled:
        out = subprocess.run([_cuda_tool("cu++filt")], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout
        names = [n for n in names if not n.startswith("_Z")] + out.splitlines()
    return {i for i in map(parse_scatter_name, names) if i is not None}


def compiled_scatter_instances(lib_path: str) -> set:
    """Every scatter instantiation in the library's device code (cuobjdump -symbols)."""
    out = subprocess.run([_cuda_tool("cuobjdump"), "-symbols", lib_path], capture_output=True, text=True, check=True).stdout
    return scatter_instances(re.findall(r"\b(_Z\S*k_scatter\S*)", out))


def scatter_inst(mode: int, fast: bool, V: str, peer: bool, aligned: bool, env=None) -> ScatterInst:
    """The instantiation launch_scatter_kv<FAST, V, PEER, ALIGNED, KIND> (dfd_launch.cuh) launches; `mode` is the
    ScatterKind: 0 (TwoPass) is k_scatter on the two-pass tiling, 1 (OnePass) k_scatter_onepass and 2 (FollowUp) k_scatter
    on the single-pass tiling.  The aligned write-out pads KV by ceil(62 * ALIGNED_MAX_N / THREADS) rows per thread
    (TILE_KV / ONEPASS_KV, dfd_launch.cuh)."""
    d = _launch_defines(os.environ if env is None else env)
    threads = d["DFD_TILE_THREADS"]
    K = d["DFD_TILE_K"] if mode == 0 else d["DFD_ONEPASS_K"]
    KV = K + (62 * d["ALIGNED_MAX_N"] + threads - 1) // threads if aligned else K
    return ScatterInst("k_scatter_onepass" if mode == 1 else "k_scatter", K, KV, bool(fast), V, bool(peer))


def use_aligned(N: int, peer: bool) -> bool:
    """dfd::use_aligned (dfd_launch.cuh): the aligned write-out runs for peer launches of up to ALIGNED_MAX_N destinations."""
    return peer and N <= _launch_defines({})["ALIGNED_MAX_N"]


_ROUTES = {(0, False): "dfd_partition_device, and the local partition of the NCCL mode and the push transport (dfd_exchange.cu)",
           (0, True): "EXCHANGE_FUSED (fused_shuffle_locked) and the exact re-run after a single-pass sub-window overflow "
                      "(dfd_exchange_collect)",
           (1, False): "dfd_partition_device_onepass",
           (1, True): "dfd_shuffle_device_onepass with fixed-width non-null columns (onepass_supported, dfd_exchange.cu)",
           (2, False): "dfd_partition_device_onepass: bit columns, or fixed-width columns past the first MAX_COLS_PER_LAUNCH",
           (2, True): "dfd_shuffle_device_onepass: fixed-width columns past the first MAX_COLS_PER_LAUNCH"}


def scatter_dispatch(env=None):
    """Restatement of the scatter dispatch of dfd_api.cu (PartitionJob::run_scatter, run_onepass) and dfd_launch.cuh.
    Returns {instantiation: route} for every instantiation an input reaches.  The rules:
    - widths: two-pass and follow-up launches go out one group per column width {8, 4, 16, 2, 1, 0 = bit columns}
      (PartitionJob::launch_width_groups), each mapped to V by launch_scatter_w;
    - bit columns (Boolean values, validity bitmaps) exist only in local calls: peer calls reject them
      (PartitionJob::prepare), and neither they nor single-pass launches have a bit instantiation (launch_scatter_w);
    - the single-pass launch moves the first MAX_COLS_PER_LAUNCH fixed-width columns with ring_w = min(widest, 8)
      (PartitionJob::run_onepass): V is u8, u16, u32 or u64, never uint4;
    - it takes the FAST key path only with an 8-byte ring (`fast_i64 && ring_w >= 8`, run_onepass; the guards in
      launch_scatter_kv compile no single-pass kernel outside these two rules); two-pass and follow-up launches take it
      whenever the key is fast_i64 (launch_width_groups);
    - follow-up launches (mode 2, ScatterKind::FollowUp) move the bit columns and the fixed-width columns past the first
      launch (run_onepass);
    - ALIGNED = use_aligned(N, PEER) (launch_scatter_t): ALIGNED only for peer launches at N <= 16 (peer launches occur
      on both sides of that bound)."""
    reach = {}
    for mode in (0, 1, 2):
        for width, V in WIDTH_V.items():
            if mode == 1 and width not in (1, 2, 4, 8):
                continue
            for peer in (False, True):
                if peer and width == 0:
                    continue
                for fast in (False, True):
                    if mode == 1 and fast and width != 8:
                        continue
                    for aligned in ((False, True) if peer else (False,)):
                        reach[scatter_inst(mode, fast, V, peer, aligned, env)] = (
                            f"{_ROUTES[mode, peer]}; V = {V}, {'Int64 fast key' if fast else 'generic key'}" +
                            (f", N {'<=' if aligned else '>'} 16" if peer else ""))
    return reach


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


# ------------------------------------------- single-pass write-out slot counts ----
# Restatements of how many write-out slots one tile of k_scatter_onepass uses (dfd_kernels.cuh), and inputs built to use
# as many as the tile's row count allows.  A tile holds T threads * KP (ROWS branch) or KV (aligned write-out) slots; a
# pair or row past that cap would be dropped without a fault.

PAIR_ALIGN_MAX_N = 16  # dfd_kernels.cuh: up to this N the local pairs of a run are padded to aligned 32-pair spans


def onepass_run_pairs(o: int, cnt: int, N: int) -> int:
    """Pairs of the run [o, o + cnt) of absolute output rows in the local single-pass write-out (the ROWS branch's `np`):
    the run cut on even output rows, plus, for N <= PAIR_ALIGN_MAX_N, a front pad of (o >> 1) mod 32 pairs and a round up
    to 32 pairs."""
    if cnt == 0:
        return 0
    wmask = 31 if N <= PAIR_ALIGN_MAX_N else 0
    return ((((o + cnt - 1) >> 1) - (o >> 1) + 1 + ((o >> 1) & wmask)) + wmask) & ~wmask


def aligned_run_slots(o: int, cnt: int) -> int:
    """Virtual slots of the run [o, o + cnt) in the aligned write-out (compute_slots with KV > K): a front pad of o mod 32
    rows, rounded up to 32."""
    return (o % 32 + cnt + 31) & ~31 if cnt else 0


def run_starts(cnt: np.ndarray, base) -> np.ndarray:
    """o[t][p] = base[p] + rows of destination p in tiles before t: the first output row of every tile's run."""
    cnt = np.asarray(cnt, dtype=np.int64)
    o = np.zeros_like(cnt)
    o[1:] = np.cumsum(cnt, axis=0)[:-1]
    return o + np.asarray(base, dtype=np.int64)[None, :]


def tile_slots(cnt: np.ndarray, base, N: int, aligned: bool = False) -> np.ndarray:
    """Write-out slots each tile uses: pairs (local single-pass) or aligned virtual rows."""
    o = run_starts(cnt, base)
    f = (lambda a, c: aligned_run_slots(a, c)) if aligned else (lambda a, c: onepass_run_pairs(a, c, N))
    return np.array([sum(f(int(o[t, p]), int(cnt[t, p])) for p in range(N)) for t in range(len(cnt))], dtype=np.int64)


def _slot_modulus(N: int, aligned: bool) -> int:
    """Slots of a run depend on its start and count only modulo this (counts c and c + M differ by a whole number of
    32-pair or 32-row spans)."""
    return 32 if aligned else (64 if N <= PAIR_ALIGN_MAX_N else 2)


def _best_residues(score: np.ndarray, rows: int, M: int, exact: bool):
    """r[p] in 1..M maximising sum score[p][r - 1], with sum r <= rows and, if `exact`, sum r = rows (mod M): the rest
    of the tile's rows then go out in whole blocks of M rows (a dynamic programme over the sum of r)."""
    N = len(score)
    neg = -1e18
    dp = np.full(N * M + 1, neg)
    dp[0] = 0.0
    choice = np.zeros((N, N * M + 1), dtype=np.int64)
    for p in range(N):
        new = np.full_like(dp, neg)
        for r in range(1, M + 1):
            cand = np.full_like(dp, neg)
            cand[r:] = dp[:-r] + score[p][r - 1]
            better = cand > new
            new[better] = cand[better]
            choice[p][better] = r
        dp = new
    sums = np.arange(len(dp))
    ok = (sums <= rows) & ((sums % M == rows % M) if exact else True)
    s = int(np.argmax(np.where(ok, dp, neg)))
    r = np.zeros(N, dtype=np.int64)
    for p in reversed(range(N)):
        r[p] = choice[p][s]
        s -= r[p]
    return r


def _spread(r: np.ndarray, rows: int, M: int) -> np.ndarray:
    """Counts r + M * k summing to `rows`: the blocks go round-robin from destination 0."""
    blocks, N = (rows - int(r.sum())) // M, len(r)
    assert blocks >= 0 and int(r.sum()) + blocks * M == rows
    return r + M * (blocks // N + (np.arange(N) < blocks % N))


def _lead_destination_0(cnt: np.ndarray, M: int, margin: int) -> np.ndarray:
    """Move whole blocks of M rows (run-start residues unchanged) from other destinations to destination 0 until its
    total exceeds every other by at least `margin` rows."""
    cnt = cnt.copy()
    while True:
        tot = cnt.sum(axis=0)
        q = int(np.argmax(tot[1:])) + 1 if cnt.shape[1] > 1 else 0
        if q == 0 or tot[0] >= tot[q] + margin:
            return cnt
        t = int(np.argmax(cnt[:, q]))
        assert cnt[t, q] > M, "no block left to move"
        cnt[t, q] -= M
        cnt[t, 0] += M


def worst_case_counts(N: int, T: int, full_tiles: int, base, aligned: bool = False) -> np.ndarray:
    """cnt[tile][p] for `full_tiles` tiles of T rows and a ragged last tile, built to fill the write-out slots: tiles
    alternate between setting the run starts (as many as the row sum allows reach o = M - 1 mod M: o = 63 mod 64, a full
    31-pair front pad and an odd start, for the local pairs at N <= 16; o odd above that; o = 31 mod 32 for the aligned
    write-out) and spending them (counts that maximise the slots; at o = 63 that is a count = 2 mod 64, which pays the
    full round-up too).  Tile 0 starts at `base` and always sets; the ragged last tile always spends, with as many rows
    (<= T) as its best counts allow.  Destination 0 ends with the largest total.  Every choice is exhaustive over the
    residues, so each tile takes the most slots its start residues and row count permit."""
    M = _slot_modulus(N, aligned)
    slots = (lambda o, c: aligned_run_slots(o, c)) if aligned else (lambda o, c: onepass_run_pairs(o, c, N))
    per_row = 1.0 if aligned else 0.5
    o = np.asarray(base, dtype=np.int64) % M
    rows_out = []
    for t in range(full_tiles + 1):
        last = t == full_tiles
        spend = last or (t > 0 and (full_tiles - t) % 2 == 0)
        score = np.zeros((N, M))
        for p in range(N):
            for r in range(1, M + 1):
                score[p][r - 1] = slots(int(o[p]) + M, r) - per_row * r  # (+ M: a start past 0, same residues)
                if not spend:
                    score[p][r - 1] += 1000.0 * ((o[p] + r) % M == M - 1)
        r = _best_residues(score, T, M, exact=not last)
        rows = T if not last else int(r.sum()) + (T - int(r.sum())) // M * M
        rows_out.append(_spread(r, rows, M))
        o = (o + r) % M
    return _lead_destination_0(np.array(rows_out, dtype=np.int64), M, 2 * M)


def residue_sweep_counts(N: int, T: int, base, end0: int, M: int = 64) -> np.ndarray:
    """cnt[tile][p] under which every destination's run starts at every residue mod M in some tile: each full tile lets
    all destinations but one (in turn) move to a residue they have not started at yet, the remaining one takes what the
    row sum leaves.  A ragged last tile makes destination 0's total = end0 (mod M), and destination 0 ends with the
    largest total."""
    base = np.asarray(base, dtype=np.int64)
    o, seen, rows_out = base % M, [set() for _ in range(N)], []
    while True:
        for p in range(N):
            seen[p].add(int(o[p]))
        if all(len(s) == M for s in seen) or len(rows_out) > 4 * M:
            break
        forced = len(rows_out) % N
        r = np.zeros(N, dtype=np.int64)
        for p in range(N):
            if p != forced:
                want = min(set(range(M)) - seen[p], default=int(o[p]) + 1)
                r[p] = (want - o[p]) % M or M
        r[forced] = (T - int(r.sum())) % M or M
        rows_out.append(_spread(r, T, M))
        o = (o + r) % M
    r = np.ones(N, dtype=np.int64)
    r[0] = (end0 - sum(int(c[0]) for c in rows_out)) % M or M
    rows_out.append(_spread(r, int(r.sum()) + (T - int(r.sum())) // M * M, M))
    return _lead_destination_0(np.array(rows_out, dtype=np.int64), M, 2 * M)


def region_construction(make, N: int, delta: int, M: int):
    """(cnt, region_rows) with region_rows = destination 0's total (the largest) + delta, where `make(base_residues)` builds
    the counts against run starts p * region_rows: only region_rows mod M matters, so each residue is tried until the
    counts it gives agree with it."""
    tried = []
    for r0 in sorted(range(M), key=lambda r: (r - 1 - delta) % M):  # the usual answer first: a total of 1 (mod M)
        cnt = make([(p * r0) % M for p in range(N)])
        rr = int(cnt[:, 0].sum()) + delta
        if rr % M == r0:
            return cnt, rr
        tried.append(r0)
    raise AssertionError(f"no consistent region size for N={N}, delta={delta}")


def keys_for_counts(cnt: np.ndarray, dest_of_pool: np.ndarray, seed: int) -> np.ndarray:
    """Pool indices, one per row, such that tile t holds cnt[t][p] rows whose dest_of_pool is p, shuffled within the tile
    (so the rank of a row is not its position).  Each row is drawn at random from the pool entries of its destination."""
    rng = np.random.Generator(np.random.PCG64(seed))
    pools = [np.nonzero(dest_of_pool == p)[0] for p in range(cnt.shape[1])]
    assert all(len(q) for q in pools), "a destination no key of the pool reaches"
    out = []
    for row in cnt:
        tile = np.concatenate([rng.choice(pools[p], int(c)) for p, c in enumerate(row)] + [np.zeros(0, dtype=np.int64)])
        rng.shuffle(tile)
        out.append(tile)
    return np.concatenate(out).astype(np.int64)


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
