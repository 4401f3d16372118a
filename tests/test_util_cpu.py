"""CPU checks of the test helpers that other tests build their inputs from: the tile geometry the edge sizes derive from,
the destination tables and row limits of the 32-bit limit tests, and the crafted PartialReduce group keys that all hash
to one slot."""
import random

import numpy as np

from tests.util import (M64, PARTITION_MAX_ROWS, REDUCE_HASH_SEED, REDUCE_MAX_ROWS, ScatterInst, dest_lut, domain_values, edge_sizes,
                        keys_on_slot, mix64, onepass_regions_accepted, parse_scatter_name, reduce_slot_of_i64_key, reduce_table_slots,
                        scatter_inst, scatter_instances, tile_geometry, unmix64, use_aligned)


def test_tile_geometry_defaults_and_overrides():
    assert tile_geometry({}) == (256 * 6, 256 * 10)
    assert tile_geometry({"DFD_NVCC_DEFS": "-DDFD_TILE_THREADS=128 -DDFD_TILE_K=4 -DDFD_TILE_MIN_CTAS=8"}) == (128 * 4, 128 * 10)
    assert tile_geometry({"DFD_NVCC_DEFS": "-DDFD_ONEPASS_K=8"}) == (256 * 6, 256 * 8)
    assert tile_geometry({"DFD_NVCC_DEFS_ONEPASS": "-DDFD_ONEPASS_K=12 -DDFD_ONEPASS_NB=3"}) == (256 * 6, 256 * 12)
    sizes = set(edge_sizes({}))
    assert {1535, 1536, 1537, 3072, 3073, 2559, 2560, 2561, 5120, 5121} <= sizes and {0, 1, 31, 32, 33, 2047, 2048, 2049} <= sizes
    assert {511, 512, 513, 1024, 1025} <= set(edge_sizes({"DFD_NVCC_DEFS": "-DDFD_TILE_THREADS=128 -DDFD_TILE_K=4"}))


def test_scatter_kernel_names_parse_in_every_demangler_format():
    """cu++filt (the library's symbol table) and the GNU demangler (profiler kernel names) spell template arguments
    differently; both, and the mangled name, give the same instantiation."""
    want = ScatterInst("k_scatter_onepass", 10, 14, True, "u32", True)
    assert parse_scatter_name("void dfd::k_scatter_onepass<(int)256, (int)10, (int)14, (int)3, (int)1, (int)3, (bool)1, unsigned int, "
                              "(bool)1>(dfd::ScatterParams)") == want
    assert parse_scatter_name("void dfd::k_scatter_onepass<256, 10, 14, 3, 1, 3, true, unsigned int, true>(dfd::ScatterParams)") == want
    assert scatter_instances(["_ZN3dfd17k_scatter_onepassILi256ELi10ELi14ELi3ELi1ELi3ELb1EjLb1EEEvNS_13ScatterParamsE", "k_scan_tiles"]) == {want}
    assert parse_scatter_name("void dfd::k_scatter<256, 6, 10, 6, false, dfd::BitColumn, false>(dfd::ScatterParams)") == \
        ScatterInst("k_scatter", 6, 10, False, "bit", False)
    assert parse_scatter_name("void dfd::k_scatter<(int)256, (int)10, (int)10, (int)4, (bool)0, uint4, (bool)1>(dfd::ScatterParams)") == \
        ScatterInst("k_scatter", 10, 10, False, "uint4", True)
    assert parse_scatter_name("void dfd::k_tile_hist<256, 6, true, 2>(dfd::KeySet, unsigned int)") is None
    # the dispatch restatement names instantiations the same way
    assert scatter_inst(1, True, "u32", True, True, {}) == want
    assert scatter_inst(0, False, "bit", False, True, {}) == ScatterInst("k_scatter", 6, 10, False, "bit", False)
    assert scatter_inst(2, False, "u8", True, True, {}) == ScatterInst("k_scatter", 10, 14, False, "u8", True)
    assert use_aligned(16, True) and not use_aligned(17, True) and not use_aligned(8, False)


def test_mix64_matches_the_murmur_finaliser_and_inverts():
    rnd = random.Random(3)
    xs = [0, 1, M64, 1 << 63] + [rnd.getrandbits(64) for _ in range(2000)]
    # the same finaliser in wrapping uint64 arithmetic, as the device computes it
    v = np.array(xs, dtype=np.uint64)
    with np.errstate(over="ignore"):
        v ^= v >> np.uint64(33)
        v *= np.uint64(0xFF51AFD7ED558CCD)
        v ^= v >> np.uint64(33)
        v *= np.uint64(0xC4CEB9FE1A85EC53)
        v ^= v >> np.uint64(33)
    assert [mix64(x) for x in xs] == v.tolist()
    for x in xs:
        assert unmix64(mix64(x)) == x and mix64(unmix64(x)) == x


def test_limit_luts_match_the_python_oracle_for_every_domain_value():
    """The destination tables of the limit tests (C oracle) against the pure-Python ahash restatement, for every key of
    each domain at each partition count the tests use; a null key goes to destination 0."""
    from oracle import oracle_py

    for kind, width, Ns in (("u8", 1, (2, 7)), ("i16", 2, (3, 4, 5)), ("i64", 8, (8,))):
        vals = domain_values(kind)
        assert len(set(vals.tolist())) == len(vals) == (256 if kind == "u8" else 1 << 16)
        hashes = [oracle_py.hash_one_int(int(v), width) for v in vals]
        for N in Ns:
            lut = dest_lut(kind, N)
            assert lut.tolist() == [h % N for h in hashes], (kind, N)
            assert set(lut.tolist()) == set(range(N)), (kind, N)  # every destination is reachable
    assert oracle_py.create_hashes([("int", 1, [None])], 1) == [0]
    assert domain_values("i16")[0x8000] == -(1 << 15) and domain_values("i16")[0xFFFF] == -1  # index = the value's bits


def test_row_limits_of_the_abi():
    """The row-count checks the limit tests cross, restated: dense calls take up to 2^32 - 1 rows; single-pass regions
    need N * region_rows < 2^32 - 1, so 3 x 1 431 655 764 = 2^32 - 4 and 2 x (2^31 - 1) = 2^32 - 2 (the largest accepted
    product) pass and any product of 2^32 - 1 or more is refused; PartialReduce takes up to 2^31 rows, whose group table
    of 2^32 slots is the most a u32 mask addresses."""
    assert PARTITION_MAX_ROWS == 0xFFFFFFFF
    assert 3 * 1_431_655_764 == (1 << 32) - 4 and onepass_regions_accepted(1_431_655_764, 3, 3_900_000_000)
    assert 2 * ((1 << 31) - 1) == (1 << 32) - 2 and onepass_regions_accepted((1 << 31) - 1, 2, (1 << 32) - 3)
    assert not onepass_regions_accepted(1_431_655_765, 3, 64) and 3 * 1_431_655_765 == (1 << 32) - 1
    assert not onepass_regions_accepted((1 << 32) - 1, 1, 64) and not onepass_regions_accepted(1 << 31, 2, 64)
    assert not onepass_regions_accepted(1_431_655_764, 3, (1 << 32) - 3)  # too small for the rows
    # the largest accepted product, over every partition count a single-pass call takes
    for N in range(1, 257):
        best = ((1 << 32) - 2) // N
        assert onepass_regions_accepted(best, N, 1) and not onepass_regions_accepted(best + 1, N, 1)
    assert reduce_table_slots(REDUCE_MAX_ROWS) == 1 << 32 and reduce_table_slots(REDUCE_MAX_ROWS + 1) == 1 << 33
    assert reduce_table_slots(REDUCE_MAX_ROWS) - 1 == 0xFFFFFFFF  # the table mask still fits 32 bits


def test_crafted_reduce_keys_all_land_on_the_last_slot():
    n_keys, reps = 3000, 3
    slots = reduce_table_slots(n_keys * reps)
    assert slots == 32768 and reduce_table_slots(1) == 64 and reduce_table_slots(32) == 64 and reduce_table_slots(33) == 128
    keys = keys_on_slot(n_keys, slots - 1, slots, seed=9)
    assert len(set(keys.tolist())) == n_keys
    for k in keys.tolist():
        assert reduce_slot_of_i64_key(k, slots) == slots - 1
        assert mix64(REDUCE_HASH_SEED ^ (k & M64)) & (slots - 1) == slots - 1


def test_constructed_destination_runs_reach_the_slot_bounds():
    """The single-pass layout constructions: every tile gives its intended counts under the destination table, and the
    restated pair and slot totals reach the bounds the write-out caps are sized for.  T = 2560 (the default tiling)."""
    from tests.util import (aligned_run_slots, keys_for_counts, onepass_run_pairs, region_construction, residue_sweep_counts,
                            run_starts, tile_slots, worst_case_counts)

    T = 2560
    # the run restatements on hand-checked runs: o = 63, count 2 pays a 31-pair front pad, 2 pairs and a 31-pair round up
    assert onepass_run_pairs(63, 2, 16) == 64 and onepass_run_pairs(64, 2, 16) == 32 and onepass_run_pairs(5, 0, 16) == 0
    assert onepass_run_pairs(63, 2, 17) == 2 and onepass_run_pairs(62, 2, 17) == 1 and onepass_run_pairs(1, 3, 256) == 2
    assert aligned_run_slots(31, 2) == 64 and aligned_run_slots(32, 2) == 32 and aligned_run_slots(7, 0) == 0
    for N, kind in ((16, "i64"), (8, "i16"), (17, "i64"), (256, "i16")):
        M = 64 if N <= 16 else 2
        lut = dest_lut(kind, N)
        for delta in (1, 0, 31, -1):
            cnt, rr = region_construction(lambda b: worst_case_counts(N, T, 3, b), N, delta, M)
            tot = cnt.sum(axis=0)
            assert rr == tot.max() + delta and tot[0] == tot.max() and (tot.sum() <= rr * N)
            assert (cnt[:-1].sum(axis=1) == T).all() and 0 < cnt[-1].sum() <= T and (cnt >= 1).all()
            idx = keys_for_counts(cnt, lut, seed=N + delta)
            starts = np.concatenate([[0], np.cumsum(cnt.sum(axis=1))])
            for t in range(len(cnt)):
                assert np.array_equal(np.bincount(lut[idx[starts[t]:starts[t + 1]]], minlength=N), cnt[t]), (N, delta, t)
            pairs = tile_slots(cnt, np.arange(N) * rr, N)
            rows = cnt.sum(axis=1)
            if N == 16 and delta == 1:
                # every run of the ragged last tile starts at 63 (mod 64) with a count of 2 (mod 64): exactly rows / 2 + 63 N
                o = run_starts(cnt, np.arange(N) * rr)
                assert (o[-1] % 64 == 63).all() and (cnt[-1] % 64 == 2).all()
                assert rows[-1] == 2528 and pairs[-1] == rows[-1] // 2 + 63 * N == 2272
            if N <= 16:
                assert pairs.max() >= T // 2 + 63 * N - 63 and (pairs <= rows // 2 + 63 * N).all()
            elif N == 256:
                assert (pairs[1:] == T // 2 + N).all()  # every run odd-started with an even count
            else:  # N = 17: full tiles keep the parity of the sum of the starts, so one run of 17 starts even
                assert (pairs[1:-1] == T // 2 + N - 1).all()
            assert (pairs <= (T // 2 + 63 * 16 + 255) // 256 * 256).all()  # within the KP cap of the default build
    # the aligned write-out of a peer launch: sub-windows of 32-row multiples, full tiles reach T + 62 N less one run's pad
    cnt = worst_case_counts(16, T, 3, [0] * 16, aligned=True)
    slots = tile_slots(cnt, np.arange(16) * 4096, 16, aligned=True)
    assert slots[1] == T + 62 * 16 - 32 and (slots <= T + 62 * 16).all()
    # every run start residue mod 64, for every destination
    for N in (3, 8):
        cnt, rr = region_construction(lambda b: residue_sweep_counts(N, T, b, (1 - 0) % 64), N, 0, 64)
        o = run_starts(cnt, np.arange(N) * rr) % 64
        assert all(set(o[:, p].tolist()) == set(range(64)) for p in range(N))
        idx = keys_for_counts(cnt, dest_lut("i64", N), seed=N)
        assert np.array_equal(np.bincount(dest_lut("i64", N)[idx], minlength=N), cnt.sum(axis=0))
