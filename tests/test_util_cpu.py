"""CPU checks of the test helpers that other tests build their inputs from: the tile geometry the edge sizes derive from,
and the crafted PartialReduce group keys that all hash to one slot."""
import random

import numpy as np

from tests.util import (M64, REDUCE_HASH_SEED, edge_sizes, keys_on_slot, mix64, reduce_slot_of_i64_key, reduce_table_slots,
                        tile_geometry, unmix64)


def test_tile_geometry_defaults_and_overrides():
    assert tile_geometry({}) == (256 * 6, 256 * 10)
    assert tile_geometry({"DFD_NVCC_DEFS": "-DDFD_TILE_THREADS=128 -DDFD_TILE_K=4 -DDFD_TILE_MIN_CTAS=8"}) == (128 * 4, 128 * 10)
    assert tile_geometry({"DFD_NVCC_DEFS": "-DDFD_ONEPASS_K=8"}) == (256 * 6, 256 * 8)
    assert tile_geometry({"DFD_NVCC_DEFS_ONEPASS": "-DDFD_ONEPASS_K=12 -DDFD_ONEPASS_NB=3"}) == (256 * 6, 256 * 12)
    sizes = set(edge_sizes({}))
    assert {1535, 1536, 1537, 3072, 3073, 2559, 2560, 2561, 5120, 5121} <= sizes and {0, 1, 31, 32, 33, 2047, 2048, 2049} <= sizes
    assert {511, 512, 513, 1024, 1025} <= set(edge_sizes({"DFD_NVCC_DEFS": "-DDFD_TILE_THREADS=128 -DDFD_TILE_K=4"}))


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


def test_crafted_reduce_keys_all_land_on_the_last_slot():
    n_keys, reps = 3000, 3
    slots = reduce_table_slots(n_keys * reps)
    assert slots == 32768 and reduce_table_slots(1) == 64 and reduce_table_slots(32) == 64 and reduce_table_slots(33) == 128
    keys = keys_on_slot(n_keys, slots - 1, slots, seed=9)
    assert len(set(keys.tolist())) == n_keys
    for k in keys.tolist():
        assert reduce_slot_of_i64_key(k, slots) == slots - 1
        assert mix64(REDUCE_HASH_SEED ^ (k & M64)) & (slots - 1) == slots - 1
