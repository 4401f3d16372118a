"""GPU parity tests of the single-pass kernel at the edges of its sub-tile ring items: every column of a tile arrives as
S items of T / S rows (2S for 16-byte columns), so a ragged last tile can end inside, exactly at, or one row past any of
those ranges, and some items of the last tile are empty.  Bar: bit-exact per destination, including row order."""
import os
import re

import numpy as np
import pyarrow as pa
import pytest

from tests.test_onepass_gpu import check_against_oracle
from tests.util import LAUNCH_HEADER, cfg2_columns, tile_geometry

pytestmark = pytest.mark.gpu


def onepass_split(env=None):
    """S (ring items per column of a tile) as build.py compiles it: the default of csrc/dfd_launch.cuh, or the
    -DDFD_ONEPASS_SPLIT= option of DFD_NVCC_DEFS_ONEPASS."""
    env = os.environ if env is None else env
    with open(LAUNCH_HEADER) as f:
        s = int(re.search(r"#define\s+DFD_ONEPASS_SPLIT\s+(\d+)", f.read()).group(1))
    m = re.search(r"-DDFD_ONEPASS_SPLIT=(\d+)", env.get("DFD_NVCC_DEFS_ONEPASS", ""))
    return int(m.group(1)) if m else s


def subtile_edge_sizes():
    """Row counts whose last tile ends at or one row either side of every sub-item boundary, for 8-byte items (T / S rows)
    and for the half-size items of 16-byte columns (T / 2S rows), in a single-tile and in a three-tile table."""
    t = tile_geometry()[1]
    step = t // (2 * onepass_split())
    sizes = set()
    for tiles in (0, 2):
        for b in range(1, t // step + 1):
            edge = tiles * t + b * step
            sizes |= {edge - 1, edge, edge + 1}
    return sorted(sizes)


@pytest.mark.parametrize("n_rows", subtile_edge_sizes())
def test_onepass_subtile_edges(ctx, n_rows):
    check_against_oracle(ctx, cfg2_columns(n_rows, 3), [0], 8)


@pytest.mark.parametrize("n_rows", [r for r in subtile_edge_sizes() if r > tile_geometry()[1]][::3])
def test_onepass_subtile_edges_mixed_widths(ctx, n_rows):
    # one launch moves 1-, 4-, 8- and 16-byte columns: each width's items split the tile at its own boundaries
    rng = np.random.Generator(np.random.PCG64(n_rows))
    key = rng.integers(-(2**63), 2**63 - 1, n_rows, dtype=np.int64)
    c8 = pa.array(rng.integers(0, 255, n_rows, dtype=np.uint8))
    c32 = pa.array(rng.integers(-(2**31), 2**31 - 1, n_rows, dtype=np.int32))
    raw = rng.integers(0, 255, n_rows * 16, dtype=np.uint8).tobytes()
    dec = pa.Array.from_buffers(pa.decimal128(38, 0), n_rows, [None, pa.py_buffer(raw)])
    for N in (8, 48):
        check_against_oracle(ctx, [key, c8, c32, dec], [0], N)
