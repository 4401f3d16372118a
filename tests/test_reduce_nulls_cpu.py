"""The null-aware exact reference of the device PartialReduce that test_reduce_nulls_gpu.py compares against, checked here
against pyarrow's group_by (NULL keys form one group; an all-null SUM / MIN / MAX is null), and the header's statement
of the nullable contract.

The reference works on numpy columns as the device reads them: integers as their type, floats as bit patterns (the
SUM_F64 state as float64), 128-bit decimals as (n, 2) int64 (low half first).  Every null is given by a bool array (True =
valid) beside its column; the bytes under a null are never read."""
import os
import re
from decimal import Decimal

import numpy as np
import pyarrow as pa
import pytest

from datafusion_distributed_b200 import _native as nv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1

# op -> (numpy dtype of the state column, how it merges)
OP_KIND = {
    nv.AGG_SUM_I64: (np.int64, "sum"), nv.AGG_SUM_F64: (np.float64, "sum_f64"), nv.AGG_SUM_I128: (np.int64, "sum_i128"),
    nv.AGG_MIN_I64: (np.int64, "int"), nv.AGG_MAX_I64: (np.int64, "int"), nv.AGG_MIN_F64: (np.uint64, "float"),
    nv.AGG_MAX_F64: (np.uint64, "float"),
    nv.AGG_MIN_I32: (np.int32, "int"), nv.AGG_MAX_I32: (np.int32, "int"), nv.AGG_MIN_I16: (np.int16, "int"),
    nv.AGG_MAX_I16: (np.int16, "int"), nv.AGG_MIN_I8: (np.int8, "int"), nv.AGG_MAX_I8: (np.int8, "int"),
    nv.AGG_MIN_U64: (np.uint64, "int"), nv.AGG_MAX_U64: (np.uint64, "int"), nv.AGG_MIN_U32: (np.uint32, "int"),
    nv.AGG_MAX_U32: (np.uint32, "int"), nv.AGG_MIN_U16: (np.uint16, "int"), nv.AGG_MAX_U16: (np.uint16, "int"),
    nv.AGG_MIN_U8: (np.uint8, "int"), nv.AGG_MAX_U8: (np.uint8, "int"), nv.AGG_MIN_I128: (np.int64, "i128"),
    nv.AGG_MAX_I128: (np.int64, "i128"), nv.AGG_MIN_F32: (np.uint32, "float"), nv.AGG_MAX_F32: (np.uint32, "float"),
    nv.AGG_MIN_F16: (np.uint16, "float"), nv.AGG_MAX_F16: (np.uint16, "float"),
}
ALL_OPS = sorted(OP_KIND)
MINMAX_OPS = [op for op in ALL_OPS if OP_KIND[op][1] not in ("sum", "sum_f64", "sum_i128")]


def is_max(op):
    return op in (nv.AGG_MAX_I64, nv.AGG_MAX_F64) or (op >= nv.AGG_MIN_I32 and (op - nv.AGG_MIN_I32) % 2 == 1)


def is_wide(op):
    return OP_KIND[op][1] in ("sum_i128", "i128")


def sentinel(op):
    """The value a MIN / MAX can never lose to (MIN: the top of the op's order, MAX: the bottom), as one element of the
    state column: the value the device starts a state from when its group's first row is null."""
    dt, kind = OP_KIND[op]
    if kind == "i128":
        return np.array([-1, (1 << 63) - 1] if not is_max(op) else [0, -(1 << 63)], dtype=np.int64)
    if kind == "float":
        w = 8 * np.dtype(dt).itemsize
        return dt((1 << (w - 1)) - 1 if not is_max(op) else (1 << w) - 1)
    info = np.iinfo(dt)
    return dt(info.min if is_max(op) else info.max)


def _total_order(bits):
    """totalOrder keys of float bit patterns (an unsigned array), as signed integers of the same width."""
    w = 8 * bits.dtype.itemsize
    s = bits.view(f"i{w // 8}")
    return s ^ ((s >> (w - 1)) & ((1 << (w - 1)) - 1)).astype(s.dtype)


def reduce_state(op, col, valid, gid, n_groups):
    """Merge one state column by group id: -> (values[n_groups] (zero under nulls), valid[n_groups]).  Only the valid
    rows count; a group without one is null."""
    dt, kind = OP_KIND[op]
    rows = np.nonzero(valid)[0] if valid is not None else np.arange(len(gid))
    g = gid[rows]
    order = np.argsort(g, kind="stable")
    rows, g = rows[order], g[order]
    present, seg = np.unique(g, return_index=True)
    out_valid = np.zeros(n_groups, dtype=bool)
    out_valid[present] = True
    out = np.zeros((n_groups, 2) if is_wide(op) else n_groups, dtype=np.int64 if is_wide(op) else dt)
    if len(rows) == 0:
        return out, out_valid
    red = np.maximum if is_max(op) else np.minimum
    c = col[rows]
    if kind == "sum":
        out[present] = np.add.reduceat(c.view(np.uint64), seg).view(np.int64)  # wraps mod 2^64
    elif kind == "sum_f64":
        out[present] = np.add.reduceat(c, seg) + 0.0  # (+0.0 + x: a group of -0.0 values sums to +0.0)
    elif kind == "sum_i128":
        lo, hi = c[:, 0].view(np.uint64), c[:, 1].view(np.uint64)
        limbs = [np.add.reduceat(x, seg).tolist() for x in (lo & 0xFFFFFFFF, lo >> 32, hi & 0xFFFFFFFF, hi >> 32)]
        tot = [(a + (b << 32) + (d << 64) + (e << 96)) & ((1 << 128) - 1) for a, b, d, e in zip(*limbs)]
        out[present, 0] = np.array([t & M64 for t in tot], dtype=np.uint64).view(np.int64)
        out[present, 1] = np.array([t >> 64 for t in tot], dtype=np.uint64).view(np.int64)
    elif kind == "i128":  # the signed high halves, then the unsigned low halves of the rows that hold the group's best high
        lo, hi = c[:, 0].view(np.uint64), c[:, 1]
        ghi = red.reduceat(hi, seg)
        on_top = hi == np.repeat(ghi, np.diff(np.append(seg, len(rows))))
        glo = red.reduceat(np.where(on_top, lo, np.uint64(0) if is_max(op) else np.uint64(M64)), seg)
        out[present, 0] = glo.view(np.int64)
        out[present, 1] = ghi
    elif kind == "float":
        k = red.reduceat(_total_order(c), seg)
        w = 8 * c.dtype.itemsize
        out[present] = (k ^ ((k >> (w - 1)) & ((1 << (w - 1)) - 1)).astype(k.dtype)).view(c.dtype)
    else:
        out[present] = red.reduceat(c, seg)
    return out, out_valid


def key_matrix(keys, key_valid):
    """One int64 row per input row that identifies its group: per key column its valid flag, then its value's 64-bit
    words, zero under a null (so the bytes there never count)."""
    parts = []
    for k, v in zip(keys, key_valid):
        valid = np.ones(len(k), dtype=bool) if v is None else v
        parts.append(valid.astype(np.int64)[:, None])
        words = k.astype(np.int64)[:, None] if k.ndim == 1 else k.astype(np.int64)
        parts.append(np.where(valid[:, None], words, 0))
    return np.concatenate(parts, axis=1)


def reference_reduce(keys, key_valid, states, state_valid, ops):
    """The null-aware exact PartialReduce of one partition.  keys / states: numpy columns; key_valid / state_valid: bool
    arrays or None (no nulls).  -> (group key matrix (key_matrix rows, one per group, sorted), [(values, valid)] per state
    column in that group order)."""
    m = key_matrix(keys, key_valid)
    groups, gid = np.unique(m, axis=0, return_inverse=True)
    gid = gid.reshape(-1)
    return groups, [reduce_state(op, c, v, gid, len(groups)) for op, c, v in zip(ops, states, state_valid)]


# ------------------------------------------------------------------- tests ----

def _i128_column(values):
    v = [x & ((1 << 128) - 1) for x in values]
    return np.stack([np.array([x & M64 for x in v], dtype=np.uint64).view(np.int64),
                     np.array([x >> 64 for x in v], dtype=np.uint64).view(np.int64)], axis=1)


def _i128_value(row):
    x = (int(np.uint64(row[1].view(np.uint64))) << 64) | int(row[0].view(np.uint64))
    return x - (1 << 128) if x >> 127 else x


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reference_matches_pyarrow_group_by(seed):
    """Int32 and Int64 nullable keys, Int64 and Decimal128 nullable states: SUM / MIN / MAX of the reference equal
    pyarrow's group_by aggregate, NULL key group and all-null results included.  Bytes under nulls are garbage."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n = 4000
    k1 = rng.integers(0, 20, n).astype(np.int32)
    k2 = rng.integers(-3, 3, n).astype(np.int64)
    kv1, kv2 = rng.random(n) > 0.2, rng.random(n) > 0.1
    s = rng.integers(-(10 ** 12), 10 ** 12, n).astype(np.int64)
    dec = [int(x) for x in rng.integers(-(10 ** 15), 10 ** 15, n)]
    # a share of rows in groups whose states are all null: every row of key (k1 = 19) has null states
    sv = (rng.random(n) > 0.5) & (k1 != 19)
    dv = (rng.random(n) > 0.3) & (k1 != 19)
    garbage = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
    k1g = np.where(kv1, k1, garbage.astype(np.int32))
    k2g = np.where(kv2, k2, garbage)
    sg = np.where(sv, s, garbage)
    dcol = _i128_column(dec)
    dcol[~dv] = np.stack([garbage, garbage[::-1]], axis=1)[~dv]

    table = pa.table({
        "k1": pa.array(k1, mask=~kv1), "k2": pa.array(k2, mask=~kv2), "s": pa.array(s, mask=~sv),
        "d": pa.array([Decimal(x) for x in dec], type=pa.decimal128(38, 0), mask=~dv),
    })
    aggs = [("s", "sum"), ("s", "min"), ("s", "max"), ("d", "sum"), ("d", "min"), ("d", "max")]
    got_pa = table.group_by(["k1", "k2"]).aggregate(aggs).to_pylist()
    want_pa = {(r["k1"], r["k2"]): tuple(r[f"{c}_{a}"] for c, a in aggs) for r in got_pa}

    ops = [nv.AGG_SUM_I64, nv.AGG_MIN_I64, nv.AGG_MAX_I64, nv.AGG_SUM_I128, nv.AGG_MIN_I128, nv.AGG_MAX_I128]
    states = [sg, sg, sg, dcol, dcol, dcol]
    groups, merged = reference_reduce([k1g, k2g], [kv1, kv2], states, [sv, sv, sv, dv, dv, dv], ops)
    assert len(groups) == len(want_pa)
    mine = {}
    for gi, row in enumerate(groups.tolist()):
        key = (row[1] if row[0] else None, row[3] if row[2] else None)
        vals = []
        for j, (vals_j, valid_j) in enumerate(merged):
            if not valid_j[gi]:
                vals.append(None)
                assert not vals_j[gi].any(), "the bytes of a null state are not zero"
            elif is_wide(ops[j]):
                vals.append(Decimal(_i128_value(vals_j[gi])))
            else:
                vals.append(int(vals_j[gi]))
        mine[key] = tuple(vals)
    assert mine == want_pa
    assert (None, None) in mine or not ((~kv1) & (~kv2)).any()
    assert any(v[0] is None for v in mine.values())  # the all-null state groups are there and null


def test_null_key_bytes_and_distinct_null_positions():
    """(NULL, 1), (1, NULL) and (NULL, NULL) are three groups, whatever bytes lie under the nulls."""
    k1 = np.array([7, 1, 9, 1, 5, 3], dtype=np.int64)
    v1 = np.array([False, True, False, True, False, False])
    k2 = np.array([1, 2, 1, 8, 6, 4], dtype=np.int64)
    v2 = np.array([True, False, True, False, False, False])
    groups, _ = reference_reduce([k1, k2], [v1, v2], [], [], [])
    assert groups.tolist() == [[0, 0, 0, 0], [0, 0, 1, 1], [1, 1, 0, 0]]


def test_header_states_the_nullable_contract():
    text = open(os.path.join(ROOT, "include", "dfd_b200.h")).read()
    block = text[text.index("device-side PartialReduce ahead of the shuffle"):text.index("typedef enum {\n    DFD_AGG_SUM_I64")]
    assert not re.search(r"nullable group keys\s*/\s*states:\s*DFD_ERR_UNSUPPORTED", block), "the old refusal is still stated"
    assert "Fixed-width non-null keys and states" not in block
    for phrase in ("out_cols[c].validity", "4-byte aligned", "ceil(n_rows / 32) * 4", "(NULL, NULL)", "5 when a MIN / MAX"):
        assert phrase in block, phrase
