"""CPU tests of the PartialReduce's Boolean and var-width group keys: the exact Python group-by the GPU tests compare with
(checked here on constructed edge cases), the restated string hash of dfd_reduce.cu, the header's statement of the new
output contract, and the binding's unchanged symbol list."""
import os
import re

import numpy as np

from tests.util import M64, REDUCE_HASH_SEED, ROOT, mix64

NULL_KEY_TAG = 0x6A09E667F3BCC909  # dfd_reduce.cu: hashed in place of a null key


def reference_group_by(keys, states, ops, rows):
    """{key tuple: [merged state per state column]} of `rows`.  keys[k] is a list of Python values (bytes / bool / int, or
    None for a null key); a null equals a null of its column and nothing else.  states[j] is an int64 array merged by
    ops[j]: "count", "sum" (wrapping mod 2^64, as SUM_I64), "min" or "max"."""
    groups = {}
    for r in rows:
        groups.setdefault(tuple(k[r] for k in keys), []).append(r)
    out = {}
    for key, rs in groups.items():
        merged = []
        for s, op in zip(states, ops):
            v = [int(s[r]) for r in rs]
            if op == "count":
                merged.append(len(v))
            elif op == "sum":
                t = sum(v) & M64
                merged.append(t - (1 << 64) if t >> 63 else t)
            else:
                merged.append(min(v) if op == "min" else max(v))
        out[key] = merged
    return out


def string_key_hash(keys):
    """dfd_reduce.cu key_hash over KeyParams for one row: per key, a null mixes NULL_KEY_TAG; bytes mix their length, then
    each 8-byte little-endian chunk (the last zero-padded); a Boolean mixes 0 / 1; an int mixes its width's bits."""
    h = REDUCE_HASH_SEED
    for k in keys:
        if k is None:
            h = mix64(h ^ NULL_KEY_TAG)
        elif isinstance(k, (bytes, bytearray)):
            h = mix64(h ^ len(k))
            for i in range(0, len(k), 8):
                h = mix64(h ^ int.from_bytes(k[i:i + 8], "little"))
        elif isinstance(k, bool):
            h = mix64(h ^ int(k))
        else:
            raise TypeError(type(k))
    return h


def home_slot(keys, slots):
    return string_key_hash(keys) & 0xFFFFFFFF & (slots - 1)


def test_null_is_not_the_empty_string():
    k = [b"", None, b"", None, b"a", b"a\x00"]
    got = reference_group_by([k], [np.ones(6, dtype=np.int64)], ["count"], range(6))
    assert got == {(b"",): [2], (None,): [2], (b"a",): [1], (b"a\x00",): [1]}


def test_prefixes_are_distinct_groups():
    k = [b"abc", b"ab", b"a", b"", b"abc", b"abcd", b"ab"]
    got = reference_group_by([k], [np.arange(7, dtype=np.int64)], ["sum"], range(7))
    assert got == {(b"abc",): [4], (b"ab",): [7], (b"a",): [2], (b"",): [3], (b"abcd",): [5]}


def test_boolean_keys_with_nulls_make_three_groups():
    k = [True, None, False, True, None, False, False]
    v = np.array([5, -1, 3, 9, 7, 2, 8], dtype=np.int64)
    got = reference_group_by([k], [v, v], ["min", "max"], range(7))
    assert got == {(True,): [5, 9], (None,): [-1, 7], (False,): [2, 8]}


def test_second_key_splits_groups_equal_in_the_first():
    k1 = [b"x", b"x", b"x", None, None]
    k2 = [False, True, False, None, True]
    got = reference_group_by([k1, k2], [np.ones(5, dtype=np.int64)], ["count"], range(5))
    assert got == {(b"x", False): [2], (b"x", True): [1], (None, None): [1], (None, True): [1]}


def test_restated_hash_mixes_the_length():
    assert len({string_key_hash([s]) for s in (b"", b"\x00", b"\x00" * 8, b"\x00" * 9)}) == 4
    assert string_key_hash([None]) != string_key_hash([b""])
    assert string_key_hash([True]) != string_key_hash([False])


def _reduce_block():
    text = open(os.path.join(ROOT, "include", "dfd_b200.h")).read()
    return text[text.index("device-side PartialReduce ahead of the shuffle"):text.index("typedef enum {\n    DFD_AGG_SUM_I64")]


def test_header_states_the_key_contract():
    block = " ".join(re.sub(r"\n \*", " ", _reduce_block()).split())  # (the comment's lines joined)
    for phrase in ("DFD_COL_UTF8", "DFD_COL_LARGE_UTF8", "DFD_COL_BINARY", "DFD_COL_BOOL", "n_rows + 1 entries",
                   "values_bytes", "DFD_ERR_CAPACITY", "before any output", "ceil(n_rows / 32) * 4",
                   "+ 4 per var-width key", "state column", "DFD_ERR_UNSUPPORTED"):
        assert phrase in block, phrase
    assert "Fixed-width non-null keys and states" not in block
    assert "5 when a MIN / MAX" in _reduce_block()


def test_source_keeps_the_fixed_key_launches_and_adds_the_key_kernels():
    src = open(os.path.join(ROOT, "datafusion_distributed_b200", "csrc", "dfd_reduce.cu")).read()
    assert len(re.findall(r"const unsigned grid = \(unsigned\)\(c->sm_count \* 8\);", src)) == 1
    for k in ("k_group_insert", "k_group_count", "k_group_place", "k_group_combine"):
        assert len(re.findall(rf"\b{k}<<<grid, 256,", src)) == 1, k
        assert len(re.findall(rf"__launch_bounds__\(256\) {k}\b", src)) == 1, k
    for k in ("k_insert_keys", "k_count_keys", "k_place_keys", "k_copy_key_bytes"):
        assert re.search(rf"__launch_bounds__\(256\) {k}\b", src), k


def test_binding_symbols_are_unchanged():
    from datafusion_distributed_b200 import _native as nv

    # the same one reduce entry point with its 12 arguments, no other reduce symbol, and the 27 ops
    assert [s for s in nv.SIGNATURES if "reduce" in s] == ["dfd_partial_reduce_device"]
    assert len(nv.SIGNATURES["dfd_partial_reduce_device"][1]) == 12
    text = open(os.path.join(ROOT, "include", "dfd_b200.h")).read()
    assert [s for s in re.findall(r"\b(dfd_\w+)\s*\(", text) if "reduce" in s] == ["dfd_partial_reduce_device"]
    assert len([n for n in dir(nv) if n.startswith("AGG_")]) == 27
