"""CPU tests of the oracle itself (no GPU): C restatement vs the independent
pure-Python restatement, the committed golden vectors and SURVEY.md §8(c)."""
import random

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as orc
from oracle import oracle_py as op
from tests.util import cfg2_columns, golden, seed_tuples


def test_survey_8c_vectors():
    g = golden()
    for k, hx in g["survey_8c"].items():
        assert format(orc.hash_one_int(int(k), 8), "016x") == hx
        assert format(op.hash_one_int(int(k), 8), "016x") == hx
    tk = g["survey_8c_two_key"]
    h = orc.create_hashes([np.array([tk["c0"]], dtype=np.int64), np.array([tk["c1"]], dtype=np.int64)], 1)[0]
    assert format(int(h), "016x") == tk["hash"]
    assert int(h) % 8 == 5


def test_golden_ints_and_strings():
    g = golden()
    for e in g["ints"]:
        assert format(orc.hash_one_int(int(e["value"]), e["width"]), "016x") == e["hash"]
    for e in g["strings"]:
        s = bytes.fromhex(e["hex"])
        assert format(orc.hash_one_str(s), "016x") == e["str_hash"]
        assert format(orc.hash_one_bytes(s), "016x") == e["bytes_hash"]
    for e in g["seeded"]:
        assert format(orc.hash_one_int(int(e["value"]), 8, tuple(e["seeds"])), "016x") == e["hash"]


def test_golden_rows_multi_column_with_nulls():
    g = golden()
    rows = g["rows_i64_i32_utf8"]
    a = pa.array([None if r["i64"] is None else int(r["i64"]) for r in rows], type=pa.uint64())
    b = pa.array([None if r["i32"] is None else int(r["i32"]) for r in rows], type=pa.uint32())
    c = pa.array([None if r["utf8_hex"] is None else bytes.fromhex(r["utf8_hex"]) for r in rows], type=pa.binary())
    c = c.cast(pa.string(), safe=False) if False else pa.Array.from_buffers(pa.string(), len(c), c.buffers(), null_count=c.null_count)
    h = orc.create_hashes([a, b, c], len(rows))
    for i, r in enumerate(rows):
        assert format(int(h[i]), "016x") == r["hash"], i
        for n, m in r["mod"].items():
            assert int(h[i]) % int(n) == m


def test_c_matches_python_restatement_randomised():
    rnd = random.Random(5)
    n = 500
    a = [rnd.choice([None, rnd.getrandbits(63)]) for _ in range(n)]
    s = [rnd.choice([None, bytes(rnd.getrandbits(8) for _ in range(rnd.randint(0, 40)))]) for _ in range(n)]
    bl = [rnd.choice([None, True, False]) for _ in range(n)]
    d = [rnd.choice([None, rnd.getrandbits(15)]) for _ in range(n)]
    cols_c = [pa.array(a, type=pa.int64()), pa.array(s, type=pa.binary()), pa.array(bl), pa.array(d, type=pa.int16())]
    cols_p = [("int", 8, a), ("bytes", 0, s), ("bool", 1, bl), ("int", 2, d)]
    assert orc.create_hashes(cols_c, n).tolist() == op.create_hashes(cols_p, n)
    # sliced (offset != 0) arrays
    sl = [c.slice(17, 300) for c in cols_c]
    slp = [(k, w, v[17:317]) for k, w, v in cols_p]
    assert orc.create_hashes(sl, 300).tolist() == op.create_hashes(slp, 300)


@pytest.mark.parametrize("seeds", seed_tuples())
def test_c_matches_python_restatement_seeded(seeds):
    """The C oracle against the Python restatement under every seed tuple of the device hash tests: each column kind
    alone (integers of 1 to 16 bytes, Boolean, Utf8, Binary, LargeUtf8, intervals), three keys in all 8 null patterns,
    and the whole set sliced at Arrow offsets 1-7, 13 and 37."""
    import struct

    rnd = random.Random(sum(seeds) % 1009)
    st = op.with_seeds(*seeds)
    n = 240
    nullable = lambda v, j: [None if (i >> j) % 2 and j < 3 else x for i, x in enumerate(v)]  # keys 0-2: r % 8's null pattern
    ints = [(w, [rnd.getrandbits(8 * w) for _ in range(n)]) for w in (1, 2, 4, 8, 16)]
    raw = [bytes(rnd.getrandbits(8) for _ in range(rnd.choice([0, 1, 3, 7, 8, 9, 16, 17, 33, 70]))) for _ in range(n)]
    cols_p = [("str", 0, raw), ("bytes", 0, raw), ("bool", 1, [rnd.random() < 0.5 for _ in range(n)])]
    cols_p += [("int", w, v) for w, v in ints]
    cols_p += [("str", 0, [rnd.choice([None, b"", x]) for x in raw])]
    cols_p = [(k, w, nullable(v, j)) for j, (k, w, v) in enumerate(cols_p)]

    def to_arrow(kind, w, v, large=False):
        if kind == "bool":
            return pa.array(v, type=pa.bool_())
        if kind == "int" and w == 16:
            valid = np.array([x is not None for x in v])
            data = b"".join((x or 0).to_bytes(16, "little") for x in v)
            return pa.Array.from_buffers(pa.decimal128(38, 0), n, [pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()),
                                                                    pa.py_buffer(data)], null_count=int((~valid).sum()))
        if kind == "int":
            return pa.array(v, type={1: pa.uint8(), 2: pa.uint16(), 4: pa.uint32(), 8: pa.uint64()}[w])
        b = pa.array(v, type=pa.binary())
        if kind == "bytes":
            return b
        s = pa.Array.from_buffers(pa.string(), n, b.buffers(), null_count=b.null_count)
        return s.cast(pa.large_string()) if large else s

    cols_c = [to_arrow(*c) for c in cols_p]
    large = to_arrow("str", 0, cols_p[0][2], large=True)
    for c, p in [(large, cols_p[0])] + list(zip(cols_c, cols_p)):
        assert orc.create_hashes([c], n, seeds).tolist() == op.create_hashes([p], n, st), (p[0], p[1])
    assert orc.create_hashes(cols_c[:3], n, seeds).tolist() == op.create_hashes(cols_p[:3], n, st)
    for off in [1, 2, 3, 4, 5, 6, 7, 13, 37]:
        m = n - off - 3
        sl = [c.slice(off, m) for c in cols_c]
        slp = [(k, w, v[off:off + m]) for k, w, v in cols_p]
        assert orc.create_hashes(sl, m, seeds).tolist() == op.create_hashes(slp, m, st), off
    dt = [(rnd.getrandbits(32) - (1 << 31), rnd.getrandbits(32) - (1 << 31)) for _ in range(n)]
    mdn = [(rnd.getrandbits(32) - (1 << 31), rnd.getrandbits(32) - (1 << 31), rnd.getrandbits(64) - (1 << 63)) for _ in range(n)]
    h = orc.create_hashes([("interval_day_time", np.frombuffer(b"".join(struct.pack("<ii", *x) for x in dt), dtype=np.uint8))], n, seeds)
    assert h.tolist() == [op.hash_one_interval_day_time(*x, st=st) for x in dt]
    h = orc.create_hashes([("interval_month_day_nano", np.frombuffer(b"".join(struct.pack("<iiq", *x) for x in mdn), dtype=np.uint8))], n, seeds)
    assert h.tolist() == [op.hash_one_interval_month_day_nano(*x, st=st) for x in mdn]


def test_null_keys_keep_previous_hash():
    # invariant (v): a null key contributes nothing; all-null single key => hash 0 => partition 0
    a = pa.array([None, None, 5], type=pa.int64())
    h = orc.create_hashes([a], 3)
    assert h[0] == 0 and h[1] == 0 and h[2] == op.hash_one_int(5)
    b = pa.array([7, None, None], type=pa.int64())
    h2 = orc.create_hashes([a, b], 3)
    assert h2[0] == op.combine_hashes(op.hash_one_int(7), 0)
    assert h2[1] == 0
    assert h2[2] == op.hash_one_int(5)


def test_signed_ints_hash_as_same_width_unsigned():
    # i32 -1 hashes as 0x00000000ffffffff (not sign-extended)
    assert orc.hash_one_int(-1, 4) == op.hash_one_int(0xFFFFFFFF, 8)
    v = np.array([-1], dtype=np.int32)
    assert orc.create_hashes([v], 1)[0] == op.hash_one_int(0xFFFFFFFF, 8)


@pytest.mark.parametrize("N", [1, 2, 3, 8, 12, 48, 1000])
def test_repartition_table_properties(N):
    cols = cfg2_columns(50_000, 4)
    outs, counts, starts = orc.repartition_table(cols, [0], N, 1024, 1)
    dest = orc.partition_ids([cols[0]], len(cols[0]), N)
    assert counts.sum() == len(cols[0])
    for p in range(N):
        idx = np.nonzero(dest == p)[0]  # input order
        for c in range(len(cols)):
            assert np.array_equal(outs[c][starts[p]:starts[p + 1]], cols[c][idx])
    # consistency with the power-of-two invariant (vi): (h % (P*T)) % P == h % P
    if N % 4 == 0:
        dest4 = orc.partition_ids([cols[0]], len(cols[0]), 4)
        assert np.array_equal(dest % 4, dest4)


def test_repartition_table_multithreaded_is_same_row_set():
    cols = cfg2_columns(100_000, 3)
    o1, c1, s1 = orc.repartition_table(cols, [0], 8, 8192, 1)
    o4, c4, s4 = orc.repartition_table(cols, [0], 8, 8192, 4)
    assert np.array_equal(c1, c4)
    for p in range(8):
        a = np.sort(o1[1][s1[p]:s1[p + 1]])
        b = np.sort(o4[1][s4[p]:s4[p + 1]])
        assert np.array_equal(a, b)


def test_distribution_sanity():
    dest = orc.partition_ids([np.arange(100_000, dtype=np.int64)], 100_000, 8)
    counts = np.bincount(dest, minlength=8)
    assert counts.min() >= 12_300 and counts.max() <= 12_700


def test_flight_proxy_reference_arm_is_a_correct_shuffle():
    """The CPU+Flight stand-in used by `bench.py --impl reference --gpus N` delivers the right row sets."""
    import pyarrow as pa

    from oracle.flight_proxy import FlightShuffleProxy

    n, T, P = 30_000, 2, 4
    cols = cfg2_columns(n, 3)
    px = FlightShuffleProxy(["c0", "c1", "c2"], T, T, P, "lz4")
    try:
        prod = [[c[r * n // T:(r + 1) * n // T] for c in cols] for r in range(T)]
        dt, rows, tables = px.run(prod, 1)
        assert rows == n
        dest = orc.partition_ids([cols[0]], n, P * T)
        for ci in range(T):
            got = np.sort(pa.concat_tables(tables[ci]).column("c1").to_numpy())
            assert np.array_equal(got, np.sort(cols[1][(dest // P) == ci]))
    finally:
        px.close()


def test_interval_keys_hash_field_by_field():
    """Arrow's IntervalDayTime / IntervalMonthDayNano derive `Hash` (one write per field); DataFusion hashes them through
    that impl (hash_utils `hash_value!(.., IntervalDayTime, IntervalMonthDayNano)`), NOT as one 64/128-bit integer."""
    import struct

    from oracle import oracle_py as op

    g = golden()["intervals"]
    dt = [e for e in g if e["type"] == "day_time"]
    raw = b"".join(struct.pack("<ii", e["days"], e["millis"]) for e in dt)
    h = orc.create_hashes([("interval_day_time", np.frombuffer(raw, dtype=np.uint8))], len(dt))
    assert [format(int(x), "016x") for x in h] == [e["hash"] for e in dt]
    mdn = [e for e in g if e["type"] == "month_day_nano"]
    raw = b"".join(struct.pack("<iiq", e["months"], e["days"], int(e["nanos"])) for e in mdn)
    h = orc.create_hashes([("interval_month_day_nano", np.frombuffer(raw, dtype=np.uint8))], len(mdn))
    assert [format(int(x), "016x") for x in h] == [e["hash"] for e in mdn]
    # and it differs from hashing the same bytes as one integer
    e = dt[0]
    as_int = int.from_bytes(struct.pack("<ii", e["days"], e["millis"]), "little")
    assert format(op.hash_one_int(as_int, 8), "016x") != e["hash"]
