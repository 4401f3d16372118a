"""Host buffers and the oracle check of dfd_shuffle_host for every column kind (tests/test_host_shuffle_gpu.py,
tests/mgpu_host_shuffle_check.py, scripts/host_shuffle_profile.py).

Inputs are pyarrow arrays at offset 0 (their host buffers are what the library reads).  Outputs are numpy buffers of
`cap` rows with FILL guard bytes behind every capacity, so a write past one shows.  `verify` compares each output buffer
with what the oracle's row order implies, byte for byte: values (junk under nulls included), validity and Boolean bits,
string offsets continued across chunks and the dense string bytes."""
from __future__ import annotations

import random

import numpy as np

FILL = 0xAB
GUARD = 64


def mixed_arrays(n, seed, nulls=True):
    """The mixed schema of tests/test_exchange_gpu.py (Int64, Utf8, LargeUtf8, Boolean, Int32, Float64), typed explicitly so
    that an all-null or empty column keeps its type."""
    import pyarrow as pa

    rnd = random.Random(seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    none = [None] if nulls else []
    key = pa.array([rnd.choice(none + [rnd.getrandbits(30)]) for _ in range(n)], type=pa.int64())
    s = pa.array([rnd.choice(none + ["", "N", "O", "phrase %d" % rnd.getrandbits(16), "x" * rnd.randint(0, 50)]) for _ in range(n)], type=pa.string())
    ls = pa.array([rnd.choice(none + ["L" * rnd.randint(0, 9)]) for _ in range(n)], type=pa.large_string())
    bl = pa.array([rnd.choice(none + [True, False]) for _ in range(n)], type=pa.bool_())
    i32 = pa.array([rnd.choice(none + [rnd.getrandbits(31)]) for _ in range(n)], type=pa.int32())
    f64 = pa.array(rng.standard_normal(n))
    return [key, s, ls, bl, i32, f64]


def kind_of(t):
    import pyarrow as pa

    from datafusion_distributed_b200 import _native as nv

    if pa.types.is_boolean(t):
        return nv.COL_BOOL, 0
    if pa.types.is_string(t):
        return nv.COL_UTF8, 0
    if pa.types.is_large_string(t):
        return nv.COL_LARGE_UTF8, 0
    if pa.types.is_binary(t):
        return nv.COL_BINARY, 0
    return nv.COL_FIXED, t.bit_width // 8


def is_var(t):
    import pyarrow as pa

    return pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_binary(t)


def in_columns(arrays, n):
    """DeviceColumn descriptors over the HOST buffers of `arrays` (offset 0; a validity bitmap only if there are nulls)."""
    import datafusion_distributed_b200 as dfd

    cols = []
    for a in arrays:
        assert a.offset == 0
        b = a.buffers()
        kind, width = kind_of(a.type)
        validity = b[0].address if (b[0] is not None and a.null_count > 0) else 0
        if is_var(a.type):
            cols.append(dfd.DeviceColumn(kind, 0, b[2].address if b[2] is not None else 0, b[1].address, validity, 0, n, a, a.type,
                                         b[2].size if b[2] is not None else 0))
        else:
            cols.append(dfd.DeviceColumn(kind, width, b[1].address, 0, validity, 0, n, a, a.type))
    return cols


def string_bytes(a, idx=None):
    """Bytes of the rows idx (all rows by default) of a var-width array at offset 0, a null row's bytes included."""
    import pyarrow as pa

    dt = np.int64 if pa.types.is_large_string(a.type) else np.int32
    off = np.frombuffer(a.buffers()[1], dtype=dt)[:len(a) + 1].astype(np.int64)
    lens = off[1:] - off[:-1]
    return int(lens.sum() if idx is None else lens[idx].sum())


def _words(rows):
    return (rows + 31) // 32 * 4


class HostOut:
    """Output buffers of `cap` rows for `types` (bitmaps as whole 32-bit words); a validity buffer for columns with
    nullable[i]; string columns get nbytes[i] bytes."""

    def __init__(self, types, cap, nullable, nbytes):
        import datafusion_distributed_b200 as dfd

        self.types, self.cap, self.bufs, self.cols = types, cap, {}, []
        for i, t in enumerate(types):
            kind, width = kind_of(t)
            validity = self._buf(i, "validity", _words(cap)) if nullable[i] else 0
            if kind == 1:  # Boolean
                self.cols.append(dfd.DeviceColumn(kind, 0, self._buf(i, "values", _words(cap)), 0, validity, 0, cap, self, t))
            elif is_var(t):
                ow = 8 if kind == 3 else 4
                self.cols.append(dfd.DeviceColumn(kind, 0, self._buf(i, "values", nbytes[i]), self._buf(i, "offsets", (cap + 1) * ow), validity, 0, cap,
                                                  self, t, nbytes[i]))
            else:
                self.cols.append(dfd.DeviceColumn(kind, width, self._buf(i, "values", cap * width), 0, validity, 0, cap, self, t))

    def _buf(self, i, what, n):
        b = np.full(n + GUARD, FILL, dtype=np.uint8)
        self.bufs[(i, what)] = (b, n)
        return b.ctypes.data


def _bits_of(a, which):
    """The bits of rows [0, len) of a's validity (which = 0; all ones without a bitmap) or Boolean values (which = 1)."""
    b = a.buffers()[which]
    if b is None:
        return np.ones(len(a), dtype=np.uint8)
    return np.unpackbits(np.frombuffer(b, dtype=np.uint8), bitorder="little")[a.offset:a.offset + len(a)]


def expected_order(dests, n_rows, n_chunks, P, rank=0):
    """World 1 (or this worker's own rows): row indices in output order, and chunk_part_starts[n_chunks][P+1]."""
    order, cps = [], np.zeros((n_chunks, P + 1), dtype=np.int64)
    at = 0
    for ch in range(n_chunks):
        lo, hi = n_rows * ch // n_chunks, n_rows * (ch + 1) // n_chunks
        d = dests[lo:hi]
        for q in range(P):
            cps[ch, q] = at
            idx = lo + np.nonzero(d == rank * P + q)[0]
            order.append(idx)
            at += len(idx)
        cps[ch, P] = at
    return (np.concatenate(order) if order else np.zeros(0, np.int64)).astype(np.int64), cps


def verify(out: HostOut, sources, total):
    """sources[i]: list of (array, row indices) whose concatenation is column i's expected output rows, in order."""
    for i, t in enumerate(out.types):
        parts = sources[i]
        kind, width = kind_of(t)
        w = _words(total)
        if (i, "validity") in out.bufs:
            vb, n = out.bufs[(i, "validity")]
            want = np.concatenate([_bits_of(a, 0)[idx] for a, idx in parts] + [np.zeros(w * 8 - total, np.uint8)])
            assert np.array_equal(np.unpackbits(vb[:w], bitorder="little"), want), (i, "validity")
            assert (vb[w:] == FILL).all(), (i, "validity written past the words of the rows")
        if kind == 1:
            vb, n = out.bufs[(i, "values")]
            want = np.concatenate([_bits_of(a, 1)[idx] for a, idx in parts] + [np.zeros(w * 8 - total, np.uint8)])
            assert np.array_equal(np.unpackbits(vb[:w], bitorder="little"), want), (i, "boolean values")
            assert (vb[w:] == FILL).all(), (i, "boolean values written past the words of the rows")
        elif is_var(t):
            ow = 8 if kind == 3 else 4
            dt = np.int64 if ow == 8 else np.int32
            lens, data = [], []
            for a, idx in parts:
                off = np.frombuffer(a.buffers()[1], dtype=dt)[a.offset:a.offset + len(a) + 1].astype(np.int64)
                raw = np.frombuffer(a.buffers()[2], dtype=np.uint8) if a.buffers()[2] is not None else np.zeros(0, np.uint8)
                lens.append(off[1:][idx] - off[:-1][idx])
                data += [raw[off[k]:off[k + 1]] for k in idx]
            lens = np.concatenate(lens) if lens else np.zeros(0, np.int64)
            want_off = np.concatenate([[0], np.cumsum(lens)]).astype(dt)
            ob, n = out.bufs[(i, "offsets")]
            assert np.array_equal(ob[:(total + 1) * ow].view(dt), want_off), (i, "offsets")
            assert (ob[(total + 1) * ow:] == FILL).all(), (i, "offsets written past the rows")
            nb = int(want_off[-1])
            vb, n = out.bufs[(i, "values")]
            want = np.concatenate(data) if data else np.zeros(0, np.uint8)
            assert np.array_equal(vb[:nb], want), (i, "string bytes")
            assert (vb[nb:] == FILL).all(), (i, "string bytes written past the data")
        else:
            vb, n = out.bufs[(i, "values")]
            want = np.concatenate([np.frombuffer(a.buffers()[1], dtype=np.uint8)[:(a.offset + len(a)) * width].reshape(-1, width)[a.offset:][idx] for a, idx in parts])
            assert np.array_equal(vb[:total * width].reshape(-1, width), want.reshape(-1, width)), (i, "values")
            assert (vb[total * width:] == FILL).all(), (i, "values written past the rows")
