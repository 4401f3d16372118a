"""CPU tests of FixedSizeList payload in the host operator: which schemas dfd_repartition_supported admits, and the staging
arithmetic of dfd_host_staging.h (the child range of a piece of rows, the bit rows appended to a chunk) against pyarrow."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pyarrow as pa
import pytest

from datafusion_distributed_b200 import _native as nv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ACCEPTED_CHILDREN = ["c", "C", "s", "S", "i", "I", "l", "L", "e", "f", "g", "d:9,2", "d:38,0", "d:9,2,32", "d:18,4,64", "tdD", "tdm",
                     "tts", "ttm", "ttu", "ttn", "tss:", "tsn:UTC", "tDs", "tDn", "tiM", "tiD", "tin", "b"]
REFUSED_CHILDREN = ["u", "U", "z", "Z", "vu", "vz", "w:4", "w:12", "w:16", "+l", "+w:2", "+s", "n", "d:76,0,256"]


def _schema(fmt, child_fmt, child_dict=False):
    keep = []

    def node(f, name):
        s = nv.ArrowSchemaStruct()
        s.format, s.name, s.flags = f.encode(), name, 2
        keep.append(s)
        return s

    col = node(fmt, b"emb")
    if child_fmt is not None:
        item = node(child_fmt, b"item")
        if child_dict:
            item.dictionary = C.addressof(node("u", b""))
        kids = (C.POINTER(nv.ArrowSchemaStruct) * 1)(C.pointer(item))
        keep.append(kids)
        col.n_children, col.children = 1, C.cast(kids, C.c_void_p)
    top = node("+s", b"")
    kids = (C.POINTER(nv.ArrowSchemaStruct) * 2)(C.pointer(node("l", b"id")), C.pointer(col))
    keep.append(kids)
    top.n_children, top.children = 2, C.cast(kids, C.c_void_p)
    return top, keep


def supported(fmt, child_fmt, key=0, child_dict=False):
    lib = nv.lib()
    top, _keep = _schema(fmt, child_fmt, child_dict)
    rc = lib.dfd_repartition_supported(C.byref(top), (C.c_int32 * 1)(key), 1)
    return rc, lib.dfd_last_error().decode()


def test_repartition_supported_admits_exactly_the_fixed_size_list_shapes(built):
    for child in ACCEPTED_CHILDREN:
        for n in (1, 3, 768):
            assert supported(f"+w:{n}", child) == (0, supported(f"+w:{n}", child)[1]), (n, child)
        assert nv.lib().dfd_schema_supported(C.byref(_schema("+w:7", child)[0])) == 0, child
    for child in REFUSED_CHILDREN:
        rc, msg = supported("+w:4", child)
        assert rc == 6 and "emb" in msg, (child, rc, msg)
    for fmt, child, key, cdict in [("+w:4", "f", 1, False), ("+w:0", "f", 0, False), ("+w:", "f", 0, False), ("+w:4x", "f", 0, False),
                                   ("+w:4", None, 0, False), ("+w:4", "i", 0, True)]:
        rc, msg = supported(fmt, child, key, cdict)
        assert rc == 6 and "emb" in msg, (fmt, child, key, cdict, rc, msg)
    assert "hash keys" in supported("+w:4", "f", 1)[1]
    # FixedSizeBinary outside 1/2/4/8/16 bytes stays refused everywhere
    assert nv.lib().dfd_arrow_format_layout(b"w:12", None, None) == 6


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("fsl_staging") / "libfsl_staging_shim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "datafusion_distributed_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "fsl_staging_shim.cpp"), "-o", out])
    return C.CDLL(out)


def _fsl(rnd, t, n, rows, offset, child_offset):
    ne = child_offset + (offset + rows) * n
    rng = np.random.Generator(np.random.PCG64(rnd.getrandbits(32)))
    w = 0 if pa.types.is_boolean(t) else t.bit_width // 8
    vals = np.packbits(rng.random(ne) < 0.5, bitorder="little").tobytes() if w == 0 else rng.integers(0, 256, ne * w, dtype=np.uint8).tobytes()
    valid = np.packbits(rng.random(ne) < 0.7, bitorder="little").tobytes()
    child = pa.Array.from_buffers(t, ne - child_offset, [pa.py_buffer(valid), pa.py_buffer(vals)], null_count=-1, offset=child_offset)
    return pa.Array.from_buffers(pa.list_(t, n), rows, [None], offset=offset, children=[child]), w


def test_staging_arithmetic_matches_pyarrow(shim):
    """Pieces of sliced FixedSizeList batches staged one after the other: the child bytes each piece copies are the bytes of
    pyarrow's flatten() of that piece, and the concatenated bit rows are the flattened validity / Boolean values."""
    rnd = random.Random(3)
    out4 = (C.c_int64 * 4)()
    for _ in range(200):
        t = rnd.choice([pa.int8(), pa.float32(), pa.decimal128(20, 2), pa.bool_()])
        n = rnd.choice([1, 3, 7, 8, 9, 33, 64])
        chunk_valid = np.full(4096, 0xAA, dtype=np.uint8)
        chunk_bool = np.full(4096, 0x55, dtype=np.uint8)
        at, want_valid, want_bool = 0, [], []
        for _piece in range(rnd.randint(1, 4)):
            rows, offset, coff = rnd.randint(0, 40), rnd.randint(0, 40), rnd.randint(0, 20)
            a, w = _fsl(rnd, t, n, rows + 10, offset, coff)
            lo = rnd.randint(0, 10)  # rows [lo, lo + rows) of the batch
            piece = a.slice(lo, rows)
            flat = piece.flatten()
            shim.t_fsl_span(C.c_int64(a.values.offset), C.c_int64(a.offset + lo), C.c_int64(rows), C.c_int64(n), C.c_int64(w), out4)
            first_bit, n_bits, first_byte, n_bytes = list(out4)
            assert first_bit == flat.offset and n_bits == len(flat) == rows * n
            if w:
                raw = np.frombuffer(a.values.buffers()[1], dtype=np.uint8)[first_byte:first_byte + n_bytes]
                assert np.array_equal(raw, np.frombuffer(flat.buffers()[1], dtype=np.uint8)[flat.offset * w:(flat.offset + len(flat)) * w])
            bufs = a.values.buffers()
            vbits = np.frombuffer(bufs[0], dtype=np.uint8)
            shim.t_append_bit_rows(chunk_valid.ctypes.data_as(C.c_void_p), C.c_int64(at), vbits.ctypes.data_as(C.c_void_p), C.c_int64(a.values.offset),
                                   C.c_int64(a.offset + lo), C.c_int64(rows), C.c_int64(n))
            want_valid += flat.is_valid().to_pylist()
            if w == 0:
                bbits = np.frombuffer(bufs[1], dtype=np.uint8)
                shim.t_append_bit_rows(chunk_bool.ctypes.data_as(C.c_void_p), C.c_int64(at), bbits.ctypes.data_as(C.c_void_p),
                                       C.c_int64(a.values.offset), C.c_int64(a.offset + lo), C.c_int64(rows), C.c_int64(n))
                raw_bits = np.unpackbits(bbits, bitorder="little")[flat.offset:flat.offset + len(flat)]
                want_bool += [bool(b) for b in raw_bits]
            at += rows
        got = np.unpackbits(chunk_valid, bitorder="little")[:at * n].astype(bool).tolist()
        assert got == want_valid
        if t == pa.bool_():
            assert np.unpackbits(chunk_bool, bitorder="little")[:at * n].astype(bool).tolist() == want_bool
        # a NULL bitmap (a nullable child without one) appends ones
        ones = np.zeros(64, dtype=np.uint8)
        shim.t_append_bit_rows(ones.ctypes.data_as(C.c_void_p), C.c_int64(1), None, C.c_int64(5), C.c_int64(2), C.c_int64(3), C.c_int64(n if n <= 33 else 33))
        k = n if n <= 33 else 33
        assert np.unpackbits(ones, bitorder="little")[:4 * k].tolist() == [0] * k + [1] * (3 * k)
