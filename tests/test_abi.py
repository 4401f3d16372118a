"""CPU tests of the drop-in boundary: the C-ABI library builds for sm_90a,
loads, exports every symbol include/dfd_b200.h declares, and fails loudly
(no CPU fallback) when there is no CUDA device."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "dfd_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dfd_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_what_python_binds(built):
    from datafusion_distributed_b200 import _native as nv

    assert sorted(nv.SIGNATURES) == declared_symbols()


def test_library_exports_every_declared_symbol(built):
    from datafusion_distributed_b200 import _native as nv

    L = nv.lib()
    for name in declared_symbols():
        assert hasattr(L, name), name
    assert L.dfd_abi_version() == 1
    assert L.dfd_status_name(6) == b"DFD_ERR_UNSUPPORTED"


def test_library_is_sm90a_and_has_the_kernels(built):
    from datafusion_distributed_b200 import LIB_PATH

    out = subprocess.run(["cuobjdump", "-lelf", LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out
    sass = subprocess.run(["cuobjdump", "-sass", LIB_PATH], capture_output=True, text=True).stdout
    for k in ("k_scatter", "k_tile_hist", "k_scan_tiles", "k_partition_ids"):
        assert k in sass, k
    assert "VOTE" in sass  # warp-ballot ranking is in the scatter kernel


def test_compiled_scatter_instantiations_are_exactly_the_reachable_ones(built):
    """Every scatter instantiation in the library is one the dispatch launches for some input (tests/util.py
    scatter_dispatch), and every reachable one is compiled.  tests/test_instantiations_gpu.py launches each of them."""
    from datafusion_distributed_b200 import LIB_PATH
    from tests.util import compiled_scatter_instances, scatter_dispatch

    compiled = compiled_scatter_instances(LIB_PATH)
    reach = scatter_dispatch()
    assert sorted(compiled - set(reach)) == [], "compiled, but no input launches them"
    assert sorted(set(reach) - compiled) == []
    assert len(reach) == 79  # (a change of the dispatch must revisit the GPU module's cases)


def test_header_compiles_as_plain_c(tmp_path):
    src = tmp_path / "t.c"
    src.write_text('#include "dfd_b200.h"\nint main(void){ struct ArrowArray a; (void)a; return DFD_OK; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src),
                           "-o", str(tmp_path / "t.o")])


def test_no_cpu_fallback_without_gpu(built):
    """On a box without CUDA the context constructor must raise; with CUDA it must work."""
    import datafusion_distributed_b200 as dfd
    from datafusion_distributed_b200 import _native as nv

    n = C.c_int(-1)
    st = nv.lib().dfd_device_count(C.byref(n))
    if st == 0 and n.value > 0:
        pytest.skip("GPU present")
    with pytest.raises(dfd.DfdError) as ei:
        dfd.WorkerContext(0)
    assert ei.value.status == 3  # DFD_ERR_CUDA
    assert "no CPU fallback" in str(ei.value)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "datafusion_distributed_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                assert "oracle" not in open(os.path.join(dp, f)).read().lower(), os.path.join(dp, f)


def test_schema_support_helpers_run_without_a_gpu(built):
    """dfd_arrow_format_layout / dfd_schema_supported: the pure-host predicates the plan hook uses."""
    import ctypes as C

    import pyarrow as pa

    from datafusion_distributed_b200 import _native as nv

    L = nv.lib()
    expect = {b"l": (0, 8), b"L": (0, 8), b"i": (0, 4), b"s": (0, 2), b"c": (0, 1), b"g": (0, 8), b"f": (0, 4), b"e": (0, 2), b"b": (1, 0),
              b"u": (2, 0), b"U": (3, 0), b"z": (4, 0), b"d:38,10": (0, 16), b"d:9,2,32": (0, 4), b"tsn:": (0, 8), b"tsu:UTC": (0, 8),
              b"tdD": (0, 4), b"tdm": (0, 8), b"ttu": (0, 8), b"tts": (0, 4), b"tDn": (0, 8), b"tiM": (0, 4), b"tiD": (0, 8), b"tin": (0, 16)}
    for fmt, (kind, width) in expect.items():
        k, w = C.c_int32(-1), C.c_int32(-1)
        assert L.dfd_arrow_format_layout(fmt, C.byref(k), C.byref(w)) == 0, fmt
        assert (k.value, w.value) == (kind, width), fmt
    for fmt, (kind, width) in {b"vu": (2, 0), b"vz": (4, 0)}.items():  # Utf8View / BinaryView move as Utf8 / Binary on the device
        k, w = C.c_int32(-1), C.c_int32(-1)
        assert L.dfd_arrow_format_layout(fmt, C.byref(k), C.byref(w)) == 0 and (k.value, w.value) == (kind, width), fmt
    # LargeBinary moves like LargeUtf8 (int64 offsets + bytes), FixedSizeBinary(1/2/4/8/16) like an N-byte value: payload only
    for fmt, (kind, width) in {b"Z": (3, 0), b"w:16": (0, 16), b"w:4": (0, 4)}.items():
        k, w = C.c_int32(-1), C.c_int32(-1)
        assert L.dfd_arrow_format_layout(fmt, C.byref(k), C.byref(w)) == 0 and (k.value, w.value) == (kind, width), fmt
    for fmt in (b"+l", b"+s", b"d:76,0,256", b"w:12", b"w:32", b"n"):
        assert L.dfd_arrow_format_layout(fmt, None, None) == 6, fmt  # DFD_ERR_UNSUPPORTED

    def supported(schema):
        cs = nv.ArrowSchemaStruct()
        schema._export_to_c(C.addressof(cs))
        try:
            return L.dfd_schema_supported(C.byref(cs)), L.dfd_last_error().decode()
        finally:
            C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))

    ok = pa.schema([("id", pa.int64()), ("metric", pa.float64()), ("flag", pa.bool_()), ("label", pa.string()), ("raw", pa.uint8()),
                    ("ts", pa.timestamp("ns")), ("count", pa.int32()), ("price", pa.decimal128(15, 2)), ("blob", pa.binary())])
    assert supported(ok)[0] == 0
    # the reference's bench fixture (src/execution_plans/benchmarks/fixture.rs:13-33): Dictionary<Int32, Utf8> is supported
    # (indices scattered, dictionary by reference), and so are view types and List<Utf8> (lengths + bytes as hidden columns)
    assert supported(pa.schema([("id", pa.int64()), ("category", pa.dictionary(pa.int32(), pa.string())), ("v", pa.string_view()),
                                ("bv", pa.binary_view()), ("d8", pa.dictionary(pa.int8(), pa.int64()))]))[0] == 0
    st, why = supported(pa.schema([("id", pa.int64()), ("nested", pa.dictionary(pa.int32(), pa.list_(pa.int32())))]))
    assert st == 6 and "dictionary value type" in why
    assert supported(pa.schema([("id", pa.int64()), ("tags", pa.list_(pa.string())), ("blobs", pa.list_(pa.binary()))]))[0] == 0
    # the reference's 9-column fixture schema, whole
    fixture = pa.schema([pa.field("id", pa.int64(), False), pa.field("metric", pa.float64(), False), ("flag", pa.bool_()), ("label", pa.string()),
                         ("category", pa.dictionary(pa.int32(), pa.string())), pa.field("raw", pa.uint8(), False),
                         pa.field("ts", pa.timestamp("ns"), False), pa.field("count", pa.int32(), False), ("tags", pa.list_(pa.string()))])
    assert supported(fixture)[0] == 0
    assert supported(pa.schema([("id", pa.int64()), ("nums", pa.list_(pa.int32())), ("xs", pa.list_(pa.float64()))]))[0] == 0  # primitive children too
    st, why = supported(pa.schema([("id", pa.int64()), ("nested", pa.list_(pa.list_(pa.int32())))]))
    assert st == 6 and "nested" in why
    st, why = supported(pa.schema([("id", pa.int64()), ("flags", pa.list_(pa.bool_()))]))
    assert st == 6 and "flags" in why
    st, why = supported(pa.schema([("id", pa.int64()), ("s", pa.struct([("a", pa.int32())]))]))
    assert st == 6 and "s" in why

    # dfd_repartition_supported: the same, with the hash keys taken into account (what the plan hook asks)
    def repartition_supported(schema, keys):
        cs = nv.ArrowSchemaStruct()
        schema._export_to_c(C.addressof(cs))
        try:
            return L.dfd_repartition_supported(C.byref(cs), (C.c_int32 * len(keys))(*keys), len(keys)), L.dfd_last_error().decode()
        finally:
            C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))

    wide = pa.schema([("id", pa.int64()), ("uuid", pa.binary(16)), ("blob", pa.large_binary()), ("tags", pa.list_(pa.string())), ("label", pa.string_view()),
                      ("cat", pa.dictionary(pa.int32(), pa.string())), ("dv", pa.dictionary(pa.int32(), pa.string_view())),
                      ("db", pa.dictionary(pa.int16(), pa.large_binary()))])
    assert supported(wide)[0] == 0
    assert repartition_supported(wide, [0])[0] == 0 and repartition_supported(wide, [0, 4, 5])[0] == 0
    for key, word in ((1, "payload"), (2, "payload"), (3, "list"), (6, "view-typed"), (7, "dictionary values")):
        st, why = repartition_supported(wide, [0, key])
        assert st == 6 and word in why, (key, why)
    assert repartition_supported(wide, [9])[0] == 1 and repartition_supported(wide, [])[0] == 1  # DFD_ERR_INVALID_ARGUMENT
