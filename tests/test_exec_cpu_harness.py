"""The host operator's HOST logic on the CPU.

`csrc/dfd_exec.cu` (chunk coalescing, bitmap / offset staging, list and view conversion, slicing the destination-sorted
chunk into Arrow batches, error fan-out, back-pressure, the pinned-chunk cache) normally needs a GPU.  Here the object
file nvcc built for the PRODUCT is linked — in a temporary directory, for this test only — against a host stand-in of the
CUDA runtime (tests/cpu_harness/fake_cudart.cpp) and against the CPU oracle in place of the kernels
(tests/cpu_harness/harness_dfd.cu), and the bodies of the GPU tests in tests/test_exec_gpu.py are run against it.  What
this checks is everything around the kernels; the kernels themselves are checked by `-m gpu`.  The product package never
loads this library (no CPU fallback): it exists only under pytest's tmp directory."""
import ctypes as C
import os
import subprocess
import types

import pyarrow as pa
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "cpu_harness")
CSRC = os.path.join(ROOT, "datafusion_distributed_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-Xcompiler", "-fPIC"]


def _build_harness(tmp):
    if os.environ.get("DFD_TEST_HARNESS_SO"):  # a prebuilt variant of the harness, e.g. compiled with -fsanitize=address
        return os.environ["DFD_TEST_HARNESS_SO"]  # (recipe: tests/cpu_harness/README.md); still test-only
    from datafusion_distributed_b200 import build as b
    from oracle import oracle as orc

    b.build()
    oracle_so = orc.build()
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC, "-I", os.path.join(ROOT, "oracle")]
    exec_obj = b.object_path("dfd_exec.cu")  # the product's own object (what libdfd_b200.so was linked from)
    newest = max(os.path.getmtime(os.path.join(d, f)) for d in (CSRC, os.path.join(ROOT, "include")) for f in os.listdir(d))
    if not os.path.exists(exec_obj) or os.path.getmtime(exec_obj) < newest:
        exec_obj = os.path.join(tmp, "dfd_exec.o")
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(CSRC, "dfd_exec.cu"), "-o", exec_obj])
    dfd_obj, rt_obj, out = os.path.join(tmp, "harness_dfd.o"), os.path.join(tmp, "fake_cudart.o"), os.path.join(tmp, "libdfd_exec_harness.so")
    subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(HARNESS, "harness_dfd.cu"), "-o", dfd_obj])
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-c", os.path.join(HARNESS, "fake_cudart.cpp"), "-o", rt_obj])
    # -Bsymbolic: the library's calls to cuda* / dfd_* bind to ITS OWN definitions even when the process has already loaded the
    # real CUDA runtime or libdfd_b200.so (other tests of the same session do)
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", out, exec_obj, dfd_obj, rt_obj, oracle_so,
                           f"-Wl,-rpath,{os.path.dirname(oracle_so)}", "-lpthread"])
    return out


class HarnessError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"status {status}: {message}")
        self.status = status
        self.message = message


class _Ctx:
    def __init__(self, lib):
        self.lib = lib
        lib.harness_ctx_create.restype = C.c_void_p
        self.handle = C.c_void_p(lib.harness_ctx_create())

    def close(self):
        if self.handle:
            self.lib.harness_ctx_destroy(self.handle)
        self.handle = C.c_void_p()


def _make_namespace(lib):
    """An object that looks like the `datafusion_distributed_b200` package to the GPU test bodies, bound to the harness."""
    import datafusion_distributed_b200 as dfd
    from datafusion_distributed_b200 import _native as nv

    VP = C.c_void_p
    sig = {
        "dfd_last_error": (C.c_char_p, []),
        "dfd_repartition_exec_create": (C.c_int, [VP, VP, C.POINTER(C.c_int32), C.c_int, C.c_uint32, C.POINTER(nv.DfdExecOptions), C.POINTER(VP)]),
        "dfd_repartition_exec_destroy": (None, [VP]),
        "dfd_repartition_exec_push": (C.c_int, [VP, VP]),
        "dfd_repartition_exec_finish": (C.c_int, [VP]),
        "dfd_repartition_exec_abort": (C.c_int, [VP, C.c_char_p]),
        "dfd_repartition_exec_run": (C.c_int, [VP, VP]),
        "dfd_repartition_exec_execute": (C.c_int, [VP, C.c_uint32, VP]),
        "dfd_repartition_exec_stats": (C.c_int, [VP, C.POINTER(nv.DfdExecStats)]),
        "harness_ctx_destroy": (None, [VP]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args

    def check(status):
        if status != 0:
            raise HarnessError(status, lib.dfd_last_error().decode("utf-8", "replace"))

    class RepartitionExec:  # same surface as datafusion_distributed_b200.execution_plans.RepartitionExec
        def __init__(self, ctx, schema, partitioning, chunk_rows=0, pipeline_depth=0, pinned_pool_chunks=0, max_pinned_chunks=0):
            self.ctx, self.schema, self.partitioning = ctx, schema, partitioning
            cs = nv.ArrowSchemaStruct()
            schema._export_to_c(C.addressof(cs))
            keys = (C.c_int32 * len(partitioning.key_cols))(*partitioning.key_cols)
            opts = nv.DfdExecOptions(chunk_rows, pipeline_depth, pinned_pool_chunks, max_pinned_chunks, 0)
            self._h = VP()
            try:
                check(lib.dfd_repartition_exec_create(ctx.handle, C.addressof(cs), keys, len(partitioning.key_cols), partitioning.partition_count,
                                                      C.byref(opts), C.byref(self._h)))
            finally:
                if cs.release:
                    C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))

        def push_batch(self, batch):
            ca = nv.ArrowArrayStruct()
            batch._export_to_c(C.addressof(ca))
            check(lib.dfd_repartition_exec_push(self._h, C.addressof(ca)))

        def finish(self):
            check(lib.dfd_repartition_exec_finish(self._h))

        def abort(self, message):
            check(lib.dfd_repartition_exec_abort(self._h, message.encode()))

        def run(self, reader):
            cs = nv.ArrowArrayStreamStruct()
            reader._export_to_c(C.addressof(cs))
            check(lib.dfd_repartition_exec_run(self._h, C.addressof(cs)))

        def execute(self, partition):
            cs = nv.ArrowArrayStreamStruct()
            check(lib.dfd_repartition_exec_execute(self._h, partition, C.addressof(cs)))
            return pa.RecordBatchReader._import_from_c(C.addressof(cs))

        def stats(self):
            st = nv.DfdExecStats()
            check(lib.dfd_repartition_exec_stats(self._h, C.byref(st)))
            return {k: getattr(st, k) for k, _ in st._fields_}

        def close(self):
            if self._h:
                lib.dfd_repartition_exec_destroy(self._h)
            self._h = VP()

    return types.SimpleNamespace(RepartitionExec=RepartitionExec, Partitioning=dfd.Partitioning, DfdError=HarnessError)


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    lib = C.CDLL(_build_harness(str(tmp_path_factory.mktemp("exec_harness"))))
    ns = _make_namespace(lib)
    ctx = _Ctx(lib)
    yield ns, ctx
    ctx.close()


# the GPU test bodies that exercise host logic only (everything except the pinned-input / device-export helpers)
CASES = [
    ("test_cfg1_shape_matches_oracle_exactly", dict(batch_rows=8192, chunk_rows=0)),
    ("test_cfg1_shape_matches_oracle_exactly", dict(batch_rows=1024, chunk_rows=10_000)),
    ("test_cfg1_shape_matches_oracle_exactly", dict(batch_rows=100_000, chunk_rows=65_536)),
    ("test_nullable_bool_mixed_widths_and_sliced_batches", {}),
    ("test_run_from_reader_and_empty_inputs", {}),
    ("test_operator_errors", {}),
    ("test_abort_fails_every_partition_stream_after_the_queued_rows", {}),
    ("test_utf8_keys_and_payload_through_the_operator", {}),
    ("test_all_empty_strings_chunk", {}),
    ("test_utf8view_and_dictionary_columns_round_trip", {}),
    ("test_small_batches_of_every_shape_coalesce_into_full_chunks", {}),
    ("test_reference_bench_fixture_schema_with_list_column", dict(keys=[0])),
    ("test_reference_bench_fixture_schema_with_list_column", dict(keys=[3])),
    ("test_reference_bench_fixture_schema_with_list_column", dict(keys=[4, 0])),
    ("test_reference_bench_fixture_schema_with_list_column", dict(keys=[7, 2])),
    ("test_list_column_edge_shapes", {}),
    ("test_bounded_pinned_pool_blocks_the_producer_until_consumers_release", {}),
    ("test_pinned_chunks_are_reused_by_the_next_operator_of_the_same_shape", {}),
    ("test_large_binary_and_fixed_size_binary_travel_as_payload", {}),
    ("test_lists_of_primitives_travel_as_payload", {}),
    ("test_equal_dictionaries_of_consecutive_batches_share_a_chunk", {}),
]


@pytest.mark.parametrize("name,kwargs", CASES, ids=[f"{n}-{i}" for i, (n, _) in enumerate(CASES)])
def test_host_logic_of_the_operator_against_the_oracle(harness, monkeypatch, name, kwargs):
    from tests import test_exec_gpu as G

    ns, ctx = harness
    monkeypatch.setattr(G, "dfd", ns)
    ctx.lib.harness_kernel_launches.restype = C.c_uint64
    ctx.lib.harness_kernel_launches.argtypes = [C.c_void_p]
    before = ctx.lib.harness_kernel_launches(ctx.handle)
    getattr(G, name)(ctx, **kwargs)
    if name != "test_operator_errors":  # (that one never gets as far as a chunk)
        assert ctx.lib.harness_kernel_launches(ctx.handle) > before  # the operator really ran through the stand-in partitioner


def _key_cases():
    from tests import test_exec_keys_gpu as K

    return K.HARNESS_CASES


@pytest.mark.parametrize("body,args", _key_cases(), ids=[f"{b}-{'-'.join(map(str, a))}" for b, a in _key_cases()])
def test_key_types_through_the_operator_against_the_oracle(harness, monkeypatch, body, args):
    """The bodies of tests/test_exec_keys_gpu.py (every key format, every Dictionary<K, V> key, unsigned indices past the
    signed range) with the operator's host logic on the stand-in partitioner."""
    from tests import test_exec_keys_gpu as K

    _, ctx = harness
    monkeypatch.setattr(K, "native", lambda: ctx.lib)
    getattr(K, body)(ctx, *args)


def test_the_product_package_never_loads_the_harness():
    """The harness is test infrastructure: nothing under the product package or the bench refers to it."""
    for top in ("datafusion_distributed_b200", "bench.py", "bench_workloads.py", "__graft_entry__.py"):
        paths = [os.path.join(ROOT, top)] if top.endswith(".py") else [os.path.join(dp, f) for dp, _, fs in os.walk(os.path.join(ROOT, top)) for f in fs
                                                                          if f.endswith((".py", ".cu", ".cuh", ".h"))]
        for p in paths:
            text = open(p, errors="replace").read()
            assert "cpu_harness" not in text and "fake_cudart" not in text and "libdfd_exec_harness" not in text, p


def _fixture_like_table(n, seed=5):
    import random

    import numpy as np

    rnd = random.Random(seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    words = ["", "a", "hello", "x" * 13, "a-much-longer-string-than-twelve-bytes"]
    label = pa.array([None if rnd.random() < 0.1 else rnd.choice(words) + str(rnd.getrandbits(12)) for _ in range(n)], type=pa.string())
    cat = pa.DictionaryArray.from_arrays(pa.array([rnd.choice([None, 0, 1, 2]) for _ in range(n)], type=pa.int32()), pa.array(["red", None, "blue"]))
    tags = pa.array([None if rnd.random() < 0.1 else [rnd.choice([None, "t1", "tag-two"]) for _ in range(rnd.randint(0, 3))] for _ in range(n)],
                    type=pa.list_(pa.string()))
    return pa.table([pa.array(rng.integers(0, 2**40, n, dtype=np.int64)), pa.array([rnd.choice([None, True, False]) for _ in range(n)]), label,
                     label.cast(pa.string_view()), cat, tags], names=["id", "flag", "label", "view", "category", "tags"])


def _run_once(ns, ctx, table, keys, **opts):
    ex = ns.RepartitionExec(ctx, table.schema, ns.Partitioning.Hash(keys, 4), **opts)
    try:
        for rb in table.to_batches(max_chunksize=500):
            ex.push_batch(rb)
        ex.finish()
        rows = sum(ex.execute(p).read_all().num_rows for p in range(4))
    finally:
        ex.close()
    return rows


def test_no_allocation_outlives_the_operator_and_its_context(harness):
    """Leak check on the stand-in runtime: after operators with every column kind (dictionary KEY included) are closed and
    their worker context destroyed (which empties the pinned-chunk cache), every device / pinned allocation has been freed."""
    import gc

    ns, _ = harness
    lib = harness[1].lib
    lib.harness_live_allocations.restype = C.c_long
    base = lib.harness_live_allocations()
    ctx = _Ctx(lib)
    table = _fixture_like_table(3000)
    assert _run_once(ns, ctx, table, [0], chunk_rows=1024) == 3000
    assert _run_once(ns, ctx, table, [4, 2], chunk_rows=256, pinned_pool_chunks=2) == 3000   # dictionary + string keys
    assert _run_once(ns, ctx, table, [0], chunk_rows=1024) == 3000                          # takes its chunks from the cache
    gc.collect()
    assert lib.harness_live_allocations() > base  # (the context still caches the pinned chunks of the finished operators)
    ctx.close()
    gc.collect()
    assert lib.harness_live_allocations() == base


@pytest.mark.parametrize("what,name", [(0, "cudaMalloc"), (1, "cudaHostAlloc"), (2, "cudaMemcpyAsync")])
def test_injected_cuda_failures_surface_as_errors_and_leak_nothing(harness, what, name):
    """Fail the n-th cudaMalloc / cudaHostAlloc / cudaMemcpyAsync for n = 1, 2, 3, ... of an operator's life (create, stage,
    flush, D2H): the failure must come back as an error from create / push / finish or from a partition stream — never a
    crash, never a hang — and once everything is closed no allocation is left behind."""
    import gc

    ns, _ = harness
    lib = harness[1].lib
    lib.harness_live_allocations.restype = C.c_long
    lib.harness_fail_nth.argtypes = [C.c_int, C.c_long]
    table = _fixture_like_table(1500)
    failures = 0
    for n in list(range(1, 40)) + [60, 90, 150, 400]:
        base = lib.harness_live_allocations()
        ctx = _Ctx(lib)
        lib.harness_fail_nth(what, n)
        try:
            rows = _run_once(ns, ctx, table, [4, 0], chunk_rows=512)
            assert rows == 1500  # the countdown was longer than this operator's life (or the failing call was not on its path)
        except (HarnessError, pa.ArrowException, OSError) as e:
            failures += 1
            assert "fake CUDA" in str(e) or "failed" in str(e) or "alloc" in str(e).lower() or "cuda" in str(e).lower(), str(e)
        finally:
            lib.harness_fail_nth(what, 0)
            ctx.close()
            gc.collect()
        assert lib.harness_live_allocations() == base, (name, n)
    assert failures >= 5, (name, failures)
