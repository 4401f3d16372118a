"""The device-output path of the host operator (device_output, execute_device, run_device) on the CPU harness.

The bodies of tests/test_exec_device_output_gpu.py run against the product's dfd_exec object linked with the stand-in CUDA
runtime and the host restatements of the staging and emit launches (tests/cpu_harness/harness_stage.cu, harness_emit.cu):
"device" chunks are host memory, so the helper copies them with memmove.  What this checks is the operator's host logic
around the kernels — which buffers the partitioner is handed, chunk ownership and reuse, events, dictionary upload and
reference, the stream wrappers, the refusals — and it is the view of that logic an address sanitizer can run: the recipe
of tests/cpu_harness/README.md with harness_stage.cu and harness_emit.cu compiled like harness_dfd.cu, fake_cudart_events.cpp
in place of fake_cudart.cpp, and the library named by DFD_TEST_OUTPUT_HARNESS_SO."""
import ctypes as C
import gc
import os
import subprocess

import pyarrow as pa
import pytest

from tests.test_exec_cpu_harness import CSRC, HARNESS, NVCC, NVCC_FLAGS, ROOT, _Ctx, _fixture_like_table, _make_namespace

SOURCES = ("harness_dfd.cu", "harness_stage.cu", "harness_emit.cu")


def _build_output_harness(tmp, sources=SOURCES):
    """The host-logic harness plus the host restatements of the staging launches and of launch_emit_chunk (without the
    latter the operator object's weak reference stays unresolved and a device-output operator cannot be created)."""
    if os.environ.get("DFD_TEST_OUTPUT_HARNESS_SO") and sources == SOURCES:  # a prebuilt variant, e.g. with -fsanitize=address
        return os.environ["DFD_TEST_OUTPUT_HARNESS_SO"]
    from datafusion_distributed_b200 import build as b
    from oracle import oracle as orc

    b.build()
    oracle_so = orc.build()
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC, "-I", os.path.join(ROOT, "oracle")]
    exec_obj = b.object_path("dfd_exec.cu")  # the product's own object
    newest = max(os.path.getmtime(os.path.join(d, f)) for d in (CSRC, os.path.join(ROOT, "include")) for f in os.listdir(d))
    if not os.path.exists(exec_obj) or os.path.getmtime(exec_obj) < newest:
        exec_obj = os.path.join(tmp, "dfd_exec.o")
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(CSRC, "dfd_exec.cu"), "-o", exec_obj])
    objs = [exec_obj]
    for src in sources:
        objs.append(os.path.join(tmp, src.replace(".cu", ".o")))
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(HARNESS, src), "-o", objs[-1]])
    objs.append(os.path.join(tmp, "fake_cudart_events.o"))  # (fake_cudart.cpp with its events counted and failable)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-c", os.path.join(HARNESS, "fake_cudart_events.cpp"), "-o", objs[-1]])
    out = os.path.join(tmp, "libdfd_exec_output_harness.so")
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", out] + objs + [oracle_so, f"-Wl,-rpath,{os.path.dirname(oracle_so)}", "-lpthread"])
    return out


def _namespace(lib):
    """The harness namespace of tests/test_exec_cpu_harness.py with the device sides of the operator bound too."""
    from datafusion_distributed_b200 import _native as nv
    from datafusion_distributed_b200.execution_plans import DeviceBatchStream

    ns = _make_namespace(lib)
    VP = C.c_void_p
    for name in ("dfd_repartition_exec_push_device", "dfd_repartition_exec_run_device"):
        getattr(lib, name).restype, getattr(lib, name).argtypes = C.c_int, [VP, VP]
    lib.dfd_repartition_exec_execute_device.restype, lib.dfd_repartition_exec_execute_device.argtypes = C.c_int, [VP, C.c_uint32, VP]

    def check(status):
        if status != 0:
            raise ns.DfdError(status, lib.dfd_last_error().decode("utf-8", "replace"))

    class RepartitionExec(ns.RepartitionExec):
        def __init__(self, ctx, schema, partitioning, chunk_rows=0, pipeline_depth=0, pinned_pool_chunks=0, max_pinned_chunks=0, device_output=False):
            self.ctx, self.schema, self.partitioning = ctx, schema, partitioning
            cs = nv.ArrowSchemaStruct()
            schema._export_to_c(C.addressof(cs))
            keys = (C.c_int32 * len(partitioning.key_cols))(*partitioning.key_cols)
            opts = nv.DfdExecOptions(chunk_rows, pipeline_depth, pinned_pool_chunks, max_pinned_chunks, int(device_output))
            self._h = VP()
            try:
                check(lib.dfd_repartition_exec_create(ctx.handle, C.addressof(cs), keys, len(partitioning.key_cols), partitioning.partition_count,
                                                      C.byref(opts), C.byref(self._h)))
            finally:
                if cs.release:
                    C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))

        def push_device_batch(self, device_array):
            check(lib.dfd_repartition_exec_push_device(self._h, device_array if isinstance(device_array, int) else C.addressof(device_array)))

        def run_device(self, stream):
            check(lib.dfd_repartition_exec_run_device(self._h, C.addressof(stream)))

        def execute_device(self, partition):
            cs = nv.ArrowDeviceArrayStreamStruct()
            check(lib.dfd_repartition_exec_execute_device(self._h, partition, C.addressof(cs)))
            return DeviceBatchStream(cs)

    ns.RepartitionExec = RepartitionExec
    return ns


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    lib = C.CDLL(_build_output_harness(str(tmp_path_factory.mktemp("exec_output_harness"))))
    lib.harness_live_allocations.restype = C.c_long
    lib.harness_live_events.restype = C.c_long
    lib.harness_fail_nth.argtypes = [C.c_int, C.c_long]
    lib.harness_fail_nth_event.argtypes = [C.c_long]
    ns = _namespace(lib)
    ctx = _Ctx(lib)
    yield ns, ctx
    ctx.close()


def _bind(monkeypatch, harness):
    from tests import device_batches as DB
    from tests import device_outputs as DO
    from tests import test_exec_device_input_gpu as IN
    from tests import test_exec_device_output_gpu as G

    ns, ctx = harness
    monkeypatch.setattr(G, "dfd", ns)
    monkeypatch.setattr(IN, "dfd", ns)
    monkeypatch.setattr(DB, "ALLOC", DB.host_alloc)
    monkeypatch.setattr(DO, "COPY", DO.host_copy)
    monkeypatch.setattr(DO, "WAIT", None)
    return G, ctx


CASES = [
    ("test_fixed_width_batches_move_nothing_over_pcie", dict(batch_rows=8192, chunk_rows=0)),
    ("test_fixed_width_batches_move_nothing_over_pcie", dict(batch_rows=1024, chunk_rows=10_000)),
    ("test_fixed_width_batches_move_nothing_over_pcie", dict(batch_rows=100_000, chunk_rows=65_536)),
    ("test_nullable_bool_mixed_widths_sliced", dict(keys=[0])),
    ("test_nullable_bool_mixed_widths_sliced", dict(keys=[5, 2])),
    ("test_strings_as_keys_and_payload", dict(keys=[1])),
    ("test_strings_as_keys_and_payload", dict(keys=[3, 1])),
    ("test_views_of_every_length_class", dict(keys=[0])),
    ("test_views_of_every_length_class", dict(keys=[2, 0])),
    ("test_dictionaries_as_payload_and_as_key", dict(keys=[0])),
    ("test_dictionaries_as_payload_and_as_key", dict(keys=[1, 0])),
    ("test_device_input_batches_with_dictionaries_live_until_their_output_is_released", {}),
    ("test_reference_fixture_schema", dict(keys=[0], N=8)),
    ("test_reference_fixture_schema", dict(keys=[0, 3], N=17)),
    ("test_lists_of_strings_binaries_and_primitives", {}),
    ("test_bounded_pool_blocks_the_producer_until_consumers_release_device_batches", {}),
    ("test_device_chunks_are_reused_once_consumers_release", {}),
    ("test_abort_and_input_errors_reach_every_device_stream_after_the_queued_batches", {}),
    ("test_streams_of_the_wrong_kind_are_refused", {}),
    ("test_run_device_pulls_a_device_stream", {}),
]


@pytest.mark.parametrize("name,kwargs", CASES, ids=[f"{n}-{i}" for i, (n, _) in enumerate(CASES)])
def test_device_output_host_logic(harness, monkeypatch, name, kwargs):
    G, ctx = _bind(monkeypatch, harness)
    getattr(G, name)(ctx, **kwargs)


def _run_device_output(ns, ctx, batches, device_input):
    """One device-output operator over `batches`, every stream drained; returns (rows out, keys of the device batches pushed)."""
    from tests import device_batches as DB

    ex, pushed = None, []
    try:
        ex = ns.RepartitionExec(ctx, batches[0].schema, ns.Partitioning.Hash([4, 0], 4), chunk_rows=512, device_output=True)
        for rb in batches:
            if device_input:
                b = DB.DeviceBatch(rb, alloc=DB.host_alloc)
                pushed.append(b.key)
                ex.push_device_batch(b.device_array)
            else:
                ex.push_batch(rb)
        ex.finish()
        return sum(b.array.length for p in range(4) for b in ex.execute_device(p)), pushed
    finally:
        if ex is not None:
            ex.close()


@pytest.mark.parametrize("device_input", [False, True], ids=["host-input", "device-input"])
def test_device_output_leaves_no_chunk_event_or_input_behind(harness, device_input):
    """Every device chunk (its buffers, list scratch, uploaded dictionaries), every event and every held input batch is
    freed once the operator and its context are gone."""
    from tests import device_batches as DB

    ns, hctx = harness
    lib = hctx.lib
    base, base_events = lib.harness_live_allocations(), lib.harness_live_events()
    ctx = _Ctx(lib)
    rows, pushed = _run_device_output(ns, ctx, _fixture_like_table(3_000).to_batches(max_chunksize=500), device_input)
    assert rows == 3_000
    ctx.close()
    gc.collect()
    assert lib.harness_live_allocations() == base and lib.harness_live_events() == base_events
    assert not set(pushed) & DB.live_batches()
    assert sorted(k for k in DB.RELEASED if k in set(pushed)) == sorted(pushed)


@pytest.mark.parametrize("device_input", [False, True], ids=["host-input", "device-input"])
@pytest.mark.parametrize("what,name", [(0, "cudaMalloc"), (3, "cudaEventCreateWithFlags"), (2, "cudaMemcpyAsync")])
def test_injected_cuda_failures_on_device_output_surface_as_errors_and_leak_nothing(harness, what, name, device_input):
    """Fail the n-th cudaMalloc / cudaEventCreateWithFlags / cudaMemcpyAsync of a device-output operator's life (create, the
    chunk pool, string-byte growth, list scratch, dictionary upload, flush): the failure comes back as an error from create /
    push / finish or from a stream — never a crash — and afterwards no allocation, event or input batch is left behind."""
    from tests import device_batches as DB

    ns, hctx = harness
    lib = hctx.lib
    batches = _fixture_like_table(1_500).to_batches(max_chunksize=500)
    failures = 0
    for n in list(range(1, 60)) + [90, 150, 400]:
        base, base_events = lib.harness_live_allocations(), lib.harness_live_events()
        ctx = _Ctx(lib)
        arm = lib.harness_fail_nth_event if what == 3 else (lambda k: lib.harness_fail_nth(what, k))
        arm(n)
        before = set(DB.live_batches())
        try:
            rows, _ = _run_device_output(ns, ctx, batches, device_input)
            assert rows == 1_500  # (the countdown was longer than this operator's life)
        except (ns.DfdError, pa.ArrowException, OSError) as e:
            failures += 1
            assert "fake CUDA" in str(e) or "failed" in str(e) or "alloc" in str(e).lower() or "cuda" in str(e).lower(), str(e)
        finally:
            arm(0)
            ctx.close()
            gc.collect()
        assert DB.live_batches() <= before, (name, n)
        assert lib.harness_live_allocations() == base and lib.harness_live_events() == base_events, (name, n)
    assert failures >= 5, (name, failures)


def test_an_operator_object_linked_without_the_emit_kernel_refuses_device_output(built, tmp_path):
    """Without harness_emit.cu the operator object still links (its reference to launch_emit_chunk is weak) and host output
    works as ever; creating a device-output operator fails with DFD_ERR_UNSUPPORTED."""
    lib = C.CDLL(_build_output_harness(str(tmp_path), sources=("harness_dfd.cu", "harness_stage.cu")))
    ns = _namespace(lib)
    ctx = _Ctx(lib)
    rb = pa.record_batch([pa.array(range(10), type=pa.int64())], names=["k"])
    with pytest.raises(ns.DfdError) as ei:
        ns.RepartitionExec(ctx, rb.schema, ns.Partitioning.Hash([0], 2), device_output=True)
    assert ei.value.status == 6 and "emit kernel" in ei.value.message
    ex = ns.RepartitionExec(ctx, rb.schema, ns.Partitioning.Hash([0], 2))
    ex.push_batch(rb)
    ex.finish()
    assert sum(ex.execute(p).read_all().num_rows for p in range(2)) == 10
    ex.close()
    ctx.close()


def test_a_device_output_option_other_than_0_or_1_is_refused(harness):
    from datafusion_distributed_b200 import _native as nv

    ns, ctx = harness
    schema = pa.schema([("k", pa.int64())])
    cs = nv.ArrowSchemaStruct()
    schema._export_to_c(C.addressof(cs))
    h = C.c_void_p()
    opts = nv.DfdExecOptions(0, 0, 0, 0, 2)
    rc = ctx.lib.dfd_repartition_exec_create(ctx.handle, C.addressof(cs), (C.c_int32 * 1)(0), 1, 2, C.byref(opts), C.byref(h))
    C.CFUNCTYPE(None, C.c_void_p)(cs.release)(C.addressof(cs))
    assert rc == 1 and not h.value and b"device_output" in ctx.lib.dfd_last_error()
