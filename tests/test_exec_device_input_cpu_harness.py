"""The device-input path of the host operator (dfd_repartition_exec_push_device) on the CPU harness.

The bodies of tests/test_exec_device_input_gpu.py run against the product's dfd_exec object linked with the stand-in CUDA
runtime and the host restatements of the staging kernels (tests/cpu_harness/harness_stage.cu): the "device" batches are
host copies, which the stand-in runtime treats as device memory.  What this checks is the operator's host logic around
the kernels — sizes read-back, chunk cuts, buffer growth, dictionary host copies, release of the pushed batches, the
refusals — and it is the view of that logic an address sanitizer can run (tests/cpu_harness/README.md)."""
import ctypes as C
import os
import subprocess

import pytest

from tests.test_exec_cpu_harness import CSRC, HARNESS, NVCC, NVCC_FLAGS, ROOT, _Ctx, _make_namespace


def _build_device_harness(tmp):
    """The host-logic harness of tests/test_exec_cpu_harness.py plus tests/cpu_harness/harness_stage.cu, the host restatement
    of the two staging launches (without it the operator object's weak references to them stay unresolved and push_device
    refuses every batch)."""
    if os.environ.get("DFD_TEST_DEVICE_HARNESS_SO"):  # a prebuilt variant, e.g. with -fsanitize=address (recipe below)
        return os.environ["DFD_TEST_DEVICE_HARNESS_SO"]
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
    for src in ("harness_dfd.cu", "harness_stage.cu"):
        objs.append(os.path.join(tmp, src.replace(".cu", ".o")))
        subprocess.check_call([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(HARNESS, src), "-o", objs[-1]])
    objs.append(os.path.join(tmp, "fake_cudart.o"))
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-Wall", "-c", os.path.join(HARNESS, "fake_cudart.cpp"), "-o", objs[-1]])
    out = os.path.join(tmp, "libdfd_exec_device_harness.so")
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", out] + objs + [oracle_so, f"-Wl,-rpath,{os.path.dirname(oracle_so)}", "-lpthread"])
    return out


# AddressSanitizer variant: the recipe of tests/cpu_harness/README.md with harness_stage.cu compiled like harness_dfd.cu and
# linked in, the library named by DFD_TEST_DEVICE_HARNESS_SO.


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    from datafusion_distributed_b200 import _native as nv

    lib = C.CDLL(_build_device_harness(str(tmp_path_factory.mktemp("exec_device_harness"))))
    ns = _make_namespace(lib)
    lib.dfd_repartition_exec_push_device.restype = C.c_int
    lib.dfd_repartition_exec_push_device.argtypes = [C.c_void_p, C.c_void_p]

    class RepartitionExec(ns.RepartitionExec):
        def push_device_batch(self, device_array):
            addr = device_array if isinstance(device_array, int) else C.addressof(device_array)
            rc = lib.dfd_repartition_exec_push_device(self._h, addr)
            if rc != 0:
                raise ns.DfdError(rc, lib.dfd_last_error().decode("utf-8", "replace"))

    ns.RepartitionExec = RepartitionExec
    ctx = _Ctx(lib)
    yield ns, ctx, nv
    ctx.close()


CASES = [
    ("test_fixed_width_batches", dict(batch_rows=8192, chunk_rows=0)),
    ("test_fixed_width_batches", dict(batch_rows=1024, chunk_rows=10_000)),
    ("test_fixed_width_batches", dict(batch_rows=100_000, chunk_rows=65_536)),
    ("test_nullable_bool_mixed_widths_sliced", dict(keys=[0])),
    ("test_nullable_bool_mixed_widths_sliced", dict(keys=[5, 2])),
    ("test_strings_as_keys_and_payload", dict(keys=[1])),
    ("test_strings_as_keys_and_payload", dict(keys=[3, 1])),
    ("test_all_empty_strings", {}),
    ("test_views_inline_and_out_of_line_over_several_buffers", {}),
    ("test_dictionary_payload_shared_and_cut_chunks", {}),
    ("test_lists_of_strings_binaries_and_primitives", {}),
    ("test_reference_fixture_schema_at_8192_row_batches", dict(keys=[0, 3])),
    ("test_large_binary_and_fixed_size_binary_payload", {}),
    ("test_back_pressure_with_concurrent_consumers", {}),
    ("test_abort_after_device_pushes_releases_the_batches", {}),
    ("test_refusals_release_the_batch_and_fail_the_operator", {}),
]


def _bind(monkeypatch, harness):
    from tests import device_batches as DB
    from tests import test_exec_device_input_gpu as G

    ns, ctx, _ = harness
    monkeypatch.setattr(G, "dfd", ns)
    monkeypatch.setattr(DB, "ALLOC", DB.host_alloc)
    return G, ctx


@pytest.mark.parametrize("name,kwargs", CASES, ids=[f"{n}-{i}" for i, (n, _) in enumerate(CASES)])
def test_device_input_host_logic(harness, monkeypatch, name, kwargs):
    G, ctx = _bind(monkeypatch, harness)
    getattr(G, name)(ctx, **kwargs)


def _key_cases():
    from tests import test_exec_keys_gpu as K

    return [("check_key_format", (f,)) for f in K.KEY_FORMATS] + [("check_dictionary_key", (i, v)) for i, v in K.DICT_CASES[::5]]


@pytest.mark.parametrize("body,args", _key_cases(), ids=[f"{b}-{'-'.join(map(str, a))}" for b, a in _key_cases()])
def test_device_input_key_types(harness, monkeypatch, body, args):
    G, ctx = _bind(monkeypatch, harness)
    getattr(G, body)(ctx, *args)


def test_device_input_leaves_no_allocation_behind(harness, monkeypatch):
    """Every stand-in device / pinned allocation the device path makes (sizes read-back, view scratch, dictionary hashes)
    is freed once the operators and their context are gone."""
    import gc

    G, _ = _bind(monkeypatch, harness)
    ns, hctx, _ = harness
    lib = hctx.lib
    lib.harness_live_allocations.restype = C.c_long
    base = lib.harness_live_allocations()
    ctx = _Ctx(lib)
    t = G.reference_fixture_table(3_000, 2)
    G.run_both(ctx, t.schema, t.to_batches(max_chunksize=500), [4, 3], 4, chunk_rows=1_024)
    ctx.close()
    gc.collect()
    assert lib.harness_live_allocations() == base


@pytest.mark.parametrize("what,name", [(0, "cudaMalloc"), (1, "cudaHostAlloc"), (2, "cudaMemcpyAsync")])
def test_injected_cuda_failures_on_device_input_surface_as_errors_and_leak_nothing(harness, what, name):
    """The device-input counterpart of test_exec_cpu_harness.py::test_injected_cuda_failures_surface_as_errors_and_leak_nothing:
    fail the n-th cudaMalloc / cudaHostAlloc / cudaMemcpyAsync of an operator fed device batches (create, sizes read-back,
    dictionary copies, staging, flush, D2H).  The failure comes back as an error, never a crash; once everything is closed
    no allocation is left behind, and every pushed batch has been released exactly once."""
    import gc

    import pyarrow as pa

    from tests import device_batches as DB
    from tests.test_exec_cpu_harness import _fixture_like_table

    ns, hctx, _ = harness
    lib = hctx.lib
    lib.harness_live_allocations.restype = C.c_long
    lib.harness_fail_nth.argtypes = [C.c_int, C.c_long]
    batches = _fixture_like_table(1500).to_batches(max_chunksize=500)
    failures = 0
    for n in list(range(1, 40)) + [60, 90, 150, 400]:
        base = lib.harness_live_allocations()
        ctx = _Ctx(lib)
        lib.harness_fail_nth(what, n)
        ex, pushed = None, []
        try:
            ex = ns.RepartitionExec(ctx, batches[0].schema, ns.Partitioning.Hash([4, 0], 4), chunk_rows=512)
            for rb in batches:
                b = DB.DeviceBatch(rb, alloc=DB.host_alloc)
                pushed.append(b.key)
                ex.push_device_batch(b.device_array)
            ex.finish()
            assert sum(ex.execute(p).read_all().num_rows for p in range(4)) == 1500  # (the failing call was not on this path)
        except (ns.DfdError, pa.ArrowException, OSError) as e:
            failures += 1
            assert "fake CUDA" in str(e) or "failed" in str(e) or "alloc" in str(e).lower() or "cuda" in str(e).lower(), str(e)
        finally:
            lib.harness_fail_nth(what, 0)
            if ex is not None:
                ex.close()
            ctx.close()
            gc.collect()
        assert not set(pushed) & DB.live_batches(), (name, n)
        assert sorted(k for k in DB.RELEASED if k in set(pushed)) == sorted(pushed), (name, n)  # each exactly once
        assert lib.harness_live_allocations() == base, (name, n)
    assert failures >= 5, (name, failures)


def test_an_operator_object_linked_without_the_staging_kernels_refuses_device_batches(built, tmp_path):
    """The host-logic harness WITHOUT harness_stage.cu: the operator object still loads (its references to the staging
    launches are weak), host batches work as ever, and a device batch is refused with DFD_ERR_UNSUPPORTED and released."""
    import pyarrow as pa

    from tests import device_batches as DB
    from tests.test_exec_cpu_harness import _build_harness

    lib = C.CDLL(_build_harness(str(tmp_path)))
    ns = _make_namespace(lib)
    lib.dfd_repartition_exec_push_device.restype = C.c_int
    lib.dfd_repartition_exec_push_device.argtypes = [C.c_void_p, C.c_void_p]
    ctx = _Ctx(lib)
    rb = pa.record_batch([pa.array(range(10), type=pa.int64())], names=["k"])
    ex = ns.RepartitionExec(ctx, rb.schema, ns.Partitioning.Hash([0], 2))
    b = DB.DeviceBatch(rb, alloc=DB.host_alloc)
    assert lib.dfd_repartition_exec_push_device(ex._h, C.addressof(b.device_array)) == 6  # DFD_ERR_UNSUPPORTED
    assert b"staging kernels" in lib.dfd_last_error()
    assert b.key not in DB.live_batches()
    ex.close()
    ex = ns.RepartitionExec(ctx, rb.schema, ns.Partitioning.Hash([0], 2))
    ex.push_batch(rb)
    ex.finish()
    assert sum(ex.execute(p).read_all().num_rows for p in range(2)) == 10
    ex.close()
    ctx.close()
