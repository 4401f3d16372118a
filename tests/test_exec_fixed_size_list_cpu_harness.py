"""FixedSizeList payload through the host operator on the CPU harness.

The bodies of tests/test_exec_fixed_size_list_gpu.py run against the product's dfd_exec object linked with the stand-in CUDA
runtime, the host restatements of the staging and emit launches, and tests/cpu_harness/harness_bit_rows.cu: the harness's
partitioner with a host stand-in of the bit-row gather (k_gather_bit_rows).  What this checks is the operator's host logic —
the schema walk, host and device staging of values and bit rows, chunk sizing, the nested output arrays of host and device
chunks — plus a leak check and a fault-injection sweep; the kernels are checked by -m gpu."""
import ctypes as C
import gc

import pyarrow as pa
import pytest

from tests.test_exec_cpu_harness import _Ctx
from tests.test_exec_device_output_cpu_harness import _build_output_harness, _namespace

SOURCES = ("harness_bit_rows.cu", "harness_stage.cu", "harness_emit.cu")  # (harness_bit_rows.cu includes harness_dfd.cu)


@pytest.fixture(scope="module")
def harness(built, tmp_path_factory):
    lib = C.CDLL(_build_output_harness(str(tmp_path_factory.mktemp("exec_fsl_harness")), sources=SOURCES))
    lib.harness_live_allocations.restype = C.c_long
    lib.harness_fail_nth.argtypes = [C.c_int, C.c_long]
    ns = _namespace(lib)
    ctx = _Ctx(lib)
    yield ns, ctx
    ctx.close()


def _bind(monkeypatch, harness):
    from tests import device_batches as DB
    from tests import device_outputs as DO
    from tests import test_exec_fixed_size_list_gpu as G

    ns, ctx = harness
    monkeypatch.setattr(G, "dfd", ns)
    monkeypatch.setattr(DB, "ALLOC", DB.host_alloc)
    monkeypatch.setattr(DO, "COPY", DO.host_copy)
    monkeypatch.setattr(DO, "WAIT", None)
    return G, ctx


CASES = ([("test_every_child_type", ())] + [("check_n", (n, c)) for n in (1, 3, 8, 33, 768) for c in ("f32", "bool")] +
         [("check_nulls", (c,)) for c in ("parent", "child", "both", "no_bitmap", "null_count_zero", "non_nullable_child")] +
         [("check_slicing", (t,)) for t in (pa.int16(), pa.bool_())] + [("check_batching", (r,)) for r in (0, 64, 1000)] +
         [("check_mixed_schema", (N,)) for N in (1, 3, 17)] + [("check_chunk_sizing", ())])


@pytest.mark.parametrize("body,args", CASES, ids=[f"{b}-{'-'.join(map(str, a))}" for b, a in CASES])
def test_fixed_size_list_host_logic(harness, monkeypatch, body, args):
    G, ctx = _bind(monkeypatch, harness)
    getattr(G, body)(ctx, *args)


def _batches(G, n=1500):
    import numpy as np

    rng = np.random.Generator(np.random.PCG64(5))
    col = G.fsl_array(rng, pa.float32(), 7, n, parent_nulls=0.1, child_nulls=0.2, offset=3, child_offset=2)
    bits = G.fsl_array(rng, pa.bool_(), 9, n, child_nulls=0.1)
    rb = G._batch(G._keys(rng, n), col, bits)
    return [rb.slice(lo, 500) for lo in range(0, n, 500)]


def test_no_allocation_outlives_the_operators(harness, monkeypatch):
    """Every stand-in device / pinned allocation of FixedSizeList operators in the four modes is freed with them and their context."""
    G, _ = _bind(monkeypatch, harness)
    ns, hctx = harness
    lib = hctx.lib
    base = lib.harness_live_allocations()
    ctx = _Ctx(lib)
    b = _batches(G)
    for mode in G.MODES:
        G.run_mode(ctx, mode, b[0].schema, b, [0], 4, chunk_rows=512)
    ctx.close()
    gc.collect()
    assert lib.harness_live_allocations() == base


@pytest.mark.parametrize("what,name", [(0, "cudaMalloc"), (1, "cudaHostAlloc"), (2, "cudaMemcpyAsync")])
@pytest.mark.parametrize("mode", ["hh", "dd"])
def test_injected_cuda_failures_surface_as_errors_and_leak_nothing(harness, monkeypatch, what, name, mode):
    """Fail the n-th cudaMalloc / cudaHostAlloc / cudaMemcpyAsync of a FixedSizeList operator's life: an error comes back,
    never a crash, and once everything is closed no allocation is left behind."""
    G, _ = _bind(monkeypatch, harness)
    ns, hctx = harness
    lib = hctx.lib
    b = _batches(G)
    failures = 0
    for n in list(range(1, 40)) + [60, 90, 150]:
        base = lib.harness_live_allocations()
        ctx = _Ctx(lib)
        lib.harness_fail_nth(what, n)
        try:
            # (the output batches are dropped here: they hold the chunks the leak check counts)
            assert sum(x.num_rows for s in G.run_mode(ctx, mode, b[0].schema, b, [0], 4, chunk_rows=512)[0] for x in s) == 1500
        except (ns.DfdError, pa.ArrowException, OSError) as e:
            failures += 1
            assert "fake CUDA" in str(e) or "failed" in str(e) or "alloc" in str(e).lower() or "cuda" in str(e).lower(), str(e)
        finally:
            lib.harness_fail_nth(what, 0)
            ctx.close()
            gc.collect()
        assert lib.harness_live_allocations() == base, (name, n)
    assert failures >= (5 if mode == "hh" or what == 0 else 1), (name, failures)  # (device in, device out: few pinned allocations / copies)
