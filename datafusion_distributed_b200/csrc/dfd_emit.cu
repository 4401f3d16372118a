// dfd_emit.cu — finishing a DEVICE-resident output chunk of the host operator (dfd_repartition_exec_execute_device).
//
// A host-output chunk is finished on a CPU thread once its D2H copy has landed: dfd::host::build_views walks every row of
// a view column, and a scalar loop turns the gathered byte offsets of a list's lengths column into element offsets.  A
// device-output chunk never leaves the GPU, so k_emit_chunk does both there, for ALL such columns of a chunk in ONE launch
// on the compute stream behind the partition kernels: a table of jobs, blockIdx.y picks the job (as in k_stage_batch).
#include <cuda_runtime.h>

#include "dfd_internal.h"

namespace {

constexpr int EMIT_BLOCK = 256;
constexpr int EMIT_MAX_GRID_X = 1024;
constexpr int EMIT_MAX_JOBS = 32;

struct EmitTable {
    int32_t n_jobs;
    dfd::EmitJob jobs[EMIT_MAX_JOBS];
};

// the low k bytes of a little-endian word (k <= 0: none, k >= 4: all)
__device__ __forceinline__ uint32_t low_bytes(int k) { return k <= 0 ? 0u : k >= 4 ? ~0u : (1u << (8 * k)) - 1u; }

}  // namespace

__global__ void __launch_bounds__(EMIT_BLOCK) k_emit_chunk(const __grid_constant__ EmitTable t) {
    const dfd::EmitJob& j = t.jobs[blockIdx.y];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    if (j.op == dfd::EMIT_LIST_OFFSETS) {
        int32_t* off = (int32_t*)j.dst;
        for (int64_t r = tid; r <= j.n; r += stride) off[r] >>= 2;
        return;
    }
    const int32_t* __restrict__ off = (const int32_t*)j.off;
    const uint32_t* __restrict__ words = (const uint32_t*)j.bytes;  // (the bytes buffer starts 4-byte aligned)
    uint4* __restrict__ views = (uint4*)j.dst;
    if (tid == 0) *(int64_t*)j.dst2 = (int64_t)off[j.n];  // the array's one variadic data buffer holds the chunk's bytes
    for (int64_t r = tid; r < j.n; r += stride) {
        const int32_t o = off[r], len = off[r + 1] - o;
        // bytes [o, o + take) sit at any byte alignment: the aligned words that hold them, funnel-shifted into place.  A word is
        // loaded only when it holds one of those bytes, so nothing past the last string byte's word is read
        const int32_t take = len > 12 ? 4 : len, sh = (o & 3) * 8;
        const int64_t end = (int64_t)o + take, w0 = o >> 2;
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) w[k] = (w0 + k) * 4 < end ? words[w0 + k] : 0u;
        uint4 v;
        v.x = (uint32_t)len;
        v.y = __funnelshift_r(w[0], w[1], sh) & low_bytes(take);
        if (len > 12) {  // length | 4-byte prefix | buffer index 0 | offset
            v.z = 0u;
            v.w = (uint32_t)o;
        } else {         // length | up to 12 inline bytes, zero padded
            v.z = __funnelshift_r(w[1], w[2], sh) & low_bytes(take - 4);
            v.w = __funnelshift_r(w[2], w[3], sh) & low_bytes(take - 8);
        }
        views[r] = v;  // one 16-byte store
    }
}

int dfd::launch_emit_chunk(const EmitJob* jobs, int n_jobs, cudaStream_t s) {
    for (int j0 = 0; j0 < n_jobs; j0 += EMIT_MAX_JOBS) {
        EmitTable t;
        t.n_jobs = n_jobs - j0 < EMIT_MAX_JOBS ? n_jobs - j0 : EMIT_MAX_JOBS;
        int64_t units = 1;
        for (int k = 0; k < t.n_jobs; ++k) {
            t.jobs[k] = jobs[j0 + k];
            if (t.jobs[k].n + 1 > units) units = t.jobs[k].n + 1;
        }
        const int64_t g = (units + EMIT_BLOCK - 1) / EMIT_BLOCK;
        k_emit_chunk<<<dim3((unsigned)(g > EMIT_MAX_GRID_X ? EMIT_MAX_GRID_X : g), (unsigned)t.n_jobs), EMIT_BLOCK, 0, s>>>(t);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_error(e, "k_emit_chunk");
    }
    return DFD_OK;
}
