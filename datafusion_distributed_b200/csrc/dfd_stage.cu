// dfd_stage.cu — device-side chunk assembly for DEVICE-resident input batches (dfd_repartition_exec_push_device).
//
// The host operator (dfd_exec.cu) builds the same chunk layout as for host batches — fixed-width values appended,
// bitmaps concatenated at bit granularity, string offsets re-based onto the chunk's byte buffer, views converted to
// offsets + bytes, lists split into their three hidden columns — but here every buffer is written on the device, straight
// from the producer's buffers.  All appends of one pushed batch are ONE launch of k_stage_batch: a table of jobs, one
// per (column, buffer), blockIdx.y picks the job.  k_stage_sizes reads what the host needs to know of variable-width
// columns before it can place their bytes (byte ranges, list element ranges, view byte totals).
#include <cuda_runtime.h>

#include "dfd_internal.h"

namespace {

constexpr int STAGE_BLOCK = 256;
constexpr int STAGE_MAX_GRID_X = 512;

struct StageTable {
    int32_t n_jobs;
    dfd::StageJob jobs[dfd::STAGE_MAX_JOBS];
};
struct SizeTable {
    int32_t n_jobs;
    dfd::StageSize jobs[dfd::STAGE_MAX_JOBS];
};

// dst[0, n) = src[0, n) in units of U once src and dst agree modulo sizeof(U): bytes up to the first aligned unit, units,
// then the remaining bytes
template <typename U>
__device__ __forceinline__ void copy_units(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int64_t n, int64_t tid, int64_t stride) {
    const int64_t mis = (int64_t)((sizeof(U) - ((uintptr_t)dst & (sizeof(U) - 1))) & (sizeof(U) - 1));
    const int64_t head = mis < n ? mis : n;
    const int64_t body = (n - head) / (int64_t)sizeof(U);
    const int64_t tail = head + body * (int64_t)sizeof(U);
    for (int64_t i = tid; i < head; i += stride) dst[i] = src[i];
    const U* s = (const U*)(src + head);
    U* d = (U*)(dst + head);
    for (int64_t i = tid; i < body; i += stride) d[i] = s[i];
    for (int64_t i = tail + tid; i < n; i += stride) dst[i] = src[i];
}

__device__ __forceinline__ void stage_copy(const uint8_t* src, uint8_t* dst, int64_t n, int64_t tid, int64_t stride) {
    const uintptr_t x = (uintptr_t)src ^ (uintptr_t)dst;
    if ((x & 15) == 0) copy_units<uint4>(src, dst, n, tid, stride);
    else if ((x & 7) == 0) copy_units<uint2>(src, dst, n, tid, stride);
    else if ((x & 3) == 0) copy_units<uint32_t>(src, dst, n, tid, stride);
    else copy_units<uint8_t>(src, dst, n, tid, stride);
}

// bits [p0, p0 + 32) of the bitmap `src`, as one word; bits outside [lo, hi) read as 0 and bytes outside that range are not
// touched (the producer's buffer may end there)
__device__ __forceinline__ uint32_t load_bits32(const uint8_t* __restrict__ src, int64_t p0, int64_t lo, int64_t hi) {
    const int64_t byte0 = p0 >= 0 ? p0 >> 3 : -((-p0 + 7) >> 3);
    const int sh = (int)(p0 - byte0 * 8);
    const int64_t blo = lo >> 3, bhi = (hi - 1) >> 3;
    uint32_t w0 = 0, w1 = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int64_t bi = byte0 + k;
        if (bi >= blo && bi <= bhi) w0 |= (uint32_t)src[bi] << (8 * k);
    }
    if (byte0 + 4 >= blo && byte0 + 4 <= bhi) w1 = src[byte0 + 4];
    return __funnelshift_r(w0, w1, sh);  // (the k_push_runs idea: two words, one funnel shift)
}

// bits k of a 32-bit word whose bit 0 is bitmap position p0, for the positions in [lo, hi)
__device__ __forceinline__ uint32_t range_mask(int64_t p0, int64_t lo, int64_t hi) {
    const int64_t l = lo - p0 > 0 ? lo - p0 : 0, h = hi - p0 < 32 ? hi - p0 : 32;
    if (h <= l) return 0u;
    const uint64_t m = ((h >= 32 ? ~0ull : ((1ull << h) - 1)) & ~((1ull << l) - 1));
    return (uint32_t)m;
}

__device__ __forceinline__ int64_t load_off(const void* p, int ow, int64_t i) {
    return ow == 8 ? ((const int64_t*)p)[i] : (int64_t)((const int32_t*)p)[i];
}

}  // namespace

__global__ void __launch_bounds__(STAGE_BLOCK) k_stage_batch(const __grid_constant__ StageTable t) {
    const dfd::StageJob j = t.jobs[blockIdx.y];  // (a copy: registers, no local-memory round trip)
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    switch (j.op) {
        case dfd::STAGE_COPY:
            stage_copy((const uint8_t*)j.src, (uint8_t*)j.dst, j.n, tid, stride);
            break;
        case dfd::STAGE_BITS: {
            const int64_t end = j.b + j.n;
            if (end <= j.c) break;
            uint32_t* dst = (uint32_t*)j.dst;
            const uint8_t* src = (const uint8_t*)j.src;
            for (int64_t w = (j.c >> 5) + tid; w <= (end - 1) >> 5; w += stride) {
                const int64_t p0 = w * 32;
                const uint32_t v = src ? load_bits32(src, j.a + (p0 - j.b), j.a, j.a + j.n) : ~0u;
                const uint32_t keep = range_mask(p0, p0, j.c);  // bits below c: what earlier appends wrote
                uint32_t out = (v & range_mask(p0, j.b, end)) | range_mask(p0, j.c, j.b);
                if (keep) out |= dst[w] & keep;
                dst[w] = out;
            }
            break;
        }
        case dfd::STAGE_OFFSETS: {
            const int64_t first = load_off(j.src, j.ow_in, 0);
            for (int64_t r = tid; r <= j.n; r += stride) {
                const int64_t v = j.base + j.scale * (load_off(j.src, j.ow_in, r) - first);
                if (j.ow_out == 8) ((int64_t*)j.dst)[r] = v;
                else ((int32_t*)j.dst)[r] = (int32_t)v;
            }
            break;
        }
        case dfd::STAGE_LIST_OFFSETS: {
            const int32_t* loff = (const int32_t*)j.src;
            const int32_t* coff = (const int32_t*)j.src2;
            const int64_t first = coff[loff[0]];
            for (int64_t r = tid; r <= j.n; r += stride) ((int32_t*)j.dst)[r] = (int32_t)(j.base + coff[loff[r]] - first);
            break;
        }
        case dfd::STAGE_DIFF32: {
            const int32_t* s = (const int32_t*)j.src;
            for (int64_t k = tid; k < j.n; k += stride) ((int32_t*)j.dst)[k] = s[k + 1] - s[k];
            break;
        }
        case dfd::STAGE_FILL32:
            for (int64_t k = tid; k < j.n; k += stride) ((int32_t*)j.dst)[k] = (int32_t)j.base;
            break;
        case dfd::STAGE_BIT_BYTES: {
            const uint8_t* s = (const uint8_t*)j.src;
            for (int64_t k = tid; k < j.n; k += stride)
                ((uint8_t*)j.dst)[k] = s ? (uint8_t)((s[(j.a + k) >> 3] >> ((j.a + k) & 7)) & 1) : (uint8_t)1;
            break;
        }
        case dfd::STAGE_VIEW_BYTES: {
            const uint8_t* views = (const uint8_t*)j.src;
            const uint8_t* const* bufs = (const uint8_t* const*)j.src2;
            const int32_t* off = (const int32_t*)j.src3;
            for (int64_t r = tid; r < j.n; r += stride) {
                const int32_t o = off[r], len = off[r + 1] - o;
                if (len <= 0) continue;
                const uint8_t* v = views + r * 16;
                const uint8_t* src = v + 4;
                if (len > 12) {
                    const int32_t buf = *(const int32_t*)(v + 8), pos = *(const int32_t*)(v + 12);
                    src = bufs[buf] + pos;
                }
                uint8_t* d = (uint8_t*)j.dst + o;
                for (int32_t k = 0; k < len; ++k) d[k] = src[k];
            }
            break;
        }
    }
}

__global__ void __launch_bounds__(STAGE_BLOCK) k_stage_sizes(const __grid_constant__ SizeTable t) {
    const dfd::StageSize& j = t.jobs[blockIdx.y];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    if (j.op == dfd::STAGE_SIZE_VIEW) {
        unsigned long long sum = 0;
        for (int64_t r = tid; r < j.n; r += stride) {
            const int64_t i = j.lo + r;
            int32_t len = *(const int32_t*)((const uint8_t*)j.off + i * 16);
            if (j.valid && !((j.valid[i >> 3] >> (i & 7)) & 1)) len = 0;
            j.lens[r] = len;
            sum += (unsigned long long)(int64_t)len;
        }
        __shared__ unsigned long long part[STAGE_BLOCK / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = sum;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long s = 0;
            for (int w = 0; w < STAGE_BLOCK / 32; ++w) s += part[w];
            if (s) atomicAdd((unsigned long long*)j.out, s);
        }
        return;
    }
    if (tid != 0) return;
    const int64_t a = load_off(j.off, j.ow, j.lo), b = load_off(j.off, j.ow, j.lo + j.n);
    j.out[0] = a;
    j.out[1] = b;
    if (j.op == dfd::STAGE_SIZE_LIST && j.off2 && a >= 0 && b >= a) {
        j.out[2] = ((const int32_t*)j.off2)[a];
        j.out[3] = ((const int32_t*)j.off2)[b];
    }
}

namespace {
int64_t job_units(const dfd::StageJob& j) {
    switch (j.op) {
        case dfd::STAGE_COPY: return j.n / 16 + 1;
        case dfd::STAGE_BITS: return (j.b + j.n - j.c + 31) / 32 + 1;
        case dfd::STAGE_OFFSETS: case dfd::STAGE_LIST_OFFSETS: return j.n + 1;
        default: return j.n;
    }
}
unsigned grid_x(int64_t units) {
    const int64_t g = (units + STAGE_BLOCK - 1) / STAGE_BLOCK;
    return (unsigned)(g < 1 ? 1 : g > STAGE_MAX_GRID_X ? STAGE_MAX_GRID_X : g);
}
}  // namespace

int dfd::launch_stage_batch(const StageJob* jobs, int n_jobs, cudaStream_t s) {
    for (int j0 = 0; j0 < n_jobs; j0 += STAGE_MAX_JOBS) {
        StageTable t;
        t.n_jobs = n_jobs - j0 < STAGE_MAX_JOBS ? n_jobs - j0 : STAGE_MAX_JOBS;
        int64_t units = 0;
        for (int k = 0; k < t.n_jobs; ++k) {
            t.jobs[k] = jobs[j0 + k];
            const int64_t u = job_units(t.jobs[k]);
            if (u > units) units = u;
        }
        k_stage_batch<<<dim3(grid_x(units), (unsigned)t.n_jobs), STAGE_BLOCK, 0, s>>>(t);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_error(e, "k_stage_batch");
    }
    return DFD_OK;
}

int dfd::launch_stage_sizes(const StageSize* jobs, int n_jobs, cudaStream_t s) {
    for (int j0 = 0; j0 < n_jobs; j0 += STAGE_MAX_JOBS) {
        SizeTable t;
        t.n_jobs = n_jobs - j0 < STAGE_MAX_JOBS ? n_jobs - j0 : STAGE_MAX_JOBS;
        int64_t units = 1;
        for (int k = 0; k < t.n_jobs; ++k) {
            t.jobs[k] = jobs[j0 + k];
            if (t.jobs[k].op == STAGE_SIZE_VIEW && t.jobs[k].n > units) units = t.jobs[k].n;
        }
        k_stage_sizes<<<dim3(grid_x(units), (unsigned)t.n_jobs), STAGE_BLOCK, 0, s>>>(t);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_error(e, "k_stage_sizes");
    }
    return DFD_OK;
}
