// dfd_gather.cu — fixed-width payload columns that no scatter instantiation moves, gathered after K2 through d_src (the
// input row of every output row, the scattered iota column K4 also reads).
//
// k_gather_rows moves values of any width outside {1, 2, 4, 8, 16} bytes: the rows of a FixedSizeList column (an
// embedding of n floats is one 4n-byte value).  It reads every input row once and writes every output byte once; the
// only extra traffic is the 4-byte d_src entry per row (and the 4-byte iota row K2 scatters to build it).
//
// k_gather_bit_rows moves rows of n BITS: the child validity of a FixedSizeList<T, n> with a nullable child, or the values
// of a FixedSizeList<Boolean, n>.  Output bits [j n, (j + 1) n) are input bits [(in_offset + src[j]) n, ... + n).
#include <cuda_runtime.h>

#include "dfd_internal.h"

namespace {

constexpr int GATHER_BLOCK = 256;

// read-only, no L1 allocation: every source row is read once
template <typename U> __device__ __forceinline__ U ld_once(const U* p);
template <> __device__ __forceinline__ uint4 ld_once<uint4>(const uint4* p) {
    uint4 v;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
template <> __device__ __forceinline__ uint2 ld_once<uint2>(const uint2* p) {
    uint2 v;
    asm("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
template <> __device__ __forceinline__ uint32_t ld_once<uint32_t>(const uint32_t* p) {
    uint32_t v;
    asm("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
template <> __device__ __forceinline__ uint8_t ld_once<uint8_t>(const uint8_t* p) {
    uint32_t v;
    asm("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return (uint8_t)v;
}
__device__ __forceinline__ void st_once(uint4* p, uint4 v) { __stcs(p, v); }
__device__ __forceinline__ void st_once(uint2* p, uint2 v) { __stcs(p, v); }
__device__ __forceinline__ void st_once(uint32_t* p, uint32_t v) { __stcs((unsigned*)p, (unsigned)v); }
__device__ __forceinline__ void st_once(uint8_t* p, uint8_t v) { __stcs((unsigned char*)p, (unsigned char)v); }

}  // namespace

// out row j (w bytes) = in row in_offset + src[j], in units U (w, in and out are multiples of sizeof(U)).  A group of
// 2^lanes_log2 lanes copies one row, lane-strided: one lane per row below 16 bytes, else as many lanes as the row has
// units, up to a warp (a whole warp on a 16- or 24-byte row would leave most lanes idle).  Index arithmetic is 64-bit: rows x w passes 2^32 bytes for wide rows.
template <typename U>
__global__ void __launch_bounds__(GATHER_BLOCK) k_gather_rows(const uint8_t* __restrict__ in, int64_t in_offset, const uint32_t* __restrict__ src,
                                                             int64_t n_rows, int64_t w, uint8_t* __restrict__ out, int lanes_log2) {
    const int64_t units = w / (int64_t)sizeof(U);
    const int64_t lanes = 1ll << lanes_log2;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t lane = t & (lanes - 1), n_groups = ((int64_t)gridDim.x * blockDim.x) >> lanes_log2;
    for (int64_t j = t >> lanes_log2; j < n_rows; j += n_groups) {
        const U* __restrict__ s = (const U*)(in + ((int64_t)src[j] + in_offset) * w);
        U* __restrict__ d = (U*)(out + j * w);
        int64_t k = lane;
        for (; k + 3 * lanes < units; k += 4 * lanes) {  // four loads in flight before the first store
            const U a = ld_once(s + k), b = ld_once(s + k + lanes), c = ld_once(s + k + 2 * lanes), e = ld_once(s + k + 3 * lanes);
            st_once(d + k, a);
            st_once(d + k + lanes, b);
            st_once(d + k + 2 * lanes, c);
            st_once(d + k + 3 * lanes, e);
        }
        for (; k < units; k += lanes) st_once(d + k, ld_once(s + k));
    }
}

// One thread per output 32-bit word: it assembles the word from the (up to 32) row segments it covers, each read with at most
// two aligned 32-bit loads and one funnel shift, and stores it once.  No atomics, no read-modify-write: every run writes the
// same words.  A segment is read from the word that holds its first bit and, only when it crosses into it, the word that
// holds its last bit.  Bits past n_rows x n in the last word are zero.  All bit indices are 64-bit (4 Mi rows x 1024 bits
// is already 2^32 bits).
__global__ void __launch_bounds__(GATHER_BLOCK) k_gather_bit_rows(const uint32_t* __restrict__ in, int64_t in_bit0, const uint32_t* __restrict__ src,
                                                                  int64_t n_rows, int64_t n, uint32_t* __restrict__ out) {
    const int64_t total = n_rows * n, n_words = (total + 31) >> 5;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n_words; q += stride) {
        const int64_t o0 = q << 5, o1 = o0 + 32 < total ? o0 + 32 : total;
        int64_t j = o0 / n, row_end = (j + 1) * n;
        uint32_t acc = 0;
        for (int64_t o = o0; o < o1; ++j, row_end += n) {
            const int64_t seg_end = row_end < o1 ? row_end : o1;
            const int len = (int)(seg_end - o);
            const int64_t s = in_bit0 + (int64_t)__ldg(src + j) * n + (o - (row_end - n));  // first source bit of the segment
            const int sh = (int)(s & 31);
            const uint32_t lo = __ldg(in + (s >> 5));
            const uint32_t hi = sh + len > 32 ? __ldg(in + (s >> 5) + 1) : 0u;
            const uint32_t v = __funnelshift_r(lo, hi, sh);
            acc |= (len == 32 ? v : v & ((1u << len) - 1u)) << (int)(o - o0);
            o = seg_end;
        }
        __stcs((unsigned*)out + q, acc);
    }
}

namespace {

// enough CTAs to fill every SM once (grid-stride loops do the rest), fewer when the work is small
template <typename K>
unsigned gather_grid(K kernel, int64_t threads_needed, int sm_count) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, GATHER_BLOCK, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    const int64_t need = (threads_needed + GATHER_BLOCK - 1) / GATHER_BLOCK;
    const int64_t cap = (int64_t)per_sm * sm_count;
    return (unsigned)(need < 1 ? 1 : need < cap ? need : cap);
}

template <typename U>
int launch_rows(const void* in, int64_t in_offset, const uint32_t* src, int64_t n_rows, int64_t w, void* out, int sm_count, cudaStream_t s) {
    const int64_t units = w / (int64_t)sizeof(U);
    int lanes_log2 = 0;
    if (w >= 16)
        while (lanes_log2 < 5 && (1ll << lanes_log2) < units) ++lanes_log2;
    const unsigned grid = gather_grid(k_gather_rows<U>, n_rows << lanes_log2, sm_count);
    k_gather_rows<U><<<grid, GATHER_BLOCK, 0, s>>>((const uint8_t*)in, in_offset, src, n_rows, w, (uint8_t*)out, lanes_log2);
    CUDA_TRY(cudaGetLastError(), "k_gather_rows");
    return DFD_OK;
}

}  // namespace

int dfd::launch_gather_rows(const void* in, int64_t in_offset, const uint32_t* src, int64_t n_rows, int64_t w, void* out, int sm_count,
                            cudaStream_t s) {
    if (n_rows <= 0) return DFD_OK;
    // the widest copy unit the width and both base pointers allow
    const uint64_t a = (uint64_t)w | (uint64_t)(uintptr_t)in | (uint64_t)(uintptr_t)out;
    if ((a & 15) == 0) return launch_rows<uint4>(in, in_offset, src, n_rows, w, out, sm_count, s);
    if ((a & 7) == 0) return launch_rows<uint2>(in, in_offset, src, n_rows, w, out, sm_count, s);
    if ((a & 3) == 0) return launch_rows<uint32_t>(in, in_offset, src, n_rows, w, out, sm_count, s);
    return launch_rows<uint8_t>(in, in_offset, src, n_rows, w, out, sm_count, s);
}

int dfd::launch_gather_bit_rows(const void* in, int64_t in_offset, const uint32_t* src, int64_t n_rows, int64_t n, void* out, int sm_count,
                                cudaStream_t s) {
    if (n_rows <= 0) return DFD_OK;
    if (n < 1) return set_error(DFD_ERR_INVALID_ARGUMENT, "bit rows of %lld bits", (long long)n);
    if ((uintptr_t)out & 3) return set_error(DFD_ERR_INVALID_ARGUMENT, "bit-row output must be 4-byte aligned");
    // the input is read in aligned words: start at the word below it, its leading bytes count as bits
    const uintptr_t mis = (uintptr_t)in & 3;
    const int64_t bit0 = in_offset * n + (int64_t)mis * 8;
    const unsigned grid = gather_grid(k_gather_bit_rows, (n_rows * n + 31) >> 5, sm_count);
    k_gather_bit_rows<<<grid, GATHER_BLOCK, 0, s>>>((const uint32_t*)((const uint8_t*)in - mis), bit0, src, n_rows, n, (uint32_t*)out);
    CUDA_TRY(cudaGetLastError(), "k_gather_bit_rows");
    return DFD_OK;
}
