// writeout_patterns.cu — the write side of the cfg-2 single-pass scatter and nothing else (scripts/writeout_patterns.py).
//
// Each tile of T = 2560 input rows is split into 8 destination runs whose lengths and exact output offsets come from the
// host.  Slot i of a tile, in destination order, is read from input row row0 + i (sequential reads, 8 B per row and
// column) and written to the output row of its run, with consecutive lanes on consecutive output rows as in
// k_scatter_onepass.  No hashing, ranking or look-back: only the store pattern differs between the instantiations.
//   PAT 0  8-byte lanes, runs at their own row alignment (the kernel today)
//   PAT 1  8-byte lanes, each run padded so that every warp's 32 rows are one aligned 256-B span
//   PAT 2  16-byte row pairs on even output rows; a run's odd head row and odd tail row are single 8-byte stores
//   PAT 3  PAT 2, each run padded so that every warp's 32 pairs are one aligned 512-B span
// CS: st.global.cs (streaming) stores, else the default policy.
#include <cstdint>

#include <cuda_runtime.h>

namespace {

constexpr int THREADS = 256;
constexpr int T = 2560;
constexpr int D = 8;
constexpr int MAX_COLS = 8;

struct Args {
    const unsigned long long* in[MAX_COLS];
    unsigned long long* out[MAX_COLS];
    const uint32_t* cnt;   // [n_tiles][D] rows of each run
    const uint32_t* orow;  // [n_tiles][D] output row of each run's first row
    long long n_rows;
    int n_tiles, n_cols;
};

template <bool CS>
__device__ __forceinline__ void st8(unsigned long long* p, unsigned long long v) {
    if (CS) asm volatile("st.global.cs.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
    else asm volatile("st.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
template <bool CS>
__device__ __forceinline__ void st16(unsigned long long* p, unsigned long long a, unsigned long long b) {
    if (CS) asm volatile("st.global.cs.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
    else asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}

// items per thread: rows (PAT 0), padded rows (PAT 1: < 62 pad per run), pairs (PAT 2: one extra per run),
// padded pairs (PAT 3: < 62 pad per run)
template <int PAT>
__host__ __device__ constexpr int items() {
    return PAT == 0 ? T / THREADS
         : PAT == 1 ? (T + 62 * D + THREADS - 1) / THREADS
         : PAT == 2 ? (T / 2 + D + THREADS - 1) / THREADS
                    : (T / 2 + D + 62 * D + THREADS - 1) / THREADS;
}

template <int PAT, bool CS>
__global__ void __launch_bounds__(THREADS) k_writeout(const __grid_constant__ Args A) {
    constexpr int KI = items<PAT>();
    __shared__ uint32_t TS[D + 1], VS[D + 1], O0[D], CNT[D];
    for (int tile = blockIdx.x; tile < A.n_tiles; tile += gridDim.x) {
        const long long row0 = (long long)tile * T;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t ts = 0, vs = 0;
            for (int d = 0; d < D; ++d) {
                const uint32_t c = A.cnt[tile * D + d], o = A.orow[tile * D + d];
                TS[d] = ts;
                VS[d] = vs;
                O0[d] = o;
                CNT[d] = c;
                ts += c;
                const uint32_t pairs = c ? ((o + c + 1) >> 1) - (o >> 1) : 0;
                if (PAT == 0) vs += c;
                if (PAT == 1) vs += c ? (c + (o & 31u) + 31u) & ~31u : 0;
                if (PAT == 2) vs += pairs;
                if (PAT == 3) vs += pairs ? (pairs + ((o >> 1) & 31u) + 31u) & ~31u : 0;
            }
            TS[D] = ts;
            VS[D] = vs;
        }
        __syncthreads();
        // this thread's items: output row (first row of the pair), source slot, live-row mask (bit 0: row, bit 1: row + 1)
        uint32_t orow[KI], src[KI], mask[KI];
#pragma unroll
        for (int k = 0; k < KI; ++k) {
            const uint32_t v = k * THREADS + threadIdx.x;
            mask[k] = 0;
            orow[k] = 0;
            src[k] = 0;
            if (v >= VS[D]) continue;
            int d = 0;
#pragma unroll
            for (int e = 1; e < D; ++e) d += v >= VS[e];
            const uint32_t r = v - VS[d], o = O0[d], c = CNT[d];
            if (PAT == 0) {
                orow[k] = o + r;
                src[k] = TS[d] + r;
                mask[k] = 1;
            } else if (PAT == 1) {
                const uint32_t head = o & 31u;
                if (r >= head && r < head + c) {
                    orow[k] = o - head + r;
                    src[k] = TS[d] + r - head;
                    mask[k] = 1;
                }
            } else {
                uint32_t q = r;
                if (PAT == 3) {
                    q = r - ((o >> 1) & 31u);  // wraps in the head pad: dead
                    if (q >= ((o + c + 1) >> 1) - (o >> 1)) continue;
                }
                const uint32_t pr = ((o >> 1) + q) * 2u;
                const bool lo = pr >= o, hi = pr + 1u < o + c;
                orow[k] = lo ? pr : pr + 1u;
                src[k] = TS[d] + orow[k] - o;
                mask[k] = lo && hi ? 3u : 1u;
            }
        }
#pragma unroll 1
        for (int col = 0; col < A.n_cols; ++col) {
            const unsigned long long* in = A.in[col] + row0;
            unsigned long long* out = A.out[col];
#pragma unroll
            for (int k = 0; k < KI; ++k) {
                if (mask[k] == 3u) st16<CS>(out + orow[k], in[src[k]], in[src[k] + 1]);
                else if (mask[k]) st8<CS>(out + orow[k], in[src[k]]);
            }
        }
    }
}

template <int PAT, bool CS>
int launch(const Args& a, int grid, cudaStream_t s) {
    k_writeout<PAT, CS><<<grid, THREADS, 0, s>>>(a);
    return (int)cudaGetLastError();
}

}  // namespace

// pattern 0..3 (see the top of the file); returns a cudaError_t
extern "C" int writeout_launch(int pattern, int cs, const void* const* in, void* const* out, int n_cols, const uint32_t* cnt,
                               const uint32_t* orow, long long n_rows, int n_tiles, int grid, void* stream) {
    if (n_cols < 1 || n_cols > MAX_COLS) return (int)cudaErrorInvalidValue;
    Args a{};
    for (int c = 0; c < n_cols; ++c) {
        a.in[c] = (const unsigned long long*)in[c];
        a.out[c] = (unsigned long long*)out[c];
    }
    a.cnt = cnt;
    a.orow = orow;
    a.n_rows = n_rows;
    a.n_tiles = n_tiles;
    a.n_cols = n_cols;
    cudaStream_t s = (cudaStream_t)stream;
    switch (pattern * 2 + (cs ? 1 : 0)) {
        case 0: return launch<0, false>(a, grid, s);
        case 1: return launch<0, true>(a, grid, s);
        case 2: return launch<1, false>(a, grid, s);
        case 3: return launch<1, true>(a, grid, s);
        case 4: return launch<2, false>(a, grid, s);
        case 5: return launch<2, true>(a, grid, s);
        case 6: return launch<3, false>(a, grid, s);
        case 7: return launch<3, true>(a, grid, s);
        default: return (int)cudaErrorInvalidValue;
    }
}

// resident CTAs per SM of a pattern's kernel (the persistent grid is a multiple of the SM count, at most this)
extern "C" int writeout_occupancy(int pattern, int* per_sm) {
    const void* f = pattern == 0 ? (const void*)k_writeout<0, true>
                  : pattern == 1 ? (const void*)k_writeout<1, true>
                  : pattern == 2 ? (const void*)k_writeout<2, true>
                                 : (const void*)k_writeout<3, true>;
    return (int)cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, f, THREADS, 0);
}
