// dfd_launch.cuh — tile geometry and the template dispatch of the scatter kernels.
// launch_scatter_impl<PEER, KIND> is explicitly instantiated once per (PEER, KIND), each in a translation unit of its own
// (dfd_scatter_<kind>_<local|peer>.cu), so that the kernels compile in parallel.  Everywhere else the extern template
// declarations in dfd_internal.h keep the compiler from instantiating it again: dfd_api.cu includes this header for the
// tile geometry only.
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>
#include <type_traits>

#include "dfd_internal.h"
#include "dfd_kernels.cuh"

namespace dfd {

// Tile geometry of K1/K2 (rows per CTA = THREADS * K).
#ifndef DFD_TILE_THREADS
#define DFD_TILE_THREADS 256
#endif
#ifndef DFD_TILE_K
#define DFD_TILE_K 6
#endif
#ifndef DFD_TILE_MIN_CTAS
#define DFD_TILE_MIN_CTAS 6
#endif
// single-pass kernel: ring depth (sub-tile items in flight per CTA), items per column of a tile, resident CTAs per SM
#ifndef DFD_ONEPASS_NB
#define DFD_ONEPASS_NB 3
#endif
#ifndef DFD_ONEPASS_SPLIT
#define DFD_ONEPASS_SPLIT 1
#endif
#ifndef DFD_ONEPASS_MIN_CTAS
// (a register cap of 72 per thread; with NB = 3 a CTA needs 70.5 KB of shared memory at cfg-2, so 3 of them would fit per SM)
#define DFD_ONEPASS_MIN_CTAS 3
#endif
#ifndef DFD_ONEPASS_CTAS_PER_SM
// persistent grid: at most this many CTAs per SM (fewer if the occupancy API says so).  3 fit at cfg-2 but the store
// stream of 3 runs slower than that of 2 on H100 (DESIGN.md 4.1)
#define DFD_ONEPASS_CTAS_PER_SM 2
#endif
#ifndef DFD_ONEPASS_K
#define DFD_ONEPASS_K 10  // rows per consumer thread per tile (tile = 256 x K rows): larger tiles amortise ranking / look-back
#endif
constexpr int ONEPASS_K = DFD_ONEPASS_K;
constexpr int FOLLOW_MIN_CTAS = 4;  // follow-up k_scatter launches on the single-pass tiling
constexpr int ONEPASS_NB = DFD_ONEPASS_NB;
constexpr int ONEPASS_SPLIT = DFD_ONEPASS_SPLIT;
constexpr int ONEPASS_MIN_CTAS = DFD_ONEPASS_MIN_CTAS;
constexpr int ONEPASS_CTAS_PER_SM = DFD_ONEPASS_CTAS_PER_SM;
constexpr int TILE_THREADS = DFD_TILE_THREADS;
constexpr int TILE_K = DFD_TILE_K;
constexpr int TILE_MIN_CTAS = DFD_TILE_MIN_CTAS;
// aligned write-out (see k_scatter and use_aligned): up to ALIGNED_MAX_N destinations; each run wastes < 62 virtual slots
constexpr uint32_t ALIGNED_MAX_N = 16;
static_assert(ALIGNED_MAX_N == PAIR_ALIGN_MAX_N, "the single-pass local write-out aligns warps for the same N");
// The aligned write-out gives NVLink peer stores full-size write packets, so only peer launches take it.  A local
// single-pass launch aligns its stores without it (its KV == K write-out stores warp-aligned output-row pairs, see
// k_scatter_onepass).
constexpr bool use_aligned(uint32_t N, bool peer) { return peer && N <= ALIGNED_MAX_N; }
constexpr int TILE_KV = TILE_K + (62 * (int)ALIGNED_MAX_N + TILE_THREADS - 1) / TILE_THREADS;
constexpr int TILE_ROWS = TILE_THREADS * TILE_K;
constexpr int ONEPASS_KV = ONEPASS_K + (62 * (int)ALIGNED_MAX_N + TILE_THREADS - 1) / TILE_THREADS;
constexpr int ONEPASS_ROWS = TILE_THREADS * ONEPASS_K;

// The most dynamic shared memory any scatter launch of a partitioner with N destinations can ask for: two-pass launches
// of every staged width (1 B also stands for bit columns), follow-up and single-pass launches where single-pass calls
// exist (N <= ONEPASS_MAX_N), local and peer, and for peer launches also with the aligned write-out wherever use_aligned
// turns it on (N <= ALIGNED_MAX_N).  dfd_partitioner_create refuses an N for which this exceeds 227 KiB, so no launch of
// an accepted partitioner fails for lack of shared memory.
inline size_t scatter_smem_worst(uint32_t N) {
    size_t worst = 0;
    const auto keep = [&worst](size_t b) { worst = b > worst ? b : worst; };
    for (const bool peer : {false, true}) {
        for (const bool aligned : {false, true}) {
            if (aligned && !use_aligned(N, peer)) continue;
            for (const int width : {1, 2, 4, 8, 16}) {
                keep(scatter_smem_bytes<TILE_THREADS, TILE_K>(N, width, peer, aligned));
                if (N > ONEPASS_MAX_N) continue;
                keep(scatter_smem_bytes<TILE_THREADS, ONEPASS_K>(N, width, peer, aligned));
                if (width <= 8) keep(onepass_smem_bytes<TILE_THREADS, ONEPASS_K, ONEPASS_NB, ONEPASS_SPLIT>(N, width, peer, aligned));
            }
        }
    }
    return worst;
}

// KIND picks the kernel and its tiling (see ScatterKind), V the element type, ALIGNED the write-out.  The dynamic shared
// memory of every kind is sized and checked here.
template <bool FAST, typename V, bool PEER, bool ALIGNED, ScatterKind KIND>
static int launch_scatter_kv(const ScatterParams& sp, int sm_count, cudaStream_t stream) {
    cudaError_t e;
    if constexpr (KIND == ScatterKind::OnePass) {
        // run_onepass launches a ring of min(widest column, 8) bytes and takes the fast key path only with an 8-byte ring:
        // the other single-pass instantiations are never launched, so they are not compiled
        if constexpr (std::is_same<V, BitColumn>::value) {
            return set_error(DFD_ERR_INTERNAL, "bit-packed columns take the two-pass k_scatter");
        } else if constexpr (sizeof(V) > 8) {
            return set_error(DFD_ERR_INTERNAL, "the single-pass ring is at most 8 bytes wide");
        } else if constexpr (FAST && sizeof(V) < 8) {
            return set_error(DFD_ERR_INTERNAL, "the single-pass fast key path needs an 8-byte ring");
        } else {
            constexpr int KV = ALIGNED ? ONEPASS_KV : ONEPASS_K;
            auto kern = k_scatter_onepass<TILE_THREADS, ONEPASS_K, KV, ONEPASS_NB, ONEPASS_SPLIT, ONEPASS_MIN_CTAS, FAST, V, PEER>;
            const size_t smem = onepass_smem_bytes<TILE_THREADS, ONEPASS_K, ONEPASS_NB, ONEPASS_SPLIT>(sp.N, (int)sizeof(V), PEER, ALIGNED);
            if (smem > 227 * 1024) return set_error(DFD_ERR_UNSUPPORTED, "single-pass kernel needs %zu B of shared memory per CTA", smem);
            // (static per instantiation: the attribute and the occupancy are properties of the kernel + smem size)
            static thread_local size_t cfg_smem = 0;
            static thread_local int cfg_per_sm = 0;
            if (cfg_smem != smem) {
                if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
                    return cuda_error(e, "cudaFuncSetAttribute(k_scatter_onepass)");
                if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cfg_per_sm, kern, TILE_THREADS + 32, smem)) != cudaSuccess)
                    return cuda_error(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
                if (cfg_per_sm > ONEPASS_CTAS_PER_SM) cfg_per_sm = ONEPASS_CTAS_PER_SM;
                if (cfg_per_sm < 1) cfg_per_sm = 1;
                cfg_smem = smem;
            }
            int64_t grid = (int64_t)cfg_per_sm * sm_count;
            if (grid > sp.n_tiles) grid = sp.n_tiles;
            kern<<<(unsigned)grid, TILE_THREADS + 32, smem, stream>>>(sp);
        }
    } else {
        constexpr bool FOLLOW = KIND == ScatterKind::FollowUp;
        constexpr int K = FOLLOW ? ONEPASS_K : TILE_K;
        constexpr int KV = ALIGNED ? (FOLLOW ? ONEPASS_KV : TILE_KV) : K;
        constexpr int CTAS = FOLLOW ? FOLLOW_MIN_CTAS : TILE_MIN_CTAS;
        auto kern = k_scatter<TILE_THREADS, K, KV, CTAS, FAST, V, PEER>;
        const size_t smem = scatter_smem_bytes<TILE_THREADS, K>(sp.N, sp.stage_width, PEER, ALIGNED);
        if (smem > 227 * 1024)
            return set_error(DFD_ERR_UNSUPPORTED, "num_partitions %u needs %zu B of shared memory per CTA (k_scatter)", sp.N, smem);
        if (smem > 48 * 1024) {
            if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
                return cuda_error(e, "cudaFuncSetAttribute(k_scatter)");
        }
        kern<<<(unsigned)sp.n_tiles, TILE_THREADS, smem, stream>>>(sp);
    }
    e = cudaGetLastError();
    return e == cudaSuccess ? DFD_OK : cuda_error(e, "k_scatter");
}

template <bool FAST, typename V, bool PEER, ScatterKind KIND>
static int launch_scatter_t(const ScatterParams& sp, int sm_count, cudaStream_t stream) {
    if constexpr (PEER) {  // (so local launches compile no aligned instantiation)
        if (use_aligned(sp.N, PEER)) return launch_scatter_kv<FAST, V, PEER, true, KIND>(sp, sm_count, stream);
    }
    return launch_scatter_kv<FAST, V, PEER, false, KIND>(sp, sm_count, stream);
}

template <bool FAST, bool PEER, ScatterKind KIND>
static int launch_scatter_w(const ScatterParams& sp, int width, int sm_count, cudaStream_t stream) {
    switch (width) {
        case 8: return launch_scatter_t<FAST, uint64_t, PEER, KIND>(sp, sm_count, stream);
        case 4: return launch_scatter_t<FAST, uint32_t, PEER, KIND>(sp, sm_count, stream);
        case 2: return launch_scatter_t<FAST, uint16_t, PEER, KIND>(sp, sm_count, stream);
        case 1: return launch_scatter_t<FAST, uint8_t, PEER, KIND>(sp, sm_count, stream);
        case 16: return launch_scatter_t<FAST, uint4, PEER, KIND>(sp, sm_count, stream);
        default:
            if constexpr (PEER || KIND == ScatterKind::OnePass) {
                return set_error(DFD_ERR_INTERNAL, "bit-packed columns take the local k_scatter instantiation");
            } else {
                return launch_scatter_t<FAST, BitColumn, false, KIND>(sp, sm_count, stream);
            }
    }
}

template <bool PEER, ScatterKind KIND>
int launch_scatter_impl(const ScatterParams& sp, int width, bool fast, int sm_count, cudaStream_t stream) {
    return fast ? launch_scatter_w<true, PEER, KIND>(sp, width, sm_count, stream)
                : launch_scatter_w<false, PEER, KIND>(sp, width, sm_count, stream);
}

}  // namespace dfd
