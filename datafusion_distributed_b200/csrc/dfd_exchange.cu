// dfd_exchange.cu — the inter-worker exchange of the shuffle over NVLink.
//
// Replaces the reference's data plane between stage N (producers) and stage
// N+1 (consumers):
//   server  Worker::impl_execute_task  (src/worker/impl_execute_task.rs:36-169)
//           Arrow-IPC/Flight encode + gRPC stream per (consumer, producer)
//   client  WorkerConnection demux + FlightRecordBatchStream decode
//           (src/worker/worker_connection_pool.rs:143-390)
//   NetworkShuffleExec::execute: off = P*task_index, partition off+p from every
//           producer (src/execution_plans/network_shuffle.rs:213-238)
// with one worker per GPU and four transports:
//   DFD_EXCHANGE_NCCL   partition locally, all-gather the T x N count matrix,
//                       grouped ncclSend/ncclRecv per (column, destination).
//   DFD_EXCHANGE_FUSED  the K2 scatter kernel stores every run straight into
//                       the owner rank's receive window (CUDA-IPC mapped peer
//                       memory over NVLink/NVSwitch): no staging buffer, no
//                       separate send — compute and transfer are one kernel.
//   single pass         (dfd_shuffle_device_onepass, fixed-width non-null) one
//                       scatter kernel stores into fixed (partition, producer)
//                       sub-windows; counts and completion are peer-memory flags.
//   push                (dfd_shuffle_device_onepass for every other schema, and
//                       dfd_exchange_gather) partition locally, then store each
//                       destination's contiguous runs into the owner's window.
// NCCL is resolved at run time (dlopen libnccl.so.2) so the single-GPU library
// has no link-time dependency on it.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "dfd_b200.h"
#include "dfd_internal.h"

using namespace dfd;

namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*CommAbort)(ncclComm_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    std::string error;
};

NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (!api.handle) {
            api.error = std::string("dlopen(libnccl.so.2) failed: ") + (dlerror() ? dlerror() : "");
            return;
        }
#define LOAD(field, sym)                                                   \
    api.field = (decltype(api.field))dlsym(api.handle, sym);             \
    if (!api.field) { api.error = std::string("missing NCCL symbol ") + sym; return; }
        LOAD(GetVersion, "ncclGetVersion");
        LOAD(GetUniqueId, "ncclGetUniqueId");
        LOAD(CommInitRank, "ncclCommInitRank");
        LOAD(CommDestroy, "ncclCommDestroy");
        LOAD(CommAbort, "ncclCommAbort");
        LOAD(GetErrorString, "ncclGetErrorString");
        LOAD(AllGather, "ncclAllGather");
        LOAD(AllReduce, "ncclAllReduce");
        LOAD(Send, "ncclSend");
        LOAD(Recv, "ncclRecv");
        LOAD(GroupStart, "ncclGroupStart");
        LOAD(GroupEnd, "ncclGroupEnd");
#undef LOAD
    });
    return &api;
}

int nccl_error(ncclResult_t r, const char* what) {
    NcclApi* n = nccl_api();
    return set_error(DFD_ERR_NCCL, "%s: %s", what, n->GetErrorString ? n->GetErrorString(r) : "NCCL error");
}

#define NCCL_TRY(call, what)                                   \
    {                                                          \
        ncclResult_t _r = (call);                              \
        if (_r != ncclSuccess) return nccl_error(_r, what);    \
    }

// dest_base / part_starts / overflow check on the device (fused mode), from the
// all-gathered count matrix counts[T][N]: no host round trip before K2.
__global__ void k_exchange_plan(const int64_t* __restrict__ counts, int world, uint32_t P, int rank, int64_t capacity_rows,
                                int64_t* __restrict__ dest_base /*[N]*/, int64_t* __restrict__ my_part_starts /*[P+1]*/,
                                int32_t* __restrict__ abort_flag) {
    const uint32_t N = P * (uint32_t)world;
    __shared__ int overflow;
    if (threadIdx.x == 0) overflow = 0;
    __syncthreads();
    // one thread per owner rank o: walk its P partitions
    for (int o = threadIdx.x; o < world; o += blockDim.x) {
        int64_t run = 0;
        for (uint32_t q = 0; q < P; ++q) {
            const uint32_t g = (uint32_t)o * P + q;
            if (o == rank) my_part_starts[q] = run;
            int64_t before_me = 0, tot = 0;
            for (int r = 0; r < world; ++r) {
                int64_t c = counts[(int64_t)r * N + g];
                if (r < rank) before_me += c;
                tot += c;
            }
            dest_base[g] = run + before_me;
            run += tot;
        }
        if (o == rank) my_part_starts[P] = run;
        if (run > capacity_rows) atomicExch(&overflow, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) *abort_flag = overflow;
}

// ---------------------------------------------------------------------------
// Peer-memory flags of the single-pass exchange (replace ncclAllGather(counts) + ncclAllReduce(barrier)).
// ---------------------------------------------------------------------------
// consumer side, start of a shuffle: "my window is free" -> every producer's header
__global__ void k_xchg_signal_ready(ExchangeHeader* const* __restrict__ peer_hdr, int rank, int world, unsigned long long epoch) {
    const int o = threadIdx.x;
    if (o < world) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&peer_hdr[o]->ready[rank]), "l"(epoch) : "memory");
    }
}

// producer side, end of a shuffle (stream-ordered after the scatter kernels): publish my per-destination counts and my
// overflow flag into every consumer's header, then the "landed" flag; then, as consumer, wait for every producer's flag.
__global__ void __launch_bounds__(256) k_xchg_publish_wait(ExchangeHeader* __restrict__ local, ExchangeHeader* const* __restrict__ peer_hdr, int rank, int world,
                                                           uint32_t P, unsigned long long epoch, const int64_t* __restrict__ totals /*[P*world]*/,
                                                           const int32_t* __restrict__ overflow, int32_t* __restrict__ timed_out) {
    const uint32_t N = P * (uint32_t)world;
    for (uint32_t g = threadIdx.x; g < N; g += blockDim.x) peer_hdr[g / P]->counts[rank][g % P] = totals[g];
    if ((int)threadIdx.x < world) peer_hdr[threadIdx.x]->overflow[rank] = *overflow;
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < world) {
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&peer_hdr[threadIdx.x]->done[rank]), "l"(epoch) : "memory");
        const long long t_start = clock64();
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(&local->done[threadIdx.x]) : "memory");
            if (v < epoch && clock64() - t_start > (1LL << 34)) {  // ~8 s: a peer never arrived (it failed before launching)
                *timed_out = 1;
                break;
            }
        } while (v < epoch);
    }
}

// ---- push transport: flag-based all-gather of per-producer metadata, then contiguous peer-store pushes ----
// Every worker writes its `n_meta` int64 counts into EVERY worker's header (meta[rank][..]), raises meta_flag[rank] = epoch
// there, and waits until all workers' flags have arrived in its own header: an all-gather over NVLink stores.
__global__ void __launch_bounds__(256) k_xchg_allgather_meta(ExchangeHeader* __restrict__ local, ExchangeHeader* const* __restrict__ peer_hdr, int rank,
                                                             int world, unsigned long long epoch, const int64_t* __restrict__ my_meta, uint32_t n_meta,
                                                             int32_t* __restrict__ timed_out) {
    for (int o = 0; o < world; ++o)
        for (uint32_t i = threadIdx.x; i < n_meta; i += blockDim.x) peer_hdr[o]->meta[rank][i] = my_meta[i];
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < world) {
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&peer_hdr[threadIdx.x]->meta_flag[rank]), "l"(epoch) : "memory");
        const long long t_start = clock64();
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(&local->meta_flag[threadIdx.x]) : "memory");
            if (v < epoch && clock64() - t_start > (1LL << 34)) {
                *timed_out = 1;
                break;
            }
        } while (v < epoch);
    }
}

// end-of-push barrier: "my pushes have landed" into every consumer's header; wait for every producer's flag
__global__ void k_xchg_done_barrier(ExchangeHeader* __restrict__ local, ExchangeHeader* const* __restrict__ peer_hdr, int rank, int world,
                                    unsigned long long epoch, int32_t* __restrict__ timed_out) {
    if ((int)threadIdx.x < world) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&peer_hdr[threadIdx.x]->done[rank]), "l"(epoch) : "memory");
        const long long t_start = clock64();
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(&local->done[threadIdx.x]) : "memory");
            if (v < epoch && clock64() - t_start > (1LL << 34)) {
                *timed_out = 1;
                break;
            }
        } while (v < epoch);
    }
}

// One contiguous run of a destination-sorted local column -> its segment in the owner's window.
struct PushRun {
    const char* src;
    char* dst;
    long long n;       // RUN_BYTES: bytes; RUN_BITS / RUN_ONES: rows (bits); RUN_OFF32 / RUN_OFF64: entries
    long long a, b;    // RUN_BITS: a = first source bit; RUN_OFF*: dst[k] = src[k] - a + b
    int kind;
    int first_block;   // first CTA of this run in the launch (prefix over the runs)
};
enum { RUN_BYTES = 0, RUN_BITS = 1, RUN_OFF32 = 2, RUN_OFF64 = 3, RUN_ONES = 4 };
constexpr int PUSH_THREADS = 256;
constexpr long long PUSH_CHUNK = 64 * 1024;  // bytes (RUN_BYTES) / output bytes (others) per CTA

__host__ __device__ inline long long push_run_out_bytes(const PushRun& r) {
    switch (r.kind) {
        case RUN_BYTES: return r.n;
        case RUN_BITS: case RUN_ONES: return (r.n + 31) / 32 * 4;
        case RUN_OFF32: return r.n * 4;
        default: return r.n * 8;
    }
}

__global__ void __launch_bounds__(PUSH_THREADS) k_push_runs(const PushRun* __restrict__ runs, int n_runs) {
    // which run does this CTA serve?  (binary search over first_block)
    int lo = 0, hi = n_runs;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (runs[mid].first_block <= (int)blockIdx.x) lo = mid; else hi = mid;
    }
    const PushRun r = runs[lo];
    const long long c0 = (long long)((int)blockIdx.x - r.first_block) * PUSH_CHUNK;  // first OUTPUT byte of this CTA's chunk
    const long long total = push_run_out_bytes(r);
    const long long c1 = c0 + PUSH_CHUNK < total ? c0 + PUSH_CHUNK : total;
    if (r.kind == RUN_BYTES) {
        const char* s = r.src + c0;
        char* d = r.dst + c0;
        const long long n = c1 - c0;
        const unsigned mis = (unsigned)(((uintptr_t)s ^ (uintptr_t)d) & 15u);
        if (mis == 0) {  // co-aligned: 16-byte body
            long long head = (16 - ((uintptr_t)d & 15u)) & 15u;
            if (head > n) head = n;
            for (long long i = threadIdx.x; i < head; i += PUSH_THREADS) d[i] = s[i];
            const long long body = (n - head) / 16;
            const uint4* s4 = (const uint4*)(s + head);
            uint4* d4 = (uint4*)(d + head);
            for (long long i = threadIdx.x; i < body; i += PUSH_THREADS) __stcs(d4 + i, __ldcs(s4 + i));
            for (long long i = head + body * 16 + threadIdx.x; i < n; i += PUSH_THREADS) d[i] = s[i];
        } else if ((mis & 7u) == 0) {  // 8-byte co-aligned (8-byte values at an odd row distance)
            long long head = (8 - ((uintptr_t)d & 7u)) & 7u;
            if (head > n) head = n;
            for (long long i = threadIdx.x; i < head; i += PUSH_THREADS) d[i] = s[i];
            const long long body = (n - head) / 8;
            const unsigned long long* s8 = (const unsigned long long*)(s + head);
            unsigned long long* d8 = (unsigned long long*)(d + head);
            for (long long i = threadIdx.x; i < body; i += PUSH_THREADS) __stcs(d8 + i, __ldcs(s8 + i));
            for (long long i = head + body * 8 + threadIdx.x; i < n; i += PUSH_THREADS) d[i] = s[i];
        } else if ((mis & 3u) == 0) {
            long long head = (4 - ((uintptr_t)d & 3u)) & 3u;
            if (head > n) head = n;
            for (long long i = threadIdx.x; i < head; i += PUSH_THREADS) d[i] = s[i];
            const long long body = (n - head) / 4;
            const unsigned* s4 = (const unsigned*)(s + head);
            unsigned* d4 = (unsigned*)(d + head);
            for (long long i = threadIdx.x; i < body; i += PUSH_THREADS) d4[i] = s4[i];
            for (long long i = head + body * 4 + threadIdx.x; i < n; i += PUSH_THREADS) d[i] = s[i];
        } else {
            for (long long i = threadIdx.x; i < n; i += PUSH_THREADS) d[i] = s[i];
        }
    } else if (r.kind == RUN_BITS) {
        // destination words are 32-row aligned (segments start on multiples of 32 rows); source starts at bit r.a
        const unsigned* sw = (const unsigned*)r.src;
        unsigned* dw = (unsigned*)r.dst;
        for (long long w = c0 / 4 + threadIdx.x; w < c1 / 4; w += PUSH_THREADS) {
            const long long bit = r.a + w * 32;
            const long long wi = bit >> 5;
            const unsigned sh = (unsigned)(bit & 31);
            const unsigned lo32 = sw[wi];
            // (the word after the last one may lie outside the bitmap: only read it when bits of it are needed)
            const bool need_hi = sh != 0 && (w * 32 + (32 - sh)) < r.n;
            const unsigned hi32 = need_hi ? sw[wi + 1] : 0u;
            dw[w] = sh ? __funnelshift_r(lo32, hi32, sh) : lo32;
        }
    } else if (r.kind == RUN_ONES) {
        unsigned* dw = (unsigned*)r.dst;
        for (long long w = c0 / 4 + threadIdx.x; w < c1 / 4; w += PUSH_THREADS) dw[w] = 0xffffffffu;
    } else if (r.kind == RUN_OFF32) {
        const int* so = (const int*)r.src;
        int* d = (int*)r.dst;
        for (long long k = c0 / 4 + threadIdx.x; k < c1 / 4; k += PUSH_THREADS) d[k] = (int)((long long)so[k] - r.a + r.b);
    } else {
        const long long* so = (const long long*)r.src;
        long long* d = (long long*)r.dst;
        for (long long k = c0 / 8 + threadIdx.x; k < c1 / 8; k += PUSH_THREADS) d[k] = so[k] - r.a + r.b;
    }
}

}  // namespace

struct dfd_exchange {
    dfd_ctx* ctx = nullptr;
    int rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    // scratch
    int64_t* d_counts = nullptr;      // [T][N] all-gathered destination counts
    int64_t* h_counts = nullptr;      // pinned mirror
    int64_t* d_dest_base = nullptr;   // [N]
    int64_t* d_my_starts = nullptr;   // [P+1]
    int64_t* h_my_starts = nullptr;   // pinned
    int32_t* d_abort = nullptr;
    int32_t* h_abort = nullptr;       // pinned
    int32_t* d_token = nullptr;       // barrier payload
    uint32_t cap_N = 0;
    // NCCL mode staging (locally partitioned columns)
    Scratch send;
    Scratch recv_tmp;  // receiver-side temporaries (u8 images of bitmaps, string lengths)
    Scratch bytes_all; // NCCL mode: all-gathered per-destination byte counts of the string columns (reused across shuffles)
    // fused mode: receive window + peers' mappings
    void* window = nullptr;
    size_t window_bytes = 0;
    void* peer_window[MAX_RANKS] = {};
    bool window_ready = false;
    // single-pass exchange: window header flags (no NCCL on the critical path)
    ExchangeHeader** d_peer_hdr = nullptr;  // device array [T]: every worker's window header
    unsigned long long epoch = 0;           // shuffle counter (flag value)
    int32_t* d_flags = nullptr;             // [0] my scatter overflowed a sub-window, [1] a peer never arrived
    int64_t* h_seg_counts = nullptr;        // pinned [T][P] rows producer r sent to my partition q
    int32_t* h_seg_flags = nullptr;         // pinned [T] overflow flags of the producers + [T] timed-out flag
    int64_t* d_meta = nullptr;              // device [XCHG_META_MAX] my metadata for the flag all-gather
    int64_t* h_meta = nullptr;              // pinned [MAX_RANKS][XCHG_META_MAX] gathered metadata
    void* d_runs = nullptr;                 // device PushRun array
    void* h_runs = nullptr;                 // pinned staging of the same
    size_t runs_cap = 0;
    uint64_t push_shuffles = 0;
    EventRing phases;  // profiling: the three stream phases of every single-pass shuffle (dfd_exchange_phase_ms)
    uint64_t onepass_fallbacks = 0;
    // What dfd_exchange_collect / _wait / _pending_segments report on: the last shuffle, if it left a result to pick up.
    // Every shuffle entry point resets it to NONE first and sets its own kind only on success.
    struct Pending {
        enum Kind {
            NONE,
            DENSE,     // two-pass fused shuffle enqueued, not yet waited for
            REGIONS,   // single-pass shuffle enqueued: (partition, producer) sub-windows
            SEGMENTS,  // push transport: already complete, collectable until the next shuffle starts
        } kind = NONE;
        uint32_t P = 0;
        size_t row_bytes = 0;
        int64_t sub_cap = 0;                  // REGIONS: rows per sub-window
        std::vector<dfd_column> in;           // REGIONS: the input, kept for the exact two-pass re-run after an overflow
        dfd_partitioner* part = nullptr;
        int64_t rows = 0;
        std::vector<int64_t> seg_starts, seg_counts;  // SEGMENTS
    } pending;
    // host pipeline (dfd_shuffle_host): H2D | shuffle | D2H of consecutive chunks overlap
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t e_h2d[2] = {}, e_k[2] = {}, e_d2h[2] = {};
    Scratch in_stage[2];
    uint64_t bytes_sent = 0, bytes_received = 0, shuffles = 0;
};

extern "C" {

/* Pure host logic (no GPU): from the T x N count matrix, where does everything go? */
int dfd_exchange_plan(int world, uint32_t partitions_per_task, int rank, const int64_t* counts, int64_t* send_start,
                      int64_t* recv_start, int64_t* part_starts, int64_t* dest_base, int64_t* recv_rows) {
    if (world < 1 || partitions_per_task < 1 || rank < 0 || rank >= world || !counts)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_exchange_plan: bad arguments");
    const uint32_t P = partitions_per_task;
    const int64_t N = (int64_t)P * world;
    for (int64_t i = 0; i < N * world; ++i)
        if (counts[i] < 0) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_exchange_plan: negative count");
    if (send_start) {  // my locally partitioned buffer: destinations back-to-back
        int64_t run = 0;
        for (int64_t g = 0; g < N; ++g) {
            send_start[g] = run;
            run += counts[(int64_t)rank * N + g];
        }
    }
    // my receive buffer: [local partition q][producer r]  (destination-major, producers in task order)
    int64_t run = 0;
    for (uint32_t q = 0; q < P; ++q) {
        const int64_t g = (int64_t)rank * P + q;
        if (part_starts) part_starts[q] = run;
        for (int r = 0; r < world; ++r) {
            if (recv_start) recv_start[(int64_t)q * world + r] = run;
            run += counts[(int64_t)r * N + g];
        }
    }
    if (part_starts) part_starts[P] = run;
    if (recv_rows) *recv_rows = run;
    if (dest_base) {  // where MY rows of destination g start inside the owner's receive buffer
        for (int o = 0; o < world; ++o) {
            int64_t orun = 0;
            for (uint32_t q = 0; q < P; ++q) {
                const int64_t g = (int64_t)o * P + q;
                int64_t before = 0, tot = 0;
                for (int r = 0; r < world; ++r) {
                    if (r < rank) before += counts[(int64_t)r * N + g];
                    tot += counts[(int64_t)r * N + g];
                }
                dest_base[g] = orun + before;
                orun += tot;
            }
        }
    }
    return DFD_OK;
}

int dfd_nccl_unique_id(void* out_128_bytes) {
    if (!out_128_bytes) return set_error(DFD_ERR_INVALID_ARGUMENT, "out is NULL");
    NcclApi* n = nccl_api();
    if (!n->handle || !n->error.empty()) return set_error(DFD_ERR_NCCL, "%s", n->error.c_str());
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    NCCL_TRY(n->GetUniqueId(&id), "ncclGetUniqueId");
    memcpy(out_128_bytes, &id, sizeof id);
    return DFD_OK;
}

int dfd_exchange_create(dfd_ctx* ctx, int rank, int world, const void* nccl_unique_id, dfd_exchange** out) {
    if (!ctx || !out) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_exchange_create: NULL argument");
    *out = nullptr;
    if (world < 1 || world > MAX_RANKS || rank < 0 || rank >= world)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "rank %d / world %d invalid (max %d workers)", rank, world, MAX_RANKS);
    dfd_exchange* x = new (std::nothrow) dfd_exchange();
    if (!x) return set_error(DFD_ERR_OOM, "out of host memory");
    x->ctx = ctx;
    x->rank = rank;
    x->world = world;
    std::lock_guard<std::mutex> lk(ctx->mu);
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) { delete x; return cuda_error(e, "cudaSetDevice"); }
    if (world > 1) {
        if (!nccl_unique_id) { delete x; return set_error(DFD_ERR_INVALID_ARGUMENT, "nccl_unique_id is NULL"); }
        NcclApi* n = nccl_api();
        if (!n->handle || !n->error.empty()) { delete x; return set_error(DFD_ERR_NCCL, "%s", n->error.c_str()); }
        ncclUniqueId id;
        memcpy(&id, nccl_unique_id, sizeof id);
        ncclResult_t r = n->CommInitRank(&x->comm, world, id, rank);
        if (r != ncclSuccess) { delete x; return nccl_error(r, "ncclCommInitRank"); }
    }
    e = cudaMalloc((void**)&x->d_abort, 256);
    if (e == cudaSuccess) e = cudaMemset(x->d_abort, 0, 256);
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&x->h_abort, 64, cudaHostAllocPortable);
    if (e != cudaSuccess) { delete x; return cuda_error(e, "dfd_exchange_create"); }
    x->d_token = x->d_abort + 16;
    *x->h_abort = 0;
    *out = x;
    return DFD_OK;
}

void dfd_exchange_destroy(dfd_exchange* x) {
    if (!x) return;
    {
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        cudaSetDevice(x->ctx->device);
        cudaStreamSynchronize(x->ctx->stream);
        for (int r = 0; r < x->world; ++r)
            if (x->peer_window[r] && r != x->rank) cudaIpcCloseMemHandle(x->peer_window[r]);
        if (x->comm) nccl_api()->CommDestroy(x->comm);
        cudaFree(x->window);
        cudaFree(x->d_peer_hdr);
        cudaFree(x->d_flags);
        cudaFree(x->d_meta);
        cudaFree(x->d_runs);
        cudaFreeHost(x->h_meta);
        cudaFreeHost(x->h_runs);
        cudaFreeHost(x->h_seg_counts);
        cudaFreeHost(x->h_seg_flags);
        cudaFree(x->d_counts);
        cudaFree(x->d_dest_base);
        cudaFree(x->d_my_starts);
        cudaFree(x->d_abort);
        cudaFree(x->send.ptr);
        cudaFree(x->recv_tmp.ptr);
        cudaFree(x->bytes_all.ptr);
        cudaFree(x->in_stage[0].ptr);
        cudaFree(x->in_stage[1].ptr);
        for (int i = 0; i < 2; ++i) {
            if (x->e_h2d[i]) cudaEventDestroy(x->e_h2d[i]);
            if (x->e_k[i]) cudaEventDestroy(x->e_k[i]);
            if (x->e_d2h[i]) cudaEventDestroy(x->e_d2h[i]);
        }
        if (x->s_h2d) cudaStreamDestroy(x->s_h2d);
        if (x->s_d2h) cudaStreamDestroy(x->s_d2h);
        cudaFreeHost(x->h_counts);
        cudaFreeHost(x->h_my_starts);
        cudaFreeHost(x->h_abort);
    }
    delete x;
}

int dfd_exchange_rank(const dfd_exchange* x) { return x ? x->rank : -1; }
int dfd_exchange_world(const dfd_exchange* x) { return x ? x->world : 0; }

static int ensure_count_buffers(dfd_exchange* x, uint32_t N) {
    if (N <= x->cap_N) return DFD_OK;
    cudaFree(x->d_counts); cudaFree(x->d_dest_base); cudaFree(x->d_my_starts);
    cudaFreeHost(x->h_counts); cudaFreeHost(x->h_my_starts);
    x->d_counts = nullptr; x->d_dest_base = nullptr; x->d_my_starts = nullptr; x->h_counts = nullptr; x->h_my_starts = nullptr;
    x->cap_N = 0;
    CUDA_TRY(cudaMalloc((void**)&x->d_counts, sizeof(int64_t) * (size_t)N * x->world), "cudaMalloc(counts)");
    CUDA_TRY(cudaMalloc((void**)&x->d_dest_base, sizeof(int64_t) * (size_t)N), "cudaMalloc(dest_base)");
    CUDA_TRY(cudaMalloc((void**)&x->d_my_starts, sizeof(int64_t) * (size_t)(N + 1)), "cudaMalloc(my_starts)");
    CUDA_TRY(cudaHostAlloc((void**)&x->h_counts, sizeof(int64_t) * (size_t)N * x->world, cudaHostAllocPortable), "cudaHostAlloc");
    CUDA_TRY(cudaHostAlloc((void**)&x->h_my_starts, sizeof(int64_t) * (size_t)(N + 1), cudaHostAllocPortable), "cudaHostAlloc");
    x->cap_N = N;
    return DFD_OK;
}

// Checks and set-up shared by the shuffle entry points.  On success `lk` holds the context's lock, the device is set, the
// count buffers fit, the shuffle is counted and nothing is pending any more.
static int begin_shuffle(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, const dfd_column* out_cols, uint32_t P,
                         const char* fn, std::unique_lock<std::mutex>& lk) {
    if (!x || !part || !in_cols || !out_cols) return set_error(DFD_ERR_INVALID_ARGUMENT, "%s: NULL argument", fn);
    dfd_ctx* c = x->ctx;
    if (part->ctx != c) return set_error(DFD_ERR_INVALID_ARGUMENT, "partitioner and exchange belong to different contexts");
    if (P < 1 || (uint64_t)P * x->world != part->N)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "num_partitions %u != partitions_per_task %u x %d workers", part->N, P, x->world);
    lk = std::unique_lock<std::mutex>(c->mu);
    x->pending.kind = dfd_exchange::Pending::NONE;
    CUDA_TRY(cudaSetDevice(c->device), "cudaSetDevice");
    int rc = ensure_count_buffers(x, part->N);
    if (rc) return rc;
    x->shuffles++;
    return DFD_OK;
}

/* Allocate this rank's receive window and map every peer's (collective call). */
int dfd_exchange_setup_window(dfd_exchange* x, size_t window_bytes) {
    if (!x) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL exchange");
    dfd_ctx* c = x->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CUDA_TRY(cudaSetDevice(c->device), "cudaSetDevice");
    if (x->window_ready) return set_error(DFD_ERR_INVALID_ARGUMENT, "receive window already set up");
    window_bytes = (window_bytes + 255) & ~(size_t)255;
    // [ExchangeHeader | XCHG_HEADER_BYTES][window_bytes of row data]
    CUDA_TRY(cudaMalloc(&x->window, window_bytes + XCHG_HEADER_BYTES), "cudaMalloc(receive window)");
    CUDA_TRY(cudaMemset(x->window, 0, XCHG_HEADER_BYTES), "cudaMemset(window header)");
    x->window_bytes = window_bytes;
    x->peer_window[x->rank] = x->window;
    if (x->world > 1) {
        NcclApi* n = nccl_api();
        // every worker derives slot sizes, column offsets and overflow checks from ITS window_bytes and applies
        // them to every peer's window: the sizes must agree, so they travel with the IPC handles
        struct Rec { cudaIpcMemHandle_t handle; unsigned long long bytes; } mine;
        memset(&mine, 0, sizeof mine);
        CUDA_TRY(cudaIpcGetMemHandle(&mine.handle, x->window), "cudaIpcGetMemHandle");
        mine.bytes = (unsigned long long)window_bytes;
        char* d_h = nullptr;
        const size_t hs = sizeof(Rec);
        CUDA_TRY(cudaMalloc((void**)&d_h, hs * (size_t)(x->world + 1)), "cudaMalloc(handles)");
        CUDA_TRY(cudaMemcpyAsync(d_h + hs * x->world, &mine, hs, cudaMemcpyHostToDevice, c->stream), "H2D handle");
        NCCL_TRY(n->AllGather(d_h + hs * x->world, d_h, hs, ncclInt8, x->comm, c->stream), "ncclAllGather(handles)");
        std::vector<Rec> all(x->world);
        CUDA_TRY(cudaMemcpyAsync(all.data(), d_h, hs * x->world, cudaMemcpyDeviceToHost, c->stream), "D2H handles");
        CUDA_TRY(cudaStreamSynchronize(c->stream), "sync");
        cudaFree(d_h);
        for (int r = 0; r < x->world; ++r)
            if (all[r].bytes != (unsigned long long)window_bytes) {
                cudaFree(x->window);
                x->window = nullptr;
                x->peer_window[x->rank] = nullptr;
                return set_error(DFD_ERR_INVALID_ARGUMENT, "receive windows must have the same size on every worker: rank %d has %llu B, rank %d has %zu B",
                                 r, all[r].bytes, x->rank, window_bytes);
            }
        for (int r = 0; r < x->world; ++r) {
            if (r == x->rank) continue;
            cudaError_t e = cudaIpcOpenMemHandle(&x->peer_window[r], all[r].handle, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) return cuda_error(e, "cudaIpcOpenMemHandle (peer receive window)");
        }
    }
    {
        std::vector<ExchangeHeader*> hdrs(x->world);
        for (int r = 0; r < x->world; ++r) hdrs[r] = (ExchangeHeader*)x->peer_window[r];
        CUDA_TRY(cudaMalloc((void**)&x->d_peer_hdr, sizeof(ExchangeHeader*) * (size_t)x->world), "cudaMalloc(peer headers)");
        CUDA_TRY(cudaMemcpy(x->d_peer_hdr, hdrs.data(), sizeof(ExchangeHeader*) * (size_t)x->world, cudaMemcpyHostToDevice), "H2D peer headers");
        CUDA_TRY(cudaMalloc((void**)&x->d_flags, 64), "cudaMalloc(flags)");
        CUDA_TRY(cudaMemset(x->d_flags, 0, 64), "cudaMemset(flags)");
        CUDA_TRY(cudaHostAlloc((void**)&x->h_seg_counts, sizeof(int64_t) * MAX_RANKS * XCHG_MAX_P, cudaHostAllocPortable), "cudaHostAlloc");
        CUDA_TRY(cudaHostAlloc((void**)&x->h_seg_flags, sizeof(int32_t) * (MAX_RANKS + 16), cudaHostAllocPortable), "cudaHostAlloc");
        CUDA_TRY(cudaMalloc((void**)&x->d_meta, sizeof(int64_t) * XCHG_META_MAX), "cudaMalloc(meta)");
        CUDA_TRY(cudaHostAlloc((void**)&x->h_meta, sizeof(int64_t) * MAX_RANKS * XCHG_META_MAX, cudaHostAllocPortable), "cudaHostAlloc");
    }
    if (x->world > 1) {
        // the header memset above must be complete on every worker before anyone's first flag store can arrive
        NcclApi* n = nccl_api();
        NCCL_TRY(n->AllReduce(x->d_token, x->d_token, 1, ncclInt32, ncclSum, x->comm, c->stream), "ncclAllReduce(window barrier)");
        CUDA_TRY(cudaStreamSynchronize(c->stream), "sync");
    }
    x->window_ready = true;
    return DFD_OK;
}

static size_t row_bytes_of(const dfd_column* cols, int n_cols) {
    size_t rb = 0;
    for (int i = 0; i < n_cols; ++i) rb += cols[i].kind == DFD_COL_FIXED ? (size_t)cols[i].width : 0;
    return rb;
}

// Window slot `slot` of `n_slots` of the fused transports (the window is split so that a chunked host pipeline can drain one
// slot while the next chunk lands in the other).  Identical on every rank: capacity rounded down to `row_align` rows, column
// i at byte offset capacity * sum(width[0..i)).  outs: the columns as the peer scatter sees them (values = byte offset into
// every rank's slot, peer_base[r]); out_cols: this rank's own slot.  Returns the capacity in rows.
static int64_t layout_window_slot(const dfd_exchange* x, const dfd_column* in_cols, int n_cols, size_t rb, int slot, int n_slots,
                                  int64_t row_align, void** peer_base, std::vector<dfd_column>& outs, dfd_column* out_cols) {
    const size_t slot_bytes = (x->window_bytes / (size_t)n_slots) & ~(size_t)255;
    const int64_t capacity_rows = (int64_t)(slot_bytes / rb) / row_align * row_align;
    for (int r = 0; r < x->world; ++r) peer_base[r] = (char*)x->peer_window[r] + XCHG_HEADER_BYTES + (size_t)slot * slot_bytes;
    outs.resize(n_cols);
    size_t off = 0;
    for (int i = 0; i < n_cols; ++i) {
        outs[i] = in_cols[i];
        outs[i].validity = nullptr;
        outs[i].offset = 0;
        out_cols[i] = outs[i];
        outs[i].values = (void*)off;
        out_cols[i].values = (char*)peer_base[x->rank] + off;
        off += (size_t)capacity_rows * (size_t)in_cols[i].width;
    }
    return capacity_rows;
}

// Completes a two-pass fused shuffle with a stream synchronize: x->h_my_starts then holds this worker's part_starts[P+1].
static int fused_shuffle_finish(dfd_exchange* x, uint32_t P, size_t rb) {
    CUDA_TRY(cudaStreamSynchronize(x->ctx->stream), "fused shuffle");
    if (*x->h_abort)
        return set_error(DFD_ERR_CAPACITY, "a receive window slot is too small for this shuffle (window %zu B)", x->window_bytes);
    x->bytes_received += (uint64_t)x->h_my_starts[P] * rb;
    return DFD_OK;
}

// Two-pass fused shuffle of device columns into window slot `slot` of `n_slots`.  With `sync` it completes inside the call;
// without, it stays pending (DENSE) for dfd_exchange_wait / _collect.  `e_k`, if given, is recorded right after the last
// kernel / barrier of this shuffle.
static int fused_shuffle_locked(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows,
                                uint32_t P, int slot, int n_slots, dfd_column* out_cols, cudaEvent_t e_k, bool sync = true) {
    dfd_ctx* c = x->ctx;
    const uint32_t N = part->N;
    const int T = x->world;
    NcclApi* n = T > 1 ? nccl_api() : nullptr;
    cudaStream_t s = c->stream;
    if (!x->window_ready) return set_error(DFD_ERR_INVALID_ARGUMENT, "fused exchange needs dfd_exchange_setup_window first");
    const size_t rb = row_bytes_of(in_cols, n_cols);
    if (rb == 0) return set_error(DFD_ERR_INVALID_ARGUMENT, "no fixed-width columns");
    void* peer_base[MAX_RANKS];
    std::vector<dfd_column> outs;
    const int64_t capacity_rows = layout_window_slot(x, in_cols, n_cols, rb, slot, n_slots, 16, peer_base, outs, out_cols);
    int rc;
    PartitionJob job;
    if ((rc = job.prepare(part, in_cols, n_cols, n_rows, outs.data(), true, s))) return rc;
    if ((rc = job.run_hist_scan())) return rc;
    if (T > 1) {
        NCCL_TRY(n->AllGather(job.d_totals, x->d_counts, N, ncclInt64, x->comm, s), "ncclAllGather(counts)");
    } else {
        CUDA_TRY(cudaMemcpyAsync(x->d_counts, job.d_totals, sizeof(int64_t) * N, cudaMemcpyDeviceToDevice, s), "copy counts");
    }
    k_exchange_plan<<<1, 32, 0, s>>>(x->d_counts, T, P, x->rank, capacity_rows, x->d_dest_base, x->d_my_starts, x->d_abort);
    CUDA_TRY(cudaGetLastError(), "k_exchange_plan");
    c->metrics.kernel_launches++;
    if ((rc = job.run_scatter(x->d_dest_base, peer_base, T, P, x->d_abort))) return rc;
    // every producer's stores must have landed before any consumer reads its window
    if (T > 1) NCCL_TRY(n->AllReduce(x->d_token, x->d_token, 1, ncclInt32, ncclSum, x->comm, s), "ncclAllReduce(barrier)");
    if (e_k) CUDA_TRY(cudaEventRecord(e_k, s), "record");
    CUDA_TRY(cudaMemcpyAsync(x->h_my_starts, x->d_my_starts, sizeof(int64_t) * (P + 1), cudaMemcpyDeviceToHost, s), "D2H starts");
    CUDA_TRY(cudaMemcpyAsync(x->h_abort, x->d_abort, sizeof(int32_t), cudaMemcpyDeviceToHost, s), "D2H flag");
    x->bytes_sent += (uint64_t)n_rows * rb;
    if (sync) return fused_shuffle_finish(x, P, rb);
    x->pending.kind = dfd_exchange::Pending::DENSE;
    x->pending.P = P;
    x->pending.row_bytes = rb;
    return DFD_OK;
}

// ---- single-pass fused shuffle ------------------------------------------------------------------
// Every (consumer partition q, producer r) pair owns a fixed sub-window of the consumer's receive window, so a producer
// needs no global counts before its first store: ONE k_scatter_onepass<PEER> launch hashes, ranks, resolves its tile
// cursors by look-back and stores straight into the owners' windows over NVLink.  Counts, overflow and completion
// travel as peer-memory flags (window headers) written by two tiny kernels — no NCCL call on the critical path.
// The reference makes the same promise: a consumer partition is the MERGE of one stream per producer, in no
// particular inter-producer order (src/execution_plans/network_shuffle.rs:230-237 `select_all`).
// (decided from the SCHEMA — column kinds and the nullable flags the caller passes in out_cols[].validity — so that every
//  worker takes the same transport whether or not its own rows contain nulls)
static bool onepass_supported(const dfd_partitioner* part, const dfd_column* cols, const dfd_column* out_cols, int n_cols, uint32_t P) {
    if (part->N > ONEPASS_MAX_N || P > XCHG_MAX_P || n_cols < 1) return false;
    for (int i = 0; i < n_cols; ++i)
        if (cols[i].kind != DFD_COL_FIXED || cols[i].validity || out_cols[i].validity) return false;
    return true;
}

static int onepass_shuffle_locked(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows, uint32_t P,
                                  int slot, int n_slots, dfd_column* out_cols) {
    dfd_ctx* c = x->ctx;
    const int T = x->world;
    cudaStream_t s = c->stream;
    if (!x->window_ready) return set_error(DFD_ERR_INVALID_ARGUMENT, "fused exchange needs dfd_exchange_setup_window first");
    const size_t rb = row_bytes_of(in_cols, n_cols);
    void* peer_base[MAX_RANKS];
    std::vector<dfd_column> outs;
    const int64_t capacity_rows = layout_window_slot(x, in_cols, n_cols, rb, slot, n_slots, 32, peer_base, outs, out_cols);
    const int64_t sub_cap = capacity_rows / ((int64_t)P * T) / 32 * 32;  // rows per (partition, producer) sub-window
    if (sub_cap < 32) return set_error(DFD_ERR_CAPACITY, "receive window (%zu B) too small for %u x %d sub-windows", x->window_bytes, P, T);
    const unsigned long long epoch = ++x->epoch;
    ExchangeHeader* hdr = (ExchangeHeader*)x->window;
    int rc;
    cudaEvent_t* pe = nullptr;
    if (c->profiling) {
        if ((rc = x->phases.next(&pe))) return rc;
        x->phases.commit();
        cudaEventRecord(pe[0], s);
    }
    // consumer half: my window is free (everything enqueued on my stream so far — i.e. my reads of the previous shuffle — is ordered before)
    k_xchg_signal_ready<<<1, 32, 0, s>>>(x->d_peer_hdr, x->rank, T, epoch);
    if (pe) cudaEventRecord(pe[1], s);
    CUDA_TRY(cudaGetLastError(), "k_xchg_signal_ready");
    CUDA_TRY(cudaMemsetAsync(x->d_flags, 0, 8, s), "memset flags");
    PartitionJob job;
    job.onepass_tiling = true;
    if ((rc = job.prepare(part, in_cols, n_cols, n_rows, outs.data(), true, s))) return rc;
    PartitionJob::OnePassLayout L;
    L.region_stride = sub_cap;
    L.peer_base = peer_base;
    L.world = T;
    L.rank = x->rank;
    L.parts_per_rank = P;
    L.d_totals = x->d_counts;
    L.d_overflow = x->d_flags;
    L.ready_flags = hdr->ready;
    L.ready_epoch = epoch;
    if ((rc = job.run_onepass(L))) return rc;
    if (pe) cudaEventRecord(pe[2], s);
    // producer half: counts + overflow + "landed" flag into every consumer's header; consumer half: wait for all producers
    k_xchg_publish_wait<<<1, 256, 0, s>>>(hdr, x->d_peer_hdr, x->rank, T, P, epoch, x->d_counts, x->d_flags, x->d_flags + 1);
    CUDA_TRY(cudaGetLastError(), "k_xchg_publish_wait");
    if (pe) cudaEventRecord(pe[3], s);
    c->metrics.kernel_launches += 2;
    CUDA_TRY(cudaMemcpy2DAsync(x->h_seg_counts, sizeof(int64_t) * P, hdr->counts, sizeof(long long) * XCHG_MAX_P, sizeof(int64_t) * P, (size_t)T,
                               cudaMemcpyDeviceToHost, s), "D2H counts");
    CUDA_TRY(cudaMemcpyAsync(x->h_seg_flags, hdr->overflow, sizeof(int32_t) * (size_t)T, cudaMemcpyDeviceToHost, s), "D2H overflow flags");
    CUDA_TRY(cudaMemcpyAsync(x->h_seg_flags + MAX_RANKS, x->d_flags + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s), "D2H timeout flag");
    x->bytes_sent += (uint64_t)n_rows * rb;
    dfd_exchange::Pending& pd = x->pending;
    pd.kind = dfd_exchange::Pending::REGIONS;
    pd.P = P;
    pd.row_bytes = rb;
    pd.sub_cap = sub_cap;
    pd.in.assign(in_cols, in_cols + n_cols);
    pd.part = part;
    pd.rows = n_rows;
    return DFD_OK;
}

// ---- push transport: every column kind over NVLink, no NCCL --------------------------------------
// 1. (shuffle only) partition locally (K1/K1b/K2 + K4) into a destination-sorted staging buffer — any column kind;
// 2. all-gather the per-slice row / byte counts through the window headers (k_xchg_allgather_meta); its flag
//    also tells the producers that this worker's window is free again;
// 3. every worker derives EVERY consumer's window layout from the same count matrices: a consumer's window is a list
//    of segments (which (producer, slice) lands where is the ROUTE: shuffle / coalesce / broadcast), each starting on a
//    32-row boundary (bitmaps are pushed word-aligned, no atomics) with >= 1 spare row (a segment's n+1 string
//    offsets never touch its neighbour);
// 4. k_push_runs stores each slice's contiguous runs — values, shifted bitmaps, re-based string offsets, string
//    bytes — straight into the owners' segments (16-byte vectors when co-aligned), then k_xchg_done_barrier.
// The consumer reads Arrow-shaped buffers in place: one values / offsets / bitmap buffer per column, segment s
// = rows [seg_start[s], +seg_count[s]).
namespace {

// Which (producer task, local slice) feeds which consumer segment.
//   SHUFFLE   (NetworkShuffleExec, src/execution_plans/network_shuffle.rs:213-238): producer r holds N = P*T slices
//             (global partitions); slice g goes to consumer g / P as segment (g % P) * T + r.
//   COALESCE  (NetworkCoalesceExec, src/execution_plans/network_coalesce.rs:170-240): producer r holds P slices (its own
//             partitions, no repartition); consumer c reads the contiguous group of producers task_group(T, c, C):
//             segment (r - group.start) * P + g; groups shorter than the longest are padded with empty segments.
//   BROADCAST (NetworkBroadcastExec, src/execution_plans/network_broadcast.rs:224-249): every consumer receives every
//             producer's P slices: segment g * T + r on each of the C consumers.
struct Route {
    int kind;
    uint32_t P;
    int T;  // producer tasks == workers
    int C;  // consumer tasks (<= workers)
    uint32_t n_slices() const { return kind == DFD_ROUTE_SHUFFLE ? P * (uint32_t)T : P; }
    void group(int c, int* start, int* len, int* max_len) const {  // task_group(input_task_count = T, task_index = c, task_count = C)
        const int base = T / C, extra = T % C;
        *len = base + (c < extra ? 1 : 0);
        *start = c * base + (c < extra ? c : extra);
        *max_len = base + (extra > 0 ? 1 : 0);
    }
    uint32_t n_segments(int o) const {
        if (o >= C) return 0;
        if (kind == DFD_ROUTE_COALESCE) { int s, l, m; group(o, &s, &l, &m); return (uint32_t)m * P; }
        return P * (uint32_t)T;
    }
    // source of consumer o's segment s: producer r and its slice g (r = -1: padding segment)
    void source(int o, uint32_t s, int* r, uint32_t* g) const {
        if (kind == DFD_ROUTE_SHUFFLE) { *r = (int)(s % (uint32_t)T); *g = (uint32_t)o * P + s / (uint32_t)T; }
        else if (kind == DFD_ROUTE_BROADCAST) { *r = (int)(s % (uint32_t)T); *g = s / (uint32_t)T; }
        else {
            int st, l, m;
            group(o, &st, &l, &m);
            const int off = (int)(s / P);
            *r = off < l ? st + off : -1;
            *g = s % P;
        }
    }
};

struct PushCol {
    int kind, width, ow, var_index;
    bool nullable, in_valid;
    const char* values;
    const char* offsets;
    const char* validity;
    int64_t offset;  // Arrow logical offset of the source column
};

size_t al(size_t v) { return (v + 255) & ~(size_t)255; }

// How the push transport and NCCL mode move column i: kind, offset width, index among the string columns, and whether a
// validity lane travels — the SCHEMA's flag (out_cols[i].validity != NULL on entry, the same on every worker) or a bitmap
// in this worker's input.  values / offsets / validity / offset describe in_cols[i].
int describe_columns(const dfd_column* in_cols, const dfd_column* out_cols, int n_cols, std::vector<PushCol>& pc) {
    pc.assign(n_cols, PushCol{});
    int V = 0;
    for (int i = 0; i < n_cols; ++i) {
        const dfd_column& ic = in_cols[i];
        PushCol& q = pc[i];
        q.kind = ic.kind; q.width = ic.width; q.ow = ic.kind == DFD_COL_LARGE_UTF8 ? 8 : 4; q.var_index = -1;
        if (ic.kind == DFD_COL_UTF8 || ic.kind == DFD_COL_LARGE_UTF8 || ic.kind == DFD_COL_BINARY) q.var_index = V++;
        else if (ic.kind != DFD_COL_FIXED && ic.kind != DFD_COL_BOOL) return set_error(DFD_ERR_UNSUPPORTED, "column %d: unknown column kind %d", i, ic.kind);
        q.in_valid = ic.validity != nullptr;
        q.nullable = out_cols[i].validity != nullptr || q.in_valid;
        q.values = (const char*)ic.values; q.offsets = (const char*)ic.offsets; q.validity = (const char*)ic.validity; q.offset = ic.offset;
    }
    return DFD_OK;
}

int n_var_cols(const std::vector<PushCol>& pc) {
    int V = 0;
    for (const PushCol& q : pc) V += q.var_index >= 0;
    return V;
}

__global__ void k_slice_rows(const int64_t* __restrict__ starts, uint32_t n, int64_t* __restrict__ rows) {
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n; g += gridDim.x * blockDim.x) rows[g] = starts[g + 1] - starts[g];
}

}  // namespace

// Steps 2-4 for `n_slices` consecutive row ranges [starts[g], starts[g+1]) of device columns `pc` (d_starts: device copy).
static int push_slices_locked(dfd_exchange* x, const std::vector<PushCol>& pc, const dfd_column* proto_cols, const Route& R,
                              const int64_t* d_starts, char* scratch /* >= (V+1) * n_slices * 8 B, device */, dfd_column* out_cols) {
    dfd_ctx* c = x->ctx;
    const int T = x->world;
    const int n_cols = (int)pc.size();
    cudaStream_t s = c->stream;
    const int V = n_var_cols(pc);
    const uint32_t NS = R.n_slices();
    const uint32_t n_meta = (uint32_t)(1 + V) * NS;
    if (n_meta > XCHG_META_MAX)
        return set_error(DFD_ERR_UNSUPPORTED, "push transport: (1 + %d string columns) x %u slices exceeds %u metadata entries", V, NS, XCHG_META_MAX);
    int rc;
    // my metadata: rows per slice, then bytes per slice of every string column (+ local: first byte of every slice)
    k_slice_rows<<<(NS + 255) / 256, 256, 0, s>>>(d_starts, NS, x->d_meta);
    CUDA_TRY(cudaGetLastError(), "k_slice_rows");
    int64_t* d_first = (int64_t*)scratch;
    for (const PushCol& q : pc)
        if (q.var_index >= 0 &&
            (rc = launch_var_dest_bytes(q.offsets + (size_t)q.offset * q.ow, q.ow, d_starts, NS, x->d_meta + (size_t)NS * (1 + q.var_index),
                                        d_first + (size_t)NS * q.var_index, s)))
            return rc;
    const unsigned long long epoch = ++x->epoch;
    ExchangeHeader* hdr = (ExchangeHeader*)x->window;
    CUDA_TRY(cudaMemsetAsync(x->d_flags, 0, 8, s), "memset flags");
    k_xchg_allgather_meta<<<1, 256, 0, s>>>(hdr, x->d_peer_hdr, x->rank, T, epoch, x->d_meta, n_meta, x->d_flags + 1);
    CUDA_TRY(cudaGetLastError(), "k_xchg_allgather_meta");
    CUDA_TRY(cudaMemcpy2DAsync(x->h_meta, sizeof(int64_t) * XCHG_META_MAX, hdr->meta, sizeof(long long) * XCHG_META_MAX, sizeof(int64_t) * n_meta,
                               (size_t)T, cudaMemcpyDeviceToHost, s), "D2H meta");
    std::vector<int64_t> h_first((size_t)(V ? V : 1) * NS), h_starts(NS + 1);
    if (V) CUDA_TRY(cudaMemcpyAsync(h_first.data(), d_first, sizeof(int64_t) * (size_t)V * NS, cudaMemcpyDeviceToHost, s), "D2H first");
    CUDA_TRY(cudaMemcpyAsync(h_starts.data(), d_starts, sizeof(int64_t) * (NS + 1), cudaMemcpyDeviceToHost, s), "D2H starts");
    CUDA_TRY(cudaMemcpyAsync(x->h_seg_flags + MAX_RANKS, x->d_flags + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s), "D2H timeout flag");
    CUDA_TRY(cudaStreamSynchronize(s), "push: metadata exchange");
    if (x->h_seg_flags[MAX_RANKS]) return set_error(DFD_ERR_INTERNAL, "a peer worker never published its metadata (did it fail?)");
    auto rows_of = [&](int r, uint32_t g) { return x->h_meta[(size_t)r * XCHG_META_MAX + g]; };
    auto bytes_of = [&](int r, int v, uint32_t g) { return x->h_meta[(size_t)r * XCHG_META_MAX + (size_t)NS * (1 + v) + g]; };
    // ---- every consumer's layout, from the same matrices on every worker
    struct Layout {
        std::vector<int64_t> seg_start;               // [n_segments] rows
        std::vector<std::vector<int64_t>> bseg_start; // [V][n_segments] bytes
        std::vector<size_t> reg_values, reg_off, reg_valid;  // byte offsets of the column regions in the window
    };
    std::vector<Layout> lay(T);
    for (int o = 0; o < T; ++o) {
        Layout& Lo = lay[o];
        const uint32_t nseg = R.n_segments(o);
        Lo.seg_start.assign(nseg, 0);
        Lo.bseg_start.assign(V, std::vector<int64_t>(nseg, 0));
        int64_t run = 0;
        std::vector<int64_t> brun(V, 0), bmax(V, 0);  // bmax: the largest string offset any segment of the column holds
        for (uint32_t sg = 0; sg < nseg; ++sg) {
            int r;
            uint32_t g;
            R.source(o, sg, &r, &g);
            Lo.seg_start[sg] = run;
            const int64_t rows = r >= 0 ? rows_of(r, g) : 0;
            run = (run + rows + 1 + 31) / 32 * 32;  // 32-row aligned, >= 1 spare row
            for (int v = 0; v < V; ++v) {
                const int64_t nb = r >= 0 ? bytes_of(r, v, g) : 0;
                Lo.bseg_start[v][sg] = brun[v];
                if (rows > 0) bmax[v] = brun[v] + nb;
                brun[v] = (brun[v] + nb + 15) / 16 * 16;
            }
        }
        // A Utf8 / Binary segment's int32 offsets index the column's one byte region, 16-byte padding included: a
        // consumer whose offsets would pass INT32_MAX cannot take this round, exactly like one whose window is too small.
        int narrow = -1;
        for (int i = 0; i < n_cols && narrow < 0; ++i)
            if (pc[i].var_index >= 0 && pc[i].ow == 4 && bmax[pc[i].var_index] > INT32_MAX) narrow = i;
        Lo.reg_values.assign(n_cols, 0); Lo.reg_off.assign(n_cols, 0); Lo.reg_valid.assign(n_cols, 0);
        size_t off = 0;
        for (int i = 0; i < n_cols; ++i) {
            const PushCol& q = pc[i];
            if (q.kind == DFD_COL_FIXED) { Lo.reg_values[i] = off; off += al((size_t)run * q.width + 16); }
            else if (q.kind == DFD_COL_BOOL) { Lo.reg_values[i] = off; off += al((size_t)run / 8 + 16); }
            else {
                Lo.reg_off[i] = off; off += al((size_t)(run + 1) * q.ow + 16);
                Lo.reg_values[i] = off; off += al((size_t)brun[q.var_index] + 16);
            }
            if (q.nullable) { Lo.reg_valid[i] = off; off += al((size_t)run / 8 + 16); }
        }
        if (off > x->window_bytes || narrow >= 0) {
            // Every worker takes this branch (same matrices).  Nobody may start the next exchange — and overwrite its metadata
            // slots in the peers' headers — before every worker has read THIS epoch's metadata: close the epoch with the
            // done barrier, exactly as a successful exchange does (the back-pressured stream retries at once with a finer
            // round, dfd_shuffle_stream_next).
            k_xchg_done_barrier<<<1, 32, 0, s>>>(hdr, x->d_peer_hdr, x->rank, T, epoch, x->d_flags + 1);
            CUDA_TRY(cudaGetLastError(), "k_xchg_done_barrier");
            c->metrics.kernel_launches += 2;
            CUDA_TRY(cudaMemcpyAsync(x->h_seg_flags + MAX_RANKS, x->d_flags + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s), "D2H timeout flag");
            CUDA_TRY(cudaStreamSynchronize(s), "push exchange (capacity)");
            if (x->h_seg_flags[MAX_RANKS]) return set_error(DFD_ERR_INTERNAL, "a peer worker never acknowledged the over-full round (did it fail?)");
            if (narrow >= 0)
                return set_error(DFD_ERR_CAPACITY, "column %d: consumer %d would hold string offsets up to %lld, past the int32 offsets of "
                                                   "Utf8 / Binary", narrow, o, (long long)bmax[pc[narrow].var_index]);
            return set_error(DFD_ERR_CAPACITY, "consumer %d needs %zu B of receive window for this exchange, windows hold %zu B", o, off, x->window_bytes);
        }
    }
    // ---- my runs as producer: walk every consumer's segments and emit the ones I feed
    std::vector<PushRun> runs;
    for (int o = 0; o < T; ++o) {
        const Layout& Lo = lay[o];
        char* dst_base = (char*)x->peer_window[o] + XCHG_HEADER_BYTES;
        for (uint32_t sg = 0; sg < R.n_segments(o); ++sg) {
            int r;
            uint32_t g;
            R.source(o, sg, &r, &g);
            if (r != x->rank) continue;
            const int64_t cnt = rows_of(r, g), seg = Lo.seg_start[sg], first_row = h_starts[g];
            if (cnt <= 0) continue;
            for (int i = 0; i < n_cols; ++i) {
                const PushCol& qc = pc[i];
                PushRun pr{};
                if (qc.kind == DFD_COL_FIXED) {
                    pr.kind = RUN_BYTES; pr.src = qc.values + (size_t)(qc.offset + first_row) * qc.width;
                    pr.dst = dst_base + Lo.reg_values[i] + (size_t)seg * qc.width; pr.n = cnt * qc.width;
                    runs.push_back(pr);
                    if (o != x->rank) x->bytes_sent += (uint64_t)pr.n;
                } else if (qc.kind == DFD_COL_BOOL) {
                    pr.kind = RUN_BITS; pr.src = qc.values; pr.a = qc.offset + first_row; pr.dst = dst_base + Lo.reg_values[i] + (size_t)seg / 8; pr.n = cnt;
                    runs.push_back(pr);
                } else {
                    const int v = qc.var_index;
                    const int64_t first = h_first[(size_t)v * NS + g], nb = bytes_of(r, v, g), bseg = Lo.bseg_start[v][sg];
                    pr.kind = qc.ow == 8 ? RUN_OFF64 : RUN_OFF32; pr.src = qc.offsets + (size_t)(qc.offset + first_row) * qc.ow; pr.a = first; pr.b = bseg;
                    pr.dst = dst_base + Lo.reg_off[i] + (size_t)seg * qc.ow; pr.n = cnt + 1;
                    runs.push_back(pr);
                    if (nb > 0) {
                        PushRun b{};
                        b.kind = RUN_BYTES; b.src = qc.values + first; b.dst = dst_base + Lo.reg_values[i] + bseg; b.n = nb;
                        runs.push_back(b);
                        if (o != x->rank) x->bytes_sent += (uint64_t)nb;
                    }
                }
                if (qc.nullable) {
                    PushRun vr{};
                    vr.kind = qc.in_valid ? RUN_BITS : RUN_ONES; vr.src = qc.in_valid ? qc.validity : nullptr; vr.a = qc.offset + first_row;
                    vr.dst = dst_base + Lo.reg_valid[i] + (size_t)seg / 8; vr.n = cnt;
                    runs.push_back(vr);
                }
            }
        }
    }
    int blocks = 0;
    for (PushRun& r : runs) {
        r.first_block = blocks;
        blocks += (int)((push_run_out_bytes(r) + PUSH_CHUNK - 1) / PUSH_CHUNK);
    }
    if (!runs.empty()) {
        const size_t need = runs.size() * sizeof(PushRun);
        if (need > x->runs_cap) {
            cudaFree(x->d_runs); cudaFreeHost(x->h_runs);
            x->d_runs = nullptr; x->h_runs = nullptr; x->runs_cap = 0;
            CUDA_TRY(cudaMalloc(&x->d_runs, need * 2), "cudaMalloc(push runs)");
            CUDA_TRY(cudaHostAlloc(&x->h_runs, need * 2, cudaHostAllocPortable), "cudaHostAlloc(push runs)");
            x->runs_cap = need * 2;
        }
        memcpy(x->h_runs, runs.data(), need);
        CUDA_TRY(cudaMemcpyAsync(x->d_runs, x->h_runs, need, cudaMemcpyHostToDevice, s), "H2D push runs");
        k_push_runs<<<(unsigned)blocks, PUSH_THREADS, 0, s>>>((const PushRun*)x->d_runs, (int)runs.size());
        CUDA_TRY(cudaGetLastError(), "k_push_runs");
        c->metrics.kernel_launches++;
    }
    k_xchg_done_barrier<<<1, 32, 0, s>>>(hdr, x->d_peer_hdr, x->rank, T, epoch, x->d_flags + 1);
    CUDA_TRY(cudaGetLastError(), "k_xchg_done_barrier");
    c->metrics.kernel_launches += 3;
    CUDA_TRY(cudaMemcpyAsync(x->h_seg_flags + MAX_RANKS, x->d_flags + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s), "D2H timeout flag");
    CUDA_TRY(cudaStreamSynchronize(s), "push exchange");
    if (x->h_seg_flags[MAX_RANKS]) return set_error(DFD_ERR_INTERNAL, "a peer worker never finished its pushes (did it fail?)");
    // ---- my view as consumer
    const Layout& Me = lay[x->rank];
    char* my_base = (char*)x->window + XCHG_HEADER_BYTES;
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        out_cols[i] = proto_cols[i];
        out_cols[i].offset = 0;
        out_cols[i].values = my_base + Me.reg_values[i];
        out_cols[i].offsets = q.var_index >= 0 ? (void*)(my_base + Me.reg_off[i]) : nullptr;
        out_cols[i].validity = q.nullable ? (uint8_t*)(my_base + Me.reg_valid[i]) : nullptr;
        out_cols[i].values_bytes = 0;
    }
    const uint32_t nseg = R.n_segments(x->rank);
    dfd_exchange::Pending& pd = x->pending;
    pd.seg_starts.assign(Me.seg_start.begin(), Me.seg_start.end());
    pd.seg_counts.assign(nseg, 0);
    uint64_t rows = 0;
    for (uint32_t sg = 0; sg < nseg; ++sg) {
        int r;
        uint32_t g;
        R.source(x->rank, sg, &r, &g);
        pd.seg_counts[sg] = r >= 0 ? rows_of(r, g) : 0;
        rows += (uint64_t)pd.seg_counts[sg];
    }
    for (int i = 0; i < n_cols; ++i)
        if (pc[i].kind == DFD_COL_FIXED) x->bytes_received += rows * (uint64_t)pc[i].width;
    x->push_shuffles++;
    pd.kind = dfd_exchange::Pending::SEGMENTS;
    return DFD_OK;
}

// Local partition (K1/K1b/K2 + K4) of in_cols into a destination-sorted copy in x->send, for the push transport and NCCL
// mode: destination g is rows [part->d_part_starts[g], part->d_part_starts[g + 1]) of every staged column, and pc (from
// describe_columns) is pointed at the copies.  The `extra_bytes` behind them are the caller's (*extra).  *d_totals: rows per
// destination.
static int stage_locally(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows, std::vector<PushCol>& pc,
                         size_t extra_bytes, char** extra, const int64_t** d_totals) {
    dfd_ctx* c = x->ctx;
    std::vector<size_t> st_values(n_cols), st_off(n_cols), st_valid(n_cols);
    std::vector<int64_t> cap_bytes(n_cols, 0);
    size_t stage_bytes = 0;
    const size_t bm = al((size_t)((n_rows + 63) / 64 * 8 + 16));
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        if (q.kind == DFD_COL_FIXED) {
            st_values[i] = stage_bytes; stage_bytes += al((size_t)n_rows * q.width + 16);
        } else if (q.kind == DFD_COL_BOOL) {
            st_values[i] = stage_bytes; stage_bytes += bm;
        } else {
            cap_bytes[i] = in_cols[i].values_bytes > 0 ? in_cols[i].values_bytes : 16;
            st_off[i] = stage_bytes; stage_bytes += al((size_t)(n_rows + 1) * q.ow + 16);
            st_values[i] = stage_bytes; stage_bytes += al((size_t)cap_bytes[i] + 16);
        }
        if (q.in_valid) { st_valid[i] = stage_bytes; stage_bytes += bm; }
    }
    int rc;
    if ((rc = x->send.ensure(stage_bytes + extra_bytes + 256, c->device))) return rc;
    char* sb = (char*)x->send.ptr;
    std::vector<dfd_column> staged(n_cols);
    for (int i = 0; i < n_cols; ++i) {
        PushCol& q = pc[i];
        staged[i] = in_cols[i];
        staged[i].values = sb + st_values[i];
        staged[i].offsets = q.var_index >= 0 ? (void*)(sb + st_off[i]) : nullptr;
        staged[i].validity = q.in_valid ? (uint8_t*)(sb + st_valid[i]) : nullptr;
        staged[i].offset = 0;
        staged[i].values_bytes = cap_bytes[i];
        q.values = (const char*)staged[i].values;
        q.offsets = (const char*)staged[i].offsets;
        q.validity = (const char*)staged[i].validity;
        q.offset = 0;
    }
    PartitionJob job;
    if ((rc = job.prepare(part, in_cols, n_cols, n_rows, staged.data(), false, c->stream))) return rc;
    if ((rc = job.run_hist_scan())) return rc;
    if ((rc = job.run_scatter(part->d_part_starts, nullptr, 1, 1, nullptr))) return rc;
    *extra = sb + stage_bytes;
    *d_totals = job.d_totals;
    return DFD_OK;
}

static int push_shuffle_locked(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows, uint32_t P,
                               dfd_column* out_cols) {
    if (!x->window_ready) return set_error(DFD_ERR_INVALID_ARGUMENT, "fused exchange needs dfd_exchange_setup_window first");
    std::vector<PushCol> pc;
    char* scratch;
    const int64_t* d_totals;
    int rc = describe_columns(in_cols, out_cols, n_cols, pc);
    if (rc == DFD_OK) rc = stage_locally(x, part, in_cols, n_cols, n_rows, pc, al((size_t)(n_var_cols(pc) + 1) * part->N * 8 + 64), &scratch, &d_totals);
    if (rc) return rc;
    return push_slices_locked(x, pc, in_cols, Route{DFD_ROUTE_SHUFFLE, P, x->world, x->world}, part->d_part_starts, scratch, out_cols);
}

/* The shuffle: producer task `rank` holds n_rows local rows; afterwards this
 * worker, as consumer task `rank`, holds its P = partitions_per_task
 * destinations (global partitions rank*P .. rank*P+P-1), each contiguous, rows
 * from the producers in task order. */
int dfd_shuffle_device(dfd_exchange* x, dfd_partitioner* part, int mode, const dfd_column* in_cols, int n_cols,
                       int64_t n_rows, uint32_t partitions_per_task, dfd_column* out_cols, int64_t out_capacity_rows,
                       int64_t* part_starts_host) {
    if (!part_starts_host) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_shuffle_device: NULL argument");
    const uint32_t P = partitions_per_task;
    std::unique_lock<std::mutex> lk;
    int rc = begin_shuffle(x, part, in_cols, out_cols, P, "dfd_shuffle_device", lk);
    if (rc) return rc;
    dfd_ctx* c = x->ctx;
    const uint32_t N = part->N;
    const int T = x->world;
    NcclApi* n = T > 1 ? nccl_api() : nullptr;
    cudaStream_t s = c->stream;

    if (mode == DFD_EXCHANGE_FUSED) {
        rc = fused_shuffle_locked(x, part, in_cols, n_cols, n_rows, P, 0, 1, out_cols, nullptr);
        if (rc) return rc;
        memcpy(part_starts_host, x->h_my_starts, sizeof(int64_t) * (P + 1));
        return DFD_OK;
    }
    if (mode != DFD_EXCHANGE_NCCL) return set_error(DFD_ERR_INVALID_ARGUMENT, "unknown exchange mode %d", mode);

    // ---- NCCL mode: partition locally into a staging buffer, then grouped send/recv ----
    // Every column kind the local partitioner supports travels: fixed-width values as they are,
    // bitmaps (validity, booleans) as one byte per row, strings as (lengths, bytes); the receiver
    // rebuilds bitmaps and offsets (k_bytes_to_bits, lengths -> offsets scan).
    std::vector<PushCol> pc;
    if ((rc = describe_columns(in_cols, out_cols, n_cols, pc))) return rc;
    for (int i = 0; i < n_cols; ++i) {
        const dfd_column& oc = out_cols[i];
        if (oc.kind != in_cols[i].kind || oc.width != in_cols[i].width || !oc.values)
            return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: out layout mismatch", i);
        if (pc[i].in_valid && !oc.validity)
            return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: input has nulls but out validity is NULL (nullable columns need a validity "
                                                       "buffer on EVERY worker)", i);
        if (pc[i].var_index >= 0 && !oc.offsets) return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: out offsets is NULL", i);
    }
    // After these checks pc[i].nullable == (out_cols[i].validity != NULL), the schema's flag: every worker sends the same lanes.
    // Conversion buffers, u8 per row: the "values lane" (a boolean column's values, a string column's lengths) and the
    // validity lane, on the sender behind the staged columns and on the receiver in x->recv_tmp.
    struct Conv { size_t send_values, send_valid, recv_values, recv_valid; };
    std::vector<Conv> cv(n_cols);
    auto lane_width = [](const PushCol& q) { return q.kind == DFD_COL_BOOL ? (size_t)1 : (size_t)q.ow; };
    const size_t V = (size_t)n_var_cols(pc);
    size_t conv_bytes = 0;
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        if (q.kind != DFD_COL_FIXED) { cv[i].send_values = conv_bytes; conv_bytes += al((size_t)(n_rows + 1) * lane_width(q) + 16); }
        if (q.nullable) { cv[i].send_valid = conv_bytes; conv_bytes += al((size_t)n_rows + 16); }
    }
    const size_t meta_off = conv_bytes;  // per string column: bytes[N] | first[N] (device)
    conv_bytes += al(V * 2 * N * 8 + 64);
    char* cb;
    const int64_t* d_totals;
    if ((rc = stage_locally(x, part, in_cols, n_cols, n_rows, pc, conv_bytes, &cb, &d_totals))) return rc;
    if (T > 1) {
        NCCL_TRY(n->AllGather(d_totals, x->d_counts, N, ncclInt64, x->comm, s), "ncclAllGather(counts)");
    } else {
        CUDA_TRY(cudaMemcpyAsync(x->d_counts, d_totals, sizeof(int64_t) * N, cudaMemcpyDeviceToDevice, s), "copy counts");
    }
    CUDA_TRY(cudaMemcpyAsync(x->h_counts, x->d_counts, sizeof(int64_t) * (size_t)N * T, cudaMemcpyDeviceToHost, s), "D2H counts");
    // sender-side conversions + per-destination byte counts of the string columns
    std::vector<int> var_cols;
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        uint8_t* send_valid = (uint8_t*)(cb + cv[i].send_valid);
        if (q.in_valid && (rc = launch_bits_to_bytes((const uint8_t*)q.validity, 0, n_rows, send_valid, s))) return rc;
        if (q.nullable && !q.in_valid && n_rows > 0)  // no nulls among my rows: all-valid lane
            CUDA_TRY(cudaMemsetAsync(send_valid, 1, (size_t)n_rows, s), "memset");
        if (q.kind == DFD_COL_BOOL && (rc = launch_bits_to_bytes((const uint8_t*)q.values, 0, n_rows, (uint8_t*)(cb + cv[i].send_values), s))) return rc;
        if (q.var_index >= 0) {
            if ((rc = launch_offsets_to_lengths(q.offsets, q.ow, n_rows, cb + cv[i].send_values, s))) return rc;
            int64_t* d_meta = (int64_t*)(cb + meta_off) + (size_t)q.var_index * 2 * N;
            if ((rc = launch_var_dest_bytes(q.offsets, q.ow, part->d_part_starts, N, d_meta, d_meta + N, s))) return rc;
            var_cols.push_back(i);
        }
    }
    // byte-count matrices of the string columns: all-gather [T][N] per column
    std::vector<int64_t> h_first(V * N), h_bytes(V * (size_t)T * N);
    int64_t* d_bytes_all = nullptr;
    if (V) {
        if ((rc = x->bytes_all.ensure(sizeof(int64_t) * V * (size_t)T * N + 256, c->device))) return rc;
        d_bytes_all = (int64_t*)x->bytes_all.ptr;
        for (size_t v = 0; v < V; ++v) {
            int64_t* d_meta = (int64_t*)(cb + meta_off) + v * 2 * N;
            if (T > 1) {
                ncclResult_t r = n->AllGather(d_meta, d_bytes_all + v * (size_t)T * N, N, ncclInt64, x->comm, s);
                if (r != ncclSuccess) return nccl_error(r, "ncclAllGather(byte counts)");
            } else {
                cudaMemcpyAsync(d_bytes_all + v * N, d_meta, sizeof(int64_t) * N, cudaMemcpyDeviceToDevice, s);
            }
            cudaMemcpyAsync(h_first.data() + v * N, d_meta + N, sizeof(int64_t) * N, cudaMemcpyDeviceToHost, s);
        }
        cudaMemcpyAsync(h_bytes.data(), d_bytes_all, sizeof(int64_t) * V * (size_t)T * N, cudaMemcpyDeviceToHost, s);
    }
    cudaError_t se = cudaStreamSynchronize(s);
    if (se != cudaSuccess) return cuda_error(se, "count exchange");
    // The receiver rebuilds a Utf8 / Binary column's int32 offsets from lengths: no consumer may receive more than INT32_MAX
    // bytes of one.  Checked for every consumer from the all-gathered matrices, so that all workers refuse together and none
    // is left waiting in a send to a peer that refused.
    for (size_t v = 0; v < V; ++v) {
        if (pc[var_cols[v]].ow != 4) continue;
        for (int o = 0; o < T; ++o) {
            int64_t total = 0;
            for (int r = 0; r < T; ++r)
                for (uint32_t q = 0; q < P; ++q) total += h_bytes[v * (size_t)T * N + (size_t)r * N + (size_t)o * P + q];
            if (total > INT32_MAX)
                return set_error(DFD_ERR_CAPACITY, "column %d: consumer %d would receive %lld string bytes, past the int32 offsets of Utf8 / "
                                                   "Binary", var_cols[v], o, (long long)total);
        }
    }
    std::vector<int64_t> send_start(N), recv_start((size_t)P * T);
    int64_t recv_rows = 0;
    rc = dfd_exchange_plan(T, P, x->rank, x->h_counts, send_start.data(), recv_start.data(), part_starts_host, nullptr, &recv_rows);
    if (rc) return rc;
    if (recv_rows > out_capacity_rows)
        return set_error(DFD_ERR_CAPACITY, "this worker receives %lld rows but out_capacity_rows is %lld", (long long)recv_rows,
                         (long long)out_capacity_rows);
    // receive-side byte layout of every string column (same [q][r] order as the rows)
    std::vector<std::vector<int64_t>> brecv_start(V);
    for (size_t v = 0; v < V; ++v) {
        brecv_start[v].resize((size_t)P * T);
        int64_t total = 0;
        rc = dfd_exchange_plan(T, P, x->rank, h_bytes.data() + v * (size_t)T * N, nullptr, brecv_start[v].data(), nullptr, nullptr, &total);
        if (rc) return rc;
        if (total > out_cols[var_cols[v]].values_bytes)
            return set_error(DFD_ERR_CAPACITY, "column %d: receives %lld string bytes but out values_bytes is %lld", var_cols[v],
                             (long long)total, (long long)out_cols[var_cols[v]].values_bytes);
    }
    size_t rtmp = 0;
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        if (q.nullable) { cv[i].recv_valid = rtmp; rtmp += al((size_t)recv_rows + 64); }
        if (q.kind != DFD_COL_FIXED) { cv[i].recv_values = rtmp; rtmp += al((size_t)(recv_rows + 1) * lane_width(q) + 64); }
    }
    const size_t rsums = rtmp;
    rtmp += al((size_t)(recv_rows / (256 * 8) + 4) * 8);
    if ((rc = x->recv_tmp.ensure(rtmp + 256, c->device))) return rc;
    char* rt = (char*)x->recv_tmp.ptr;
    // one "lane" = one stream of w-byte units with its own T x N count matrix, send starts [N] and receive starts [P][T]:
    // the row lanes, then the bytes of every string column
    struct Lane { const char* src; char* dst; size_t w; const int64_t* cnt; const int64_t* send; const int64_t* recv; };
    std::vector<Lane> lanes;
    auto row_lane = [&](const char* src, char* dst, size_t w) { lanes.push_back({src, dst, w, x->h_counts, send_start.data(), recv_start.data()}); };
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        if (q.kind == DFD_COL_FIXED) row_lane(q.values, (char*)out_cols[i].values, (size_t)q.width);
        else row_lane(cb + cv[i].send_values, rt + cv[i].recv_values, lane_width(q));
        if (q.nullable) row_lane(cb + cv[i].send_valid, rt + cv[i].recv_valid, 1);
    }
    for (size_t v = 0; v < V; ++v)
        lanes.push_back({pc[var_cols[v]].values, (char*)out_cols[var_cols[v]].values, 1, h_bytes.data() + v * (size_t)T * N, h_first.data() + v * N,
                         brecv_start[v].data()});
    if (T > 1) NCCL_TRY(n->GroupStart(), "ncclGroupStart");
    for (const Lane& ln : lanes) {
        for (uint32_t g = 0; g < N; ++g) {  // my units of destination g -> its owner
            const int peer = (int)(g / P);
            const int64_t units = ln.cnt[(int64_t)x->rank * N + g];
            if (units == 0) continue;
            if (peer == x->rank) {
                CUDA_TRY(cudaMemcpyAsync(ln.dst + (size_t)ln.recv[(size_t)(g % P) * T + x->rank] * ln.w, ln.src + (size_t)ln.send[g] * ln.w,
                                         (size_t)units * ln.w, cudaMemcpyDeviceToDevice, s), "local segment copy");
            } else {
                NCCL_TRY(n->Send(ln.src + (size_t)ln.send[g] * ln.w, (size_t)units * ln.w, ncclInt8, peer, x->comm, s), "ncclSend");
                x->bytes_sent += (uint64_t)units * ln.w;
            }
        }
        for (int r = 0; r < T; ++r) {  // every producer's units of my P destinations
            if (r == x->rank) continue;
            for (uint32_t q = 0; q < P; ++q) {
                const int64_t units = ln.cnt[(int64_t)r * N + (int64_t)x->rank * P + q];
                if (units == 0) continue;
                NCCL_TRY(n->Recv(ln.dst + (size_t)ln.recv[(size_t)q * T + r] * ln.w, (size_t)units * ln.w, ncclInt8, r, x->comm, s), "ncclRecv");
                x->bytes_received += (uint64_t)units * ln.w;
            }
        }
    }
    if (T > 1) NCCL_TRY(n->GroupEnd(), "ncclGroupEnd");
    // receiver-side rebuild of bitmaps and offsets
    for (int i = 0; i < n_cols; ++i) {
        const PushCol& q = pc[i];
        if (q.nullable && (rc = launch_bytes_to_bits((const uint8_t*)(rt + cv[i].recv_valid), recv_rows, out_cols[i].validity, s))) return rc;
        if (q.kind == DFD_COL_BOOL && (rc = launch_bytes_to_bits((const uint8_t*)(rt + cv[i].recv_values), recv_rows, out_cols[i].values, s))) return rc;
        if (q.var_index >= 0 &&
            (rc = launch_lengths_to_offsets(rt + cv[i].recv_values, q.ow, recv_rows, (unsigned long long*)(rt + rsums), out_cols[i].offsets, s)))
            return rc;
    }
    CUDA_TRY(cudaStreamSynchronize(s), "nccl exchange");
    return DFD_OK;
}

/* Host-to-host shuffle (the end-to-end path of the multi-worker exchange): this worker's rows live in
 * HOST column buffers, its received destinations are delivered into HOST (ideally pinned) buffers.
 * The rows are cut into `n_chunks` equal pieces (every worker must pass the same n_chunks: each chunk
 * is one collective fused shuffle) and pipelined: H2D of chunk i+1 and D2H of chunk i-1 overlap the
 * shuffle of chunk i (two input stages, two receive-window slots).  Output: chunk-major — chunk i's
 * destination q occupies rows [chunk_part_starts[i*(P+1)+q], chunk_part_starts[i*(P+1)+q+1]) of
 * every out column (absolute row offsets), exactly like a stream of per-destination record batches. */
int dfd_shuffle_host(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows,
                     uint32_t partitions_per_task, int n_chunks, const dfd_column* out_cols, int64_t out_capacity_rows,
                     int64_t* chunk_part_starts) {
    if (!x || !part || !in_cols || !out_cols || !chunk_part_starts || n_chunks < 1 || n_rows < 0)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_shuffle_host: bad arguments");
    const uint32_t P = partitions_per_task;
    for (int i = 0; i < n_cols; ++i)
        if (in_cols[i].kind != DFD_COL_FIXED || in_cols[i].validity || in_cols[i].offset != 0 || out_cols[i].kind != DFD_COL_FIXED ||
            out_cols[i].width != in_cols[i].width || !in_cols[i].values || !out_cols[i].values)
            return set_error(DFD_ERR_UNSUPPORTED, "column %d: dfd_shuffle_host moves fixed-width non-null columns", i);
    std::unique_lock<std::mutex> lk;
    int rc = begin_shuffle(x, part, in_cols, out_cols, P, "dfd_shuffle_host", lk);
    if (rc) return rc;
    x->shuffles += (uint64_t)n_chunks - 1;  // one collective fused shuffle per chunk
    dfd_ctx* c = x->ctx;
    if (!x->s_h2d) {
        CUDA_TRY(cudaStreamCreateWithFlags(&x->s_h2d, cudaStreamNonBlocking), "stream");
        CUDA_TRY(cudaStreamCreateWithFlags(&x->s_d2h, cudaStreamNonBlocking), "stream");
        for (int i = 0; i < 2; ++i) {
            CUDA_TRY(cudaEventCreateWithFlags(&x->e_h2d[i], cudaEventDisableTiming), "event");
            CUDA_TRY(cudaEventCreateWithFlags(&x->e_k[i], cudaEventDisableTiming), "event");
            CUDA_TRY(cudaEventCreateWithFlags(&x->e_d2h[i], cudaEventDisableTiming), "event");
        }
    }
    const int64_t max_chunk = (n_rows + n_chunks - 1) / n_chunks + 1;
    std::vector<size_t> col_off(n_cols);
    size_t stage_bytes = 0;
    for (int i = 0; i < n_cols; ++i) {
        col_off[i] = stage_bytes;
        stage_bytes += ((size_t)max_chunk * in_cols[i].width + 255) & ~(size_t)255;
    }
    for (int k = 0; k < 2; ++k)
        if ((rc = x->in_stage[k].ensure(stage_bytes + 256, c->device))) return rc;
    auto chunk_lo = [&](int i) { return (int64_t)((__int128)n_rows * i / n_chunks); };
    auto issue_h2d = [&](int i) -> int {
        const int k = i & 1;
        const int64_t lo = chunk_lo(i), rows = chunk_lo(i + 1) - lo;
        if (i >= 2) CUDA_TRY(cudaStreamWaitEvent(x->s_h2d, x->e_k[k], 0), "wait");  // kernels of chunk i-2 read this stage
        for (int cidx = 0; cidx < n_cols; ++cidx) {
            const size_t w = (size_t)in_cols[cidx].width;
            if (rows)
                CUDA_TRY(cudaMemcpyAsync((char*)x->in_stage[k].ptr + col_off[cidx], (const char*)in_cols[cidx].values + (size_t)lo * w,
                                         (size_t)rows * w, cudaMemcpyHostToDevice, x->s_h2d), "H2D");
        }
        CUDA_TRY(cudaEventRecord(x->e_h2d[k], x->s_h2d), "record");
        return DFD_OK;
    };
    int64_t out_row = 0;
    if ((rc = issue_h2d(0))) return rc;
    std::vector<dfd_column> dev_in(n_cols), win(n_cols);
    for (int i = 0; i < n_chunks; ++i) {
        const int k = i & 1;
        if (i + 1 < n_chunks && (rc = issue_h2d(i + 1))) return rc;
        const int64_t rows = chunk_lo(i + 1) - chunk_lo(i);
        for (int cidx = 0; cidx < n_cols; ++cidx) {
            dev_in[cidx] = in_cols[cidx];
            dev_in[cidx].values = (char*)x->in_stage[k].ptr + col_off[cidx];
        }
        CUDA_TRY(cudaStreamWaitEvent(c->stream, x->e_h2d[k], 0), "wait");
        if (i >= 2) CUDA_TRY(cudaStreamWaitEvent(c->stream, x->e_d2h[k], 0), "wait");  // my window slot k has been drained
        if ((rc = fused_shuffle_locked(x, part, dev_in.data(), n_cols, rows, P, k, 2, win.data(), x->e_k[k]))) return rc;
        const int64_t got = x->h_my_starts[P];
        if (out_row + got > out_capacity_rows)
            return set_error(DFD_ERR_CAPACITY, "dfd_shuffle_host: out buffers hold %lld rows, need more than %lld", (long long)out_capacity_rows,
                             (long long)(out_row + got));
        for (uint32_t q = 0; q <= P; ++q) chunk_part_starts[(size_t)i * (P + 1) + q] = out_row + x->h_my_starts[q];
        for (int cidx = 0; cidx < n_cols; ++cidx) {
            const size_t w = (size_t)in_cols[cidx].width;
            if (got)
                CUDA_TRY(cudaMemcpyAsync((char*)out_cols[cidx].values + (size_t)out_row * w, win[cidx].values, (size_t)got * w,
                                         cudaMemcpyDeviceToHost, x->s_d2h), "D2H");
        }
        CUDA_TRY(cudaEventRecord(x->e_d2h[k], x->s_d2h), "record");
        out_row += got;
    }
    CUDA_TRY(cudaStreamSynchronize(x->s_d2h), "D2H drain");
    return DFD_OK;
}

/* Fused shuffle without the final host synchronisation: everything is enqueued on the context's
 * stream and the call returns; out_cols are set (window pointers) immediately.  Completion,
 * the capacity check and part_starts are delivered by dfd_exchange_wait.  Back-to-back calls
 * pipeline on the stream (each overwrites the window, so consume or wait in between if the data
 * matters). */
int dfd_shuffle_device_async(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows,
                             uint32_t partitions_per_task, dfd_column* out_cols) {
    std::unique_lock<std::mutex> lk;
    int rc = begin_shuffle(x, part, in_cols, out_cols, partitions_per_task, "dfd_shuffle_device_async", lk);
    if (rc) return rc;
    return fused_shuffle_locked(x, part, in_cols, n_cols, n_rows, partitions_per_task, 0, 1, out_cols, nullptr, /*sync=*/false);
}

int dfd_exchange_wait(dfd_exchange* x, int64_t* part_starts_host) {
    if (!x) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL exchange");
    dfd_ctx* c = x->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CUDA_TRY(cudaSetDevice(c->device), "cudaSetDevice");
    dfd_exchange::Pending& pd = x->pending;
    if (pd.kind != dfd_exchange::Pending::DENSE) return set_error(DFD_ERR_INVALID_ARGUMENT, "no asynchronous shuffle is pending");
    pd.kind = dfd_exchange::Pending::NONE;
    int rc = fused_shuffle_finish(x, pd.P, pd.row_bytes);
    if (rc) return rc;
    if (part_starts_host) memcpy(part_starts_host, x->h_my_starts, sizeof(int64_t) * (pd.P + 1));
    return DFD_OK;
}

/* Single-pass fused shuffle (asynchronous): see onepass_shuffle_locked.  Falls back to the two-pass fused path
 * (dense layout) when the schema / partition count is outside the single-pass kernel's envelope. */
int dfd_shuffle_device_onepass(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows,
                               uint32_t partitions_per_task, dfd_column* out_cols) {
    const uint32_t P = partitions_per_task;
    std::unique_lock<std::mutex> lk;
    int rc = begin_shuffle(x, part, in_cols, out_cols, P, "dfd_shuffle_device_onepass", lk);
    if (rc) return rc;
    if (!onepass_supported(part, in_cols, out_cols, n_cols, P))  // nullable / boolean / string columns (or > 256 partitions):
        return push_shuffle_locked(x, part, in_cols, n_cols, n_rows, P, out_cols);  // the push transport moves every column kind
    return onepass_shuffle_locked(x, part, in_cols, n_cols, n_rows, P, 0, 1, out_cols);
}

/* Complete the last dfd_shuffle_device_onepass: per local partition q and producer r, rows
 * [seg_starts[q*T + r], +seg_counts[q*T + r]) of every out column.  If a sub-window overflowed on ANY worker
 * (every worker sees every producer's flag, so all take the same branch) the shuffle is re-run through the two-pass
 * fused path with exact counts; the segments then describe its dense layout. */
// Segment q * T + r = producer r's counts[r * stride + q] rows of my partition q: back to back from x->h_my_starts[q] in the
// dense layout (sub_cap 0), else at the start of its sub-window of sub_cap rows.  Returns the rows of all segments.
static uint64_t fill_segments(const dfd_exchange* x, uint32_t P, const int64_t* counts, size_t stride, int64_t sub_cap, int64_t* seg_starts,
                              int64_t* seg_counts) {
    const int T = x->world;
    uint64_t rows = 0;
    for (uint32_t q = 0; q < P; ++q) {
        int64_t run = sub_cap ? (int64_t)q * T * sub_cap : x->h_my_starts[q];
        for (int r = 0; r < T; ++r) {
            const int64_t cnt = counts[(size_t)r * stride + q];
            if (seg_starts) seg_starts[(size_t)q * T + r] = run;
            if (seg_counts) seg_counts[(size_t)q * T + r] = cnt;
            run += sub_cap ? sub_cap : cnt;
            rows += (uint64_t)cnt;
        }
    }
    return rows;
}

int dfd_exchange_collect(dfd_exchange* x, dfd_column* out_cols, int64_t* seg_starts, int64_t* seg_counts) {
    if (!x) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL exchange");
    dfd_ctx* c = x->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CUDA_TRY(cudaSetDevice(c->device), "cudaSetDevice");
    const int T = x->world;
    dfd_exchange::Pending& pd = x->pending;
    const uint32_t P = pd.P;
    int rc;
    switch (pd.kind) {
        case dfd_exchange::Pending::SEGMENTS:  // the push transport completes inside the call: hand out its segments
            for (size_t i = 0; i < pd.seg_starts.size(); ++i) {
                if (seg_starts) seg_starts[i] = pd.seg_starts[i];
                if (seg_counts) seg_counts[i] = pd.seg_counts[i];
            }
            return DFD_OK;
        case dfd_exchange::Pending::DENSE:  // dense two-pass layout: producers contiguous per partition
            pd.kind = dfd_exchange::Pending::NONE;
            if ((rc = fused_shuffle_finish(x, P, pd.row_bytes))) return rc;
            CUDA_TRY(cudaMemcpy(x->h_counts, x->d_counts, sizeof(int64_t) * (size_t)P * T * T, cudaMemcpyDeviceToHost), "D2H counts");
            fill_segments(x, P, x->h_counts + (size_t)x->rank * P, (size_t)P * T, 0, seg_starts, seg_counts);
            return DFD_OK;
        case dfd_exchange::Pending::REGIONS:
            break;
        default:
            return set_error(DFD_ERR_INVALID_ARGUMENT, "no shuffle is pending");
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream), "single-pass shuffle");
    pd.kind = dfd_exchange::Pending::NONE;
    if (x->h_seg_flags[MAX_RANKS]) return set_error(DFD_ERR_INTERNAL, "a peer worker never signalled completion of the shuffle (did it fail?)");
    bool overflow = false;
    for (int r = 0; r < T; ++r) overflow |= x->h_seg_flags[r] != 0;
    if (overflow) {
        // exact re-run: counts all-gather -> plan -> two-pass peer scatter (every worker takes this branch)
        x->onepass_fallbacks++;
        std::vector<dfd_column> outs(pd.in.size());
        if ((rc = fused_shuffle_locked(x, pd.part, pd.in.data(), (int)pd.in.size(), pd.rows, P, 0, 1, outs.data(), nullptr, /*sync=*/true))) return rc;
        if (out_cols) for (size_t i = 0; i < outs.size(); ++i) out_cols[i] = outs[i];
        fill_segments(x, P, x->h_seg_counts, P, 0, seg_starts, seg_counts);
        return DFD_OK;
    }
    x->bytes_received += fill_segments(x, P, x->h_seg_counts, P, pd.sub_cap, seg_starts, seg_counts) * pd.row_bytes;
    return DFD_OK;
}

/* ---- back-pressure: a shuffle delivered in rounds -------------------------------------------------------------
 * The reference throttles producers with a per-connection byte budget (src/worker/worker_connection_pool.rs:151-153,
 * 251-257): a consumer that cannot take more data yet slows its producers down, it never fails the query.  Here the
 * bounded resource is the consumer's receive window: when a round does not fit (DFD_ERR_CAPACITY, detected from the
 * same global count matrices on every worker, so all workers agree), the remaining rows of EVERY producer are cut
 * into finer row ranges and the round is retried with less data; the consumer drains the window between rounds. */
struct dfd_shuffle_stream {
    dfd_exchange* x = nullptr;
    dfd_partitioner* part = nullptr;
    std::vector<dfd_column> in_cols;
    std::vector<uint8_t> nullable;
    int64_t n_rows = 0;
    uint32_t P = 0;
    // progress as a fraction num / den of every producer's rows (identical on all workers)
    uint64_t num = 0, den = 1;
    uint64_t rounds = 0, splits = 0;
};

int dfd_shuffle_stream_begin(dfd_exchange* x, dfd_partitioner* part, const dfd_column* in_cols, int n_cols, int64_t n_rows,
                             uint32_t partitions_per_task, const uint8_t* nullable, dfd_shuffle_stream** out) {
    if (!x || !part || !in_cols || !out || n_rows < 0 || n_cols < 1) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_shuffle_stream_begin: bad arguments");
    if (part->ctx != x->ctx) return set_error(DFD_ERR_INVALID_ARGUMENT, "partitioner and exchange belong to different contexts");
    if (partitions_per_task < 1 || (uint64_t)partitions_per_task * x->world != part->N)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "num_partitions %u != partitions_per_task %u x %d workers", part->N, partitions_per_task, x->world);
    dfd_shuffle_stream* st = new (std::nothrow) dfd_shuffle_stream();
    if (!st) return set_error(DFD_ERR_OOM, "out of host memory");
    st->x = x; st->part = part; st->n_rows = n_rows; st->P = partitions_per_task;
    st->in_cols.assign(in_cols, in_cols + n_cols);
    st->nullable.assign((size_t)n_cols, 0);
    for (int i = 0; i < n_cols; ++i) st->nullable[i] = (nullable ? nullable[i] != 0 : false) || in_cols[i].validity != nullptr;
    *out = st;
    return DFD_OK;
}

void dfd_shuffle_stream_end(dfd_shuffle_stream* st) { delete st; }

int dfd_shuffle_stream_stats(const dfd_shuffle_stream* st, uint64_t* rounds, uint64_t* splits) {
    if (!st) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL stream");
    if (rounds) *rounds = st->rounds;
    if (splits) *splits = st->splits;
    return DFD_OK;
}

/* Collective.  Delivers the next round into the receive window: out_cols / segments (P x T) are valid until the next call.
 * *done is set to 1 when every row has been delivered (this call then delivered nothing). */
int dfd_shuffle_stream_next(dfd_shuffle_stream* st, dfd_column* out_cols, int64_t* seg_starts, int64_t* seg_counts, int* done) {
    if (!st || !out_cols || !done) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_shuffle_stream_next: NULL argument");
    dfd_exchange* x = st->x;
    const int n_cols = (int)st->in_cols.size();
    const size_t nseg = (size_t)st->P * x->world;
    if (st->num == st->den) {
        *done = 1;
        for (size_t i = 0; i < nseg; ++i) { if (seg_starts) seg_starts[i] = 0; if (seg_counts) seg_counts[i] = 0; }
        return DFD_OK;
    }
    *done = 0;
    for (;;) {
        const int64_t lo = (int64_t)((unsigned __int128)st->n_rows * st->num / st->den);
        const int64_t hi = (int64_t)((unsigned __int128)st->n_rows * (st->num + 1) / st->den);
        std::vector<dfd_column> cols(st->in_cols);
        for (int i = 0; i < n_cols; ++i) {
            cols[i].offset += lo;
            out_cols[i] = dfd_column{};
            out_cols[i].validity = st->nullable[i] ? (uint8_t*)1 : nullptr;  // the schema's nullable flag (see dfd_shuffle_device_onepass)
        }
        int rc = dfd_shuffle_device_onepass(x, st->part, cols.data(), n_cols, hi - lo, st->P, out_cols);
        if (rc == DFD_OK) rc = dfd_exchange_collect(x, out_cols, seg_starts, seg_counts);
        if (rc == DFD_OK) {
            st->num += 1;
            st->rounds++;
            return DFD_OK;
        }
        if (rc != DFD_ERR_CAPACITY) return rc;
        // the round does not fit some consumer's window: every worker saw the same counts and splits the same way
        if (st->den > (uint64_t)1 << 40) return set_error(DFD_ERR_CAPACITY, "receive windows too small even for single-row rounds");
        st->num *= 2;
        st->den *= 2;
        st->splits++;
    }
}

/* Pure host arithmetic of NetworkCoalesceExec's task grouping (src/execution_plans/network_coalesce.rs:264-289 `task_group`). */
int dfd_coalesce_task_group(int input_task_count, int task_index, int task_count, int* start_task, int* len, int* max_len) {
    if (input_task_count < 0 || task_index < 0 || task_count < 0 || !start_task || !len || !max_len)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_coalesce_task_group: bad arguments");
    if (task_count == 0) { *start_task = 0; *len = 0; *max_len = 0; return DFD_OK; }
    Route R{DFD_ROUTE_COALESCE, 1, input_task_count, task_count};
    R.group(task_index, start_task, len, max_len);
    if (task_index >= task_count) *len = 0;
    return DFD_OK;
}

int dfd_route_segment_source(int route, uint32_t partitions, int producer_tasks, int consumer_tasks, int consumer, uint32_t segment,
                             int* producer, uint32_t* slice, uint32_t* n_segments) {
    if ((route != DFD_ROUTE_SHUFFLE && route != DFD_ROUTE_COALESCE && route != DFD_ROUTE_BROADCAST) || partitions < 1 || producer_tasks < 1 ||
        consumer_tasks < 1 || consumer_tasks > producer_tasks || consumer < 0 || consumer >= producer_tasks)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_route_segment_source: bad arguments");
    if (route == DFD_ROUTE_SHUFFLE && consumer_tasks != producer_tasks)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_route_segment_source: a shuffle has as many consumer tasks as workers");
    const Route R{route, partitions, producer_tasks, consumer_tasks};
    const uint32_t n = R.n_segments(consumer);
    if (n_segments) *n_segments = n;
    if (producer || slice) {
        if (segment >= n) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_route_segment_source: segment %u out of range [0,%u)", segment, n);
        int r = -1;
        uint32_t g = 0;
        R.source(consumer, segment, &r, &g);
        if (producer) *producer = r;
        if (slice) *slice = g;
    }
    return DFD_OK;
}

/* Coalesce / broadcast over the same NVLink transport (no repartition): this worker, as producer task `rank`, holds
 * `P` partitions = the row slices [slice_starts[j], slice_starts[j+1]) of in_cols. */
int dfd_exchange_gather(dfd_exchange* x, int route, const dfd_column* in_cols, int n_cols, const int64_t* slice_starts, uint32_t P,
                        int consumer_tasks, dfd_column* out_cols) {
    if (!x || !in_cols || !out_cols || !slice_starts || P < 1 || n_cols < 1)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_exchange_gather: bad arguments");
    if (route != DFD_ROUTE_COALESCE && route != DFD_ROUTE_BROADCAST && route != DFD_ROUTE_SHUFFLE)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "unknown route %d", route);
    if (consumer_tasks < 1 || consumer_tasks > x->world || (route == DFD_ROUTE_SHUFFLE && consumer_tasks != x->world))
        return set_error(DFD_ERR_INVALID_ARGUMENT, "consumer_tasks %d not in [1, %d workers] (pre-partitioned shuffle: == workers)", consumer_tasks, x->world);
    const uint32_t n_slices = route == DFD_ROUTE_SHUFFLE ? P * (uint32_t)x->world : P;
    dfd_ctx* c = x->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    x->pending.kind = dfd_exchange::Pending::NONE;
    CUDA_TRY(cudaSetDevice(c->device), "cudaSetDevice");
    if (!x->window_ready) return set_error(DFD_ERR_INVALID_ARGUMENT, "the exchange needs dfd_exchange_setup_window first");
    cudaStream_t s = c->stream;
    std::vector<PushCol> pc;
    int rc = describe_columns(in_cols, out_cols, n_cols, pc);
    if (rc) return rc;
    // device copy of the slice boundaries + scratch for the per-slice byte offsets
    const size_t need = ((size_t)(n_slices + 1) * 8 + 255) / 256 * 256 + (size_t)(n_var_cols(pc) + 1) * n_slices * 8 + 256;
    if ((rc = x->recv_tmp.ensure(need, c->device))) return rc;
    int64_t* d_starts = (int64_t*)x->recv_tmp.ptr;
    char* scratch = (char*)x->recv_tmp.ptr + ((size_t)(n_slices + 1) * 8 + 255) / 256 * 256;
    for (uint32_t j = 0; j < n_slices; ++j)
        if (slice_starts[j + 1] < slice_starts[j]) return set_error(DFD_ERR_INVALID_ARGUMENT, "slice_starts must be non-decreasing");
    CUDA_TRY(cudaMemcpyAsync(d_starts, slice_starts, sizeof(int64_t) * (n_slices + 1), cudaMemcpyHostToDevice, s), "H2D slice starts");
    CUDA_TRY(cudaStreamSynchronize(s), "sync");  // (slice_starts is caller memory)
    Route R{route, P, x->world, consumer_tasks};
    x->shuffles++;
    return push_slices_locked(x, pc, in_cols, R, d_starts, scratch, out_cols);
}

uint32_t dfd_exchange_pending_segments(const dfd_exchange* x) {
    return x && x->pending.kind == dfd_exchange::Pending::SEGMENTS ? (uint32_t)x->pending.seg_starts.size() : 0;
}

int dfd_exchange_stats(dfd_exchange* x, uint64_t* bytes_sent, uint64_t* bytes_received, uint64_t* shuffles) {
    if (!x) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL exchange");
    if (bytes_sent) *bytes_sent = x->bytes_sent;
    if (bytes_received) *bytes_received = x->bytes_received;
    if (shuffles) *shuffles = x->shuffles;
    return DFD_OK;
}

uint64_t dfd_exchange_onepass_fallbacks(const dfd_exchange* x) { return x ? x->onepass_fallbacks : 0; }

/* Mean CUDA-event durations (ms) of the three stream phases of the single-pass shuffles recorded while the context was in
 * profiling mode: [0] k_xchg_signal_ready, [1] k_scatter_onepass<PEER> (+ follow-up launches), [2] k_xchg_publish_wait
 * (flag stores + waiting for the slowest producer).  Synchronises; resets the accumulators. */
int dfd_exchange_phase_ms(dfd_exchange* x, double* out3, uint64_t* n_shuffles) {
    if (!x || !out3) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL argument");
    dfd_ctx* c = x->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CUDA_TRY(cudaSetDevice(c->device), "cudaSetDevice");
    CUDA_TRY(cudaStreamSynchronize(c->stream), "sync");
    EventRing& r = x->phases;
    if (int rc = r.drain()) return rc;
    for (int k = 0; k < 3; ++k) out3[k] = r.calls ? r.sum_ms[k] / (double)r.calls : 0.0;
    if (n_shuffles) *n_shuffles = r.calls;
    r.reset();
    return DFD_OK;
}

}  // extern "C"
