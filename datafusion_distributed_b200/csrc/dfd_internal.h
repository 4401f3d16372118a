// dfd_internal.h — host-side objects behind the opaque C ABI handles.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "dfd_b200.h"
#include "dfd_hash.cuh"
#include "dfd_types.cuh"

namespace dfd {

int set_error(int code, const char* fmt, ...);
int cuda_error(cudaError_t e, const char* what);

#define CUDA_TRY(call, what)                                   \
    {                                                          \
        cudaError_t _e = (call);                               \
        if (_e != cudaSuccess) return dfd::cuda_error(_e, what); \
    }

struct Scratch {
    void* ptr = nullptr;
    size_t bytes = 0;
    int ensure(size_t need, int device);
};

// Profiling: the CUDA events of up to CALLS calls, four per call (three consecutive phases), recorded without a sync.
// The phase durations are summed when the ring is full and whenever the owner reads them.  (Inline: the exchange is
// also linked without dfd_api.cu.)
struct EventRing {
    static constexpr size_t CALLS = 64;
    std::vector<cudaEvent_t> ev;     // 4 per call, created on first use
    size_t pending = 0;              // calls recorded, not yet summed
    double sum_ms[3] = {0, 0, 0};    // phase durations of the calls summed since reset()
    uint64_t calls = 0;              // ... and their number

    EventRing() = default;
    EventRing(const EventRing&) = delete;
    EventRing& operator=(const EventRing&) = delete;
    ~EventRing() {
        for (cudaEvent_t e : ev) cudaEventDestroy(e);
    }
    // The event quad of the next call (summing the ring first if it is full); commit() once its last event is recorded.
    int next(cudaEvent_t** quad) {
        if (ev.empty()) {
            ev.resize(4 * CALLS);
            for (cudaEvent_t& e : ev) cudaEventCreate(&e);
        }
        if (pending == CALLS) {
            if (int rc = drain()) return rc;
        }
        *quad = &ev[4 * pending];
        return DFD_OK;
    }
    void commit() { ++pending; }
    // Waits for the recorded calls and adds their phase durations to the sums.
    int drain() {
        if (pending == 0) return DFD_OK;
        CUDA_TRY(cudaEventSynchronize(ev[4 * pending - 1]), "partition kernels");
        for (size_t i = 0; i < pending; ++i)
            for (int k = 0; k < 3; ++k) {
                float ms = 0;
                cudaEventElapsedTime(&ms, ev[4 * i + k], ev[4 * i + k + 1]);
                sum_ms[k] += ms;
            }
        calls += pending;
        pending = 0;
        return DFD_OK;
    }
    void reset() {
        sum_ms[0] = sum_ms[1] = sum_ms[2] = 0;
        calls = 0;
    }
};

}  // namespace dfd

// One worker == one GPU (reference `Worker`, src/worker/worker_service.rs:39-49).
struct dfd_ctx {
    int device = 0;
    int sm_count = 132;
    size_t l2_bytes = 0;
    cudaStream_t stream = nullptr;  // compute stream: K1/K1b/K2 launch here
    dfd::EventRing phases;          // profiling: K1 / K1b / K2 phases of every partition call (dfd_metrics hist/scan/scatter_ms)
    cudaEvent_t timer_a = nullptr, timer_b = nullptr;
    bool profiling = false;
    dfd::Scratch scratch;  // tile histograms / cursors
    void* scratch_done = nullptr;  // zero-initialised "blocks done" counter inside scratch
    dfd::Scratch flush;    // L2 flush buffer
    dfd::Scratch var_scratch;  // K4: iota | src row ids | block sums
    dfd::Scratch lb;           // single-pass mode: [ticket, done | 256 B] [look-back descriptors u64 [N][n_tiles]]
    uint32_t lb_epoch = 0;     // epoch of the last single-pass launch (30 bits; descriptors of older epochs are stale)
    dfd_metrics metrics = {};
    std::shared_ptr<void> pinned_cache;  // host operator: pinned output chunks of finished operators (dfd_exec.cu: PinnedCache)
    std::mutex mu;
};

// ≙ DataFusion BatchPartitioner::Hash { exprs, num_partitions, hash_buffer, random_state }
struct dfd_partitioner {
    dfd_ctx* ctx = nullptr;
    uint32_t N = 0;
    std::vector<int32_t> key_cols;
    std::vector<int32_t> key_modes;  // dfd_key_hash_mode per key column
    struct KeyDict { const uint64_t* hashes = nullptr; const uint8_t* validity = nullptr; bool index_unsigned = false; };
    std::vector<KeyDict> key_dicts;  // DFD_KEY_HASH_DICTIONARY: device hashes / validity of the dictionary values
    dfd::HashState st{};
    dfd::ModN mod{};
    int64_t* d_part_starts = nullptr;  // [N+1]
    // single-pass (region layout) state: results of the last dfd_partition_device_onepass
    int64_t* d_counts = nullptr;       // [N] rows per destination | [N] dest_base | [N] dest_cap (exact re-run) | overflow flag
    int64_t* h_pin = nullptr;          // pinned: [N] counts, then the overflow flag
    enum { LAST_NONE = 0, LAST_DENSE = 1, LAST_REGIONS = 2 } last = LAST_NONE;
    std::vector<dfd_column> last_in, last_out;
    int64_t last_rows = 0, last_stride = 0;
    bool bit_rows = false;             // accept COL_BIT_ROWS columns (set by the host operator for its own partitioner only)
};

namespace dfd {
using Ctx = ::dfd_ctx;
using Partitioner = ::dfd_partitioner;

// What a scatter launch is: the two-pass k_scatter on the K1 tiling (TILE_K), the single-pass k_scatter_onepass
// (ONEPASS_K), or a follow-up k_scatter on the single-pass tiling: further width groups / bit columns of a single-pass
// call, driven by the per-tile counts and cursors the single-pass launch left in hist_out / base_out.
enum class ScatterKind { TwoPass, OnePass, FollowUp };

// One partition call split into its stages so the exchange can put the count
// all-gather between K1b and K2.  Caller holds ctx->mu and has set the device.
struct PartitionJob {
    Partitioner* p = nullptr;
    cudaStream_t stream = nullptr;
    bool peer = false;
    KeySet ks{};
    std::vector<PayloadCol> passes;
    struct VarCol { dfd_column in, out; };
    std::vector<VarCol> var_cols;        // K4: variable-width payload columns
    uint32_t* d_src = nullptr;            // K4 and the gathers: input row of every output row (scattered iota)
    unsigned long long* d_block_sums = nullptr;
    uint64_t bytes = 0;
    int64_t n_rows = 0, n_tiles = 0;
    bool var_bytes_known = false;        // set before prepare(): in_cols[i].values_bytes IS the byte count of a var-width input (no D2H read + sync)
    bool onepass_tiling = false;         // set before prepare(): tile the rows for the single-pass kernel (ONEPASS_K rows per thread)
    bool gather_wide = false;            // set before prepare(): accept fixed widths outside {1,2,4,8,16} (two-pass local calls)
    struct GatherCol { const void* in; void* out; int64_t in_offset, width; };
    std::vector<GatherCol> gathers;      // wide fixed-width columns, gathered through d_src after K2 (k_gather_rows)
    std::vector<GatherCol> bit_gathers;  // COL_BIT_ROWS columns (width = bits per row), gathered the same way (k_gather_bit_rows)
    int64_t out_rows = -1;               // rows of the OUTPUT row space (-1: n_rows; single-pass regions: N * region_rows)
    uint32_t* d_hist = nullptr;
    uint32_t* d_base = nullptr;
    int64_t* d_totals = nullptr;  // [N] rows per destination (after run_hist_scan)
    unsigned* d_done = nullptr;
    uint16_t* d_dest_cache = nullptr;  // two-pass, non-trivial keys: destination of every row (written by K1, read by every K2 launch)
    cudaEvent_t* ev = nullptr;
    int prepare(Partitioner* part, const dfd_column* in_cols, int n_cols, int64_t rows, const dfd_column* out_cols,
                bool peer_mode, cudaStream_t st);
    int run_hist_scan();
    int run_scatter(const int64_t* dest_base, void* const* peer_base, int world, uint32_t parts_per_rank,
                    const int32_t* abort_flag);
    int run_varwidth();  // called by run_scatter after the fixed-width launches
    int run_gathers();   // called by run_scatter after the fixed-width launches
    // Single-pass K2 (no K1/K1b): destinations live in fixed regions; see k_scatter<..., ONEPASS>.
    struct OnePassLayout {
        const int64_t* d_dest_base = nullptr;  // device [N] region starts (rows); nullptr: region_stride formula
        const int64_t* d_dest_cap = nullptr;   // device [N] region capacities; nullptr: region_stride
        int64_t region_stride = 0;
        void* const* peer_base = nullptr;      // peer mode: every rank's window slot
        int world = 1, rank = 0;
        uint32_t parts_per_rank = 1;
        int64_t* d_totals = nullptr;           // device [N] out: rows per destination
        int32_t* d_overflow = nullptr;         // device out: set to 1 if a region is too small (caller zeroes it)
        const unsigned long long* ready_flags = nullptr;  // peer mode: "window free" flags in my header (see ExchangeHeader)
        unsigned long long ready_epoch = 0;
    };
    int run_onepass(const OnePassLayout& L);

  private:
    int scatter_params(ScatterParams& sp, void* const* peer_base, int world, uint32_t parts_per_rank) const;
    int launch_width_groups(ScatterParams& sp, const std::vector<PayloadCol>& cols, ScatterKind kind, int* launches);
    void finish(int launches);
};

constexpr uint32_t ONEPASS_MAX_N = 256;  // above this the per-tile look-back costs more than the K1 pass it replaces

// Small conversion kernels the exchange uses for bit-packed / variable-width columns (defined in dfd_api.cu).
int launch_bits_to_bytes(const uint8_t* bits, int64_t bit_offset, int64_t n, uint8_t* out, cudaStream_t s);
int launch_bytes_to_bits(const uint8_t* in, int64_t n, void* out_words, cudaStream_t s);
int launch_offsets_to_lengths(const void* off, int ow, int64_t n, void* len, cudaStream_t s);
int launch_var_dest_bytes(const void* off, int ow, const int64_t* part_starts, uint32_t N, int64_t* bytes, int64_t* first, cudaStream_t s);
int launch_lengths_to_offsets(const void* len, int ow, int64_t n, unsigned long long* block_sums /*[n/2048 + 2]*/, void* out_off, cudaStream_t s);

// Gather after K2 through src, the input row of every output row (kernel in dfd_gather.cu): out row j (w bytes) = in row
// in_offset + src[j], for the fixed widths no scatter instantiation moves.
int launch_gather_rows(const void* in, int64_t in_offset, const uint32_t* src, int64_t n_rows, int64_t w, void* out, int sm_count, cudaStream_t s);
// The same for rows of n bits (a bitmap of n_rows x n bits, row r at bit (in_offset + r) x n): out bits [j n, (j + 1) n) = in
// bits [(in_offset + src[j]) n, ...).  Every output word up to bit n_rows x n is written whole; its bits past the end are zero.
int launch_gather_bit_rows(const void* in, int64_t in_offset, const uint32_t* src, int64_t n_rows, int64_t n, void* out, int sm_count, cudaStream_t s);
// Fixed widths the scatter instantiations move; other widths are gathered (two-pass local partition calls only).
inline bool scatter_width(int64_t w) { return w == 1 || w == 2 || w == 4 || w == 8 || w == 16; }

// Device-side chunk assembly for device-resident input batches (dfd_repartition_exec_push_device; kernels in dfd_stage.cu).
// One StageJob appends one buffer of one column to the open chunk; all jobs of a pushed batch go out in one launch
// (STAGE_MAX_JOBS per launch, as a __grid_constant__ table).  Offsets are re-based as dst[r] = base + scale * (src[r] - src[0]).
enum StageOp : int32_t {
    STAGE_COPY = 0,      // dst[0, n) = src[0, n) (bytes)
    STAGE_BITS = 1,      // bitmap append: dst bits [c, b) = 1, dst bits [b, b + n) = src bits [a, a + n) (src NULL: all ones)
    STAGE_OFFSETS = 2,   // dst[r] = base + scale * (src[r] - src[0]), r in [0, n]; ow_in / ow_out = 4 or 8 bytes
    STAGE_LIST_OFFSETS = 3,  // list child bytes: dst[r] = base + src2[src[r]] - src2[src[0]], r in [0, n] (int32 list + child offsets)
    STAGE_DIFF32 = 4,    // element lengths: dst[k] = src[k + 1] - src[k], k < n (int32)
    STAGE_FILL32 = 5,    // dst[k] = (int32) base, k < n
    STAGE_BIT_BYTES = 6, // dst[k] = bit a + k of src (src NULL: 1), one byte each, k < n
    STAGE_VIEW_BYTES = 7,  // 16-byte views src[0, n) -> bytes at dst + src3[r] (src3 = int32 offsets, src2 = data buffer table)
};
struct StageJob {
    int32_t op = STAGE_COPY, ow_in = 4, ow_out = 4, pad = 0;
    const void* src = nullptr;
    const void* src2 = nullptr;
    const void* src3 = nullptr;
    void* dst = nullptr;
    int64_t n = 0, a = 0, b = 0, c = 0, base = 0, scale = 1;
};
constexpr int STAGE_MAX_JOBS = 32;
// The two staging launches are WEAK references of the operator object: it also links without dfd_stage.cu (a build of the
// operator's host logic on its own, with no device code), and push_device then refuses device batches with an error —
// never a fallback.  libdfd_b200.so always links dfd_stage.cu, so there both are defined.
__attribute__((weak)) int launch_stage_batch(const StageJob* jobs, int n_jobs, cudaStream_t s);

// What the host must know of a var-width column before it stages rows [lo, lo + n): read back once per pushed batch.
enum StageSizeOp : int32_t {
    STAGE_SIZE_RANGE = 0,  // out[0] = off[lo], out[1] = off[lo + n] (ow = 4 or 8)
    STAGE_SIZE_LIST = 1,   // out[0] = e0 = off[lo], out[1] = e1 = off[lo + n]; with off2 (child offsets): out[2] = off2[e0], out[3] = off2[e1]
    STAGE_SIZE_VIEW = 2,   // lens[r] = length of view lo + r (0 when null), out[0] += sum of lens (caller zeroes out)
};
struct StageSize {
    int32_t op = STAGE_SIZE_RANGE, ow = 4;
    const void* off = nullptr;
    const void* off2 = nullptr;
    const uint8_t* valid = nullptr;
    int64_t lo = 0, n = 0;
    int32_t* lens = nullptr;
    int64_t* out = nullptr;  // 4 values
};
__attribute__((weak)) int launch_stage_sizes(const StageSize* jobs, int n_jobs, cudaStream_t s);

// Device-resident OUTPUT (dfd_repartition_exec_execute_device; kernel in dfd_emit.cu): what the host does per row when it
// finishes a host chunk, done on the device for a device chunk — all view and list columns of a chunk in one launch.
enum EmitOp : int32_t {
    EMIT_VIEWS = 0,        // int32 off[0, n] + bytes -> n 16-byte views at dst (bit-identical to host::build_views) and the
                           //   int64 variadic buffer size off[n] at dst2
    EMIT_LIST_OFFSETS = 1, // dst[r] >>= 2, r in [0, n]: byte offsets into the 4-byte lengths -> element offsets (int32, in place)
};
struct EmitJob {
    int32_t op = EMIT_VIEWS, pad = 0;
    const void* off = nullptr;    // views: int32 offsets
    const void* bytes = nullptr;  // views: the string bytes, a 4-byte aligned buffer of off[n] bytes
    void* dst = nullptr;
    void* dst2 = nullptr;
    int64_t n = 0;
};
// Weak like the staging launches: without dfd_emit.cu the operator object still links, and creating a device-output operator
// fails with DFD_ERR_UNSUPPORTED.  libdfd_b200.so always links it.
__attribute__((weak)) int launch_emit_chunk(const EmitJob* jobs, int n_jobs, cudaStream_t s);

// One scatter launch of a width group (template in dfd_launch.cuh).  Each (PEER, KIND) is instantiated in a translation unit
// of its own (dfd_scatter_<kind>_<local|peer>.cu) so that they compile in parallel; nowhere else.
template <bool PEER, ScatterKind KIND>
int launch_scatter_impl(const ScatterParams& sp, int width, bool fast, int sm_count, cudaStream_t stream);
extern template int launch_scatter_impl<false, ScatterKind::TwoPass>(const ScatterParams&, int, bool, int, cudaStream_t);
extern template int launch_scatter_impl<true, ScatterKind::TwoPass>(const ScatterParams&, int, bool, int, cudaStream_t);
extern template int launch_scatter_impl<false, ScatterKind::OnePass>(const ScatterParams&, int, bool, int, cudaStream_t);
extern template int launch_scatter_impl<true, ScatterKind::OnePass>(const ScatterParams&, int, bool, int, cudaStream_t);
extern template int launch_scatter_impl<false, ScatterKind::FollowUp>(const ScatterParams&, int, bool, int, cudaStream_t);
extern template int launch_scatter_impl<true, ScatterKind::FollowUp>(const ScatterParams&, int, bool, int, cudaStream_t);

// Column kinds that only the host operator hands to hash_columns_locked, never part of the C ABI: Interval(DayTime) (8 bytes)
// and Interval(MonthDayNano) (16 bytes) dictionary VALUES, hashed field by field like interval keys (KEY_HASH_INTERVAL_*).
constexpr int32_t COL_INTERVAL_DAY_TIME = 5, COL_INTERVAL_MONTH_DAY_NANO = 6;
// Payload kind of the host operator's own partitioner (dfd_partitioner::bit_rows), never part of the C ABI: rows of `width`
// BITS each in a bitmap (`values`, bit 0 of row r at bit (offset + r) x width), moved by k_gather_bit_rows.  The bit rows of a
// FixedSizeList column: its child's validity, or the values of a Boolean child.  May carry a row validity bitmap.
constexpr int32_t COL_BIT_ROWS = 7;

// create_hashes over device columns -> raw u64 row hashes (dictionary values, parity hook).  Besides the DFD_COL_* kinds a
// column may be COL_INTERVAL_DAY_TIME / COL_INTERVAL_MONTH_DAY_NANO.  Caller holds ctx->mu.
int hash_columns_locked(Ctx* c, const dfd_column* cols, int n_cols, int64_t n_rows, const uint64_t* seeds, uint64_t* hashes_device, cudaStream_t stream);

// Launches K1 -> K1b -> K2 on `stream`; caller holds ctx->mu and has set the device.
// Fixed-width values of any width >= 1 are accepted: widths outside {1,2,4,8,16} are gathered after K2.
int partition_device_locked(Partitioner* p, const dfd_column* in_cols, int n_cols, int64_t n_rows,
                            const dfd_column* out_cols, cudaStream_t stream, bool var_bytes_known = false);

}  // namespace dfd
