// include/dfd_b200.hpp — C++17 host-side mirror of the reference's operator surface for the
// hash-repartition shuffle, layered on the C ABI (dfd_b200.h).  Header-only, no CUDA headers needed.
//
// The reference is compiled Rust; its toolchain is absent from the build image, so this is the
// compiled-language host side a C++ engine (or a cxx/bindgen bridge) would use.  Names and
// argument meaning follow the reference:
//   Partitioning::Hash(exprs, n), scale_partitioning     src/execution_plans/common.rs:17-26
//   Stage / ExecutionTask / DistributedTaskContext        src/stage.rs:71-106
//   RepartitionExec::try_new(input, Hash) + execute(p)    (DataFusion; built at network_shuffle.rs:126-134)
//   NetworkShuffleExec::try_new / execute                 src/execution_plans/network_shuffle.rs:115-157, 213-238
// Errors: every failing C call becomes a dfd::Error carrying the dfd_status code (the Rust shim maps
// the same codes onto DataFusionError, see INTEGRATION.md).
#pragma once
#include <array>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "dfd_b200.h"

namespace dfd {

class Error : public std::runtime_error {
public:
    Error(int status, const std::string& msg) : std::runtime_error(std::string(dfd_status_name(status)) + ": " + msg), status_(status) {}
    int status() const { return status_; }

private:
    int status_;
};

inline void check(int status) {
    if (status != DFD_OK) throw Error(status, dfd_last_error());
}

// `Partitioning::Hash(exprs, n)` restricted to column-reference expressions.
struct Partitioning {
    std::vector<int32_t> key_cols;
    uint32_t partition_count = 0;
    static Partitioning Hash(std::vector<int32_t> keys, uint32_t n) { return Partitioning{std::move(keys), n}; }
};

// src/execution_plans/common.rs:17-26
template <typename F>
inline Partitioning scale_partitioning(const Partitioning& p, F f) {
    return Partitioning{p.key_cols, static_cast<uint32_t>(f(p.partition_count))};
}

struct ExecutionTask {  // src/stage.rs:85-89 (here a worker's "url" is its rank on the NVSwitch box)
    int url = -1;
};

struct Stage {  // src/stage.rs:71-82
    std::array<uint8_t, 16> query_id{};
    size_t num = 0;
    Partitioning plan;
    std::vector<ExecutionTask> tasks;
};

struct DistributedTaskContext {  // src/stage.rs:92-106
    size_t task_index = 0;
    size_t task_count = 1;
};

// One worker == one GPU (reference `Worker`, src/worker/worker_service.rs:39-49).
class WorkerContext {
public:
    explicit WorkerContext(int device = 0) { check(dfd_ctx_create(device, &ctx_)); }
    ~WorkerContext() { dfd_ctx_destroy(ctx_); }
    WorkerContext(const WorkerContext&) = delete;
    WorkerContext& operator=(const WorkerContext&) = delete;
    dfd_ctx* get() const { return ctx_; }
    void synchronize() { check(dfd_ctx_synchronize(ctx_)); }
    void* device_alloc(size_t bytes) { void* p = nullptr; check(dfd_device_alloc(ctx_, bytes, &p)); return p; }
    void device_free(void* p) { check(dfd_device_free(ctx_, p)); }
    void* host_alloc(size_t bytes) { void* p = nullptr; check(dfd_host_alloc(ctx_, bytes, &p)); return p; }
    void host_free(void* p) { check(dfd_host_free(ctx_, p)); }
    void h2d(void* dst, const void* src, size_t n) { check(dfd_memcpy_h2d(ctx_, dst, src, n)); }
    void d2h(void* dst, const void* src, size_t n) { check(dfd_memcpy_d2h(ctx_, dst, src, n)); }
    dfd_metrics metrics() { dfd_metrics m; check(dfd_metrics_get(ctx_, &m)); return m; }

private:
    dfd_ctx* ctx_ = nullptr;
};

inline dfd_column fixed_column(void* values, int32_t width, uint8_t* validity = nullptr, int64_t offset = 0) {
    return dfd_column{DFD_COL_FIXED, width, values, nullptr, validity, offset, 0};
}

// ≙ DataFusion `BatchPartitioner::try_new(Partitioning::Hash(..))` on one GPU.
class HashPartitioner {
public:
    HashPartitioner(WorkerContext& ctx, const Partitioning& p, const uint64_t* seeds = nullptr) : partitioning_(p) {
        check(dfd_partitioner_create(ctx.get(), p.partition_count, p.key_cols.data(), (int)p.key_cols.size(), seeds, &h_));
    }
    ~HashPartitioner() { dfd_partitioner_destroy(h_); }
    HashPartitioner(const HashPartitioner&) = delete;
    HashPartitioner& operator=(const HashPartitioner&) = delete;
    dfd_partitioner* get() const { return h_; }
    const Partitioning& partitioning() const { return partitioning_; }
    // device columns in -> device columns out (destination-sorted), returns part_starts[N+1]
    std::vector<int64_t> partition(const std::vector<dfd_column>& in, int64_t n_rows, const std::vector<dfd_column>& out) {
        std::vector<int64_t> starts(partitioning_.partition_count + 1);
        check(dfd_partition_device(h_, in.data(), (int)in.size(), n_rows, out.data(), starts.data()));
        return starts;
    }

private:
    Partitioning partitioning_;
    dfd_partitioner* h_ = nullptr;
};

// `RepartitionExec::try_new(input, Partitioning::Hash(exprs, n))` with host Arrow batches in/out.
class RepartitionExec {
public:
    RepartitionExec(WorkerContext& ctx, const ArrowSchema* schema, const Partitioning& p, const dfd_exec_options* opts = nullptr)
        : partitioning_(p) {
        check(dfd_repartition_exec_create(ctx.get(), schema, p.key_cols.data(), (int)p.key_cols.size(), p.partition_count, opts, &h_));
    }
    ~RepartitionExec() { dfd_repartition_exec_destroy(h_); }
    RepartitionExec(const RepartitionExec&) = delete;
    RepartitionExec& operator=(const RepartitionExec&) = delete;
    const char* name() const { return "RepartitionExec"; }
    const Partitioning& output_partitioning() const { return partitioning_; }
    void push_batch(ArrowArray* batch) { check(dfd_repartition_exec_push(h_, batch)); }  // ownership moves
    void finish() { check(dfd_repartition_exec_finish(h_)); }
    void abort(const std::string& message) { check(dfd_repartition_exec_abort(h_, message.c_str())); }  // input failed: every stream ends with EIO + message
    void run(ArrowArrayStream* input) { check(dfd_repartition_exec_run(h_, input)); }
    // ≙ ExecutionPlan::execute(partition, ctx) -> SendableRecordBatchStream
    void execute(uint32_t partition, ArrowArrayStream* out) { check(dfd_repartition_exec_execute(h_, partition, out)); }
    // device-resident batches in / out (an operator created with dfd_exec_options.device_output = 1 for the output side)
    void push_device_batch(ArrowDeviceArray* batch) { check(dfd_repartition_exec_push_device(h_, batch)); }  // ownership moves
    void run_device(ArrowDeviceArrayStream* input) { check(dfd_repartition_exec_run_device(h_, input)); }
    void execute_device(uint32_t partition, ArrowDeviceArrayStream* out) { check(dfd_repartition_exec_execute_device(h_, partition, out)); }

private:
    Partitioning partitioning_;
    dfd_repartition_exec* h_ = nullptr;
};

// One worker's endpoint of the NVLink exchange (≙ WorkerConnectionPool + the ExecuteTask server).
class ShuffleExchange {
public:
    static std::array<uint8_t, 128> unique_id() {
        std::array<uint8_t, 128> id{};
        check(dfd_nccl_unique_id(id.data()));
        return id;
    }
    ShuffleExchange(WorkerContext& ctx, int rank, int world, const void* nccl_id) : rank_(rank), world_(world) {
        check(dfd_exchange_create(ctx.get(), rank, world, nccl_id, &h_));
    }
    ~ShuffleExchange() { dfd_exchange_destroy(h_); }
    ShuffleExchange(const ShuffleExchange&) = delete;
    ShuffleExchange& operator=(const ShuffleExchange&) = delete;
    void setup_window(size_t bytes) { check(dfd_exchange_setup_window(h_, bytes)); }
    dfd_exchange* get() const { return h_; }
    int rank() const { return rank_; }
    int world() const { return world_; }

private:
    dfd_exchange* h_ = nullptr;
    int rank_, world_;
};

// Consumer side of the shuffle for device-resident columns.
class NetworkShuffleExec {
public:
    // network_shuffle.rs:115-157: input must be hash partitioned; the producer's RepartitionExec is
    // rescaled to Hash(keys, P * task_count) while this node keeps advertising Hash(keys, P).
    static NetworkShuffleExec try_new(const Partitioning& input, std::array<uint8_t, 16> query_id, size_t num, size_t task_count,
                                      size_t input_task_count) {
        if (input.key_cols.empty()) throw Error(DFD_ERR_INVALID_ARGUMENT, "NetworkShuffleExec input must be hash partitioned");
        NetworkShuffleExec n;
        n.properties_ = input;
        n.task_count_ = task_count;
        n.input_stage_.query_id = query_id;
        n.input_stage_.num = num;
        n.input_stage_.plan = scale_partitioning(input, [&](uint32_t p) { return p * (uint32_t)task_count; });
        n.input_stage_.tasks.assign(input_task_count, ExecutionTask{});
        return n;
    }
    const char* name() const { return "NetworkShuffleExec"; }
    const Partitioning& output_partitioning() const { return properties_; }
    const Stage& input_stage() const { return input_stage_; }

    // The collective: this worker contributes `in` as producer task `rank` and receives its P destinations.
    // FUSED mode fills `out` with pointers into the receive window; NCCL mode writes into caller buffers.
    void shuffle(WorkerContext& ctx, ShuffleExchange& x, const std::vector<dfd_column>& in, int64_t n_rows, std::vector<dfd_column>& out,
                 int mode = DFD_EXCHANGE_FUSED, int64_t out_capacity_rows = 0) {
        if ((size_t)x.world() != task_count_ || input_stage_.tasks.size() != task_count_)
            throw Error(DFD_ERR_INVALID_ARGUMENT, "one producer and one consumer task per GPU worker");
        if (!part_) part_ = std::make_unique<HashPartitioner>(ctx, input_stage_.plan);
        out.resize(in.size());
        starts_.assign(properties_.partition_count + 1, 0);
        check(dfd_shuffle_device(x.get(), part_->get(), mode, in.data(), (int)in.size(), n_rows, properties_.partition_count, out.data(),
                                 out_capacity_rows, starts_.data()));
    }
    // ≙ execute(partition, ctx): rows with hash % (P*T) == P*task_index + partition are rows [first, second)
    std::pair<int64_t, int64_t> execute(size_t partition, const DistributedTaskContext&) const {
        if (partition + 1 >= starts_.size()) throw Error(DFD_ERR_INVALID_ARGUMENT, "partition out of range (or shuffle() has not run)");
        return {starts_[partition], starts_[partition + 1]};
    }

private:
    Partitioning properties_;
    Stage input_stage_;
    size_t task_count_ = 1;
    std::unique_ptr<HashPartitioner> part_;
    std::vector<int64_t> starts_;
};

}  // namespace dfd
