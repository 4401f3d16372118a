//! Raw declarations of the entry points of `include/dfd_b200.h` this shim binds (host operator + plan-hook predicates).
//! The Arrow structs are arrow-rs' own `#[repr(C)]` mirrors of the Arrow C Data / C Stream interface
//! (`include/arrow_c_abi.h` is the same layout).
#![allow(non_camel_case_types)]

use std::ffi::{c_char, c_int, c_void};

use arrow::ffi::{FFI_ArrowArray, FFI_ArrowSchema};
use arrow::ffi_stream::FFI_ArrowArrayStream;

#[repr(C)]
pub struct dfd_ctx {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct dfd_repartition_exec {
    _opaque: [u8; 0],
}

/// `dfd_exec_options` (include/dfd_b200.h): zero = the library's default for every field.
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct dfd_exec_options {
    pub chunk_rows: i64,
    pub pipeline_depth: i32,
    pub pinned_pool_chunks: i32,
    pub max_pinned_chunks: i32,
    pub device_output: i32,
}

/// `dfd_exec_stats` (include/dfd_b200.h).
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct dfd_exec_stats {
    pub rows_in: u64,
    pub rows_out: u64,
    pub bytes_h2d: u64,
    pub bytes_d2h: u64,
    pub pinned_chunks: u64,
    pub pinned_chunks_allocated: u64,
    pub pinned_chunks_reused: u64,
    pub ns_push: u64,
    pub ns_wait_d2h: u64,
    pub ns_wait_pool: u64,
}

/// `struct ArrowDeviceArray` of the Arrow C Device Data Interface (`include/arrow_c_abi.h`): a record batch whose buffers
/// live on a GPU; `sync_event` is NULL or a `cudaEvent_t*`.
#[repr(C)]
pub struct ArrowDeviceArray {
    pub array: FFI_ArrowArray,
    pub device_id: i64,
    pub device_type: i32,
    pub sync_event: *mut c_void,
    pub reserved: [i64; 3],
}
pub const ARROW_DEVICE_CUDA: i32 = 2;

/// `struct ArrowDeviceArrayStream` of the Arrow C Device stream interface (`include/arrow_c_abi.h`).
#[repr(C)]
pub struct ArrowDeviceArrayStream {
    pub device_type: i32,
    pub get_schema: Option<unsafe extern "C" fn(*mut ArrowDeviceArrayStream, *mut FFI_ArrowSchema) -> c_int>,
    pub get_next: Option<unsafe extern "C" fn(*mut ArrowDeviceArrayStream, *mut ArrowDeviceArray) -> c_int>,
    pub get_last_error: Option<unsafe extern "C" fn(*mut ArrowDeviceArrayStream) -> *const c_char>,
    pub release: Option<unsafe extern "C" fn(*mut ArrowDeviceArrayStream)>,
    pub private_data: *mut c_void,
}

// dfd_status (include/dfd_b200.h)
pub const DFD_OK: c_int = 0;
pub const DFD_ERR_INVALID_ARGUMENT: c_int = 1;
pub const DFD_ERR_OOM: c_int = 2;
pub const DFD_ERR_CUDA: c_int = 3;
pub const DFD_ERR_NCCL: c_int = 4;
pub const DFD_ERR_INTERNAL: c_int = 5;
pub const DFD_ERR_UNSUPPORTED: c_int = 6;
pub const DFD_ERR_CAPACITY: c_int = 7;

extern "C" {
    pub fn dfd_last_error() -> *const c_char;
    pub fn dfd_ctx_create(device: c_int, out: *mut *mut dfd_ctx) -> c_int;
    pub fn dfd_ctx_destroy(ctx: *mut dfd_ctx);
    /// Pure host predicate (no GPU touched): can the GPU operator move every column of this record-batch schema?
    pub fn dfd_schema_supported(schema: *const FFI_ArrowSchema) -> c_int;
    /// The same with the hash key columns taken into account (lists / LargeBinary / FixedSizeBinary move as payload only).
    pub fn dfd_repartition_supported(schema: *const FFI_ArrowSchema, key_cols: *const i32, n_keys: c_int) -> c_int;
    /// `RepartitionExec::try_new(input, Partitioning::Hash(cols, n))` (network_shuffle.rs:126-134)
    pub fn dfd_repartition_exec_create(
        ctx: *mut dfd_ctx,
        schema: *const FFI_ArrowSchema,
        key_cols: *const i32,
        n_keys: c_int,
        num_partitions: u32,
        opts: *const dfd_exec_options,
        out: *mut *mut dfd_repartition_exec,
    ) -> c_int;
    /// One input `RecordBatch`; ownership of `*batch` moves to the operator (its `release` is cleared). Single producer.
    pub fn dfd_repartition_exec_push(x: *mut dfd_repartition_exec, batch: *mut FFI_ArrowArray) -> c_int;
    /// One GPU-resident input batch (same device as the context); ownership of `batch.array` moves to the operator. An
    /// operator takes either host batches (`push`) or device batches, decided by the first non-empty push.
    pub fn dfd_repartition_exec_push_device(x: *mut dfd_repartition_exec, batch: *mut ArrowDeviceArray) -> c_int;
    pub fn dfd_repartition_exec_finish(x: *mut dfd_repartition_exec) -> c_int;
    /// The input failed: every partition stream ends with EIO + `message` (RepartitionExec forwards input errors likewise).
    pub fn dfd_repartition_exec_abort(x: *mut dfd_repartition_exec, message: *const c_char) -> c_int;
    /// `plan.execute(partition, ctx)` (impl_execute_task.rs:77-86): a blocking Arrow C stream of that destination's batches.
    pub fn dfd_repartition_exec_execute(x: *mut dfd_repartition_exec, partition: u32, out: *mut FFI_ArrowArrayStream) -> c_int;
    /// The same for an operator created with `device_output = 1`: a blocking Arrow C Device stream of GPU-resident batches,
    /// each with a `sync_event` the consumer's stream waits on; a batch is released after the consumer's device reads.
    pub fn dfd_repartition_exec_execute_device(x: *mut dfd_repartition_exec, partition: u32, out: *mut ArrowDeviceArrayStream) -> c_int;
    /// Pulls a stream of GPU-resident batches to exhaustion (through `push_device`), then finishes; releases the stream once.
    pub fn dfd_repartition_exec_run_device(x: *mut dfd_repartition_exec, input: *mut ArrowDeviceArrayStream) -> c_int;
    pub fn dfd_repartition_exec_stats(x: *mut dfd_repartition_exec, out: *mut dfd_exec_stats) -> c_int;
    pub fn dfd_repartition_exec_destroy(x: *mut dfd_repartition_exec);
}
