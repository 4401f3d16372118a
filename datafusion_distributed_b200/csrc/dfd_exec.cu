// dfd_exec.cu — host-side operator: RepartitionExec(Hash) with HOST Arrow batches.
//
// Mirrors the producer half of the reference's shuffle as an operator:
//   RepartitionExec::try_new(input, Partitioning::Hash(exprs, P * task_count))
//     (src/execution_plans/network_shuffle.rs:126-134)
//   plan.execute(partition, ctx) -> SendableRecordBatchStream
//     (src/worker/impl_execute_task.rs:77-86)
// over the Arrow C Data / C Stream interfaces.  Input batches are copied to the
// GPU in chunks (H2D stream), partitioned by K1/K1b/K2 (compute stream), copied
// back into pooled pinned memory (D2H stream) and handed out as zero-copy
// per-destination slices — the three stages of consecutive chunks overlap, so
// end-to-end time approaches max(H2D, D2H) over PCIe.
#include <cuda_runtime.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "dfd_b200.h"
#include "dfd_host_staging.h"
#include "dfd_internal.h"

using namespace dfd;

namespace {

struct FieldInfo {
    std::string name, format;
    int64_t flags = 0;
    int32_t kind = DFD_COL_FIXED;   // layout the DEVICE sees (a Utf8View column is Utf8 there; a dictionary column is its indices)
    int32_t width = 0;
    bool view = false;             // Arrow Utf8View / BinaryView ("vu" / "vz"): converted to offsets + bytes on input, back to views on output
    // List<Utf8 / Binary> payload: the visible field is a PLACEHOLDER without a device column of its own; its rows travel as
    // three hidden Binary device columns appended after the visible fields (all scattered by the same K2/K4 passes):
    //   h_len   row -> the int32 LENGTHS of its child elements (4 bytes per element); carries the list's validity bitmap
    //   h_bytes row -> the bytes of its child strings (contiguous per row)
    //   h_valid row -> one byte per child element (its validity), only when the child field is nullable
    // After the scatter the child offsets are an exclusive scan of the gathered lengths and the child validity is re-packed.
    bool list = false, hidden = false;
    int h_len = -1, h_bytes = -1, h_valid = -1;
    int owner = -1, role = 0;  // hidden columns: the list field they belong to; role 1 = lengths, 2 = bytes, 3 = element validity
    std::string child_name, child_format;
    int64_t child_flags = 0;
    int32_t child_width = 0;       // list child: 0 = Utf8 / Binary (offsets + bytes), > 0 = fixed-width primitive of that many bytes
    bool nodev() const { return list; }
    bool dict = false;             // dictionary-encoded: `format` is the index type, dict_* describe the values
    bool dict_index_unsigned = false;  // UInt8/16/32/64 indices ("C" "S" "I" "L")
    std::string dict_format;
    int64_t dict_flags = 0;
    int32_t dict_kind = DFD_COL_FIXED, dict_width = 0;
    bool var() const { return kind == DFD_COL_UTF8 || kind == DFD_COL_LARGE_UTF8 || kind == DFD_COL_BINARY; }
    size_t ow() const { return kind == DFD_COL_LARGE_UTF8 ? 8 : 4; }  // offset width of var-width kinds
};

// LargeBinary and FixedSizeBinary values are hashed by DataFusion as byte slices with a length prefix; the device hashes a
// LARGE_UTF8 column as strings and a FIXED column as an integer: such columns travel as payload but cannot be hash keys.
bool hashable_format(const char* f) { return f[0] != 'Z' && f[0] != 'w'; }

// Interval(DayTime) / Interval(MonthDayNano) values hash field by field (arrow's derived Hash), as keys and as the values of
// a dictionary key alike; everything else is one integer / byte-slice write.
int32_t interval_key_mode(const std::string& f) {
    return f == "tiD" ? DFD_KEY_HASH_INTERVAL_DAY_TIME : f == "tin" ? DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO : DFD_KEY_HASH_PLAIN;
}

// Arrow format string -> physical layout (Arrow C data interface, "Data type description")
bool parse_format(const char* f, int32_t* kind, int32_t* width) {
    *kind = DFD_COL_FIXED;
    switch (f[0]) {
        case 'b': *kind = DFD_COL_BOOL; *width = 0; return f[1] == 0;
        case 'c': case 'C': *width = 1; return f[1] == 0;
        case 's': case 'S': *width = 2; return f[1] == 0;
        case 'e': *width = 2; return f[1] == 0;
        case 'i': case 'I': case 'f': *width = 4; return f[1] == 0;
        case 'l': case 'L': case 'g': *width = 8; return f[1] == 0;
        case 'u': *kind = DFD_COL_UTF8; *width = 0; return f[1] == 0;
        case 'U': *kind = DFD_COL_LARGE_UTF8; *width = 0; return f[1] == 0;
        case 'z': *kind = DFD_COL_BINARY; *width = 0; return f[1] == 0;
        case 'Z': *kind = DFD_COL_LARGE_UTF8; *width = 0; return f[1] == 0;  // LargeBinary MOVES like LargeUtf8 (int64 offsets + bytes); payload only
        case 'w': {  // FixedSizeBinary(N), N in {1, 2, 4, 8, 16} (e.g. 16-byte UUIDs): N-byte values; payload only
            int nb = 0;
            if (sscanf(f, "w:%d", &nb) != 1 || (nb != 1 && nb != 2 && nb != 4 && nb != 8 && nb != 16)) return false;
            *width = nb;
            return true;
        }
        case 'v':  // Utf8View / BinaryView: 16-byte views + variadic data buffers; hashed over the string bytes exactly like Utf8 / Binary
            if (f[1] == 'u' && f[2] == 0) { *kind = DFD_COL_UTF8; *width = 0; return true; }
            if (f[1] == 'z' && f[2] == 0) { *kind = DFD_COL_BINARY; *width = 0; return true; }
            return false;
        case 'd': {  // d:precision,scale[,bitwidth]
            int p = 0, s = 0, bw = 128;
            int n = sscanf(f, "d:%d,%d,%d", &p, &s, &bw);
            if (n < 2) return false;
            if (bw != 128 && bw != 64 && bw != 32) return false;
            *width = bw / 8;
            return true;
        }
        case 't':
            if (f[1] == 'd') { *width = f[2] == 'D' ? 4 : 8; return f[2] == 'D' || f[2] == 'm'; }  // date32/date64
            if (f[1] == 't') { *width = (f[2] == 's' || f[2] == 'm') ? 4 : 8; return true; }    // time32/time64
            if (f[1] == 's' || f[1] == 'D') { *width = 8; return true; }                           // timestamp / duration
            if (f[1] == 'i') { *width = f[2] == 'M' ? 4 : (f[2] == 'D' ? 8 : 16); return true; }   // intervals
            return false;
    }
    return false;
}

struct PinnedPool;

// An input record batch shared by everything that still points into it: in-flight H2D copies and, for dictionary
// columns, the dictionaries of the output batches (which travel by reference).  Released when the last user lets go.
struct SharedInput {
    ArrowArray array;
    explicit SharedInput(const ArrowArray& a) : array(a) {}
    ~SharedInput() {
        if (array.release) array.release(&array);
    }
};

// One D2H landing buffer (pinned): all columns of one chunk, destination-sorted.
struct OutChunk {
    std::vector<void*> views;        // per column: 16-byte views of a Utf8View / BinaryView column (host, built at emission)
    std::vector<int64_t> view_sizes; // per column: the "variadic buffer sizes" buffer of such an array (one data buffer)
    std::vector<std::shared_ptr<SharedInput>> inputs;  // input batches whose dictionaries this chunk's batches reference
    std::vector<void*> values;    // per column: values (fixed / bool) or string bytes (var-width, grown on demand)
    std::vector<void*> validity;  // per column (may be null)
    std::vector<void*> offsets;   // per column (var-width only)
    std::vector<size_t> data_cap; // per column: capacity of `values` for var-width columns
    std::atomic<int> refs{0};
    std::shared_ptr<PinnedPool> pool;
};

void destroy_out_chunk(OutChunk* c) {
    for (void* p : c->values)
        if (p) cudaFreeHost(p);
    for (void* p : c->validity)
        if (p) cudaFreeHost(p);
    for (void* p : c->offsets)
        if (p) cudaFreeHost(p);
    for (void* p : c->views) free(p);
    delete c;
}

// Pinned output chunks of FINISHED operators, kept by the worker context for the next operator with the same column
// layout and chunk size.  Pinning memory is slow (cudaHostAlloc of a 64 MiB chunk costs milliseconds — as long as
// moving several chunks over PCIe), and a worker runs the same stage shapes again and again: the reference's workers
// get the same effect from their caching allocator (mimalloc, benchmarks/cdk/bin/worker.rs:32).  Bounded by bytes
// (DFD_PINNED_CACHE_BYTES, default 4 GiB); freed with the context.
struct PinnedCache {
    struct Entry {
        std::string layout;
        int64_t chunk_rows;
        OutChunk* chunk;
        size_t bytes;
    };
    std::mutex mu;
    std::vector<Entry> entries;
    size_t bytes = 0, max_bytes = (size_t)4 << 30;
    int device = 0;
    PinnedCache() {
        if (const char* e = getenv("DFD_PINNED_CACHE_BYTES")) max_bytes = (size_t)strtoull(e, nullptr, 10);
    }
    OutChunk* take(const std::string& layout, int64_t chunk_rows) {
        std::lock_guard<std::mutex> lk(mu);
        for (size_t i = entries.size(); i-- > 0;)
            if (entries[i].chunk_rows == chunk_rows && entries[i].layout == layout) {
                OutChunk* c = entries[i].chunk;
                bytes -= entries[i].bytes;
                entries.erase(entries.begin() + (long)i);
                return c;
            }
        return nullptr;
    }
    bool put(const std::string& layout, int64_t chunk_rows, OutChunk* c, size_t nbytes) {  // false: over budget, caller frees
        std::lock_guard<std::mutex> lk(mu);
        if (bytes + nbytes > max_bytes) return false;
        entries.push_back(Entry{layout, chunk_rows, c, nbytes});
        bytes += nbytes;
        return true;
    }
    ~PinnedCache() {
        cudaSetDevice(device);
        for (Entry& e : entries) destroy_out_chunk(e.chunk);
    }
};

std::shared_ptr<PinnedCache> pinned_cache_of(dfd_ctx* ctx) {  // caller holds no lock; the slot is written once under ctx->mu
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!ctx->pinned_cache) {
        auto pc = std::make_shared<PinnedCache>();
        pc->device = ctx->device;
        ctx->pinned_cache = pc;
    }
    return std::static_pointer_cast<PinnedCache>(ctx->pinned_cache);
}

struct PinnedPool : std::enable_shared_from_this<PinnedPool> {
    int device = 0;
    int64_t chunk_rows = 0;
    std::vector<FieldInfo> fields;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<OutChunk*> free_list;
    std::vector<OutChunk*> all;
    size_t max_chunks = 0;  // 0 = unbounded; otherwise acquire() blocks until a consumer returns a chunk (back-pressure)
    std::weak_ptr<PinnedCache> cache;  // the worker context's cache (gone once the context is destroyed)
    std::string layout;                // what makes two pools' chunks interchangeable: per field kind / width / nullable / view
    std::atomic<uint64_t> n_allocated{0}, n_reused{0};  // chunks pinned by this pool / taken over from the context's cache

    static size_t value_bytes(const FieldInfo& f, int64_t rows) {
        if (f.var()) return 0;  // string bytes are sized per chunk
        return f.kind == DFD_COL_BOOL ? (size_t)((rows + 63) / 64 * 8 + 8) : (size_t)rows * (size_t)f.width;
    }
    static size_t bitmap_bytes(int64_t rows) { return (size_t)((rows + 63) / 64 * 8 + 8); }

    void set_fields(const std::vector<FieldInfo>& fs) {
        fields = fs;
        layout.clear();
        for (const FieldInfo& f : fields) {
            char b[64];
            snprintf(b, sizeof b, "%d:%d:%d:%d:%d;", (int)f.kind, (int)f.width, (int)((f.flags & ARROW_FLAG_NULLABLE) != 0), (int)f.view, (int)f.nodev());
            layout += b;
        }
    }
    size_t chunk_bytes(const OutChunk* c) const {  // pinned bytes one chunk holds right now
        size_t n = 0;
        for (size_t i = 0; i < fields.size(); ++i) {
            const FieldInfo& f = fields[i];
            if (f.nodev()) continue;
            n += f.var() ? c->data_cap[i] + (size_t)(chunk_rows + 16) * f.ow() : value_bytes(f, chunk_rows);
            if (f.flags & ARROW_FLAG_NULLABLE) n += bitmap_bytes(chunk_rows);
        }
        return n;
    }

    // A pooled pinned chunk.  With a bound (`max_chunks`), the producer BLOCKS here until a consumer has released a chunk:
    // that is the operator's back-pressure (the reference bounds the same hand-off with its byte budget,
    // src/worker/worker_connection_pool.rs:151-153, 251-257).
    OutChunk* acquire() {
        {
            std::unique_lock<std::mutex> lk(mu);
            if (max_chunks && free_list.empty() && all.size() >= max_chunks) cv.wait(lk, [&] { return !free_list.empty(); });
            if (!free_list.empty()) {
                OutChunk* c = free_list.back();
                free_list.pop_back();
                return c;
            }
        }
        if (std::shared_ptr<PinnedCache> pc = cache.lock())
            if (OutChunk* c = pc->take(layout, chunk_rows)) {  // a chunk a finished operator of the same shape left behind
                c->refs.store(0);
                c->inputs.clear();
                n_reused.fetch_add(1);
                std::lock_guard<std::mutex> lk(mu);
                all.push_back(c);
                return c;
            }
        OutChunk* c = new (std::nothrow) OutChunk();
        if (!c) return nullptr;
        cudaSetDevice(device);
        for (const FieldInfo& f : fields) {
            void* v = nullptr;
            void* b = nullptr;
            void* o = nullptr;
            bool ok = true;
            if (f.nodev()) {  // list placeholder: no buffers of its own
                c->values.push_back(nullptr); c->validity.push_back(nullptr); c->offsets.push_back(nullptr); c->data_cap.push_back(0);
                c->views.push_back(nullptr); c->view_sizes.push_back(0);
                continue;
            }
            if (!f.var() && cudaHostAlloc(&v, value_bytes(f, chunk_rows), cudaHostAllocPortable) != cudaSuccess) ok = false;
            if (ok && (f.flags & ARROW_FLAG_NULLABLE) && cudaHostAlloc(&b, bitmap_bytes(chunk_rows), cudaHostAllocPortable) != cudaSuccess) ok = false;
            if (ok && f.var() && cudaHostAlloc(&o, (size_t)(chunk_rows + 16) * f.ow(), cudaHostAllocPortable) != cudaSuccess) ok = false;
            if (!ok) {  // free what this chunk already holds: nothing leaks on a failed allocation
                if (v) cudaFreeHost(v);
                if (b) cudaFreeHost(b);
                if (o) cudaFreeHost(o);
                destroy_out_chunk(c);
                return nullptr;
            }
            c->values.push_back(v);
            c->validity.push_back(b);
            c->offsets.push_back(o);
            c->data_cap.push_back(0);
            c->views.push_back(f.view ? malloc((size_t)(chunk_rows + 16) * 16) : nullptr);
            c->view_sizes.push_back(0);
        }
        n_allocated.fetch_add(1);
        std::lock_guard<std::mutex> lk(mu);
        all.push_back(c);
        return c;
    }
    void give_back(OutChunk* c) {
        c->inputs.clear();  // (drops the references to the input batches whose dictionaries were handed out)
        {
            std::lock_guard<std::mutex> lk(mu);
            free_list.push_back(c);
        }
        cv.notify_one();
    }
    // The pool dies with its operator and the last output batch: its chunks go to the context's cache (if the context is
    // still there and the cache has room), otherwise the memory is unpinned.
    ~PinnedPool() {
        std::shared_ptr<PinnedCache> pc = cache.lock();
        cudaSetDevice(device);
        for (OutChunk* c : all) {
            c->inputs.clear();
            if (!pc || !pc->put(layout, chunk_rows, c, chunk_bytes(c))) destroy_out_chunk(c);
        }
    }
};

void chunk_unref(OutChunk* c) {
    if (c->refs.fetch_sub(1) == 1) {
        std::shared_ptr<PinnedPool> pool = std::move(c->pool);  // keep the pool alive past give_back
        pool->give_back(c);
    }
}

// ---- Arrow C Data export of one destination's slice of a chunk -------------
struct BatchPriv {
    OutChunk* chunk;
    std::vector<ArrowArray> children;
    std::vector<ArrowArray*> child_ptrs;
    std::vector<const void*> child_bufs;  // 4 per child (validity, values|offsets|views, string bytes, variadic sizes)
    std::vector<ArrowArray> grand;        // per child: the values array of a list column (child of the child)
    std::vector<ArrowArray*> grand_ptrs;
    std::vector<const void*> grand_bufs;  // 3 per child (validity, offsets, bytes of the list's values array)
    std::vector<ArrowArray> dicts;        // per child: shallow copy of the input dictionary (dictionary columns)
    std::vector<std::shared_ptr<SharedInput>> dict_owner;  // keeps that dictionary's batch alive
    const void* struct_bufs[1] = {nullptr};
};

void dict_release(ArrowArray* a) { a->release = nullptr; }  // (the buffers belong to the SharedInput held by the batch)

void child_release(ArrowArray* a) { a->release = nullptr; }

void batch_release(ArrowArray* a) {
    BatchPriv* p = (BatchPriv*)a->private_data;
    for (ArrowArray& c : p->children) {
        if (c.dictionary && c.dictionary->release) c.dictionary->release(c.dictionary);
        if (c.release) c.release(&c);
    }
    chunk_unref(p->chunk);
    delete p;
    a->release = nullptr;
}

struct SchemaPriv {
    std::vector<FieldInfo> fields;
    std::vector<ArrowSchema> children;
    std::vector<ArrowSchema*> child_ptrs;
    std::vector<ArrowSchema> dicts;  // per child: schema of the dictionary values (dictionary columns)
    std::vector<ArrowSchema> items;  // per child: the item field of a list column
    std::vector<ArrowSchema*> item_ptrs;
};

void schema_child_release(ArrowSchema* s) { s->release = nullptr; }
void schema_release(ArrowSchema* s) {
    SchemaPriv* p = (SchemaPriv*)s->private_data;
    for (ArrowSchema& c : p->children)
        if (c.release) c.release(&c);
    delete p;
    s->release = nullptr;
}

int export_schema(const std::vector<FieldInfo>& fields, ArrowSchema* out) {
    SchemaPriv* p = new (std::nothrow) SchemaPriv();
    if (!p) return ENOMEM;
    for (const FieldInfo& f : fields)
        if (!f.hidden) p->fields.push_back(f);  // (hidden list columns are an implementation detail)
    const size_t nf = p->fields.size();
    p->children.resize(nf);
    p->child_ptrs.resize(nf);
    p->dicts.resize(nf);
    p->items.resize(nf);
    p->item_ptrs.resize(nf);
    for (size_t i = 0; i < nf; ++i) {
        ArrowSchema& c = p->children[i];
        memset(&c, 0, sizeof c);
        c.format = p->fields[i].format.c_str();
        c.name = p->fields[i].name.c_str();
        c.flags = p->fields[i].flags;
        c.release = schema_child_release;
        if (p->fields[i].list) {
            ArrowSchema& it = p->items[i];
            memset(&it, 0, sizeof it);
            it.format = p->fields[i].child_format.c_str();
            it.name = p->fields[i].child_name.c_str();
            it.flags = p->fields[i].child_flags;
            it.release = schema_child_release;
            p->item_ptrs[i] = &it;
            c.n_children = 1;
            c.children = &p->item_ptrs[i];
        }
        if (p->fields[i].dict) {
            ArrowSchema& d = p->dicts[i];
            memset(&d, 0, sizeof d);
            d.format = p->fields[i].dict_format.c_str();
            d.name = "";
            d.flags = p->fields[i].dict_flags;
            d.release = schema_child_release;
            c.dictionary = &d;
        }
        p->child_ptrs[i] = &c;
    }
    memset(out, 0, sizeof *out);
    out->format = "+s";
    out->name = "";
    out->n_children = (int64_t)nf;
    out->children = p->child_ptrs.data();
    out->release = schema_release;
    out->private_data = p;
    return 0;
}

struct PartQueue {
    std::deque<ArrowArray> batches;
};

using HeldInput = std::shared_ptr<SharedInput>;  // an input batch whose buffers an in-flight H2D still reads

struct VarPrep {  // rows of one variable-width device column as they will be staged: n + 1 source offsets (the first being
    const char* off = nullptr;   // `first`) and the bytes they span
    int64_t first = 0;
    const char* bytes = nullptr;
    int64_t nbytes = 0;
};

struct DictId {  // identity of a dictionary: values buffer, offset, length
    const void* p = nullptr;
    int64_t offset = 0, length = 0;
    bool operator==(const DictId& o) const { return p == o.p && offset == o.offset && length == o.length; }
};

struct Slot {
    std::vector<void*> d_in, d_in_valid, d_out, d_out_valid;  // per column device buffers
    std::vector<void*> d_in_off, d_out_off;                   // var-width: offsets buffers
    std::vector<size_t> in_cap, out_cap;                      // var-width: capacity of d_in / d_out (string bytes)
    std::vector<int64_t> first_off, data_bytes;               // var-width: first input offset / byte count of the chunk
    std::vector<uint8_t*> h_valid, h_bool;                    // pinned, allocated on first use: the chunk's validity / boolean bitmaps,
                                                              //   concatenated on the host at bit granularity (bit r = row r of the chunk)
    std::vector<char*> h_off;                                 // pinned: the chunk's var-width offsets, re-based onto the chunk's byte buffer
    std::vector<DictId> dict_id;                              // dictionary columns: identity of the chunk's dictionary
    std::vector<dfd::Scratch> list_tmp;                       // list fields: [child offsets | child validity bits | scan block sums] (device)
    std::vector<dfd::Scratch> dict_buf;                       // dictionary KEY columns: [hashes | offsets | data | validity] of the values
    std::vector<const uint64_t*> dict_hashes;                 //   device pointers handed to the partitioner for this chunk
    std::vector<const uint8_t*> dict_valid;
    int64_t* h_part_starts = nullptr;                        // pinned [N+1]
    cudaEvent_t e_h2d = nullptr, e_k = nullptr, e_d2h = nullptr;
    bool k_recorded = false, d2h_recorded = false;
    // state of the chunk currently in this slot
    int64_t rows = 0;
    std::vector<bool> has_valid;
    OutChunk* out = nullptr;
    bool in_flight = false;
    std::vector<HeldInput> held;
    std::vector<HeldInput> dict_held;  // device input: host copies of the dictionaries of the batches in `held` (what the output references)
};

enum InputMode { INPUT_UNSET = 0, INPUT_HOST = 1, INPUT_DEVICE = 2 };

}  // namespace

struct dfd_repartition_exec {
    dfd_ctx* ctx = nullptr;
    dfd_partitioner* part = nullptr;
    std::vector<FieldInfo> fields;
    std::vector<int> key_of_field;  // index into the partitioner's key list, or -1
    size_t n_visible = 0;           // fields [0, n_visible) are the schema's columns; the rest are hidden device columns (lists)
    std::vector<int> dev_fields;    // fields that own a device column, in launch order; dev_pos[field] = its position there
    std::vector<int> dev_pos;
    uint32_t N = 0;
    int64_t chunk_rows = 0;
    int depth = 3;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    std::vector<Slot> slots;
    int cur = 0;              // slot being filled
    bool cur_open = false;
    std::shared_ptr<PinnedPool> pool;
    // output side
    std::mutex mu;
    std::condition_variable cv;
    std::vector<PartQueue> queues;
    bool finished = false;
    int error_code = 0;
    std::string error;
    // counters: written by the producer thread, read by dfd_repartition_exec_stats from any thread (relaxed atomics)
    std::atomic<uint64_t> rows_in{0}, bytes_h2d{0}, bytes_d2h{0};
    uint64_t rows_out = 0;  // (under `mu`)
    std::atomic<uint64_t> ns_push{0}, ns_wait_d2h{0}, ns_wait_pool{0};  // producer-thread time: inside push/finish; of which blocked on a D2H / on the pinned pool
    // host scratch of the batch being staged (pageable: an H2D from it has been staged by the time cudaMemcpyAsync returns)
    std::vector<std::vector<char>> tmp_off, tmp_bytes;
    std::vector<VarPrep> prep;
    // device input (push_device): the first non-empty push decides whether the operator takes host or device batches
    int input_mode = INPUT_UNSET;
    dfd::Scratch d_sizes;                  // k_stage_sizes results, 4 x int64 per var-width column
    int64_t* h_sizes = nullptr;            // pinned: their read-back
    cudaEvent_t e_sizes = nullptr;
    std::vector<dfd::Scratch> view_tmp;    // view fields: [lengths | offsets | scan block sums | data buffer table] (device)
    std::vector<std::vector<int64_t>> dsz; // per visible field: the read-back sizes of the rows being staged
};

namespace {

struct ScopedNs {  // adds the scope's wall time to a counter
    std::atomic<uint64_t>& acc;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    explicit ScopedNs(std::atomic<uint64_t>& a) : acc(a) {}
    ~ScopedNs() { acc += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(); }
};

int fail(dfd_repartition_exec* x, int code, const std::string& msg) {
    {
        std::lock_guard<std::mutex> lk(x->mu);
        if (!x->error_code) {
            x->error_code = code;
            x->error = msg;
        }
        x->finished = true;
    }
    x->cv.notify_all();
    return set_error(code, "%s", msg.c_str());
}

#define XCUDA(x, call, what)                                                           \
    {                                                                                  \
        cudaError_t _e = (call);                                                       \
        if (_e != cudaSuccess) return fail((x), DFD_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(_e)); \
    }

// hand the finished chunk in `s` to the per-destination queues
int emit_slot(dfd_repartition_exec* x, Slot& s) {
    if (!s.in_flight) return DFD_OK;
    {
        const auto t0 = std::chrono::steady_clock::now();
        XCUDA(x, cudaEventSynchronize(s.e_d2h), "D2H");
        x->ns_wait_d2h += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    }
    OutChunk* oc = s.out;
    for (const FieldInfo& f : x->fields)  // the output batches reference the inputs' dictionaries (device input: their host copies)
        if (f.dict) { oc->inputs = x->input_mode == INPUT_DEVICE ? s.dict_held : s.held; break; }
    s.held.clear();
    s.dict_held.clear();
    s.out = nullptr;
    s.in_flight = false;
    const size_t C = x->n_visible;  // the output batches carry the schema's columns; hidden list columns are folded into their list
    int made = 0;
    for (size_t c = 0; c < C; ++c) {
        if (!x->fields[c].list) continue;
        int32_t* lo32 = (int32_t*)oc->offsets[(size_t)x->fields[c].h_len];  // byte offsets into the 4-byte lengths -> element offsets
        for (int64_t r = 0; r <= s.rows; ++r) lo32[r] >>= 2;
    }
    for (size_t c = 0; c < C; ++c) {
        if (!x->fields[c].view) continue;
        // Utf8View output: 16-byte views over the chunk's single data buffer (inline when <= 12 bytes)
        const int32_t* off = (const int32_t*)oc->offsets[c];
        const int64_t rows = s.rows;
        dfd::host::build_views(off, (const uint8_t*)oc->values[c], rows, (uint8_t*)oc->views[c]);
        oc->view_sizes[c] = off[rows];
    }
    oc->refs.store(1);  // guard while slicing
    oc->pool = x->pool;
    for (uint32_t p = 0; p < x->N; ++p) {
        int64_t start = s.h_part_starts[p], cnt = s.h_part_starts[p + 1] - start;
        if (cnt <= 0) continue;  // like the reference, only non-empty partitions are emitted
        BatchPriv* bp = new (std::nothrow) BatchPriv();
        if (!bp) return fail(x, DFD_ERR_OOM, "out of host memory");
        bp->chunk = oc;
        bp->children.resize(C);
        bp->child_ptrs.resize(C);
        bp->child_bufs.resize(4 * C);
        bp->dicts.resize(C);
        bp->grand.resize(C);
        bp->grand_ptrs.resize(C);
        bp->grand_bufs.resize(3 * C);
        for (size_t c = 0; c < C; ++c) {
            ArrowArray& a = bp->children[c];
            memset(&a, 0, sizeof a);
            bool hv = s.has_valid[c];
            const FieldInfo& f = x->fields[c];
            if (f.list) {
                // List<Utf8>: list offsets + validity from the lengths column, values array (offsets from the device scan, bytes, validity)
                const size_t hl = (size_t)f.h_len, hb = (size_t)f.h_bytes;
                const bool lv = s.has_valid[hl];
                bp->child_bufs[4 * c] = lv ? oc->validity[hl] : nullptr;
                bp->child_bufs[4 * c + 1] = oc->offsets[hl];
                ArrowArray& g = bp->grand[c];
                memset(&g, 0, sizeof g);
                bp->grand_bufs[3 * c] = f.h_valid >= 0 ? oc->values[(size_t)f.h_valid] : nullptr;
                bp->grand_bufs[3 * c + 1] = f.child_width > 0 ? oc->values[hb] : oc->values[hl];  // primitive child: [validity, values]
                bp->grand_bufs[3 * c + 2] = oc->values[hb];
                g.length = s.data_bytes[hl] / 4;
                g.null_count = f.h_valid >= 0 ? -1 : 0;
                g.n_buffers = f.child_width > 0 ? 2 : 3;
                g.buffers = &bp->grand_bufs[3 * c];
                g.release = child_release;
                bp->grand_ptrs[c] = &g;
                a.length = cnt;
                a.offset = start;
                a.null_count = lv ? -1 : 0;
                a.n_buffers = 2;
                a.buffers = &bp->child_bufs[4 * c];
                a.n_children = 1;
                a.children = &bp->grand_ptrs[c];
                a.release = child_release;
                bp->child_ptrs[c] = &a;
                continue;
            }
            const bool var = f.var();
            bp->child_bufs[4 * c] = hv ? oc->validity[c] : nullptr;
            bp->child_bufs[4 * c + 1] = f.view ? oc->views[c] : (var ? oc->offsets[c] : oc->values[c]);
            bp->child_bufs[4 * c + 2] = var ? oc->values[c] : nullptr;
            bp->child_bufs[4 * c + 3] = f.view ? (const void*)&oc->view_sizes[c] : nullptr;
            a.length = cnt;
            a.offset = start;  // zero-copy slice of the chunk-wide destination-sorted buffer
            a.null_count = hv ? -1 : 0;
            a.n_buffers = f.view ? 4 : (var ? 3 : 2);  // view arrays: validity, views, one data buffer, variadic buffer sizes
            a.buffers = &bp->child_bufs[4 * c];
            a.release = child_release;
            if (f.dict && !oc->inputs.empty()) {
                // the dictionary travels by reference: a shallow copy of the input batch's dictionary, kept alive by the shared input
                const ArrowArray* src = oc->inputs.back()->array.children[c]->dictionary;
                bp->dicts[c] = *src;
                bp->dicts[c].release = dict_release;
                bp->dicts[c].private_data = nullptr;
                bp->dict_owner.push_back(oc->inputs.back());
                a.dictionary = &bp->dicts[c];
            }
            bp->child_ptrs[c] = &a;
        }
        ArrowArray top;
        memset(&top, 0, sizeof top);
        top.length = cnt;
        top.null_count = 0;
        top.n_buffers = 1;
        top.buffers = bp->struct_bufs;
        top.n_children = (int64_t)C;
        top.children = bp->child_ptrs.data();
        top.release = batch_release;
        top.private_data = bp;
        oc->refs.fetch_add(1);
        ++made;
        {
            std::lock_guard<std::mutex> lk(x->mu);
            x->queues[p].batches.push_back(top);
            x->rows_out += (uint64_t)cnt;
        }
    }
    chunk_unref(oc);  // drop the guard (returns the chunk to the pool if nothing was emitted)
    (void)made;
    x->cv.notify_all();
    return DFD_OK;
}

// run the kernels + D2H for the chunk accumulated in the current slot
int flush_current(dfd_repartition_exec* x) {
    if (!x->cur_open) return DFD_OK;
    Slot& s = x->slots[x->cur];
    dfd_ctx* c = x->ctx;
    const size_t C = x->fields.size();
    x->cur_open = false;
    if (s.rows == 0) return DFD_OK;
    // the pinned landing buffer of this chunk FIRST, before the context lock is taken: with max_pinned_chunks this is where
    // the producer waits for a consumer to release a chunk (back-pressure), and other operators of the same worker context
    // must keep running meanwhile
    {
        const auto t0 = std::chrono::steady_clock::now();
        s.out = x->pool->acquire();
        x->ns_wait_pool += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    }
    if (!s.out) return fail(x, DFD_ERR_OOM, "pinned host allocation failed");
    std::lock_guard<std::mutex> lk(c->mu);
    XCUDA(x, cudaSetDevice(c->device), "cudaSetDevice");
    for (int fi : x->dev_fields) {  // the buffers concatenated on the host while staging: bitmaps and re-based offsets
        if (x->input_mode == INPUT_DEVICE) break;  // (device input: k_stage_batch built them in place)
        const size_t i = (size_t)fi;
        const FieldInfo& f = x->fields[i];
        const size_t bm = (size_t)((s.rows + 7) / 8);
        if (s.has_valid[i]) {
            XCUDA(x, cudaMemcpyAsync(s.d_in_valid[i], s.h_valid[i], bm, cudaMemcpyHostToDevice, x->s_h2d), "H2D validity");
            x->bytes_h2d += bm;
        }
        if (f.kind == DFD_COL_BOOL) {
            XCUDA(x, cudaMemcpyAsync(s.d_in[i], s.h_bool[i], bm, cudaMemcpyHostToDevice, x->s_h2d), "H2D boolean values");
            x->bytes_h2d += bm;
        }
        if (f.var()) {
            XCUDA(x, cudaMemcpyAsync(s.d_in_off[i], s.h_off[i], (size_t)(s.rows + 1) * f.ow(), cudaMemcpyHostToDevice, x->s_h2d), "H2D offsets");
            x->bytes_h2d += (size_t)(s.rows + 1) * f.ow();
        }
    }
    XCUDA(x, cudaEventRecord(s.e_h2d, x->s_h2d), "record h2d");
    XCUDA(x, cudaStreamWaitEvent(c->stream, s.e_h2d, 0), "wait h2d");
    if (s.d2h_recorded) XCUDA(x, cudaStreamWaitEvent(c->stream, s.e_d2h, 0), "wait d2h");
    const size_t D = x->dev_fields.size();  // device columns: every field except the list placeholders (+ the hidden list columns)
    std::vector<dfd_column> in(D), out(D);
    for (size_t k = 0; k < D; ++k) {
        const size_t i = (size_t)x->dev_fields[k];
        const FieldInfo& f = x->fields[i];
        if (f.var()) {
            // (values_bytes = the bytes staged into this chunk: the offsets were built here, so the partitioner need not read them back)
            in[k] = dfd_column{f.kind, 0, s.d_in[i], s.d_in_off[i], s.has_valid[i] ? (uint8_t*)s.d_in_valid[i] : nullptr, 0, s.data_bytes[i]};
            out[k] = dfd_column{f.kind, 0, s.d_out[i], s.d_out_off[i], s.has_valid[i] ? (uint8_t*)s.d_out_valid[i] : nullptr, 0, (int64_t)s.out_cap[i]};
        } else {
            in[k] = dfd_column{f.kind, f.width, s.d_in[i], nullptr, s.has_valid[i] ? (uint8_t*)s.d_in_valid[i] : nullptr, 0, 0};
            out[k] = dfd_column{f.kind, f.width, s.d_out[i], nullptr, s.has_valid[i] ? (uint8_t*)s.d_out_valid[i] : nullptr, 0, 0};
        }
        if (f.kind == DFD_COL_BOOL)
            XCUDA(x, cudaMemsetAsync(s.d_out[i], 0, PinnedPool::bitmap_bytes(s.rows), c->stream), "memset");
        if (s.has_valid[i]) XCUDA(x, cudaMemsetAsync(s.d_out_valid[i], 0, PinnedPool::bitmap_bytes(s.rows), c->stream), "memset");
    }
    for (size_t i = 0; i < C; ++i)  // dictionary keys of this chunk (caller holds the context lock: set the fields directly)
        if (x->fields[i].dict && x->key_of_field[i] >= 0) {
            x->part->key_modes[(size_t)x->key_of_field[i]] = dfd::KEY_HASH_DICTIONARY;
            x->part->key_dicts[(size_t)x->key_of_field[i]] = dfd_partitioner::KeyDict{s.dict_hashes[i], s.dict_valid[i], x->fields[i].dict_index_unsigned};
        }
    int rc = partition_device_locked(x->part, in.data(), (int)D, s.rows, out.data(), c->stream, /*var_bytes_known=*/true);
    if (rc) return fail(x, rc, dfd_last_error());
    // list fields: child offsets = exclusive scan of the gathered element lengths; child validity bytes -> bitmap
    std::vector<const void*> d2h_src(C, nullptr);
    std::vector<size_t> d2h_nb(C, 0);
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        if (!f.list) continue;
        const int64_t ne = s.data_bytes[(size_t)f.h_len] / 4;
        auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
        const size_t o_off = 0, o_bits = al((size_t)(ne + 1) * 4 + 16), o_sums = o_bits + al((size_t)(ne + 63) / 64 * 8 + 16);
        const size_t total = o_sums + al((size_t)(ne / 2048 + 4) * 8);
        int rc2 = s.list_tmp[i].ensure(total, c->device);
        if (rc2) return fail(x, rc2, dfd_last_error());
        char* lt = (char*)s.list_tmp[i].ptr;
        if (f.child_width > 0) {  // primitive child: no child offsets; the gathered lengths themselves are not needed on the host
            d2h_src[(size_t)f.h_len] = lt + o_off;
            d2h_nb[(size_t)f.h_len] = 0;
        } else {
            if ((rc2 = launch_lengths_to_offsets(s.d_out[(size_t)f.h_len], 4, ne, (unsigned long long*)(lt + o_sums), lt + o_off, c->stream)))
                return fail(x, rc2, dfd_last_error());
            d2h_src[(size_t)f.h_len] = lt + o_off;
            d2h_nb[(size_t)f.h_len] = (size_t)(ne + 1) * 4;
        }
        if (f.h_valid >= 0) {
            if ((rc2 = launch_bytes_to_bits((const uint8_t*)s.d_out[(size_t)f.h_valid], ne, lt + o_bits, c->stream))) return fail(x, rc2, dfd_last_error());
            d2h_src[(size_t)f.h_valid] = lt + o_bits;
            d2h_nb[(size_t)f.h_valid] = (size_t)((ne + 31) / 32 * 4);
        }
    }
    XCUDA(x, cudaMemcpyAsync(s.h_part_starts, x->part->d_part_starts, sizeof(int64_t) * (x->N + 1), cudaMemcpyDeviceToHost, c->stream),
          "D2H part_starts");
    XCUDA(x, cudaEventRecord(s.e_k, c->stream), "record k");
    s.k_recorded = true;
    // D2H of the destination-sorted chunk into the pooled pinned buffer taken above
    XCUDA(x, cudaStreamWaitEvent(x->s_d2h, s.e_k, 0), "wait k");
    for (size_t k = 0; k < D; ++k) {
        const size_t i = (size_t)x->dev_fields[k];
        const FieldInfo& f = x->fields[i];
        size_t nb = f.kind == DFD_COL_BOOL ? (size_t)((s.rows + 7) / 8) : (size_t)s.rows * f.width;
        const void* src = s.d_out[i];
        if (f.var()) {
            nb = (size_t)s.data_bytes[i];
            if (d2h_src[i]) { src = d2h_src[i]; nb = d2h_nb[i]; }  // list columns: scanned child offsets / re-packed child validity
            if (s.out->data_cap[i] < nb || !s.out->values[i]) {  // grow this pinned chunk's string buffer (never NULL, even for 0 bytes)
                if (s.out->values[i]) cudaFreeHost(s.out->values[i]);
                s.out->values[i] = nullptr;
                s.out->data_cap[i] = 0;
                size_t want = nb + nb / 4 + 64;
                XCUDA(x, cudaHostAlloc(&s.out->values[i], want, cudaHostAllocPortable), "cudaHostAlloc(string bytes)");
                s.out->data_cap[i] = want;
            }
            if (!f.hidden || f.role == 1) {  // (the per-row offsets of the hidden bytes / validity columns are not needed on the host)
                XCUDA(x, cudaMemcpyAsync(s.out->offsets[i], s.d_out_off[i], (size_t)(s.rows + 1) * f.ow(), cudaMemcpyDeviceToHost, x->s_d2h), "D2H offsets");
                x->bytes_d2h += (size_t)(s.rows + 1) * f.ow();
            }
        }
        if (nb) XCUDA(x, cudaMemcpyAsync(s.out->values[i], src, nb, cudaMemcpyDeviceToHost, x->s_d2h), "D2H");
        x->bytes_d2h += nb;
        if (s.has_valid[i]) {
            XCUDA(x, cudaMemcpyAsync(s.out->validity[i], s.d_out_valid[i], (size_t)((s.rows + 7) / 8), cudaMemcpyDeviceToHost, x->s_d2h), "D2H");
            x->bytes_d2h += (size_t)((s.rows + 7) / 8);
        }
    }
    XCUDA(x, cudaEventRecord(s.e_d2h, x->s_d2h), "record d2h");
    s.d2h_recorded = true;
    s.in_flight = true;
    return DFD_OK;
}

// make the next slot current: emit whatever it still holds, fence its buffers
int open_next_slot(dfd_repartition_exec* x) {
    x->cur = (x->cur + 1) % x->depth;
    Slot& s = x->slots[x->cur];
    int rc = emit_slot(x, s);
    if (rc) return rc;
    // H2D into this slot must not overtake the kernels that last read it
    if (s.k_recorded) {
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
        XCUDA(x, cudaStreamWaitEvent(x->s_h2d, s.e_k, 0), "wait k (h2d)");
    }
    s.rows = 0;
    std::fill(s.has_valid.begin(), s.has_valid.end(), false);
    std::fill(s.data_bytes.begin(), s.data_bytes.end(), 0);
    std::fill(s.dict_id.begin(), s.dict_id.end(), DictId{});
    x->cur_open = true;
    return DFD_OK;
}

using dfd::host::append_bits;  // (bit-granular bitmap concatenation: dfd_host_staging.h, CPU-tested)

const uint8_t* validity_of(const ArrowArray* c) {
    return (c->null_count != 0 && c->n_buffers > 0 && c->buffers[0]) ? (const uint8_t*)c->buffers[0] : nullptr;
}

DictId dict_identity(const ArrowArray* d) {
    return DictId{d->n_buffers > 0 ? d->buffers[d->n_buffers - 1] : nullptr, d->offset, d->length};
}

bool same_dictionary(const FieldInfo& f, const ArrowArray* mine, const ArrowArray* theirs);
int grow_var_bytes(dfd_repartition_exec* x, int64_t n, bool* fits);

// Host-side preparation of rows [start, start + n) of `b` for the open chunk: where every variable-width device column's
// offsets and bytes come from (views and lists are converted to offsets + bytes here, index arithmetic only), and whether
// these rows can JOIN the chunk (`*fits`): same dictionaries, and string bytes within the offset width.  The chunk's
// byte buffers grow here when the rows need more room.
int prepare_rows(dfd_repartition_exec* x, const ArrowArray* b, int64_t start, int64_t n, bool* fits) {
    Slot& s = x->slots[x->cur];
    *fits = true;
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        const int64_t lo = c->offset + start;
        if (validity_of(c) && !(f.flags & ARROW_FLAG_NULLABLE) && c->null_count > 0)
            return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": nulls in a column the schema declares non-nullable");
        if (f.list) {
            // List<Utf8 / Binary> -> three hidden Binary columns: row -> its elements' int32 lengths, row -> its elements' bytes
            // (one contiguous range of the child's data buffer), row -> one validity byte per element
            if (c->n_children != 1 || !c->children[0]) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": list array without a child");
            const ArrowArray* v = c->children[0];
            const int32_t* loff = (const int32_t*)c->buffers[1];
            const int32_t cw = f.child_width;
            const int32_t* coff = cw > 0 ? nullptr : (const int32_t*)v->buffers[1] + v->offset;
            const uint8_t* cvalid = validity_of(v);
            const int64_t e0 = loff[lo], e1 = loff[lo + n], ne = e1 - e0;
            if (ne < 0) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": list offsets are not monotonic");
            if (ne * 4 > 0x7fffffffLL || ne * (int64_t)(cw > 0 ? cw : 1) > 0x7fffffffLL)
                return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": too many list elements in one chunk");
            const size_t hl = (size_t)f.h_len, hb = (size_t)f.h_bytes;
            std::vector<char>& ol = x->tmp_off[hl];
            std::vector<char>& dl = x->tmp_bytes[hl];
            std::vector<char>& ob = x->tmp_off[hb];
            ol.resize((size_t)(n + 1) * 4);
            ob.resize((size_t)(n + 1) * 4);
            dl.resize((size_t)ne * 4 + 16);
            int32_t* ov32 = nullptr;
            char* dvb = nullptr;
            if (f.h_valid >= 0) {
                std::vector<char>& ov = x->tmp_off[(size_t)f.h_valid];
                std::vector<char>& dv = x->tmp_bytes[(size_t)f.h_valid];
                ov.resize((size_t)(n + 1) * 4);
                dv.resize((size_t)ne + 16);
                ov32 = (int32_t*)ov.data();
                dvb = dv.data();
            }
            if (cw > 0) {
                dfd::host::split_list_rows_fixed(loff, cw, cvalid, v->offset, lo, n, (int32_t*)ol.data(), (int32_t*)ob.data(), (int32_t*)dl.data(), ov32, dvb);
                x->prep[hb] = VarPrep{ob.data(), 0, (const char*)v->buffers[1] + (size_t)(v->offset + e0) * (size_t)cw, ne * (int64_t)cw};
            } else {
                dfd::host::split_list_rows(loff, coff, cvalid, v->offset, lo, n, (int32_t*)ol.data(), (int32_t*)ob.data(), (int32_t*)dl.data(), ov32, dvb);
                x->prep[hb] = VarPrep{ob.data(), 0, (const char*)v->buffers[2] + coff[e0], (int64_t)coff[e1] - coff[e0]};
            }
            x->prep[hl] = VarPrep{ol.data(), 0, dl.data(), ne * 4};
            if (f.h_valid >= 0) x->prep[(size_t)f.h_valid] = VarPrep{(const char*)ov32, 0, dvb, ne};
        } else if (f.var() && f.view) {
            // Utf8View / BinaryView -> offsets + contiguous bytes (16-byte views: len | 12 inline bytes, or len | prefix |
            // buffer index | offset into one of the variadic data buffers); from here on an ordinary Utf8 / Binary column
            std::vector<char>& vo = x->tmp_off[i];
            std::vector<char>& vb = x->tmp_bytes[i];
            vo.resize((size_t)(n + 1) * 4);
            int32_t* off32 = (int32_t*)vo.data();
            const uint8_t* views = (const uint8_t*)c->buffers[1];
            const int64_t total = dfd::host::view_offsets(views, validity_of(c), lo, n, off32);
            if (total < 0) return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": more than 2 GiB of view data in one chunk");
            vb.resize((size_t)total + 16);
            dfd::host::view_bytes(views, c->buffers + 2, lo, n, off32, vb.data());
            x->prep[i] = VarPrep{vo.data(), 0, vb.data(), total};
        } else if (f.var()) {
            const size_t ow = f.ow();
            const char* offs = (const char*)c->buffers[1];
            int64_t first, last;
            if (ow == 4) { first = ((const int32_t*)offs)[lo]; last = ((const int32_t*)offs)[lo + n]; }
            else { first = ((const int64_t*)offs)[lo]; last = ((const int64_t*)offs)[lo + n]; }
            if (last < first) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": offsets are not monotonic");
            x->prep[i] = VarPrep{offs + (size_t)lo * ow, first, (const char*)c->buffers[2] + first, last - first};
        } else if (f.dict) {
            if (!c->dictionary) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": dictionary array without a dictionary");
            // one dictionary per chunk (it travels by reference).  A batch whose dictionary is a different OBJECT with the same
            // values (readers re-materialise the dictionary for every batch) joins the chunk and is served by the chunk's first one
            const DictId id = dict_identity(c->dictionary);
            if (s.rows > 0 && !(s.dict_id[i] == id)) {
                const ArrowArray* mine = !s.held.empty() && s.held.front()->array.children[i] ? s.held.front()->array.children[i]->dictionary : nullptr;
                if (!same_dictionary(f, mine, c->dictionary)) *fits = false;
            }
        }
    }
    if (!*fits) return DFD_OK;
    return grow_var_bytes(x, n, fits);
}

// Does a dictionary with other buffers (`theirs`) hold the same values as the chunk's (`mine`)?  Both in host memory.
bool same_dictionary(const FieldInfo& f, const ArrowArray* mine, const ArrowArray* theirs) {
    const bool dvar = f.dict_kind == DFD_COL_UTF8 || f.dict_kind == DFD_COL_LARGE_UTF8 || f.dict_kind == DFD_COL_BINARY;
    const bool comparable = mine && f.dict_format[0] != 'v' && mine->length == theirs->length && mine->n_buffers == theirs->n_buffers &&
                            mine->length <= (1 << 16);  // (a linear comparison per batch: only worth it for small dictionaries — a batch's own)
    return comparable && dfd::host::flat_arrays_equal(mine->length, dvar ? (f.dict_kind == DFD_COL_LARGE_UTF8 ? 8 : 4) : 0,
                                                      f.dict_kind == DFD_COL_BOOL ? 0 : f.dict_width, mine->buffers, mine->offset, mine->null_count,
                                                      theirs->buffers, theirs->offset, theirs->null_count);
}

// The string bytes `x->prep` says rows [.., + n) add: cut the chunk early (`*fits` = false) when they would pass what 32-bit
// offsets address, otherwise grow the chunk's byte buffers when they need more room.
int grow_var_bytes(dfd_repartition_exec* x, int64_t n, bool* fits) {
    Slot& s = x->slots[x->cur];
    for (int fi : x->dev_fields) {
        const size_t h = (size_t)fi;
        const FieldInfo& f = x->fields[h];
        if (!f.var()) continue;
        const int64_t need = s.data_bytes[h] + x->prep[h].nbytes;
        if (f.ow() == 4 && need > 0x7fffffffLL) {
            if (s.rows > 0) { *fits = false; return DFD_OK; }
            return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": more than 2 GiB of string data in one chunk (use a smaller chunk_rows or LargeUtf8)");
        }
        if ((size_t)need <= s.in_cap[h]) continue;
        // grow the chunk's byte buffers, keeping what is already staged (the copy is ordered after the H2D appends on the same
        // stream; cudaFree waits for it).  Sized for a FULL chunk at the bytes per row seen so far, and at least doubled, so
        // that growth is rare and the following batches join the chunk instead of cutting it
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
        size_t want = (size_t)need + (size_t)need / 4 + 256;
        if (want < 2 * s.in_cap[h]) want = 2 * s.in_cap[h];
        const double per_row = (double)need / (double)(s.rows + n);
        double full = per_row * (double)x->chunk_rows * 1.25;
        if (full > (double)(1ull << 30)) full = (double)(1ull << 30);
        if ((size_t)full > want) want = (size_t)full;
        if (f.ow() == 4 && want > 0x7fffffffull + 256) want = 0x7fffffffull + 256;
        void* bigger = nullptr;
        XCUDA(x, cudaMalloc(&bigger, want), "cudaMalloc(string bytes)");
        if (s.data_bytes[h] > 0) {
            cudaError_t ce = cudaMemcpyAsync(bigger, s.d_in[h], (size_t)s.data_bytes[h], cudaMemcpyDeviceToDevice, x->s_h2d);
            if (ce != cudaSuccess) {
                cudaFree(bigger);
                return fail(x, DFD_ERR_CUDA, std::string("grow string bytes: ") + cudaGetErrorString(ce));
            }
        }
        cudaFree(s.d_in[h]);
        cudaFree(s.d_out[h]);
        s.d_in[h] = bigger;
        s.d_out[h] = nullptr;
        s.in_cap[h] = want;
        s.out_cap[h] = 0;
        XCUDA(x, cudaMalloc(&s.d_out[h], want), "cudaMalloc(string bytes)");
        s.out_cap[h] = want;
    }
    return DFD_OK;
}

// copy rows [start, start + n) of `b` (prepared by prepare_rows) to the end of the open chunk.  Fixed-width values and
// string bytes go to the device straight from the batch; bitmaps (validity, boolean values) and string offsets are
// concatenated on the host — bit-granular, offsets re-based onto the chunk's byte buffer — and follow when the chunk is
// flushed.  A column gets a validity bitmap from the first batch that has one (earlier rows count as valid).
int stage_rows(dfd_repartition_exec* x, const ArrowArray* b, int64_t start, int64_t n) {
    Slot& s = x->slots[x->cur];
    std::lock_guard<std::mutex> lk(x->ctx->mu);
    XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
    auto host_bitmap = [&](std::vector<uint8_t*>& v, size_t i) -> uint8_t* {
        if (!v[i] && cudaHostAlloc((void**)&v[i], PinnedPool::bitmap_bytes(x->chunk_rows) + 8, cudaHostAllocPortable) != cudaSuccess) v[i] = nullptr;
        return v[i];
    };
    auto stage_validity = [&](size_t i, const uint8_t* valid, int64_t lo) -> int {
        if (!valid && !s.has_valid[i]) return DFD_OK;
        uint8_t* hb = host_bitmap(s.h_valid, i);
        if (!hb) return fail(x, DFD_ERR_OOM, "pinned host allocation failed");
        if (!s.has_valid[i]) {
            append_bits(hb, 0, nullptr, 0, s.rows);
            s.has_valid[i] = true;
        }
        append_bits(hb, s.rows, valid, lo, n);
        return DFD_OK;
    };
    auto stage_var = [&](size_t h) -> int {
        const VarPrep& p = x->prep[h];
        const int64_t base = s.data_bytes[h];
        if (x->fields[h].ow() == 4) {
            int32_t* dst = (int32_t*)s.h_off[h] + s.rows;
            const int32_t* src = (const int32_t*)p.off;
            const int64_t delta = base - p.first;
            for (int64_t r = 0; r <= n; ++r) dst[r] = (int32_t)(src[r] + delta);
        } else {
            int64_t* dst = (int64_t*)s.h_off[h] + s.rows;
            const int64_t* src = (const int64_t*)p.off;
            const int64_t delta = base - p.first;
            for (int64_t r = 0; r <= n; ++r) dst[r] = src[r] + delta;
        }
        if (p.nbytes) XCUDA(x, cudaMemcpyAsync((char*)s.d_in[h] + base, p.bytes, (size_t)p.nbytes, cudaMemcpyHostToDevice, x->s_h2d), "H2D");
        s.data_bytes[h] = base + p.nbytes;
        x->bytes_h2d += (size_t)p.nbytes;
        return DFD_OK;
    };
    int rc2 = DFD_OK;
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        const int64_t lo = c->offset + start;
        const uint8_t* valid = (f.flags & ARROW_FLAG_NULLABLE) ? validity_of(c) : nullptr;
        if (f.list) {
            if ((rc2 = stage_var((size_t)f.h_len)) || (rc2 = stage_var((size_t)f.h_bytes))) return rc2;
            if (f.h_valid >= 0 && (rc2 = stage_var((size_t)f.h_valid))) return rc2;
            if ((rc2 = stage_validity((size_t)f.h_len, valid, lo))) return rc2;  // the list's own validity rides on the lengths column
            continue;
        }
        if (f.dict && s.rows == 0) s.dict_id[i] = dict_identity(c->dictionary);
        if (f.dict && x->key_of_field[i] >= 0 && s.rows == 0) {
            // dictionary KEY: hash the dictionary values once per chunk on the device (DataFusion hash_dictionary); rows pick dict_hashes[index]
            const ArrowArray* d = c->dictionary;
            const int64_t dn = d->offset + d->length;
            const bool dvar = f.dict_kind == DFD_COL_UTF8 || f.dict_kind == DFD_COL_LARGE_UTF8 || f.dict_kind == DFD_COL_BINARY;
            const size_t dow = f.dict_kind == DFD_COL_LARGE_UTF8 ? 8 : 4;
            const bool dhv = d->null_count != 0 && d->n_buffers > 0 && d->buffers[0] != nullptr;
            int64_t dbytes = 0;
            if (dvar) dbytes = dow == 4 ? ((const int32_t*)d->buffers[1])[dn] : ((const int64_t*)d->buffers[1])[dn];
            auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
            const size_t o_hash = 0, o_off = al((size_t)(d->length + 1) * 8), o_data = o_off + al(dvar ? (size_t)(dn + 1) * dow : 0);
            const size_t vbytes = f.dict_kind == DFD_COL_BOOL ? (size_t)((dn + 7) / 8) : (dvar ? (size_t)dbytes : (size_t)dn * f.dict_width);
            const size_t o_valid = o_data + al(vbytes + 16), total = o_valid + al((size_t)((dn + 7) / 8) + 16);
            rc2 = s.dict_buf[i].ensure(total, x->ctx->device);
            if (rc2) return fail(x, rc2, dfd_last_error());
            char* db = (char*)s.dict_buf[i].ptr;
            if (dvar) XCUDA(x, cudaMemcpyAsync(db + o_off, d->buffers[1], (size_t)(dn + 1) * dow, cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary offsets");
            if (vbytes) XCUDA(x, cudaMemcpyAsync(db + o_data, d->buffers[dvar ? 2 : 1], vbytes, cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary values");
            if (dhv) XCUDA(x, cudaMemcpyAsync(db + o_valid, d->buffers[0], (size_t)((dn + 7) / 8), cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary validity");
            const int32_t dmode = interval_key_mode(f.dict_format);  // interval values hash field by field, as interval keys do
            const int32_t hkind = dmode == DFD_KEY_HASH_INTERVAL_DAY_TIME ? COL_INTERVAL_DAY_TIME
                                  : dmode == DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO ? COL_INTERVAL_MONTH_DAY_NANO : f.dict_kind;
            dfd_column dc{hkind, f.dict_width, db + o_data, dvar ? (void*)(db + o_off) : nullptr, dhv ? (uint8_t*)(db + o_valid) : nullptr, d->offset,
                          (int64_t)vbytes};
            rc2 = hash_columns_locked(x->ctx, &dc, 1, d->length, nullptr, (uint64_t*)(db + o_hash), x->s_h2d);
            if (rc2) return fail(x, rc2, dfd_last_error());
            s.dict_hashes[i] = (const uint64_t*)(db + o_hash);
            // the validity handed to the partitioner is indexed by dictionary index (0-based): re-base with the values' offset
            s.dict_valid[i] = dhv ? (const uint8_t*)(db + o_valid) : nullptr;
            if (dhv && d->offset != 0) return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": sliced dictionary values with nulls are not supported yet");
            x->bytes_h2d += vbytes + (dvar ? (size_t)(dn + 1) * dow : 0);
        }
        if (f.var()) {
            if ((rc2 = stage_var(i))) return rc2;
        } else if (f.kind == DFD_COL_FIXED) {
            const char* src = (const char*)c->buffers[1] + (size_t)lo * f.width;
            char* dst = (char*)s.d_in[i] + (size_t)s.rows * f.width;
            XCUDA(x, cudaMemcpyAsync(dst, src, (size_t)n * f.width, cudaMemcpyHostToDevice, x->s_h2d), "H2D");
            x->bytes_h2d += (size_t)n * f.width;
        } else {  // boolean values: one more bitmap
            uint8_t* hb = host_bitmap(s.h_bool, i);
            if (!hb) return fail(x, DFD_ERR_OOM, "pinned host allocation failed");
            append_bits(hb, s.rows, (const uint8_t*)c->buffers[1], lo, n);
        }
        if ((rc2 = stage_validity(i, valid, lo))) return rc2;
    }
    s.rows += n;
    return DFD_OK;
}

// emit every in-flight chunk (oldest first) whose D2H has already completed
int emit_ready(dfd_repartition_exec* x) {
    for (int i = 1; i <= x->depth; ++i) {
        Slot& s = x->slots[(x->cur + i) % x->depth];
        if (!s.in_flight) continue;
        cudaError_t q = cudaEventQuery(s.e_d2h);
        if (q == cudaErrorNotReady) break;  // keep emission in chunk order
        if (q != cudaSuccess) return fail(x, DFD_ERR_CUDA, std::string("D2H: ") + cudaGetErrorString(q));
        int rc = emit_slot(x, s);
        if (rc) return rc;
    }
    return DFD_OK;
}

// ---- device input (dfd_repartition_exec_push_device): the same chunks, assembled on the device by k_stage_* ---------------

// the host waits for everything enqueued on the staging stream so far (read-backs of sizes / dictionaries)
int wait_staging(dfd_repartition_exec* x) {
    {
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
        if (!x->e_sizes) XCUDA(x, cudaEventCreateWithFlags(&x->e_sizes, cudaEventDisableTiming), "cudaEventCreate");
        XCUDA(x, cudaEventRecord(x->e_sizes, x->s_h2d), "record read-back");
    }
    XCUDA(x, cudaEventSynchronize(x->e_sizes), "read-back");
    return DFD_OK;
}

// Host copies of the dictionaries of one device batch.  The output batches are host arrays and reference these (held by
// the chunk), so a device batch need not outlive the device work that reads it.
struct HostDicts {
    std::vector<ArrowArray> kids;  // per column: only `dictionary` is set
    std::vector<ArrowArray*> kid_ptrs;
    std::vector<ArrowArray> dicts;
    std::vector<std::vector<const void*>> bufs;
    std::vector<std::vector<char>> mem;
};
void host_dicts_release(ArrowArray* a) {
    delete (HostDicts*)a->private_data;
    a->release = nullptr;
}

int host_dictionaries(dfd_repartition_exec* x, const ArrowArray* b, HeldInput* out) {
    const size_t C = x->n_visible;
    std::unique_ptr<HostDicts> h(new HostDicts());
    h->kids.resize(C);
    h->kid_ptrs.resize(C);
    h->dicts.resize(C);
    h->bufs.resize(C);
    for (size_t i = 0; i < C; ++i) {
        memset(&h->kids[i], 0, sizeof(ArrowArray));
        h->kids[i].release = child_release;
        h->kid_ptrs[i] = &h->kids[i];
    }
    auto copy = [&](const void* src, size_t n) -> const void* {  // D2H on the staging stream (after the producer's event)
        h->mem.emplace_back(n + 8);
        char* dst = h->mem.back().data();
        if (n && cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, x->s_h2d) != cudaSuccess) return nullptr;
        x->bytes_d2h += n;
        return dst;
    };
    for (int phase = 0; phase < 2; ++phase) {  // 0: validity, values, offsets, views, variadic sizes; 1: the bytes they locate
        {
            std::lock_guard<std::mutex> lk(x->ctx->mu);
            XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
            for (size_t i = 0; i < C; ++i) {
                const FieldInfo& f = x->fields[i];
                const ArrowArray* d = f.dict ? b->children[i]->dictionary : nullptr;
                if (!d) continue;  // (prepare refuses a dictionary column without a dictionary)
                const int64_t dn = d->offset + d->length;
                const bool view = f.dict_format[0] == 'v';
                const bool dvar = !view && (f.dict_kind == DFD_COL_UTF8 || f.dict_kind == DFD_COL_LARGE_UTF8 || f.dict_kind == DFD_COL_BINARY);
                const size_t dow = f.dict_kind == DFD_COL_LARGE_UTF8 ? 8 : 4;
                std::vector<const void*>& hb = h->bufs[i];
                bool ok = true;
                if (phase == 0) {
                    if (d->n_buffers < (view ? 3 : dvar ? 3 : 2) || !d->buffers || !d->buffers[1])
                        return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": malformed dictionary");
                    hb.assign((size_t)d->n_buffers, nullptr);
                    if (d->null_count != 0 && d->buffers[0]) ok &= (hb[0] = copy(d->buffers[0], (size_t)((dn + 7) / 8))) != nullptr;
                    const size_t nb1 = f.dict_kind == DFD_COL_BOOL ? (size_t)((dn + 7) / 8) : view ? (size_t)dn * 16 : dvar ? (size_t)(dn + 1) * dow : (size_t)dn * f.dict_width;
                    ok &= (hb[1] = copy(d->buffers[1], nb1)) != nullptr;
                    if (view) ok &= (hb[(size_t)d->n_buffers - 1] = copy(d->buffers[d->n_buffers - 1], (size_t)(d->n_buffers - 3) * 8)) != nullptr;
                } else if (dvar) {
                    const int64_t last = dow == 8 ? ((const int64_t*)hb[1])[dn] : ((const int32_t*)hb[1])[dn];
                    ok &= (hb[2] = copy(d->buffers[2], (size_t)(last > 0 ? last : 0))) != nullptr;
                } else if (view) {
                    const int64_t* sizes = (const int64_t*)hb[(size_t)d->n_buffers - 1];
                    for (int64_t k = 0; k + 3 < d->n_buffers; ++k) ok &= (hb[(size_t)k + 2] = copy(d->buffers[k + 2], (size_t)sizes[k])) != nullptr;
                }
                if (!ok) return fail(x, DFD_ERR_CUDA, "column " + f.name + ": D2H of the dictionary failed");
            }
        }
        if (int rc = wait_staging(x)) return rc;
    }
    for (size_t i = 0; i < C; ++i) {
        const ArrowArray* d = x->fields[i].dict ? b->children[i]->dictionary : nullptr;
        if (!d) continue;
        ArrowArray& hd = h->dicts[i];
        hd = *d;
        hd.buffers = h->bufs[i].data();
        hd.n_children = 0;
        hd.children = nullptr;
        hd.dictionary = nullptr;
        hd.release = child_release;
        hd.private_data = nullptr;
        h->kids[i].dictionary = &hd;
    }
    ArrowArray top;
    memset(&top, 0, sizeof top);
    top.length = b->length;
    top.n_children = (int64_t)C;
    top.children = h->kid_ptrs.data();
    top.release = host_dicts_release;
    top.private_data = h.release();
    *out = std::make_shared<SharedInput>(top);
    return DFD_OK;
}

struct ViewTmp {  // byte offsets of the parts of a view field's device scratch, for n rows and `nbuf` variadic buffers
    size_t lens, off, sums, ptrs, total;
    ViewTmp(int64_t n, int64_t nbuf) {
        auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
        lens = 0;
        off = al((size_t)n * 4 + 16);
        sums = off + al((size_t)(n + 1) * 4 + 16);
        ptrs = sums + al((size_t)(n / 2048 + 4) * 8);
        total = ptrs + al((size_t)(nbuf > 0 ? nbuf : 1) * 8);
    }
};

// Device counterpart of prepare_rows: the same checks and chunk cuts.  Variable-width columns need their byte counts on
// the host (buffer growth, the 2 GiB cut of 32-bit offsets, values_bytes): k_stage_sizes computes them for all such
// columns at once, and the host reads them back (one small D2H and one wait; never for fixed-width-only schemas).
int prepare_rows_device(dfd_repartition_exec* x, const ArrowArray* b, const HeldInput& dicts, int64_t start, int64_t n, bool* fits) {
    Slot& s = x->slots[x->cur];
    *fits = true;
    std::vector<StageSize> jobs;
    std::vector<size_t> job_field;
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        const int64_t lo = c->offset + start;
        if (validity_of(c) && !(f.flags & ARROW_FLAG_NULLABLE) && c->null_count > 0)
            return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": nulls in a column the schema declares non-nullable");
        StageSize j;
        j.lo = lo;
        j.n = n;
        if (f.list) {
            if (c->n_children != 1 || !c->children[0]) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": list array without a child");
            const ArrowArray* v = c->children[0];
            j.op = STAGE_SIZE_LIST;
            j.off = c->buffers[1];
            j.off2 = f.child_width > 0 ? nullptr : (const int32_t*)v->buffers[1] + v->offset;
        } else if (f.var() && f.view) {
            j.op = STAGE_SIZE_VIEW;  // (j.lens: set once the field's scratch is sized, below)
            j.off = c->buffers[1];
            j.valid = validity_of(c);
        } else if (f.var()) {
            j.op = STAGE_SIZE_RANGE;
            j.ow = (int32_t)f.ow();
            j.off = c->buffers[1];
        } else {
            if (f.dict) {
                if (!c->dictionary) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": dictionary array without a dictionary");
                const DictId id = dict_identity(c->dictionary);  // (identity of the DEVICE dictionary; values compared on the host copies)
                if (s.rows > 0 && !(s.dict_id[i] == id)) {
                    const ArrowArray* mine = !s.dict_held.empty() ? s.dict_held.front()->array.children[i]->dictionary : nullptr;
                    if (!same_dictionary(f, mine, dicts->array.children[i]->dictionary)) *fits = false;
                }
            }
            continue;
        }
        jobs.push_back(j);
        job_field.push_back(i);
    }
    if (!*fits || jobs.empty()) return DFD_OK;
    const size_t nb = jobs.size() * 4 * sizeof(int64_t);
    {
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
        if (int rc = x->d_sizes.ensure(nb, x->ctx->device)) return fail(x, rc, dfd_last_error());
        if (!x->h_sizes) XCUDA(x, cudaHostAlloc((void**)&x->h_sizes, x->fields.size() * 4 * sizeof(int64_t), cudaHostAllocPortable), "cudaHostAlloc(sizes)");
        for (size_t k = 0; k < jobs.size(); ++k) {
            jobs[k].out = (int64_t*)x->d_sizes.ptr + 4 * k;
            if (jobs[k].op != STAGE_SIZE_VIEW) continue;
            const ViewTmp vt(n, b->children[job_field[k]]->n_buffers - 3);
            if (int rc = x->view_tmp[job_field[k]].ensure(vt.total, x->ctx->device)) return fail(x, rc, dfd_last_error());
            jobs[k].lens = (int32_t*)((char*)x->view_tmp[job_field[k]].ptr + vt.lens);
        }
        XCUDA(x, cudaMemsetAsync(x->d_sizes.ptr, 0, nb, x->s_h2d), "memset sizes");
        int rc = launch_stage_sizes(jobs.data(), (int)jobs.size(), x->s_h2d);
        for (size_t k = 0; k < jobs.size() && !rc; ++k) {  // views: offsets = exclusive scan of the lengths
            if (jobs[k].op != STAGE_SIZE_VIEW) continue;
            const ViewTmp vt(n, b->children[job_field[k]]->n_buffers - 3);
            char* t = (char*)x->view_tmp[job_field[k]].ptr;
            rc = launch_lengths_to_offsets(t + vt.lens, 4, n, (unsigned long long*)(t + vt.sums), t + vt.off, x->s_h2d);
        }
        if (rc) return fail(x, rc, dfd_last_error());
        XCUDA(x, cudaMemcpyAsync(x->h_sizes, x->d_sizes.ptr, nb, cudaMemcpyDeviceToHost, x->s_h2d), "D2H sizes");
    }
    if (int rc = wait_staging(x)) return rc;
    for (size_t k = 0; k < jobs.size(); ++k) {
        const size_t i = job_field[k];
        const FieldInfo& f = x->fields[i];
        const int64_t* r = x->h_sizes + 4 * k;
        x->dsz[i].assign(r, r + 4);
        if (f.list) {
            const int64_t ne = r[1] - r[0], cw = f.child_width;
            if (ne < 0 || (cw == 0 && r[3] < r[2])) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": list offsets are not monotonic");
            if (ne * 4 > 0x7fffffffLL || ne * (cw > 0 ? cw : 1) > 0x7fffffffLL)
                return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": too many list elements in one chunk");
            x->prep[(size_t)f.h_len].nbytes = ne * 4;
            x->prep[(size_t)f.h_bytes].nbytes = cw > 0 ? ne * cw : r[3] - r[2];
            if (f.h_valid >= 0) x->prep[(size_t)f.h_valid].nbytes = ne;
        } else if (f.view) {
            if (r[0] > 0x7fffffffLL) return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": more than 2 GiB of view data in one chunk");
            x->prep[i].nbytes = r[0];
        } else {
            if (r[1] < r[0]) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": offsets are not monotonic");
            x->prep[i].first = r[0];
            x->prep[i].nbytes = r[1] - r[0];
        }
    }
    return grow_var_bytes(x, n, fits);
}

// Device counterpart of stage_rows: append rows [start, start + n) of the device batch `b` to the open chunk — every buffer
// of every column in ONE k_stage_batch launch (plus a small H2D of the data buffer table of each view column).
int stage_rows_device(dfd_repartition_exec* x, const ArrowArray* b, const HeldInput& dicts, int64_t start, int64_t n) {
    Slot& s = x->slots[x->cur];
    std::lock_guard<std::mutex> lk(x->ctx->mu);
    XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
    std::vector<StageJob> jobs;
    auto validity = [&](size_t i, const uint8_t* valid, int64_t lo) {
        if (!valid && !s.has_valid[i]) return;
        StageJob j;
        j.op = STAGE_BITS;
        j.src = valid;
        j.a = lo;
        j.dst = s.d_in_valid[i];
        j.b = s.rows;
        j.c = s.has_valid[i] ? s.rows : 0;  // the first batch with a validity bitmap: earlier rows of the chunk count as valid
        j.n = n;
        s.has_valid[i] = true;
        jobs.push_back(j);
    };
    auto offsets = [&](size_t h, const void* src, int ow_in, int64_t scale) {
        StageJob j;
        j.op = STAGE_OFFSETS;
        j.src = src;
        j.ow_in = ow_in;
        j.ow_out = (int32_t)x->fields[h].ow();
        j.dst = (char*)s.d_in_off[h] + (size_t)s.rows * x->fields[h].ow();
        j.n = n;
        j.base = s.data_bytes[h];
        j.scale = scale;
        return j;
    };
    auto bytes = [&](size_t h, StageJob j) {  // (after the column's offsets job, which takes the old byte count as its base)
        j.dst = (char*)s.d_in[h] + s.data_bytes[h];
        jobs.push_back(j);
        s.data_bytes[h] += x->prep[h].nbytes;
    };
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        const int64_t lo = c->offset + start;
        const uint8_t* valid = (f.flags & ARROW_FLAG_NULLABLE) ? validity_of(c) : nullptr;
        if (f.list) {
            const ArrowArray* v = c->children[0];
            const size_t hl = (size_t)f.h_len, hb = (size_t)f.h_bytes;
            const int32_t* loff = (const int32_t*)c->buffers[1] + lo;
            const int32_t* coff = f.child_width > 0 ? nullptr : (const int32_t*)v->buffers[1] + v->offset;
            const int64_t e0 = x->dsz[i][0], ne = x->dsz[i][1] - e0, cw = f.child_width;
            jobs.push_back(offsets(hl, loff, 4, 4));
            StageJob len;
            if (cw > 0) { len.op = STAGE_FILL32; len.base = cw; }
            else { len.op = STAGE_DIFF32; len.src = coff + e0; }
            len.n = ne;
            bytes(hl, len);
            if (cw > 0) {
                jobs.push_back(offsets(hb, loff, 4, cw));
            } else {
                StageJob lo_ = offsets(hb, loff, 4, 1);
                lo_.op = STAGE_LIST_OFFSETS;
                lo_.src2 = coff;
                jobs.push_back(lo_);
            }
            StageJob cp;
            cp.src = cw > 0 ? (const char*)v->buffers[1] + (size_t)(v->offset + e0) * (size_t)cw : (const char*)v->buffers[2] + x->dsz[i][2];
            cp.n = x->prep[hb].nbytes;
            bytes(hb, cp);
            if (f.h_valid >= 0) {
                const size_t hv = (size_t)f.h_valid;
                jobs.push_back(offsets(hv, loff, 4, 1));
                StageJob vb;
                vb.op = STAGE_BIT_BYTES;
                vb.src = validity_of(v);
                vb.a = v->offset + e0;
                vb.n = ne;
                bytes(hv, vb);
            }
            validity(hl, valid, lo);  // the list's own validity rides on the lengths column
            continue;
        }
        if (f.dict && s.rows == 0) s.dict_id[i] = dict_identity(c->dictionary);
        if (f.dict && x->key_of_field[i] >= 0 && s.rows == 0) {
            // dictionary KEY: hash the device-resident values in place once per chunk (DataFusion hash_dictionary)
            const ArrowArray* d = c->dictionary;
            const ArrowArray* hd = dicts->array.children[i]->dictionary;  // (host copy: the byte count of string values)
            const int64_t dn = d->offset + d->length;
            const bool dvar = f.dict_kind == DFD_COL_UTF8 || f.dict_kind == DFD_COL_LARGE_UTF8 || f.dict_kind == DFD_COL_BINARY;
            const bool dhv = d->null_count != 0 && d->n_buffers > 0 && d->buffers[0] != nullptr;
            int64_t dbytes = 0;
            if (dvar) dbytes = f.dict_kind == DFD_COL_LARGE_UTF8 ? ((const int64_t*)hd->buffers[1])[dn] : ((const int32_t*)hd->buffers[1])[dn];
            const size_t vbytes = f.dict_kind == DFD_COL_BOOL ? (size_t)((dn + 7) / 8) : (dvar ? (size_t)dbytes : (size_t)dn * f.dict_width);
            int rc = s.dict_buf[i].ensure((size_t)(d->length + 1) * 8, x->ctx->device);
            if (rc) return fail(x, rc, dfd_last_error());
            const int32_t dmode = interval_key_mode(f.dict_format);
            const int32_t hkind = dmode == DFD_KEY_HASH_INTERVAL_DAY_TIME ? COL_INTERVAL_DAY_TIME
                                  : dmode == DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO ? COL_INTERVAL_MONTH_DAY_NANO : f.dict_kind;
            dfd_column dc{hkind, f.dict_width, (void*)d->buffers[dvar ? 2 : 1], dvar ? (void*)d->buffers[1] : nullptr, dhv ? (uint8_t*)d->buffers[0] : nullptr,
                          d->offset, (int64_t)vbytes};
            rc = hash_columns_locked(x->ctx, &dc, 1, d->length, nullptr, (uint64_t*)s.dict_buf[i].ptr, x->s_h2d);
            if (rc) return fail(x, rc, dfd_last_error());
            s.dict_hashes[i] = (const uint64_t*)s.dict_buf[i].ptr;
            s.dict_valid[i] = dhv ? (const uint8_t*)d->buffers[0] : nullptr;  // (the first batch of the chunk stays held until its D2H is done)
            if (dhv && d->offset != 0) return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": sliced dictionary values with nulls are not supported yet");
        }
        if (f.var() && f.view) {
            // Utf8View / BinaryView: lengths and their scan came with the sizes; the data buffer table goes to the device
            const int64_t nbuf = c->n_buffers - 3;  // (validity, views, data buffers..., variadic sizes: the sizes are not read)
            const ViewTmp vt(n, nbuf);
            char* t = (char*)x->view_tmp[i].ptr;
            if (nbuf > 0)
                XCUDA(x, cudaMemcpyAsync(t + vt.ptrs, c->buffers + 2, (size_t)nbuf * sizeof(void*), cudaMemcpyHostToDevice, x->s_h2d), "H2D view buffer table");
            jobs.push_back(offsets(i, t + vt.off, 4, 1));
            StageJob vb;
            vb.op = STAGE_VIEW_BYTES;
            vb.src = (const uint8_t*)c->buffers[1] + (size_t)lo * 16;
            vb.src2 = t + vt.ptrs;
            vb.src3 = t + vt.off;
            vb.n = n;
            bytes(i, vb);
        } else if (f.var()) {
            jobs.push_back(offsets(i, (const char*)c->buffers[1] + (size_t)lo * f.ow(), (int)f.ow(), 1));
            StageJob cp;
            cp.src = (const char*)c->buffers[2] + x->prep[i].first;
            cp.n = x->prep[i].nbytes;
            bytes(i, cp);
        } else if (f.kind == DFD_COL_FIXED) {
            StageJob cp;
            cp.src = (const char*)c->buffers[1] + (size_t)lo * f.width;
            cp.dst = (char*)s.d_in[i] + (size_t)s.rows * f.width;
            cp.n = n * f.width;
            jobs.push_back(cp);
        } else {  // boolean values: one more bitmap
            StageJob bv;
            bv.op = STAGE_BITS;
            bv.src = c->buffers[1];
            bv.a = lo;
            bv.dst = s.d_in[i];
            bv.b = bv.c = s.rows;
            bv.n = n;
            jobs.push_back(bv);
        }
        validity(i, valid, lo);
    }
    if (int rc = launch_stage_batch(jobs.data(), (int)jobs.size(), x->s_h2d)) return fail(x, rc, dfd_last_error());
    s.rows += n;
    return DFD_OK;
}

// After an error or an abort of a device-input operator: wait for the device work that still reads the pushed batches,
// then release them (the producer gets its memory back now, not when the operator is destroyed).
void release_device_inputs(dfd_repartition_exec* x) {
    {
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        cudaSetDevice(x->ctx->device);
        cudaStreamSynchronize(x->s_h2d);
        cudaStreamSynchronize(x->ctx->stream);
        cudaStreamSynchronize(x->s_d2h);
    }
    for (Slot& s : x->slots) {
        s.held.clear();
        s.dict_held.clear();
    }
}

}  // namespace

extern "C" {

int dfd_arrow_format_layout(const char* format, int32_t* kind, int32_t* width) {
    int32_t k = 0, w = 0;
    if (!format || !parse_format(format, &k, &w))
        return set_error(DFD_ERR_UNSUPPORTED, "Arrow format '%s' is not supported by the GPU shuffle path", format ? format : "(null)");
    if (kind) *kind = k;
    if (width) *width = w;
    return DFD_OK;
}

// List<Utf8> / List<Binary> / List<fixed-width primitive> (int32 list offsets): the nested shapes the shuffle path moves
// (payload only).  *child_width = 0 for string children, the value width for primitive ones (array_agg / median states).
static bool list_child_ok(const ArrowSchema* c, int32_t* child_width = nullptr) {
    if (!c->format || strcmp(c->format, "+l") != 0 || c->n_children != 1 || !c->children || !c->children[0]) return false;
    const ArrowSchema* v = c->children[0];
    if (!v->format || v->dictionary || v->n_children != 0) return false;
    int32_t k = 0, w = 0;
    if (strcmp(v->format, "u") == 0 || strcmp(v->format, "z") == 0) w = 0;
    else if (parse_format(v->format, &k, &w) && k == DFD_COL_FIXED && v->format[0] != 'w') { /* ints, floats, decimals, dates, times */ }
    else return false;
    if (child_width) *child_width = w;
    return true;
}

// One column of the record-batch schema: can the operator move it, and — if it is hash key `is_key` — hash it like DataFusion?
static int check_column(const ArrowSchema* c, long long i, bool is_key) {
    const char* name = c->name ? c->name : "";
    int32_t k, w;
    if (list_child_ok(c)) {  // List<Utf8 / Binary>: payload only
        if (is_key) return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): list columns cannot be hash keys", i, name);
        return DFD_OK;
    }
    if (!c->format || !parse_format(c->format, &k, &w))
        return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): Arrow format '%s' is not supported", i, name, c->format ? c->format : "(null)");
    if (c->dictionary) {  // Dictionary<integer index, flat values>: indices are scattered, the dictionary travels by reference
        if (k != DFD_COL_FIXED || !strchr("cCsSiIlL", c->format[0]) || c->format[1])
            return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary index type '%s' is not an integer", i, name, c->format);
        int32_t dk, dw;
        const ArrowSchema* d = c->dictionary;
        if (d->dictionary || d->n_children > 0 || !d->format || !parse_format(d->format, &dk, &dw))
            return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary value type '%s' is not supported", i, name, d->format ? d->format : "(null)");
        if (is_key && d->format[0] == 'v')
            return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary KEY with view-typed values is not supported", i, name);
        if (is_key && !hashable_format(d->format))
            return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary values of type '%s' cannot be hash keys", i, name, d->format);
        return DFD_OK;
    }
    if (is_key && !hashable_format(c->format))
        return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): columns of type '%s' travel as payload but cannot be hash keys", i, name, c->format);
    return DFD_OK;
}

int dfd_schema_supported(const struct ArrowSchema* schema) {
    if (!schema || !schema->format || strcmp(schema->format, "+s") != 0)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "schema must be a struct (record batch) schema");
    for (int64_t i = 0; i < schema->n_children; ++i)
        if (int rc = check_column(schema->children[i], (long long)i, false)) return rc;
    return DFD_OK;
}

int dfd_repartition_supported(const struct ArrowSchema* schema, const int32_t* key_cols, int n_keys) {
    if (!schema || !schema->format || strcmp(schema->format, "+s") != 0)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "schema must be a struct (record batch) schema");
    if (n_keys < 1 || n_keys > MAX_KEYS || !key_cols) return set_error(DFD_ERR_INVALID_ARGUMENT, "n_keys %d not in [1, %d]", n_keys, MAX_KEYS);
    for (int k = 0; k < n_keys; ++k)
        if (key_cols[k] < 0 || key_cols[k] >= schema->n_children) return set_error(DFD_ERR_INVALID_ARGUMENT, "key column index out of range");
    for (int64_t i = 0; i < schema->n_children; ++i) {
        bool is_key = false;
        for (int k = 0; k < n_keys; ++k) is_key |= key_cols[k] == i;
        if (int rc = check_column(schema->children[i], (long long)i, is_key)) return rc;
    }
    return DFD_OK;
}

int dfd_repartition_exec_create(dfd_ctx* ctx, const struct ArrowSchema* schema, const int32_t* key_cols, int n_keys,
                                uint32_t num_partitions, const dfd_exec_options* opts, dfd_repartition_exec** out) {
    if (!ctx || !schema || !out) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_create: NULL argument");
    *out = nullptr;
    if (!schema->format || strcmp(schema->format, "+s") != 0)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "schema must be a struct (record batch) schema, got format '%s'",
                         schema->format ? schema->format : "(null)");
    for (int64_t i = 0; i < schema->n_children; ++i) {  // (the same checks the plan hook runs through dfd_repartition_supported)
        bool is_key = false;
        for (int k = 0; k < n_keys; ++k) is_key |= key_cols && key_cols[k] == i;
        if (int rc = check_column(schema->children[i], (long long)i, is_key)) return rc;
    }
    std::unique_ptr<dfd_repartition_exec> x(new (std::nothrow) dfd_repartition_exec());
    if (!x) return set_error(DFD_ERR_OOM, "out of host memory");
    x->ctx = ctx;
    x->N = num_partitions;
    for (int64_t i = 0; i < schema->n_children; ++i) {
        const ArrowSchema* c = schema->children[i];
        FieldInfo f;
        f.name = c->name ? c->name : "";
        f.format = c->format ? c->format : "";
        f.flags = c->flags;
        int key_index = -1;
        for (int k = 0; k < n_keys; ++k)
            if (key_cols && key_cols[k] == i) key_index = k;
        int32_t child_width = 0;
        if (list_child_ok(c, &child_width)) {
            if (key_index >= 0) return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): list columns cannot be hash keys", (long long)i, f.name.c_str());
            f.list = true;
            f.child_width = child_width;
            f.kind = -1;
            f.width = 0;
            f.child_name = c->children[0]->name ? c->children[0]->name : "item";
            f.child_format = c->children[0]->format;
            f.child_flags = c->children[0]->flags;
            x->key_of_field.push_back(-1);
            x->fields.push_back(f);
            continue;
        }
        if (!parse_format(f.format.c_str(), &f.kind, &f.width))
            return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): Arrow format '%s' is not supported", (long long)i, f.name.c_str(), f.format.c_str());
        f.view = f.format[0] == 'v';
        if (c->dictionary) {
            const ArrowSchema* d = c->dictionary;
            if (f.kind != DFD_COL_FIXED || !strchr("cCsSiIlL", f.format[0]) || f.format[1])
                return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary index type '%s' is not an integer", (long long)i, f.name.c_str(), f.format.c_str());
            f.dict = true;
            f.dict_index_unsigned = strchr("CSIL", f.format[0]) != nullptr;
            f.dict_format = d->format ? d->format : "";
            f.dict_flags = d->flags;
            if (d->dictionary || d->n_children > 0 || !parse_format(f.dict_format.c_str(), &f.dict_kind, &f.dict_width))
                return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary value type '%s' is not supported", (long long)i, f.name.c_str(), f.dict_format.c_str());
            if (key_index >= 0 && f.dict_format[0] == 'v')
                return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary KEY with view-typed values is not supported", (long long)i, f.name.c_str());
        }
        x->key_of_field.push_back(key_index);
        x->fields.push_back(f);
    }
    for (int k = 0; k < n_keys; ++k)
        if (!key_cols || key_cols[k] < 0 || key_cols[k] >= (int)x->fields.size())
            return set_error(DFD_ERR_INVALID_ARGUMENT, "key column index out of range");
    // hidden device columns of the list fields, appended after the visible ones
    x->n_visible = x->fields.size();
    for (size_t i = 0; i < x->n_visible; ++i) {
        if (!x->fields[i].list) continue;
        auto hidden = [&](const char* tag, bool nullable) {
            FieldInfo h;
            h.name = x->fields[i].name + "." + tag;
            h.format = "z";
            h.kind = DFD_COL_BINARY;
            h.width = 0;
            h.hidden = true;
            h.owner = (int)i;
            h.role = tag[0] == 'l' ? 1 : tag[0] == 'b' ? 2 : 3;
            h.flags = nullable ? ARROW_FLAG_NULLABLE : 0;
            x->key_of_field.push_back(-1);
            x->fields.push_back(h);
            return (int)x->fields.size() - 1;
        };
        x->fields[i].h_len = hidden("lengths", (x->fields[i].flags & ARROW_FLAG_NULLABLE) != 0);
        x->fields[i].h_bytes = hidden("bytes", false);
        if (x->fields[i].child_flags & ARROW_FLAG_NULLABLE) x->fields[i].h_valid = hidden("validity", false);
    }
    x->dev_pos.assign(x->fields.size(), -1);
    for (size_t i = 0; i < x->fields.size(); ++i)
        if (!x->fields[i].nodev()) {
            x->dev_pos[i] = (int)x->dev_fields.size();
            x->dev_fields.push_back((int)i);
        }
    std::vector<int32_t> dev_keys(n_keys);
    for (int k = 0; k < n_keys; ++k) dev_keys[k] = x->dev_pos[(size_t)key_cols[k]];  // keys address the compact device column list
    int rc = dfd_partitioner_create(ctx, num_partitions, dev_keys.data(), n_keys, nullptr, &x->part);
    if (rc) return rc;  // (x has no CUDA resources yet; unique_ptr frees it)
    for (int k = 0; k < n_keys; ++k) {  // interval keys hash field by field (arrow's derived Hash), not as one integer
        const int mode = interval_key_mode(x->fields[(size_t)key_cols[k]].format);  // (a dictionary field's format is its index type)
        if (mode != DFD_KEY_HASH_PLAIN && (rc = dfd_partitioner_set_key_hash_mode(x->part, k, mode))) {
            dfd_partitioner_destroy(x->part);
            x->part = nullptr;
            return rc;
        }
    }
    x->chunk_rows = (opts && opts->chunk_rows > 0) ? opts->chunk_rows : (int64_t)(4 << 20);
    x->chunk_rows = (x->chunk_rows + 63) / 64 * 64;
    x->depth = (opts && opts->pipeline_depth > 0) ? opts->pipeline_depth : 3;
    if (x->depth < 2) x->depth = 2;
    int pool_chunks = (opts && opts->pinned_pool_chunks > 0) ? opts->pinned_pool_chunks : x->depth + 1;
    x->queues.resize(num_partitions);

    cudaError_t e;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        e = cudaSetDevice(ctx->device);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&x->s_h2d, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&x->s_d2h, cudaStreamNonBlocking);
        const size_t C = x->fields.size();
        x->slots.resize(x->depth);
        for (Slot& s : x->slots) {
            s.d_in.assign(C, nullptr); s.d_in_valid.assign(C, nullptr); s.d_out.assign(C, nullptr); s.d_out_valid.assign(C, nullptr);
            s.has_valid.assign(C, false);
            s.h_valid.assign(C, nullptr); s.h_bool.assign(C, nullptr); s.h_off.assign(C, nullptr); s.dict_id.assign(C, DictId{});
            s.d_in_off.assign(C, nullptr); s.d_out_off.assign(C, nullptr);
            s.in_cap.assign(C, 0); s.out_cap.assign(C, 0);
            s.first_off.assign(C, 0); s.data_bytes.assign(C, 0);
            s.dict_buf.resize(C); s.dict_hashes.assign(C, nullptr); s.dict_valid.assign(C, nullptr);
            s.list_tmp.resize(C);
            for (size_t i = 0; i < C && e == cudaSuccess; ++i) {
                const FieldInfo& f = x->fields[i];
                if (f.nodev()) continue;  // list placeholder: its rows live in the hidden columns
                if (f.var()) {  // offsets now, string bytes on demand
                    e = cudaMalloc(&s.d_in_off[i], (size_t)(x->chunk_rows + 16) * f.ow());
                    if (e == cudaSuccess) e = cudaHostAlloc((void**)&s.h_off[i], (size_t)(x->chunk_rows + 16) * f.ow(), cudaHostAllocPortable);
                    if (e == cudaSuccess) e = cudaMalloc(&s.d_out_off[i], (size_t)(x->chunk_rows + 16) * f.ow());
                    if (e == cudaSuccess && (f.flags & ARROW_FLAG_NULLABLE)) {
                        e = cudaMalloc(&s.d_in_valid[i], PinnedPool::bitmap_bytes(x->chunk_rows) + 8);
                        if (e == cudaSuccess) e = cudaMalloc(&s.d_out_valid[i], PinnedPool::bitmap_bytes(x->chunk_rows) + 8);
                    }
                    continue;
                }
                size_t vb = PinnedPool::value_bytes(f, x->chunk_rows) + 16 * (size_t)(f.width ? f.width : 1);
                e = cudaMalloc(&s.d_in[i], vb);
                if (e == cudaSuccess) e = cudaMalloc(&s.d_out[i], vb);
                if (e == cudaSuccess && (f.flags & ARROW_FLAG_NULLABLE)) {
                    e = cudaMalloc(&s.d_in_valid[i], PinnedPool::bitmap_bytes(x->chunk_rows) + 8);
                    if (e == cudaSuccess) e = cudaMalloc(&s.d_out_valid[i], PinnedPool::bitmap_bytes(x->chunk_rows) + 8);
                }
            }
            if (e == cudaSuccess) e = cudaHostAlloc((void**)&s.h_part_starts, sizeof(int64_t) * (num_partitions + 1), cudaHostAllocPortable);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.e_h2d, cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.e_k, cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.e_d2h, cudaEventDisableTiming);
        }
    }
    if (e != cudaSuccess) {
        int code = cuda_error(e, "dfd_repartition_exec_create allocations");
        dfd_repartition_exec_destroy(x.release());
        return code;
    }
    x->pool = std::make_shared<PinnedPool>();
    x->pool->device = ctx->device;
    x->pool->chunk_rows = x->chunk_rows;
    x->pool->set_fields(x->fields);
    x->pool->cache = pinned_cache_of(ctx);
    x->pool->max_chunks = (opts && opts->max_pinned_chunks > 0) ? (size_t)opts->max_pinned_chunks : 0;
    if (x->pool->max_chunks && x->pool->max_chunks < (size_t)pool_chunks) x->pool->max_chunks = (size_t)pool_chunks;
    std::vector<OutChunk*> pre;
    for (int i = 0; i < pool_chunks; ++i) {
        OutChunk* c = x->pool->acquire();
        if (!c) {
            dfd_repartition_exec_destroy(x.release());
            return set_error(DFD_ERR_OOM, "pinned pool allocation failed");
        }
        pre.push_back(c);
    }
    for (OutChunk* c : pre) x->pool->give_back(c);
    x->tmp_off.resize(x->fields.size());
    x->tmp_bytes.resize(x->fields.size());
    x->prep.resize(x->fields.size());
    x->view_tmp.resize(x->fields.size());
    x->dsz.assign(x->fields.size(), std::vector<int64_t>(4, 0));
    x->cur = x->depth - 1;  // open_next_slot() starts at slot 0
    *out = x.release();
    return DFD_OK;
}

void dfd_repartition_exec_destroy(dfd_repartition_exec* x) {
    if (!x) return;
    {
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        cudaSetDevice(x->ctx->device);
        if (x->s_h2d) cudaStreamSynchronize(x->s_h2d);
        if (x->s_d2h) cudaStreamSynchronize(x->s_d2h);
        cudaStreamSynchronize(x->ctx->stream);
        cudaFree(x->d_sizes.ptr);
        for (dfd::Scratch& b : x->view_tmp) cudaFree(b.ptr);
        if (x->h_sizes) cudaFreeHost(x->h_sizes);
        if (x->e_sizes) cudaEventDestroy(x->e_sizes);
        for (Slot& s : x->slots) {
            s.held.clear();
            s.dict_held.clear();
            if (s.out) { s.out->refs.store(1); s.out->pool = x->pool; chunk_unref(s.out); }
            for (void* p : s.d_in) cudaFree(p);
            for (void* p : s.d_in_valid) cudaFree(p);
            for (void* p : s.d_out) cudaFree(p);
            for (void* p : s.d_out_valid) cudaFree(p);
            for (void* p : s.d_in_off) cudaFree(p);
            for (void* p : s.d_out_off) cudaFree(p);
            for (uint8_t* p : s.h_valid) if (p) cudaFreeHost(p);
            for (uint8_t* p : s.h_bool) if (p) cudaFreeHost(p);
            for (char* p : s.h_off) if (p) cudaFreeHost(p);
            for (dfd::Scratch& b : s.dict_buf) cudaFree(b.ptr);
            for (dfd::Scratch& b : s.list_tmp) cudaFree(b.ptr);
            if (s.h_part_starts) cudaFreeHost(s.h_part_starts);
            if (s.e_h2d) cudaEventDestroy(s.e_h2d);
            if (s.e_k) cudaEventDestroy(s.e_k);
            if (s.e_d2h) cudaEventDestroy(s.e_d2h);
        }
        if (x->s_h2d) cudaStreamDestroy(x->s_h2d);
        if (x->s_d2h) cudaStreamDestroy(x->s_d2h);
    }
    for (PartQueue& q : x->queues)
        for (ArrowArray& a : q.batches)
            if (a.release) a.release(&a);
    if (x->part) dfd_partitioner_destroy(x->part);
    delete x;
}

int dfd_repartition_exec_push(dfd_repartition_exec* x, struct ArrowArray* batch) {
    if (!x || !batch) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_push: NULL argument");
    ScopedNs timed(x->ns_push);
    auto drop = [&]() { if (batch->release) batch->release(batch); };
    if (x->finished) { drop(); return set_error(DFD_ERR_INVALID_ARGUMENT, "push after finish/error: %s", x->error.c_str()); }
    if (batch->n_children != (int64_t)x->n_visible) {
        drop();
        return fail(x, DFD_ERR_INVALID_ARGUMENT, "batch has " + std::to_string(batch->n_children) + " columns, schema has " + std::to_string(x->n_visible));
    }
    const int64_t R = batch->length;
    x->rows_in += (uint64_t)R;
    if (R == 0) { drop(); return DFD_OK; }
    if (x->input_mode == INPUT_DEVICE) {
        drop();
        const int rc = fail(x, DFD_ERR_INVALID_ARGUMENT, "host batch pushed to an operator that takes device batches (push_device)");
        release_device_inputs(x);
        return rc;
    }
    for (int64_t i = 0; i < batch->n_children; ++i)
        if (batch->children[i]->length < R || (batch->offset != 0)) {
            drop();
            return fail(x, DFD_ERR_INVALID_ARGUMENT, "record batch children shorter than the batch, or non-zero struct offset");
        }
    x->input_mode = INPUT_HOST;
    // ownership of the batch moves to a shared holder: every chunk that stages rows from it (and, for dictionary columns,
    // every output batch that references its dictionaries) keeps it alive
    HeldInput holder = std::make_shared<SharedInput>(*batch);
    batch->release = nullptr;
    const ArrowArray* in = &holder->array;
    int rc = DFD_OK;
    int64_t done = 0;
    while (done < R) {
        if (!x->cur_open && (rc = open_next_slot(x))) return rc;
        Slot& s = x->slots[x->cur];
        const int64_t room = x->chunk_rows - s.rows;
        if (room == 0) {
            if ((rc = flush_current(x))) return rc;
            continue;
        }
        const int64_t n = R - done < room ? R - done : room;
        // batches of every shape are APPENDED to the open chunk (bitmaps concatenated at bit granularity, string offsets
        // re-based); the chunk is cut early only when these rows cannot join it: another dictionary, or string bytes beyond
        // what 32-bit offsets address
        bool fits = true;
        if ((rc = prepare_rows(x, in, done, n, &fits))) return rc;
        if (!fits) {
            if ((rc = flush_current(x))) return rc;
            continue;  // (prepared again against an empty chunk, which always fits or grows)
        }
        if ((rc = stage_rows(x, in, done, n))) return rc;
        s.held.push_back(holder);
        done += n;
        if (s.rows == x->chunk_rows && (rc = flush_current(x))) return rc;
    }
    return emit_ready(x);
}

int dfd_repartition_exec_push_device(dfd_repartition_exec* x, struct ArrowDeviceArray* batch) {
    if (!x || !batch) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_push_device: NULL argument");
    ScopedNs timed(x->ns_push);
    ArrowArray* a = &batch->array;
    auto drop = [&]() { if (a->release) a->release(a); };
    if (x->finished) { drop(); return set_error(DFD_ERR_INVALID_ARGUMENT, "push after finish/error: %s", x->error.c_str()); }
    auto refuse = [&](int code, const std::string& msg) {  // the batch is released, the operator fails (and lets go of earlier batches)
        drop();
        const int rc = fail(x, code, msg);
        if (x->input_mode == INPUT_DEVICE) release_device_inputs(x);
        return rc;
    };
    if (!launch_stage_batch || !launch_stage_sizes)  // (weak: see dfd_internal.h)
        return refuse(DFD_ERR_UNSUPPORTED, "device input: this build of the operator has no staging kernels (dfd_stage.cu)");
    if (batch->device_type != ARROW_DEVICE_CUDA || batch->device_id != (int64_t)x->ctx->device)
        return refuse(DFD_ERR_INVALID_ARGUMENT, "device batch of device type " + std::to_string((int)batch->device_type) + ", device " +
                                                    std::to_string(batch->device_id) + ": the operator takes CUDA batches of device " +
                                                    std::to_string(x->ctx->device));
    if (a->n_children != (int64_t)x->n_visible)
        return refuse(DFD_ERR_INVALID_ARGUMENT, "batch has " + std::to_string(a->n_children) + " columns, schema has " + std::to_string(x->n_visible));
    const int64_t R = a->length;
    x->rows_in += (uint64_t)R;
    if (R == 0) { drop(); return DFD_OK; }
    if (x->input_mode == INPUT_HOST)
        return refuse(DFD_ERR_INVALID_ARGUMENT, "device batch pushed to an operator that takes host batches (push / run)");
    for (int64_t i = 0; i < a->n_children; ++i)
        if (a->children[i]->length < R || (a->offset != 0))
            return refuse(DFD_ERR_INVALID_ARGUMENT, "record batch children shorter than the batch, or non-zero struct offset");
    x->input_mode = INPUT_DEVICE;
    if (batch->sync_event) {  // the staging stream waits for the producer's work; the host does not
        cudaError_t e;
        {
            std::lock_guard<std::mutex> lk(x->ctx->mu);
            e = cudaSetDevice(x->ctx->device);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(x->s_h2d, *(cudaEvent_t*)batch->sync_event, 0);
        }
        if (e != cudaSuccess) return refuse(DFD_ERR_CUDA, std::string("wait on the batch's sync_event: ") + cudaGetErrorString(e));
    }
    // ownership moves to a shared holder, as in push(): released once the chunks that read it have been emitted
    HeldInput holder = std::make_shared<SharedInput>(*a);
    a->release = nullptr;
    const ArrowArray* in = &holder->array;
    auto bail = [&](int rc) {
        release_device_inputs(x);
        return rc;
    };
    int rc = DFD_OK;
    HeldInput dicts;
    for (const FieldInfo& f : x->fields)
        if (f.dict) {
            if ((rc = host_dictionaries(x, in, &dicts))) return bail(rc);
            break;
        }
    int64_t done = 0;
    while (done < R) {
        if (!x->cur_open && (rc = open_next_slot(x))) return bail(rc);
        Slot& s = x->slots[x->cur];
        const int64_t room = x->chunk_rows - s.rows;
        if (room == 0) {
            if ((rc = flush_current(x))) return bail(rc);
            continue;
        }
        const int64_t n = R - done < room ? R - done : room;
        bool fits = true;
        if ((rc = prepare_rows_device(x, in, dicts, done, n, &fits))) return bail(rc);
        if (!fits) {
            if ((rc = flush_current(x))) return bail(rc);
            continue;
        }
        if ((rc = stage_rows_device(x, in, dicts, done, n))) return bail(rc);
        s.held.push_back(holder);
        if (dicts) s.dict_held.push_back(dicts);
        done += n;
        if (s.rows == x->chunk_rows && (rc = flush_current(x))) return bail(rc);
    }
    if ((rc = emit_ready(x))) return bail(rc);
    return DFD_OK;
}

int dfd_repartition_exec_finish(dfd_repartition_exec* x) {
    if (!x) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL exec");
    if (x->finished) return x->error_code ? set_error(x->error_code, "%s", x->error.c_str()) : DFD_OK;
    ScopedNs timed(x->ns_push);
    int rc = flush_current(x);
    if (rc) return rc;
    for (int i = 0; i < x->depth; ++i) {
        int si = (x->cur + 1 + i) % x->depth;
        if ((rc = emit_slot(x, x->slots[si]))) return rc;
    }
    {
        std::lock_guard<std::mutex> lk(x->mu);
        x->finished = true;
    }
    x->cv.notify_all();
    return DFD_OK;
}

int dfd_repartition_exec_abort(dfd_repartition_exec* x, const char* message) {
    if (!x) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL exec");
    if (x->finished) return DFD_OK;  // already finished or failed: the first outcome stands
    fail(x, DFD_ERR_INTERNAL, std::string("aborted by the producer: ") + (message ? message : "input failed"));
    if (x->input_mode == INPUT_DEVICE) release_device_inputs(x);
    return DFD_OK;
}

int dfd_repartition_exec_run(dfd_repartition_exec* x, struct ArrowArrayStream* input) {
    if (!x || !input || !input->get_next) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_run: NULL argument");
    int rc = DFD_OK;
    for (;;) {
        ArrowArray a;
        memset(&a, 0, sizeof a);
        int e = input->get_next(input, &a);
        if (e != 0) {
            const char* m = input->get_last_error ? input->get_last_error(input) : nullptr;
            rc = fail(x, DFD_ERR_INTERNAL, std::string("input stream error: ") + (m ? m : "unknown"));
            break;
        }
        if (!a.release) break;  // end of stream
        if ((rc = dfd_repartition_exec_push(x, &a))) break;
    }
    if (input->release) input->release(input);
    if (rc) return rc;
    return dfd_repartition_exec_finish(x);
}

/* ---- output streams (ArrowArrayStream per destination) ------------------- */

namespace {
struct OutStreamPriv {
    dfd_repartition_exec* x;
    uint32_t partition;
    std::string last_error;
};

int os_get_schema(ArrowArrayStream* s, ArrowSchema* out) {
    OutStreamPriv* p = (OutStreamPriv*)s->private_data;
    return export_schema(p->x->fields, out);
}

int os_get_next(ArrowArrayStream* s, ArrowArray* out) {
    OutStreamPriv* p = (OutStreamPriv*)s->private_data;
    dfd_repartition_exec* x = p->x;
    std::unique_lock<std::mutex> lk(x->mu);
    PartQueue& q = x->queues[p->partition];
    x->cv.wait(lk, [&] { return !q.batches.empty() || x->finished; });
    if (!q.batches.empty()) {
        *out = q.batches.front();
        q.batches.pop_front();
        return 0;
    }
    if (x->error_code) {  // errors fan out to every partition stream (worker_connection_pool.rs:393-397)
        p->last_error = x->error;
        return EIO;
    }
    memset(out, 0, sizeof *out);  // release == NULL: end of stream
    return 0;
}

const char* os_last_error(ArrowArrayStream* s) {
    OutStreamPriv* p = (OutStreamPriv*)s->private_data;
    return p->last_error.empty() ? nullptr : p->last_error.c_str();
}

void os_release(ArrowArrayStream* s) {
    delete (OutStreamPriv*)s->private_data;
    s->release = nullptr;
}
}  // namespace

int dfd_repartition_exec_execute(dfd_repartition_exec* x, uint32_t partition, struct ArrowArrayStream* out) {
    if (!x || !out) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_execute: NULL argument");
    if (partition >= x->N) return set_error(DFD_ERR_INVALID_ARGUMENT, "partition %u out of range [0,%u)", partition, x->N);
    OutStreamPriv* p = new (std::nothrow) OutStreamPriv{x, partition, {}};
    if (!p) return set_error(DFD_ERR_OOM, "out of host memory");
    out->get_schema = os_get_schema;
    out->get_next = os_get_next;
    out->get_last_error = os_last_error;
    out->release = os_release;
    out->private_data = p;
    return DFD_OK;
}

namespace {
struct DevExportPriv {
    std::vector<ArrowArray> children;
    std::vector<ArrowArray*> child_ptrs;
    std::vector<const void*> bufs;  // 3 per child
    const void* struct_bufs[1] = {nullptr};
    cudaEvent_t event = nullptr;
    int device = 0;
};
void dev_child_release(ArrowArray* a) { a->release = nullptr; }
void dev_export_release(ArrowArray* a) {
    DevExportPriv* p = (DevExportPriv*)a->private_data;
    for (ArrowArray& c : p->children)
        if (c.release) c.release(&c);
    if (p->event) {
        cudaSetDevice(p->device);
        cudaEventDestroy(p->event);
    }
    delete p;
    a->release = nullptr;
}
}  // namespace

int dfd_export_partition_device(dfd_ctx* ctx, const dfd_column* cols, int n_cols, int64_t first_row, int64_t n_rows,
                                struct ArrowDeviceArray* out) {
    if (!ctx || !out || n_cols < 0 || (n_cols > 0 && !cols) || first_row < 0 || n_rows < 0)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_export_partition_device: bad arguments");
    DevExportPriv* p = new (std::nothrow) DevExportPriv();
    if (!p) return set_error(DFD_ERR_OOM, "out of host memory");
    p->device = ctx->device;
    p->children.resize(n_cols);
    p->child_ptrs.resize(n_cols);
    p->bufs.resize(3 * (size_t)n_cols);
    for (int i = 0; i < n_cols; ++i) {
        const dfd_column& c = cols[i];
        ArrowArray& a = p->children[i];
        memset(&a, 0, sizeof a);
        const bool var = c.kind == DFD_COL_UTF8 || c.kind == DFD_COL_LARGE_UTF8 || c.kind == DFD_COL_BINARY;
        p->bufs[3 * i] = c.validity;
        p->bufs[3 * i + 1] = var ? c.offsets : c.values;
        p->bufs[3 * i + 2] = var ? c.values : nullptr;
        a.length = n_rows;
        a.offset = c.offset + first_row;
        a.null_count = c.validity ? -1 : 0;
        a.n_buffers = var ? 3 : 2;
        a.buffers = &p->bufs[3 * i];
        a.release = dev_child_release;
        p->child_ptrs[i] = &a;
    }
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        cudaError_t e = cudaSetDevice(ctx->device);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->event, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(p->event, ctx->stream);
        if (e != cudaSuccess) {
            if (p->event) cudaEventDestroy(p->event);
            delete p;
            return cuda_error(e, "dfd_export_partition_device");
        }
    }
    memset(out, 0, sizeof *out);
    out->array.length = n_rows;
    out->array.null_count = 0;
    out->array.n_buffers = 1;
    out->array.buffers = p->struct_bufs;
    out->array.n_children = n_cols;
    out->array.children = p->child_ptrs.data();
    out->array.release = dev_export_release;
    out->array.private_data = p;
    out->device_id = ctx->device;
    out->device_type = ARROW_DEVICE_CUDA;
    out->sync_event = &p->event;
    return DFD_OK;
}

int dfd_repartition_exec_stats(dfd_repartition_exec* x, dfd_exec_stats* out) {
    if (!x || !out) return set_error(DFD_ERR_INVALID_ARGUMENT, "NULL argument");
    std::lock_guard<std::mutex> lk(x->mu);
    out->rows_in = x->rows_in;
    out->rows_out = x->rows_out;
    out->bytes_h2d = x->bytes_h2d;
    out->bytes_d2h = x->bytes_d2h;
    out->pinned_chunks = 0;
    if (x->pool) {
        std::lock_guard<std::mutex> pl(x->pool->mu);
        out->pinned_chunks = (uint64_t)x->pool->all.size();
    }
    out->pinned_chunks_allocated = x->pool ? x->pool->n_allocated.load() : 0;
    out->pinned_chunks_reused = x->pool ? x->pool->n_reused.load() : 0;
    out->ns_push = x->ns_push;
    out->ns_wait_d2h = x->ns_wait_d2h;
    out->ns_wait_pool = x->ns_wait_pool;
    return DFD_OK;
}

}  // extern "C"
