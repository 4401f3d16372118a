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
// end-to-end time approaches max(H2D, D2H) over PCIe.  Input batches may also be
// device-resident (push_device), and an operator created for device output keeps
// its chunks on the GPU: the partition kernels write pooled DEVICE chunks in place
// and the streams carry ArrowDeviceArray slices of them (execute_device).
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
    int role = 0;  // hidden columns: 1 = lengths, 2 = bytes, 3 = element validity
    std::string child_name, child_format;
    int64_t child_flags = 0;
    int32_t child_width = 0;       // list child: 0 = Utf8 / Binary (offsets + bytes), > 0 = fixed-width primitive of that many bytes
    bool nodev() const { return list; }
    // FixedSizeList<T, n> payload (n = fsl_n): the field is the device column of its rows and carries the list's validity.
    // Its values are the child's, n x child_width bytes per row (kind FIXED), or for a Boolean child (child_width 0) n bits
    // per row (kind COL_BIT_ROWS).  A nullable child adds one hidden COL_BIT_ROWS column (h_valid): its validity, n bits per row.
    bool fsl = false;
    int32_t fsl_n = 0;
    bool dict = false;             // dictionary-encoded: `format` is the index type, dict_* describe the values
    bool dict_index_unsigned = false;  // UInt8/16/32/64 indices ("C" "S" "I" "L")
    std::string dict_format;
    int64_t dict_flags = 0;
    int32_t dict_kind = DFD_COL_FIXED, dict_width = 0;
    static bool var_kind(int32_t k) { return k == DFD_COL_UTF8 || k == DFD_COL_LARGE_UTF8 || k == DFD_COL_BINARY; }
    bool var() const { return var_kind(kind); }
    size_t ow() const { return kind == DFD_COL_LARGE_UTF8 ? 8 : 4; }  // offset width of var-width kinds
    bool dict_var() const { return var_kind(dict_kind); }             // dictionary values with offsets + bytes
    size_t dict_ow() const { return dict_kind == DFD_COL_LARGE_UTF8 ? 8 : 4; }
    int32_t dict_hash_kind() const;                                    // how the device hashes the dictionary values
};

// LargeBinary and FixedSizeBinary values are hashed by DataFusion as byte slices with a length prefix; the device hashes a
// LARGE_UTF8 column as strings and a FIXED column as an integer: such columns travel as payload but cannot be hash keys.
bool hashable_format(const char* f) { return f[0] != 'Z' && f[0] != 'w'; }

// Interval(DayTime) / Interval(MonthDayNano) values hash field by field (arrow's derived Hash), as keys and as the values of
// a dictionary key alike; everything else is one integer / byte-slice write.
int32_t interval_key_mode(const std::string& f) {
    return f == "tiD" ? DFD_KEY_HASH_INTERVAL_DAY_TIME : f == "tin" ? DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO : DFD_KEY_HASH_PLAIN;
}

int32_t FieldInfo::dict_hash_kind() const {
    const int32_t mode = interval_key_mode(dict_format);
    return mode == DFD_KEY_HASH_INTERVAL_DAY_TIME ? COL_INTERVAL_DAY_TIME : mode == DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO ? COL_INTERVAL_MONTH_DAY_NANO : dict_kind;
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

// All columns of one chunk, destination-sorted: the D2H landing buffer (pinned) of a host-output operator, or the buffers the
// partition kernels write in place (device memory) of a device-output operator.
struct OutChunk {
    bool device = false;             // device-output operator: every buffer below is device memory
    cudaEvent_t event = nullptr;     // device chunks: recorded after the last kernel that writes the chunk (the batches' sync_event)
    std::vector<void*> views;        // per column: 16-byte views of a Utf8View / BinaryView column (host chunks: built at emission)
    std::vector<int64_t> view_sizes; // per column: the "variadic buffer sizes" buffer of such an array (one data buffer) ...
    int64_t* d_view_sizes = nullptr; //   ... and where it lives for a device chunk (one int64 per column)
    std::vector<const void*> child_off, child_valid;  // per list column: offsets / validity bitmap of its values array
    std::vector<dfd::Scratch> list_tmp;  // device chunks, per list column: [child offsets | child validity bits | scan block sums]
    struct Dict {                    // device chunks, host input: the chunk's dictionary of a column, uploaded once per chunk
        dfd::Scratch mem;
        ArrowArray array;            //   (shallow: length / offset / null_count of the input's; `buffers` point into mem)
        std::vector<const void*> bufs;
    };
    std::vector<Dict> dicts;
    std::vector<std::shared_ptr<SharedInput>> inputs;  // input batches whose dictionaries this chunk's batches reference
    std::vector<void*> values;    // per column: values (fixed / bool) or string bytes (var-width, grown on demand)
    std::vector<void*> validity;  // per column (may be null)
    std::vector<void*> offsets;   // per column (var-width only)
    std::vector<size_t> data_cap; // per column: capacity of `values` for var-width columns
    std::atomic<int> refs{0};
    std::shared_ptr<PinnedPool> pool;
};

// chunk memory of either kind
cudaError_t chunk_alloc(bool device, void** p, size_t n) { return device ? cudaMalloc(p, n) : cudaHostAlloc(p, n, cudaHostAllocPortable); }
void chunk_free(bool device, void* p) {
    if (!p) return;
    if (device) cudaFree(p);
    else cudaFreeHost(p);
}

void destroy_out_chunk(OutChunk* c) {
    for (void* p : c->values) chunk_free(c->device, p);
    for (void* p : c->validity) chunk_free(c->device, p);
    for (void* p : c->offsets) chunk_free(c->device, p);
    for (void* p : c->views)
        if (c->device) cudaFree(p);
        else free(p);
    for (dfd::Scratch& t : c->list_tmp) cudaFree(t.ptr);
    for (OutChunk::Dict& d : c->dicts) cudaFree(d.mem.ptr);
    cudaFree(c->d_view_sizes);
    if (c->event) cudaEventDestroy(c->event);
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

// The operator's pool of output chunks: pinned chunks, or device chunks for a device-output operator (same bound, same counters).
struct PinnedPool : std::enable_shared_from_this<PinnedPool> {
    int device = 0;
    int64_t chunk_rows = 0;
    std::vector<FieldInfo> fields;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<OutChunk*> free_list;
    std::vector<OutChunk*> all;
    size_t max_chunks = 0;  // 0 = unbounded; otherwise acquire() blocks until a consumer returns a chunk (back-pressure)
    bool device_out = false;  // the chunks are device memory, each with its event; they are not kept past the pool (no context cache)
    std::weak_ptr<PinnedCache> cache;  // the worker context's cache (gone once the context is destroyed)
    std::string layout;                // what makes two pools' chunks interchangeable: per field kind / width / nullable / view
    std::atomic<uint64_t> n_allocated{0}, n_reused{0};  // chunks pinned by this pool / taken over from the context's cache

    static size_t value_bytes(const FieldInfo& f, int64_t rows) {
        if (f.var()) return 0;  // string bytes are sized per chunk
        if (f.kind == COL_BIT_ROWS) return bitmap_bytes(rows * f.width);
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
        c->device = device_out;
        c->child_off.assign(fields.size(), nullptr);
        c->child_valid.assign(fields.size(), nullptr);
        if (device_out) {
            c->list_tmp.resize(fields.size());
            c->dicts.resize(fields.size());
            if (cudaEventCreateWithFlags(&c->event, cudaEventDisableTiming) != cudaSuccess ||
                cudaMalloc((void**)&c->d_view_sizes, sizeof(int64_t) * fields.size()) != cudaSuccess) {
                destroy_out_chunk(c);
                return nullptr;
            }
        }
        // (device chunks are what the scatter kernels write: sized like the slot's own output buffers of a host-output operator)
        const size_t pad = device_out ? 8 : 0;
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
            void* vw = nullptr;
            const size_t vpad = device_out ? 16 * (size_t)(f.width ? f.width : 1) : 0;
            if (!f.var() && chunk_alloc(device_out, &v, value_bytes(f, chunk_rows) + vpad) != cudaSuccess) ok = false;
            if (ok && (f.flags & ARROW_FLAG_NULLABLE) && chunk_alloc(device_out, &b, bitmap_bytes(chunk_rows) + pad) != cudaSuccess) ok = false;
            if (ok && f.var() && chunk_alloc(device_out, &o, (size_t)(chunk_rows + 16) * f.ow()) != cudaSuccess) ok = false;
            if (ok && f.view) {
                if (!device_out) vw = malloc((size_t)(chunk_rows + 16) * 16);
                else if (cudaMalloc(&vw, (size_t)(chunk_rows + 16) * 16) != cudaSuccess) ok = false;
            }
            if (!ok) {  // free what this chunk already holds: nothing leaks on a failed allocation
                chunk_free(device_out, v);
                chunk_free(device_out, b);
                chunk_free(device_out, o);
                destroy_out_chunk(c);
                return nullptr;
            }
            c->values.push_back(v);
            c->validity.push_back(b);
            c->offsets.push_back(o);
            c->data_cap.push_back(0);
            c->views.push_back(vw);
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
        if (p->fields[i].list || p->fields[i].fsl) {
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

struct VarPrep {  // rows of one variable-width device column as they will be staged: the first source offset and the
    int64_t first = 0;  // byte count (lists and views are staged from zero-based offsets built for them)
    int64_t nbytes = 0;
};

struct Span {  // what rows [lo, lo + n) of a visible variable-width field span in its buffers
    int64_t first = 0, last = 0;              // offsets at lo and lo + n (lists: element offsets; views: 0 and the byte total)
    int64_t child_first = 0, child_last = 0;  // lists of strings: the child offsets at those elements
};

struct FieldTmp {  // per field: the rows being staged
    std::vector<char> off, bytes;  // host input: offsets / bytes built for a view field or a hidden list column
    VarPrep prep;                  // variable-width device columns
    Span span;                     // visible variable-width and list fields
    dfd::Scratch view_dev;         // view fields, device input: [lengths | offsets | scan block sums | data buffer table]
};

struct DictId {  // identity of a dictionary: values buffer, offset, length
    const void* p = nullptr;
    int64_t offset = 0, length = 0;
    bool operator==(const DictId& o) const { return p == o.p && offset == o.offset && length == o.length; }
};

struct SlotCol {  // one field of a slot
    void *d_in = nullptr, *d_in_valid = nullptr, *d_out = nullptr, *d_out_valid = nullptr;  // device buffers
    void *d_in_off = nullptr, *d_out_off = nullptr;  // var-width: offsets buffers
    size_t in_cap = 0, out_cap = 0;                  // var-width: capacity of d_in / d_out (string bytes)
    int64_t data_bytes = 0;                          // var-width: byte count of the chunk
    uint8_t *h_valid = nullptr, *h_bool = nullptr;   // pinned, allocated on first use: the chunk's validity / boolean bitmaps,
                                                     //   concatenated on the host at bit granularity (bit r = row r of the chunk)
    char* h_off = nullptr;                           // pinned: the chunk's var-width offsets, re-based onto the chunk's byte buffer
    bool has_valid = false;
    DictId dict_id;                                  // dictionary fields: identity of the chunk's dictionary
    dfd::Scratch list_tmp;                           // list fields: [child offsets | child validity bits | scan block sums] (device)
    dfd::Scratch dict_buf;                           // dictionary KEY fields: [hashes | offsets | data | validity] of the values
    const uint64_t* dict_hashes = nullptr;           //   device pointers handed to the partitioner for this chunk
    const uint8_t* dict_valid = nullptr;
};

struct Slot {
    std::vector<SlotCol> col;  // per field
    int64_t* h_part_starts = nullptr;  // pinned [N+1]
    cudaEvent_t e_h2d = nullptr, e_k = nullptr, e_d2h = nullptr;
    bool k_recorded = false, d2h_recorded = false;
    // state of the chunk currently in this slot
    int64_t rows = 0;
    OutChunk* out = nullptr;
    bool in_flight = false;
    std::vector<HeldInput> held;
    std::vector<HeldInput> dict_held;  // what the output batches' dictionaries reference: the batches in `held` (host input)
                                       //   or host copies of their dictionaries (device input); empty without dictionary fields
};

enum InputMode { INPUT_UNSET = 0, INPUT_HOST = 1, INPUT_DEVICE = 2 };

}  // namespace

struct dfd_repartition_exec {
    dfd_ctx* ctx = nullptr;
    dfd_partitioner* part = nullptr;
    std::vector<FieldInfo> fields;
    std::vector<int> key_of_field;  // index into the partitioner's key list, or -1
    size_t n_visible = 0;           // fields [0, n_visible) are the schema's columns; the rest are hidden device columns (lists)
    std::vector<int> dev_fields;    // fields that own a device column, in launch order
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
    // per field: the batch being staged (host memory is pageable: an H2D from it has been staged by the time
    // cudaMemcpyAsync returns)
    std::vector<FieldTmp> tmp;
    // the first non-empty push decides whether the operator takes host (push) or device (push_device) batches
    int input_mode = INPUT_UNSET;
    bool device_out = false;               // dfd_exec_options.device_output: chunks stay on the device, streams carry ArrowDeviceArray
    dfd::Scratch d_sizes;                  // device input: k_stage_sizes results, 4 x int64 per var-width column
    int64_t* h_sizes = nullptr;            // pinned: their read-back
    cudaEvent_t e_sizes = nullptr;
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
        ScopedNs waited(x->ns_wait_d2h);
        XCUDA(x, cudaEventSynchronize(s.e_d2h), "D2H");
    }
    OutChunk* oc = s.out;
    if (!oc->device) {
        oc->inputs = std::move(s.dict_held);  // the output batches reference the inputs' dictionaries
    } else {
        // a device batch cannot reference host memory: its dictionary is the device input batch's own (that batch lives until
        // the chunk's last batch is released), or the copy flush_current uploaded into the chunk (host input)
        oc->inputs.clear();
        if (x->input_mode == INPUT_DEVICE && !s.dict_held.empty()) oc->inputs.push_back(s.held.back());
    }
    s.held.clear();
    s.dict_held.clear();
    s.out = nullptr;
    s.in_flight = false;
    const size_t C = x->n_visible;  // the output batches carry the schema's columns; hidden list columns are folded into their list
    for (size_t c = 0; c < C; ++c) {  // (a device chunk has had this loop and the next done by k_emit_chunk)
        if (!x->fields[c].list || oc->device) continue;
        int32_t* lo32 = (int32_t*)oc->offsets[(size_t)x->fields[c].h_len];  // byte offsets into the 4-byte lengths -> element offsets
        for (int64_t r = 0; r <= s.rows; ++r) lo32[r] >>= 2;
    }
    for (size_t c = 0; c < C; ++c) {
        if (!x->fields[c].view || oc->device) continue;
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
            bool hv = s.col[c].has_valid;
            const FieldInfo& f = x->fields[c];
            if (f.list) {
                // List<Utf8>: list offsets + validity from the lengths column, values array (offsets from the device scan, bytes, validity)
                const size_t hl = (size_t)f.h_len, hb = (size_t)f.h_bytes;
                const bool lv = s.col[hl].has_valid;
                bp->child_bufs[4 * c] = lv ? oc->validity[hl] : nullptr;
                bp->child_bufs[4 * c + 1] = oc->offsets[hl];
                ArrowArray& g = bp->grand[c];
                memset(&g, 0, sizeof g);
                bp->grand_bufs[3 * c] = f.h_valid >= 0 ? oc->child_valid[c] : nullptr;
                bp->grand_bufs[3 * c + 1] = f.child_width > 0 ? oc->values[hb] : oc->child_off[c];  // primitive child: [validity, values]
                bp->grand_bufs[3 * c + 2] = oc->values[hb];
                g.length = s.col[hl].data_bytes / 4;
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
            if (f.fsl) {
                // FixedSizeList: a zero-copy slice of the parent (its validity) over the chunk-wide child, whose element
                // (start + i) x n starts row i of the slice
                bp->child_bufs[4 * c] = hv ? oc->validity[c] : nullptr;
                ArrowArray& g = bp->grand[c];
                memset(&g, 0, sizeof g);
                bp->grand_bufs[3 * c] = f.h_valid >= 0 ? oc->values[(size_t)f.h_valid] : nullptr;
                bp->grand_bufs[3 * c + 1] = oc->values[c];
                g.length = s.rows * f.fsl_n;
                g.null_count = f.h_valid >= 0 ? -1 : 0;
                g.n_buffers = 2;
                g.buffers = &bp->grand_bufs[3 * c];
                g.release = child_release;
                bp->grand_ptrs[c] = &g;
                a.length = cnt;
                a.offset = start;
                a.null_count = hv ? -1 : 0;
                a.n_buffers = 1;
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
            bp->child_bufs[4 * c + 3] = !f.view ? nullptr : oc->device ? (const void*)(oc->d_view_sizes + c) : (const void*)&oc->view_sizes[c];
            a.length = cnt;
            a.offset = start;  // zero-copy slice of the chunk-wide destination-sorted buffer
            a.null_count = hv ? -1 : 0;
            a.n_buffers = f.view ? 4 : (var ? 3 : 2);  // view arrays: validity, views, one data buffer, variadic buffer sizes
            a.buffers = &bp->child_bufs[4 * c];
            a.release = child_release;
            if (f.dict && (!oc->inputs.empty() || oc->device)) {
                // the dictionary travels by reference: a shallow copy of the input batch's dictionary, kept alive by the shared
                // input — or of the chunk's own uploaded copy, kept alive by the chunk
                const ArrowArray* src = !oc->inputs.empty() ? oc->inputs.back()->array.children[c]->dictionary : &oc->dicts[c].array;
                bp->dicts[c] = *src;
                bp->dicts[c].release = dict_release;
                bp->dicts[c].private_data = nullptr;
                if (!oc->inputs.empty()) bp->dict_owner.push_back(oc->inputs.back());
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
        {
            std::lock_guard<std::mutex> lk(x->mu);
            x->queues[p].batches.push_back(top);
            x->rows_out += (uint64_t)cnt;
        }
    }
    chunk_unref(oc);  // drop the guard (returns the chunk to the pool if nothing was emitted)
    x->cv.notify_all();
    return DFD_OK;
}

// bytes of the values [0, offset + length) of dictionary `d`, which is in host memory
size_t dict_value_bytes(const FieldInfo& f, const ArrowArray* d) {
    const int64_t dn = d->offset + d->length;
    if (f.dict_kind == DFD_COL_BOOL) return (size_t)((dn + 7) / 8);
    if (!f.dict_var()) return (size_t)dn * f.dict_width;
    return (size_t)(f.dict_ow() == 8 ? ((const int64_t*)d->buffers[1])[dn] : ((const int32_t*)d->buffers[1])[dn]);
}

// the string bytes of column i of a chunk need room for nb bytes (the buffer is never NULL, even for 0 bytes)
int grow_chunk_bytes(dfd_repartition_exec* x, OutChunk* oc, size_t i, size_t nb) {
    if (oc->data_cap[i] >= nb && oc->values[i]) return DFD_OK;
    chunk_free(oc->device, oc->values[i]);
    oc->values[i] = nullptr;
    oc->data_cap[i] = 0;
    const size_t want = (nb + nb / 4 + 64 + 15) & ~(size_t)15;
    XCUDA(x, chunk_alloc(oc->device, &oc->values[i], want), "chunk allocation (string bytes)");
    oc->data_cap[i] = want;
    return DFD_OK;
}

// Device output, host input: every buffer of dictionary `d` (host memory) of column i goes to memory the chunk owns, once per
// chunk, on the H2D stream.  Caller holds the context lock.
int upload_dictionary(dfd_repartition_exec* x, OutChunk* oc, size_t i, const ArrowArray* d) {
    const FieldInfo& f = x->fields[i];
    const int64_t dn = d->offset + d->length, nbuf = d->n_buffers;
    const bool view = f.dict_format[0] == 'v', dvar = !view && f.dict_var();
    if (nbuf < (view || dvar ? 3 : 2) || !d->buffers || !d->buffers[1])
        return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": malformed dictionary");
    std::vector<size_t> nb((size_t)nbuf, 0);
    if (d->null_count != 0 && d->buffers[0]) nb[0] = (size_t)((dn + 7) / 8);
    nb[1] = f.dict_kind == DFD_COL_BOOL ? (size_t)((dn + 7) / 8) : view ? (size_t)dn * 16 : dvar ? (size_t)(dn + 1) * f.dict_ow() : (size_t)dn * f.dict_width;
    if (dvar) nb[2] = dict_value_bytes(f, d);
    if (view) {  // the variadic data buffers and, last, their sizes (on the device too)
        for (int64_t k = 0; k + 3 < nbuf; ++k) nb[(size_t)k + 2] = (size_t)((const int64_t*)d->buffers[nbuf - 1])[k];
        nb[(size_t)nbuf - 1] = (size_t)(nbuf - 3) * 8;
    }
    auto al = [](size_t v) { return (v + 16 + 255) & ~(size_t)255; };
    size_t total = 0;
    for (size_t n : nb) total += al(n);
    OutChunk::Dict& od = oc->dicts[i];
    if (int rc = od.mem.ensure(total, x->ctx->device)) return fail(x, rc, dfd_last_error());
    od.bufs.assign((size_t)nbuf, nullptr);
    char* at = (char*)od.mem.ptr;
    for (size_t k = 0; k < (size_t)nbuf; at += al(nb[k]), ++k) {
        if (!d->buffers[k] || (k == 0 && !nb[0])) continue;
        if (nb[k]) XCUDA(x, cudaMemcpyAsync(at, d->buffers[k], nb[k], cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary");
        x->bytes_h2d += nb[k];
        od.bufs[k] = at;
    }
    od.array = *d;
    od.array.buffers = od.bufs.data();
    return DFD_OK;
}

// run the kernels + D2H for the chunk accumulated in the current slot (device output: the kernels write the chunk in place)
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
        ScopedNs waited(x->ns_wait_pool);
        s.out = x->pool->acquire();
    }
    if (!s.out) return fail(x, DFD_ERR_OOM, x->device_out ? "device chunk allocation failed" : "pinned host allocation failed");
    OutChunk* oc = s.out;
    const bool dev = oc->device;
    std::lock_guard<std::mutex> lk(c->mu);
    XCUDA(x, cudaSetDevice(c->device), "cudaSetDevice");
    if (dev) {
        for (int fi : x->dev_fields)  // the scatter kernels write the chunk's own buffers: room for the string bytes first
            if (x->fields[(size_t)fi].var())
                if (int rc = grow_chunk_bytes(x, oc, (size_t)fi, (size_t)s.col[(size_t)fi].data_bytes)) return rc;
        for (size_t i = 0; i < x->n_visible && x->input_mode == INPUT_HOST; ++i)
            if (x->fields[i].dict && !s.dict_held.empty())
                if (int rc = upload_dictionary(x, oc, i, s.dict_held.back()->array.children[i]->dictionary)) return rc;
    }
    for (int fi : x->dev_fields) {  // the buffers concatenated on the host while staging: bitmaps and re-based offsets
        if (x->input_mode == INPUT_DEVICE) break;  // (device input: k_stage_batch built them in place)
        const FieldInfo& f = x->fields[(size_t)fi];
        SlotCol& sc = s.col[(size_t)fi];
        const size_t bm = (size_t)((s.rows + 7) / 8);
        if (sc.has_valid) {
            XCUDA(x, cudaMemcpyAsync(sc.d_in_valid, sc.h_valid, bm, cudaMemcpyHostToDevice, x->s_h2d), "H2D validity");
            x->bytes_h2d += bm;
        }
        if (f.kind == DFD_COL_BOOL || f.kind == COL_BIT_ROWS) {
            const size_t nb = f.kind == DFD_COL_BOOL ? bm : (size_t)((s.rows * f.width + 7) / 8);
            XCUDA(x, cudaMemcpyAsync(sc.d_in, sc.h_bool, nb, cudaMemcpyHostToDevice, x->s_h2d), "H2D boolean values");
            x->bytes_h2d += nb;
        }
        if (f.var()) {
            XCUDA(x, cudaMemcpyAsync(sc.d_in_off, sc.h_off, (size_t)(s.rows + 1) * f.ow(), cudaMemcpyHostToDevice, x->s_h2d), "H2D offsets");
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
        const SlotCol& sc = s.col[i];
        // where the scatter kernels write: the slot's output buffers (copied to the pinned chunk below), or the device chunk itself
        void* o_values = dev ? oc->values[i] : sc.d_out;
        uint8_t* o_valid = !sc.has_valid ? nullptr : (uint8_t*)(dev ? oc->validity[i] : sc.d_out_valid);
        if (f.var()) {
            // (values_bytes = the bytes staged into this chunk: the offsets were built here, so the partitioner need not read them back)
            in[k] = dfd_column{f.kind, 0, sc.d_in, sc.d_in_off, sc.has_valid ? (uint8_t*)sc.d_in_valid : nullptr, 0, sc.data_bytes};
            out[k] = dfd_column{f.kind, 0, o_values, dev ? oc->offsets[i] : sc.d_out_off, o_valid, 0, (int64_t)(dev ? oc->data_cap[i] : sc.out_cap)};
        } else {
            in[k] = dfd_column{f.kind, f.width, sc.d_in, nullptr, sc.has_valid ? (uint8_t*)sc.d_in_valid : nullptr, 0, 0};
            out[k] = dfd_column{f.kind, f.width, o_values, nullptr, o_valid, 0, 0};
        }
        if (f.kind == DFD_COL_BOOL)
            XCUDA(x, cudaMemsetAsync(o_values, 0, PinnedPool::bitmap_bytes(s.rows), c->stream), "memset");
        if (sc.has_valid) XCUDA(x, cudaMemsetAsync(o_valid, 0, PinnedPool::bitmap_bytes(s.rows), c->stream), "memset");
    }
    for (size_t i = 0; i < C; ++i)  // dictionary keys of this chunk (caller holds the context lock: set the fields directly)
        if (x->fields[i].dict && x->key_of_field[i] >= 0) {
            x->part->key_modes[(size_t)x->key_of_field[i]] = dfd::KEY_HASH_DICTIONARY;
            x->part->key_dicts[(size_t)x->key_of_field[i]] = dfd_partitioner::KeyDict{s.col[i].dict_hashes, s.col[i].dict_valid, x->fields[i].dict_index_unsigned};
        }
    int rc = partition_device_locked(x->part, in.data(), (int)D, s.rows, out.data(), c->stream, /*var_bytes_known=*/true);
    if (rc) return fail(x, rc, dfd_last_error());
    // list fields: child offsets = exclusive scan of the gathered element lengths; child validity bytes -> bitmap
    std::vector<const void*> d2h_src(C, nullptr);
    std::vector<size_t> d2h_nb(C, 0);
    auto scattered = [&](int field) -> void* { return dev ? oc->values[(size_t)field] : s.col[(size_t)field].d_out; };
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        if (!f.list) continue;
        const int64_t ne = s.col[(size_t)f.h_len].data_bytes / 4;
        auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
        const size_t o_off = 0, o_bits = al((size_t)(ne + 1) * 4 + 16), o_sums = o_bits + al((size_t)(ne + 63) / 64 * 8 + 16);
        const size_t total = o_sums + al((size_t)(ne / 2048 + 4) * 8);
        dfd::Scratch& tmp = dev ? oc->list_tmp[i] : s.col[i].list_tmp;  // (a device chunk's batches point into it)
        int rc2 = tmp.ensure(total, c->device);
        if (rc2) return fail(x, rc2, dfd_last_error());
        char* lt = (char*)tmp.ptr;
        if (dev) {
            oc->child_off[i] = lt + o_off;
            oc->child_valid[i] = lt + o_bits;
        }
        if (f.child_width > 0) {  // primitive child: no child offsets; the gathered lengths themselves are not needed on the host
            d2h_src[(size_t)f.h_len] = lt + o_off;
            d2h_nb[(size_t)f.h_len] = 0;
        } else {
            if ((rc2 = launch_lengths_to_offsets(scattered(f.h_len), 4, ne, (unsigned long long*)(lt + o_sums), lt + o_off, c->stream)))
                return fail(x, rc2, dfd_last_error());
            d2h_src[(size_t)f.h_len] = lt + o_off;
            d2h_nb[(size_t)f.h_len] = (size_t)(ne + 1) * 4;
        }
        if (f.h_valid >= 0) {
            if ((rc2 = launch_bytes_to_bits((const uint8_t*)scattered(f.h_valid), ne, lt + o_bits, c->stream))) return fail(x, rc2, dfd_last_error());
            d2h_src[(size_t)f.h_valid] = lt + o_bits;
            d2h_nb[(size_t)f.h_valid] = (size_t)((ne + 31) / 32 * 4);
        }
    }
    XCUDA(x, cudaMemcpyAsync(s.h_part_starts, x->part->d_part_starts, sizeof(int64_t) * (x->N + 1), cudaMemcpyDeviceToHost, c->stream),
          "D2H part_starts");
    XCUDA(x, cudaEventRecord(s.e_k, c->stream), "record k");
    s.k_recorded = true;
    if (dev) {
        // No D2H: what emission waits for is the copy of part_starts alone.  Views and list offsets are finished by one more
        // kernel, and the chunk's own event, recorded behind it, is what the consumers of its batches wait on.
        XCUDA(x, cudaEventRecord(s.e_d2h, c->stream), "record part_starts");
        std::vector<EmitJob> jobs;
        for (size_t i = 0; i < x->n_visible; ++i) {
            const FieldInfo& f = x->fields[i];
            EmitJob j;
            j.n = s.rows;
            if (f.view) {
                j.off = oc->offsets[i];
                j.bytes = oc->values[i];
                j.dst = oc->views[i];
                j.dst2 = oc->d_view_sizes + i;
            } else if (f.list) {
                j.op = EMIT_LIST_OFFSETS;
                j.dst = oc->offsets[(size_t)f.h_len];
            } else {
                continue;
            }
            jobs.push_back(j);
        }
        if (!jobs.empty())
            if (int rc2 = launch_emit_chunk(jobs.data(), (int)jobs.size(), c->stream)) return fail(x, rc2, dfd_last_error());
        XCUDA(x, cudaEventRecord(oc->event, c->stream), "record chunk");
        s.d2h_recorded = true;
        s.in_flight = true;
        return DFD_OK;
    }
    // D2H of the destination-sorted chunk into the pooled pinned buffer taken above
    XCUDA(x, cudaStreamWaitEvent(x->s_d2h, s.e_k, 0), "wait k");
    for (size_t k = 0; k < D; ++k) {
        const size_t i = (size_t)x->dev_fields[k];
        const FieldInfo& f = x->fields[i];
        const SlotCol& sc = s.col[i];
        size_t nb = f.kind == DFD_COL_BOOL ? (size_t)((s.rows + 7) / 8) : (size_t)s.rows * f.width;
        if (f.kind == COL_BIT_ROWS) nb = (size_t)((s.rows * f.width + 31) / 32) * 4;  // (whole words, as the gather wrote them)
        const void* src = sc.d_out;
        if (f.var()) {
            nb = (size_t)sc.data_bytes;
            if (d2h_src[i]) { src = d2h_src[i]; nb = d2h_nb[i]; }  // list columns: scanned child offsets / re-packed child validity
            if (int rc2 = grow_chunk_bytes(x, oc, i, nb)) return rc2;
            if (!f.hidden || f.role == 1) {  // (the per-row offsets of the hidden bytes / validity columns are not needed on the host)
                XCUDA(x, cudaMemcpyAsync(s.out->offsets[i], sc.d_out_off, (size_t)(s.rows + 1) * f.ow(), cudaMemcpyDeviceToHost, x->s_d2h), "D2H offsets");
                x->bytes_d2h += (size_t)(s.rows + 1) * f.ow();
            }
        }
        if (nb) XCUDA(x, cudaMemcpyAsync(s.out->values[i], src, nb, cudaMemcpyDeviceToHost, x->s_d2h), "D2H");
        x->bytes_d2h += nb;
        if (sc.has_valid) {
            XCUDA(x, cudaMemcpyAsync(s.out->validity[i], sc.d_out_valid, (size_t)((s.rows + 7) / 8), cudaMemcpyDeviceToHost, x->s_d2h), "D2H");
            x->bytes_d2h += (size_t)((s.rows + 7) / 8);
        }
    }
    for (size_t i = 0; i < x->n_visible; ++i)  // the values arrays of list columns: scanned offsets / re-packed validity, as copied above
        if (x->fields[i].list) {
            oc->child_off[i] = oc->values[(size_t)x->fields[i].h_len];
            oc->child_valid[i] = x->fields[i].h_valid >= 0 ? oc->values[(size_t)x->fields[i].h_valid] : nullptr;
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
    for (SlotCol& sc : s.col) {
        sc.has_valid = false;
        sc.data_bytes = 0;
        sc.dict_id = DictId{};
    }
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

// Does a dictionary with other buffers (`theirs`) hold the same values as the chunk's (`mine`)?  Both in host memory.
bool same_dictionary(const FieldInfo& f, const ArrowArray* mine, const ArrowArray* theirs) {
    const bool comparable = mine && f.dict_format[0] != 'v' && mine->length == theirs->length && mine->n_buffers == theirs->n_buffers &&
                            mine->length <= (1 << 16);  // (a linear comparison per batch: only worth it for small dictionaries — a batch's own)
    return comparable && dfd::host::flat_arrays_equal(mine->length, f.dict_var() ? (int)f.dict_ow() : 0,
                                                      f.dict_kind == DFD_COL_BOOL ? 0 : f.dict_width, mine->buffers, mine->offset, mine->null_count,
                                                      theirs->buffers, theirs->offset, theirs->null_count);
}

// the host waits for everything enqueued on the staging stream so far (read-backs of sizes / dictionaries of device input)
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

// The string bytes the `prep` of the fields say rows [.., + n) add: cut the chunk early (`*fits` = false) when they would
// pass what 32-bit offsets address, otherwise grow the chunk's byte buffers when they need more room.
int grow_var_bytes(dfd_repartition_exec* x, int64_t n, bool* fits) {
    Slot& s = x->slots[x->cur];
    for (int fi : x->dev_fields) {
        const FieldInfo& f = x->fields[(size_t)fi];
        SlotCol& sc = s.col[(size_t)fi];
        if (!f.var()) continue;
        const int64_t need = sc.data_bytes + x->tmp[(size_t)fi].prep.nbytes;
        if (f.ow() == 4 && need > 0x7fffffffLL) {
            if (s.rows > 0) { *fits = false; return DFD_OK; }
            return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": more than 2 GiB of string data in one chunk (use a smaller chunk_rows or LargeUtf8)");
        }
        if ((size_t)need <= sc.in_cap) continue;
        // grow the chunk's byte buffers, keeping what is already staged (the copy is ordered after the H2D appends on the same
        // stream; cudaFree waits for it).  Sized for a FULL chunk at the bytes per row seen so far, and at least doubled, so
        // that growth is rare and the following batches join the chunk instead of cutting it
        std::lock_guard<std::mutex> lk(x->ctx->mu);
        XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
        size_t want = (size_t)need + (size_t)need / 4 + 256;
        if (want < 2 * sc.in_cap) want = 2 * sc.in_cap;
        const double per_row = (double)need / (double)(s.rows + n);
        double full = per_row * (double)x->chunk_rows * 1.25;
        if (full > (double)(1ull << 30)) full = (double)(1ull << 30);
        if ((size_t)full > want) want = (size_t)full;
        if (f.ow() == 4 && want > 0x7fffffffull + 256) want = 0x7fffffffull + 256;
        void* bigger = nullptr;
        XCUDA(x, cudaMalloc(&bigger, want), "cudaMalloc(string bytes)");
        if (sc.data_bytes > 0) {
            cudaError_t ce = cudaMemcpyAsync(bigger, sc.d_in, (size_t)sc.data_bytes, cudaMemcpyDeviceToDevice, x->s_h2d);
            if (ce != cudaSuccess) {
                cudaFree(bigger);
                return fail(x, DFD_ERR_CUDA, std::string("grow string bytes: ") + cudaGetErrorString(ce));
            }
        }
        cudaFree(sc.d_in);
        cudaFree(sc.d_out);
        sc.d_in = bigger;
        sc.d_out = nullptr;
        sc.in_cap = want;
        sc.out_cap = 0;
        if (x->device_out) continue;  // (the scatter writes the chunk's own buffer, grown when the chunk is flushed)
        XCUDA(x, cudaMalloc(&sc.d_out, want), "cudaMalloc(string bytes)");
        sc.out_cap = want;
    }
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

// Host input: what rows [start, start + n) of the visible variable-width fields span, read from the batch.  View fields are
// converted to offsets + contiguous bytes here (16-byte views: len | 12 inline bytes, or len | prefix | buffer index |
// offset into one of the variadic data buffers); from then on they are ordinary Utf8 / Binary columns.
void measure_host(dfd_repartition_exec* x, const ArrowArray* b, int64_t start, int64_t n) {
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        const int64_t lo = c->offset + start;
        FieldTmp& t = x->tmp[i];
        if (f.list) {
            const int32_t* loff = (const int32_t*)c->buffers[1];
            t.span = Span{loff[lo], loff[lo + n]};
            if (f.child_width == 0 && t.span.last >= t.span.first) {  // (decreasing list offsets are refused without reading the child's)
                const ArrowArray* v = c->children[0];
                const int32_t* coff = (const int32_t*)v->buffers[1] + v->offset;
                t.span.child_first = coff[t.span.first];
                t.span.child_last = coff[t.span.last];
            }
        } else if (f.view) {
            t.off.resize((size_t)(n + 1) * 4);
            int32_t* off32 = (int32_t*)t.off.data();
            const uint8_t* views = (const uint8_t*)c->buffers[1];
            const int64_t total = dfd::host::view_offsets(views, validity_of(c), lo, n, off32);  // (-1: past 32-bit offsets)
            if (total >= 0) {
                t.bytes.resize((size_t)total + 16);
                dfd::host::view_bytes(views, c->buffers + 2, lo, n, off32, t.bytes.data());
            }
            t.span = Span{0, total};
        } else if (f.var()) {
            const void* offs = c->buffers[1];
            if (f.ow() == 4) t.span = Span{((const int32_t*)offs)[lo], ((const int32_t*)offs)[lo + n]};
            else t.span = Span{((const int64_t*)offs)[lo], ((const int64_t*)offs)[lo + n]};
        }
    }
}

// Device input: the same spans, computed by k_stage_sizes for all such fields at once and read back (one small D2H and one
// wait; never for schemas without variable-width fields).  View fields also get their lengths' scan in the device scratch.
int measure_device(dfd_repartition_exec* x, const ArrowArray* b, int64_t start, int64_t n) {
    std::vector<StageSize> jobs;
    std::vector<size_t> job_field;
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        StageSize j;
        j.lo = c->offset + start;
        j.n = n;
        j.off = c->buffers[1];
        if (f.list) {
            const ArrowArray* v = c->children[0];
            j.op = STAGE_SIZE_LIST;
            j.off2 = f.child_width > 0 ? nullptr : (const int32_t*)v->buffers[1] + v->offset;
        } else if (f.view) {
            j.op = STAGE_SIZE_VIEW;  // (j.lens: set once the field's scratch is sized, below)
            j.valid = validity_of(c);
        } else if (f.var()) {
            j.op = STAGE_SIZE_RANGE;
            j.ow = (int32_t)f.ow();
        } else {
            continue;
        }
        jobs.push_back(j);
        job_field.push_back(i);
    }
    if (jobs.empty()) return DFD_OK;
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
            if (int rc = x->tmp[job_field[k]].view_dev.ensure(vt.total, x->ctx->device)) return fail(x, rc, dfd_last_error());
            jobs[k].lens = (int32_t*)((char*)x->tmp[job_field[k]].view_dev.ptr + vt.lens);
        }
        XCUDA(x, cudaMemsetAsync(x->d_sizes.ptr, 0, nb, x->s_h2d), "memset sizes");
        int rc = launch_stage_sizes(jobs.data(), (int)jobs.size(), x->s_h2d);
        for (size_t k = 0; k < jobs.size() && !rc; ++k) {  // views: offsets = exclusive scan of the lengths
            if (jobs[k].op != STAGE_SIZE_VIEW) continue;
            const ViewTmp vt(n, b->children[job_field[k]]->n_buffers - 3);
            char* t = (char*)x->tmp[job_field[k]].view_dev.ptr;
            rc = launch_lengths_to_offsets(t + vt.lens, 4, n, (unsigned long long*)(t + vt.sums), t + vt.off, x->s_h2d);
        }
        if (rc) return fail(x, rc, dfd_last_error());
        XCUDA(x, cudaMemcpyAsync(x->h_sizes, x->d_sizes.ptr, nb, cudaMemcpyDeviceToHost, x->s_h2d), "D2H sizes");
    }
    if (int rc = wait_staging(x)) return rc;
    for (size_t k = 0; k < jobs.size(); ++k) {
        const int64_t* r = x->h_sizes + 4 * k;
        x->tmp[job_field[k]].span = jobs[k].op == STAGE_SIZE_VIEW ? Span{0, r[0]} : Span{r[0], r[1], r[2], r[3]};
    }
    return DFD_OK;
}

// Can rows [start, start + n) of `b` join the open chunk (`*fits`), and what do they add?  One pass over the columns checks
// what the schema promises and cuts the chunk at another dictionary; the spans of the variable-width fields are measured
// where the batch lives and checked here; then the chunk's byte buffers grow, or the chunk is cut when the rows' string
// bytes would pass what 32-bit offsets address.
int prepare_rows(dfd_repartition_exec* x, const ArrowArray* b, const HeldInput& dicts, int64_t start, int64_t n, bool* fits) {
    Slot& s = x->slots[x->cur];
    *fits = true;
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const ArrowArray* c = b->children[i];
        if (validity_of(c) && !(f.flags & ARROW_FLAG_NULLABLE) && c->null_count > 0)
            return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": nulls in a column the schema declares non-nullable");
        if ((f.list || f.fsl) && (c->n_children != 1 || !c->children[0]))
            return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": list array without a child");
        if (f.fsl && validity_of(c->children[0]) && !(f.child_flags & ARROW_FLAG_NULLABLE) && c->children[0]->null_count > 0)
            return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": nulls in a list child the schema declares non-nullable");
        if (!f.dict) continue;
        if (!c->dictionary) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": dictionary array without a dictionary");
        // one dictionary per chunk (it travels by reference).  A batch whose dictionary is a different OBJECT with the same
        // values (readers re-materialise the dictionary for every batch) joins the chunk and is served by the chunk's first
        // one.  Identities are those of the batch's own dictionary; values are compared in host memory (`dicts`)
        const DictId id = dict_identity(c->dictionary);
        if (s.rows == 0) {
            s.col[i].dict_id = id;
        } else if (!(s.col[i].dict_id == id)) {
            const ArrowArray* mine = !s.dict_held.empty() ? s.dict_held.front()->array.children[i]->dictionary : nullptr;
            if (!same_dictionary(f, mine, dicts->array.children[i]->dictionary)) *fits = false;
        }
    }
    if (!*fits) return DFD_OK;
    if (x->input_mode == INPUT_DEVICE) {
        if (int rc = measure_device(x, b, start, n)) return rc;
    } else {
        measure_host(x, b, start, n);
    }
    for (size_t i = 0; i < x->n_visible; ++i) {
        const FieldInfo& f = x->fields[i];
        const Span& sp = x->tmp[i].span;
        if (f.list) {
            const int64_t ne = sp.last - sp.first, cw = f.child_width;
            if (ne < 0 || (cw == 0 && sp.child_last < sp.child_first))
                return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": list offsets are not monotonic");
            if (ne * 4 > 0x7fffffffLL || ne * (cw > 0 ? cw : 1) > 0x7fffffffLL)
                return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": too many list elements in one chunk");
            x->tmp[(size_t)f.h_len].prep = VarPrep{0, ne * 4};
            x->tmp[(size_t)f.h_bytes].prep = VarPrep{0, cw > 0 ? ne * cw : sp.child_last - sp.child_first};
            if (f.h_valid >= 0) x->tmp[(size_t)f.h_valid].prep = VarPrep{0, ne};
        } else if (f.view) {
            if (sp.last < 0 || sp.last > 0x7fffffffLL) return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": more than 2 GiB of view data in one chunk");
            x->tmp[i].prep = VarPrep{0, sp.last};
        } else if (f.var()) {
            if (sp.last < sp.first) return fail(x, DFD_ERR_INVALID_ARGUMENT, "column " + f.name + ": offsets are not monotonic");
            x->tmp[i].prep = VarPrep{sp.first, sp.last - sp.first};
        }
    }
    return grow_var_bytes(x, n, fits);
}

size_t dict_hash_bytes(int64_t length) { return (size_t)(length + 1) * 8; }

// Dictionary KEY field i: hash its values once per chunk on the device (DataFusion hash_dictionary); the chunk's rows pick
// dict_hashes[index].  `values` are in device memory; the hashes go to the front of the slot's dict_buf (host input copies
// the values behind them).  Caller holds the context lock.
int hash_dictionary(dfd_repartition_exec* x, size_t i, dfd_column values, int64_t length) {
    const FieldInfo& f = x->fields[i];
    SlotCol& sc = x->slots[x->cur].col[i];
    // the validity handed to the partitioner is indexed by dictionary index (0-based): it must start at the values' first bit
    if (values.validity && values.offset != 0)
        return fail(x, DFD_ERR_UNSUPPORTED, "column " + f.name + ": sliced dictionary values with nulls are not supported yet");
    values.kind = f.dict_hash_kind();  // (interval values hash field by field, as interval keys do)
    int rc = sc.dict_buf.ensure(dict_hash_bytes(length), x->ctx->device);
    if (!rc) rc = hash_columns_locked(x->ctx, &values, 1, length, nullptr, (uint64_t*)sc.dict_buf.ptr, x->s_h2d);
    if (rc) return fail(x, rc, dfd_last_error());
    sc.dict_hashes = (const uint64_t*)sc.dict_buf.ptr;
    sc.dict_valid = values.validity;
    return DFD_OK;
}

// Host input: copy rows [start, start + n) of `b` (admitted by prepare_rows) to the end of the open chunk.  Fixed-width
// values and string bytes go to the device straight from the batch; bitmaps (validity, boolean values) and string offsets
// are concatenated on the host — bit-granular, offsets re-based onto the chunk's byte buffer — and follow when the chunk is
// flushed.  A column gets a validity bitmap from the first batch that has one (earlier rows count as valid).
int stage_rows_host(dfd_repartition_exec* x, const ArrowArray* b, const HeldInput&, int64_t start, int64_t n) {
    Slot& s = x->slots[x->cur];
    std::lock_guard<std::mutex> lk(x->ctx->mu);
    XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
    auto host_bitmap = [&](uint8_t*& p, int64_t bits_per_row = 1) -> uint8_t* {
        if (!p && cudaHostAlloc((void**)&p, PinnedPool::bitmap_bytes(x->chunk_rows * bits_per_row) + 8, cudaHostAllocPortable) != cudaSuccess) p = nullptr;
        return p;
    };
    auto stage_validity = [&](size_t i, const uint8_t* valid, int64_t lo) -> int {
        SlotCol& sc = s.col[i];
        if (!valid && !sc.has_valid) return DFD_OK;
        uint8_t* hb = host_bitmap(sc.h_valid);
        if (!hb) return fail(x, DFD_ERR_OOM, "pinned host allocation failed");
        if (!sc.has_valid) {
            append_bits(hb, 0, nullptr, 0, s.rows);
            sc.has_valid = true;
        }
        append_bits(hb, s.rows, valid, lo, n);
        return DFD_OK;
    };
    auto stage_var = [&](size_t h, const void* off, const char* bytes) -> int {  // n + 1 source offsets (from prep.first), their bytes
        SlotCol& sc = s.col[h];
        const VarPrep& p = x->tmp[h].prep;
        const int64_t delta = sc.data_bytes - p.first;
        if (x->fields[h].ow() == 4) {
            int32_t* dst = (int32_t*)sc.h_off + s.rows;
            const int32_t* src = (const int32_t*)off;
            for (int64_t r = 0; r <= n; ++r) dst[r] = (int32_t)(src[r] + delta);
        } else {
            int64_t* dst = (int64_t*)sc.h_off + s.rows;
            const int64_t* src = (const int64_t*)off;
            for (int64_t r = 0; r <= n; ++r) dst[r] = src[r] + delta;
        }
        if (p.nbytes) XCUDA(x, cudaMemcpyAsync((char*)sc.d_in + sc.data_bytes, bytes, (size_t)p.nbytes, cudaMemcpyHostToDevice, x->s_h2d), "H2D");
        sc.data_bytes += p.nbytes;
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
            // List<Utf8 / Binary / primitive> -> three hidden Binary columns: row -> its elements' int32 lengths, row -> its
            // elements' bytes (one contiguous range of the child's data), row -> one validity byte per element
            const ArrowArray* v = c->children[0];
            const int32_t* loff = (const int32_t*)c->buffers[1];
            const int32_t cw = f.child_width;
            const int64_t e0 = x->tmp[i].span.first, ne = x->tmp[i].span.last - e0;
            FieldTmp& tl = x->tmp[(size_t)f.h_len];
            FieldTmp& tb = x->tmp[(size_t)f.h_bytes];
            tl.off.resize((size_t)(n + 1) * 4);
            tb.off.resize((size_t)(n + 1) * 4);
            tl.bytes.resize((size_t)ne * 4 + 16);
            int32_t* ov32 = nullptr;
            char* dvb = nullptr;
            if (f.h_valid >= 0) {
                FieldTmp& tv = x->tmp[(size_t)f.h_valid];
                tv.off.resize((size_t)(n + 1) * 4);
                tv.bytes.resize((size_t)ne + 16);
                ov32 = (int32_t*)tv.off.data();
                dvb = tv.bytes.data();
            }
            const char* child_bytes;
            if (cw > 0) {
                dfd::host::split_list_rows_fixed(loff, cw, validity_of(v), v->offset, lo, n, (int32_t*)tl.off.data(), (int32_t*)tb.off.data(),
                                                 (int32_t*)tl.bytes.data(), ov32, dvb);
                child_bytes = (const char*)v->buffers[1] + (size_t)(v->offset + e0) * (size_t)cw;
            } else {
                dfd::host::split_list_rows(loff, (const int32_t*)v->buffers[1] + v->offset, validity_of(v), v->offset, lo, n, (int32_t*)tl.off.data(),
                                           (int32_t*)tb.off.data(), (int32_t*)tl.bytes.data(), ov32, dvb);
                child_bytes = (const char*)v->buffers[2] + x->tmp[i].span.child_first;
            }
            if ((rc2 = stage_var((size_t)f.h_len, tl.off.data(), tl.bytes.data())) || (rc2 = stage_var((size_t)f.h_bytes, tb.off.data(), child_bytes))) return rc2;
            if (f.h_valid >= 0 && (rc2 = stage_var((size_t)f.h_valid, ov32, dvb))) return rc2;
            if ((rc2 = stage_validity((size_t)f.h_len, valid, lo))) return rc2;  // the list's own validity rides on the lengths column
            continue;
        }
        if (f.fsl) {
            // FixedSizeList: the child values of the rows go to the device straight from the batch; bit rows (Boolean values,
            // child validity) are concatenated on the host like any bitmap, n bits per row
            const ArrowArray* v = c->children[0];
            const dfd::host::FslSpan sp = dfd::host::fsl_span(v->offset, lo, n, f.fsl_n, f.child_width);
            auto bit_rows = [&](size_t h, const uint8_t* src) -> int {
                uint8_t* hb = host_bitmap(s.col[h].h_bool, f.fsl_n);
                if (!hb) return fail(x, DFD_ERR_OOM, "pinned host allocation failed");
                append_bits(hb, s.rows * f.fsl_n, src, sp.first_bit, sp.n_bits);
                return DFD_OK;
            };
            if (f.kind == DFD_COL_FIXED) {
                if (sp.n_bytes) XCUDA(x, cudaMemcpyAsync((char*)s.col[i].d_in + (size_t)s.rows * f.width, (const char*)v->buffers[1] + sp.first_byte, sp.n_bytes,
                                                         cudaMemcpyHostToDevice, x->s_h2d), "H2D");
                x->bytes_h2d += sp.n_bytes;
            } else if ((rc2 = bit_rows(i, (const uint8_t*)v->buffers[1]))) {
                return rc2;
            }
            if (f.h_valid >= 0 && (rc2 = bit_rows((size_t)f.h_valid, validity_of(v)))) return rc2;  // (no bitmap: all valid)
            if ((rc2 = stage_validity(i, valid, lo))) return rc2;
            continue;
        }
        if (f.dict && x->key_of_field[i] >= 0 && s.rows == 0) {
            // dictionary KEY: its values go to the device, behind the room for their hashes
            const ArrowArray* d = c->dictionary;
            const int64_t dn = d->offset + d->length;
            const uint8_t* dvalid = validity_of(d);
            const size_t nb_off = f.dict_var() ? (size_t)(dn + 1) * f.dict_ow() : 0, vbytes = dict_value_bytes(f, d);
            auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
            const size_t o_off = al(dict_hash_bytes(d->length)), o_data = o_off + al(nb_off);
            const size_t o_valid = o_data + al(vbytes + 16), total = o_valid + al((size_t)((dn + 7) / 8) + 16);
            if ((rc2 = s.col[i].dict_buf.ensure(total, x->ctx->device))) return fail(x, rc2, dfd_last_error());
            char* db = (char*)s.col[i].dict_buf.ptr;
            if (nb_off) XCUDA(x, cudaMemcpyAsync(db + o_off, d->buffers[1], nb_off, cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary offsets");
            if (vbytes) XCUDA(x, cudaMemcpyAsync(db + o_data, d->buffers[f.dict_var() ? 2 : 1], vbytes, cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary values");
            if (dvalid) XCUDA(x, cudaMemcpyAsync(db + o_valid, dvalid, (size_t)((dn + 7) / 8), cudaMemcpyHostToDevice, x->s_h2d), "H2D dictionary validity");
            x->bytes_h2d += vbytes + nb_off;
            const dfd_column dc{f.dict_kind, f.dict_width, db + o_data, nb_off ? db + o_off : nullptr, dvalid ? (uint8_t*)(db + o_valid) : nullptr, d->offset,
                                (int64_t)vbytes};
            if ((rc2 = hash_dictionary(x, i, dc, d->length))) return rc2;
        }
        if (f.view) {
            if ((rc2 = stage_var(i, x->tmp[i].off.data(), x->tmp[i].bytes.data()))) return rc2;
        } else if (f.var()) {
            if ((rc2 = stage_var(i, (const char*)c->buffers[1] + (size_t)lo * f.ow(), (const char*)c->buffers[2] + x->tmp[i].prep.first))) return rc2;
        } else if (f.kind == DFD_COL_FIXED) {
            const char* src = (const char*)c->buffers[1] + (size_t)lo * f.width;
            char* dst = (char*)s.col[i].d_in + (size_t)s.rows * f.width;
            XCUDA(x, cudaMemcpyAsync(dst, src, (size_t)n * f.width, cudaMemcpyHostToDevice, x->s_h2d), "H2D");
            x->bytes_h2d += (size_t)n * f.width;
        } else {  // boolean values: one more bitmap
            uint8_t* hb = host_bitmap(s.col[i].h_bool);
            if (!hb) return fail(x, DFD_ERR_OOM, "pinned host allocation failed");
            append_bits(hb, s.rows, (const uint8_t*)c->buffers[1], lo, n);
        }
        if ((rc2 = stage_validity(i, valid, lo))) return rc2;
    }
    s.rows += n;
    return DFD_OK;
}

// Device input: append rows [start, start + n) of the device batch `b` to the open chunk — every buffer of every column in
// ONE k_stage_batch launch (plus a small H2D of the data buffer table of each view column).
int stage_rows_device(dfd_repartition_exec* x, const ArrowArray* b, const HeldInput& dicts, int64_t start, int64_t n) {
    Slot& s = x->slots[x->cur];
    std::lock_guard<std::mutex> lk(x->ctx->mu);
    XCUDA(x, cudaSetDevice(x->ctx->device), "cudaSetDevice");
    std::vector<StageJob> jobs;
    auto validity = [&](size_t i, const uint8_t* valid, int64_t lo) {
        SlotCol& sc = s.col[i];
        if (!valid && !sc.has_valid) return;
        StageJob j;
        j.op = STAGE_BITS;
        j.src = valid;
        j.a = lo;
        j.dst = sc.d_in_valid;
        j.b = s.rows;
        j.c = sc.has_valid ? s.rows : 0;  // the first batch with a validity bitmap: earlier rows of the chunk count as valid
        j.n = n;
        sc.has_valid = true;
        jobs.push_back(j);
    };
    auto offsets = [&](size_t h, const void* src, int ow_in, int64_t scale) {
        StageJob j;
        j.op = STAGE_OFFSETS;
        j.src = src;
        j.ow_in = ow_in;
        j.ow_out = (int32_t)x->fields[h].ow();
        j.dst = (char*)s.col[h].d_in_off + (size_t)s.rows * x->fields[h].ow();
        j.n = n;
        j.base = s.col[h].data_bytes;
        j.scale = scale;
        return j;
    };
    auto bytes = [&](size_t h, StageJob j) {  // (after the column's offsets job, which takes the old byte count as its base)
        j.dst = (char*)s.col[h].d_in + s.col[h].data_bytes;
        jobs.push_back(j);
        s.col[h].data_bytes += x->tmp[h].prep.nbytes;
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
            const int64_t e0 = x->tmp[i].span.first, ne = x->tmp[i].span.last - e0, cw = f.child_width;
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
            cp.src = cw > 0 ? (const char*)v->buffers[1] + (size_t)(v->offset + e0) * (size_t)cw : (const char*)v->buffers[2] + x->tmp[i].span.child_first;
            cp.n = x->tmp[hb].prep.nbytes;
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
        if (f.fsl) {
            // FixedSizeList: one copy of the rows' child values, or bitmap appends of n bits per row (Boolean values, child validity)
            const ArrowArray* v = c->children[0];
            const dfd::host::FslSpan sp = dfd::host::fsl_span(v->offset, lo, n, f.fsl_n, f.child_width);
            auto bit_rows = [&](size_t h, const void* src) {
                StageJob bj;
                bj.op = STAGE_BITS;
                bj.src = src;
                bj.a = sp.first_bit;
                bj.dst = s.col[h].d_in;
                bj.b = bj.c = s.rows * f.fsl_n;
                bj.n = sp.n_bits;
                jobs.push_back(bj);
            };
            if (f.kind == DFD_COL_FIXED) {
                StageJob cp;
                cp.src = (const char*)v->buffers[1] + sp.first_byte;
                cp.dst = (char*)s.col[i].d_in + (size_t)s.rows * f.width;
                cp.n = (int64_t)sp.n_bytes;
                jobs.push_back(cp);
            } else {
                bit_rows(i, v->buffers[1]);
            }
            if (f.h_valid >= 0) bit_rows((size_t)f.h_valid, validity_of(v));  // (no bitmap: all valid)
            validity(i, valid, lo);
            continue;
        }
        if (f.dict && x->key_of_field[i] >= 0 && s.rows == 0) {
            // dictionary KEY: hash the device-resident values in place (the first batch of the chunk stays held until its D2H
            // is done); the host copy gives the byte count of string values
            const ArrowArray* d = c->dictionary;
            const dfd_column dc{f.dict_kind, f.dict_width, (void*)d->buffers[f.dict_var() ? 2 : 1], f.dict_var() ? (void*)d->buffers[1] : nullptr,
                                (uint8_t*)validity_of(d), d->offset, (int64_t)dict_value_bytes(f, dicts->array.children[i]->dictionary)};
            if (int rc = hash_dictionary(x, i, dc, d->length)) return rc;
        }
        if (f.view) {
            // Utf8View / BinaryView: lengths and their scan came with the sizes; the data buffer table goes to the device
            const int64_t nbuf = c->n_buffers - 3;  // (validity, views, data buffers..., variadic sizes: the sizes are not read)
            const ViewTmp vt(n, nbuf);
            char* t = (char*)x->tmp[i].view_dev.ptr;
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
            cp.src = (const char*)c->buffers[2] + x->tmp[i].prep.first;
            cp.n = x->tmp[i].prep.nbytes;
            bytes(i, cp);
        } else if (f.kind == DFD_COL_FIXED) {
            StageJob cp;
            cp.src = (const char*)c->buffers[1] + (size_t)lo * f.width;
            cp.dst = (char*)s.col[i].d_in + (size_t)s.rows * f.width;
            cp.n = n * f.width;
            jobs.push_back(cp);
        } else {  // boolean values: one more bitmap
            StageJob bv;
            bv.op = STAGE_BITS;
            bv.src = c->buffers[1];
            bv.a = lo;
            bv.dst = s.col[i].d_in;
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
                const bool dvar = !view && f.dict_var();
                const size_t dow = f.dict_ow();
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

// The device and pinned buffers of one pipeline slot: offsets and bitmaps for a full chunk now, string bytes on demand
// (caller holds the context lock).  A device-output operator has no d_out* buffers: its scatter writes the chunk.  free_slot frees whatever it holds.
cudaError_t alloc_slot(const dfd_repartition_exec* x, Slot& s) {
    s.col.resize(x->fields.size());
    const size_t bitmap = PinnedPool::bitmap_bytes(x->chunk_rows) + 8;
    for (size_t i = 0; i < x->fields.size(); ++i) {
        const FieldInfo& f = x->fields[i];
        SlotCol& sc = s.col[i];
        if (f.nodev()) continue;  // list placeholder: its rows live in the hidden columns
        cudaError_t e;
        if (f.var()) {
            const size_t ob = (size_t)(x->chunk_rows + 16) * f.ow();
            e = cudaMalloc(&sc.d_in_off, ob);
            if (e == cudaSuccess) e = cudaHostAlloc((void**)&sc.h_off, ob, cudaHostAllocPortable);
            if (e == cudaSuccess && !x->device_out) e = cudaMalloc(&sc.d_out_off, ob);
        } else {
            const size_t vb = PinnedPool::value_bytes(f, x->chunk_rows) + 16 * (size_t)(f.width ? f.width : 1);
            e = cudaMalloc(&sc.d_in, vb);
            if (e == cudaSuccess && !x->device_out) e = cudaMalloc(&sc.d_out, vb);
        }
        if (e == cudaSuccess && (f.flags & ARROW_FLAG_NULLABLE)) {
            e = cudaMalloc(&sc.d_in_valid, bitmap);
            if (e == cudaSuccess && !x->device_out) e = cudaMalloc(&sc.d_out_valid, bitmap);
        }
        if (e != cudaSuccess) return e;
    }
    cudaError_t e = cudaHostAlloc((void**)&s.h_part_starts, sizeof(int64_t) * (x->N + 1), cudaHostAllocPortable);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.e_h2d, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.e_k, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.e_d2h, cudaEventDisableTiming);
    return e;
}

void free_slot(dfd_repartition_exec* x, Slot& s) {  // (caller holds the context lock, the streams are idle)
    s.held.clear();
    s.dict_held.clear();
    if (s.out) { s.out->refs.store(1); s.out->pool = x->pool; chunk_unref(s.out); }
    for (SlotCol& sc : s.col) {
        for (void* p : {sc.d_in, sc.d_in_valid, sc.d_out, sc.d_out_valid, sc.d_in_off, sc.d_out_off, sc.dict_buf.ptr, sc.list_tmp.ptr}) cudaFree(p);
        for (void* p : {(void*)sc.h_valid, (void*)sc.h_bool, (void*)sc.h_off})
            if (p) cudaFreeHost(p);
    }
    if (s.h_part_starts) cudaFreeHost(s.h_part_starts);
    if (s.e_h2d) cudaEventDestroy(s.e_h2d);
    if (s.e_k) cudaEventDestroy(s.e_k);
    if (s.e_d2h) cudaEventDestroy(s.e_d2h);
}

// A refused batch is released and the operator fails; a device-input operator also lets go of the batches it holds.
int refuse(dfd_repartition_exec* x, ArrowArray* a, int code, const std::string& msg) {
    if (a->release) a->release(a);
    const int rc = fail(x, code, msg);
    if (x->input_mode == INPUT_DEVICE) release_device_inputs(x);
    return rc;
}

int refuse_after_finish(dfd_repartition_exec* x, ArrowArray* a) {  // (the operator's first outcome stands)
    if (a->release) a->release(a);
    return set_error(DFD_ERR_INVALID_ARGUMENT, "push after finish/error: %s", x->error.c_str());
}

// What push and push_device share after their own checks: the checks of the batch against the schema and the operator's
// input kind, then the chunk loop.  Batches of every shape are APPENDED to the open chunk (bitmaps concatenated at bit
// granularity, string offsets re-based); the chunk is cut early only when rows cannot join it: another dictionary, or
// string bytes beyond what 32-bit offsets address.
int push_rows(dfd_repartition_exec* x, ArrowArray* a, int mode, void* sync_event) {
    if (a->n_children != (int64_t)x->n_visible)
        return refuse(x, a, DFD_ERR_INVALID_ARGUMENT, "batch has " + std::to_string(a->n_children) + " columns, schema has " + std::to_string(x->n_visible));
    const int64_t R = a->length;
    x->rows_in += (uint64_t)R;
    if (R == 0) {
        if (a->release) a->release(a);
        return DFD_OK;
    }
    if (x->input_mode != INPUT_UNSET && x->input_mode != mode)
        return refuse(x, a, DFD_ERR_INVALID_ARGUMENT, mode == INPUT_HOST ? "host batch pushed to an operator that takes device batches (push_device)"
                                                                        : "device batch pushed to an operator that takes host batches (push / run)");
    for (int64_t i = 0; i < a->n_children; ++i)
        if (a->children[i]->length < R || (a->offset != 0))
            return refuse(x, a, DFD_ERR_INVALID_ARGUMENT, "record batch children shorter than the batch, or non-zero struct offset");
    x->input_mode = mode;
    if (sync_event) {  // the staging stream waits for the producer's work; the host does not
        cudaError_t e;
        {
            std::lock_guard<std::mutex> lk(x->ctx->mu);
            e = cudaSetDevice(x->ctx->device);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(x->s_h2d, *(cudaEvent_t*)sync_event, 0);
        }
        if (e != cudaSuccess) return refuse(x, a, DFD_ERR_CUDA, std::string("wait on the batch's sync_event: ") + cudaGetErrorString(e));
    }
    // ownership of the batch moves to a shared holder: every chunk that stages rows from it keeps it alive (host input: so
    // does every output batch that references its dictionaries)
    HeldInput holder = std::make_shared<SharedInput>(*a);
    a->release = nullptr;
    const ArrowArray* in = &holder->array;
    auto bail = [&](int rc) {
        if (mode == INPUT_DEVICE) release_device_inputs(x);
        return rc;
    };
    int rc = DFD_OK;
    HeldInput dicts;  // what the output batches' dictionaries reference: the batch itself, or host copies of a device batch's
    for (const FieldInfo& f : x->fields)
        if (f.dict) {
            if (mode == INPUT_HOST) dicts = holder;
            else if ((rc = host_dictionaries(x, in, &dicts))) return bail(rc);
            break;
        }
    const auto stage_rows = mode == INPUT_HOST ? stage_rows_host : stage_rows_device;
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
        if ((rc = prepare_rows(x, in, dicts, done, n, &fits))) return bail(rc);
        if (!fits) {
            if ((rc = flush_current(x))) return bail(rc);
            continue;  // (prepared again against an empty chunk, which always fits or grows)
        }
        if ((rc = stage_rows(x, in, dicts, done, n))) return bail(rc);
        s.held.push_back(holder);
        if (dicts) s.dict_held.push_back(dicts);
        done += n;
        if (s.rows == x->chunk_rows && (rc = flush_current(x))) return bail(rc);
    }
    if ((rc = emit_ready(x))) return bail(rc);
    return DFD_OK;
}

ArrowArray& array_of(ArrowArray& a) { return a; }
ArrowArray& array_of(ArrowDeviceArray& a) { return a.array; }

// run and run_device: pull `input` to exhaustion through `push`, release it, finish
template <typename Stream, typename Batch>
int pull_stream(dfd_repartition_exec* x, Stream* input, int (*push)(dfd_repartition_exec*, Batch*)) {
    int rc = DFD_OK;
    for (;;) {
        Batch a;
        memset(&a, 0, sizeof a);
        int e = input->get_next(input, &a);
        if (e != 0) {
            const char* m = input->get_last_error ? input->get_last_error(input) : nullptr;
            rc = fail(x, DFD_ERR_INTERNAL, std::string("input stream error: ") + (m ? m : "unknown"));
            if (x->input_mode == INPUT_DEVICE) release_device_inputs(x);
            break;
        }
        if (!array_of(a).release) break;  // end of stream
        if ((rc = push(x, &a))) break;
    }
    if (input->release) input->release(input);
    if (rc) return rc;
    return dfd_repartition_exec_finish(x);
}
}  // namespace

// The chunk size of an operator created with chunk_rows = 0: 4 Mi rows, or, for a schema with a FixedSizeList column (whose
// rows can be kilobytes: an embedding), the largest multiple of 64 rows up to that whose fixed-width buffers (values, bit
// rows, bitmaps) fit FSL_CHUNK_BUDGET — what cfg-2's 4 Mi rows x 64 B hold.  Each of the pipeline's in-slots, out-slots and
// output chunks holds one such chunk.
constexpr int64_t DEFAULT_CHUNK_ROWS = 4 << 20;
constexpr int64_t FSL_CHUNK_BUDGET = (int64_t)256 << 20;

static int64_t default_chunk_rows(const std::vector<FieldInfo>& fields) {
    bool fsl = false;
    int64_t bits = 0;  // fixed-width bits per row
    for (const FieldInfo& f : fields) {
        fsl |= f.fsl;
        if (f.nodev() || f.var()) continue;
        bits += f.kind == DFD_COL_BOOL ? 1 : f.kind == COL_BIT_ROWS ? f.width : 8 * (int64_t)f.width;
        if (f.flags & ARROW_FLAG_NULLABLE) bits += 1;
    }
    if (!fsl || bits == 0) return DEFAULT_CHUNK_ROWS;
    const int64_t rows = FSL_CHUNK_BUDGET * 8 / bits / 64 * 64;
    return rows < 64 ? 64 : rows > DEFAULT_CHUNK_ROWS ? DEFAULT_CHUNK_ROWS : rows;
}

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
static bool list_child_ok(const ArrowSchema* c, int32_t* child_width) {
    if (!c->format || strcmp(c->format, "+l") != 0 || c->n_children != 1 || !c->children || !c->children[0]) return false;
    const ArrowSchema* v = c->children[0];
    if (!v->format || v->dictionary || v->n_children != 0) return false;
    int32_t k = 0, w = 0;
    if (strcmp(v->format, "u") == 0 || strcmp(v->format, "z") == 0) w = 0;
    else if (parse_format(v->format, &k, &w) && k == DFD_COL_FIXED && v->format[0] != 'w') { /* ints, floats, decimals, dates, times */ }
    else return false;
    *child_width = w;
    return true;
}

// FixedSizeList<T, n> ("+w:n", n >= 1) payload: the child is a Boolean or a fixed-width primitive that list_child_ok takes.
// Fills `f` (0 = the column is not a FixedSizeList), or refuses it naming the column.
static int fixed_size_list_child(const ArrowSchema* c, long long i, bool is_key, FieldInfo* f) {
    const char* name = c->name ? c->name : "";
    if (!c->format || strncmp(c->format, "+w:", 3) != 0) return DFD_OK;
    if (is_key) return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): FixedSizeList columns cannot be hash keys", i, name);
    char* end = nullptr;
    const long long n = strtoll(c->format + 3, &end, 10);
    if (end == c->format + 3 || *end || n < 1)
        return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): FixedSizeList format '%s' is not supported (n >= 1)", i, name, c->format);
    const ArrowSchema* v = c->n_children == 1 && c->children ? c->children[0] : nullptr;
    int32_t k = 0, w = 0;
    if (!v || !v->format || c->dictionary || v->dictionary || v->n_children != 0 || !parse_format(v->format, &k, &w) ||
        !(k == DFD_COL_BOOL || (k == DFD_COL_FIXED && v->format[0] != 'w')))
        return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): FixedSizeList child type '%s' is not supported (fixed-width primitives and Boolean only)", i,
                         name, v && v->format ? v->format : "(none)");
    if (n * (w ? w : 1) > 0x7fffffffLL) return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): FixedSizeList rows of more than 2 GiB", i, name);
    f->fsl = true;
    f->fsl_n = (int32_t)n;
    f->child_width = w;
    f->kind = k == DFD_COL_BOOL ? COL_BIT_ROWS : DFD_COL_FIXED;
    f->width = k == DFD_COL_BOOL ? (int32_t)n : (int32_t)(n * w);
    f->child_name = v->name ? v->name : "item";
    f->child_format = v->format;
    f->child_flags = v->flags;
    return DFD_OK;
}

// One column `i` of the record-batch schema: can the operator move it, and — if it is a hash key — hash it like DataFusion?
// Fills `f` with what the operator keeps of it.
static int describe_column(const ArrowSchema* c, long long i, bool is_key, FieldInfo* f) {
    const char* name = c->name ? c->name : "";
    f->name = name;
    f->format = c->format ? c->format : "";
    f->flags = c->flags;
    if (list_child_ok(c, &f->child_width)) {  // List<Utf8 / Binary / primitive>: payload only
        if (is_key) return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): list columns cannot be hash keys", i, name);
        f->list = true;
        f->kind = -1;
        f->width = 0;
        f->child_name = c->children[0]->name ? c->children[0]->name : "item";
        f->child_format = c->children[0]->format;
        f->child_flags = c->children[0]->flags;
        return DFD_OK;
    }
    if (int rc = fixed_size_list_child(c, i, is_key, f)) return rc;
    if (f->fsl) return DFD_OK;
    if (!c->format || !parse_format(c->format, &f->kind, &f->width))
        return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): Arrow format '%s' is not supported", i, name, c->format ? c->format : "(null)");
    f->view = c->format[0] == 'v';
    if (c->dictionary) {  // Dictionary<integer index, flat values>: indices are scattered, the dictionary travels by reference
        if (f->kind != DFD_COL_FIXED || !strchr("cCsSiIlL", c->format[0]) || c->format[1])
            return set_error(DFD_ERR_UNSUPPORTED, "column %lld (%s): dictionary index type '%s' is not an integer", i, name, c->format);
        const ArrowSchema* d = c->dictionary;
        f->dict = true;
        f->dict_index_unsigned = strchr("CSIL", c->format[0]) != nullptr;
        f->dict_format = d->format ? d->format : "";
        f->dict_flags = d->flags;
        if (d->dictionary || d->n_children > 0 || !d->format || !parse_format(d->format, &f->dict_kind, &f->dict_width))
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
    for (int64_t i = 0; i < schema->n_children; ++i) {
        FieldInfo f;
        if (int rc = describe_column(schema->children[i], (long long)i, false, &f)) return rc;
    }
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
        FieldInfo f;
        if (int rc = describe_column(schema->children[i], (long long)i, is_key, &f)) return rc;
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
    std::unique_ptr<dfd_repartition_exec> x(new (std::nothrow) dfd_repartition_exec());
    if (!x) return set_error(DFD_ERR_OOM, "out of host memory");
    x->ctx = ctx;
    x->N = num_partitions;
    if (opts && opts->device_output != 0 && opts->device_output != 1)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_exec_options.device_output is %d: 0 (host output) or 1 (device output)", (int)opts->device_output);
    x->device_out = opts && opts->device_output == 1;
    if (x->device_out && !launch_emit_chunk)  // (weak: see dfd_internal.h)
        return set_error(DFD_ERR_UNSUPPORTED, "device output: this build of the operator has no emit kernel (dfd_emit.cu)");
    for (int64_t i = 0; i < schema->n_children; ++i) {  // (the same rules the plan hook checks through dfd_repartition_supported)
        int key_index = -1;
        for (int k = 0; k < n_keys; ++k)
            if (key_cols && key_cols[k] == i) key_index = k;
        FieldInfo f;
        if (int rc = describe_column(schema->children[i], (long long)i, key_index >= 0, &f)) return rc;
        x->key_of_field.push_back(key_index);
        x->fields.push_back(f);
    }
    for (int k = 0; k < n_keys; ++k)
        if (!key_cols || key_cols[k] < 0 || key_cols[k] >= (int)x->fields.size())
            return set_error(DFD_ERR_INVALID_ARGUMENT, "key column index out of range");
    // hidden device columns of the list fields, appended after the visible ones
    x->n_visible = x->fields.size();
    for (size_t i = 0; i < x->n_visible; ++i) {
        if (x->fields[i].fsl && (x->fields[i].child_flags & ARROW_FLAG_NULLABLE)) {  // the child's validity: n bits per row
            FieldInfo h;
            h.name = x->fields[i].name + ".validity";
            h.format = x->fields[i].format;
            h.kind = COL_BIT_ROWS;
            h.width = x->fields[i].fsl_n;
            h.hidden = true;
            h.role = 3;
            x->key_of_field.push_back(-1);
            x->fields.push_back(h);
            x->fields[i].h_valid = (int)x->fields.size() - 1;
        }
        if (!x->fields[i].list) continue;
        auto hidden = [&](const char* tag, bool nullable) {
            FieldInfo h;
            h.name = x->fields[i].name + "." + tag;
            h.format = "z";
            h.kind = DFD_COL_BINARY;
            h.width = 0;
            h.hidden = true;
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
    std::vector<int> dev_pos(x->fields.size(), -1);  // field -> its position among the device columns
    for (size_t i = 0; i < x->fields.size(); ++i)
        if (!x->fields[i].nodev()) {
            dev_pos[i] = (int)x->dev_fields.size();
            x->dev_fields.push_back((int)i);
        }
    std::vector<int32_t> dev_keys(n_keys);
    for (int k = 0; k < n_keys; ++k) dev_keys[k] = dev_pos[(size_t)key_cols[k]];  // keys address the compact device column list
    int rc = dfd_partitioner_create(ctx, num_partitions, dev_keys.data(), n_keys, nullptr, &x->part);
    if (rc) return rc;  // (x has no CUDA resources yet; unique_ptr frees it)
    x->part->bit_rows = true;  // (FixedSizeList bit rows)
    for (int k = 0; k < n_keys; ++k) {  // interval keys hash field by field (arrow's derived Hash), not as one integer
        const int mode = interval_key_mode(x->fields[(size_t)key_cols[k]].format);  // (a dictionary field's format is its index type)
        if (mode != DFD_KEY_HASH_PLAIN && (rc = dfd_partitioner_set_key_hash_mode(x->part, k, mode))) {
            dfd_partitioner_destroy(x->part);
            x->part = nullptr;
            return rc;
        }
    }
    x->chunk_rows = (opts && opts->chunk_rows > 0) ? opts->chunk_rows : default_chunk_rows(x->fields);
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
        x->slots.resize(x->depth);
        for (Slot& s : x->slots)
            if (e == cudaSuccess) e = alloc_slot(x.get(), s);
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
    x->pool->device_out = x->device_out;
    if (!x->device_out) x->pool->cache = pinned_cache_of(ctx);
    x->pool->max_chunks = (opts && opts->max_pinned_chunks > 0) ? (size_t)opts->max_pinned_chunks : 0;
    if (x->pool->max_chunks && x->pool->max_chunks < (size_t)pool_chunks) x->pool->max_chunks = (size_t)pool_chunks;
    std::vector<OutChunk*> pre;
    for (int i = 0; i < pool_chunks; ++i) {
        OutChunk* c = x->pool->acquire();
        if (!c) {
            const bool device_out = x->device_out;
            dfd_repartition_exec_destroy(x.release());
            return set_error(DFD_ERR_OOM, device_out ? "device chunk pool allocation failed" : "pinned pool allocation failed");
        }
        pre.push_back(c);
    }
    for (OutChunk* c : pre) x->pool->give_back(c);
    x->tmp.resize(x->fields.size());
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
        for (FieldTmp& t : x->tmp) cudaFree(t.view_dev.ptr);
        if (x->h_sizes) cudaFreeHost(x->h_sizes);
        if (x->e_sizes) cudaEventDestroy(x->e_sizes);
        for (Slot& s : x->slots) free_slot(x, s);
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
    if (x->finished) return refuse_after_finish(x, batch);
    return push_rows(x, batch, INPUT_HOST, nullptr);
}

int dfd_repartition_exec_push_device(dfd_repartition_exec* x, struct ArrowDeviceArray* batch) {
    if (!x || !batch) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_push_device: NULL argument");
    ScopedNs timed(x->ns_push);
    ArrowArray* a = &batch->array;
    if (x->finished) return refuse_after_finish(x, a);
    if (!launch_stage_batch || !launch_stage_sizes)  // (weak: see dfd_internal.h)
        return refuse(x, a, DFD_ERR_UNSUPPORTED, "device input: this build of the operator has no staging kernels (dfd_stage.cu)");
    if (batch->device_type != ARROW_DEVICE_CUDA || batch->device_id != (int64_t)x->ctx->device)
        return refuse(x, a, DFD_ERR_INVALID_ARGUMENT, "device batch of device type " + std::to_string((int)batch->device_type) + ", device " +
                                                          std::to_string(batch->device_id) + ": the operator takes CUDA batches of device " +
                                                          std::to_string(x->ctx->device));
    return push_rows(x, a, INPUT_DEVICE, batch->sync_event);
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
    return pull_stream(x, input, dfd_repartition_exec_push);
}

int dfd_repartition_exec_run_device(dfd_repartition_exec* x, struct ArrowDeviceArrayStream* input) {
    if (!x || !input || !input->get_next) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_run_device: NULL argument");
    if (input->device_type != ARROW_DEVICE_CUDA) {
        const int type = (int)input->device_type;
        if (input->release) input->release(input);
        return set_error(DFD_ERR_INVALID_ARGUMENT, "device stream of device type %d: the operator takes CUDA streams", type);
    }
    return pull_stream(x, input, dfd_repartition_exec_push_device);
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

// the next batch of the stream's destination (blocking); *out is released (release == NULL) at the end of the stream
int next_batch(OutStreamPriv* p, ArrowArray* out) {
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

int os_get_next(ArrowArrayStream* s, ArrowArray* out) { return next_batch((OutStreamPriv*)s->private_data, out); }

// The device streams hand out the same queued batches, wrapped: the buffers of a device-output operator's chunks are device
// memory, and the chunk's event says when they are written.
int ds_get_schema(ArrowDeviceArrayStream* s, ArrowSchema* out) { return export_schema(((OutStreamPriv*)s->private_data)->x->fields, out); }
int ds_get_next(ArrowDeviceArrayStream* s, ArrowDeviceArray* out) {
    OutStreamPriv* p = (OutStreamPriv*)s->private_data;
    memset(out, 0, sizeof *out);
    if (int e = next_batch(p, &out->array)) return e;
    if (!out->array.release) return 0;
    out->device_id = p->x->ctx->device;
    out->device_type = ARROW_DEVICE_CUDA;
    out->sync_event = &((BatchPriv*)out->array.private_data)->chunk->event;
    return 0;
}
const char* ds_last_error(ArrowDeviceArrayStream* s) {
    OutStreamPriv* p = (OutStreamPriv*)s->private_data;
    return p->last_error.empty() ? nullptr : p->last_error.c_str();
}
void ds_release(ArrowDeviceArrayStream* s) {
    delete (OutStreamPriv*)s->private_data;
    s->release = nullptr;
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
    if (x->device_out) return set_error(DFD_ERR_INVALID_ARGUMENT, "execute on a device-output operator: its streams are taken with execute_device");
    OutStreamPriv* p = new (std::nothrow) OutStreamPriv{x, partition, {}};
    if (!p) return set_error(DFD_ERR_OOM, "out of host memory");
    out->get_schema = os_get_schema;
    out->get_next = os_get_next;
    out->get_last_error = os_last_error;
    out->release = os_release;
    out->private_data = p;
    return DFD_OK;
}

int dfd_repartition_exec_execute_device(dfd_repartition_exec* x, uint32_t partition, struct ArrowDeviceArrayStream* out) {
    if (!x || !out) return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_repartition_exec_execute_device: NULL argument");
    if (partition >= x->N) return set_error(DFD_ERR_INVALID_ARGUMENT, "partition %u out of range [0,%u)", partition, x->N);
    if (!x->device_out)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "execute_device on a host-output operator: create it with dfd_exec_options.device_output = 1");
    OutStreamPriv* p = new (std::nothrow) OutStreamPriv{x, partition, {}};
    if (!p) return set_error(DFD_ERR_OOM, "out of host memory");
    out->device_type = ARROW_DEVICE_CUDA;
    out->get_schema = ds_get_schema;
    out->get_next = ds_get_next;
    out->get_last_error = ds_last_error;
    out->release = ds_release;
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
