// TEST INFRASTRUCTURE (CPU suite only): the functions csrc/dfd_exec.cu imports from the rest of the library, restated
// on the host with the CPU oracle (oracle/df_oracle.c) in place of the kernels, for the host-logic harness described in
// fake_cudart.cpp.  partition_device_locked == K1/K1b/K2/K4 (dense, stable, destination-sorted output + part_starts),
// hash_columns_locked == create_hashes over device columns, launch_lengths_to_offsets / launch_bytes_to_bits == the two
// small conversion kernels.  Pointers named "device" are host pointers here.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>
#include <atomic>
#include <chrono>

#include "dfd_b200.h"
#include "dfd_internal.h"
#include "df_oracle.h"

int harness_partition(dfd_partitioner* p, const dfd_column* in, int n_cols, int64_t n, const dfd_column* out);
int harness_destinations(dfd_partitioner* p, const dfd_column* in, int n_cols, int64_t n, std::vector<uint64_t>* hashes);

namespace {
std::atomic<uint64_t> g_ns_kernels{0};  // time spent in the stand-ins of the kernels (not host logic of the operator)
struct KernelTime {
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    ~KernelTime() { g_ns_kernels += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(); }
};
thread_local std::string g_err;
inline bool bit(const uint8_t* b, int64_t i) { return (b[i >> 3] >> (i & 7)) & 1; }
inline void set_bit(uint8_t* b, int64_t i) { b[i >> 3] = (uint8_t)(b[i >> 3] | (1u << (i & 7))); }
orc_random_state state_of(const uint64_t* seeds) {
    return seeds ? orc_state_with_seeds(seeds[0], seeds[1], seeds[2], seeds[3]) : orc_repartition_random_state();
}
}  // namespace

int dfd::set_error(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
int dfd::cuda_error(cudaError_t e, const char* what) { return set_error(DFD_ERR_CUDA, "%s: fake CUDA error %d", what, (int)e); }

int dfd::Scratch::ensure(size_t need, int) {
    if (need <= bytes) return DFD_OK;
    cudaFree(ptr);  // (the stand-in runtime: the operator releases these with cudaFree too)
    ptr = nullptr;
    bytes = 0;
    cudaError_t e = cudaMalloc(&ptr, need + need / 4 + 256);
    if (e != cudaSuccess) return cuda_error(e, "cudaMalloc(scratch)");
    bytes = need + need / 4 + 256;
    return DFD_OK;
}

int dfd::launch_lengths_to_offsets(const void* len, int ow, int64_t n, unsigned long long*, void* out_off, cudaStream_t) {
    KernelTime kernel_time;
    if (ow == 8) {
        int64_t run = 0;
        for (int64_t i = 0; i < n; ++i) { ((int64_t*)out_off)[i] = run; run += ((const int64_t*)len)[i]; }
        ((int64_t*)out_off)[n > 0 ? n : 0] = run;
    } else {
        int64_t run = 0;
        for (int64_t i = 0; i < n; ++i) { ((int32_t*)out_off)[i] = (int32_t)run; run += ((const int32_t*)len)[i]; }
        ((int32_t*)out_off)[n > 0 ? n : 0] = (int32_t)run;
    }
    return DFD_OK;
}

int dfd::launch_bytes_to_bits(const uint8_t* in, int64_t n, void* out_words, cudaStream_t) {
    KernelTime kernel_time;
    if (n <= 0) return DFD_OK;
    memset(out_words, 0, (size_t)((n + 31) / 32) * 4);
    for (int64_t i = 0; i < n; ++i)
        if (in[i]) set_bit((uint8_t*)out_words, i);
    return DFD_OK;
}

static orc_column to_orc(const dfd_column& c, int mode) {
    orc_column o{};
    o.kind = mode == DFD_KEY_HASH_INTERVAL_DAY_TIME ? ORC_INTERVAL_DAY_TIME : mode == DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO ? ORC_INTERVAL_MONTH_DAY_NANO : c.kind;
    o.width = c.width;
    o.values = c.values;
    o.offsets = c.offsets;
    o.validity = c.validity;
    o.offset = c.offset;
    return o;
}

int dfd::hash_columns_locked(Ctx*, const dfd_column* cols, int n_cols, int64_t n_rows, const uint64_t* seeds, uint64_t* hashes_device, cudaStream_t) {
    KernelTime kernel_time;
    if (!cols || n_cols < 1 || n_rows < 0 || !hashes_device) return set_error(DFD_ERR_INVALID_ARGUMENT, "hash_columns: bad arguments");
    std::vector<orc_column> oc;
    for (int i = 0; i < n_cols; ++i)  // (the operator's interval dictionary values arrive as the internal interval kinds)
        oc.push_back(to_orc(cols[i], cols[i].kind == dfd::COL_INTERVAL_DAY_TIME         ? DFD_KEY_HASH_INTERVAL_DAY_TIME
                                     : cols[i].kind == dfd::COL_INTERVAL_MONTH_DAY_NANO ? DFD_KEY_HASH_INTERVAL_MONTH_DAY_NANO
                                                                                        : DFD_KEY_HASH_PLAIN));
    const orc_random_state st = state_of(seeds);
    memset(hashes_device, 0, sizeof(uint64_t) * (size_t)n_rows);
    orc_create_hashes(oc.data(), n_cols, n_rows, &st, hashes_device);
    return DFD_OK;
}

int dfd::partition_device_locked(Partitioner* p, const dfd_column* in, int n_cols, int64_t n, const dfd_column* out, cudaStream_t, bool) {
    return harness_partition(p, in, n_cols, n, out);
}

// the stand-in of K1/K1b/K2/K4 (also used by the exchange harness, harness_exchange.cu)
// create_hashes over the key columns -> destination id of every row (h % N)
int harness_destinations(dfd_partitioner* p, const dfd_column* in, int n_cols, int64_t n, std::vector<uint64_t>* hashes) {
    using dfd::set_error;
    const orc_random_state st = orc_repartition_random_state();
    std::vector<uint64_t>& h = *hashes;
    h.assign((size_t)n, 0);
    std::vector<uint64_t> one((size_t)n);
    for (size_t k = 0; k < p->key_cols.size(); ++k) {
        if (p->key_cols[k] >= n_cols) return set_error(DFD_ERR_INVALID_ARGUMENT, "key column %d out of range", p->key_cols[k]);
        const dfd_column& c = in[p->key_cols[k]];
        const int mode = p->key_modes[k];
        if (mode == dfd::KEY_HASH_DICTIONARY) {
            const dfd_partitioner::KeyDict& d = p->key_dicts[k];
            for (int64_t i = 0; i < n; ++i) {
                const int64_t j = i + c.offset;
                if (c.validity && !bit(c.validity, j)) continue;
                int64_t idx;
                switch (c.width) {
                    case 8: idx = ((const int64_t*)c.values)[j]; break;
                    case 4: idx = d.index_unsigned ? (int64_t)((const uint32_t*)c.values)[j] : ((const int32_t*)c.values)[j]; break;
                    case 2: idx = d.index_unsigned ? (int64_t)((const uint16_t*)c.values)[j] : ((const int16_t*)c.values)[j]; break;
                    default: idx = d.index_unsigned ? (int64_t)((const uint8_t*)c.values)[j] : ((const int8_t*)c.values)[j]; break;
                }
                if (d.validity && !bit(d.validity, idx)) continue;
                h[(size_t)i] = k >= 1 ? orc_combine_hashes(d.hashes[idx], h[(size_t)i]) : d.hashes[idx];
            }
            continue;
        }
        const orc_column oc = to_orc(c, mode);
        std::fill(one.begin(), one.end(), 0);
        orc_create_hashes(&oc, 1, n, &st, one.data());  // hash_one(value) for every valid row
        for (int64_t i = 0; i < n; ++i) {
            if (c.validity && !bit(c.validity, i + c.offset)) continue;
            h[(size_t)i] = k >= 1 ? orc_combine_hashes(one[(size_t)i], h[(size_t)i]) : one[(size_t)i];
        }
    }
    return DFD_OK;
}

int harness_partition(dfd_partitioner* p, const dfd_column* in, int n_cols, int64_t n, const dfd_column* out) {
    using dfd::set_error;
    KernelTime kernel_time;
    const uint32_t N = p->N;
    std::vector<uint64_t> h;
    if (int rc = harness_destinations(p, in, n_cols, n, &h)) return rc;
    // ---- stable partition: row indices grouped by destination, in row order
    std::vector<int64_t> counts(N), starts(N + 1);
    std::vector<uint32_t> idx((size_t)(n > 0 ? n : 1));
    orc_partition_indices(h.data(), n, N, counts.data(), idx.data(), starts.data());
    memcpy(p->d_part_starts, starts.data(), sizeof(int64_t) * (N + 1));
    // ---- take, column by column
    auto gather_bits = [&](const uint8_t* src, int64_t src_off, uint8_t* dst) {
        memset(dst, 0, (size_t)((n + 31) / 32) * 4);
        for (int64_t o = 0; o < n; ++o)
            if (bit(src, (int64_t)idx[(size_t)o] + src_off)) set_bit(dst, o);
    };
    for (int ci = 0; ci < n_cols; ++ci) {
        const dfd_column& ic = in[ci];
        const dfd_column& oc = out[ci];
        if (ic.kind != oc.kind || ic.width != oc.width) return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: in/out layout mismatch", ci);
        if (ic.kind == DFD_COL_FIXED) {
            const size_t w = (size_t)ic.width;
            for (int64_t o = 0; o < n; ++o) memcpy((char*)oc.values + (size_t)o * w, (const char*)ic.values + ((size_t)idx[(size_t)o] + (size_t)ic.offset) * w, w);
        } else if (ic.kind == DFD_COL_BOOL) {
            gather_bits((const uint8_t*)ic.values, ic.offset, (uint8_t*)oc.values);
        } else {
            const bool large = ic.kind == DFD_COL_LARGE_UTF8;
            auto off_at = [&](int64_t r) -> int64_t { return large ? ((const int64_t*)ic.offsets)[r + ic.offset] : (int64_t)((const int32_t*)ic.offsets)[r + ic.offset]; };
            int64_t run = 0;
            for (int64_t o = 0; o < n; ++o) {
                const int64_t r = idx[(size_t)o], a = off_at(r), b = off_at(r + 1);
                if (large) ((int64_t*)oc.offsets)[o] = run; else ((int32_t*)oc.offsets)[o] = (int32_t)run;
                if (run + (b - a) > oc.values_bytes) return set_error(DFD_ERR_CAPACITY, "column %d: out values_bytes too small", ci);
                if (b > a) memcpy((char*)oc.values + run, (const char*)ic.values + a, (size_t)(b - a));
                run += b - a;
            }
            if (large) ((int64_t*)oc.offsets)[n] = run; else ((int32_t*)oc.offsets)[n] = (int32_t)run;
        }
        if (ic.validity) {
            if (!oc.validity) return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: input has a validity bitmap but out validity is NULL", ci);
            gather_bits(ic.validity, ic.offset, oc.validity);
        }
    }
    p->ctx->metrics.kernel_launches += 3;
    return DFD_OK;
}

extern "C" {

const char* dfd_last_error(void) { return g_err.c_str(); }

int dfd_partitioner_create(dfd_ctx* c, uint32_t num_partitions, const int32_t* key_cols, int n_keys, const uint64_t*, dfd_partitioner** out) {
    if (!c || !out) return dfd::set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_partitioner_create: NULL argument");
    *out = nullptr;
    if (num_partitions < 1 || num_partitions > DFD_MAX_PARTITIONS) return dfd::set_error(DFD_ERR_INVALID_ARGUMENT, "num_partitions %u not in [1, %u]", num_partitions, DFD_MAX_PARTITIONS);
    if (n_keys < 1 || n_keys > dfd::MAX_KEYS || !key_cols) return dfd::set_error(DFD_ERR_INVALID_ARGUMENT, "n_keys %d not in [1, %d]", n_keys, dfd::MAX_KEYS);
    dfd_partitioner* p = new dfd_partitioner();
    p->ctx = c;
    p->N = num_partitions;
    p->key_cols.assign(key_cols, key_cols + n_keys);
    p->key_modes.assign((size_t)n_keys, DFD_KEY_HASH_PLAIN);
    p->key_dicts.assign((size_t)n_keys, dfd_partitioner::KeyDict{});
    p->d_part_starts = (int64_t*)calloc(num_partitions + 1, sizeof(int64_t));
    *out = p;
    return DFD_OK;
}

void dfd_partitioner_destroy(dfd_partitioner* p) {
    if (!p) return;
    free(p->d_part_starts);
    delete p;
}

int dfd_partitioner_set_key_hash_mode(dfd_partitioner* p, int key_index, int mode) {
    if (!p || key_index < 0 || key_index >= (int)p->key_modes.size()) return dfd::set_error(DFD_ERR_INVALID_ARGUMENT, "bad key index");
    p->key_modes[(size_t)key_index] = mode;
    return DFD_OK;
}

// the harness's worker context (the product's dfd_ctx_create needs a GPU)
dfd_ctx* harness_ctx_create(void) { return new dfd_ctx(); }
void harness_ctx_destroy(dfd_ctx* c) {
    if (!c) return;
    c->pinned_cache.reset();
    delete c;
}
uint64_t harness_kernel_launches(dfd_ctx* c) { return c ? c->metrics.kernel_launches : 0; }
uint64_t harness_kernel_ns(void) { return g_ns_kernels.load(); }

}  // extern "C"
