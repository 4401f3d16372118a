// dfd_reduce.cu — device-side PartialReduce ahead of the shuffle.
//
// The reference inserts AggregateExec(mode = PartialReduce) ABOVE the producers' hash RepartitionExec
// (src/distributed_planner/partial_reduce_below_network_shuffles.rs:17-100; plan shape tests/distributed_aggregation.rs:63-67):
// after hash repartitioning, rows with equal group keys sit in the same destination partition, so merging their
// aggregate states there shrinks what crosses the network.  Here the partitioned table is already on the GPU
// (output of dfd_partition_device), so the merge runs on it in place of a PCIe round trip:
//   k_group_insert   open-addressing table of REPRESENTATIVE ROW indices (one u32 per slot): a row claims an empty slot
//                    with atomicCAS or joins the group whose representative has equal key bytes (any number / width of
//                    fixed-width keys — the keys themselves are never copied into the table)
//   k_group_count    groups per destination partition (representatives only)      -> exclusive scan (host, N+1 values)
//   k_group_place    every group gets an output row inside its partition; key columns copied, states initialised
//   k_group_combine  every input row folds its states into its group's output row with atomics (k_combine_nullable, the
//                    same code skipping null states and setting the output bits, when a state column has a bitmap)
//                    (SUM i64 / f64 / i128 (two 64-bit adds with carry); MIN / MAX of signed and unsigned 8- to 64-bit
//                    integers, of 128-bit decimals and of f16 / f32 / f64 under totalOrder: native atomicMin / atomicMax
//                    at 32 and 64 bits, CAS loops at 8 (on the enclosing 32-bit word), 16 and 128 bits and for floats)
//   k_group_clear    only when a MIN / MAX state column has an input bitmap: zeroes the value of every such state that
//                    no valid row reached (it still holds the sentinel k_group_place started it from)
// Nullable keys and states: a null key equals a null of its column and nothing else (its bytes are never read); a null
// state is skipped, and an output state is valid when one of its group's input states is.
// Boolean and var-width (Utf8 / LargeUtf8 / Binary) keys: a call with one runs k_insert_keys / k_count_keys /
// k_place_keys in place of insert / count / place (the same bodies over a KeyParams table; the fixed-key kernels never
// see it).  Strings compare and hash by length and bytes; k_count_keys also sums the representatives' key bytes per
// column, so the host checks the output capacity at its one sync.  k_place_keys writes each group's key length into the
// output offsets (and its representative row into out_rep); then, ONE COLUMN AT A TIME, the K4 scan (k_len_block_sums,
// k_var_scan_block_sums, k_len_write_offsets) turns the lengths into offsets in place and k_copy_key_bytes copies the
// representatives' bytes.  So a call makes 4 (+1 for k_group_clear) + 4 per var-width key launches.
// Integer / byte work; random access into an L2-resident table for the cardinalities PartialReduce is used for.
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>
#include <vector>

#include "dfd_b200.h"
#include "dfd_internal.h"

using namespace dfd;

namespace {

constexpr int MAX_REDUCE_COLS = 32;
constexpr uint32_t SLOT_EMPTY = 0xffffffffu;

struct ReduceCol {
    const char* in;
    char* out;
    const uint8_t* in_valid;  // input bitmap, or NULL; row r's bit is bit in_bit + r counted from this byte
    uint32_t* out_valid;      // output bitmap (4-byte aligned), or NULL for a non-null output column
    int32_t width;
    int32_t op;  // dfd_agg_op, or -1 for a group key
    int32_t in_bit;  // 0..7
};

struct ReduceParams {
    ReduceCol col[MAX_REDUCE_COLS];
    int32_t n_cols;
    int32_t key_idx[MAX_KEYS];
    int32_t n_keys;
    int64_t n_rows;
    int64_t n_groups;       // output rows (k_group_clear only)
    uint32_t N;
    uint32_t table_mask;
    uint32_t* table;        // [table_mask + 1] representative row of every slot
    uint32_t* row_slot;     // [n_rows] slot of every row's group
    uint32_t* slot_out;     // [table_mask + 1] output row of the slot's group
    const int64_t* part_starts;  // [N+1] input partition boundaries (device)
    unsigned long long* group_count;  // [N]
    int64_t* out_starts;    // [N+1] (device)
    unsigned long long* cursor;  // [N]
};

// What a Boolean or var-width key column adds to its ReduceCol (in_valid / out_valid / in_bit stay there).
struct KeyExt {
    int32_t kind;          // dfd_col_kind; DFD_COL_FIXED: a fixed-width key, read through its ReduceCol
    int32_t bit;           // Boolean: the values' bit offset 0..7 (row r's bit is bit + r counted from `in`)
    const void* in_off;    // var-width: the input offsets from the Arrow offset on (entry r = row r's start)
    const uint8_t* in;     // var-width: the input bytes (offsets index them); Boolean: the value bitmap
    void* out_off;         // var-width: output offsets (int32 / int64 as the input's)
    uint8_t* out;          // var-width: output bytes; Boolean: output words (4-byte aligned)
};

// The launches of a call with a Boolean or var-width key: ReduceParams plus one KeyExt per column (key columns only).
struct KeyParams {
    ReduceParams P;
    KeyExt key[MAX_REDUCE_COLS];
    uint32_t* out_rep;               // [n_rows] representative row of every output row (read by k_copy_key_bytes)
    unsigned long long* key_bytes;   // [MAX_KEYS] bytes of the groups' representatives, per key (var-width keys)
};

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}

__device__ __forceinline__ bool valid_at(const ReduceCol& c, int64_t row) {
    const int64_t b = (int64_t)c.in_bit + row;
    return (c.in_valid[b >> 3] >> (b & 7)) & 1;
}

// Sets output row o's bit.  Other rows of the word belong to other groups, so the update is atomic.
__device__ __forceinline__ void set_valid(uint32_t* bits, int64_t o) { atomicOr(bits + (o >> 5), 1u << (o & 31)); }

constexpr uint64_t NULL_KEY_TAG = 0x6a09e667f3bcc909ULL;  // hashed in place of a null key's bytes

// h folded with the fixed-width key of `row` in column c, as key_hash<NULLS>(ReduceParams) does it.  (Only the KeyParams
// overload calls this: key_hash<NULLS>(ReduceParams) keeps its own copy of the switch, which compiles to the instruction
// sequence the fixed-key kernels have always had; a call to this helper there does not.)
__device__ __forceinline__ uint64_t mix_fixed(uint64_t h, const ReduceCol& c, int64_t row) {
    const char* p = c.in + row * (int64_t)c.width;
    switch (c.width) {
        case 8: h = mix64(h ^ *(const uint64_t*)p); break;
        case 4: h = mix64(h ^ *(const uint32_t*)p); break;
        case 2: h = mix64(h ^ *(const uint16_t*)p); break;
        case 1: h = mix64(h ^ *(const uint8_t*)p); break;
        default: h = mix64(mix64(h ^ ((const uint64_t*)p)[0]) ^ ((const uint64_t*)p)[1]); break;
    }
    return h;
}

__device__ __forceinline__ bool fixed_equal(const ReduceCol& c, int64_t a, int64_t b) {
    const char* pa = c.in + a * (int64_t)c.width;
    const char* pb = c.in + b * (int64_t)c.width;
    bool eq;
    switch (c.width) {
        case 8: eq = *(const uint64_t*)pa == *(const uint64_t*)pb; break;
        case 4: eq = *(const uint32_t*)pa == *(const uint32_t*)pb; break;
        case 2: eq = *(const uint16_t*)pa == *(const uint16_t*)pb; break;
        case 1: eq = *pa == *pb; break;
        default: eq = ((const uint64_t*)pa)[0] == ((const uint64_t*)pb)[0] && ((const uint64_t*)pa)[1] == ((const uint64_t*)pb)[1]; break;
    }
    return eq;
}

template <bool NULLS>
__device__ __forceinline__ uint64_t key_hash(const ReduceParams& P, int64_t row) {
    uint64_t h = 0x9e3779b97f4a7c15ULL;
    for (int k = 0; k < P.n_keys; ++k) {
        const ReduceCol& c = P.col[P.key_idx[k]];
        if (NULLS && c.in_valid && !valid_at(c, row)) {
            h = mix64(h ^ NULL_KEY_TAG);
            continue;
        }
        const char* p = c.in + row * (int64_t)c.width;
        switch (c.width) {
            case 8: h = mix64(h ^ *(const uint64_t*)p); break;
            case 4: h = mix64(h ^ *(const uint32_t*)p); break;
            case 2: h = mix64(h ^ *(const uint16_t*)p); break;
            case 1: h = mix64(h ^ *(const uint8_t*)p); break;
            default: h = mix64(mix64(h ^ ((const uint64_t*)p)[0]) ^ ((const uint64_t*)p)[1]); break;
        }
    }
    return h;
}

template <bool NULLS>
__device__ __forceinline__ bool keys_equal(const ReduceParams& P, int64_t a, int64_t b) {
    for (int k = 0; k < P.n_keys; ++k) {
        const ReduceCol& c = P.col[P.key_idx[k]];
        if (NULLS && c.in_valid) {  // a null equals a null of the same column and nothing else
            const bool va = valid_at(c, a);
            if (va != valid_at(c, b)) return false;
            if (!va) continue;
        }
        if (!fixed_equal(c, a, b)) return false;
    }
    return true;
}

// ---- Boolean and var-width keys (KeyParams) ----

__device__ __forceinline__ bool bool_at(const KeyExt& k, int64_t row) {
    const int64_t b = (int64_t)k.bit + row;
    return (k.in[b >> 3] >> (b & 7)) & 1;
}

// Start and length of row r's bytes (int64 offsets for LargeUtf8, int32 for Utf8 / Binary).
__device__ __forceinline__ int64_t var_start(const KeyExt& k, int64_t row, int64_t& len) {
    if (k.kind == DFD_COL_LARGE_UTF8) {
        const int64_t* o = (const int64_t*)k.in_off;
        len = o[row + 1] - o[row];
        return o[row];
    }
    const int32_t* o = (const int32_t*)k.in_off;
    len = (int64_t)o[row + 1] - o[row];
    return o[row];
}

// The bytes [p, p + len) as little-endian 8-byte chunks, the last one zero-padded.  Only the aligned 8-byte words that
// hold one of the bytes are loaded, and each chunk is funnel-shifted out of two of them (as k_emit_chunk reads views):
// nothing past the word of the last byte is read, whatever the address.  So equal bytes give equal chunks anywhere.
struct ByteChunks {
    const uint64_t* w;  // the aligned word that holds the next chunk's first byte
    uint64_t lo;        // *w
    int64_t left;       // bytes not yet returned
    unsigned sh;        // bit position of a chunk's first byte in its word
    __device__ __forceinline__ ByteChunks(const uint8_t* p, int64_t len)
        : w((const uint64_t*)((uintptr_t)p & ~(uintptr_t)7)), lo(0), left(len), sh(((unsigned)(uintptr_t)p & 7u) * 8u) {
        if (len > 0) lo = *w;
    }
    __device__ __forceinline__ uint64_t next() {  // (while left > 0)
        const bool more = left > (int64_t)(8u - sh / 8u);  // word w + 1 holds one of the bytes
        const uint64_t hi = more ? w[1] : 0;
        uint64_t v = sh ? (lo >> sh) | (hi << (64u - sh)) : lo;
        if (left < 8) v &= (1ULL << (8 * left)) - 1ULL;
        left -= 8;
        ++w;
        lo = hi;
        return v;
    }
};

// The length first, so "", "a" and "a\0" hash (and compare) apart, then one mix64 per 8-byte chunk.
__device__ __forceinline__ uint64_t mix_bytes(uint64_t h, const uint8_t* p, int64_t len) {
    h = mix64(h ^ (uint64_t)len);
    for (ByteChunks b(p, len); b.left > 0;) h = mix64(h ^ b.next());
    return h;
}

template <bool NULLS>
__device__ __forceinline__ uint64_t key_hash(const KeyParams& K, int64_t row) {
    const ReduceParams& P = K.P;
    uint64_t h = 0x9e3779b97f4a7c15ULL;
    for (int k = 0; k < P.n_keys; ++k) {
        const ReduceCol& c = P.col[P.key_idx[k]];
        const KeyExt& kc = K.key[P.key_idx[k]];
        if (NULLS && c.in_valid && !valid_at(c, row)) {
            h = mix64(h ^ NULL_KEY_TAG);
        } else if (kc.kind == DFD_COL_FIXED) {
            h = mix_fixed(h, c, row);
        } else if (kc.kind == DFD_COL_BOOL) {
            h = mix64(h ^ (uint64_t)bool_at(kc, row));
        } else {
            int64_t len;
            const int64_t s = var_start(kc, row, len);
            h = mix_bytes(h, kc.in + s, len);
        }
    }
    return h;
}

template <bool NULLS>
__device__ __forceinline__ bool keys_equal(const KeyParams& K, int64_t a, int64_t b) {
    const ReduceParams& P = K.P;
    for (int k = 0; k < P.n_keys; ++k) {
        const ReduceCol& c = P.col[P.key_idx[k]];
        const KeyExt& kc = K.key[P.key_idx[k]];
        if (NULLS && c.in_valid) {
            const bool va = valid_at(c, a);
            if (va != valid_at(c, b)) return false;
            if (!va) continue;
        }
        if (kc.kind == DFD_COL_FIXED) {
            if (!fixed_equal(c, a, b)) return false;
        } else if (kc.kind == DFD_COL_BOOL) {
            if (bool_at(kc, a) != bool_at(kc, b)) return false;
        } else {
            int64_t la, lb;
            const int64_t sa = var_start(kc, a, la), sb = var_start(kc, b, lb);
            if (la != lb) return false;
            ByteChunks ca(kc.in + sa, la), cb(kc.in + sb, lb);
            while (ca.left > 0)
                if (ca.next() != cb.next()) return false;
        }
    }
    return true;
}

__device__ __forceinline__ uint32_t partition_of(const int64_t* starts, uint32_t N, int64_t row) {
    uint32_t lo = 0, hi = N;  // last p with starts[p] <= row
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (starts[mid] <= row) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ const ReduceParams& reduce_params(const ReduceParams& P) { return P; }
__device__ __forceinline__ const ReduceParams& reduce_params(const KeyParams& K) { return K.P; }

// Every kernel that reads or writes bitmaps has two launches of one body: NULLS = false is the code of a call without
// them (k_group_insert / _place / _combine), NULLS = true the one of a call with them (k_*_nullable).  Insert and place
// have a third, over KeyParams with NULLS = true, for a call with a Boolean or var-width key (k_insert_keys /
// k_place_keys).
template <bool NULLS, typename Params>
__device__ __forceinline__ void insert_rows(const Params& K) {
    const ReduceParams& P = reduce_params(K);
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < P.n_rows; row += (int64_t)gridDim.x * blockDim.x) {
        uint32_t s = (uint32_t)key_hash<NULLS>(K, row) & P.table_mask;
        for (;;) {
            uint32_t rep = P.table[s];
            if (rep == SLOT_EMPTY) {
                rep = atomicCAS(P.table + s, SLOT_EMPTY, (uint32_t)row);
                if (rep == SLOT_EMPTY) break;  // this row represents a new group
            }
            if (keys_equal<NULLS>(K, (int64_t)rep, row)) break;
            s = (s + 1) & P.table_mask;
        }
        P.row_slot[row] = s;
    }
}

__global__ void __launch_bounds__(256) k_group_insert(const __grid_constant__ ReduceParams P) { insert_rows<false>(P); }
__global__ void __launch_bounds__(256) k_insert_nullable(const __grid_constant__ ReduceParams P) { insert_rows<true>(P); }
__global__ void __launch_bounds__(256) k_insert_keys(const __grid_constant__ KeyParams K) { insert_rows<true>(K); }

__global__ void __launch_bounds__(256) k_group_count(const __grid_constant__ ReduceParams P) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= (int64_t)P.table_mask; s += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t rep = P.table[s];
        if (rep != SLOT_EMPTY) atomicAdd(P.group_count + partition_of(P.part_starts, P.N, (int64_t)rep), 1ULL);
    }
}

// k_group_count, plus the key bytes of every var-width key summed over the representatives (a null adds none): each
// thread sums its slots, then one atomic per warp and key.  Every lane of a warp makes the same number of passes (the
// table's size and the grid's stride are multiples of 32), so the whole warp reaches the shuffles.
__global__ void __launch_bounds__(256) k_count_keys(const __grid_constant__ KeyParams K) {
    const ReduceParams& P = K.P;
    unsigned long long bytes[MAX_KEYS];
#pragma unroll
    for (int k = 0; k < MAX_KEYS; ++k) bytes[k] = 0;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= (int64_t)P.table_mask; s += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t rep = P.table[s];
        if (rep == SLOT_EMPTY) continue;
        atomicAdd(P.group_count + partition_of(P.part_starts, P.N, (int64_t)rep), 1ULL);
#pragma unroll
        for (int k = 0; k < MAX_KEYS; ++k) {
            if (k >= P.n_keys) break;
            const ReduceCol& c = P.col[P.key_idx[k]];
            const KeyExt& kc = K.key[P.key_idx[k]];
            if (kc.kind < DFD_COL_UTF8 || (c.in_valid && !valid_at(c, (int64_t)rep))) continue;
            int64_t len;
            var_start(kc, (int64_t)rep, len);
            bytes[k] += (unsigned long long)len;
        }
    }
#pragma unroll
    for (int k = 0; k < MAX_KEYS; ++k) {
        if (k >= P.n_keys) break;
        unsigned long long v = bytes[k];
#pragma unroll
        for (int sh = 16; sh >= 1; sh >>= 1) v += __shfl_xor_sync(0xffffffffu, v, sh);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(K.key_bytes + k, v);
    }
}

// The start of a MIN / MAX whose representative is null: the end of the op's order that every value can replace, so that
// it stays only if no valid row reaches the state (k_group_clear then zeroes it) or if a valid row holds exactly these
// bits.  Signed integers: the type's maximum / minimum; unsigned: all ones / 0; floats: totalOrder's top +NaN 0x7f..f /
// bottom -NaN 0xf..f.  -> the low 64 bits; the I128 high halves (0x7f..f / 0x80..0) are set in state_init.  (MIN_I64 /
// MAX_I64 always start from their sentinel, valid representative or not.)
__device__ __forceinline__ uint64_t minmax_sentinel(int op) {
    switch (op) {
        case DFD_AGG_MIN_I32: return 0x7fffffffu;
        case DFD_AGG_MAX_I32: return 0x80000000u;
        case DFD_AGG_MIN_I16: return 0x7fffu;
        case DFD_AGG_MAX_I16: return 0x8000u;
        case DFD_AGG_MIN_I8: return 0x7fu;
        case DFD_AGG_MAX_I8: return 0x80u;
        case DFD_AGG_MIN_F64: return 0x7fffffffffffffffULL;
        case DFD_AGG_MIN_F32: return 0x7fffffffu;
        case DFD_AGG_MIN_F16: return 0x7fffu;
        case DFD_AGG_MAX_F64: case DFD_AGG_MAX_F32: case DFD_AGG_MAX_F16: case DFD_AGG_MIN_U64: case DFD_AGG_MIN_U32:
        case DFD_AGG_MIN_U16: case DFD_AGG_MIN_U8: case DFD_AGG_MIN_I128: return ~0ULL;  // (cut to the state's width)
        default: return 0;  // MAX_U64 / U32 / U16 / U8, MAX_I128
    }
}

// `rep` = the group's representative row.  Float MIN / MAX start from its value, not from +-inf: an all-NaN group then
// yields one of its own NaNs, and folding the representative in again in k_group_combine changes nothing.  The MIN / MAX
// ops of the other widths start from it too (no sentinel per type), unless it is null.  Float SUM starts from +0.0
// (dfd_b200.h): a group of only -0.0 values sums to +0.0.
__device__ __forceinline__ void state_init(const ReduceCol& c, char* dst, int64_t rep, bool rep_valid) {
    switch (c.op) {
        case DFD_AGG_SUM_I64: case DFD_AGG_SUM_F64: *(uint64_t*)dst = 0; break;
        case DFD_AGG_SUM_I128: ((uint64_t*)dst)[0] = 0; ((uint64_t*)dst)[1] = 0; break;
        case DFD_AGG_MIN_I64: *(long long*)dst = 0x7fffffffffffffffLL; break;
        case DFD_AGG_MAX_I64: *(long long*)dst = (long long)0x8000000000000000ULL; break;
        case DFD_AGG_MIN_F64: case DFD_AGG_MAX_F64:
            if (rep_valid) { *(uint64_t*)dst = *(const uint64_t*)(c.in + rep * 8); break; }
            [[fallthrough]];
        default: {  // MIN / MAX of every other width (aligned to it, dfd_partial_reduce_device checks)
            if (!rep_valid) {
                const uint64_t v = minmax_sentinel(c.op);
                switch (c.width) {
                    case 1: *(uint8_t*)dst = (uint8_t)v; break;
                    case 2: *(uint16_t*)dst = (uint16_t)v; break;
                    case 4: *(uint32_t*)dst = (uint32_t)v; break;
                    case 8: *(uint64_t*)dst = v; break;
                    default: ((uint64_t*)dst)[0] = v; ((uint64_t*)dst)[1] = c.op == DFD_AGG_MIN_I128 ? 0x7fffffffffffffffULL : 0x8000000000000000ULL; break;
                }
                break;
            }
            const char* src = c.in + rep * (int64_t)c.width;
            switch (c.width) {
                case 1: *dst = *src; break;
                case 2: *(uint16_t*)dst = *(const uint16_t*)src; break;
                case 4: *(uint32_t*)dst = *(const uint32_t*)src; break;
                case 8: *(uint64_t*)dst = *(const uint64_t*)src; break;
                default: ((uint64_t*)dst)[0] = ((const uint64_t*)src)[0]; ((uint64_t*)dst)[1] = ((const uint64_t*)src)[1]; break;
            }
        }
    }
}

// Output row o of key column c <- the representative's key (a null key's row: bit clear, value bytes zero).
__device__ __forceinline__ void place_key(const ReduceParams&, int, const ReduceCol& col, char* dst, int64_t rep, int64_t, bool valid) {
    const char* src = col.in + rep * col.width;
    for (int b = 0; b < col.width; ++b) dst[b] = valid ? src[b] : 0;
}

// ... a Boolean key: its bit (the words of rows [0, G) are zero before); a var-width key: its length, 0 for a null,
// into the output offsets, which the scan then turns into offsets in place, and the representative into out_rep.
__device__ __forceinline__ void place_key(const KeyParams& K, int c, const ReduceCol& col, char* dst, int64_t rep, int64_t o, bool valid) {
    const KeyExt& kc = K.key[c];
    if (kc.kind == DFD_COL_FIXED) {
        place_key(K.P, c, col, dst, rep, o, valid);
    } else if (kc.kind == DFD_COL_BOOL) {
        if (valid && bool_at(kc, rep)) set_valid((uint32_t*)kc.out, o);
    } else {
        int64_t len = 0;
        if (valid) var_start(kc, rep, len);
        if (kc.kind == DFD_COL_LARGE_UTF8) ((int64_t*)kc.out_off)[o] = len;
        else ((int32_t*)kc.out_off)[o] = (int32_t)len;
        K.out_rep[o] = (uint32_t)rep;
    }
}

template <bool NULLS, typename Params>
__device__ __forceinline__ void place_groups(const Params& K) {
    const ReduceParams& P = reduce_params(K);
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= (int64_t)P.table_mask; s += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t rep = P.table[s];
        if (rep == SLOT_EMPTY) continue;
        const uint32_t p = partition_of(P.part_starts, P.N, (int64_t)rep);
        const int64_t o = P.out_starts[p] + (int64_t)atomicAdd(P.cursor + p, 1ULL);
        P.slot_out[s] = (uint32_t)o;
        for (int c = 0; c < P.n_cols; ++c) {
            const ReduceCol& col = P.col[c];
            char* dst = col.out + o * (int64_t)col.width;
            const bool valid = !NULLS || !col.in_valid || valid_at(col, (int64_t)rep);
            if (col.op < 0) {
                place_key(K, c, col, dst, (int64_t)rep, o, valid);
            } else {
                state_init(col, dst, (int64_t)rep, valid);
            }
            if (NULLS && col.out_valid && valid) set_valid(col.out_valid, o);  // k_combine_nullable: the other valid rows
        }
    }
}

__global__ void __launch_bounds__(256) k_group_place(const __grid_constant__ ReduceParams P) { place_groups<false>(P); }
__global__ void __launch_bounds__(256) k_place_nullable(const __grid_constant__ ReduceParams P) { place_groups<true>(P); }
__global__ void __launch_bounds__(256) k_place_keys(const __grid_constant__ KeyParams K) { place_groups<true>(K); }

// Output bytes of one var-width key column: output row j gets its representative row's bytes (none for a null or empty
// one), at the offsets k_len_write_offsets left.  k_var_copy_bytes's scheme: a warp takes 32 consecutive output rows,
// every lane resolves its row's (source, destination, length), then the warp copies the rows one after the other with
// all 32 lanes on consecutive bytes, 8 bytes a lane when a long row and its destination are co-aligned.
template <typename OFF>
__global__ void __launch_bounds__(256) k_copy_key_bytes(const OFF* __restrict__ in_off, const uint8_t* __restrict__ in_data,
                                                        const uint8_t* __restrict__ in_valid, int64_t in_bit,
                                                        const uint32_t* __restrict__ out_rep, const OFF* __restrict__ out_off,
                                                        uint8_t* __restrict__ out_data, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = ((((int64_t)blockIdx.x * blockDim.x) + threadIdx.x) >> 5) << 5; base < n; base += n_warps << 5) {
        const int64_t j = base + lane;
        int64_t so = 0, dof = 0, len = 0;
        if (j < n) {
            const int64_t r = (int64_t)out_rep[j];
            const int64_t b = in_bit + r;
            if (!in_valid || ((in_valid[b >> 3] >> (b & 7)) & 1)) {
                so = (int64_t)in_off[r];
                len = (int64_t)in_off[r + 1] - so;
            }
            dof = (int64_t)out_off[j];
        }
        unsigned todo = __ballot_sync(0xffffffffu, len > 0);
        while (todo) {
            const int l = __ffs(todo) - 1;
            todo &= todo - 1;
            const uint8_t* s = in_data + __shfl_sync(0xffffffffu, so, l);
            uint8_t* d = out_data + __shfl_sync(0xffffffffu, dof, l);
            const int64_t L = __shfl_sync(0xffffffffu, len, l);
            if (L >= 256 && (((uintptr_t)s ^ (uintptr_t)d) & 7) == 0) {  // long, co-aligned: byte head, 8-byte body
                const int64_t head = (int64_t)((8 - ((uintptr_t)d & 7)) & 7);
                if (lane < head) d[lane] = s[lane];
                const int64_t words = (L - head) >> 3;
                const uint64_t* s8 = (const uint64_t*)(s + head);
                uint64_t* d8 = (uint64_t*)(d + head);
                for (int64_t i = lane; i < words; i += 32) d8[i] = s8[i];
                for (int64_t i = head + (words << 3) + lane; i < L; i += 32) d[i] = s[i];
            } else {
                for (int64_t i = lane; i < L; i += 32) d[i] = s[i];
            }
        }
    }
}

// IEEE 754 totalOrder as a signed integer: flipping the magnitude bits of negative values makes the int64 order
// -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN, with NaNs ordered by payload.  Only identical bits tie, so the
// merged MIN / MAX is the same whatever order the rows arrive in.
// Float32 / Float16 likewise at their width.
struct TotalOrder {
    __device__ long long operator()(unsigned long long bits) const {
        return (long long)(bits ^ ((unsigned long long)((long long)bits >> 63) >> 1));
    }
    __device__ int operator()(unsigned bits) const { return (int)(bits ^ ((unsigned)((int)bits >> 31) >> 1)); }
    __device__ short operator()(unsigned short bits) const { return (short)(bits ^ ((unsigned short)((short)bits >> 15) >> 1)); }
};
struct SignedOrder {
    __device__ short operator()(unsigned short b) const { return (short)b; }
    __device__ signed char operator()(unsigned char b) const { return (signed char)b; }
};
struct UnsignedOrder {
    template <typename W> __device__ W operator()(W b) const { return b; }
};

// MIN / MAX of a 16-, 32- or 64-bit word by CAS, values compared as order(value).  The loop exits on a value a single load
// or an atomic returned, and writes only when v wins, so the result is the bits of one input row.
template <bool MAX, typename W, typename Order>
__device__ __forceinline__ void atomic_minmax_cas(W* a, W v, Order order) {
    const auto vk = order(v);
    W old = *a;
    while (MAX ? vk > order(old) : vk < order(old)) {
        const W prev = atomicCAS(a, old, v);
        if (prev == old) break;
        old = prev;
    }
}

// 1-byte MIN / MAX: CAS on the aligned 32-bit word that holds the byte, replacing that byte only.  The word's other bytes
// may be other groups' rows, updated at the same moment (a CAS that loses to one of them retries with its new bytes), or
// lie outside the column: a CAS stores them as it found them, and only if no byte of the word moved, so they never change.
template <bool MAX, typename Order>
__device__ __forceinline__ void atomic_minmax_u8(unsigned char* p, unsigned char v, Order order) {
    unsigned* w = (unsigned*)((uintptr_t)p & ~(uintptr_t)3);
    const unsigned sh = ((unsigned)(uintptr_t)p & 3u) * 8u;
    const auto vk = order(v);
    unsigned old = *w;
    while (MAX ? vk > order((unsigned char)(old >> sh)) : vk < order((unsigned char)(old >> sh))) {
        const unsigned prev = atomicCAS(w, old, (old & ~(0xffu << sh)) | ((unsigned)v << sh));
        if (prev == old) break;
        old = prev;
    }
}

// One 128-bit compare-and-swap (sm_90, PTX ISA 8.3): *a = n if *a == c.  Returns the old value in (lo, hi).
__device__ __forceinline__ void atomic_cas_b128(unsigned long long* a, unsigned long long& lo, unsigned long long& hi,
                                                unsigned long long nlo, unsigned long long nhi) {
    asm volatile(
        "{\n\t.reg .b128 d, c, n;\n\t"
        "mov.b128 c, {%0, %1};\n\t"
        "mov.b128 n, {%3, %4};\n\t"
        "atom.global.cas.b128 d, [%2], c, n;\n\t"
        "mov.b128 {%0, %1}, d;\n\t}"
        : "+l"(lo), "+l"(hi)
        : "l"(__cvta_generic_to_global(a)), "l"(nlo), "l"(nhi)
        : "memory");
}

// 128-bit MIN / MAX (Decimal128): CAS on the whole 16-byte word, never two 64-bit updates (unlike SUM_I128, a MIN / MAX
// cannot be split into halves).  Order: the signed high halves, then the unsigned low halves.  Two 64-bit loads of the
// word may tear, so the loop trusts them for one thing only: a state only moves towards its result, so a v that loses on
// the high half alone, which one load reads whole, never wins.  Any other exit rests on a value the CAS returned: when v
// does not beat the loaded guess, the CAS writes the guess back unchanged, which succeeds only if the guess was real.
template <bool MAX>
__device__ __forceinline__ void atomic_minmax_i128(unsigned long long* a, unsigned long long vlo, long long vhi) {
    long long hi = *(volatile long long*)(a + 1);
    if (MAX ? vhi < hi : vhi > hi) return;
    unsigned long long lo = *(volatile unsigned long long*)a;
    for (bool exact = false;; exact = true) {
        const bool wins = MAX ? (vhi > hi || (vhi == hi && vlo > lo)) : (vhi < hi || (vhi == hi && vlo < lo));
        if (!wins && exact) return;
        unsigned long long plo = lo, phi = (unsigned long long)hi;
        atomic_cas_b128(a, plo, phi, wins ? vlo : lo, wins ? (unsigned long long)vhi : (unsigned long long)hi);
        if (plo == lo && (long long)phi == hi) return;
        lo = plo;
        hi = (long long)phi;
    }
}

template <bool NULLS>
__device__ __forceinline__ void combine_rows(const ReduceParams& P) {
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < P.n_rows; row += (int64_t)gridDim.x * blockDim.x) {
        const int64_t o = (int64_t)P.slot_out[P.row_slot[row]];
        for (int c = 0; c < P.n_cols; ++c) {
            const ReduceCol& col = P.col[c];
            if (col.op < 0) continue;
            if (NULLS && col.in_valid) {  // (then out_valid is set too: dfd_partial_reduce_device checks)
                if (!valid_at(col, row)) continue;
                // a plain load first, so that the rows of one hot group do not all queue on the bitmap word's atomic
                uint32_t* w = col.out_valid + (o >> 5);
                if (!((*w >> (o & 31)) & 1u)) atomicOr(w, 1u << (o & 31));
            }
            const char* src = col.in + row * (int64_t)col.width;
            char* dst = col.out + o * (int64_t)col.width;
            switch (col.op) {
                case DFD_AGG_SUM_I64: atomicAdd((unsigned long long*)dst, *(const unsigned long long*)src); break;
                case DFD_AGG_SUM_F64: atomicAdd((double*)dst, *(const double*)src); break;
                case DFD_AGG_MIN_I64: atomicMin((long long*)dst, *(const long long*)src); break;
                case DFD_AGG_MAX_I64: atomicMax((long long*)dst, *(const long long*)src); break;
                case DFD_AGG_MIN_F64: atomic_minmax_cas<false>((unsigned long long*)dst, *(const unsigned long long*)src, TotalOrder{}); break;
                case DFD_AGG_MAX_F64: atomic_minmax_cas<true>((unsigned long long*)dst, *(const unsigned long long*)src, TotalOrder{}); break;
                case DFD_AGG_MIN_I32: atomicMin((int*)dst, *(const int*)src); break;
                case DFD_AGG_MAX_I32: atomicMax((int*)dst, *(const int*)src); break;
                case DFD_AGG_MIN_U64: atomicMin((unsigned long long*)dst, *(const unsigned long long*)src); break;
                case DFD_AGG_MAX_U64: atomicMax((unsigned long long*)dst, *(const unsigned long long*)src); break;
                case DFD_AGG_MIN_U32: atomicMin((unsigned*)dst, *(const unsigned*)src); break;
                case DFD_AGG_MAX_U32: atomicMax((unsigned*)dst, *(const unsigned*)src); break;
                case DFD_AGG_MIN_I16: atomic_minmax_cas<false>((unsigned short*)dst, *(const unsigned short*)src, SignedOrder{}); break;
                case DFD_AGG_MAX_I16: atomic_minmax_cas<true>((unsigned short*)dst, *(const unsigned short*)src, SignedOrder{}); break;
                case DFD_AGG_MIN_U16: atomic_minmax_cas<false>((unsigned short*)dst, *(const unsigned short*)src, UnsignedOrder{}); break;
                case DFD_AGG_MAX_U16: atomic_minmax_cas<true>((unsigned short*)dst, *(const unsigned short*)src, UnsignedOrder{}); break;
                case DFD_AGG_MIN_F16: atomic_minmax_cas<false>((unsigned short*)dst, *(const unsigned short*)src, TotalOrder{}); break;
                case DFD_AGG_MAX_F16: atomic_minmax_cas<true>((unsigned short*)dst, *(const unsigned short*)src, TotalOrder{}); break;
                case DFD_AGG_MIN_I8: atomic_minmax_u8<false>((unsigned char*)dst, *(const unsigned char*)src, SignedOrder{}); break;
                case DFD_AGG_MAX_I8: atomic_minmax_u8<true>((unsigned char*)dst, *(const unsigned char*)src, SignedOrder{}); break;
                case DFD_AGG_MIN_U8: atomic_minmax_u8<false>((unsigned char*)dst, *(const unsigned char*)src, UnsignedOrder{}); break;
                case DFD_AGG_MAX_U8: atomic_minmax_u8<true>((unsigned char*)dst, *(const unsigned char*)src, UnsignedOrder{}); break;
                case DFD_AGG_MIN_F32: atomic_minmax_cas<false>((unsigned*)dst, *(const unsigned*)src, TotalOrder{}); break;
                case DFD_AGG_MAX_F32: atomic_minmax_cas<true>((unsigned*)dst, *(const unsigned*)src, TotalOrder{}); break;
                case DFD_AGG_MIN_I128:
                    atomic_minmax_i128<false>((unsigned long long*)dst, ((const unsigned long long*)src)[0], ((const long long*)src)[1]);
                    break;
                case DFD_AGG_MAX_I128:
                    atomic_minmax_i128<true>((unsigned long long*)dst, ((const unsigned long long*)src)[0], ((const long long*)src)[1]);
                    break;
                case DFD_AGG_SUM_I128: {
                    // two's complement 128-bit add as two 64-bit atomics: each add propagates its OWN carry exactly once
                    const unsigned long long lo = ((const unsigned long long*)src)[0], hi = ((const unsigned long long*)src)[1];
                    const unsigned long long old = atomicAdd((unsigned long long*)dst, lo);
                    const unsigned long long carry = (old + lo) < old ? 1ULL : 0ULL;
                    atomicAdd((unsigned long long*)dst + 1, hi + carry);
                    break;
                }
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_group_combine(const __grid_constant__ ReduceParams P) { combine_rows<false>(P); }
__global__ void __launch_bounds__(256) k_combine_nullable(const __grid_constant__ ReduceParams P) { combine_rows<true>(P); }

__host__ __device__ __forceinline__ bool is_minmax(int op) {
    return op >= 0 && op != DFD_AGG_SUM_I64 && op != DFD_AGG_SUM_F64 && op != DFD_AGG_SUM_I128;
}

// Zeroes the value of every MIN / MAX state (of a column with an input bitmap) that no valid row reached: it still holds
// the sentinel k_group_place started it from.  Launched after k_group_combine, only when such a column exists.
__global__ void __launch_bounds__(256) k_group_clear(const __grid_constant__ ReduceParams P) {
    for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < P.n_groups; o += (int64_t)gridDim.x * blockDim.x) {
        for (int c = 0; c < P.n_cols; ++c) {
            const ReduceCol& col = P.col[c];
            if (!col.in_valid || !is_minmax(col.op)) continue;
            if ((col.out_valid[o >> 5] >> (o & 31)) & 1u) continue;
            char* dst = col.out + o * (int64_t)col.width;
            switch (col.width) {
                case 1: *(uint8_t*)dst = 0; break;
                case 2: *(uint16_t*)dst = 0; break;
                case 4: *(uint32_t*)dst = 0; break;
                case 8: *(uint64_t*)dst = 0; break;
                default: ((uint64_t*)dst)[0] = 0; ((uint64_t*)dst)[1] = 0; break;
            }
        }
    }
}

// Bytes of a state column of `op`; 0 for a value outside dfd_agg_op.
int agg_width(int op) {
    switch (op) {
        case DFD_AGG_SUM_I128: case DFD_AGG_MIN_I128: case DFD_AGG_MAX_I128: return 16;
        case DFD_AGG_SUM_I64: case DFD_AGG_SUM_F64: case DFD_AGG_MIN_I64: case DFD_AGG_MAX_I64: case DFD_AGG_MIN_F64:
        case DFD_AGG_MAX_F64: case DFD_AGG_MIN_U64: case DFD_AGG_MAX_U64: return 8;
        case DFD_AGG_MIN_I32: case DFD_AGG_MAX_I32: case DFD_AGG_MIN_U32: case DFD_AGG_MAX_U32: case DFD_AGG_MIN_F32:
        case DFD_AGG_MAX_F32: return 4;
        case DFD_AGG_MIN_I16: case DFD_AGG_MAX_I16: case DFD_AGG_MIN_U16: case DFD_AGG_MAX_U16: case DFD_AGG_MIN_F16:
        case DFD_AGG_MAX_F16: return 2;
        case DFD_AGG_MIN_I8: case DFD_AGG_MAX_I8: case DFD_AGG_MIN_U8: case DFD_AGG_MAX_U8: return 1;
        default: return 0;
    }
}

}  // namespace

extern "C" int dfd_partial_reduce_device(dfd_ctx* c, const dfd_column* in_cols, int n_cols, int64_t n_rows, const int32_t* key_cols, int n_keys,
                                         const int32_t* agg_ops, const int64_t* part_starts_device, uint32_t num_partitions,
                                         const dfd_column* out_cols, int64_t* out_part_starts_host, int64_t* out_part_starts_device) {
    if (!c || !in_cols || !out_cols || !key_cols || !agg_ops || !part_starts_device || !out_part_starts_host)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_partial_reduce_device: NULL argument");
    if (n_cols < 1 || n_cols > MAX_REDUCE_COLS || n_keys < 1 || n_keys > MAX_KEYS || n_rows < 0 || n_rows >= 0xffffffffLL || num_partitions < 1)
        return set_error(DFD_ERR_INVALID_ARGUMENT, "dfd_partial_reduce_device: bad sizes (columns <= %d, keys <= %d, rows < 2^32)", MAX_REDUCE_COLS, MAX_KEYS);
    // the table has the next power of two >= 2 * n_rows slots, addressed through a u32 mask: at most 2^32 slots
    if (n_rows > ((int64_t)1 << 31))
        return set_error(DFD_ERR_UNSUPPORTED, "dfd_partial_reduce_device: n_rows %lld > 2^31 per call (32-bit hash table slots)", (long long)n_rows);
    KeyParams K{};  // (only the k_*_keys launches read past K.P)
    ReduceParams& P = K.P;
    P.n_cols = n_cols;
    P.n_keys = n_keys;
    P.n_rows = n_rows;
    P.N = num_partitions;
    for (int k = 0; k < n_keys; ++k) {
        if (key_cols[k] < 0 || key_cols[k] >= n_cols || agg_ops[key_cols[k]] >= 0)
            return set_error(DFD_ERR_INVALID_ARGUMENT, "key column %d out of range or carries an aggregate", key_cols[k]);
        P.key_idx[k] = key_cols[k];
    }
    // which kernels run their nullable code: a key column has an input bitmap (insert); any column has a bitmap (place); a
    // state column has an input bitmap (combine); a MIN / MAX state column has one (k_group_clear runs).  `keyed`: a key is
    // Boolean or var-width (insert, count and place run their k_*_keys code); `var_keys` of them are var-width.
    bool null_keys = false, any_bitmap = false, null_states = false, clear = false, keyed = false;
    int var_keys = 0;
    for (int i = 0; i < n_cols; ++i) {
        const dfd_column& ic = in_cols[i];
        const dfd_column& oc = out_cols[i];
        const int op = agg_ops[i];
        bool is_key = false;
        for (int k = 0; k < n_keys; ++k) is_key |= key_cols[k] == i;
        if (is_key && ic.kind >= DFD_COL_BOOL && ic.kind <= DFD_COL_BINARY) {  // a Boolean or var-width key
            const bool var = ic.kind != DFD_COL_BOOL;
            const int ow = ic.kind == DFD_COL_LARGE_UTF8 ? 8 : 4;
            if (oc.kind != ic.kind)
                return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: a key of kind %d needs an output of the same kind, not %d", i, ic.kind, oc.kind);
            if (!ic.values || !oc.values) return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: values is NULL", i);
            if (var && (!ic.offsets || !oc.offsets))
                return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: a var-width key needs input and output offsets", i);
            if (var && (uintptr_t)oc.offsets % (uintptr_t)ow != 0)
                return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: the output offsets %p are not %d-byte aligned", i, oc.offsets, ow);
            if (!var && (uintptr_t)oc.values % 4 != 0)
                return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: the Boolean output %p is not 4-byte aligned", i, oc.values);
            if (ic.validity && !oc.validity)
                return set_error(DFD_ERR_UNSUPPORTED, "column %d has a validity bitmap but its output has none (a non-null output column)", i);
            if ((uintptr_t)oc.validity % 4 != 0)
                return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: the output validity bitmap %p is not 4-byte aligned", i, (void*)oc.validity);
            P.col[i] = ReduceCol{nullptr, nullptr, ic.validity ? ic.validity + (ic.offset >> 3) : nullptr, (uint32_t*)oc.validity, 0, op,
                                 (int32_t)(ic.offset & 7)};
            K.key[i] = var ? KeyExt{ic.kind, 0, (const char*)ic.offsets + ic.offset * ow, (const uint8_t*)ic.values, oc.offsets, (uint8_t*)oc.values}
                           : KeyExt{ic.kind, (int32_t)(ic.offset & 7), nullptr, (const uint8_t*)ic.values + (ic.offset >> 3), nullptr, (uint8_t*)oc.values};
            keyed = true;
            var_keys += var;
            any_bitmap |= ic.validity || oc.validity;
            continue;
        }
        if (ic.kind != DFD_COL_FIXED || out_cols[i].kind != DFD_COL_FIXED || out_cols[i].width != ic.width)
            return set_error(DFD_ERR_UNSUPPORTED, "column %d: partial reduce moves fixed-width columns (keys and aggregate states)", i);
        if (ic.validity && !out_cols[i].validity)
            return set_error(DFD_ERR_UNSUPPORTED, "column %d has a validity bitmap but its output has none (a non-null output column)", i);
        if ((uintptr_t)out_cols[i].validity % 4 != 0)
            return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: the output validity bitmap %p is not 4-byte aligned", i, (void*)out_cols[i].validity);
        if (op < 0 && !is_key) return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d is neither a group key nor an aggregate state", i);
        const int need = op < 0 ? ic.width : agg_width(op);
        if (op > DFD_AGG_MAX_F16 || ic.width != need || (op < 0 && ic.width != 1 && ic.width != 2 && ic.width != 4 && ic.width != 8 && ic.width != 16))
            return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: aggregate op %d does not match value width %d", i, op, ic.width);
        P.col[i] = ReduceCol{(const char*)ic.values + ic.offset * (int64_t)ic.width, (char*)out_cols[i].values,
                             ic.validity ? ic.validity + (ic.offset >> 3) : nullptr, (uint32_t*)out_cols[i].validity, ic.width, op,
                             (int32_t)(ic.offset & 7)};
        null_keys |= ic.validity && op < 0;
        any_bitmap |= ic.validity || out_cols[i].validity;
        null_states |= ic.validity && op >= 0;
        clear |= ic.validity && is_minmax(op);
        if (!ic.values || !out_cols[i].values) return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: values is NULL", i);
        // the MIN / MAX ops numbered 7 and up load and update whole values: each must sit at an address aligned
        // to its width (an input 128-bit value, read as two 64-bit halves, to 8 bytes; an output one, a 128-bit atomic's
        // target, to 16)
        if (op >= DFD_AGG_MIN_I32 && ((uintptr_t)P.col[i].in % (uintptr_t)(ic.width < 8 ? ic.width : 8) != 0 ||
                                      (uintptr_t)P.col[i].out % (uintptr_t)ic.width != 0))
            return set_error(DFD_ERR_INVALID_ARGUMENT, "column %d: aggregate op %d needs values aligned to their width %d (input %p, output %p)",
                             i, op, ic.width, (const void*)P.col[i].in, (void*)P.col[i].out);
    }
    std::lock_guard<std::mutex> lk(c->mu);
    cudaError_t e = cudaSetDevice(c->device);
    if (e != cudaSuccess) return cuda_error(e, "cudaSetDevice");
    cudaStream_t s = c->stream;
    const uint32_t N = num_partitions;
    if (n_rows == 0) {
        for (uint32_t p = 0; p <= N; ++p) out_part_starts_host[p] = 0;
        if (out_part_starts_device && (e = cudaMemsetAsync(out_part_starts_device, 0, sizeof(int64_t) * (N + 1), s)) != cudaSuccess)
            return cuda_error(e, "cudaMemsetAsync");
        for (int i = 0; i < n_cols; ++i)  // entry 0 of a var-width key's offsets
            if (K.key[i].kind >= DFD_COL_UTF8 &&
                (e = cudaMemsetAsync(K.key[i].out_off, 0, K.key[i].kind == DFD_COL_LARGE_UTF8 ? 8 : 4, s)) != cudaSuccess)
                return cuda_error(e, "cudaMemsetAsync(offsets)");
        return DFD_OK;
    }
    uint64_t slots = 64;
    while (slots < (uint64_t)n_rows * 2) slots <<= 1;  // load factor <= 0.5
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t table_b = al(slots * 4), rowslot_b = al((size_t)n_rows * 4), small_b = al((size_t)(3 * N + 2 + (keyed ? MAX_KEYS : 0)) * 8);
    // var-width keys: out_rep [n_rows] and the block sums of the offset scan [n_rows / 2048 + 2]
    const size_t rep_b = var_keys ? rowslot_b : 0, sums_b = var_keys ? al(((size_t)n_rows / 2048 + 2) * 8) : 0;
    int rc = c->var_scratch.ensure(2 * table_b + rowslot_b + small_b + rep_b + sums_b + 256, c->device);
    if (rc) return rc;
    char* base = (char*)c->var_scratch.ptr;
    P.table = (uint32_t*)base;
    P.slot_out = (uint32_t*)(base + table_b);
    P.row_slot = (uint32_t*)(base + 2 * table_b);
    P.group_count = (unsigned long long*)(base + 2 * table_b + rowslot_b);
    P.cursor = P.group_count + N;
    P.out_starts = (int64_t*)(P.cursor + N);
    P.part_starts = part_starts_device;
    P.table_mask = (uint32_t)(slots - 1);
    K.key_bytes = (unsigned long long*)(P.out_starts + N + 1);
    K.out_rep = var_keys ? (uint32_t*)(base + 2 * table_b + rowslot_b + small_b) : nullptr;
    unsigned long long* block_sums = (unsigned long long*)(base + 2 * table_b + rowslot_b + small_b + rep_b);
    if ((e = cudaMemsetAsync(P.table, 0xff, slots * 4, s)) != cudaSuccess) return cuda_error(e, "cudaMemsetAsync(table)");
    if ((e = cudaMemsetAsync(P.group_count, 0, small_b, s)) != cudaSuccess) return cuda_error(e, "cudaMemsetAsync(counters)");
    const unsigned grid = (unsigned)(c->sm_count * 8);
    if (keyed)
        k_insert_keys<<<grid, 256, 0, s>>>(K);
    else if (null_keys)
        k_insert_nullable<<<grid, 256, 0, s>>>(P);
    else
        k_group_insert<<<grid, 256, 0, s>>>(P);
    if (keyed)
        k_count_keys<<<grid, 256, 0, s>>>(K);
    else
        k_group_count<<<grid, 256, 0, s>>>(P);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error(e, "k_group_insert / k_group_count");
    c->metrics.kernel_launches += 2;  // (a capacity refusal below launches nothing more)
    std::vector<unsigned long long> counts(N), key_bytes(MAX_KEYS);
    if ((e = cudaMemcpyAsync(counts.data(), P.group_count, sizeof(unsigned long long) * N, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (keyed && (e = cudaMemcpyAsync(key_bytes.data(), K.key_bytes, sizeof(unsigned long long) * MAX_KEYS, cudaMemcpyDeviceToHost, s)) != cudaSuccess) ||
        (e = cudaStreamSynchronize(s)) != cudaSuccess)
        return cuda_error(e, "partial reduce: group counts");
    for (int k = 0; k < n_keys; ++k) {  // before any output is written
        const int i = key_cols[k];
        if (K.key[i].kind >= DFD_COL_UTF8 && key_bytes[k] > (unsigned long long)out_cols[i].values_bytes)
            return set_error(DFD_ERR_CAPACITY, "column %d: the groups' keys need %llu bytes, the output holds %lld", i, key_bytes[k],
                             (long long)out_cols[i].values_bytes);
    }
    out_part_starts_host[0] = 0;
    for (uint32_t p = 0; p < N; ++p) out_part_starts_host[p + 1] = out_part_starts_host[p] + (int64_t)counts[p];
    if ((e = cudaMemcpyAsync(P.out_starts, out_part_starts_host, sizeof(int64_t) * (N + 1), cudaMemcpyHostToDevice, s)) != cudaSuccess)
        return cuda_error(e, "H2D out_starts");
    if (out_part_starts_device &&
        (e = cudaMemcpyAsync(out_part_starts_device, out_part_starts_host, sizeof(int64_t) * (N + 1), cudaMemcpyHostToDevice, s)) != cudaSuccess)
        return cuda_error(e, "H2D out_starts");
    P.n_groups = out_part_starts_host[N];
    for (int i = 0; i < n_cols; ++i)  // the words of output rows [0, G); k_group_place and k_group_combine set the valid ones
        if (P.col[i].out_valid && (e = cudaMemsetAsync(P.col[i].out_valid, 0, (size_t)((P.n_groups + 31) / 32) * 4, s)) != cudaSuccess)
            return cuda_error(e, "cudaMemsetAsync(output validity)");
    for (int i = 0; i < n_cols; ++i)  // likewise the value words of a Boolean key; k_place_keys sets the true ones
        if (K.key[i].kind == DFD_COL_BOOL && (e = cudaMemsetAsync(K.key[i].out, 0, (size_t)((P.n_groups + 31) / 32) * 4, s)) != cudaSuccess)
            return cuda_error(e, "cudaMemsetAsync(Boolean key)");
    if (keyed)
        k_place_keys<<<grid, 256, 0, s>>>(K);
    else if (any_bitmap)
        k_place_nullable<<<grid, 256, 0, s>>>(P);
    else
        k_group_place<<<grid, 256, 0, s>>>(P);
    if (null_states)
        k_combine_nullable<<<grid, 256, 0, s>>>(P);
    else
        k_group_combine<<<grid, 256, 0, s>>>(P);
    if (clear) k_group_clear<<<grid, 256, 0, s>>>(P);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error(e, "k_group_place / k_group_combine / k_group_clear");
    // var-width keys, one column at a time: the lengths k_place_keys left in entries [0, G) of the output offsets become the
    // offsets [0, G] in place (each scan thread reads its entries before it writes them), then the bytes are copied
    for (int i = 0; i < n_cols; ++i) {
        const KeyExt& kc = K.key[i];
        if (kc.kind < DFD_COL_UTF8) continue;
        const int ow = kc.kind == DFD_COL_LARGE_UTF8 ? 8 : 4;
        if ((rc = launch_lengths_to_offsets(kc.out_off, ow, P.n_groups, block_sums, kc.out_off, s))) return rc;
        const int64_t blocks = (P.n_groups + 255) / 256;
        const unsigned copy_grid = (unsigned)(blocks > 0x7fffffffLL ? 0x7fffffffLL : blocks);
        if (ow == 8)
            k_copy_key_bytes<int64_t><<<copy_grid, 256, 0, s>>>((const int64_t*)kc.in_off, kc.in, P.col[i].in_valid, P.col[i].in_bit, K.out_rep,
                                                               (const int64_t*)kc.out_off, kc.out, P.n_groups);
        else
            k_copy_key_bytes<int32_t><<<copy_grid, 256, 0, s>>>((const int32_t*)kc.in_off, kc.in, P.col[i].in_valid, P.col[i].in_bit, K.out_rep,
                                                               (const int32_t*)kc.out_off, kc.out, P.n_groups);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error(e, "k_copy_key_bytes");
    }
    c->metrics.kernel_launches += (clear ? 3 : 2) + 4 * var_keys;
    if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return cuda_error(e, "partial reduce");  // (out_part_starts_host is caller memory)
    return DFD_OK;
}
