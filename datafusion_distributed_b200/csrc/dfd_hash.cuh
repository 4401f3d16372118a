// dfd_hash.cuh — device-side hashing for the repartition path (sm_90a).
//
// Bit-for-bit the arithmetic DataFusion 53 runs in
//   BatchPartitioner::partition (Hash arm) -> create_hashes(keys, REPARTITION_RANDOM_STATE)
//   -> ahash 0.8.12 fallback hasher -> `hash % num_partitions`
// (third-party crates the reference pins in Cargo.lock:32-33,1960-1985,2572-2574
// and calls through src/execution_plans/network_shuffle.rs:126-134 and
// src/worker/impl_execute_task.rs:77-86).  Integer work only: two 64x64->128
// multiplies per fixed-width key (IMAD.WIDE chains), no tensor cores.
#pragma once
#include <cstdint>

namespace dfd {

constexpr int MAX_KEYS = 8;

// ahash RandomState after with_seeds(); AHasher::from_random_state takes
// buffer = k1, pad = k0, extra_keys = [k2, k3].
struct HashState {
    uint64_t k0, k1, k2, k3;
};

constexpr uint64_t AHASH_MULTIPLE = 6364136223846793005ULL;
constexpr unsigned AHASH_ROT = 23;

enum ColKind : int32_t { COL_FIXED = 0, COL_BOOL = 1, COL_UTF8 = 2, COL_LARGE_UTF8 = 3, COL_BINARY = 4 };

struct KeyCol {
    const void* values;
    const void* offsets;
    const uint8_t* validity;
    int64_t offset;
    int32_t kind;
    int16_t width;
    int8_t mode;              // KEY_HASH_*: how a fixed-width value is fed to the hasher
    uint8_t index_unsigned;   // KEY_HASH_DICTIONARY: the indices are UInt8/16/32/64 (zero-extended), else signed
    const uint8_t* dict_validity;  // KEY_HASH_DICTIONARY: validity bitmap of the dictionary VALUES (or nullptr); `offsets` = their u64 hashes
};

// A fixed-width key is normally ONE write_u{8..128}.  Arrow's interval structs derive `Hash`, i.e. one write
// per field (arrow-buffer IntervalDayTime {i32, i32}, IntervalMonthDayNano {i32, i32, i64}; DataFusion hash_utils
// `hash_value!(.., IntervalDayTime, IntervalMonthDayNano)` -> `state.hash_one(self)`).
// KEY_HASH_DICTIONARY: the column holds dictionary INDICES (`width` bytes, signed or unsigned per `index_unsigned`);
// DataFusion's hash_dictionary hashes the dictionary values once (create_hashes over the values array) and a row takes
// dict_hashes[key.as_usize()]; a null index or a null dictionary value leaves the running hash untouched.
enum KeyHashMode : int8_t { KEY_HASH_PLAIN = 0, KEY_HASH_INTERVAL_DAY_TIME = 1, KEY_HASH_INTERVAL_MONTH_DAY_NANO = 2, KEY_HASH_DICTIONARY = 3 };

struct KeySet {
    KeyCol col[MAX_KEYS];
    int32_t n;
    int32_t fast_i64;  // 1: exactly one non-null 8-byte fixed key with offset 0
};

// `h % n` for n in [1, 2^32) (the ABI caps n at DFD_MAX_PARTITIONS = 4096): mask for powers of two, otherwise one Barrett
// step (q = mulhi(h, floor(2^64/n)) is off by at most one) — replaces the
// ~100-instruction generic 64-bit remainder.
struct ModN {
    uint64_t magic;
    uint32_t n;
    uint32_t pow2_mask;  // n-1 when n is a power of two, else 0xffffffff marker unused
    uint32_t is_pow2;
};

__host__ inline ModN make_modn(uint32_t n) {
    ModN m;
    m.n = n;
    m.is_pow2 = (n & (n - 1)) == 0;
    m.pow2_mask = n - 1;
    m.magic = m.is_pow2 ? 0 : (~0ULL) / n;  // floor(2^64 / n) for non powers of two
    return m;
}

__device__ __forceinline__ uint32_t mod_n(uint64_t h, const ModN& m) {
    if (m.is_pow2) return (uint32_t)h & m.pow2_mask;
    uint64_t q = __umul64hi(h, m.magic);
    uint64_t r = h - q * (uint64_t)m.n;
    if (r >= m.n) r -= m.n;
    return (uint32_t)r;
}

__device__ __forceinline__ uint64_t rotl64(uint64_t x, unsigned r) {
    r &= 63;
    return (x << r) | (x >> ((64 - r) & 63));
}

// lo64(s*by) ^ hi64(s*by).  nvcc lowers this to 3 IMAD (low half) + 4 IMAD.WIDE.U32 with
// carry predicates (high half); a hand-split 32-bit-limb version was measured to be LONGER
// (extra zero-extension moves), so the intrinsic form stays.
__device__ __forceinline__ uint64_t folded_multiply(uint64_t s, uint64_t by) {
    return (s * by) ^ __umul64hi(s, by);
}

struct AHasher {
    uint64_t buffer, pad, e0, e1;
    __device__ __forceinline__ explicit AHasher(const HashState& st)
        : buffer(st.k1), pad(st.k0), e0(st.k2), e1(st.k3) {}
    __device__ __forceinline__ void update(uint64_t x) { buffer = folded_multiply(x ^ buffer, AHASH_MULTIPLE); }
    __device__ __forceinline__ void large_update(uint64_t lo, uint64_t hi) {
        uint64_t combined = folded_multiply(lo ^ e0, hi ^ e1);
        buffer = rotl64((buffer + pad) ^ combined, AHASH_ROT);
    }
    __device__ __forceinline__ uint64_t finish() const {
        return rotl64(folded_multiply(buffer, pad), (unsigned)(buffer & 63));
    }
    // little-endian read of n (1..8) bytes at an arbitrary address: the one or two ALIGNED 8-byte words that cover
    // [p, p+n) are loaded and funnel-shifted (a byte loop costs up to 8 dependent loads per call and dominated string-key
    // hashing).  Only words that contain requested bytes are touched, so nothing outside the buffer's 8-byte-aligned extent
    // is read (Arrow buffers are at least 8-byte aligned).
    static __device__ __forceinline__ uint64_t rd(const uint8_t* p, int n) {
        const uintptr_t a = (uintptr_t)p;
        const unsigned sh = (unsigned)(a & 7u) * 8u;
        const uint64_t* w = (const uint64_t*)(a & ~(uintptr_t)7);
        uint64_t v = w[0] >> sh;
        if (sh && (int)(a & 7u) + n > 8) v |= w[1] << (64u - sh);
        return n >= 8 ? v : (v & ((1ULL << (8 * n)) - 1ULL));
    }
    // AHasher::write(&[u8]) (fallback_hash.rs) with operations.rs read_small
    __device__ void write(const uint8_t* data, uint64_t len) {
        buffer = (buffer + len) * AHASH_MULTIPLE;
        if (len > 8) {
            if (len > 16) {
                large_update(rd(data + len - 16, 8), rd(data + len - 8, 8));
                while (len > 16) {
                    large_update(rd(data, 8), rd(data + 8, 8));
                    data += 16;
                    len -= 16;
                }
            } else {
                large_update(rd(data, 8), rd(data + len - 8, 8));
            }
        } else {
            uint64_t a, b;
            if (len >= 2) {
                if (len >= 4) {
                    a = rd(data, 4);
                    b = rd(data + len - 4, 4);
                } else {
                    a = rd(data, 2);
                    b = data[len - 1];
                }
            } else if (len > 0) {
                a = b = data[0];
            } else {
                a = b = 0;
            }
            large_update(a, b);
        }
    }
};

__device__ __forceinline__ uint64_t hash_one_u64(const HashState& st, uint64_t x) {
    AHasher h(st);
    h.update(x);
    return h.finish();
}

// datafusion-common hash_utils::combine_hashes
__device__ __forceinline__ uint64_t combine_hashes(uint64_t l, uint64_t r) {
    return (17ULL * 37ULL + l) * 37ULL + r;
}

__device__ __forceinline__ bool bit_is_set(const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; }

// hash_one of row `j` (already offset-adjusted) of one key column
__device__ __forceinline__ uint64_t hash_key_value(const KeyCol& c, int64_t j, const HashState& st) {
    switch (c.kind) {
        case COL_FIXED: {
            switch (c.width) {
                case 8: {
                    const uint64_t v = ((const uint64_t*)c.values)[j];
                    if (c.mode == KEY_HASH_INTERVAL_DAY_TIME) {  // {days: i32, milliseconds: i32}: two write_i32
                        AHasher h(st);
                        h.update(v & 0xffffffffULL);
                        h.update(v >> 32);
                        return h.finish();
                    }
                    return hash_one_u64(st, v);
                }
                case 4: return hash_one_u64(st, ((const uint32_t*)c.values)[j]);
                case 2: return hash_one_u64(st, ((const uint16_t*)c.values)[j]);
                case 1: return hash_one_u64(st, ((const uint8_t*)c.values)[j]);
                default: {  // 16: write_u128 -> large_update
                    const uint64_t* p = (const uint64_t*)c.values + 2 * j;
                    AHasher h(st);
                    if (c.mode == KEY_HASH_INTERVAL_MONTH_DAY_NANO) {  // {months: i32, days: i32, nanoseconds: i64}
                        h.update(p[0] & 0xffffffffULL);
                        h.update(p[0] >> 32);
                        h.update(p[1]);
                    } else {
                        h.large_update(p[0], p[1]);
                    }
                    return h.finish();
                }
            }
        }
        case COL_BOOL: return hash_one_u64(st, bit_is_set((const uint8_t*)c.values, j) ? 1 : 0);
        case COL_UTF8:
        case COL_BINARY: {
            const int32_t* off = (const int32_t*)c.offsets;
            int32_t a = off[j], b = off[j + 1];
            AHasher h(st);
            if (c.kind == COL_BINARY) h.update((uint64_t)(b - a));  // write_length_prefix
            h.write((const uint8_t*)c.values + a, (uint64_t)(b - a));
            if (c.kind == COL_UTF8) h.update(0xff);  // write_str suffix
            return h.finish();
        }
        default: {  // COL_LARGE_UTF8
            const int64_t* off = (const int64_t*)c.offsets;
            int64_t a = off[j], b = off[j + 1];
            AHasher h(st);
            h.write((const uint8_t*)c.values + a, (uint64_t)(b - a));
            h.update(0xff);
            return h.finish();
        }
    }
}

// create_hashes for one row: column 0 overwrites, column j>=1 combines,
// null key values leave the running hash untouched.
// FAST_I64 (compile time): exactly one non-null 8-byte key at offset 0 — the
// kernel instantiation for the headline workload carries none of the generic
// (string / multi-key / null) code.
template <bool FAST_I64>
__device__ __forceinline__ uint64_t row_hash(const KeySet& ks, int64_t row, const HashState& st) {
    if (FAST_I64) return hash_one_u64(st, ((const uint64_t*)ks.col[0].values)[row]);
    uint64_t h = 0;
    for (int k = 0; k < ks.n; ++k) {
        const KeyCol& c = ks.col[k];
        int64_t j = row + c.offset;
        if (c.validity && !bit_is_set(c.validity, j)) continue;
        uint64_t v;
        if (c.mode == KEY_HASH_DICTIONARY) {
            uint64_t raw;
            switch (c.width) {
                case 8: raw = ((const uint64_t*)c.values)[j]; break;
                case 4: raw = ((const uint32_t*)c.values)[j]; break;
                case 2: raw = ((const uint16_t*)c.values)[j]; break;
                default: raw = ((const uint8_t*)c.values)[j]; break;
            }
            // zero-extended load, then a shift pair sign-extends signed indices (this form leaves the generic scatter kernels'
            // registers and spills as they were with signed loads); 8-byte indices are taken as they are: a valid one is below 2^63
            const unsigned s = c.index_unsigned ? 0u : 64u - 8u * (unsigned)c.width;
            const int64_t idx = (int64_t)(raw << s) >> s;
            if (c.dict_validity && !bit_is_set(c.dict_validity, idx)) continue;
            v = ((const uint64_t*)c.offsets)[idx];
        } else {
            v = hash_key_value(c, j, st);
        }
        h = k >= 1 ? combine_hashes(v, h) : v;
    }
    return h;
}

}  // namespace dfd
