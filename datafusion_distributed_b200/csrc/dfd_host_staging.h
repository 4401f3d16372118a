// dfd_host_staging.h — the pure index arithmetic of the host operator's staging (dfd_exec.cu): no CUDA, no operator
// state, plain pointers in and out.  Kept apart so that the CPU test-suite can run exactly this code against pyarrow
// (tests/test_host_staging.py compiles it with g++): bitmap concatenation at bit granularity, Utf8View / BinaryView ->
// offsets + bytes and back, List<Utf8 / Binary> rows -> the three hidden Binary device columns.
#pragma once
#include <cstdint>
#include <cstring>

namespace dfd {
namespace host {

// append bits [lo, lo + n) of `src` (nullptr = all ones) to the bitmap `dst` at bit position `at`; bits of the last byte
// beyond at + n are left zero, so the next append continues cleanly
inline void append_bits(uint8_t* dst, int64_t at, const uint8_t* src, int64_t lo, int64_t n) {
    auto get = [&](int64_t k) -> unsigned { return src ? (unsigned)((src[(lo + k) >> 3] >> ((lo + k) & 7)) & 1) : 1u; };
    int64_t i = 0;
    for (; i < n && ((at + i) & 7); ++i) {  // head: up to the next byte boundary of the destination
        uint8_t& d = dst[(at + i) >> 3];
        const uint8_t m = (uint8_t)(1u << ((at + i) & 7));
        d = get(i) ? (uint8_t)(d | m) : (uint8_t)(d & ~m);
    }
    uint8_t* d = dst + ((at + i) >> 3);
    const int64_t nb = (n - i) >> 3;  // whole destination bytes
    if (nb > 0) {
        if (!src) {
            memset(d, 0xff, (size_t)nb);
        } else {
            const int sh = (int)((lo + i) & 7);
            const uint8_t* sp = src + ((lo + i) >> 3);
            if (sh == 0) memcpy(d, sp, (size_t)nb);
            else
                for (int64_t b = 0; b < nb; ++b) d[b] = (uint8_t)((sp[b] >> sh) | (sp[b + 1] << (8 - sh)));
        }
        i += nb * 8;
        d += nb;
    }
    if (i < n) {  // tail: a partial byte, upper bits zero
        unsigned v = 0;
        for (int64_t k = i; k < n; ++k) v |= get(k) << (k - i);
        *d = (uint8_t)v;
    }
}

// Utf8View / BinaryView rows [lo, lo + n) -> int32 offsets (off32[0] = 0 ... off32[n] = total bytes); a null row has length 0.
// 16-byte views: int32 length | 12 inline bytes, or int32 length | 4-byte prefix | int32 buffer index | int32 offset.
// Returns the total byte count, or -1 when it does not fit 32-bit offsets.
inline int64_t view_offsets(const uint8_t* views, const uint8_t* valid, int64_t lo, int64_t n, int32_t* off32) {
    int64_t total = 0;
    for (int64_t r = 0; r < n; ++r) {
        const uint8_t* v = views + (size_t)(lo + r) * 16;
        int32_t len;
        memcpy(&len, v, 4);
        if (valid && !((valid[(lo + r) >> 3] >> ((lo + r) & 7)) & 1)) len = 0;
        off32[r] = (int32_t)total;
        total += len;
        if (total > 0x7fffffffLL) return -1;
    }
    off32[n] = (int32_t)total;
    return total;
}

// ... and their bytes, contiguous in row order (`data_buffers` = the array's variadic data buffers, i.e. buffers + 2)
inline void view_bytes(const uint8_t* views, const void* const* data_buffers, int64_t lo, int64_t n, const int32_t* off32, char* out) {
    for (int64_t r = 0; r < n; ++r) {
        const int32_t len = off32[r + 1] - off32[r];
        if (!len) continue;
        const uint8_t* v = views + (size_t)(lo + r) * 16;
        int32_t buf, pos;
        memcpy(&buf, v + 8, 4);
        memcpy(&pos, v + 12, 4);
        const uint8_t* src = len <= 12 ? v + 4 : (const uint8_t*)data_buffers[buf] + pos;
        memcpy(out + off32[r], src, (size_t)len);
    }
}

// offsets + bytes -> 16-byte views over ONE data buffer (buffer index 0), inline when <= 12 bytes: the output side
inline void build_views(const int32_t* off, const uint8_t* data, int64_t rows, uint8_t* views) {
    for (int64_t r = 0; r < rows; ++r) {
        uint8_t* v = views + (size_t)r * 16;
        const int32_t o = off[r], len = off[r + 1] - o;
        memset(v, 0, 16);
        memcpy(v, &len, 4);
        if (len <= 12) {
            memcpy(v + 4, data + o, (size_t)len);
        } else {
            const int32_t zero = 0;
            memcpy(v + 4, data + o, 4);
            memcpy(v + 8, &zero, 4);
            memcpy(v + 12, &o, 4);
        }
    }
}

// List<Utf8 / Binary> rows [lo, lo + n) -> the hidden device columns' host staging:
//   len_off[n + 1]   byte offsets of every row into the LENGTHS column (4 bytes per child element)
//   bytes_off[n + 1] byte offsets of every row into the child strings' bytes (relative to the first element's first byte)
//   lengths[ne]      int32 length of every child element
//   valid_off[n + 1], valid_bytes[ne]  (optional: pass nullptr) one validity byte per child element
// `loff` = the list's int32 offsets, `coff` = the child's int32 offsets already advanced by the child's array offset,
// `cvalid` / `cvalid_offset` = the child's validity bitmap (nullptr: all valid) and the child's array offset.
// Returns the number of child elements ne (callers size lengths / valid_bytes with loff[lo + n] - loff[lo] beforehand).
inline int64_t split_list_rows(const int32_t* loff, const int32_t* coff, const uint8_t* cvalid, int64_t cvalid_offset, int64_t lo, int64_t n,
                               int32_t* len_off, int32_t* bytes_off, int32_t* lengths, int32_t* valid_off, char* valid_bytes) {
    const int64_t e0 = loff[lo], e1 = loff[lo + n], ne = e1 - e0;
    for (int64_t r = 0; r <= n; ++r) {
        len_off[r] = (int32_t)(4 * ((int64_t)loff[lo + r] - e0));
        bytes_off[r] = coff[loff[lo + r]] - coff[e0];
    }
    for (int64_t k = 0; k < ne; ++k) lengths[k] = coff[e0 + k + 1] - coff[e0 + k];
    if (valid_off) {
        for (int64_t r = 0; r <= n; ++r) valid_off[r] = (int32_t)((int64_t)loff[lo + r] - e0);
        if (!cvalid) {
            memset(valid_bytes, 1, (size_t)ne);
        } else {
            // bits [first, first + ne) of the child's validity -> one byte each: bit by bit up to a byte boundary of the
            // bitmap, then eight at a time (byte b -> 8 bytes: replicate, isolate bit i in byte i, normalise to 0 / 1)
            const int64_t first = cvalid_offset + e0;
            int64_t k = 0;
            for (; k < ne && ((first + k) & 7); ++k) valid_bytes[k] = (char)((cvalid[(first + k) >> 3] >> ((first + k) & 7)) & 1);
            const uint8_t* src = cvalid + ((first + k) >> 3);
            for (; k + 8 <= ne; k += 8, ++src) {
                const uint64_t spread = ((uint64_t)*src * 0x0101010101010101ULL) & 0x8040201008040201ULL;
                const uint64_t ones = ((spread + 0x7f7f7f7f7f7f7f7fULL) >> 7) & 0x0101010101010101ULL;  // byte i = 1 iff byte i of spread != 0
                memcpy(valid_bytes + k, &ones, 8);  // (little endian: byte 0 = bit 0)
            }
            for (; k < ne; ++k) valid_bytes[k] = (char)((cvalid[(first + k) >> 3] >> ((first + k) & 7)) & 1);
        }
    }
    return ne;
}

// List<fixed-width primitive> rows (child values of `w` bytes, no child offsets): the same three hidden columns — every element
// still owns one int32 in the LENGTHS column (its value, w, is not used: the column is what carries the per-row element counts
// and the list's validity through the scatter), the BYTES column is the rows' contiguous ranges of the child's values buffer.
inline int64_t split_list_rows_fixed(const int32_t* loff, int32_t w, const uint8_t* cvalid, int64_t cvalid_offset, int64_t lo, int64_t n, int32_t* len_off,
                                     int32_t* bytes_off, int32_t* lengths, int32_t* valid_off, char* valid_bytes) {
    const int64_t e0 = loff[lo], e1 = loff[lo + n], ne = e1 - e0;
    for (int64_t r = 0; r <= n; ++r) {
        const int64_t k = (int64_t)loff[lo + r] - e0;
        len_off[r] = (int32_t)(4 * k);
        bytes_off[r] = (int32_t)(k * w);
        if (valid_off) valid_off[r] = (int32_t)k;
    }
    for (int64_t k = 0; k < ne; ++k) lengths[k] = w;
    if (valid_off) {
        if (!cvalid) {
            memset(valid_bytes, 1, (size_t)ne);
        } else {
            const int64_t first = cvalid_offset + e0;
            for (int64_t k = 0; k < ne; ++k) valid_bytes[k] = (char)((cvalid[(first + k) >> 3] >> ((first + k) & 7)) & 1);
        }
    }
    return ne;
}

// FixedSizeList<T, n> rows [lo, lo + rows) (lo counts the parent's array offset) over a child at array offset `child_offset`
// (counted in elements, as every Arrow offset): the child elements they span, child_offset + lo x n onwards, as bits (the
// child's validity bitmap, or its values when T is Boolean) and as bytes of a child of w bytes per element (w = 0: Boolean).
struct FslSpan {
    int64_t first_bit, n_bits;
    size_t first_byte, n_bytes;
};
inline FslSpan fsl_span(int64_t child_offset, int64_t lo, int64_t rows, int64_t n, int64_t w) {
    const int64_t e0 = child_offset + lo * n, ne = rows * n;
    return FslSpan{e0, ne, (size_t)(e0 * w), (size_t)(ne * w)};
}

// Do two flat Arrow arrays hold the same values?  (dictionaries of consecutive batches: readers re-materialise the same
// dictionary for every batch, and a chunk can keep ONE of them for all its rows.)  `var_ow` = 0 for fixed-width values of
// `width` bytes (0 = bit-packed booleans), 4 / 8 for Utf8 / Binary / LargeUtf8 offsets.  Buffers follow the Arrow C layout:
// validity (may be NULL = all valid), then values, or offsets + data.  Null slots compare equal whatever lies under them.
inline bool flat_arrays_equal(int64_t length, int var_ow, int width, const void* const* a_bufs, int64_t a_offset, int64_t a_nulls, const void* const* b_bufs,
                              int64_t b_offset, int64_t b_nulls) {
    const uint8_t* av = a_nulls != 0 ? (const uint8_t*)a_bufs[0] : nullptr;
    const uint8_t* bv = b_nulls != 0 ? (const uint8_t*)b_bufs[0] : nullptr;
    auto valid = [](const uint8_t* v, int64_t i) { return !v || ((v[i >> 3] >> (i & 7)) & 1); };
    for (int64_t i = 0; i < length; ++i) {
        const bool x = valid(av, a_offset + i), y = valid(bv, b_offset + i);
        if (x != y) return false;
        if (!x) continue;
        if (var_ow == 0 && width == 0) {  // booleans
            if (valid((const uint8_t*)a_bufs[1], a_offset + i) != valid((const uint8_t*)b_bufs[1], b_offset + i)) return false;
        } else if (var_ow == 0) {
            if (memcmp((const char*)a_bufs[1] + (size_t)(a_offset + i) * (size_t)width, (const char*)b_bufs[1] + (size_t)(b_offset + i) * (size_t)width, (size_t)width) != 0)
                return false;
        } else {
            int64_t a0, a1, b0, b1;
            if (var_ow == 8) {
                a0 = ((const int64_t*)a_bufs[1])[a_offset + i]; a1 = ((const int64_t*)a_bufs[1])[a_offset + i + 1];
                b0 = ((const int64_t*)b_bufs[1])[b_offset + i]; b1 = ((const int64_t*)b_bufs[1])[b_offset + i + 1];
            } else {
                a0 = ((const int32_t*)a_bufs[1])[a_offset + i]; a1 = ((const int32_t*)a_bufs[1])[a_offset + i + 1];
                b0 = ((const int32_t*)b_bufs[1])[b_offset + i]; b1 = ((const int32_t*)b_bufs[1])[b_offset + i + 1];
            }
            if (a1 - a0 != b1 - b0) return false;
            if (a1 > a0 && memcmp((const char*)a_bufs[2] + a0, (const char*)b_bufs[2] + b0, (size_t)(a1 - a0)) != 0) return false;
        }
    }
    return true;
}

}  // namespace host
}  // namespace dfd
