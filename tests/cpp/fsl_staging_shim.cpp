// Test-only C wrapper around the host operator's FixedSizeList staging arithmetic (csrc/dfd_host_staging.h), compiled with
// plain g++ by tests/test_fixed_size_list_cpu.py: the child range of a piece of rows, and its bit rows appended to a chunk.
#include "dfd_host_staging.h"

extern "C" {
void t_fsl_span(int64_t child_offset, int64_t lo, int64_t rows, int64_t n, int64_t w, int64_t* out) {
    const dfd::host::FslSpan s = dfd::host::fsl_span(child_offset, lo, rows, n, w);
    out[0] = s.first_bit;
    out[1] = s.n_bits;
    out[2] = (int64_t)s.first_byte;
    out[3] = (int64_t)s.n_bytes;
}
// rows [lo, lo + rows) of a FixedSizeList<*, n> whose bitmap `src` (child validity or Boolean values; NULL = all ones) starts
// at the child's array offset, appended at row `at` of the chunk's bit-row bitmap `dst` (what stage_rows_host does)
void t_append_bit_rows(uint8_t* dst, int64_t at, const uint8_t* src, int64_t child_offset, int64_t lo, int64_t rows, int64_t n) {
    const dfd::host::FslSpan s = dfd::host::fsl_span(child_offset, lo, rows, n, 0);
    dfd::host::append_bits(dst, at * n, src, s.first_bit, s.n_bits);
}
}
