// TEST INFRASTRUCTURE (CPU suite only): harness_dfd.cu with the host operator's FixedSizeList bit-row columns added, for the
// harness that tests/test_exec_fixed_size_list_cpu_harness.py links in its place (the product's dfd_exec object + this file +
// harness_stage.cu + harness_emit.cu + fake_cudart_events.cpp).  harness_dfd.cu's stand-in of partition_device_locked is
// compiled under another name; the one defined here hands it every other column plus an iota column (the product's d_src,
// the input row of every output row) and then gathers the COL_BIT_ROWS columns through it: the host stand-in of
// k_gather_bit_rows.  Pointers named "device" are host pointers here.
#define partition_device_locked partition_device_locked_without_bit_rows
#include "harness_dfd.cu"
#undef partition_device_locked

#include "dfd_host_staging.h"

namespace dfd {
int partition_device_locked(Partitioner* p, const dfd_column* in, int n_cols, int64_t n, const dfd_column* out, cudaStream_t stream,
                            bool var_bytes_known = false);
}

int dfd::partition_device_locked(Partitioner* p, const dfd_column* in, int n_cols, int64_t n, const dfd_column* out, cudaStream_t stream, bool known) {
    std::vector<dfd_column> rest_in, rest_out, bits_in, bits_out;
    for (int i = 0; i < n_cols; ++i) {
        if (in[i].kind == COL_BIT_ROWS && p->bit_rows) {
            bits_in.push_back(in[i]);
            bits_out.push_back(out[i]);
        } else {
            rest_in.push_back(in[i]);
            rest_out.push_back(out[i]);
        }
    }
    if (bits_in.empty()) return partition_device_locked_without_bit_rows(p, in, n_cols, n, out, stream, known);
    std::vector<uint32_t> iota((size_t)n + 1), src((size_t)n + 1);
    for (int64_t r = 0; r < n; ++r) iota[(size_t)r] = (uint32_t)r;
    rest_in.push_back(dfd_column{DFD_COL_FIXED, 4, iota.data(), nullptr, nullptr, 0, 0});
    rest_out.push_back(dfd_column{DFD_COL_FIXED, 4, src.data(), nullptr, nullptr, 0, 0});
    if (int rc = partition_device_locked_without_bit_rows(p, rest_in.data(), (int)rest_in.size(), n, rest_out.data(), stream, known)) return rc;
    KernelTime kernel_time;
    for (size_t k = 0; k < bits_in.size(); ++k) {
        const dfd_column& ic = bits_in[k];
        const dfd_column& oc = bits_out[k];
        const int64_t w = ic.width;
        memset(oc.values, 0, (size_t)((n * w + 31) / 32) * 4);  // (whole words, bits past the last row zero)
        for (int64_t j = 0; j < n; ++j)
            dfd::host::append_bits((uint8_t*)oc.values, j * w, (const uint8_t*)ic.values, ((int64_t)src[(size_t)j] + ic.offset) * w, w);
        if (ic.validity) {
            memset(oc.validity, 0, (size_t)((n + 31) / 32) * 4);
            for (int64_t j = 0; j < n; ++j)
                if (bit(ic.validity, (int64_t)src[(size_t)j] + ic.offset)) set_bit(oc.validity, j);
        }
        p->ctx->metrics.kernel_launches++;
    }
    return DFD_OK;
}
