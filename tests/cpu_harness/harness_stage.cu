// TEST INFRASTRUCTURE (CPU suite only): the two staging launches of device-resident input (csrc/dfd_stage.cu) restated
// on the host with dfd_host_staging.h, job by job, for the device-input harness that
// tests/test_exec_device_input_cpu_harness.py links (the product's dfd_exec object + harness_dfd.cu + fake_cudart.cpp +
// this file).  Pointers named "device" are host pointers here.
#include <cstdint>
#include <cstring>

#include "dfd_host_staging.h"
#include "dfd_internal.h"

namespace {
inline bool bit(const uint8_t* b, int64_t i) { return (b[i >> 3] >> (i & 7)) & 1; }
inline int64_t off_at(const void* p, int ow, int64_t i) { return ow == 8 ? ((const int64_t*)p)[i] : (int64_t)((const int32_t*)p)[i]; }
}  // namespace

int dfd::launch_stage_batch(const StageJob* jobs, int n_jobs, cudaStream_t) {
    for (int k = 0; k < n_jobs; ++k) {
        const StageJob& j = jobs[k];
        switch (j.op) {
            case STAGE_COPY:
                if (j.n) memcpy(j.dst, j.src, (size_t)j.n);
                break;
            case STAGE_BITS:
                if (j.c < j.b) dfd::host::append_bits((uint8_t*)j.dst, j.c, nullptr, 0, j.b - j.c);
                dfd::host::append_bits((uint8_t*)j.dst, j.b, (const uint8_t*)j.src, j.a, j.n);
                break;
            case STAGE_OFFSETS:
                for (int64_t r = 0; r <= j.n; ++r) {
                    const int64_t v = j.base + j.scale * (off_at(j.src, j.ow_in, r) - off_at(j.src, j.ow_in, 0));
                    if (j.ow_out == 8) ((int64_t*)j.dst)[r] = v;
                    else ((int32_t*)j.dst)[r] = (int32_t)v;
                }
                break;
            case STAGE_LIST_OFFSETS: {
                const int32_t* l = (const int32_t*)j.src;
                const int32_t* c = (const int32_t*)j.src2;
                for (int64_t r = 0; r <= j.n; ++r) ((int32_t*)j.dst)[r] = (int32_t)(j.base + c[l[r]] - c[l[0]]);
                break;
            }
            case STAGE_DIFF32:
                for (int64_t i = 0; i < j.n; ++i) ((int32_t*)j.dst)[i] = ((const int32_t*)j.src)[i + 1] - ((const int32_t*)j.src)[i];
                break;
            case STAGE_FILL32:
                for (int64_t i = 0; i < j.n; ++i) ((int32_t*)j.dst)[i] = (int32_t)j.base;
                break;
            case STAGE_BIT_BYTES:
                for (int64_t i = 0; i < j.n; ++i) ((uint8_t*)j.dst)[i] = j.src ? (uint8_t)bit((const uint8_t*)j.src, j.a + i) : (uint8_t)1;
                break;
            case STAGE_VIEW_BYTES:
                dfd::host::view_bytes((const uint8_t*)j.src, (const void* const*)j.src2, 0, j.n, (const int32_t*)j.src3, (char*)j.dst);
                break;
            default:
                return set_error(DFD_ERR_INTERNAL, "stage job %d: unknown op %d", k, j.op);
        }
    }
    return DFD_OK;
}

int dfd::launch_stage_sizes(const StageSize* jobs, int n_jobs, cudaStream_t) {
    for (int k = 0; k < n_jobs; ++k) {
        const StageSize& j = jobs[k];
        if (j.op == STAGE_SIZE_VIEW) {
            int64_t total = 0;  // (lengths of the views, a null row as 0)
            for (int64_t r = 0; r < j.n; ++r) {
                int32_t len;
                memcpy(&len, (const uint8_t*)j.off + (size_t)(j.lo + r) * 16, 4);
                if (j.valid && !bit(j.valid, j.lo + r)) len = 0;
                j.lens[r] = len;
                total += len;
            }
            j.out[0] += total;
            continue;
        }
        const int64_t a = off_at(j.off, j.ow, j.lo), b = off_at(j.off, j.ow, j.lo + j.n);
        j.out[0] = a;
        j.out[1] = b;
        if (j.op == STAGE_SIZE_LIST && j.off2 && a >= 0 && b >= a) {
            j.out[2] = ((const int32_t*)j.off2)[a];
            j.out[3] = ((const int32_t*)j.off2)[b];
        }
    }
    return DFD_OK;
}
