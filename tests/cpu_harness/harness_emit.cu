// TEST INFRASTRUCTURE (CPU suite only): the launch that finishes a device-output chunk (csrc/dfd_emit.cu) restated on the
// host with dfd_host_staging.h, job by job, for the device-output harness that
// tests/test_exec_device_output_cpu_harness.py links (the product's dfd_exec object + harness_dfd.cu + harness_stage.cu +
// fake_cudart.cpp + this file).  Pointers named "device" are host pointers here.
#include <cstdint>

#include "dfd_host_staging.h"
#include "dfd_internal.h"

int dfd::launch_emit_chunk(const EmitJob* jobs, int n_jobs, cudaStream_t) {
    for (int k = 0; k < n_jobs; ++k) {
        const EmitJob& j = jobs[k];
        if (j.op == EMIT_VIEWS) {
            dfd::host::build_views((const int32_t*)j.off, (const uint8_t*)j.bytes, j.n, (uint8_t*)j.dst);
            *(int64_t*)j.dst2 = ((const int32_t*)j.off)[j.n];
        } else if (j.op == EMIT_LIST_OFFSETS) {
            for (int64_t r = 0; r <= j.n; ++r) ((int32_t*)j.dst)[r] >>= 2;
        } else {
            return set_error(DFD_ERR_INTERNAL, "emit job %d: unknown op %d", k, j.op);
        }
    }
    return DFD_OK;
}
