// dfd_scatter_onepass_local.cu — single-pass k_scatter_onepass instantiations, local mode (see dfd_launch.cuh).
#include "dfd_launch.cuh"

namespace dfd {
template int launch_scatter_impl<false, ScatterKind::OnePass>(const ScatterParams&, int, bool, int, cudaStream_t);
}  // namespace dfd

#ifdef DFD_ONEPASS_CLOCKS
// phase-clock build only (scripts/onepass_clocks.py): copies the local-mode kernel's per-phase cycle sums (OnePassClock order)
// to out[CLK_COUNT] after the device is idle, then clears them if `reset`.  The default build has no such export.
extern "C" int dfd_onepass_clocks(unsigned long long* out, int reset) {
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out, dfd::g_onepass_clocks, sizeof(unsigned long long) * dfd::CLK_COUNT);
    if (e == cudaSuccess && reset) {
        static const unsigned long long zero[dfd::CLK_COUNT] = {};
        e = cudaMemcpyToSymbol(dfd::g_onepass_clocks, zero, sizeof(zero));
    }
    return (int)e;
}
#endif
