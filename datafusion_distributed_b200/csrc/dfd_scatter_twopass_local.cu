// dfd_scatter_twopass_local.cu — two-pass k_scatter (K1 tiling) instantiations, local mode (see dfd_launch.cuh).
#include "dfd_launch.cuh"

namespace dfd {
template int launch_scatter_impl<false, ScatterKind::TwoPass>(const ScatterParams&, int, bool, int, cudaStream_t);
}  // namespace dfd
