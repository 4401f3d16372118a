// dfd_scatter_follow_local.cu — follow-up k_scatter on the single-pass tiling instantiations, local mode (see dfd_launch.cuh).
#include "dfd_launch.cuh"

namespace dfd {
template int launch_scatter_impl<false, ScatterKind::FollowUp>(const ScatterParams&, int, bool, int, cudaStream_t);
}  // namespace dfd
