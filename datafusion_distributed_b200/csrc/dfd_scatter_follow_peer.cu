// dfd_scatter_follow_peer.cu — follow-up k_scatter on the single-pass tiling instantiations, peer-store (fused exchange) mode (see dfd_launch.cuh).
#include "dfd_launch.cuh"

namespace dfd {
template int launch_scatter_impl<true, ScatterKind::FollowUp>(const ScatterParams&, int, bool, int, cudaStream_t);
}  // namespace dfd
