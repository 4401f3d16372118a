// dfd_scatter_twopass_peer.cu — two-pass k_scatter (K1 tiling) instantiations, peer-store (fused exchange) mode (see dfd_launch.cuh).
#include "dfd_launch.cuh"

namespace dfd {
template int launch_scatter_impl<true, ScatterKind::TwoPass>(const ScatterParams&, int, bool, int, cudaStream_t);
}  // namespace dfd
