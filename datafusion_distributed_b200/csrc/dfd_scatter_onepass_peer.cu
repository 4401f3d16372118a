// dfd_scatter_onepass_peer.cu — single-pass k_scatter_onepass instantiations, peer-store (fused exchange) mode (see dfd_launch.cuh).
#include "dfd_launch.cuh"

namespace dfd {
template int launch_scatter_impl<true, ScatterKind::OnePass>(const ScatterParams&, int, bool, int, cudaStream_t);
}  // namespace dfd
