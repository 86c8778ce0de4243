// k_heap.cu — thread-per-instance kernels over the binary heap (QMODE 0): long horizons / explicit large capacities.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_heap(const KernelSel& k, const Params& P, cudaStream_t stream) {
  return launch_listed<Kernels<ThreadVariants<16, 0>, ThreadVariants<32, 0>, ThreadVariants<64, 0>>>(k, P, stream);
}
}  // namespace lbft
