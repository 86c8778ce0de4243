// k_scan.cu — thread-per-instance kernels over the scan queues (QMODE 1: 64-bit keys in HBM, QMODE 2: 32-bit keys in shared
// memory), committees of <= 5, with their recording / resumable variants.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_scan(const KernelSel& k, const Params& P, cudaStream_t stream) {
  return launch_listed<Kernels<ThreadVariants<16, 2>, ThreadVariants<16, 1>>>(k, P, stream);
}
}  // namespace lbft
