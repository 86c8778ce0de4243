// k_wide.cu — warp-per-instance kernels (sim_core.cuh G = 32): small batches and large committees.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_wide(const KernelSel& k, const Params& P, cudaStream_t stream) {
  // QMODE 2 also with the instance state in shared memory; 64 authors on the calendar queue also with the compile-time
  // layout of BASELINE configs[3]
  using Special = Kernels<WideKernel<16, 2, true, 8>, WideKernel<16, 2, true, 32>, WideKernel<64, 3, false, 8, false, FX_COMMITTEE64>>;
  return launch_listed<Kernels<Special, WideVariants<16, 2>, WideVariants<16, 1>, WideVariants<16, 3>, WideVariants<32, 3>,
                               WideVariants<64, 3>, WideVariants<16, 0>, WideVariants<32, 0>, WideVariants<64, 0>>>(k, P, stream);
}
}  // namespace lbft
