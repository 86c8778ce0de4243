// k_sweep_wide.cu — warp-per-instance kernels of sweep handles (lbft_create_sweep): the twin of every plain generic wide
// instantiation (both lane groups with the state in HBM, and the two with the instance in shared memory).
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_sweep_wide(const KernelSel& k, const SweepParams& S, cudaStream_t stream) {
  using Smem = Kernels<WideKernel<16, 2, true, 8, false, FX_NONE, true>, WideKernel<16, 2, true, 32, false, FX_NONE, true>>;
  return launch_listed<Kernels<Smem, SweepWideVariants<16, 2>, SweepWideVariants<16, 1>, SweepWideVariants<16, 3>, SweepWideVariants<32, 3>,
                               SweepWideVariants<64, 3>, SweepWideVariants<16, 0>, SweepWideVariants<32, 0>, SweepWideVariants<64, 0>>>(k, S, stream);
}
}  // namespace lbft
