// k_ct_sweep_wide.cu — the commit-times twins (LBFT_FLAG_COMMIT_TIMES) of every sweep warp-per-instance kernel.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_ct_sweep_wide(const KernelSel& k, const CtParams<SweepParams>& C, cudaStream_t stream) {
  using Smem = Kernels<WideKernel<16, 2, true, 8, false, FX_NONE, true, true>, WideKernel<16, 2, true, 32, false, FX_NONE, true, true>>;
  return launch_listed<Kernels<Smem, CtWideVariants<16, 2, true>, CtWideVariants<16, 1, true>, CtWideVariants<16, 3, true>,
                               CtWideVariants<32, 3, true>, CtWideVariants<64, 3, true>, CtWideVariants<16, 0, true>,
                               CtWideVariants<32, 0, true>, CtWideVariants<64, 0, true>>>(k, C, stream);
}
}  // namespace lbft
