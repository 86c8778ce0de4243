// k_ct_wide.cu — the commit-times twins (LBFT_FLAG_COMMIT_TIMES) of the single-epoch warp-per-instance kernels: the three
// special shapes and both HBM lane groups of every queue mode.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_ct_wide(const KernelSel& k, const CtParams<Params>& C, cudaStream_t stream) {
  using Special = Kernels<WideKernel<16, 2, true, 8, false, FX_NONE, false, true>, WideKernel<16, 2, true, 32, false, FX_NONE, false, true>,
                          WideKernel<64, 3, false, 8, false, FX_COMMITTEE64, false, true>>;
  return launch_listed<Kernels<Special, CtWideVariants<16, 2, false>, CtWideVariants<16, 1, false>, CtWideVariants<16, 3, false>,
                               CtWideVariants<32, 3, false>, CtWideVariants<64, 3, false>, CtWideVariants<16, 0, false>,
                               CtWideVariants<32, 0, false>, CtWideVariants<64, 0, false>>>(k, C, stream);
}
}  // namespace lbft
