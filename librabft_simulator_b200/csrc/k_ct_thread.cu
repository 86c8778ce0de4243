// k_ct_thread.cu — the commit-times twins (LBFT_FLAG_COMMIT_TIMES) of the one-shot single-epoch thread-per-instance kernels:
// the bench kernel, the three sparse tiles over the calendar queue and the full-tile generic kernel of every queue mode.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_ct_thread(const KernelSel& k, const CtParams<Params>& C, cudaStream_t stream) {
  using Fixed = ThreadKernel<16, 2, FX_DEFAULT4, false, false, false, false, 32, false, true>;
  using SparseTiles = Kernels<ThreadKernel<16, 3, FX_PART7, false, false, false, false, 8, false, true>,
                              ThreadKernel<16, 3, FX_NONE, false, false, false, false, 8, false, true>,
                              ThreadKernel<16, 3, FX_NONE, false, false, false, false, 16, false, true>>;
  return launch_listed<Kernels<Fixed, SparseTiles, CtThread<16, 2, false>, CtThread<16, 1, false>, CtThread<16, 3, false>,
                               CtThread<32, 3, false>, CtThread<64, 3, false>, CtThread<16, 0, false>, CtThread<32, 0, false>,
                               CtThread<64, 0, false>>>(k, C, stream);
}
}  // namespace lbft
