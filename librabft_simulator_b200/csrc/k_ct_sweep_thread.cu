// k_ct_sweep_thread.cu — the commit-times twins (LBFT_FLAG_COMMIT_TIMES) of every sweep thread-per-instance kernel.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_ct_sweep_thread(const KernelSel& k, const CtParams<SweepParams>& C, cudaStream_t stream) {
  using SparseTiles = Kernels<ThreadKernel<16, 3, FX_NONE, false, false, false, false, 8, true, true>,
                              ThreadKernel<16, 3, FX_NONE, false, false, false, false, 16, true, true>>;
  return launch_listed<Kernels<SparseTiles, CtThread<16, 2, true>, CtThread<16, 1, true>, CtThread<16, 3, true>, CtThread<32, 3, true>,
                               CtThread<64, 3, true>, CtThread<16, 0, true>, CtThread<32, 0, true>, CtThread<64, 0, true>>>(k, C, stream);
}
}  // namespace lbft
