// k_sweep_thread.cu — thread-per-instance kernels of sweep handles (lbft_create_sweep): the twin of every plain generic
// thread instantiation, full tiles over each queue mode and the two sparse tiles over the calendar queue.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_sweep_thread(const KernelSel& k, const SweepParams& S, cudaStream_t stream) {
  using SparseTiles = Kernels<ThreadKernel<16, 3, FX_NONE, false, false, false, false, 8, true>,
                              ThreadKernel<16, 3, FX_NONE, false, false, false, false, 16, true>>;
  return launch_listed<Kernels<SparseTiles, SweepThread<16, 2>, SweepThread<16, 1>, SweepThread<16, 3>, SweepThread<32, 3>,
                               SweepThread<64, 3>, SweepThread<16, 0>, SweepThread<32, 0>, SweepThread<64, 0>>>(k, S, stream);
}
}  // namespace lbft
