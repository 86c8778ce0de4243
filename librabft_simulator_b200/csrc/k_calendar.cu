// k_calendar.cu — thread-per-instance kernels over the calendar queue (QMODE 3), committees of 6..64.
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_calendar(const KernelSel& k, const Params& P, cudaStream_t stream) {
  // sparse tiles: plain kernels for committees of 6..16, among them the seven-author partition shape (BASELINE configs[4])
  using SparseTiles = Kernels<ThreadKernel<16, 3, FX_PART7, false, false, false, false, 8>, ThreadKernel<16, 3, FX_NONE, false, false, false, false, 8>,
                              ThreadKernel<16, 3, FX_NONE, false, false, false, false, 16>>;
  return launch_listed<Kernels<SparseTiles, ThreadVariants<16, 3>, ThreadVariants<32, 3>, ThreadVariants<64, 3>>>(k, P, stream);
}
}  // namespace lbft
