// k_fixed.cu — the bench kernel: four authors, default capacities, the reference's own delay model; layout is a compile-time
// constant (sim_core.cuh FIXED).  BASELINE configs[2].
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_fixed(const KernelSel& k, const Params& P, cudaStream_t stream) {
  return launch_listed<Kernels<ThreadKernel<16, 2, FX_DEFAULT4>>>(k, P, stream);
}
}  // namespace lbft
