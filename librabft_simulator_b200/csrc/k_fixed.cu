// k_fixed.cu — the bench kernel: four authors, default capacities, the reference's own delay model; layout is a compile-time
// constant (sim_core.cuh FIXED).  BASELINE configs[2].
#include "kernels.cuh"
namespace lbft {
cudaError_t launch_fixed(const KernelSel& k, const Params& P, cudaStream_t stream) {
  if (k.wide || k.fixed != FX_DEFAULT4 || k.qmode != 2) return cudaErrorInvalidValue;
  constexpr int T = LaunchShape<2>::kThreads;
  const size_t dyn = (size_t)(T / 32) * 64 * (32 * 4 + 32 * 2);
  if (k.tile == 8) {  // sparse tiles: eight instances per warp (batches too small to fill the GPU with full warps)
    const uint32_t tiles = (P.num_instances + 7) / 8;
    return launch_thread<16, 2, FX_DEFAULT4, false, false, false, false, 8>((tiles * 32 + T - 1) / T, dyn, P, stream);
  }
  if (k.tile != 32) return cudaErrorInvalidValue;
  return launch_thread<16, 2, FX_DEFAULT4>((P.num_instances + T - 1) / T, dyn, P, stream);
}
}  // namespace lbft
