// sampler_probe.cu — TEST INFRASTRUCTURE: runs the device sampler (sim_core.cuh Core: Xoshiro256** seeding and steps, rand's
// range draws, the 256-layer ziggurat with its wedge and tail, the threshold walk of delay_from_z and every branch of
// sample_delay) on records with an explicit state each (sampler_ops.cuh), so that inputs a whole run reaches once in millions of
// draws, or never, reach it directly.  The cores are the kernels' own instantiations: the generic plain core, the bench
// kernel's FX_DEFAULT4 core and the sweep core bound to its record's parameter set, with G = 1, 8 or 32 lanes per record (every
// lane computes the record; the probe flags a group whose lanes disagree).  The tables are the product's and are read where
// the kernels read them: the ziggurat layers, and the thresholds when place_delay_thresholds puts them there, from shared
// memory as the thread kernels do, or all from global memory as the wide kernels do.  Built by _build.build_sampler_probe();
// never part of, linked into, or reachable from the product library.
#include <cuda_runtime.h>

#include "../../librabft_simulator_b200/csrc/kernels.cuh"
#include "sampler_ops.cuh"

namespace {

using sampler::Rec;
constexpr uint32_t kBlock = 128;

template <uint32_t CK, int G>
struct CoreOf;
template <int G>
struct CoreOf<sampler::CORE_PLAIN, G> {  // lbft_event_loop_kernel's generic core (G = 1), lbft_wide_kernel's (G = 8, 32)
  using type = typename std::conditional<G == 1, lbft::Core<lbft::TileMem<32>, 16, 3>, lbft::Core<lbft::TileMem<1>, 64, 1, lbft::FX_NONE, false, false, G>>::type;
};
template <int G>
struct CoreOf<sampler::CORE_FIXED, G> {  // the bench kernel's
  static_assert(G == 1, "the compile-time layout is a thread kernel's");
  using type = lbft::Core<lbft::TileMem<32, true>, 16, 2, lbft::FX_DEFAULT4>;
};
template <int G>
struct CoreOf<sampler::CORE_SWEEP, G> {  // lbft_sweep_event_loop_kernel's (G = 1), lbft_sweep_wide_kernel's (G = 8, 32)
  using type = typename std::conditional<G == 1, lbft::Core<lbft::TileMem<32>, 16, 3, lbft::FX_NONE, false, false, 1, false, false, false, true>,
                                         lbft::Core<lbft::TileMem<1>, 64, 1, lbft::FX_NONE, false, false, G, false, false, false, true>>::type;
};

std::string g_err;

template <uint32_t CK, int G, bool SMEM>
__global__ void __launch_bounds__(kBlock) sampler_probe_kernel(const __grid_constant__ lbft::Params P, const lbft::SweepSet* sets, uint64_t n,
                                                               Rec* recs) {
  constexpr bool SW = CK == sampler::CORE_SWEEP;
  __shared__ double s_zx[257];
  __shared__ double s_zf[257];
  __shared__ double s_thr[lbft::kThrSmem];
  const double *zx = P.zig_x, *zf = P.zig_f, *thr = P.delay_thr;
  if (SMEM) {  // as event_loop_body
    for (int i = threadIdx.x; i < 257; i += blockDim.x) {
      s_zx[i] = P.zig_x[i];
      s_zf[i] = P.zig_f[i];
    }
    const bool thr_fits = lbft::place_delay_thresholds<SW>(P, s_thr);
    __syncthreads();
    zx = s_zx;
    zf = s_zf;
    thr = thr_fits ? s_thr : P.delay_thr;
  }
  const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  if (i >= n) return;  // (whole groups)
  typename CoreOf<CK, G>::type core(P, {nullptr, 0}, zx, zf, thr);
  Rec r = recs[i];
  if constexpr (SW) core.bind_set(lbft::sweep_set_at(sets, r.set, 0));
  sampler::run_op(core, r);
  if constexpr (G > 1) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gm = G == 32 ? 0xffffffffu : ((1u << G) - 1u) << (lane & ~(uint32_t)(G - 1));
    const uint64_t w[7] = {r.s[0], r.s[1], r.s[2], r.s[3], r.result, r.draws, r.status};
    bool same = true;
    for (int k = 0; k < 7; k++) same &= __shfl_sync(gm, (unsigned long long)w[k], 0, G) == w[k];
    if (!__all_sync(gm, same)) r.status |= sampler::kLanesDisagree;
    if (threadIdx.x % G) return;
  }
  recs[i] = r;
}

template <uint32_t CK, int G, bool SMEM>
cudaError_t launch(const lbft::Params& P, const lbft::SweepSet* sets, uint64_t n, Rec* recs) {
  const uint64_t blocks = (n * G + kBlock - 1) / kBlock;
  sampler_probe_kernel<CK, G, SMEM><<<(unsigned)blocks, kBlock>>>(P, sets, n, recs);
  return cudaGetLastError();
}

template <uint32_t CK>
cudaError_t launch_core(uint32_t G, bool smem, const lbft::Params& P, const lbft::SweepSet* sets, uint64_t n, Rec* recs) {
  if (G == 1) return smem ? launch<CK, 1, true>(P, sets, n, recs) : launch<CK, 1, false>(P, sets, n, recs);
  if constexpr (CK != sampler::CORE_FIXED) {
    if (G == 8) return smem ? launch<CK, 8, true>(P, sets, n, recs) : launch<CK, 8, false>(P, sets, n, recs);
    if (G == 32) return smem ? launch<CK, 32, true>(P, sets, n, recs) : launch<CK, 32, false>(P, sets, n, recs);
  }
  return cudaErrorInvalidValue;
}

template <class T>
cudaError_t upload(T** d, const T* h, size_t count) {
  cudaError_t e = cudaMalloc(d, (count ? count : 1) * sizeof(T));
  if (e == cudaSuccess && count) e = cudaMemcpy(*d, h, count * sizeof(T), cudaMemcpyHostToDevice);
  return e;
}

}  // namespace

extern "C" {

const char* sampler_probe_last_error() { return g_err.c_str(); }

// Runs recs[0..n) on the device with `core` (sampler_ops.cuh CORE_*), G lanes per record (1, 8 or 32; the fixed core: 1), the
// tables in shared memory (smem != 0) or global memory, over the setup of `c` (sets == NULL) or of a sweep of `c` over
// sets[0..num_sets).  0, or -1 for a configuration or record out of range (sampler_ops.cuh check_records), -4 for a CUDA
// error (read either with sampler_probe_last_error).
int sampler_probe(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, uint32_t core, uint32_t G, uint32_t smem,
                  Rec* recs, uint64_t n) {
  lbft::HostSetup hs;
  if (!sampler::make_setup(c, sets, num_sets, hs, g_err) || !sampler::check_records(hs, core, recs, n, g_err)) return -1;
  if (!(G == 1 || ((G == 8 || G == 32) && core != sampler::CORE_FIXED))) {
    g_err = "G must be 1, 8 or 32 (the fixed core: 1)";
    return -1;
  }
  if (n == 0) return 0;
  lbft::Params P = hs.params;
  const std::vector<uint64_t> table = hs.set_table();
  double *d_zx = nullptr, *d_zf = nullptr, *d_thr = nullptr;
  uint64_t* d_sets = nullptr;
  Rec* d_recs = nullptr;
  const char* step = "upload";
  cudaError_t e = cudaSuccess;
  if ((e = upload(&d_zx, hs.zig_x.data(), hs.zig_x.size())) || (e = upload(&d_zf, hs.zig_f.data(), hs.zig_f.size())) ||
      (e = upload(&d_thr, hs.delay_thr.data(), hs.delay_thr.size())) || (e = upload(&d_sets, table.data(), table.size())) ||
      (e = upload(&d_recs, recs, n)))
    goto done;
  P.zig_x = d_zx;
  P.zig_f = d_zf;
  P.delay_thr = d_thr;
  step = "sampler_probe_kernel";
  {
    const lbft::SweepSet* S = reinterpret_cast<const lbft::SweepSet*>(d_sets);
    e = core == sampler::CORE_PLAIN   ? launch_core<sampler::CORE_PLAIN>(G, smem, P, S, n, d_recs)
        : core == sampler::CORE_FIXED ? launch_core<sampler::CORE_FIXED>(G, smem, P, S, n, d_recs)
                                      : launch_core<sampler::CORE_SWEEP>(G, smem, P, S, n, d_recs);
  }
  if (e || (e = cudaDeviceSynchronize())) goto done;
  step = "cudaMemcpy to the host";
  e = cudaMemcpy(recs, d_recs, n * sizeof(Rec), cudaMemcpyDeviceToHost);
done:
  if (e) g_err = std::string(step) + ": " + cudaGetErrorString(e);
  cudaFree(d_zx);
  cudaFree(d_zf);
  cudaFree(d_thr);
  cudaFree(d_sets);
  cudaFree(d_recs);
  return e ? -4 : 0;
}

}  // extern "C"
