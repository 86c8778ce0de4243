// block_threshold_probe.cu — TEST INFRASTRUCTURE: runs the lane form of the block threshold time (sim_core.cuh
// block_threshold_time_lanes, what the threshold overload of lbft_latency_stats_kernel runs per block) over synthetic
// commit-time tables, with the kernel's group shape: G lanes per instance, G the smallest power of two >= min(N, 32), 128 / G
// instances per block of 128 threads.  Tables that a real run cannot produce (ties everywhere, zero-weight first commits,
// weights at the 2^24 cap, a lone upper-half node) reach the device function this way.  Built by
// _build.build_block_threshold_probe(); never part of, linked into, or reachable from the product library.
#include <cuda_runtime.h>

#include <string>

#include "../../librabft_simulator_b200/csrc/sim_core.cuh"

namespace {

constexpr uint32_t kBlock = 128;  // lbft_api.cu kLatBlock

struct Weights {
  uint32_t w[64];  // in the parameter space, as Params::c_weights is for the kernel
};

std::string g_err;

// Instance i is a group of G lanes; for every row r < round_cap it takes k = r, so node n committed the block iff
// cc[i][n] > r, at times[i][n][r].  T[i][r]: the threshold time at W[i], INT64_MAX when unreached.
__global__ void __launch_bounds__(kBlock) block_threshold_probe_kernel(const __grid_constant__ Weights W8, lbft::Layout L, uint32_t G,
                                                                       uint32_t I, const uint32_t* cc, const int32_t* times,
                                                                       const uint32_t* W, int64_t* T) {
  const uint32_t per_block = kBlock / G;
  const uint32_t j = threadIdx.x & (G - 1);
  const uint32_t inst = blockIdx.x * per_block + threadIdx.x / G;
  if (inst >= I) return;  // (whole groups: an instance's lanes are all live or all not)
  const uint32_t N = L.num_nodes, R = L.round_cap;
  const uint32_t* icc = cc + (size_t)inst * N;
  const int32_t* t_inst = times + (size_t)inst * (N + 1) * R;
  const uint32_t warp_lane = threadIdx.x & 31;
  const uint32_t gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1u) << (warp_lane & ~(G - 1));
  const uint32_t cc0 = j < N ? icc[j] : 0u, cc1 = j + 32 < N ? icc[j + 32] : 0u;
  for (uint32_t r = 0; r < R; r++) {
    const int64_t t = lbft::block_threshold_time_lanes(L, G, gmask, j, cc0, cc1, t_inst, W8.w, r, r, W[inst]);
    if (j == 0) T[(size_t)inst * R + r] = t;
  }
}

int fail(const char* what, cudaError_t e) {
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return -4;
}

}  // namespace

extern "C" {

const char* block_threshold_probe_last_error() { return g_err.c_str(); }

// cc: [I][N] commit counts; times: [I][N + 1][round_cap] (row N, the proposed times, is not read); w: [N] voting rights
// (each <= 2^24); W: [I] thresholds; T: [I][round_cap] out.  0, or -1 for arguments out of range, -4 for a CUDA error (read
// with block_threshold_probe_last_error).
int block_threshold_probe(uint32_t N, uint32_t I, uint32_t round_cap, const uint32_t* cc, const int32_t* times, const uint32_t* w,
                          const uint32_t* W, int64_t* T) {
  if (N < 1 || N > 64 || I < 1 || round_cap < 1) {
    g_err = "N must be in 1..64, I and round_cap >= 1";
    return -1;
  }
  lbft::Layout L{};
  L.num_nodes = N;
  L.round_cap = round_cap;
  Weights W8{};
  for (uint32_t n = 0; n < N; n++) W8.w[n] = w[n];
  uint32_t G = 1;  // lbft_api.cu latency_stats: the smallest power of two >= min(N, 32)
  while (G < N && G < 32) G <<= 1;
  const size_t cc_bytes = (size_t)I * N * sizeof(uint32_t), t_bytes = (size_t)I * (N + 1) * round_cap * sizeof(int32_t),
               W_bytes = (size_t)I * sizeof(uint32_t), T_bytes = (size_t)I * round_cap * sizeof(int64_t);
  uint32_t *d_cc = nullptr, *d_W = nullptr;
  int32_t* d_t = nullptr;
  int64_t* d_T = nullptr;
  cudaError_t e = cudaSuccess;
  int rc = 0;
  const char* step = "cudaMalloc";
  if ((e = cudaMalloc(&d_cc, cc_bytes)) || (e = cudaMalloc(&d_t, t_bytes)) || (e = cudaMalloc(&d_W, W_bytes)) ||
      (e = cudaMalloc(&d_T, T_bytes)))
    goto done;
  step = "cudaMemcpy to the device";
  if ((e = cudaMemcpy(d_cc, cc, cc_bytes, cudaMemcpyHostToDevice)) || (e = cudaMemcpy(d_t, times, t_bytes, cudaMemcpyHostToDevice)) ||
      (e = cudaMemcpy(d_W, W, W_bytes, cudaMemcpyHostToDevice)))
    goto done;
  step = "block_threshold_probe_kernel";
  block_threshold_probe_kernel<<<(I + kBlock / G - 1) / (kBlock / G), kBlock>>>(W8, L, G, I, d_cc, d_t, d_W, d_T);
  if ((e = cudaGetLastError()) || (e = cudaDeviceSynchronize())) goto done;
  step = "cudaMemcpy to the host";
  e = cudaMemcpy(T, d_T, T_bytes, cudaMemcpyDeviceToHost);
done:
  if (e) rc = fail(step, e);
  cudaFree(d_cc);
  cudaFree(d_t);
  cudaFree(d_W);
  cudaFree(d_T);
  return rc;
}

}  // extern "C"
