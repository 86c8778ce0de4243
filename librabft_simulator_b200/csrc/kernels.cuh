// kernels.cuh — the two kernel templates over sim_core.cuh, their sweep twins and the per-translation-unit launchers.
//
//   lbft_event_loop_kernel<NMAX, QMODE, FIXED, REC, RES>   one THREAD per instance, 32 instances per warp tile (large batches)
//   lbft_wide_kernel<NMAX, QMODE>                          one WARP per instance (small batches, large committees)
//   lbft_sweep_event_loop_kernel / lbft_sweep_wide_kernel  the same bodies for sweep handles (lbft_create_sweep: per-instance
//                                                          delay model and NodeConfig; lbft_create_sweep_faults: and faults;
//                                                          lbft_create_sweep_rights: and voting rights;
//                                                          lbft_create_sweep_committees: and committee size;
//                                                          lbft_create_sweep_links: and link latencies;
//                                                          lbft_create_sweep_outages: and node outages)
//   lbft_ct_*_kernel                                       the same bodies with the commit-time stores (LBFT_FLAG_COMMIT_TIMES),
//                                                          a twin of every one-shot single-epoch plain and sweep kernel
//
// All do init -> event loop -> read-out in a single launch.  The instantiations are spread over several .cu files
// (k_fixed.cu, k_scan.cu, k_calendar.cu, k_heap.cu, k_wide.cu, k_sweep_thread.cu, k_sweep_wide.cu, k_ct_*.cu) so that they
// compile in parallel and the bench kernel can be rebuilt alone; lbft_api.cu only sees the launch_* functions declared at the end.
#pragma once
#include <cuda_runtime.h>

#include "host_setup.hpp"
#include "sim_core.cuh"

namespace lbft {

// The sparse-tile thread kernels keep the calendar's occupancy words in shared memory (sim_core.cuh KS); the wide kernels keep
// them in HBM: the words are L1-resident there anyway, and shared memory gains nothing.
LBFT_LAYOUT_FN uint32_t calendar_kmask_words(const Layout& L) { return (L.cal_times + 7) / 8; }

// Launch shapes of the thread-per-instance kernel: 16 warp tiles per SM, so that the 2 048 tiles of a 65 536-instance batch
// are resident in one wave on the 132 SMs of an H100 (14 per SM would leave 200 tiles for a second wave).  16 warps are four
// per SM sub-partition, i.e. <= 128 registers/thread — the bound ptxas already applies at 14.  QMODE 0/1/3: one-warp blocks.
// QMODE 2: four-warp blocks, 4 per SM, so that the ziggurat/threshold tables (6 KB) are shared by four tiles and the per-tile
// event queues (queue_cap x 32 x 6 B: 48 KB per block at queue_cap 64) fit in the 228 KB of shared memory of an SM.
template <int QMODE>
struct LaunchShape {
  static constexpr int kThreads = QMODE == 2 ? 32 * 4 : 32;  // QMODE 2: four warps per block share the 6 KB of tables
  static constexpr int kBlocksPerSm = QMODE == 2 ? 4 : 16;   // ... and four blocks per SM: 16 tiles per SM
};

// TILE: instances per warp tile.  32 fills every lane; 8 / 4 ("sparse" tiles: the other lanes of the warp retire at once) trade
// lanes for warps when the batch is too small to fill the GPU with full warps — the instances of a warp serialise through
// each other's code paths, so a warp of 8 instances finishes far sooner than a warp of 32, and four times as many warps hide
// each other's latency.  Plain kernels over the calendar queue and the shared-memory queue (whose columns keep their
// 32-entry pitch); the state layout interleaves TILE instances.
// Where a thread kernel's instances read the delay thresholds (Core::thr) from: the block's shared-memory copy `s_thr`, filled
// here by the block's threads, when the launch has a table of at most kThrSmem entries (returns true); the table in global
// memory otherwise, and always on a sweep (SW: the instances of one warp may belong to different sets, Core::bind_set).  The
// caller publishes the copy with a __syncthreads before the first read.
template <bool SW>
__device__ __forceinline__ bool place_delay_thresholds(const Params& P, double* s_thr) {
  const bool thr_fits = !SW && P.delay_kmax != 0 && P.delay_kmax + 2 <= kThrSmem;
  if (thr_fits)
    for (uint32_t i = threadIdx.x; i < P.delay_kmax + 2; i += blockDim.x) s_thr[i] = P.delay_thr[i];
  return thr_fits;
}
// The body of both thread kernels (lbft_event_loop_kernel, lbft_sweep_event_loop_kernel), given the kernel's shared memory.
// SW (sweep handles): the instance's parameter set supplies the delay model and NodeConfig, on a fault sweep (`records` bit 0:
// `sets` heads a SweepSetFaults table) the silent nodes and partition plan, and on a rights sweep (bit 1: a SweepSetRights table)
// the voting rights, quorum and leaders, on a committee sweep (bit 2, a rights sweep too) the committee size, and on a links
// sweep (bit 3, a SweepSetLinks table) the link latencies, and on an outage sweep (bit 4, a SweepSetLinks table) the outage
// windows; its thresholds are read through L1 from the concatenated table, as the
// instances of one warp may belong to different sets.
// CT: the commit-time stores (sim_core.cuh Core CT) into `times`, [num_instances][N + 1][round_cap].
template <int NMAX, int QMODE, int FX, bool REC, bool RES, bool EP, bool TDS, int TILE, bool SW, bool CT = false>
__device__ __forceinline__ void event_loop_body(const Params& P, double* s_zx, double* s_zf, double* s_thr, uint32_t* s_queue,
                                                const uint32_t* set_of, const SweepSet* sets, int32_t* times = nullptr,
                                                uint32_t records = 0) {
  static_assert(TILE == 32 || ((QMODE == 3 || QMODE == 2) && !REC && !RES && !EP && !TDS), "sparse tiles: plain kernels over the calendar / shared-memory queue");
  for (int i = threadIdx.x; i < 257; i += blockDim.x) {
    s_zx[i] = P.zig_x[i];
    s_zf[i] = P.zig_f[i];
  }
  const bool thr_fits = place_delay_thresholds<SW>(P, s_thr);
  __syncthreads();
  const uint32_t gthread = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t tile = gthread >> 5, lane = gthread & 31;
  const uint32_t inst = tile * TILE + lane;
  if (lane >= TILE || inst >= P.num_instances) return;
  const uint32_t total_words = FX ? fixed_layout(FX).total_words : P.L.total_words;
  // the compact encoding (FX_DEFAULT4, Core::PACK) keeps its node words and slots in lane blocks (TileMem LB)
  using Mem = TileMem<TILE, FX == FX_DEFAULT4>;
  Mem mem{P.state + (size_t)tile * total_words * TILE, lane};
  uint32_t* sk = nullptr;
  uint16_t* sd = nullptr;
  if (QMODE == 2) {
    const uint32_t warp = threadIdx.x >> 5, qcap = P.L.queue_cap;
    uint32_t* base = s_queue + (size_t)warp * (qcap * 32 + qcap * 16);  // keys (qcap*32 words) + payload (qcap*32 halves)
    sk = base + lane;
    sd = reinterpret_cast<uint16_t*>(base + qcap * 32) + lane;
  }
  // sparse tiles over the calendar queue: the kind-occupancy words of the tile's instances in shared memory, a column per
  // lane (sim_core.cuh KS; the host only selects sparse tiles when 14 warps' worth fits, host_setup.hpp)
  constexpr bool KS = QMODE == 3 && TILE < 32;
  Core<Mem, NMAX, QMODE, FX, REC, RES, 1, EP, TDS, KS, SW, CT> core(P, mem, s_zx, s_zf, thr_fits ? s_thr : P.delay_thr, sk, sd);
  if (KS) core.km = s_queue + (size_t)(threadIdx.x >> 5) * calendar_kmask_words(FX ? fixed_layout(FX) : P.L) * TILE + lane;
  if constexpr (CT) core.ct = times + (size_t)inst * (core.L.num_nodes + 1) * core.L.round_cap;
  if constexpr (SW) {
    core.bind_set(sweep_set_at(sets, set_of[inst], records));
    core.bind_faults(records & 1);
    core.bind_rights(records & 2);
    core.bind_committee(records & 4);
    core.bind_links(records & 8);
    core.bind_outages(records & 16);
  }
  if (RES && (P.run_flags & 1u)) core.restore_regs();  // a later lbft_run_until: continue where the last launch stopped
  else core.init(P.seeds[inst]);
  core.run();
  core.finalize(inst);
  if (RES) core.save_regs();
}

template <int NMAX, int QMODE, int FX = FX_NONE, bool REC = false, bool RES = false, bool EP = false, bool TDS = false, int TILE = 32>
__global__ void __launch_bounds__(LaunchShape<QMODE>::kThreads, LaunchShape<QMODE>::kBlocksPerSm) lbft_event_loop_kernel(const __grid_constant__ Params P) {
  // The ziggurat layers are indexed by a random byte per lane: a per-block shared-memory copy (4 KB) serves the 32
  // scattered 8-byte reads of a warp in ~1-2 wavefronts; reading them through L1 from global memory instead makes the
  // whole kernel markedly slower.
  __shared__ double s_zx[257];
  __shared__ double s_zf[257];
  __shared__ double s_thr[kThrSmem];  // delay thresholds (same scattered access pattern), when they fit
  extern __shared__ uint32_t s_queue[];  // QMODE 2: per warp [queue_cap][32] u32 keys, then [queue_cap][32] u16 payload words
                                         // QMODE 3, sparse tiles: per warp [kmask words][TILE] calendar occupancy words
  event_loop_body<NMAX, QMODE, FX, REC, RES, EP, TDS, TILE, false>(P, s_zx, s_zf, s_thr, s_queue, nullptr, nullptr);
}

// A sweep handle's thread kernel (lbft_create_sweep): the generic plain kernel with per-instance parameter sets.
template <int NMAX, int QMODE, int TILE = 32>
__global__ void __launch_bounds__(LaunchShape<QMODE>::kThreads, LaunchShape<QMODE>::kBlocksPerSm) lbft_sweep_event_loop_kernel(const __grid_constant__ SweepParams S) {
  __shared__ double s_zx[257];
  __shared__ double s_zf[257];
  extern __shared__ uint32_t s_queue[];
  event_loop_body<NMAX, QMODE, FX_NONE, false, false, false, false, TILE, true>(S.P, s_zx, s_zf, nullptr, s_queue, S.set_of, S.sets, nullptr,
                                                                               sweep_records(S));
}

// ---- a group of G lanes per instance ("wide") ---------------------------------------------------------------------
// wide_warps(G) warps per block, 32 / G instances per warp (instance = global group index; the hardware block scheduler hands
// out the next block as soon as one retires, which is the work queue SURVEY §8e asks for).  The state of an instance is one
// contiguous extent (TileMem<1>: stride 1), tables are read through L1 (every lane of a group reads the same element), the
// shared-memory queue of QMODE 2 and the fan-out scratch are per group.
// Warps per block: four when a warp carries several instances; ONE when a warp is an instance (G = 32): a block is then a
// single instance, its index arithmetic folds away and blocks retire one by one, which shortens small batches; with 8 lanes
// per instance the block size makes no difference.
LBFT_LAYOUT_FN int wide_warps(int g) { return g == 32 ? 1 : 4; }
// blocks per SM the register allocation is bounded for: 16 warps per SM, <= 128 registers
LBFT_LAYOUT_FN int wide_blocks_per_sm(int g) { return 16 / wide_warps(g); }

// Shared memory of one group: [scratch][QMODE 2: queue keys, queue payload halves][SMEM: the instance state]
LBFT_LAYOUT_FN uint32_t wide_scratch_words() { return (uint32_t)((sizeof(WideScratch) + 7) / 8 * 2); }
LBFT_LAYOUT_FN uint32_t wide_queue_words(uint32_t queue_cap, int qmode) {
  return qmode == 2 ? ((queue_cap + (queue_cap + 1) / 2 + 1) & ~1u) : 0u;  // even: what follows holds 64-bit entries
}
LBFT_LAYOUT_FN uint32_t wide_smem_words_per_group(const Layout& L, int qmode, bool smem_state) {
  return wide_scratch_words() + wide_queue_words(L.queue_cap, qmode) + (smem_state ? ((L.total_words + 1) & ~1u) : 0u);
}

// SMEM: the instance's state words live in shared memory for the whole run; only the chain table (and the epoch table) is
// copied to the instance's global extent at the end, for lbft_commit_log / lbft_commit_logs.
// The body of both wide kernels (lbft_wide_kernel, lbft_sweep_wide_kernel).  SW: as event_loop_body.
template <int NMAX, int QMODE, bool SMEM, int G, bool EP, int FX, bool SW, bool CT = false>
__device__ __forceinline__ void wide_body(const Params& P, uint32_t* s_wide, const uint32_t* set_of, const SweepSet* sets,
                                          int32_t* times = nullptr, uint32_t records = 0) {
  constexpr uint32_t kPerBlock = wide_warps(G) * 32 / G;
  const uint32_t grp = threadIdx.x / G, wl = threadIdx.x % G;
  const uint32_t inst = blockIdx.x * kPerBlock + grp;
  if (inst >= P.num_instances) return;  // whole groups leave together: everything below is group-uniform
  const Layout KL = FX ? fixed_layout(FX) : P.L;
  uint32_t* base = s_wide + (size_t)grp * wide_smem_words_per_group(KL, QMODE, SMEM);
  WideScratch* ws = reinterpret_cast<WideScratch*>(base);
  uint32_t* sk = base + wide_scratch_words();
  uint16_t* sd = reinterpret_cast<uint16_t*>(sk + KL.queue_cap);
  uint32_t* gstate = P.state + (size_t)inst * KL.total_words;
  uint32_t* state = SMEM ? sk + wide_queue_words(KL.queue_cap, QMODE) : gstate;
  TileMem<1> mem{state, 0};
  Core<TileMem<1>, NMAX, QMODE, FX, false, false, G, EP, false, false, SW, CT> core(P, mem, P.zig_x, P.zig_f, P.delay_thr, sk, sd);
  core.wl = wl;
  if constexpr (CT) core.ct = times + (size_t)inst * (KL.num_nodes + 1) * KL.round_cap;
  core.gm = G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << ((threadIdx.x & 31u) & ~(uint32_t)(G - 1)));
  core.ws = ws;
  if constexpr (SW) {
    core.bind_set(sweep_set_at(sets, set_of[inst], records));
    core.bind_faults(records & 1);
    core.bind_rights(records & 2);
    core.bind_committee(records & 4);
    core.bind_links(records & 8);
    core.bind_outages(records & 16);
  }
  core.init(P.seeds[inst]);
  core.run();
  core.finalize(inst);
  if (SMEM) {
    __syncwarp(core.gm);
    for (uint32_t w = P.L.chain_base + wl; w < P.L.chain_base + 2 * P.L.round_cap; w += G) gstate[w] = state[w];
    if (EP)
      for (uint32_t w = wl; w < P.L.epochs; w += G) gstate[P.L.einit_base + w] = state[P.L.einit_base + w];
  }
}

template <int NMAX, int QMODE, bool SMEM, int G, bool EP = false, int FX = FX_NONE>
__global__ void __launch_bounds__(wide_warps(G) * 32, wide_blocks_per_sm(G)) lbft_wide_kernel(const __grid_constant__ Params P) {
  extern __shared__ __align__(8) uint32_t s_wide[];
  wide_body<NMAX, QMODE, SMEM, G, EP, FX, false>(P, s_wide, nullptr, nullptr);
}

// A sweep handle's wide kernel (lbft_create_sweep).
template <int NMAX, int QMODE, bool SMEM, int G>
__global__ void __launch_bounds__(wide_warps(G) * 32, wide_blocks_per_sm(G)) lbft_sweep_wide_kernel(const __grid_constant__ SweepParams S) {
  extern __shared__ __align__(8) uint32_t s_wide[];
  wide_body<NMAX, QMODE, SMEM, G, false, FX_NONE, true>(S.P, s_wide, S.set_of, S.sets, nullptr, sweep_records(S));
}

// The parameter block of a commit-times kernel (LBFT_FLAG_COMMIT_TIMES): the plain (Params) or sweep (SweepParams) block and
// the commit-time table, [num_instances][N + 1][round_cap] int32.  (A block of its own, so that no other kernel's parameters
// move.)
template <class KP>
struct CtParams {
  KP base;
  int32_t* times;
};

// The commit-times twins of the one-shot single-epoch kernels: the same bodies with CT set.
template <int NMAX, int QMODE, int FX, int TILE>
__global__ void __launch_bounds__(LaunchShape<QMODE>::kThreads, LaunchShape<QMODE>::kBlocksPerSm) lbft_ct_event_loop_kernel(const __grid_constant__ CtParams<Params> C) {
  __shared__ double s_zx[257];
  __shared__ double s_zf[257];
  __shared__ double s_thr[kThrSmem];
  extern __shared__ uint32_t s_queue[];
  event_loop_body<NMAX, QMODE, FX, false, false, false, false, TILE, false, true>(C.base, s_zx, s_zf, s_thr, s_queue, nullptr, nullptr, C.times);
}
template <int NMAX, int QMODE, int TILE>
__global__ void __launch_bounds__(LaunchShape<QMODE>::kThreads, LaunchShape<QMODE>::kBlocksPerSm) lbft_ct_sweep_event_loop_kernel(const __grid_constant__ CtParams<SweepParams> C) {
  __shared__ double s_zx[257];
  __shared__ double s_zf[257];
  extern __shared__ uint32_t s_queue[];
  event_loop_body<NMAX, QMODE, FX_NONE, false, false, false, false, TILE, true, true>(C.base.P, s_zx, s_zf, nullptr, s_queue, C.base.set_of,
                                                                                     C.base.sets, C.times, sweep_records(C.base));
}
template <int NMAX, int QMODE, bool SMEM, int G, int FX>
__global__ void __launch_bounds__(wide_warps(G) * 32, wide_blocks_per_sm(G)) lbft_ct_wide_kernel(const __grid_constant__ CtParams<Params> C) {
  extern __shared__ __align__(8) uint32_t s_wide[];
  wide_body<NMAX, QMODE, SMEM, G, false, FX, false, true>(C.base, s_wide, nullptr, nullptr, C.times);
}
template <int NMAX, int QMODE, bool SMEM, int G>
__global__ void __launch_bounds__(wide_warps(G) * 32, wide_blocks_per_sm(G)) lbft_ct_sweep_wide_kernel(const __grid_constant__ CtParams<SweepParams> C) {
  extern __shared__ __align__(8) uint32_t s_wide[];
  wide_body<NMAX, QMODE, SMEM, G, false, FX_NONE, true, true>(C.base.P, s_wide, C.base.set_of, C.base.sets, C.times, sweep_records(C.base));
}

// One per translation unit: launches the instantiation the selection names, or returns cudaErrorInvalidValue if the unit
// has none (lbft_api.cu reports that with the kernel's name).
cudaError_t launch_fixed(const KernelSel& k, const Params& P, cudaStream_t stream);
cudaError_t launch_scan(const KernelSel& k, const Params& P, cudaStream_t stream);
cudaError_t launch_calendar(const KernelSel& k, const Params& P, cudaStream_t stream);
cudaError_t launch_heap(const KernelSel& k, const Params& P, cudaStream_t stream);
cudaError_t launch_wide(const KernelSel& k, const Params& P, cudaStream_t stream);
cudaError_t launch_sweep_thread(const KernelSel& k, const SweepParams& S, cudaStream_t stream);
cudaError_t launch_sweep_wide(const KernelSel& k, const SweepParams& S, cudaStream_t stream);
cudaError_t launch_ct_thread(const KernelSel& k, const CtParams<Params>& C, cudaStream_t stream);
cudaError_t launch_ct_wide(const KernelSel& k, const CtParams<Params>& C, cudaStream_t stream);
cudaError_t launch_ct_sweep_thread(const KernelSel& k, const CtParams<SweepParams>& C, cudaStream_t stream);
cudaError_t launch_ct_sweep_wide(const KernelSel& k, const CtParams<SweepParams>& C, cudaStream_t stream);

// Lets `kernel` take up to the device's opt-in limit of shared memory per block, beyond the 48 KB default (the QMODE 2
// queues of four warps, the wide kernel's shared-memory instance state); `whole_carveout` also asks for the largest
// shared-memory carveout (4 such QMODE 2 blocks per SM).  The attributes belong to the kernel's handle in each device's
// context, so they are set before every launch on the current device (one process may drive several GPUs), and always to
// the same values, so host threads launching concurrently cannot undo each other's setting.
template <class Kernel>
inline cudaError_t allow_optin_smem(Kernel kernel, bool whole_carveout) {
  int dev = 0, optin = 0;
  cudaFuncAttributes fa{};
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, kernel);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
  if (e == cudaSuccess && whole_carveout)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
  return e;
}

inline const Params& params_of(const Params& P) { return P; }
inline const Params& params_of(const SweepParams& S) { return S.P; }
template <class KP>
inline const Params& params_of(const CtParams<KP>& C) { return params_of(C.base); }

// One instantiation of a kernel template: the selection that names it, and its launch.  try_launch launches it if `k` names
// it and reports whether it did.  SW: the sweep twin of the generic plain instantiation (lbft_sweep_*_kernel).  CT: the
// commit-times twin (lbft_ct_*_kernel) of the instantiation the other arguments name.
template <int NMAX, int QM, int FX = FX_NONE, bool REC = false, bool RES = false, bool EP = false, bool TDS = false, int TILE = 32,
          bool SW = false, bool CT = false>
struct ThreadKernel {
  static_assert(!SW || (FX == FX_NONE && !REC && !RES && !EP && !TDS), "sweeps: plain single-epoch generic kernels only");
  static_assert(!CT || (!REC && !RES && !EP && !TDS), "commit times: one-shot single-epoch kernels only");
  static constexpr KernelSel sel{/*wide*/ false, /*smem*/ false, /*group*/ 0, EP, TDS, TILE, NMAX, QM, FX, REC, RES, SW, CT};
  using Base = typename std::conditional<SW, SweepParams, Params>::type;
  using KParams = typename std::conditional<CT, CtParams<Base>, Base>::type;  // the kernel's parameter block
  static bool try_launch(const KernelSel& k, const KParams& KP, cudaStream_t stream, cudaError_t& e) {
    if (!same_kernel(k, sel)) return false;
    const Params& P = params_of(KP);
    constexpr int T = LaunchShape<QM>::kThreads;
    const uint32_t tiles = (P.num_instances + TILE - 1) / TILE, blocks = (tiles * 32 + T - 1) / T;
    // QMODE 2: per warp the queue keys and payload halves; sparse tiles over the calendar queue: per warp the occupancy
    // words of its instances (sim_core.cuh KS)
    const size_t dyn = QM == 2 ? (size_t)(T / 32) * P.L.queue_cap * (32 * 4 + 32 * 2)
                               : (QM == 3 && TILE < 32 ? (size_t)calendar_kmask_words(P.L) * TILE * sizeof(uint32_t) : 0);
    void (*kernel)(KParams);
    if constexpr (CT && SW) kernel = lbft_ct_sweep_event_loop_kernel<NMAX, QM, TILE>;
    else if constexpr (CT) kernel = lbft_ct_event_loop_kernel<NMAX, QM, FX, TILE>;
    else if constexpr (SW) kernel = lbft_sweep_event_loop_kernel<NMAX, QM, TILE>;
    else kernel = lbft_event_loop_kernel<NMAX, QM, FX, REC, RES, EP, TDS, TILE>;
    e = dyn > 0 ? allow_optin_smem(kernel, QM == 2) : cudaSuccess;
    if (e == cudaSuccess) {
      kernel<<<blocks, T, dyn, stream>>>(KP);
      e = cudaGetLastError();
    }
    return true;
  }
};
template <int NMAX, int QM, bool SMEM, int G, bool EP = false, int FX = FX_NONE, bool SW = false, bool CT = false>
struct WideKernel {
  static_assert(!SW || (FX == FX_NONE && !EP), "sweeps: plain single-epoch generic kernels only");
  static_assert(!CT || !EP, "commit times: single-epoch kernels only");
  static constexpr KernelSel sel{/*wide*/ true, SMEM, G, EP, /*tds*/ false, /*tile*/ 1, NMAX, QM, FX, /*rec*/ false, /*res*/ false, SW, CT};
  using Base = typename std::conditional<SW, SweepParams, Params>::type;
  using KParams = typename std::conditional<CT, CtParams<Base>, Base>::type;
  static bool try_launch(const KernelSel& k, const KParams& KP, cudaStream_t stream, cudaError_t& e) {
    if (!same_kernel(k, sel)) return false;
    const Params& P = params_of(KP);
    constexpr uint32_t kPerBlock = wide_warps(G) * 32 / G;
    const uint32_t blocks = (P.num_instances + kPerBlock - 1) / kPerBlock;
    const size_t dyn = (size_t)kPerBlock * wide_smem_words_per_group(P.L, QM, SMEM) * sizeof(uint32_t);
    void (*kernel)(KParams);
    if constexpr (CT && SW) kernel = lbft_ct_sweep_wide_kernel<NMAX, QM, SMEM, G>;
    else if constexpr (CT) kernel = lbft_ct_wide_kernel<NMAX, QM, SMEM, G, FX>;
    else if constexpr (SW) kernel = lbft_sweep_wide_kernel<NMAX, QM, SMEM, G>;
    else kernel = lbft_wide_kernel<NMAX, QM, SMEM, G, EP, FX>;
    e = dyn > 48 * 1024 ? allow_optin_smem(kernel, false) : cudaSuccess;  // (the wide kernel has no static shared memory)
    if (e == cudaSuccess) {
      kernel<<<blocks, wide_warps(G) * 32, dyn, stream>>>(KP);
      e = cudaGetLastError();
    }
    return true;
  }
};
// A list of instantiations (or of lists) that take the same parameter block KP (Params, or SweepParams for sweep kernels).
template <class... Ks>
struct Kernels {
  template <class KP>
  static bool try_launch(const KernelSel& k, const KP& kp, cudaStream_t stream, cudaError_t& e) {
    return (Ks::try_launch(k, kp, stream, e) || ...);
  }
};
template <class List, class KP>
inline cudaError_t launch_listed(const KernelSel& k, const KP& kp, cudaStream_t stream) {
  cudaError_t e = cudaErrorInvalidValue;
  List::try_launch(k, kp, stream, e);
  return e;
}

// The recording / resumable / epoch / true-data-sync variants of a generic thread kernel.
template <int NMAX, int QM>
using ThreadVariants = Kernels<ThreadKernel<NMAX, QM>, ThreadKernel<NMAX, QM, FX_NONE, true>, ThreadKernel<NMAX, QM, FX_NONE, false, true>,
                               ThreadKernel<NMAX, QM, FX_NONE, true, true>, ThreadKernel<NMAX, QM, FX_NONE, false, false, true>,
                               ThreadKernel<NMAX, QM, FX_NONE, false, false, false, true>>;
// The lane groups and the epoch variant of a generic wide kernel with its state in HBM.
template <int NMAX, int QM>
using WideVariants = Kernels<WideKernel<NMAX, QM, false, 8>, WideKernel<NMAX, QM, false, 32>, WideKernel<NMAX, QM, false, 32, true>>;
// The sweep twins of the plain generic instantiations: of a full-tile thread kernel, and of the two lane groups of a wide
// kernel with its state in HBM.
template <int NMAX, int QM>
using SweepThread = ThreadKernel<NMAX, QM, FX_NONE, false, false, false, false, 32, true>;
template <int NMAX, int QM>
using SweepWideVariants = Kernels<WideKernel<NMAX, QM, false, 8, false, FX_NONE, true>, WideKernel<NMAX, QM, false, 32, false, FX_NONE, true>>;
// The commit-times twins (k_ct_*.cu): of a full-tile generic thread kernel and of the two HBM lane groups of a generic wide
// kernel, plain (SW = false) or sweep.
template <int NMAX, int QM, bool SW>
using CtThread = ThreadKernel<NMAX, QM, FX_NONE, false, false, false, false, 32, SW, true>;
template <int NMAX, int QM, bool SW>
using CtWideVariants = Kernels<WideKernel<NMAX, QM, false, 8, false, FX_NONE, SW, true>, WideKernel<NMAX, QM, false, 32, false, FX_NONE, SW, true>>;

}  // namespace lbft
