// sweep_hostcore.cpp — TEST INFRASTRUCTURE: the device state machine (csrc/sim_core.cuh) of sweep handles (lbft_create_sweep,
// Core's SW parameter) compiled with g++, over the product's own host setup (HostSetup::build_sweep), so that a sweep can be
// checked against the oracle instance by instance without a GPU.  Never part of, linked into, or reachable from the product
// library.
#include <cstring>
#include <string>
#include <vector>

#include "../../librabft_simulator_b200/csrc/host_setup.hpp"
#include "../../librabft_simulator_b200/csrc/sim_core.cuh"

using namespace lbft;
static thread_local std::string g_err;

// Instance i runs with sets[set_of[i]], as in the product's sweep kernels; the thread-per-instance tile layout.
template <int NMAX, int QMODE>
static void run_sweep_all(const Params& P, std::vector<uint32_t>& state, const uint32_t* set_of, const SweepSet* sets) {
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * P.L.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, FX_NONE, false, false, 1, false, false, false, true> core(P, mem, P.zig_x, P.zig_f, P.delay_thr,
                                                                                         sk.data() + lane, sd.data() + lane);
    core.bind_set(sets + set_of[inst]);
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
  }
}

// FNV-1a over a byte range; over a host table, its length and then its bytes (hostcore_sweep_setup_digest)
static uint64_t fnv1a(uint64_t h, const void* p, size_t n) {
  for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 0x100000001b3ULL;
  return h;
}
template <class T>
static uint64_t fnv1a(uint64_t h, const std::vector<T>& v) {
  const uint64_t n = v.size();
  return fnv1a(fnv1a(h, &n, sizeof n), v.data(), n * sizeof(T));
}

extern "C" {
const char* hostcore_sweep_last_error(void) { return g_err.c_str(); }

// The product's lbft_kernel_info for a sweep handle of this configuration (lbft_create_sweep's host setup).
int hostcore_kernel_info_sweep(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, const uint32_t* set_of,
                               char* buf, size_t cap) {
  HostSetup hs;
  if (!hs.build_sweep(*c, sets, num_sets, set_of)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  if (!buf || cap == 0) { g_err = "NULL argument"; return LBFT_ERR_INVALID; }
  snprintf(buf, cap, "%s", kernel_name(hs.sel).c_str());
  return LBFT_OK;
}

// hostcore_setup_digest (hostcore.cpp) of a sweep handle's host setup, with the parameter sets and the set of each instance.
int hostcore_sweep_setup_digest(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, const uint32_t* set_of,
                                uint64_t* digest) {
  HostSetup hs;
  if (!hs.build_sweep(*c, sets, num_sets, set_of)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  uint64_t h = fnv1a(0xcbf29ce484222325ULL, &hs.params, offsetof(Params, seeds));
  h = fnv1a(fnv1a(fnv1a(fnv1a(h, hs.zig_x), hs.zig_f), hs.leader), hs.duration);
  h = fnv1a(fnv1a(fnv1a(h, hs.period), hs.weights), hs.delay_thr);
  *digest = fnv1a(fnv1a(h, hs.sets), hs.set_of);
  return LBFT_OK;
}

// Same outputs as the product's lbft_* getters on a sweep handle, plus the per-node last committed rounds and the state words
// per instance.
int hostcore_run_sweep(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, const uint32_t* set_of,
                       uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round, uint32_t* counters, uint32_t* status,
                       uint32_t* words_per_instance) {
  HostSetup hs;
  if (!hs.build_sweep(*c, sets, num_sets, set_of)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  Params P = hs.params;
  P.seeds = c->seeds;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.leader = hs.leader.data();
  P.duration = hs.duration.data();
  P.period = hs.period.data();
  P.weights = hs.weights.data();
  P.delay_thr = hs.delay_thr.empty() ? nullptr : hs.delay_thr.data();
  std::vector<uint32_t> state((size_t)((c->num_instances + 31) / 32) * P.L.total_words * 32, 0xdeadbeefu);
  P.state = state.data();
  P.out_commit_counts = commit_counts;
  P.out_last_state = last_states;
  P.out_lc_round = lc_round;
  P.out_counters = counters;
  P.out_status = status;
  if (words_per_instance) *words_per_instance = P.L.total_words;
  const uint32_t* so = hs.set_of.data();
  const SweepSet* ss = hs.sets.data();
  const uint32_t N = c->num_nodes, qs = P.L.queue_scan;
  if (qs == 2) run_sweep_all<16, 2>(P, state, so, ss);
  else if (qs == 1) run_sweep_all<16, 1>(P, state, so, ss);
  else if (qs == 3) {
    if (N <= 16) run_sweep_all<16, 3>(P, state, so, ss);
    else if (N <= 32) run_sweep_all<32, 3>(P, state, so, ss);
    else run_sweep_all<64, 3>(P, state, so, ss);
  } else if (N <= 16) run_sweep_all<16, 0>(P, state, so, ss);
  else if (N <= 32) run_sweep_all<32, 0>(P, state, so, ss);
  else run_sweep_all<64, 0>(P, state, so, ss);
  return LBFT_OK;
}
}  // extern "C"
