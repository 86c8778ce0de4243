// fault_hostcore.cpp — TEST INFRASTRUCTURE for fault sweeps (lbft_create_sweep_faults).  The device state machine of sweep
// handles (csrc/sim_core.cuh, Core's SW parameter, with and without the commit-time stores of CT) compiled with g++, over the
// product's own host setup (HostSetup::build_sweep_faults), each instance bound to its set's parameter and fault records as the
// product's sweep kernels bind them.  The CT runs are read out through the product's commit_times_of and latency_samples_of.
// ct_hostcore.cpp is compiled into this unit as it is (for kNotWritten and the error slot).  Never part of, linked into, or
// reachable from the product library.
#include "ct_hostcore.cpp"

namespace {
using namespace lbft;

// Instance i runs with set set_of[i], bound as the product's sweep kernels bind it: on a fault sweep from the SweepSetFaults
// table the runtime uploads (`paired`), else from the sets; the thread-per-instance tile layout (32 lanes).
template <int NMAX, int QMODE, bool CT>
void run_faults(const Params& P, std::vector<uint32_t>& state, int32_t* times, const uint32_t* set_of, const SweepSet* sets,
                const SweepSetFaults* paired) {
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    const uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * P.L.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, FX_NONE, false, false, 1, false, false, false, true, CT> core(P, mem, P.zig_x, P.zig_f, P.delay_thr,
                                                                                             sk.data() + lane, sd.data() + lane);
    if constexpr (CT) core.ct = times + (size_t)inst * (P.L.num_nodes + 1) * P.L.round_cap;
    core.bind_set(paired ? &paired[set_of[inst]].set : sets + set_of[inst]);
    core.bind_faults(paired != nullptr);
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
  }
}

template <bool CT>
void dispatch(const Params& P, std::vector<uint32_t>& state, int32_t* times, const HostSetup& hs) {
  const uint32_t N = P.L.num_nodes, qs = P.L.queue_scan;
  const uint32_t* so = hs.set_of.data();
  const SweepSet* ss = hs.sets.data();
  std::vector<SweepSetFaults> table(hs.faults.size());  // (lbft_api.cu create_on_device)
  for (size_t k = 0; k < table.size(); k++) table[k] = SweepSetFaults{hs.sets[k], hs.faults[k]};
  const SweepSetFaults* sf = table.empty() ? nullptr : table.data();
  if (qs == 2) run_faults<16, 2, CT>(P, state, times, so, ss, sf);
  else if (qs == 1) run_faults<16, 1, CT>(P, state, times, so, ss, sf);
  else if (qs == 3) {
    if (N <= 16) run_faults<16, 3, CT>(P, state, times, so, ss, sf);
    else if (N <= 32) run_faults<32, 3, CT>(P, state, times, so, ss, sf);
    else run_faults<64, 3, CT>(P, state, times, so, ss, sf);
  } else if (N <= 16) run_faults<16, 0, CT>(P, state, times, so, ss, sf);
  else if (N <= 32) run_faults<32, 0, CT>(P, state, times, so, ss, sf);
  else run_faults<64, 0, CT>(P, state, times, so, ss, sf);
}

// The host tables of `hs` and the output arrays into a parameter block.
Params bind_tables(const HostSetup& hs, const lbft_config* c, std::vector<uint32_t>& state, uint32_t* commit_counts, uint64_t* last_states,
                   uint32_t* lc_round, uint32_t* counters, uint32_t* status) {
  Params P = hs.params;
  P.seeds = c->seeds;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.leader = hs.leader.data();
  P.duration = hs.duration.data();
  P.period = hs.period.data();
  P.weights = hs.weights.data();
  P.delay_thr = hs.delay_thr.empty() ? nullptr : hs.delay_thr.data();
  state.assign((size_t)((c->num_instances + 31) / 32) * P.L.total_words * 32, 0xdeadbeefu);
  P.state = state.data();
  P.out_commit_counts = commit_counts;
  P.out_last_state = last_states;
  P.out_lc_round = lc_round;
  P.out_counters = counters;
  P.out_status = status;
  return P;
}

// sets / faults: lbft_create_sweep_faults when faults is not null, lbft_create_sweep otherwise.
bool setup(HostSetup& hs, const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, uint32_t num_sets,
           const uint32_t* set_of) {
  if (faults ? hs.build_sweep_faults(*c, sets, faults, num_sets, set_of) : hs.build_sweep(*c, sets, num_sets, set_of)) return true;
  g_ct_err = hs.error;
  return false;
}
}  // namespace

extern "C" {
const char* fault_hostcore_last_error(void) { return g_ct_err.c_str(); }

// The product's lbft_kernel_info and Layout::part_windows for a fault sweep of this configuration (faults == NULL: a sweep).
int fault_hostcore_kernel_info(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, uint32_t num_sets,
                               const uint32_t* set_of, char* buf, size_t cap, uint32_t* part_windows) {
  HostSetup hs;
  if (!setup(hs, c, sets, faults, num_sets, set_of)) return LBFT_ERR_INVALID;
  snprintf(buf, cap, "%s", kernel_name(hs.sel).c_str());
  *part_windows = hs.params.L.part_windows;
  return LBFT_OK;
}

// The SW core: the outputs of the product's lbft_* getters, plus the per-node last committed rounds.
int fault_hostcore_run(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, uint32_t num_sets,
                       const uint32_t* set_of, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round, uint32_t* counters,
                       uint32_t* status) {
  HostSetup hs;
  if (!setup(hs, c, sets, faults, num_sets, set_of)) return LBFT_ERR_INVALID;
  if (hs.sel.ct) { g_ct_err = "fault_hostcore_run runs the SW core: use fault_hostcore_run_ct for LBFT_FLAG_COMMIT_TIMES"; return LBFT_ERR_INVALID; }
  std::vector<uint32_t> state;
  const Params P = bind_tables(hs, c, state, commit_counts, last_states, lc_round, counters, status);
  dispatch<false>(P, state, nullptr, hs);
  return LBFT_OK;
}

// The SW + CT core (LBFT_FLAG_COMMIT_TIMES): the getters' outputs and lbft_commit_times (committed [I][N][cap], proposed
// [I][cap]).  With a spec (may be NULL), also lbft_latency_stats into out[num_sets] and hist[num_sets][num_bins] (may be NULL),
// grouped by set, through the product's spec check and per-instance walk.
int fault_hostcore_run_ct(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, uint32_t num_sets,
                          const uint32_t* set_of, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round, uint32_t* counters,
                          uint32_t* status, int64_t* committed, int64_t* proposed, size_t cap, const lbft_latency_spec* spec,
                          lbft_latency_summary* out, uint64_t* hist) {
  HostSetup hs;
  if (!setup(hs, c, sets, faults, num_sets, set_of)) return LBFT_ERR_INVALID;
  if (!hs.sel.ct) { g_ct_err = "commit times were not recorded: set LBFT_FLAG_COMMIT_TIMES in lbft_config.flags"; return LBFT_ERR_STATE; }
  if (cap == 0 || cap > 0xffffu) { g_ct_err = "cap must be in 1..65535 rows per instance"; return LBFT_ERR_INVALID; }
  if (spec)
    if (const char* e = latency_spec_error(hs, *spec)) { g_ct_err = e; return LBFT_ERR_INVALID; }
  const uint32_t I = c->num_instances, N = c->num_nodes;
  std::vector<uint32_t> state;
  const Params P = bind_tables(hs, c, state, commit_counts, last_states, lc_round, counters, status);
  const Layout& L = P.L;
  std::vector<int32_t> times((size_t)I * (N + 1) * L.round_cap, kNotWritten);
  dispatch<true>(P, state, times.data(), hs);
  for (uint32_t i = 0; i < I; i++) {
    const uint32_t* inst = state.data() + (size_t)(i / 32) * L.total_words * 32 + i % 32;
    const int32_t* t = times.data() + (size_t)i * (N + 1) * L.round_cap;
    if (!commit_times_of(L, inst, 32, commit_counts + (size_t)i * N, lc_round + (size_t)i * N, t, (uint32_t)cap,
                         committed + (size_t)i * N * cap, proposed + (size_t)i * cap)) {
      g_ct_err = "node logs that are not prefixes of one chain";
      return LBFT_ERR_STATE;
    }
  }
  if (!spec) return LBFT_OK;
  LatencyAccumulator acc(out, num_sets, *spec);
  for (uint32_t i = 0; i < I; i++) {
    const uint32_t g = set_of[i];
    if (!acc.admit(g, status[i])) continue;
    const bool ok = latency_samples_of(L, state.data() + (size_t)(i / 32) * L.total_words * 32 + i % 32, 32, commit_counts + (size_t)i * N,
                                       lc_round + (size_t)i * N, times.data() + (size_t)i * (N + 1) * L.round_cap, spec->proposed_from,
                                       spec->proposed_until, [&](int64_t lat) { acc.add(g, lat); });
    if (!ok) { g_ct_err = "node logs that are not prefixes of one chain"; return LBFT_ERR_STATE; }
  }
  acc.finish(hist);
  return LBFT_OK;
}
}  // extern "C"
