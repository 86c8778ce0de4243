// ct_hostcore.cpp — TEST INFRASTRUCTURE for commit times (LBFT_FLAG_COMMIT_TIMES).  Two things, so that the feature can be
// checked without a GPU:
//   * the device state machine with its commit-time stores (csrc/sim_core.cuh, Core CT) compiled with g++, over the
//     product's own host setup (HostSetup::build / build_sweep) and read out through the product's commit_times_of;
//   * the oracle (oracle/lbft_oracle.hpp), observed from outside: the run is advanced one event time at a time and every row
//     that appears in a node's committed_history() is stamped with the clock of that event time.  No protocol code changes.
// Never part of, linked into, or reachable from the product library.
//
// The oracle's C entry points are compiled into this unit as they are, for the configuration and partition-plan helpers
// they use (make_cfg, make_partition_plan): the observed runs are built exactly like the oracle's own.
#include "../../oracle/oracle_capi.cpp"

#include "../../librabft_simulator_b200/csrc/host_setup.hpp"
#include "../../librabft_simulator_b200/csrc/sim_core.cuh"

namespace {
thread_local std::string g_ct_err;
constexpr int32_t kNotWritten = 0x5eadbeef;  // fill of a fresh commit-time table: never written by a run

// The instance driver of the product's kernels for one-shot single-epoch handles with CT set: the compile-time layouts where
// fixed_shape_of finds one, the generic core otherwise; SW: a sweep handle.  Thread-per-instance tile layout (32 lanes).
template <int NMAX, int QMODE, int FX, bool SW>
void run_ct(const lbft::Params& P, std::vector<uint32_t>& state, int32_t* times, uint32_t* startup, const uint32_t* set_of,
            const lbft::SweepSet* sets) {
  using namespace lbft;
  const Layout KL = FX ? fixed_layout(FX) : P.L;
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    const uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * KL.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)KL.queue_cap * 32 : 1);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)KL.queue_cap * 32 : 1);
    constexpr bool KS = QMODE == 3 && FX != FX_NONE;  // (the compile-time calendar layouts: occupancy words in "shared memory")
    std::vector<uint32_t> km(KS ? (size_t)((KL.cal_times + 7) / 8) * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, FX, false, false, 1, false, false, KS, SW, true> core(P, mem, P.zig_x, P.zig_f, P.delay_thr,
                                                                                         sk.data() + lane, sd.data() + lane);
    core.km = km.data() + lane;
    core.ct = times + (size_t)inst * (KL.num_nodes + 1) * KL.round_cap;
    if constexpr (SW) core.bind_set(sets + set_of[inst]);
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
    if (startup)  // SimulatedNode.startup_time of every node, as the core holds it
      for (uint32_t n = 0; n < KL.num_nodes; n++) startup[(size_t)inst * KL.num_nodes + n] = core.node_ld(core.nbase(n), F_STARTUP);
  }
}

template <bool SW>
void run_dispatch(const lbft::Params& P, uint32_t N, std::vector<uint32_t>& state, int32_t* times, uint32_t* startup, const uint32_t* so,
                  const lbft::SweepSet* ss) {
  using namespace lbft;
  const int fx = SW ? (int)FX_NONE : fixed_shape_of(P);
  if constexpr (!SW) {
    if (fx == FX_DEFAULT4) return run_ct<16, 2, FX_DEFAULT4, false>(P, state, times, startup, so, ss);
    if (fx == FX_PART7) return run_ct<16, 3, FX_PART7, false>(P, state, times, startup, so, ss);
    if (fx == FX_COMMITTEE64) return run_ct<64, 3, FX_COMMITTEE64, false>(P, state, times, startup, so, ss);
  }
  const uint32_t qs = P.L.queue_scan;
  if (qs == 2) run_ct<16, 2, FX_NONE, SW>(P, state, times, startup, so, ss);
  else if (qs == 1) run_ct<16, 1, FX_NONE, SW>(P, state, times, startup, so, ss);
  else if (qs == 3) {
    if (N <= 16) run_ct<16, 3, FX_NONE, SW>(P, state, times, startup, so, ss);
    else if (N <= 32) run_ct<32, 3, FX_NONE, SW>(P, state, times, startup, so, ss);
    else run_ct<64, 3, FX_NONE, SW>(P, state, times, startup, so, ss);
  } else if (N <= 16) run_ct<16, 0, FX_NONE, SW>(P, state, times, startup, so, ss);
  else if (N <= 32) run_ct<32, 0, FX_NONE, SW>(P, state, times, startup, so, ss);
  else run_ct<64, 0, FX_NONE, SW>(P, state, times, startup, so, ss);
}

// One handle's run(s) and lbft_commit_times read-out.  first_seeds (optional): run those seeds first over the same state and
// commit-time table, as a re-seeded handle does.
int run_impl(lbft::HostSetup& hs, const lbft_config* c, const uint64_t* first_seeds, uint32_t* commit_counts, uint64_t* last_states,
             uint32_t* lc_round, uint32_t* counters, uint32_t* status, int64_t* committed, int64_t* proposed, size_t cap,
             uint32_t* startup) {
  using namespace lbft;
  if (!hs.sel.ct) { g_ct_err = "commit times were not recorded: set LBFT_FLAG_COMMIT_TIMES in lbft_config.flags"; return LBFT_ERR_STATE; }
  if (cap == 0 || cap > 0xffffu) { g_ct_err = "cap must be in 1..65535 rows per instance"; return LBFT_ERR_INVALID; }
  const uint32_t I = c->num_instances, N = c->num_nodes;
  Params P = hs.params;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.leader = hs.leader.data();
  P.duration = hs.duration.data();
  P.period = hs.period.data();
  P.weights = hs.weights.data();
  P.delay_thr = hs.delay_thr.empty() ? nullptr : hs.delay_thr.data();
  std::vector<uint32_t> state((size_t)((I + 31) / 32) * P.L.total_words * 32, 0xdeadbeefu);
  std::vector<int32_t> times((size_t)I * (N + 1) * P.L.round_cap, kNotWritten);
  P.state = state.data();
  P.out_commit_counts = commit_counts;
  P.out_last_state = last_states;
  P.out_lc_round = lc_round;
  P.out_counters = counters;
  P.out_status = status;
  const uint32_t* so = hs.set_of.empty() ? nullptr : hs.set_of.data();
  const SweepSet* ss = hs.sets.empty() ? nullptr : hs.sets.data();
  for (const uint64_t* seeds : {first_seeds, c->seeds}) {
    if (!seeds) continue;
    P.seeds = seeds;
    if (hs.sel.sweep) run_dispatch<true>(P, N, state, times.data(), startup, so, ss);
    else run_dispatch<false>(P, N, state, times.data(), startup, so, ss);
  }
  for (uint32_t i = 0; i < I; i++)
    if (!commit_times_of(P.L, state.data() + (size_t)(i / 32) * P.L.total_words * 32 + i % 32, 32, commit_counts + (size_t)i * N,
                         lc_round + (size_t)i * N, times.data() + (size_t)i * (N + 1) * P.L.round_cap, (uint32_t)cap,
                         committed + (size_t)i * N * cap, proposed ? proposed + (size_t)i * cap : nullptr)) {
      g_ct_err = "node logs that are not prefixes of one chain";
      return LBFT_ERR_STATE;
    }
  return LBFT_OK;
}
}  // namespace

extern "C" {
const char* ct_hostcore_last_error(void) { return g_ct_err.c_str(); }

// lbft_create + lbft_run + lbft_commit_times of a plain handle, with the outputs of the other getters (and lc_round), and
// startup[instance * N + node] (may be null): each node's startup time, read from the core's final state.
int ct_hostcore_run(const lbft_config* c, const uint64_t* first_seeds, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                    uint32_t* counters, uint32_t* status, int64_t* committed, int64_t* proposed, size_t cap, uint32_t* startup) {
  lbft::HostSetup hs;
  if (!hs.build(*c)) { g_ct_err = hs.error; return LBFT_ERR_INVALID; }
  return run_impl(hs, c, first_seeds, commit_counts, last_states, lc_round, counters, status, committed, proposed, cap, startup);
}

// The same for a sweep handle (lbft_create_sweep).
int ct_hostcore_run_sweep(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, const uint32_t* set_of,
                          uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round, uint32_t* counters, uint32_t* status,
                          int64_t* committed, int64_t* proposed, size_t cap) {
  lbft::HostSetup hs;
  if (!hs.build_sweep(*c, sets, num_sets, set_of)) { g_ct_err = hs.error; return LBFT_ERR_INVALID; }
  return run_impl(hs, c, nullptr, commit_counts, last_states, lc_round, counters, status, committed, proposed, cap, nullptr);
}

// The oracle's commit times of instances [first, first + count), laid out like lbft_commit_times (absolute instance ids):
// committed[(i * N + n) * cap + k] is the clock at which node n's committed_history() grew to k + 1 rows, proposed[i * cap + k]
// the NodeTime of row k of the instance's longest log plus its proposer's startup time; -1 elsewhere.  commit_counts: the
// final committed_history().len() per node.
int ct_oracle_commit_times(const lbft_config* c, uint32_t first, uint32_t count, size_t cap, int64_t* committed, int64_t* proposed,
                           uint32_t* commit_counts) {
  SimConfig base;
  if (!make_cfg(c, base, g_ct_err)) return LBFT_ERR_INVALID;
  if ((uint64_t)first + count > c->num_instances) { g_ct_err = "instance range out of bounds"; return LBFT_ERR_INVALID; }
  const uint32_t N = c->num_nodes;
  for (uint32_t i = first; i < first + count; i++) {
    SimConfig s = base;
    make_partition_plan(c, c->seeds[i], s);
    Simulator sim(c->seeds[i], s);
    int64_t* row = committed + (size_t)i * N * cap;
    std::fill(row, row + (size_t)N * cap, -1);
    std::fill(proposed + (size_t)i * cap, proposed + (size_t)(i + 1) * cap, -1);
    std::vector<uint64_t> len(N, 0);
    try {
      // loop_until(t) handles every event of time t (all at clock t) and drops the first event beyond t: a sentinel that
      // outranks every event of time t + 1 (kind 4 > every kind) is what gets dropped.
      while (!sim.pending_events.empty() && sim.pending_events.top().time <= s.max_clock) {
        const int64_t t = sim.pending_events.top().time;
        sim.pending_events.push(Simulator::Event{t + 1, 0, 4, 0, 0, -1});
        sim.loop_until(t);
        for (uint32_t n = 0; n < N; n++) {
          const uint64_t depth = sim.ledger.entries[sim.nodes[n].context.last_committed_state()].depth;
          for (uint64_t k = len[n]; k < depth && k < cap; k++) row[(size_t)n * cap + k] = t;
          len[n] = depth;
        }
      }
    } catch (const OracleError&) {
    }
    uint32_t best = 0;
    for (uint32_t n = 0; n < N; n++) {
      commit_counts[(size_t)i * N + n] = (uint32_t)len[n];
      if (len[n] > len[best]) best = n;
    }
    const std::vector<CommitEntry> h = sim.nodes[best].context.committed_history();
    for (size_t k = 0; k < h.size() && k < cap; k++) proposed[(size_t)i * cap + k] = h[k].time + sim.nodes[h[k].proposer].startup_time;
  }
  return LBFT_OK;
}
}  // extern "C"
