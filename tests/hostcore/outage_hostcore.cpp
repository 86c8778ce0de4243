// outage_hostcore.cpp — TEST INFRASTRUCTURE for outage sweeps (lbft_create_sweep_outages).  The device state machine of sweep
// handles (csrc/sim_core.cuh, Core's SW parameter, with and without the commit-time stores of CT) compiled with g++, over the
// product's own host setup (HostSetup::build_sweep_outages), each instance bound to its set's entry of the table the runtime
// uploads (HostSetup::set_table) as the product's sweep kernels bind it (sweep_set_at, bind_faults, bind_rights, bind_committee,
// bind_links, bind_outages), with the matrices and the outage schedules behind SweepParams::links / outages and the union of the
// windowed nodes in SweepParams::down_mask, as the kernels' parameter block carries them.  The runs are read out as
// link_hostcore.cpp reads them.  Also the oracle with link latencies and outage windows (outage_oracle.hpp): runs, commit logs, a
// trace of every pop with its fate, and commit times observed as ct_hostcore.cpp observes a run without them.  link_hostcore.cpp
// (and through it committee_hostcore.cpp, rights_hostcore.cpp, fault_hostcore.cpp, ct_hostcore.cpp and the oracle's C entry
// points) is compiled into this unit as it is.  Never part of, linked into, or reachable from the product library.
#include "link_hostcore.cpp"
#include "outage_oracle.hpp"

namespace {
using namespace lbft;

template <int NMAX, int QMODE, bool CT>
void run_outages(const SweepParams& S, std::vector<uint32_t>& state, int32_t* times, uint32_t records) {
  const Params& P = S.P;
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    const uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * P.L.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, FX_NONE, false, false, 1, false, false, false, true, CT> core(P, mem, P.zig_x, P.zig_f, P.delay_thr,
                                                                                             sk.data() + lane, sd.data() + lane);
    if constexpr (CT) core.ct = times + (size_t)inst * (P.L.num_nodes + 1) * P.L.round_cap;
    core.bind_set(sweep_set_at(S.sets, S.set_of[inst], records));
    core.bind_faults(records & 1);
    core.bind_rights(records & 2);
    core.bind_committee(records & 4);
    core.bind_links(records & 8);
    core.bind_outages(records & 16);
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
  }
}

template <bool CT>
void dispatch_outages(const SweepParams& S, std::vector<uint32_t>& state, int32_t* times, uint32_t rec) {
  const uint32_t N = S.P.L.num_nodes, qs = S.P.L.queue_scan;
  if (qs == 2) run_outages<16, 2, CT>(S, state, times, rec);
  else if (qs == 1) run_outages<16, 1, CT>(S, state, times, rec);
  else if (qs == 3) {
    if (N <= 16) run_outages<16, 3, CT>(S, state, times, rec);
    else if (N <= 32) run_outages<32, 3, CT>(S, state, times, rec);
    else run_outages<64, 3, CT>(S, state, times, rec);
  } else if (N <= 16) run_outages<16, 0, CT>(S, state, times, rec);
  else if (N <= 32) run_outages<32, 0, CT>(S, state, times, rec);
  else run_outages<64, 0, CT>(S, state, times, rec);
}

// outages == NULL: the links sweep harness's setups (lbft_create_sweep_links, or with links NULL too _committees, _rights,
// _faults or lbft_create_sweep), for the equivalence of empty schedules.
bool setup_outages(HostSetup& hs, const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, const uint64_t* vr,
                   const uint32_t* sizes, const uint32_t* links, const lbft_outage* outages, uint32_t num_sets, const uint32_t* set_of) {
  if (!outages) return setup_links(hs, c, sets, faults, vr, sizes, links, num_sets, set_of);
  if (hs.build_sweep_outages(*c, sets, faults, vr, sizes, links, outages, num_sets, set_of)) return true;
  g_ct_err = hs.error;
  return false;
}

// The oracle's per-node windows from `w` ([num_nodes] lbft_outage, or NULL: none), unclamped: the oracle compares the pop clock
// with the windows as given.
std::vector<std::pair<int64_t, int64_t>> oracle_windows(const lbft_config* c, const lbft_outage* w) {
  std::vector<std::pair<int64_t, int64_t>> out;
  if (w)
    for (uint32_t n = 0; n < c->num_nodes; n++) out.emplace_back(w[n].down_from, w[n].down_until);
  return out;
}
}  // namespace

extern "C" {
const char* outage_hostcore_last_error(void) { return g_ct_err.c_str(); }

// The product's lbft_kernel_info and words per instance for this sweep, the bytes of its outage schedules (HostSetup::outages,
// the region lbft_memory_info counts), the device table's records() bits and SweepParams::down_mask.
int outage_hostcore_kernel_info(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, const uint64_t* vr,
                                const uint32_t* sizes, const uint32_t* links, const lbft_outage* outages, uint32_t num_sets,
                                const uint32_t* set_of, char* buf, size_t cap, uint32_t* words, uint64_t* outage_bytes,
                                uint32_t* records, uint64_t* down_mask) {
  HostSetup hs;
  if (!setup_outages(hs, c, sets, faults, vr, sizes, links, outages, num_sets, set_of)) return LBFT_ERR_INVALID;
  snprintf(buf, cap, "%s", kernel_name(hs.sel).c_str());
  *words = hs.params.L.total_words;
  *outage_bytes = hs.outages.size() * sizeof(SweepOutage);
  *records = hs.records();
  *down_mask = hs.down_mask;
  return LBFT_OK;
}

// The SW core (SW + CT with LBFT_FLAG_COMMIT_TIMES): the outputs of the product's lbft_* getters and the per-node last committed
// rounds; proposers[I][cap] the proposer column of lbft_commit_logs (0 past a log's end).  With the flag also lbft_commit_times
// (committed [I][N][cap], proposed [I][cap]).
int outage_hostcore_run(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, const uint64_t* vr,
                        const uint32_t* sizes, const uint32_t* links, const lbft_outage* outages, uint32_t num_sets,
                        const uint32_t* set_of, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                        uint32_t* counters, uint32_t* status, uint32_t* proposers, size_t cap, int64_t* committed,
                        int64_t* proposed) {
  HostSetup hs;
  if (!setup_outages(hs, c, sets, faults, vr, sizes, links, outages, num_sets, set_of)) return LBFT_ERR_INVALID;
  if (cap == 0 || cap > 0xffffu) { g_ct_err = "cap must be in 1..65535 rows per instance"; return LBFT_ERR_INVALID; }
  const uint32_t I = c->num_instances, N = c->num_nodes;
  std::vector<uint32_t> state;
  const Params P = bind_tables(hs, c, state, commit_counts, last_states, lc_round, counters, status);
  const Layout& L = P.L;
  const std::vector<uint64_t> table = hs.set_table();
  const uint32_t rec = hs.records();
  const SweepParams S{P,
                      hs.set_of.data(),
                      reinterpret_cast<const SweepSet*>(table.data()),
                      rec & 1u,
                      (rec >> 1) & 3u,
                      hs.links.empty() ? nullptr : hs.links.data(),
                      hs.outages.empty() ? nullptr : hs.outages.data(),
                      hs.down_mask};
  std::vector<int32_t> times(hs.sel.ct ? (size_t)I * (N + 1) * L.round_cap : 0, kNotWritten);
  if (hs.sel.ct) dispatch_outages<true>(S, state, times.data(), rec);
  else dispatch_outages<false>(S, state, nullptr, rec);
  for (uint32_t i = 0; i < I; i++) {
    const uint32_t* tb = state.data() + (size_t)(i / 32) * L.total_words * 32 + i % 32;
    const uint32_t *icc = commit_counts + (size_t)i * N, *ilc = lc_round + (size_t)i * N;
    const uint32_t leaders = hs.rights.empty() ? 0u : hs.rights[hs.set_of[i]].leader_off;
    for (size_t k = 0; k < cap; k++) proposers[(size_t)i * cap + k] = 0;
    const bool ok = walk_commit_chain(L, tb, 32, icc, ilc, [&](uint32_t k, uint32_t r, uint32_t) {
      if (k < cap) proposers[(size_t)i * cap + k] = hs.leader[leaders + r % L.rspan];
    });
    if (!ok) { g_ct_err = "node logs that are not prefixes of one chain"; return LBFT_ERR_STATE; }
    if (hs.sel.ct)
      commit_times_of(L, tb, 32, icc, ilc, times.data() + (size_t)i * (N + 1) * L.round_cap, (uint32_t)cap,
                      committed + (size_t)i * N * cap, proposed + (size_t)i * cap);
  }
  return LBFT_OK;
}

// lbfo_run_batch of instances [0, num_instances) with link latencies (links[sender * num_nodes + receiver], or NULL: none) and
// outage windows (outages[n], or NULL: none): the outputs of the oracle's run_one.
int outage_oracle_run(const lbft_config* c, const uint32_t* links, const lbft_outage* outages, uint32_t* commit_counts,
                      uint64_t* last_states, lbft_instance_counters* counters, uint32_t* status) {
  SimConfig base;
  std::vector<uint32_t> m;
  if (!link_oracle_cfg(c, links, base, m)) return LBFT_ERR_INVALID;
  const auto w = oracle_windows(c, outages);
  const uint32_t N = c->num_nodes;
  for (uint32_t i = 0; i < c->num_instances; i++) {
    SimConfig s = base;
    make_partition_plan(c, c->seeds[i], s);
    OutageSimulator sim(c->seeds[i], s, m, w);
    uint32_t st = 0;
    try {
      sim.loop_until(s.max_clock);
      st |= LBFT_ST_DONE;
    } catch (const OracleError&) {
      st |= LBFT_ST_INVARIANT;
    }
    for (uint32_t n = 0; n < N; n++) {
      auto& ctx = sim.nodes[n].context;
      commit_counts[(size_t)i * N + n] = sim.ledger.entries[ctx.last_committed_state()].depth;
      last_states[(size_t)i * N + n] = ctx.last_committed_state_key();
      if (sim.nodes[n].node.timeout_and_propose_same_update) st |= LBFT_ST_INVARIANT;
      if (sim.nodes[n].node.epoch_id != 0) st |= LBFT_ST_EPOCH_CHANGE;
    }
    if (sim.rec_counters.response_records_accepted) st |= LBFT_ST_INVARIANT;
    lbft_instance_counters& k = counters[i];
    memset(&k, 0, sizeof k);
    for (int e = 0; e < 4; e++) k.processed[e] = (uint32_t)sim.counters.processed[e];
    k.timers_cancelled = (uint32_t)sim.counters.timers_cancelled;
    k.scheduled = (uint32_t)sim.event_count;
    k.max_active_round = (uint32_t)sim.max_active_round();
    k.rng_draws = (uint32_t)sim.rng.draws;
    k.max_queue = (uint32_t)sim.counters.max_queue;
    k.scheduled_notify = (uint32_t)sim.counters.scheduled_notify;
    status[i] = st;
  }
  return LBFT_OK;
}

// lbfo_commit_log with link latencies and outage windows: committed_history() of one node.
int outage_oracle_commit_log(const lbft_config* c, const uint32_t* links, const lbft_outage* outages, uint32_t instance, uint32_t node,
                             lbft_commit* out, size_t cap, size_t* n) {
  SimConfig s;
  std::vector<uint32_t> m;
  if (!link_oracle_cfg(c, links, s, m)) return LBFT_ERR_INVALID;
  if (instance >= c->num_instances || node >= c->num_nodes) { g_ct_err = "index out of range"; return LBFT_ERR_INVALID; }
  make_partition_plan(c, c->seeds[instance], s);
  OutageSimulator sim(c->seeds[instance], s, m, oracle_windows(c, outages));
  try {
    sim.loop_until(s.max_clock);
  } catch (const OracleError&) {
  }
  const std::vector<CommitEntry> h = sim.nodes[node].context.committed_history();
  *n = h.size();
  for (size_t i = 0; i < h.size() && i < cap; i++) out[i] = lbft_commit{h[i].proposer, h[i].index, h[i].time};
  return LBFT_OK;
}

// Every pop of one instance up to max_clock, in order: rows[k] = {kind, receiver, sender, pop clock, fate (PopFate)}; *n the
// count (rows past cap are not written).
int outage_oracle_trace(const lbft_config* c, const uint32_t* links, const lbft_outage* outages, uint32_t instance, int64_t* rows,
                        size_t cap, size_t* n) {
  SimConfig s;
  std::vector<uint32_t> m;
  if (!link_oracle_cfg(c, links, s, m)) return LBFT_ERR_INVALID;
  if (instance >= c->num_instances) { g_ct_err = "index out of range"; return LBFT_ERR_INVALID; }
  make_partition_plan(c, c->seeds[instance], s);
  OutageSimulator sim(c->seeds[instance], s, m, oracle_windows(c, outages));
  size_t k = 0;
  sim.on_pop = [&](int kind, Author receiver, Author sender, int64_t clk, int fate) {
    if (k < cap) {
      int64_t* r = rows + 5 * k;
      r[0] = kind; r[1] = receiver; r[2] = sender; r[3] = clk; r[4] = fate;
    }
    k++;
  };
  try {
    sim.loop_until(s.max_clock);
  } catch (const OracleError&) {
  }
  *n = k;
  return LBFT_OK;
}

// ct_oracle_commit_times of a run with link latencies and outage windows.
int outage_oracle_commit_times(const lbft_config* c, const uint32_t* links, const lbft_outage* outages, uint32_t first, uint32_t count,
                               size_t cap, int64_t* committed, int64_t* proposed, uint32_t* commit_counts) {
  SimConfig base;
  std::vector<uint32_t> m;
  if (!link_oracle_cfg(c, links, base, m)) return LBFT_ERR_INVALID;
  if ((uint64_t)first + count > c->num_instances) { g_ct_err = "instance range out of bounds"; return LBFT_ERR_INVALID; }
  const auto w = oracle_windows(c, outages);
  const uint32_t N = c->num_nodes;
  for (uint32_t i = first; i < first + count; i++) {
    SimConfig s = base;
    make_partition_plan(c, c->seeds[i], s);
    OutageSimulator sim(c->seeds[i], s, m, w);
    int64_t* row = committed + (size_t)i * N * cap;
    std::fill(row, row + (size_t)N * cap, -1);
    std::fill(proposed + (size_t)i * cap, proposed + (size_t)(i + 1) * cap, -1);
    std::vector<uint64_t> len(N, 0);
    try {
      // one event time at a time, as ct_oracle_commit_times: the sentinel of time t + 1 is the event loop_until(t) drops
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
