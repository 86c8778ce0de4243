// committee_hostcore.cpp — TEST INFRASTRUCTURE for committee sweeps (lbft_create_sweep_committees).  The device state machine of
// sweep handles (csrc/sim_core.cuh, Core's SW parameter, with and without the commit-time stores of CT) compiled with g++, over
// the product's own host setup (HostSetup::build_sweep_committees), each instance bound to its set's entry of the table the
// runtime uploads (HostSetup::set_table) as the product's sweep kernels bind it (sweep_set_at, bind_faults, bind_rights,
// bind_committee).  The runs are read out as rights_hostcore.cpp reads them: proposers from the instance's leader table, commit
// times (commit_times_of) and block-latency statistics per group over the group's weights.  rights_hostcore.cpp (and through it
// fault_hostcore.cpp and ct_hostcore.cpp) is compiled into this unit as it is.  Never part of, linked into, or reachable from the
// product library.
#include "rights_hostcore.cpp"

namespace {
using namespace lbft;

template <int NMAX, int QMODE, bool CT>
void run_committee(const Params& P, std::vector<uint32_t>& state, int32_t* times, const uint32_t* set_of, const SweepSet* table,
                   uint32_t records) {
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    const uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * P.L.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, FX_NONE, false, false, 1, false, false, false, true, CT> core(P, mem, P.zig_x, P.zig_f, P.delay_thr,
                                                                                             sk.data() + lane, sd.data() + lane);
    if constexpr (CT) core.ct = times + (size_t)inst * (P.L.num_nodes + 1) * P.L.round_cap;
    core.bind_set(sweep_set_at(table, set_of[inst], records));
    core.bind_faults(records & 1);
    core.bind_rights(records & 2);
    core.bind_committee(records & 4);
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
  }
}

template <bool CT>
void dispatch_committee(const Params& P, std::vector<uint32_t>& state, int32_t* times, const uint32_t* so, const SweepSet* t, uint32_t rec) {
  const uint32_t N = P.L.num_nodes, qs = P.L.queue_scan;
  if (qs == 2) run_committee<16, 2, CT>(P, state, times, so, t, rec);
  else if (qs == 1) run_committee<16, 1, CT>(P, state, times, so, t, rec);
  else if (qs == 3) {
    if (N <= 16) run_committee<16, 3, CT>(P, state, times, so, t, rec);
    else if (N <= 32) run_committee<32, 3, CT>(P, state, times, so, t, rec);
    else run_committee<64, 3, CT>(P, state, times, so, t, rec);
  } else if (N <= 16) run_committee<16, 0, CT>(P, state, times, so, t, rec);
  else if (N <= 32) run_committee<32, 0, CT>(P, state, times, so, t, rec);
  else run_committee<64, 0, CT>(P, state, times, so, t, rec);
}

// sizes == NULL: lbft_create_sweep_rights (vr given), lbft_create_sweep_faults (faults given) or lbft_create_sweep, for the
// equivalences.
bool setup_committee(HostSetup& hs, const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, const uint64_t* vr,
                     const uint32_t* sizes, uint32_t num_sets, const uint32_t* set_of) {
  if (!sizes) return setup_rights(hs, c, sets, faults, vr, num_sets, set_of);
  if (hs.build_sweep_committees(*c, sets, faults, vr, sizes, num_sets, set_of)) return true;
  g_ct_err = hs.error;
  return false;
}
}  // namespace

extern "C" {
const char* committee_hostcore_last_error(void) { return g_ct_err.c_str(); }

// The product's lbft_kernel_info and words per instance for this sweep, the bytes of its leader tables, the device table's
// records() bits, and each set's leader table (leaders[num_sets][round_cap + 1]; may be NULL).
int committee_hostcore_kernel_info(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, const uint64_t* vr,
                                   const uint32_t* sizes, uint32_t num_sets, const uint32_t* set_of, char* buf, size_t cap,
                                   uint32_t* words, uint64_t* leader_bytes, uint32_t* records, uint8_t* leaders) {
  HostSetup hs;
  if (!setup_committee(hs, c, sets, faults, vr, sizes, num_sets, set_of)) return LBFT_ERR_INVALID;
  snprintf(buf, cap, "%s", kernel_name(hs.sel).c_str());
  *words = hs.params.L.total_words;
  *leader_bytes = hs.leader.size();
  *records = hs.records();
  const size_t span = (size_t)hs.params.L.rspan + 1;
  if (leaders)
    for (uint32_t s = 0; s < num_sets; s++) {
      const uint32_t off = hs.rights.empty() ? 0u : hs.rights[s].leader_off;
      memcpy(leaders + s * span, hs.leader.data() + off, span);
    }
  return LBFT_OK;
}

// The SW core (SW + CT with LBFT_FLAG_COMMIT_TIMES): the outputs of the product's lbft_* getters and the per-node last committed
// rounds; proposers[I][cap] the proposer column of lbft_commit_logs (0 past a log's end), lens[I][N] its lengths (the commit
// counts: lbft_commit_logs' lens).  With the flag also lbft_commit_times (committed [I][N][cap], proposed [I][cap]) and, with
// thresholds (may be NULL), lbft_block_latency_stats_groups into out, unreached and hist (may be NULL).  The outputs are filled
// with garbage first, so that whatever the run leaves unwritten shows.
int committee_hostcore_run(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, const uint64_t* vr,
                           const uint32_t* sizes, uint32_t num_sets, const uint32_t* set_of, uint32_t* commit_counts,
                           uint64_t* last_states, uint32_t* lc_round, uint32_t* counters, uint32_t* status, uint32_t* proposers,
                           size_t cap, int64_t* committed, int64_t* proposed, const lbft_latency_spec* spec, const uint64_t* thresholds,
                           lbft_latency_summary* out, uint64_t* unreached, uint64_t* hist) {
  HostSetup hs;
  if (!setup_committee(hs, c, sets, faults, vr, sizes, num_sets, set_of)) return LBFT_ERR_INVALID;
  if (cap == 0 || cap > 0xffffu) { g_ct_err = "cap must be in 1..65535 rows per instance"; return LBFT_ERR_INVALID; }
  if (thresholds) {
    if (!hs.sel.ct) { g_ct_err = "commit times were not recorded: set LBFT_FLAG_COMMIT_TIMES in lbft_config.flags"; return LBFT_ERR_STATE; }
    if (const char* e = latency_spec_error(hs, *spec)) { g_ct_err = e; return LBFT_ERR_INVALID; }
    if (const char* e = block_latency_thresholds_error(hs, thresholds)) { g_ct_err = e; return LBFT_ERR_INVALID; }
  }
  const uint32_t I = c->num_instances, N = c->num_nodes;
  for (size_t k = 0; k < (size_t)I * N; k++) {
    commit_counts[k] = lc_round[k] = 0xdeadbeefu;
    last_states[k] = 0xdeadbeefdeadbeefULL;
  }
  std::vector<uint32_t> state;
  const Params P = bind_tables(hs, c, state, commit_counts, last_states, lc_round, counters, status);
  const Layout& L = P.L;
  const std::vector<uint64_t> table = hs.set_table();
  const SweepSet* t = reinterpret_cast<const SweepSet*>(table.data());
  std::vector<int32_t> times(hs.sel.ct ? (size_t)I * (N + 1) * L.round_cap : 0, kNotWritten);
  if (hs.sel.ct) dispatch_committee<true>(P, state, times.data(), hs.set_of.data(), t, hs.records());
  else dispatch_committee<false>(P, state, nullptr, hs.set_of.data(), t, hs.records());
  const uint32_t groups = latency_groups(hs);
  std::vector<lbft_latency_summary> unused(groups);  // (the accumulator's summaries when no statistics are asked for)
  LatencyAccumulator acc(thresholds ? out : unused.data(), groups, thresholds ? *spec : lbft_latency_spec{});
  std::vector<uint64_t> un(groups, 0);
  for (uint32_t i = 0; i < I; i++) {
    const uint32_t* tb = state.data() + (size_t)(i / 32) * L.total_words * 32 + i % 32;
    const uint32_t *icc = commit_counts + (size_t)i * N, *ilc = lc_round + (size_t)i * N;
    const uint32_t g = hs.set_of[i];
    const uint32_t leaders = hs.rights.empty() ? 0u : hs.rights[g].leader_off;
    for (size_t k = 0; k < cap; k++) proposers[(size_t)i * cap + k] = 0;
    const bool ok = walk_commit_chain(L, tb, 32, icc, ilc, [&](uint32_t k, uint32_t r, uint32_t) {
      if (k < cap) proposers[(size_t)i * cap + k] = hs.leader[leaders + r % L.rspan];
    });
    if (!ok) { g_ct_err = "node logs that are not prefixes of one chain"; return LBFT_ERR_STATE; }
    if (!hs.sel.ct) continue;
    const int32_t* ti = times.data() + (size_t)i * (N + 1) * L.round_cap;
    commit_times_of(L, tb, 32, icc, ilc, ti, (uint32_t)cap, committed + (size_t)i * N * cap, proposed + (size_t)i * cap);
    if (!thresholds || !acc.admit(g, status[i])) continue;
    const uint32_t* w = hs.rights.empty() ? P.c_weights : hs.rights[g].weights;
    block_latency_samples_of(
        L, tb, 32, icc, ilc, ti, spec->proposed_from, spec->proposed_until,
        [&](uint32_t k, uint32_t r) { return block_threshold_time(L, icc, ti, w, k, r, thresholds[g]); },
        [&](int64_t lat) { acc.add(g, lat); }, [&]() { un[g]++; });
  }
  if (thresholds) {
    acc.finish(hist);
    if (unreached) std::copy(un.begin(), un.end(), unreached);
  }
  return LBFT_OK;
}
}  // extern "C"
