// latency_hostcore.cpp — TEST INFRASTRUCTURE for commit-latency statistics (lbft_latency_stats).  The CT core of
// ct_hostcore.cpp (compiled into this unit as it is, with its instance driver and its exports) run over the product's host
// setup, then the product's spec check (latency_spec_error) and per-instance walk (latency_samples_of, latency_bin) into a host
// accumulator, with the grouping and exclusion rules of lbft_latency_stats_kernel.  Never part of, linked into, or reachable
// from the product library.
#include "ct_hostcore.cpp"

extern "C" {

// lbft_create (sets == NULL) or lbft_create_sweep, lbft_run and lbft_latency_stats.  status: the run's lbft_status.  hist may
// be NULL.  Errors are read with ct_hostcore_last_error.
int latency_hostcore_stats(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, const uint32_t* set_of,
                           const lbft_latency_spec* spec, uint32_t* status, lbft_latency_summary* out, uint64_t* hist) {
  using namespace lbft;
  HostSetup hs;
  if (!(sets ? hs.build_sweep(*c, sets, num_sets, set_of) : hs.build(*c))) { g_ct_err = hs.error; return LBFT_ERR_INVALID; }
  if (!hs.sel.ct) { g_ct_err = "commit times were not recorded: set LBFT_FLAG_COMMIT_TIMES in lbft_config.flags"; return LBFT_ERR_STATE; }
  if (const char* e = latency_spec_error(hs, *spec)) { g_ct_err = e; return LBFT_ERR_INVALID; }
  const uint32_t I = c->num_instances, N = c->num_nodes, groups = latency_groups(hs), bins = spec->num_bins;
  // the run, as ct_hostcore.cpp's run_impl makes it
  Params P = hs.params;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.leader = hs.leader.data();
  P.duration = hs.duration.data();
  P.period = hs.period.data();
  P.weights = hs.weights.data();
  P.delay_thr = hs.delay_thr.empty() ? nullptr : hs.delay_thr.data();
  const Layout& L = P.L;
  std::vector<uint32_t> state((size_t)((I + 31) / 32) * L.total_words * 32, 0xdeadbeefu);
  std::vector<int32_t> times((size_t)I * (N + 1) * L.round_cap, kNotWritten);
  std::vector<uint32_t> cc((size_t)I * N), lc((size_t)I * N), counters((size_t)I * 12);
  std::vector<uint64_t> ls((size_t)I * N);
  P.state = state.data();
  P.out_commit_counts = cc.data();
  P.out_last_state = ls.data();
  P.out_lc_round = lc.data();
  P.out_counters = counters.data();
  P.out_status = status;
  P.seeds = c->seeds;
  const uint32_t* so = hs.set_of.empty() ? nullptr : hs.set_of.data();
  const SweepSet* ss = hs.sets.empty() ? nullptr : hs.sets.data();
  if (hs.sel.sweep) run_dispatch<true>(P, N, state, times.data(), nullptr, so, ss);
  else run_dispatch<false>(P, N, state, times.data(), nullptr, so, ss);
  // the statistics
  std::vector<uint64_t> h((size_t)groups * bins, 0);
  for (uint32_t g = 0; g < groups; g++) out[g] = lbft_latency_summary{0, 0, 0, 0, INT64_MAX, -1};
  for (uint32_t i = 0; i < I; i++) {
    const uint32_t g = so ? so[i] : 0u;
    lbft_latency_summary& s = out[g];
    if (status[i] & ST_ERROR_BITS) { s.excluded++; continue; }
    s.instances++;
    const bool ok = latency_samples_of(L, state.data() + (size_t)(i / 32) * L.total_words * 32 + i % 32, 32, cc.data() + (size_t)i * N,
                                       lc.data() + (size_t)i * N, times.data() + (size_t)i * (N + 1) * L.round_cap, spec->proposed_from,
                                       spec->proposed_until, [&](int64_t lat) {
                                         s.samples++;
                                         s.sum += (uint64_t)lat;
                                         s.min = lat < s.min ? lat : s.min;
                                         s.max = lat > s.max ? lat : s.max;
                                         h[(size_t)g * bins + latency_bin(lat, spec->bin_width, bins)]++;
                                       });
    if (!ok) { g_ct_err = "node logs that are not prefixes of one chain"; return LBFT_ERR_STATE; }
  }
  for (uint32_t g = 0; g < groups; g++)
    if (out[g].samples == 0) out[g].min = -1;
  if (hist) std::copy(h.begin(), h.end(), hist);
  return LBFT_OK;
}

}  // extern "C"
