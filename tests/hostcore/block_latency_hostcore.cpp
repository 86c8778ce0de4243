// block_latency_hostcore.cpp — TEST INFRASTRUCTURE for block-latency statistics (lbft_block_latency_stats).  The CT cores of
// ct_hostcore.cpp (plain handles and sweeps) and fault_hostcore.cpp (fault sweeps), compiled into this unit as they are, run over
// the product's host setup; then the product's spec and threshold checks (latency_spec_error, block_latency_threshold_error) and
// per-instance walk (block_latency_samples_of with the serial block_threshold_time, latency_bin) into a host accumulator, with
// the grouping and exclusion rules of the kernel (the threshold overload of lbft_latency_stats_kernel); and block_threshold_time
// alone over synthetic tables, the reference of the device probe of its lane form.  Never part of, linked into, or reachable
// from the product library.
#include "fault_hostcore.cpp"

extern "C" {

// lbft_create (sets == NULL), lbft_create_sweep (faults == NULL) or lbft_create_sweep_faults, lbft_run, lbft_commit_times at
// `cap` (committed [I][N][cap], proposed [I][cap]) and lbft_block_latency_stats.  status: the run's lbft_status.  unreached and
// hist may be NULL.  Errors are read with ct_hostcore_last_error.
int block_latency_hostcore_stats(const lbft_config* c, const lbft_param_set* sets, const lbft_fault_set* faults, uint32_t num_sets,
                                 const uint32_t* set_of, const lbft_latency_spec* spec, uint64_t threshold, uint32_t* status,
                                 int64_t* committed, int64_t* proposed, size_t cap, lbft_latency_summary* out, uint64_t* unreached,
                                 uint64_t* hist) {
  using namespace lbft;
  HostSetup hs;
  const bool built = !sets ? hs.build(*c)
                           : (faults ? hs.build_sweep_faults(*c, sets, faults, num_sets, set_of) : hs.build_sweep(*c, sets, num_sets, set_of));
  if (!built) { g_ct_err = hs.error; return LBFT_ERR_INVALID; }
  if (!hs.sel.ct) { g_ct_err = "commit times were not recorded: set LBFT_FLAG_COMMIT_TIMES in lbft_config.flags"; return LBFT_ERR_STATE; }
  if (const char* e = latency_spec_error(hs, *spec)) { g_ct_err = e; return LBFT_ERR_INVALID; }
  if (const char* e = block_latency_threshold_error(hs, threshold)) { g_ct_err = e; return LBFT_ERR_INVALID; }
  if (cap == 0 || cap > 0xffffu) { g_ct_err = "cap must be in 1..65535 rows per instance"; return LBFT_ERR_INVALID; }
  const uint32_t I = c->num_instances, N = c->num_nodes, groups = latency_groups(hs);
  // the run, as ct_hostcore.cpp's run_impl and fault_hostcore.cpp's fault_hostcore_run_ct make it
  std::vector<uint32_t> cc((size_t)I * N), lc((size_t)I * N), counters((size_t)I * 12), state;
  std::vector<uint64_t> ls((size_t)I * N);
  const Params P = bind_tables(hs, c, state, cc.data(), ls.data(), lc.data(), counters.data(), status);
  const Layout& L = P.L;
  std::vector<int32_t> times((size_t)I * (N + 1) * L.round_cap, kNotWritten);
  const uint32_t* so = hs.set_of.empty() ? nullptr : hs.set_of.data();
  if (faults) dispatch<true>(P, state, times.data(), hs);
  else if (hs.sel.sweep) run_dispatch<true>(P, N, state, times.data(), nullptr, so, hs.sets.data());
  else run_dispatch<false>(P, N, state, times.data(), nullptr, so, nullptr);
  // the commit times, and the statistics
  LatencyAccumulator acc(out, groups, *spec);
  std::vector<uint64_t> un(groups, 0);
  for (uint32_t i = 0; i < I; i++) {
    const uint32_t* tb = state.data() + (size_t)(i / 32) * L.total_words * 32 + i % 32;
    const uint32_t *icc = cc.data() + (size_t)i * N, *ilc = lc.data() + (size_t)i * N;
    const int32_t* t = times.data() + (size_t)i * (N + 1) * L.round_cap;
    const bool ok = commit_times_of(L, tb, 32, icc, ilc, t, (uint32_t)cap, committed + (size_t)i * N * cap, proposed + (size_t)i * cap);
    const uint32_t g = so ? so[i] : 0u;
    if (!acc.admit(g, status[i])) continue;
    if (!ok) { g_ct_err = "node logs that are not prefixes of one chain"; return LBFT_ERR_STATE; }
    block_latency_samples_of(
        L, tb, 32, icc, ilc, t, spec->proposed_from, spec->proposed_until,
        [&](uint32_t k, uint32_t r) { return block_threshold_time(L, icc, t, P.c_weights, k, r, threshold); },
        [&](int64_t lat) { acc.add(g, lat); }, [&]() { un[g]++; });
  }
  acc.finish(hist);
  if (unreached) std::copy(un.begin(), un.end(), unreached);
  return LBFT_OK;
}

// The serial block_threshold_time over synthetic tables laid out as tests/gpuprobe/block_threshold_probe.cu takes them: cc
// [I][N], times [I][N + 1][round_cap], w [N], W [I]; for every row r, k = r.  T: [I][round_cap], INT64_MAX when unreached.
int block_threshold_hostcore_times(uint32_t N, uint32_t I, uint32_t round_cap, const uint32_t* cc, const int32_t* times,
                                   const uint32_t* w, const uint64_t* W, int64_t* T) {
  using namespace lbft;
  if (N < 1 || N > 64 || round_cap < 1) { g_ct_err = "N must be in 1..64 and round_cap >= 1"; return LBFT_ERR_INVALID; }
  Layout L{};
  L.num_nodes = N;
  L.round_cap = round_cap;
  for (uint32_t i = 0; i < I; i++)
    for (uint32_t r = 0; r < round_cap; r++)
      T[(size_t)i * round_cap + r] =
          block_threshold_time(L, cc + (size_t)i * N, times + (size_t)i * (N + 1) * round_cap, w, r, r, W[i]);
  return LBFT_OK;
}

}  // extern "C"
