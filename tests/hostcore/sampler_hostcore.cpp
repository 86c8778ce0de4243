// sampler_hostcore.cpp — TEST INFRASTRUCTURE: the host-compiled twin of the sampler probe (tests/gpuprobe/sampler_probe.cu):
// the same op dispatcher (sampler_ops.cuh) over the same Core instantiations at G = 1, compiled with g++ -ffp-contract=off, so
// that a regression in the sampler or in the probe's records fails against the oracle before a GPU run.  Its libm is the
// host's, so it also stands for what the device would compute with glibc's exp / log.  Also exports the product's tables
// (HostSetup::build / build_sweep) for the checks of build_delay_table.  Never part of, linked into, or reachable from the
// product library.
#include <cstring>

#include "../gpuprobe/sampler_ops.cuh"

using sampler::Rec;
static thread_local std::string g_err;

using PlainCore = lbft::Core<lbft::TileMem<32>, 16, 3>;
using FixedCore = lbft::Core<lbft::TileMem<32, true>, 16, 2, lbft::FX_DEFAULT4>;
using SweepCore = lbft::Core<lbft::TileMem<32>, 16, 3, lbft::FX_NONE, false, false, 1, false, false, false, true>;

template <class C>
static void run_all(const lbft::HostSetup& hs, Rec* recs, uint64_t n) {
  lbft::Params P = hs.params;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.delay_thr = hs.delay_thr.data();
  for (uint64_t i = 0; i < n; i++) {
    C core(P, {nullptr, 0}, P.zig_x, P.zig_f, P.delay_thr);
    if constexpr (std::is_same<C, SweepCore>::value) core.bind_set(&hs.sets[recs[i].set]);
    sampler::run_op(core, recs[i]);
  }
}

extern "C" {

const char* sampler_host_last_error() { return g_err.c_str(); }

// sampler_probe (sampler_probe.cu) at G = 1 on the host: the same arguments but G and smem, the same results.
int sampler_host(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, uint32_t core, Rec* recs, uint64_t n) {
  lbft::HostSetup hs;
  if (!sampler::make_setup(c, sets, num_sets, hs, g_err) || !sampler::check_records(hs, core, recs, n, g_err)) return -1;
  if (core == sampler::CORE_PLAIN) run_all<PlainCore>(hs, recs, n);
  else if (core == sampler::CORE_FIXED) run_all<FixedCore>(hs, recs, n);
  else run_all<SweepCore>(hs, recs, n);
  return 0;
}

// The product's tables: the ziggurat (zig_x / zig_f: 257 each, *zig_r), and per set (one set without `sets`) its delay model
// (models: [num_sets] SweepSet, the launch's for a plain setup) and its thresholds at thr[models[s].thr_off ..]; *thr_len the
// number of thresholds, copied up to thr_cap.  0, or -1 (sampler_host_last_error).
int sampler_tables(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, double* zig_x, double* zig_f, double* zig_r,
                   lbft::SweepSet* models, double* thr, uint64_t thr_cap, uint64_t* thr_len) {
  lbft::HostSetup hs;
  if (!sampler::make_setup(c, sets, num_sets, hs, g_err)) return -1;
  memcpy(zig_x, hs.zig_x.data(), 257 * sizeof(double));
  memcpy(zig_f, hs.zig_f.data(), 257 * sizeof(double));
  *zig_r = hs.params.zig_r;
  if (sets) {
    for (uint32_t s = 0; s < num_sets; s++) models[s] = hs.sets[s];
  } else {
    models[0] = sampler::model_of(hs, sampler::CORE_PLAIN, 0);
    models[0].thr_off = 0;
  }
  *thr_len = hs.delay_thr.size();
  memcpy(thr, hs.delay_thr.data(), (hs.delay_thr.size() < thr_cap ? hs.delay_thr.size() : thr_cap) * sizeof(double));
  return 0;
}

}  // extern "C"
