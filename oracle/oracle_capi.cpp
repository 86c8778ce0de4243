// oracle_capi.cpp — C entry points of the CPU ORACLE (TEST INFRASTRUCTURE, see lbft_oracle.hpp).
// Loaded with ctypes by tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference).
// Takes the product's lbft_config so both sides are driven by the very same bytes.
#include <atomic>
#include <chrono>
#include <string>
#include <thread>

#include "../include/lbft.h"
#include "lbft_oracle.hpp"

using namespace lbft_oracle;

static thread_local std::string g_err;

static bool make_cfg(const lbft_config* c, SimConfig& s, std::string& err) {
  if (!c || c->struct_size != sizeof(lbft_config)) { err = "bad lbft_config.struct_size"; return false; }
  if (c->num_nodes < 1 || c->num_nodes > 64) { err = "num_nodes must be in 1..64"; return false; }
  s.num_nodes = c->num_nodes;
  s.max_clock = c->max_clock;
  if (c->delay_kind == LBFT_DELAY_LOGNORMAL) s.delay = RandomDelay::lognormal(c->delay_mean, c->delay_variance);
  else if (c->delay_kind == LBFT_DELAY_UNIFORM) {
    if (c->delay_hi < c->delay_lo || c->delay_lo < 0) { err = "bad uniform delay bounds"; return false; }
    s.delay = RandomDelay::uniform(c->delay_lo, c->delay_hi);
  } else { err = "unknown delay_kind"; return false; }
  s.node.target_commit_interval = c->target_commit_interval;
  s.node.delta = c->delta;
  s.node.gamma = c->gamma;
  s.node.lambda = c->lambda;
  s.commands_per_epoch = c->commands_per_epoch;
  s.true_data_sync = (c->flags & LBFT_FLAG_TRUE_DATA_SYNC) != 0;
  if (c->voting_rights) s.voting_rights.assign(c->voting_rights, c->voting_rights + c->num_nodes);
  if (c->silent) s.silent.assign(c->silent, c->silent + c->num_nodes);
  return true;
}

// EXTENSION D.3 — the per-instance partition plan, drawn from a stream separate from the simulator's.
static void make_partition_plan(const lbft_config* c, uint64_t seed, SimConfig& s) {
  s.partitions.clear();
  if (c->partition_windows == 0 || c->num_nodes < 2) return;
  Xoshiro256StarStar r = Xoshiro256StarStar::seed_from_u64(seed ^ 0xD1B54A32D192ED03ULL);
  uint64_t nsub = c->num_nodes >= 64 ? UINT64_MAX - 1 : ((1ULL << c->num_nodes) - 2);
  for (uint32_t k = 0; k < c->partition_windows; k++) {
    int64_t t0 = (int64_t)gen_range_u64(r, (uint64_t)c->max_clock + 1);
    int64_t len = 1 + (int64_t)gen_range_u64(r, c->partition_max_len ? c->partition_max_len : 1);
    uint64_t mask = 1 + gen_range_u64(r, nsub);
    s.partitions.push_back({t0, t0 + len, mask});
  }
}

static void run_one(const lbft_config* c, const SimConfig& base, uint32_t inst, uint32_t* commit_counts,
                    uint64_t* last_states, lbft_instance_counters* counters, uint32_t* status,
                    std::vector<std::vector<CommitEntry>>* logs, std::vector<lbft_round_switch>* switches = nullptr,
                    const std::vector<int64_t>* stops = nullptr) {
  SimConfig s = base;
  uint64_t seed = c->seeds[inst];
  make_partition_plan(c, seed, s);
  uint32_t st = 0;
  Simulator sim(seed, s);
  sim.record_round_switches = switches != nullptr;
  struct Collect {  // node-major, rounds ascending within a node (the order of include/lbft.h)
    Simulator& sim; std::vector<lbft_round_switch>* out;
    ~Collect() {
      if (!out) return;
      for (size_t n = 0; n < sim.nodes_round_switch.size(); n++)
        for (auto& e : sim.nodes_round_switch[n]) out->push_back(lbft_round_switch{(uint32_t)n, (uint32_t)e.first, e.second});
    }
  } collect{sim, switches};
  try {
    // staged: loop_until called again and again on the same Simulator (simulator.rs:380) — each call drops the first
    // event beyond its clock (:383-391)
    if (stops) for (int64_t t : *stops) sim.loop_until(t);
    else sim.loop_until(s.max_clock);
    st |= LBFT_ST_DONE;
  } catch (const OracleError&) {
    st |= LBFT_ST_INVARIANT;
  }
  uint32_t N = c->num_nodes;
  for (uint32_t n = 0; n < N; n++) {
    auto& ctx = sim.nodes[n].context;
    if (commit_counts) commit_counts[(size_t)inst * N + n] = sim.ledger.entries[ctx.last_committed_state()].depth;
    if (last_states) last_states[(size_t)inst * N + n] = ctx.last_committed_state_key();
    if (sim.nodes[n].node.timeout_and_propose_same_update) st |= LBFT_ST_INVARIANT;
    if (sim.nodes[n].node.epoch_id != 0) st |= LBFT_ST_EPOCH_CHANGE;
    if (logs) logs->push_back(ctx.committed_history());
  }
  if (sim.rec_counters.response_records_accepted) st |= LBFT_ST_INVARIANT;
  if (counters) {
    lbft_instance_counters& k = counters[inst];
    memset(&k, 0, sizeof k);
    for (int i = 0; i < 4; i++) k.processed[i] = (uint32_t)sim.counters.processed[i];
    k.timers_cancelled = (uint32_t)sim.counters.timers_cancelled;
    k.scheduled = (uint32_t)sim.event_count;
    k.max_active_round = (uint32_t)sim.max_active_round();
    k.rng_draws = (uint32_t)sim.rng.draws;
    k.max_queue = (uint32_t)sim.counters.max_queue;
    k.scheduled_notify = (uint32_t)sim.counters.scheduled_notify;
  }
  if (status) status[inst] = st;
}

extern "C" {

const char* lbfo_last_error(void) { return g_err.c_str(); }

// Runs instances [first, first+count) of the batch described by `c` on `threads` host threads.
// Output arrays are indexed by absolute instance id like the product's.  Returns wall seconds of
// the run phase in *seconds (construction + loop_until of every instance).
int lbfo_run_batch(const lbft_config* c, uint32_t first, uint32_t count, uint32_t threads, uint32_t* commit_counts,
                   uint64_t* last_states, lbft_instance_counters* counters, uint32_t* status, double* seconds) {
  SimConfig base;
  if (!make_cfg(c, base, g_err)) return LBFT_ERR_INVALID;
  if ((uint64_t)first + count > c->num_instances) { g_err = "instance range out of bounds"; return LBFT_ERR_INVALID; }
  if (threads == 0) threads = 1;
  auto t0 = std::chrono::steady_clock::now();
  std::atomic<uint32_t> next{0};
  auto worker = [&]() {
    for (;;) {
      uint32_t i = next.fetch_add(1);
      if (i >= count) break;
      run_one(c, base, first + i, commit_counts, last_states, counters, status, nullptr);
    }
  };
  if (threads == 1) worker();
  else {
    std::vector<std::thread> pool;
    for (uint32_t t = 0; t < threads; t++) pool.emplace_back(worker);
    for (auto& t : pool) t.join();
  }
  auto t1 = std::chrono::steady_clock::now();
  if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
  return LBFT_OK;
}

int lbfo_commit_log(const lbft_config* c, uint32_t instance, uint32_t node, lbft_commit* out, size_t cap, size_t* n) {
  SimConfig base;
  if (!make_cfg(c, base, g_err)) return LBFT_ERR_INVALID;
  if (instance >= c->num_instances || node >= c->num_nodes) { g_err = "index out of range"; return LBFT_ERR_INVALID; }
  std::vector<std::vector<CommitEntry>> logs;
  run_one(c, base, instance, nullptr, nullptr, nullptr, nullptr, &logs);
  const auto& h = logs[node];
  if (n) *n = h.size();
  for (size_t i = 0; i < h.size() && i < cap; i++) out[i] = lbft_commit{h[i].proposer, h[i].index, h[i].time};
  return LBFT_OK;
}

// lbfo_run_batch with loop_until called once per entry of stops[] on each instance (the reference of lbft_run_until).
int lbfo_run_batch_staged(const lbft_config* c, uint32_t first, uint32_t count, uint32_t threads, const int64_t* stops,
                          size_t nstops, uint32_t* commit_counts, uint64_t* last_states, lbft_instance_counters* counters,
                          uint32_t* status) {
  SimConfig base;
  if (!make_cfg(c, base, g_err)) return LBFT_ERR_INVALID;
  if ((uint64_t)first + count > c->num_instances) { g_err = "instance range out of bounds"; return LBFT_ERR_INVALID; }
  const std::vector<int64_t> st(stops, stops + nstops);
  if (threads == 0) threads = 1;
  std::atomic<uint32_t> next{0};
  auto worker = [&]() {
    for (;;) {
      uint32_t i = next.fetch_add(1);
      if (i >= count) break;
      run_one(c, base, first + i, commit_counts, last_states, counters, status, nullptr, nullptr, &st);
    }
  };
  std::vector<std::thread> pool;
  for (uint32_t t = 1; t < threads; t++) pool.emplace_back(worker);
  worker();
  for (auto& t : pool) t.join();
  return LBFT_OK;
}

// committed_history() of one node after a staged run.
int lbfo_commit_log_staged(const lbft_config* c, uint32_t instance, uint32_t node, const int64_t* stops, size_t nstops,
                           lbft_commit* out, size_t cap, size_t* n) {
  SimConfig base;
  if (!make_cfg(c, base, g_err)) return LBFT_ERR_INVALID;
  if (instance >= c->num_instances || node >= c->num_nodes) { g_err = "index out of range"; return LBFT_ERR_INVALID; }
  const std::vector<int64_t> st(stops, stops + nstops);
  std::vector<std::vector<CommitEntry>> logs;
  run_one(c, base, instance, nullptr, nullptr, nullptr, nullptr, &logs, nullptr, &st);
  const auto& h = logs[node];
  if (n) *n = h.size();
  for (size_t i = 0; i < h.size() && i < cap; i++) out[i] = lbft_commit{h[i].proposer, h[i].index, h[i].time};
  return LBFT_OK;
}

// Round switches of a staged run of one instance (the DataWriter of each loop_until call is fed the same way; the
// log of a staged run is the concatenation, kept here in one table like the device does).
int lbfo_round_switches_staged(const lbft_config* c, uint32_t instance, const int64_t* stops, size_t nstops,
                               lbft_round_switch* out, size_t cap, size_t* n) {
  SimConfig base;
  if (!make_cfg(c, base, g_err)) return LBFT_ERR_INVALID;
  if (instance >= c->num_instances) { g_err = "index out of range"; return LBFT_ERR_INVALID; }
  const std::vector<int64_t> st(stops, stops + nstops);
  std::vector<lbft_round_switch> sw;
  run_one(c, base, instance, nullptr, nullptr, nullptr, nullptr, nullptr, &sw, &st);
  if (n) *n = sw.size();
  for (size_t i = 0; i < sw.size() && i < cap; i++) out[i] = sw[i];
  return LBFT_OK;
}

// Round switches of one instance, as DataWriter would have collected them (data_writer.rs:34-50).
int lbfo_round_switches(const lbft_config* c, uint32_t instance, lbft_round_switch* out, size_t cap, size_t* n) {
  SimConfig base;
  if (!make_cfg(c, base, g_err)) return LBFT_ERR_INVALID;
  if (instance >= c->num_instances) { g_err = "index out of range"; return LBFT_ERR_INVALID; }
  std::vector<lbft_round_switch> sw;
  run_one(c, base, instance, nullptr, nullptr, nullptr, nullptr, nullptr, &sw);
  if (n) *n = sw.size();
  for (size_t i = 0; i < sw.size() && i < cap; i++) out[i] = sw[i];
  return LBFT_OK;
}

// ---- primitives, exposed so the tests can pin them against the reference's known answers ----
uint64_t lbfo_siphash13(const uint8_t* p, size_t n) {
  SipHasher13 h;
  h.write(p, n);
  return h.finish();
}
uint64_t lbfo_state_key(const lbft_commit* log, size_t n) {  // simulated_context.rs:51-55
  SipHasher13 h;
  h.write_u64(n);
  for (size_t i = 0; i < n; i++) {
    h.write_u64(log[i].proposer);
    h.write_u64(log[i].index);
    h.write_u64((uint64_t)log[i].time);
  }
  return h.finish();
}
void lbfo_xoshiro_seq(uint64_t seed, uint64_t* out, size_t n) {
  Xoshiro256StarStar r = Xoshiro256StarStar::seed_from_u64(seed);
  for (size_t i = 0; i < n; i++) out[i] = r.next_u64();
}
uint32_t lbfo_pick_author(const uint64_t* weights, uint32_t n, uint64_t seed) {  // configuration.rs:65-75
  std::vector<std::pair<Author, uint64_t>> v;
  for (uint32_t i = 0; i < n; i++) v.push_back({(Author)i, weights[i]});
  return (uint32_t)EpochConfiguration(v).pick_author(seed);
}
uint32_t lbfo_leader(const uint64_t* weights, uint32_t n, uint64_t round) {  // pacemaker.rs:100-109
  SipHasher13 h;
  h.write_u64(round);
  return lbfo_pick_author(weights, n, h.finish());
}
uint64_t lbfo_quorum_threshold(const uint64_t* weights, uint32_t n) {  // configuration.rs:52-56
  uint64_t t = 0;
  for (uint32_t i = 0; i < n; i++) t += weights[i];
  return 2 * t / 3 + 1;
}
void lbfo_ziggurat_tables(double* x257, double* f257) {
  memcpy(x257, zig().x, sizeof(double) * 257);
  memcpy(f257, zig().f, sizeof(double) * 257);
}
void lbfo_delay_samples(uint64_t seed, double mean, double variance, int64_t* out, size_t n) {
  Xoshiro256StarStar r = Xoshiro256StarStar::seed_from_u64(seed);
  RandomDelay d = RandomDelay::lognormal(mean, variance);
  for (size_t i = 0; i < n; i++) out[i] = d.sample(r);
}
void lbfo_normal_samples(uint64_t seed, double* out, size_t n) {
  Xoshiro256StarStar r = Xoshiro256StarStar::seed_from_u64(seed);
  for (size_t i = 0; i < n; i++) out[i] = standard_normal(r);
}
void lbfo_shuffle(uint64_t seed, uint32_t* v, size_t n) {
  Xoshiro256StarStar r = Xoshiro256StarStar::seed_from_u64(seed);
  std::vector<uint32_t> w(v, v + n);
  shuffle(w, r);
  memcpy(v, w.data(), n * sizeof(uint32_t));
}
void lbfo_round_durations(int64_t delta, double gamma, double lambda, int64_t* dur, int64_t* period, size_t n) {
  for (size_t i = 0; i < n; i++) {  // pacemaker.rs:123,196  (index i <-> n = i)
    dur[i] = (int64_t)((double)delta * std::pow((double)i, gamma));
    period[i] = (int64_t)(lambda * (double)dur[i]);
  }
}

// One call of the sampler from an explicit Xoshiro256** state (tests/rng_support.py REC; the device's side of it is the sampler
// probe's record): s in / out, arg the seed, n or the bits of z / x, result the integer result or the bits of a double.
struct SamplerRec {
  uint64_t s[4];
  uint64_t arg, result;
  uint32_t op, set, draws, status;
};
static_assert(sizeof(SamplerRec) == 64, "tests/rng_support.py REC");
static uint64_t f64_bits(double d) {
  uint64_t b;
  memcpy(&b, &d, 8);
  return b;
}

// Runs recs[0..n) through the oracle's Xoshiro256StarStar, gen_range_u32 / u64, standard_normal and RandomDelay of `c`'s delay
// model, or of sets[rec.set]'s when sets is not NULL.  Ops: 0 seed_from_u64(arg), 1 next_u64, 2 gen_range_u32(arg),
// 3 gen_range_u64(arg), 4 standard_normal, 5 the LogNormal delay of z = arg, 6 RandomDelay::sample, 7 exp(arg), 8 log(arg)
// (the host libm).  status is always 0.  0, or -1 (lbfo_last_error).
int lbfo_sampler(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, SamplerRec* recs, size_t n) {
  std::vector<RandomDelay> models;
  for (uint32_t s = 0; s < (sets ? num_sets : 1u); s++) {
    lbft_config cs = *c;
    if (sets) {
      cs.delay_kind = sets[s].delay_kind;
      cs.delay_mean = sets[s].delay_mean;
      cs.delay_variance = sets[s].delay_variance;
      cs.delay_lo = sets[s].delay_lo;
      cs.delay_hi = sets[s].delay_hi;
    }
    SimConfig sc;
    if (!make_cfg(&cs, sc, g_err)) return -1;
    models.push_back(sc.delay);
  }
  for (size_t i = 0; i < n; i++) {
    SamplerRec& r = recs[i];
    if (r.set >= models.size() || r.op > 8) { g_err = "record " + std::to_string(i) + ": set or op out of range"; return -1; }
    const RandomDelay& d = models[r.set];
    Xoshiro256StarStar rng;
    memcpy(rng.s, r.s, sizeof r.s);
    double x;
    memcpy(&x, &r.arg, 8);
    uint64_t v = 0;
    switch (r.op) {
      case 0: rng = Xoshiro256StarStar::seed_from_u64(r.arg); break;
      case 1: v = rng.next_u64(); break;
      case 2: v = gen_range_u32(rng, (uint32_t)r.arg); break;
      case 3: v = gen_range_u64(rng, r.arg); break;
      case 4: v = f64_bits(standard_normal(rng)); break;
      case 5: v = (uint64_t)d.lognormal_of(x); break;
      case 6: v = (uint64_t)d.sample(rng); break;
      case 7: v = f64_bits(std::exp(x)); break;
      case 8: v = f64_bits(std::log(x)); break;
    }
    memcpy(r.s, rng.s, sizeof r.s);
    r.result = v;
    r.draws = (uint32_t)rng.draws;
    r.status = 0;
  }
  return 0;
}

int lbfo_selftest(char* buf, size_t cap);  // oracle_selftest.cpp

}  // extern "C"
