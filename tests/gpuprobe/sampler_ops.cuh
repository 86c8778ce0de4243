// sampler_ops.cuh — TEST INFRASTRUCTURE: the op dispatcher of the sampler probe (sampler_probe.cu, on the device) and of its
// host-compiled twin (tests/hostcore/sampler_hostcore.cpp).  One record is one call of a Core sampler method from an explicit
// Xoshiro256** state: seed_rng, next_u64, gen_range_u32 / u64, standard_normal, delay_from_z, sample_delay, or the raw libm
// exp / log the cold paths call (Core::normal_slow, delay_via_exp), for diagnosis.  The records, the cores and the tables are
// the product's (HostSetup::build / build_sweep); never part of, linked into, or reachable from the product library.
#pragma once
#include <string>
#include <vector>

#include "../../librabft_simulator_b200/csrc/host_setup.hpp"
#include "../../librabft_simulator_b200/csrc/sim_core.cuh"

namespace sampler {

enum : uint32_t { OP_SEED = 0, OP_NEXT_U64, OP_RANGE_U32, OP_RANGE_U64, OP_NORMAL, OP_DELAY_FROM_Z, OP_SAMPLE_DELAY, OP_EXP, OP_LOG, OP_COUNT };
// Which core runs the ops: the generic plain one, the bench kernel's compile-time layout (FX_DEFAULT4: FIXED, whose delay is
// always the table lookup), or a sweep's (SW: the delay model of the record's parameter set, bind_set).
enum : uint32_t { CORE_PLAIN = 0, CORE_FIXED = 1, CORE_SWEEP = 2 };
constexpr uint32_t kLanesDisagree = 1u << 31;  // status: the lanes of the record's group did not all compute the same record

// 64 bytes; tests/rng_support.py REC and oracle/oracle_capi.cpp lbfo_sampler read and write the same layout.
struct Rec {
  uint64_t s[4];    // in: the state (OP_SEED: ignored); out: the state after the op (OP_SEED: the state seed_rng makes)
  uint64_t arg;     // in: the seed (OP_SEED), n (OP_RANGE_*), or the bits of z (OP_DELAY_FROM_Z) / x (OP_EXP, OP_LOG)
  uint64_t result;  // out: the integer result (delays as int64), or the bits of a double result
  uint32_t op;
  uint32_t set;     // in: the parameter set (CORE_SWEEP)
  uint32_t draws;   // out: next_u64 calls the op made
  uint32_t status;  // out: Core::status (ST_DELAY_NEAR_INT, ST_TIME_OVERFLOW), and kLanesDisagree
};
static_assert(sizeof(Rec) == 64, "the layout the Python side and the oracle read");

LBFT_HD uint64_t f64_bits(double d) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t b;
  __builtin_memcpy(&b, &d, 8);
  return b;
#endif
}

template <class C>
LBFT_HD void run_op(C& core, Rec& r) {
  core.s0 = r.s[0];
  core.s1 = r.s[1];
  core.s2 = r.s[2];
  core.s3 = r.s[3];
  core.draws = 0;
  core.status = 0;
  const double x = lbft::bits_to_f64(r.arg);
  uint64_t v = 0;
  switch (r.op) {
    case OP_SEED: core.seed_rng(r.arg, core.s0, core.s1, core.s2, core.s3); break;
    case OP_NEXT_U64: v = core.next_u64(); break;
    case OP_RANGE_U32: v = core.gen_range_u32((uint32_t)r.arg); break;
    case OP_RANGE_U64: v = core.gen_range_u64(r.arg); break;
    case OP_NORMAL: v = f64_bits(core.standard_normal()); break;
    case OP_DELAY_FROM_Z: v = (uint64_t)(int64_t)core.delay_from_z(x); break;
    case OP_SAMPLE_DELAY: v = (uint64_t)(int64_t)core.sample_delay(); break;
    case OP_EXP: v = f64_bits(exp(x)); break;
    case OP_LOG: v = f64_bits(log(x)); break;
  }
  r.s[0] = core.s0;
  r.s[1] = core.s1;
  r.s[2] = core.s2;
  r.s[3] = core.s3;
  r.result = v;
  r.draws = core.draws;
  r.status = core.status;
}

// The product's tables for `c` (HostSetup::build), or for a sweep of `c` over `sets` with set s on instance s (build_sweep).
inline bool make_setup(const lbft_config* c, const lbft_param_set* sets, uint32_t num_sets, lbft::HostSetup& hs, std::string& err) {
  if (!c) {
    err = "config must not be NULL";
    return false;
  }
  bool ok;
  if (sets) {
    lbft_config cs = *c;
    cs.num_instances = num_sets;
    std::vector<uint32_t> set_of(num_sets);
    for (uint32_t s = 0; s < num_sets; s++) set_of[s] = s;
    ok = hs.build_sweep(cs, sets, num_sets, set_of.data());
  } else {
    ok = hs.build(*c);
  }
  if (!ok) err = hs.error;
  return ok;
}

// The delay model a record of `core` reads: the launch's (Params), or its parameter set's.
inline lbft::SweepSet model_of(const lbft::HostSetup& hs, uint32_t core, uint32_t set) {
  lbft::SweepSet m{};
  if (core == CORE_SWEEP) return hs.sets[set];
  const lbft::Params& p = hs.params;
  m.delay_kind = p.delay_kind;
  m.delay_const = p.delay_const;
  m.delay_const_value = p.delay_const_value;
  m.mu = p.mu;
  m.sigma = p.sigma;
  m.uni_lo = p.uni_lo;
  m.uni_span = p.uni_span;
  m.delay_kmax = p.delay_kmax;
  return m;
}

// Keeps every record inside the sampler's domain: a nonzero state, n >= 1, a finite |z| <= 14 (the host's ZMAX: the table's
// sentinels bound the walk only there) on a model with a threshold table, finite exp and positive finite log arguments for
// the diagnosis ops; the fixed core only on a model with a table (FIXED always looks the delay up), the sweep core only on a sweep.
inline bool check_records(const lbft::HostSetup& hs, uint32_t core, const Rec* recs, uint64_t n, std::string& err) {
  if (core > CORE_SWEEP || (core == CORE_SWEEP) != !hs.sets.empty()) {
    err = "core must be CORE_PLAIN / CORE_FIXED on a plain setup, CORE_SWEEP on a sweep";
    return false;
  }
  if (core == CORE_FIXED && hs.params.delay_kmax == 0) {
    err = "the fixed core needs a model with a threshold table";
    return false;
  }
  for (uint64_t i = 0; i < n; i++) {
    const Rec& r = recs[i];
    const std::string at = "record " + std::to_string(i) + ": ";
    if (r.op >= OP_COUNT) return err = at + "unknown op", false;
    if (core == CORE_SWEEP && r.set >= hs.sets.size()) return err = at + "set out of range", false;
    if (r.op != OP_SEED && r.op != OP_EXP && r.op != OP_LOG && !(r.s[0] | r.s[1] | r.s[2] | r.s[3]))
      return err = at + "the all-zero state", false;
    if ((r.op == OP_RANGE_U32 && (uint32_t)r.arg == 0) || (r.op == OP_RANGE_U64 && r.arg == 0)) return err = at + "n = 0", false;
    const double x = lbft::bits_to_f64(r.arg);
    if (r.op == OP_DELAY_FROM_Z) {
      const lbft::SweepSet m = model_of(hs, core, r.set);
      if (!(x >= -14.0 && x <= 14.0)) return err = at + "z outside [-14, 14]", false;
      if (m.delay_kmax == 0 || (core != CORE_FIXED && (m.delay_kind != LBFT_DELAY_LOGNORMAL || m.delay_const)))
        return err = at + "delay_from_z on a model without a threshold table", false;
    }
    if ((r.op == OP_EXP && !(x > -1e300 && x < 1e300)) || (r.op == OP_LOG && !(x > 0.0 && x < 1e300)))
      return err = at + "exp argument not finite, or log argument outside (0, 1e300)", false;
  }
  return true;
}

}  // namespace sampler
