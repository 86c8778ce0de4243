// lbft_oracle.hpp — CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
//
// A C++17 restatement of the LibraBFTv2 discrete-event simulator of
// novifinancial/librabft_simulator (reference checkout: /root/reference, commit cc2ec64d).
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// build, load or call this.  The product library (librabft_simulator_b200/csrc) never includes it.
//
// PARITY PINNING: no Rust toolchain exists in the build image, so the reference cannot be run.
// This restatement is pinned by the reference's own golden vectors instead (tests/test_oracle_*.py,
// oracle/oracle_selftest.cpp):
//   * librabft-v2/tests/simulated_run.rs:45-94   (seed 52 / 3 nodes, seed 48 / 8 nodes: commit counts
//     and last-committed-state keys, which are SipHash-1-3 digests of the full commit logs)
//   * bft-lib/src/unit_tests/configuration_tests.rs:6-47 (pick_author KAT, quorum thresholds)
//   * librabft-v2/src/unit_tests/record_store_tests.rs:106-292 (scripted record-store sequences)
//   * bft-lib/src/unit_tests/simulated_context_tests.rs:79-129, README.md:27 (empty-log state key)
// PARITY UNPINNED for one output: the DataWriter round-switch log (sample_round_numbers, data_writer.rs:34-50) has no
// test, golden or fixture in the reference; it is a reading of the source over the (pinned) event sequence.
// Third-party arithmetic that is NOT under /root/reference (semver pins from bft-lib/Cargo.toml:18-21,
// no lockfile): rand 0.8.3 (gen_range, shuffle), rand_distr 0.4.0 (LogNormal / ziggurat normal),
// rand_xoshiro 0.6.0 (SplitMix64 seeding, Xoshiro256**), Rust std DefaultHasher (SipHash-1-3, zero
// key).  Their published algorithms are restated below; the goldens above pin all of them.
//
// Records are identified by a per-instance creation id instead of a BCS/SipHash content hash
// (reference record hashes are not reproducible run-to-run anyway: QC vote order comes from a
// RandomState HashMap, record_store.rs:709-719).  Execution states are interned (parent, command,
// time) triples; the SipHash state key (simulated_context.rs:51-55) is computed on read-out.
// Unlike the GPU layout, NOTHING here assumes "one block / one QC per round": the store is keyed by
// id, so this oracle independently checks the invariants the device layout relies on.
#pragma once
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <optional>
#include <queue>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

namespace lbft_oracle {

// ---------------------------------------------------------------------------------------------
// SipHash-1-3, k0 = k1 = 0  (Rust std::collections::hash_map::DefaultHasher::new()).
// Call sites: simulated_context.rs:51-55 (state key), pacemaker.rs:100-109 (leader seed).
// ---------------------------------------------------------------------------------------------
struct SipHasher13 {
  uint64_t v0, v1, v2, v3;
  uint64_t tail = 0;
  unsigned ntail = 0;
  uint64_t length = 0;
  SipHasher13() {
    v0 = 0x736f6d6570736575ULL;
    v1 = 0x646f72616e646f6dULL;
    v2 = 0x6c7967656e657261ULL;
    v3 = 0x7465646279746573ULL;
  }
  static inline uint64_t rotl(uint64_t x, int b) { return (x << b) | (x >> (64 - b)); }
  inline void round() {
    v0 += v1; v1 = rotl(v1, 13); v1 ^= v0; v0 = rotl(v0, 32);
    v2 += v3; v3 = rotl(v3, 16); v3 ^= v2;
    v0 += v3; v3 = rotl(v3, 21); v3 ^= v0;
    v2 += v1; v1 = rotl(v1, 17); v1 ^= v2; v2 = rotl(v2, 32);
  }
  inline void absorb(uint64_t m) { v3 ^= m; round(); v0 ^= m; }
  void write(const uint8_t* p, size_t n) {
    length += n;
    for (size_t i = 0; i < n; i++) {
      tail |= (uint64_t)p[i] << (8 * ntail);
      if (++ntail == 8) { absorb(tail); tail = 0; ntail = 0; }
    }
  }
  void write_u64(uint64_t x) {  // write_usize / write_i64 feed 8 LE bytes
    if (ntail == 0) { length += 8; absorb(x); return; }
    uint8_t b[8];
    for (int i = 0; i < 8; i++) b[i] = (uint8_t)(x >> (8 * i));
    write(b, 8);
  }
  uint64_t finish() const {
    SipHasher13 s = *this;
    uint64_t b = (s.length << 56) | s.tail;
    s.v3 ^= b; s.round(); s.v0 ^= b;
    s.v2 ^= 0xff;
    s.round(); s.round(); s.round();
    return s.v0 ^ s.v1 ^ s.v2 ^ s.v3;
  }
};

// ---------------------------------------------------------------------------------------------
// rand_xoshiro 0.6.0: SplitMix64 seeding + Xoshiro256StarStar (simulator.rs:212, configuration.rs:66)
// ---------------------------------------------------------------------------------------------
struct Xoshiro256StarStar {
  uint64_t s[4];
  uint64_t draws = 0;  // instrumentation only
  static Xoshiro256StarStar seed_from_u64(uint64_t seed) {
    Xoshiro256StarStar r;
    uint64_t x = seed;
    for (int i = 0; i < 4; i++) {
      x += 0x9e3779b97f4a7c15ULL;
      uint64_t z = x;
      z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
      z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
      r.s[i] = z ^ (z >> 31);
    }
    return r;
  }
  static inline uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
  uint64_t next_u64() {
    draws++;
    uint64_t result = rotl(s[1] * 5, 7) * 9;
    uint64_t t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
    s[2] ^= t;
    s[3] = rotl(s[3], 45);
    return result;
  }
  uint32_t next_u32() { return (uint32_t)(next_u64() >> 32); }
};

// rand 0.8.3 UniformInt::sample_single_inclusive for usize (64-bit): configuration.rs:67
inline uint64_t gen_range_u64(Xoshiro256StarStar& rng, uint64_t n /* range 0..n, n>0 */) {
  uint64_t zone = (n << __builtin_clzll(n)) - 1;
  for (;;) {
    uint64_t v = rng.next_u64();
    unsigned __int128 m = (unsigned __int128)v * n;
    uint64_t lo = (uint64_t)m, hi = (uint64_t)(m >> 64);
    if (lo <= zone) return hi;
  }
}
// ... and for u32 (used by SliceRandom::shuffle's gen_index for len <= u32::MAX)
inline uint32_t gen_range_u32(Xoshiro256StarStar& rng, uint32_t n) {
  uint32_t zone = (n << __builtin_clz(n)) - 1;
  for (;;) {
    uint32_t v = rng.next_u32();
    uint64_t m = (uint64_t)v * n;
    uint32_t lo = (uint32_t)m, hi = (uint32_t)(m >> 32);
    if (lo <= zone) return hi;
  }
}
// rand 0.8.3 SliceRandom::shuffle (simulator.rs:343,370)
template <class T>
inline void shuffle(std::vector<T>& v, Xoshiro256StarStar& rng) {
  for (size_t i = v.size(); i-- > 1;) {
    size_t j = gen_range_u32(rng, (uint32_t)(i + 1));
    std::swap(v[i], v[j]);
  }
}

// ---------------------------------------------------------------------------------------------
// rand_distr 0.4.0: StandardNormal via 256-layer ziggurat; Normal; LogNormal.
// The crate ships decimal literals generated by its ziggurat_tables.py with "%.18f"; the tables are
// regenerated here with the same recurrence and the same rounding through "%.18f".
// ---------------------------------------------------------------------------------------------
struct ZigguratTables {
  double x[257];
  double f[257];
  double r;
  ZigguratTables() {
    const double R = 3.6541528853610088, V = 0.00492867323399;
    auto pdf = [](double t) { return std::exp(-t * t / 2.0); };
    auto pdf_inv = [](double y) { return std::sqrt(-2.0 * std::log(y)); };
    double xs[257];
    xs[0] = V / pdf(R);
    xs[1] = R;
    for (int i = 2; i < 256; i++) xs[i] = pdf_inv(V / xs[i - 1] + pdf(xs[i - 1]));
    xs[256] = 0.0;
    auto through_literal = [](double v) {
      char buf[64];
      snprintf(buf, sizeof buf, "%.18f", v);
      return strtod(buf, nullptr);
    };
    for (int i = 0; i <= 256; i++) {
      x[i] = through_literal(xs[i]);
      f[i] = through_literal(pdf(xs[i]));
    }
    r = through_literal(R);  // ZIG_NORM_R = 3.654152885361008796
  }
};
inline const ZigguratTables& zig() {
  static const ZigguratTables t;
  return t;
}
inline double f64_from_bits(uint64_t b) {
  double d;
  memcpy(&d, &b, 8);
  return d;
}
inline double open01(Xoshiro256StarStar& rng) {
  // rand 0.8 Open01 for f64: into_float_with_exponent(0) of (next_u64 >> 12), minus (1 - EPSILON/2)
  return f64_from_bits((1023ULL << 52) | (rng.next_u64() >> 12)) - (1.0 - 2.220446049250313e-16 / 2.0);
}
inline double standard_normal(Xoshiro256StarStar& rng) {
  const ZigguratTables& T = zig();
  for (;;) {
    uint64_t bits = rng.next_u64();
    unsigned i = (unsigned)(bits & 0xff);
    double u = f64_from_bits((1024ULL << 52) | (bits >> 12)) - 3.0;  // [-1, 1)
    double x = u * T.x[i];
    if (std::fabs(x) < T.x[i + 1]) return x;
    if (i == 0) {
      double xx = 1.0, yy = 0.0;
      while (-2.0 * yy < xx * xx) {
        double a = open01(rng);
        double b = open01(rng);
        xx = std::log(a) / T.r;
        yy = std::log(b);
      }
      return u < 0.0 ? xx - T.r : T.r - xx;
    }
    double g = (double)(rng.next_u64() >> 11) * (1.0 / 9007199254740992.0);  // Standard f64: 53 bits
    if (T.f[i + 1] + (T.f[i] - T.f[i + 1]) * g < std::exp(-x * x / 2.0)) return x;
  }
}

// simulator.rs:39-43,99-118 — RandomDelay.  kind 0 = the reference's LogNormal(mean, variance).
// kind 1 = EXTENSION (BASELINE config 2, SURVEY App. D.1): integer uniform on [lo, hi], one 64-bit
// gen_range draw per delay.  Not in the reference; parity for it is GPU-vs-this-oracle only.
struct RandomDelay {
  int kind = 0;
  double mu = 0, sigma = 0;
  int64_t lo = 0, hi = 0;
  static RandomDelay lognormal(double mean, double variance) {
    RandomDelay d;
    d.kind = 0;
    d.mu = std::log(mean / std::sqrt(1.0 + variance / (mean * mean)));
    d.sigma = std::sqrt(std::log(1.0 + variance / (mean * mean)));
    return d;
  }
  static RandomDelay uniform(int64_t lo, int64_t hi) {
    RandomDelay d;
    d.kind = 1;
    d.lo = lo;
    d.hi = hi;
    return d;
  }
  int64_t sample(Xoshiro256StarStar& rng) const {
    if (kind == 1) return lo + (int64_t)gen_range_u64(rng, (uint64_t)(hi - lo + 1));
    return lognormal_of(standard_normal(rng));
  }
  // The LogNormal delay of the standard normal deviate n.
  int64_t lognormal_of(double n) const {
    double v = std::exp(mu + sigma * n);  // Normal: mean + std_dev * n; LogNormal: exp
    return (int64_t)v;                    // simulator.rs:117 `v as i64`
  }
};

// ---------------------------------------------------------------------------------------------
// base types (base_types.rs:19-79)
// ---------------------------------------------------------------------------------------------
using Round = uint64_t;
using Author = int;
using NodeTime = int64_t;
using Duration = int64_t;
using EpochId = uint64_t;
constexpr NodeTime NODE_TIME_NEVER = INT64_MAX;
using StateId = int32_t;   // index into LedgerIntern; 0 = empty history
using BlockId = int32_t;   // stand-in for BlockHash
using QcId = int32_t;      // stand-in for QuorumCertificateHash

// GlobalTime <-> NodeTime (bft-lib/src/simulator.rs:120-126): a node's clock starts at its startup time.
using GlobalTime = int64_t;
inline NodeTime to_node_time(GlobalTime t, GlobalTime startup_time) { return t - startup_time; }
inline GlobalTime from_node_time(NodeTime t, GlobalTime startup_time) { return t + startup_time; }

// librabft-v2/src/util.rs:8-10
inline bool is_power2_minus1(size_t x) { return (x & (x + 1)) == 0; }
// librabft-v2/src/util.rs:12-53: merge two sequences sorted by `cmp` (< 0, 0, > 0); elements that compare Equal are kept once
// when they are `eq`, both (first sequence's first) otherwise.
template <class T, class Cmp, class Eq>
inline std::vector<T> merge_sort(const std::vector<T>& v1, const std::vector<T>& v2, Cmp cmp, Eq eq) {
  std::vector<T> result;
  size_t i = 0, j = 0;
  while (i < v1.size() && j < v2.size()) {
    const int c = cmp(v1[i], v2[j]);
    if (c < 0) result.push_back(v1[i++]);
    else if (c == 0) {
      if (eq(v1[i], v2[j])) result.push_back(v1[i]);
      else { result.push_back(v1[i]); result.push_back(v2[j]); }
      i++; j++;
    } else result.push_back(v2[j++]);
  }
  while (i < v1.size()) result.push_back(v1[i++]);
  while (j < v2.size()) result.push_back(v2[j++]);
  return result;
}
constexpr QcId QC_INITIAL = -1;

struct Command {
  Author proposer;
  uint64_t index;
  bool operator==(const Command& o) const { return proposer == o.proposer && index == o.index; }
};
struct CommitEntry {
  uint32_t proposer;
  uint32_t index;
  int64_t time;
};

// Interned SimulatedLedgerState values (simulated_context.rs:38-72).  A state is its execution
// history; two histories are equal iff (parent, command, time) chains are equal, so interning the
// triple gives the same equality as the reference's SipHash key (modulo hash collisions).
struct LedgerIntern {
  struct Entry {
    StateId parent;
    Command cmd;
    NodeTime time;
    uint32_t depth;
  };
  std::vector<Entry> entries;
  std::map<std::tuple<StateId, int, uint64_t, int64_t>, StateId> index;
  LedgerIntern() { entries.push_back({-1, {0, 0}, 0, 0}); }
  StateId execute(StateId base, const Command& c, NodeTime t) {
    auto key = std::make_tuple(base, c.proposer, c.index, t);
    auto it = index.find(key);
    if (it != index.end()) return it->second;
    StateId id = (StateId)entries.size();
    entries.push_back({base, c, t, entries[base].depth + 1});
    index.emplace(key, id);
    return id;
  }
  std::vector<CommitEntry> history(StateId s) const {
    std::vector<CommitEntry> h(entries[s].depth);
    for (StateId cur = s; cur > 0; cur = entries[cur].parent) {
      const Entry& e = entries[cur];
      h[e.depth - 1] = {(uint32_t)e.cmd.proposer, (uint32_t)e.cmd.index, e.time};
    }
    return h;
  }
  // SimulatedLedgerState::key, simulated_context.rs:51-55: Vec<(Command, NodeTime)>::hash
  uint64_t key(StateId s) const {
    SipHasher13 h;
    auto hist = history(s);
    h.write_u64(hist.size());
    for (auto& e : hist) {
      h.write_u64(e.proposer);
      h.write_u64(e.index);
      h.write_u64((uint64_t)e.time);
    }
    return h.finish();
  }
};

// configuration.rs:29-75
struct EpochConfiguration {
  std::vector<std::pair<Author, uint64_t>> authors;
  std::map<Author, uint64_t> voting_rights;
  uint64_t total_votes = 0;
  EpochConfiguration() {}
  explicit EpochConfiguration(const std::vector<std::pair<Author, uint64_t>>& a) : authors(a) {
    for (auto& p : a) {
      voting_rights[p.first] = p.second;
      total_votes += p.second;
    }
  }
  uint64_t weight(Author a) const {
    auto it = voting_rights.find(a);
    return it == voting_rights.end() ? 0 : it->second;
  }
  uint64_t quorum_threshold() const { return 2 * total_votes / 3 + 1; }
  uint64_t validity_threshold() const { return (total_votes + 2) / 3; }
  Author pick_author(uint64_t seed) const {
    Xoshiro256StarStar rng = Xoshiro256StarStar::seed_from_u64(seed);
    uint64_t target = gen_range_u64(rng, total_votes);
    for (auto& p : authors) {
      if (p.second > target) return p.first;
      target -= p.second;
    }
    abort();  // unreachable!()
  }
};

struct OracleError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

// ---------------------------------------------------------------------------------------------
// SimulatedContext (simulated_context.rs:74-274): fake crypto is dropped (signatures always verify
// for honestly built records), the ledger / fetch / commit semantics are kept exactly.
// ---------------------------------------------------------------------------------------------
struct SimulatedContext {
  Author author_ = 0;
  size_t num_nodes = 0;
  uint64_t max_command_per_epoch = 0;
  uint64_t next_fetched_command_index = 0;
  StateId last_committed_ledger_state = 0;
  std::set<StateId> pending_ledger_states;
  LedgerIntern* ledger = nullptr;
  const std::vector<uint64_t>* voting_rights_override = nullptr;  // EXTENSION (App. D.2); null = all 1

  SimulatedContext() {}
  SimulatedContext(Author a, size_t n, uint64_t cpe, LedgerIntern* l)
      : author_(a), num_nodes(n), max_command_per_epoch(cpe), ledger(l) {}
  Author author() const { return author_; }
  bool has_ledger_state(StateId s) const {  // get_ledger_state :102-108
    return s == last_committed_ledger_state || pending_ledger_states.count(s);
  }
  Command fetch() {  // :116-125
    Command c{author_, next_fetched_command_index};
    next_fetched_command_index++;
    return c;
  }
  std::optional<StateId> compute(StateId base, const Command& c, NodeTime t) {  // :128-157
    if (!has_ledger_state(base)) return std::nullopt;
    StateId ns = ledger->execute(base, c, t);
    pending_ledger_states.insert(ns);
    return ns;
  }
  void commit(StateId s) {  // :161-185
    auto it = pending_ledger_states.find(s);
    if (it == pending_ledger_states.end()) throw OracleError("Committed states should be known");
    pending_ledger_states.erase(it);
    // happened_just_before (:61-71): len+1 and equal prefix  <=>  parent == last committed
    if (ledger->entries[s].parent != last_committed_ledger_state)
      throw OracleError("commit does not extend the last committed state by one");
    last_committed_ledger_state = s;
  }
  StateId last_committed_state() const { return last_committed_ledger_state; }
  EpochId read_epoch_id(StateId s) const {  // :199-207
    if (!has_ledger_state(s)) throw OracleError("Read states should be known");
    return ledger->entries[s].depth / max_command_per_epoch;
  }
  EpochConfiguration configuration(StateId) const {  // :209-216 (uniform weight 1)
    std::vector<std::pair<Author, uint64_t>> v;
    for (size_t i = 0; i < num_nodes; i++)
      v.push_back({(Author)i, voting_rights_override ? (*voting_rights_override)[i] : 1});
    return EpochConfiguration(v);
  }
  std::vector<CommitEntry> committed_history() const { return ledger->history(last_committed_ledger_state); }
  uint64_t last_committed_state_key() const { return ledger->key(last_committed_ledger_state); }
};

// ---------------------------------------------------------------------------------------------
// Records (record.rs:52-111)
// ---------------------------------------------------------------------------------------------
struct Block {
  BlockId id;
  Command command;
  NodeTime time;
  QcId previous_quorum_certificate_hash;
  Round round;
  Author author;
};
struct Vote {
  EpochId epoch_id;
  Round round;
  BlockId certified_block_hash;
  StateId state;
  std::optional<StateId> committed_state;
  Author author;
};
struct QuorumCertificate {
  QcId id;
  EpochId epoch_id;
  Round round;
  BlockId certified_block_hash;
  StateId state;
  std::optional<StateId> committed_state;
  std::vector<Author> votes;
  Author author;
};
struct Timeout {
  EpochId epoch_id;
  Round round;
  Round highest_certified_block_round;
  Author author;
};
struct Record {
  enum Kind { BLOCK, VOTE, QC, TIMEOUT } kind;
  Block block;
  Vote vote;
  QuorumCertificate qc;
  Timeout timeout;
  static Record of(const Block& b) { Record r; r.kind = BLOCK; r.block = b; return r; }
  static Record of(const Vote& v) { Record r; r.kind = VOTE; r.vote = v; return r; }
  static Record of(const QuorumCertificate& q) { Record r; r.kind = QC; r.qc = q; return r; }
  static Record of(const Timeout& t) { Record r; r.kind = TIMEOUT; r.timeout = t; return r; }
};

// Per-instance id source standing in for content hashes.
struct IdSource {
  int32_t next_block = 0, next_qc = 0;
};

struct Counters {
  uint64_t inserts_tried[4] = {0, 0, 0, 0};
  uint64_t inserts_ok[4] = {0, 0, 0, 0};
  uint64_t response_records_accepted = 0;  // App. C.5: must stay 0 in the simulator
};

struct PacemakerState;

// ---------------------------------------------------------------------------------------------
// RecordStoreState (record_store.rs:93-843)
// ---------------------------------------------------------------------------------------------
struct RecordStoreState {
  EpochId epoch_id = 0;
  EpochConfiguration configuration;
  QcId initial_hash = QC_INITIAL;
  StateId initial_state = 0;
  std::unordered_map<BlockId, Block> blocks;
  std::unordered_map<QcId, QuorumCertificate> quorum_certificates;
  std::optional<BlockId> current_proposed_block;
  Round highest_quorum_certificate_round_ = 0;
  QcId highest_quorum_certificate_hash_ = QC_INITIAL;
  Round highest_timeout_certificate_round_ = 0;
  Round current_round_ = 1;
  Round highest_committed_round_ = 0;
  std::optional<QcId> highest_commit_certificate_hash;
  std::optional<std::vector<Timeout>> highest_timeout_certificate;
  std::map<Author, Timeout> current_timeouts;  // ascending author (SURVEY B.10)
  std::map<Author, Vote> current_votes;
  uint64_t current_timeouts_weight = 0;
  enum ElectionKind { ONGOING, WON, CLOSED } election = ONGOING;
  std::map<std::pair<BlockId, StateId>, uint64_t> ballot;
  BlockId won_block = -1;
  StateId won_state = -1;
  IdSource* ids = nullptr;
  Counters* counters = nullptr;

  RecordStoreState() {}
  RecordStoreState(QcId initial_hash_, StateId initial_state_, EpochId e, EpochConfiguration c, IdSource* i,
                   Counters* cn)
      : epoch_id(e), configuration(std::move(c)), initial_hash(initial_hash_), initial_state(initial_state_),
        highest_quorum_certificate_hash_(initial_hash_), ids(i), counters(cn) {}

  const Block* block(BlockId h) const {
    auto it = blocks.find(h);
    return it == blocks.end() ? nullptr : &it->second;
  }
  const QuorumCertificate* quorum_certificate(QcId h) const {
    auto it = quorum_certificates.find(h);
    return it == quorum_certificates.end() ? nullptr : &it->second;
  }
  // BackwardQuorumCertificateIterator :137-166
  struct BackIter {
    const RecordStoreState* store;
    QcId current;
    const QuorumCertificate* next() {
      if (current == store->initial_hash) return nullptr;
      const QuorumCertificate* qc = store->quorum_certificate(current);
      const Block* b = store->block(qc->certified_block_hash);
      current = b->previous_quorum_certificate_hash;
      return qc;
    }
  };
  BackIter back_iter(QcId h) const { return BackIter{this, h}; }

  Author pick_author(uint64_t seed) const { return configuration.pick_author(seed); }
  // PacemakerState::leader, pacemaker.rs:100-109
  Author leader(Round round) const {
    SipHasher13 h;
    h.write_u64(round);
    return pick_author(h.finish());
  }

  void update_current_round(Round round) {  // :207-219
    if (round <= current_round_) return;
    current_round_ = round;
    current_proposed_block.reset();
    current_timeouts.clear();
    current_votes.clear();
    current_timeouts_weight = 0;
    election = ONGOING;
    ballot.clear();
  }
  void update_commit_3chain_round(QcId qc_hash) {  // :221-235
    BackIter it = back_iter(qc_hash);
    const QuorumCertificate* q3 = it.next();
    const QuorumCertificate* q2 = q3 ? it.next() : nullptr;
    const QuorumCertificate* q1 = q2 ? it.next() : nullptr;
    if (q1 && q2 && q3) {
      Round r3 = q3->round, r2 = q2->round, r1 = q1->round;
      if (r3 == r2 + 1 && r2 == r1 + 1 && r1 > highest_committed_round_) {
        highest_committed_round_ = r1;
        highest_commit_certificate_hash = qc_hash;
      }
    }
  }
  std::optional<StateId> vote_committed_state(BlockId block_hash) const {  // :237-255
    const Block* b = block(block_hash);
    Round r3 = b->round;
    BackIter it = back_iter(b->previous_quorum_certificate_hash);
    const QuorumCertificate* qc2 = it.next();
    const QuorumCertificate* qc1 = qc2 ? it.next() : nullptr;
    if (qc1 && qc2) {
      Round r2 = qc2->round, r1 = qc1->round;
      if (r3 == r2 + 1 && r2 == r1 + 1) return qc1->state;
    }
    return std::nullopt;
  }

  // verify_network_record :257-417.  Returns an error string or nullptr; ids play the role of hashes.
  const char* verify_network_record(const Record& record) const {
    switch (record.kind) {
      case Record::BLOCK: {
        const Block& b = record.block;
        if (blocks.count(b.id)) return "Block was already inserted.";
        if (!(b.previous_quorum_certificate_hash == initial_hash ||
              quorum_certificates.count(b.previous_quorum_certificate_hash)))
          return "The previous QC (if any) must be verified first.";
        if (initial_hash == b.previous_quorum_certificate_hash) {
          if (!(b.round > 0)) return "Rounds must start at 1";
        } else {
          const QuorumCertificate* pqc = quorum_certificate(b.previous_quorum_certificate_hash);
          const Block* pb = block(pqc->certified_block_hash);
          if (!(b.round > pb->round)) return "Rounds must be increasing";
        }
        return nullptr;
      }
      case Record::VOTE: {
        const Vote& v = record.vote;
        if (v.epoch_id != epoch_id) return "Epoch identifier of vote must match the current epoch.";
        if (!blocks.count(v.certified_block_hash)) return "The certified block hash of a vote must be verified first.";
        if (block(v.certified_block_hash)->round != v.round) return "The round of the vote must match the certified block.";
        if (vote_committed_state(v.certified_block_hash) != v.committed_state)
          return "The committed_state value of a vote must follow the commit rule.";
        if (v.round != current_round_) return "Only accepting votes for a proposal at the current round.";
        if (current_votes.count(v.author)) return "We insert votes only for authors who haven't voted yet.";
        return nullptr;
      }
      case Record::QC: {
        const QuorumCertificate& q = record.qc;
        if (q.epoch_id != epoch_id) return "Epoch identifier of QC must match the current epoch.";
        if (quorum_certificates.count(q.id)) return "QuorumCertificate was already inserted.";
        if (!blocks.count(q.certified_block_hash)) return "The certified block hash of a QC must be verified first.";
        if (block(q.certified_block_hash)->round != q.round) return "The round of the QC must match the certified block.";
        if (q.author != block(q.certified_block_hash)->author) return "QCs must be created by the author of the certified block";
        if (vote_committed_state(q.certified_block_hash) != q.committed_state)
          return "The committed_state value of a QC must follow the commit rule.";
        uint64_t weight = 0;
        for (Author a : q.votes) weight += configuration.weight(a);
        if (!(weight >= configuration.quorum_threshold())) return "Votes in QCs must form a quorum";
        return nullptr;
      }
      case Record::TIMEOUT: {
        const Timeout& t = record.timeout;
        if (t.epoch_id != epoch_id) return "Epoch identifier of timeout must match the current epoch.";
        if (!(t.highest_certified_block_round <= highest_quorum_certificate_round_))
          return "Timeouts must refer to a known certified block round.";
        if (t.round != current_round_) return "Accepting only timeouts at the current round.";
        if (current_timeouts.count(t.author)) return "A timeout is already known for the same round and the same author";
        return nullptr;
      }
    }
    return "unreachable";
  }

  std::optional<StateId> compute_state(BlockId block_hash, SimulatedContext& context) const {  // :426-454
    const Block* b = block(block_hash);
    StateId previous_state;
    if (b->previous_quorum_certificate_hash == initial_hash) previous_state = initial_state;
    else previous_state = quorum_certificate(b->previous_quorum_certificate_hash)->state;
    return context.compute(previous_state, b->command, b->time);
  }

  // try_insert_network_record :456-541
  const char* try_insert_network_record(const Record& record, SimulatedContext& context) {
    if (const char* err = verify_network_record(record)) return err;
    switch (record.kind) {
      case Record::BLOCK: {
        const Block& b = record.block;
        if (b.round == current_round_ && leader(b.round) == b.author) current_proposed_block = b.id;
        blocks.emplace(b.id, b);
        break;
      }
      case Record::VOTE: {
        const Vote& v = record.vote;
        current_votes.emplace(v.author, v);
        if (election == ONGOING) {
          uint64_t& entry = ballot[{v.certified_block_hash, v.state}];
          entry += configuration.weight(v.author);
          if (entry >= configuration.quorum_threshold()) {
            election = WON;
            won_block = v.certified_block_hash;
            won_state = v.state;
          }
        }
        break;
      }
      case Record::QC: {
        const QuorumCertificate& q = record.qc;
        quorum_certificates.emplace(q.id, q);  // inserted BEFORE execution (:505)
        std::optional<StateId> st = compute_state(q.certified_block_hash, context);
        if (st) {
          if (*st != q.state) return "I computed a different state for a QC. This is very bad";
        } else {
          return "I failed to execute a block with a QC";  // QC stays inserted (:515-517)
        }
        if (q.round > highest_quorum_certificate_round_) {
          highest_quorum_certificate_round_ = q.round;
          highest_quorum_certificate_hash_ = q.id;
        }
        update_current_round(q.round + 1);
        update_commit_3chain_round(q.id);
        break;
      }
      case Record::TIMEOUT: {
        const Timeout& t = record.timeout;
        current_timeouts.emplace(t.author, t);
        current_timeouts_weight += configuration.weight(t.author);
        if (current_timeouts_weight >= configuration.quorum_threshold()) {
          std::vector<Timeout> tc;
          for (auto& kv : current_timeouts) tc.push_back(kv.second);
          highest_timeout_certificate = std::move(tc);
          highest_timeout_certificate_round_ = current_round_;
          update_current_round(current_round_ + 1);
        }
        break;
      }
    }
    return nullptr;
  }
  // insert_network_record :833-842 — errors are swallowed.  Returns whether it was accepted
  // (instrumentation; the reference returns nothing).
  bool insert_network_record(const Record& record, SimulatedContext& context) {
    if (counters) counters->inserts_tried[record.kind]++;
    const char* err = try_insert_network_record(record, context);
    if (!err && counters) counters->inserts_ok[record.kind]++;
    return err == nullptr;
  }

  // ---- RecordStore trait :544-843 ----
  Round current_round() const { return current_round_; }
  QcId highest_quorum_certificate_hash() const { return highest_quorum_certificate_hash_; }
  Round highest_quorum_certificate_round() const { return highest_quorum_certificate_round_; }
  Round highest_timeout_certificate_round() const { return highest_timeout_certificate_round_; }
  Round highest_committed_round() const { return highest_committed_round_; }
  std::vector<std::pair<Round, StateId>> committed_states_after(Round after_round) const {  // :557-574
    QcId cc = highest_commit_certificate_hash.value_or(initial_hash);
    BackIter it = back_iter(cc);
    it.next();
    it.next();
    std::vector<std::pair<Round, StateId>> commits;
    while (const QuorumCertificate* qc = it.next()) {
      if (qc->round <= after_round) break;
      commits.push_back({qc->round, qc->state});
    }
    std::reverse(commits.begin(), commits.end());
    return commits;
  }
  Round previous_round(BlockId block_hash) const {  // :588-598
    QcId h = block(block_hash)->previous_quorum_certificate_hash;
    if (h == initial_hash) return 0;
    return block(quorum_certificate(h)->certified_block_hash)->round;
  }
  Round second_previous_round(BlockId block_hash) const {  // :600-609
    QcId h = block(block_hash)->previous_quorum_certificate_hash;
    if (h == initial_hash) return 0;
    return previous_round(quorum_certificate(h)->certified_block_hash);
  }
  struct Proposed {
    BlockId hash;
    Round round;
    Author author;
  };
  std::optional<Proposed> proposed_block(const PacemakerState& pm) const;  // :611-634 (below)
  void create_timeout(Author author, Round round, SimulatedContext& context) {  // :636-649
    Timeout t{epoch_id, round, highest_quorum_certificate_round_, author};
    insert_network_record(Record::of(t), context);
  }
  bool has_timeout(Author author, Round round) const {  // :651-653
    return round == current_round_ && current_timeouts.count(author);
  }
  void propose_block(SimulatedContext& context, QcId previous_qc_hash, NodeTime time) {  // :655-674
    Command command = context.fetch();
    Block b{ids->next_block++, command, time, previous_qc_hash, current_round_, context.author()};
    insert_network_record(Record::of(b), context);
  }
  bool create_vote(SimulatedContext& context, BlockId certified_block_hash) {  // :676-700
    std::optional<StateId> committed_state = vote_committed_state(certified_block_hash);
    std::optional<StateId> st = compute_state(certified_block_hash, context);
    if (!st) return false;
    Vote v{epoch_id, block(certified_block_hash)->round, certified_block_hash, *st, committed_state, context.author()};
    insert_network_record(Record::of(v), context);
    return true;
  }
  bool check_for_new_quorum_certificate(SimulatedContext& context) {  // :702-738
    if (election != WON) return false;
    if (block(won_block)->author != context.author()) return false;
    std::optional<StateId> committed_state = vote_committed_state(won_block);
    std::vector<Author> authors;
    for (auto& kv : current_votes)
      if (kv.second.state == won_state) authors.push_back(kv.second.author);
    QuorumCertificate q{ids->next_qc++, epoch_id, current_round_, won_block, won_state, committed_state, authors, context.author()};
    election = CLOSED;
    insert_network_record(Record::of(q), context);
    return true;
  }
  const QuorumCertificate* highest_commit_certificate() const {  // :740-743
    if (!highest_commit_certificate_hash) return nullptr;
    return quorum_certificate(*highest_commit_certificate_hash);
  }
  const QuorumCertificate* highest_quorum_certificate() const {  // :745-747 (initial hash -> None)
    return quorum_certificate(highest_quorum_certificate_hash_);
  }
  std::vector<Timeout> timeouts() const {  // :749-756
    std::vector<Timeout> t;
    if (highest_timeout_certificate) t = *highest_timeout_certificate;
    for (auto& kv : current_timeouts) t.push_back(kv.second);
    return t;
  }
  const Vote* current_vote(Author a) const {  // :762-764
    auto it = current_votes.find(a);
    return it == current_votes.end() ? nullptr : &it->second;
  }
  std::set<Round> known_quorum_certificate_rounds() const {  // :766-799
    std::set<Round> result;
    for (QcId start : {highest_quorum_certificate_hash_, highest_commit_certificate_hash.value_or(initial_hash)}) {
      BackIter it = back_iter(start);
      size_t i = 0;
      while (const QuorumCertificate* qc = it.next()) {
        if (is_power2_minus1(i)) result.insert(qc->round);
        i++;
      }
    }
    return result;
  }
  std::vector<Record> unknown_records(const std::set<Round>& known) const {  // :801-831
    auto chain = [&](QcId start) {
      std::vector<const QuorumCertificate*> c;
      BackIter it = back_iter(start);
      while (const QuorumCertificate* qc = it.next()) {
        if (known.count(qc->round)) break;
        c.push_back(qc);
      }
      return c;
    };
    auto c1 = chain(highest_quorum_certificate_hash_);
    auto c2 = chain(highest_commit_certificate_hash.value_or(initial_hash));
    // record_store.rs:822: merge_sort(chain1, chain2, |qc1, qc2| qc2.round.cmp(&qc1.round)) — descending rounds, equal QCs once
    using QcPtr = const QuorumCertificate*;
    std::vector<QcPtr> qcs = merge_sort(
        c1, c2, [](QcPtr a, QcPtr b) { return b->round < a->round ? -1 : (b->round == a->round ? 0 : 1); },
        [](QcPtr a, QcPtr b) { return a->id == b->id; });
    std::vector<Record> result;
    for (size_t n = qcs.size(); n-- > 0;) {
      result.push_back(Record::of(*block(qcs[n]->certified_block_hash)));
      result.push_back(Record::of(*qcs[n]));
    }
    for (auto& t : timeouts()) result.push_back(Record::of(t));
    if (current_proposed_block) result.push_back(Record::of(*block(*current_proposed_block)));
    return result;
  }
};

// ---------------------------------------------------------------------------------------------
// Pacemaker (pacemaker.rs:17-221)
// ---------------------------------------------------------------------------------------------
struct PacemakerUpdateActions {
  std::optional<QcId> should_propose_block;
  std::optional<Round> should_create_timeout;
  std::vector<Author> should_send;
  bool should_broadcast = false;
  bool should_query_all = false;
  NodeTime next_scheduled_update = NODE_TIME_NEVER;
};
struct PacemakerState {
  EpochId active_epoch = 0;
  Round active_round_ = 0;
  std::optional<Author> active_leader_;
  NodeTime active_round_start_time = 0;
  Duration active_round_duration = 0;
  Duration delta = 0;
  double gamma = 0, lambda = 0;
  PacemakerState() {}
  PacemakerState(EpochId e, NodeTime t, Duration d, double g, double l)
      : active_epoch(e), active_round_start_time(t), delta(d), gamma(g), lambda(l) {}
  Round active_round() const { return active_round_; }
  std::optional<Author> active_leader() const { return active_leader_; }
  Duration duration(const RecordStoreState& rs, Round round) const {  // :111-124
    Round hccr = rs.highest_committed_round() > 0 ? rs.highest_committed_round() + 2 : 0;
    if (!(round > hccr)) throw OracleError("Active round is higher than any QC round.");
    uint64_t n = round - hccr;
    return (Duration)((double)delta * std::pow((double)n, gamma));
  }
  PacemakerUpdateActions update_pacemaker(Author local_author, EpochId epoch_id, const RecordStoreState& rs,
                                          NodeTime latest_query_all_time, NodeTime clock) {  // :142-207
    PacemakerUpdateActions actions;
    Round active_round = std::max(rs.highest_quorum_certificate_round(), rs.highest_timeout_certificate_round()) + 1;
    if (epoch_id > active_epoch || (epoch_id == active_epoch && active_round > active_round_)) {
      active_epoch = epoch_id;
      active_round_ = active_round;
      active_round_start_time = clock;
      active_leader_ = rs.leader(active_round);
      active_round_duration = duration(rs, active_round);
      if (active_leader_ != std::optional<Author>(local_author)) actions.should_send = {*active_leader_};
    }
    if (active_leader_ == std::optional<Author>(local_author) && !rs.proposed_block(*this)) {
      actions.should_propose_block = rs.highest_quorum_certificate_hash();
      actions.should_broadcast = true;
      actions.next_scheduled_update = clock;
    }
    if (!rs.has_timeout(local_author, active_round)) {
      NodeTime timeout_deadline = active_round_start_time + active_round_duration;
      if (clock >= timeout_deadline) {
        actions.should_create_timeout = active_round;
        actions.should_broadcast = true;
      } else {
        actions.next_scheduled_update = std::min(actions.next_scheduled_update, timeout_deadline);
      }
    } else {
      Duration period = (Duration)(lambda * (double)active_round_duration);
      NodeTime query_all_deadline = latest_query_all_time + period;
      if (clock >= query_all_deadline) {
        actions.should_query_all = true;
        query_all_deadline = clock + period;
      }
      actions.next_scheduled_update = std::min(actions.next_scheduled_update, query_all_deadline);
    }
    return actions;
  }
};

inline std::optional<RecordStoreState::Proposed> RecordStoreState::proposed_block(const PacemakerState& pm) const {
  if (epoch_id != pm.active_epoch || current_round_ != pm.active_round()) return std::nullopt;
  if (!pm.active_leader()) return std::nullopt;
  if (!current_proposed_block) return std::nullopt;
  const Block* b = block(*current_proposed_block);
  if (b->round != current_round_ || b->author != *pm.active_leader()) throw OracleError("proposed_block assertion");
  return Proposed{*current_proposed_block, b->round, b->author};
}

// ---------------------------------------------------------------------------------------------
// NodeState + CommitTracker (node.rs:28-407), data-sync messages and handlers (data_sync.rs)
// ---------------------------------------------------------------------------------------------
struct NodeConfig {
  Duration target_commit_interval = 100000;
  Duration delta = 20;
  double gamma = 2.0;
  double lambda = 0.5;
};
struct NodeUpdateActions {  // interfaces.rs:12-21
  NodeTime next_scheduled_update = NODE_TIME_NEVER;
  std::vector<Author> should_send;
  bool should_broadcast = false;
  bool should_query_all = false;
};
struct CommitTracker {
  EpochId epoch_id = 0;
  Round highest_committed_round = 0;
  NodeTime latest_commit_time = 0;
  Duration target_commit_interval = 0;
  struct Actions {
    NodeTime next_scheduled_update = NODE_TIME_NEVER;
    bool should_query_all = false;
  };
  Actions update_tracker(NodeTime latest_query_all_time, NodeTime clock, EpochId current_epoch_id,
                         const RecordStoreState& rs) {  // node.rs:364-396
    Actions actions;
    if (current_epoch_id > epoch_id) {
      epoch_id = current_epoch_id;
      highest_committed_round = rs.highest_committed_round();
      latest_commit_time = clock;
    } else {
      Round hcr = rs.highest_committed_round();
      if (hcr > highest_committed_round) {
        highest_committed_round = hcr;
        latest_commit_time = clock;
      }
    }
    NodeTime deadline = std::max(latest_commit_time, latest_query_all_time) + target_commit_interval;
    if (clock >= deadline) {
      actions.should_query_all = true;
      deadline = clock + target_commit_interval;
    }
    actions.next_scheduled_update = deadline;
    return actions;
  }
};

struct DataSyncNotification {  // data_sync.rs:16-39
  EpochId current_epoch = 0;
  std::optional<QuorumCertificate> highest_commit_certificate;
  std::optional<QuorumCertificate> highest_quorum_certificate;
  std::vector<Timeout> timeouts;
  std::optional<Vote> current_vote;
  std::optional<Block> proposed_block;
};
struct DataSyncRequest {  // :41-47
  EpochId current_epoch = 0;
  std::set<Round> known_quorum_certificates;
};
struct DataSyncResponse {  // :49-59
  EpochId current_epoch = 0;
  std::vector<std::pair<EpochId, std::vector<Record>>> records;
};

struct NodeState {
  RecordStoreState record_store;
  PacemakerState pacemaker;
  EpochId epoch_id = 0;
  Round latest_voted_round = 0;
  Round locked_round = 0;
  NodeTime latest_query_all_time = 0;
  CommitTracker tracker;
  std::map<EpochId, RecordStoreState> past_record_stores;
  IdSource* ids = nullptr;
  Counters* counters = nullptr;
  bool timeout_and_propose_same_update = false;  // App. C.1b watch

  // make_initial_state node.rs:87-114
  static NodeState make_initial_state(const SimulatedContext& context, const NodeConfig& config, NodeTime node_time,
                                      IdSource* ids, Counters* counters) {
    NodeState n;
    StateId initial_state = context.last_committed_state();
    EpochId epoch_id = context.read_epoch_id(initial_state);
    n.tracker.epoch_id = epoch_id;
    n.tracker.highest_committed_round = 0;
    n.tracker.latest_commit_time = node_time;
    n.tracker.target_commit_interval = config.target_commit_interval;
    n.record_store = RecordStoreState(QC_INITIAL, initial_state, epoch_id, context.configuration(initial_state), ids, counters);
    n.pacemaker = PacemakerState(epoch_id, node_time, config.delta, config.gamma, config.lambda);
    n.epoch_id = epoch_id;
    n.latest_query_all_time = node_time;
    n.ids = ids;
    n.counters = counters;
    return n;
  }
  const RecordStoreState* record_store_at(EpochId e) const {
    if (e == epoch_id) return &record_store;
    auto it = past_record_stores.find(e);
    return it == past_record_stores.end() ? nullptr : &it->second;
  }
  bool insert_network_record(EpochId e, const Record& r, SimulatedContext& ctx) {  // node.rs:150-167
    if (e == epoch_id) return record_store.insert_network_record(r, ctx);
    return false;
  }
  Round active_round() const { return pacemaker.active_round(); }

  NodeUpdateActions process_pacemaker_actions(const PacemakerUpdateActions& pa, NodeTime clock, SimulatedContext& ctx) {  // :179-202
    NodeUpdateActions actions;
    actions.next_scheduled_update = pa.next_scheduled_update;
    actions.should_broadcast = pa.should_broadcast;
    actions.should_query_all = pa.should_query_all;
    actions.should_send = pa.should_send;
    if (pa.should_create_timeout && pa.should_propose_block) timeout_and_propose_same_update = true;
    if (pa.should_create_timeout) {
      record_store.create_timeout(ctx.author(), *pa.should_create_timeout, ctx);
      latest_voted_round = std::max(latest_voted_round, *pa.should_create_timeout);
    }
    if (pa.should_propose_block) record_store.propose_block(ctx, *pa.should_propose_block, clock);
    return actions;
  }
  void process_commits(SimulatedContext& ctx) {  // :313-350
    for (auto& rs : record_store.committed_states_after(tracker.highest_committed_round)) {
      ctx.commit(rs.second);
      EpochId new_epoch_id = ctx.read_epoch_id(rs.second);
      if (new_epoch_id > epoch_id) {
        RecordStoreState fresh(QC_INITIAL, rs.second, new_epoch_id, ctx.configuration(rs.second), ids, counters);
        past_record_stores.emplace(epoch_id, std::move(record_store));
        record_store = std::move(fresh);
        epoch_id = new_epoch_id;
        latest_voted_round = 0;
        locked_round = 0;
        break;
      }
    }
  }
  NodeUpdateActions update_node(SimulatedContext& ctx, NodeTime clock) {  // :240-304
    PacemakerUpdateActions pa = pacemaker.update_pacemaker(ctx.author(), epoch_id, record_store, latest_query_all_time, clock);
    NodeUpdateActions actions = process_pacemaker_actions(pa, clock, ctx);
    if (auto pb = record_store.proposed_block(pacemaker)) {
      if (pb->round > latest_voted_round && record_store.previous_round(pb->hash) >= locked_round) {
        latest_voted_round = pb->round;
        locked_round = std::max(locked_round, record_store.second_previous_round(pb->hash));
        if (record_store.create_vote(ctx, pb->hash)) actions.should_send = {pb->author};
      }
    }
    if (record_store.check_for_new_quorum_certificate(ctx)) {
      actions.should_broadcast = true;
      actions.next_scheduled_update = clock;
    }
    process_commits(ctx);
    CommitTracker::Actions ta = tracker.update_tracker(latest_query_all_time, clock, epoch_id, record_store);
    actions.should_query_all = actions.should_query_all || ta.should_query_all;
    actions.next_scheduled_update = std::min(actions.next_scheduled_update, ta.next_scheduled_update);
    if (actions.should_query_all) latest_query_all_time = clock;
    return actions;
  }

  // ---- DataSyncNode (data_sync.rs:74-241) ----
  DataSyncRequest create_request() const {  // :62-72,179-181
    return DataSyncRequest{epoch_id, record_store.known_quorum_certificate_rounds()};
  }
  DataSyncNotification create_notification(const SimulatedContext& ctx) const {  // :82-111
    DataSyncNotification n;
    n.current_epoch = epoch_id;
    if (const QuorumCertificate* q = record_store.highest_commit_certificate()) n.highest_commit_certificate = *q;
    else if (epoch_id != 0) {
      // EpochId::previous() returns the SAME id (base_types.rs:31-37, quirk B.9.iii)
      const RecordStoreState* s = record_store_at(epoch_id);
      if (const QuorumCertificate* q2 = s->highest_commit_certificate()) n.highest_commit_certificate = *q2;
    }
    if (const QuorumCertificate* q = record_store.highest_quorum_certificate()) n.highest_quorum_certificate = *q;
    n.timeouts = record_store.timeouts();
    if (const Vote* v = record_store.current_vote(ctx.author())) n.current_vote = *v;
    if (auto pb = record_store.proposed_block(pacemaker)) {
      if (pb->author == ctx.author()) n.proposed_block = *record_store.block(pb->hash);
    }
    return n;
  }
  std::optional<DataSyncRequest> handle_notification(SimulatedContext& ctx, const DataSyncNotification& n) {  // :113-177
    bool should_sync = false;
    should_sync |= n.current_epoch > epoch_id;
    if (n.highest_commit_certificate) {
      const QuorumCertificate& q = *n.highest_commit_certificate;
      insert_network_record(q.epoch_id, Record::of(q), ctx);
      should_sync |= (q.epoch_id > epoch_id) || (q.epoch_id == epoch_id && q.round > record_store.highest_committed_round() + 2);
    }
    if (n.highest_quorum_certificate) {
      const QuorumCertificate& q = *n.highest_quorum_certificate;
      insert_network_record(q.epoch_id, Record::of(q), ctx);
      should_sync |= (q.epoch_id > epoch_id) || (q.epoch_id == epoch_id && q.round > record_store.highest_quorum_certificate_round());
    }
    if (n.proposed_block) insert_network_record(n.current_epoch, Record::of(*n.proposed_block), ctx);
    for (auto& t : n.timeouts) insert_network_record(n.current_epoch, Record::of(t), ctx);
    if (n.current_vote) insert_network_record(n.current_epoch, Record::of(*n.current_vote), ctx);
    if (should_sync) return create_request();
    return std::nullopt;
  }
  DataSyncResponse handle_request(const DataSyncRequest& req) const {  // :183-207
    DataSyncResponse resp;
    if (const RecordStoreState* s = record_store_at(req.current_epoch))
      resp.records.push_back({req.current_epoch, s->unknown_records(req.known_quorum_certificates)});
    for (EpochId i = req.current_epoch + 1; i < epoch_id + 1; i++) {
      const RecordStoreState* s = record_store_at(i);
      if (!s) throw OracleError("All record stores up to the current epoch should exist.");
      resp.records.push_back({i, s->unknown_records({})});
    }
    resp.current_epoch = epoch_id;
    return resp;
  }
  void handle_response(SimulatedContext& ctx, const DataSyncResponse& resp, NodeTime clock) {  // :209-240
    size_t num_records = resp.records.size();
    for (size_t i = 0; i < num_records; i++) {
      EpochId e = resp.records[i].first;
      if (e < epoch_id) continue;
      if (e > epoch_id) break;
      for (auto& r : resp.records[i].second) {
        bool ok = insert_network_record(e, r, ctx);
        if (ok && counters) counters->response_records_accepted++;
      }
      if (i == num_records - 1) break;
      process_commits(ctx);
      tracker.update_tracker(latest_query_all_time, clock, epoch_id, record_store);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// Simulator (simulator.rs:26-475)
// ---------------------------------------------------------------------------------------------
struct SimConfig {
  uint32_t num_nodes = 3;
  int64_t max_clock = 1000;
  RandomDelay delay = RandomDelay::lognormal(10.0, 4.0);
  NodeConfig node;
  uint64_t commands_per_epoch = 30000;
  // ---- EXTENSIONS (not in the reference; SURVEY Appendix D).  Defaults = reference behaviour. ----
  std::vector<uint64_t> voting_rights;  // empty = all 1 (simulated_context.rs:209-216)
  std::vector<uint8_t> silent;          // empty = none; silent[i] != 0: node i never handles an event
  // partition plan: windows [t0, t1) during which nodes with side bit 1 cannot exchange network
  // events with nodes with side bit 0 (decided at SEND time, after the delay is drawn).
  struct PartitionWindow {
    int64_t t0, t1;
    uint64_t side_mask;
  };
  std::vector<PartitionWindow> partitions;
  // LBFT_FLAG_TRUE_DATA_SYNC (NON-PARITY variant, SURVEY 8(f).4): handle_request runs on the node the request was sent
  // to instead of on the requester (simulator.rs:446 uses `receiver`)
  bool true_data_sync = false;
};

enum EventKind { EV_NOTIFY = 0, EV_REQUEST = 1, EV_RESPONSE = 2, EV_TIMER = 3 };

struct SimCounters {
  uint64_t processed[4] = {0, 0, 0, 0};  // popped (and not beyond max_clock), by kind
  uint64_t timers_cancelled = 0;
  uint64_t scheduled[4] = {0, 0, 0, 0};
  uint64_t max_queue = 0;
  uint64_t dropped_partition = 0;
  uint64_t scheduled_notify = 0;  // Notify events handed a creation stamp (incl. partition-dropped)
};

struct Simulator {
  struct Event {
    int64_t time;
    uint64_t stamp;
    int kind;
    Author receiver, sender;
    int payload;  // index into the payload pools (notification / request / response), -1 none
  };
  struct Cmp {  // simulator.rs:149-161: max-heap on (other.time, self.kind, other.stamp)
    bool operator()(const Event& a, const Event& b) const {
      // returns true if a is "less" (lower priority) than b
      if (a.time != b.time) return a.time > b.time;
      if (a.kind != b.kind) return a.kind < b.kind;
      return a.stamp > b.stamp;
    }
  };
  struct SimulatedNode {
    int64_t startup_time;
    int64_t ignore_scheduled_updates_until;
    NodeState node;
    SimulatedContext context;
  };

  SimConfig cfg;
  int64_t clock = 0;
  std::priority_queue<Event, std::vector<Event>, Cmp> pending_events;
  std::vector<SimulatedNode> nodes;
  uint64_t event_count = 0;
  Xoshiro256StarStar rng;
  LedgerIntern ledger;
  IdSource ids;
  Counters rec_counters;
  SimCounters counters;
  std::vector<DataSyncNotification> notif_pool;
  std::vector<DataSyncRequest> req_pool;
  std::vector<DataSyncResponse> resp_pool;
  bool payload_free = true;  // drop pool entries once delivered (keeps memory flat)

  Simulator(uint64_t seed, const SimConfig& c) : cfg(c) {  // Simulator::new :200-250
    rng = Xoshiro256StarStar::seed_from_u64(seed);
    nodes.resize(cfg.num_nodes);
    for (uint32_t index = 0; index < cfg.num_nodes; index++) {
      SimulatedNode& sn = nodes[index];
      sn.context = SimulatedContext((Author)index, cfg.num_nodes, cfg.commands_per_epoch, &ledger);
      if (!cfg.voting_rights.empty()) sn.context.voting_rights_override = &cfg.voting_rights;
      sn.node = NodeState::make_initial_state(sn.context, cfg.node, 0, &ids, &rec_counters);
      sn.startup_time = 0 + cfg.delay.sample(rng) + 1;
      push_event(sn.startup_time, EV_TIMER, (Author)index, (Author)index, -1);
      sn.ignore_scheduled_updates_until = sn.startup_time - 1;
    }
  }
  // the context pointers into `ledger` / the node pointers into ids/counters make this non-movable
  Simulator(const Simulator&) = delete;
  Simulator& operator=(const Simulator&) = delete;

  void push_event(int64_t t, int kind, Author receiver, Author sender, int payload) {  // schedule_event :252-264
    pending_events.push(Event{t, event_count, kind, receiver, sender, payload});
    event_count++;
    counters.scheduled[kind]++;
    counters.max_queue = std::max<uint64_t>(counters.max_queue, pending_events.size());
  }
  bool partitioned(Author a, Author b) const {
    for (auto& w : cfg.partitions)
      if (clock >= w.t0 && clock < w.t1 && (((w.side_mask >> a) ^ (w.side_mask >> b)) & 1)) return true;
    return false;
  }
  void schedule_network_event(int kind, Author receiver, Author sender, int payload) {  // :266-269
    int64_t t = clock + cfg.delay.sample(rng);
    // EXTENSION D.3: a partitioned message still draws its delay and consumes a creation stamp.
    // The message travels from `sender` to `receiver` for notifications/responses-to-requests alike;
    // for requests (receiver = requester) the two endpoints are the same pair.
    if (!cfg.partitions.empty() && partitioned(receiver, sender)) {
      event_count++;
      counters.dropped_partition++;
      return;
    }
    push_event(t, kind, receiver, sender, payload);
  }
  bool is_silent(Author a) const { return !cfg.silent.empty() && cfg.silent[a]; }

  void process_node_actions(int64_t clk, Author author, const NodeUpdateActions& actions) {  // :296-378
    SimulatedNode& node = nodes[author];
    // save_node (:307-309) has no observable effect in the simulator and is omitted.
    int64_t from_node =
        actions.next_scheduled_update == NODE_TIME_NEVER ? INT64_MAX : from_node_time(actions.next_scheduled_update, node.startup_time);
    int64_t new_scheduled_time = std::max(from_node, clk + 1);
    node.ignore_scheduled_updates_until = new_scheduled_time - 1;
    push_event(new_scheduled_time, EV_TIMER, author, author, -1);
    std::vector<Author> receivers;
    if (actions.should_broadcast) {
      for (uint32_t i = 0; i < cfg.num_nodes; i++)
        if ((Author)i != author) receivers.push_back((Author)i);
    } else {
      for (Author r : actions.should_send)
        if (r != author) receivers.push_back(r);
    }
    shuffle(receivers, rng);
    if (!receivers.empty()) {  // create_notification has no side effect; only materialise when sent
      int p = (int)notif_pool.size();
      notif_pool.push_back(node.node.create_notification(node.context));
      counters.scheduled_notify += receivers.size();
      for (Author r : receivers) schedule_network_event(EV_NOTIFY, r, author, p);
    }
    std::vector<Author> senders;
    if (actions.should_query_all) {
      for (uint32_t i = 0; i < cfg.num_nodes; i++)
        if ((Author)i != author) senders.push_back((Author)i);
    }
    shuffle(senders, rng);
    if (!senders.empty()) {
      int p = (int)req_pool.size();
      req_pool.push_back(node.node.create_request());
      for (Author s : senders) schedule_network_event(EV_REQUEST, author, s, p);
    }
  }

  // DataWriter state (data_writer.rs:10-17), kept when loop_until is given a csv path (simulator.rs:381).
  // PARITY UNPINNED for this output: the reference has no test or golden for DataWriter; the event
  // sequence it samples is pinned by the commit-log goldens.
  bool record_round_switches = false;
  std::vector<uint64_t> max_round_per_node;                                     // :13
  std::vector<std::vector<std::pair<uint64_t, int64_t>>> nodes_round_switch;   // :14
  // update_round_number data_writer.rs:34-50 — every node is looked at, at every pop.
  void sample_round_numbers(int64_t scheduled_time) {
    if (max_round_per_node.size() != nodes.size()) {
      max_round_per_node.assign(nodes.size(), 0);
      nodes_round_switch.assign(nodes.size(), {});
    }
    for (size_t n = 0; n < nodes.size(); n++) {
      uint64_t r = nodes[n].node.active_round();
      if (r > max_round_per_node[n]) {
        max_round_per_node[n] = r;
        nodes_round_switch[n].push_back({r, scheduled_time});
      }
    }
  }

  // loop_until :380-475
  void loop_until(int64_t max_clock) {
    while (!pending_events.empty()) {
      Event ev = pending_events.top();
      pending_events.pop();
      if (ev.time > max_clock) break;
      // :393-394 — after the max_clock test, with the event's own scheduled_time (the max() with the
      // simulator clock comes later, :399), and before the timer-cancellation test (:406).
      if (record_round_switches) sample_round_numbers(ev.time);
      int64_t clk = std::max(ev.time, clock);
      clock = clk;
      counters.processed[ev.kind]++;
      // EXTENSION D.2: a silent node never handles an event, and never answers a request.
      if (is_silent(ev.receiver) || (ev.kind == EV_REQUEST && is_silent(ev.sender))) continue;
      switch (ev.kind) {
        case EV_TIMER: {
          SimulatedNode& node = nodes[ev.receiver];
          if (clk <= node.ignore_scheduled_updates_until) {
            counters.timers_cancelled++;
            continue;
          }
          NodeUpdateActions actions = node.node.update_node(node.context, to_node_time(clk, node.startup_time));
          process_node_actions(clk, ev.receiver, actions);
          break;
        }
        case EV_NOTIFY: {
          SimulatedNode& node = nodes[ev.receiver];
          std::optional<DataSyncRequest> result = node.node.handle_notification(node.context, notif_pool[ev.payload]);
          NodeUpdateActions actions = node.node.update_node(node.context, to_node_time(clk, node.startup_time));
          if (result) {
            int p = (int)req_pool.size();
            req_pool.push_back(*result);
            schedule_network_event(EV_REQUEST, ev.receiver, ev.sender, p);
          }
          process_node_actions(clk, ev.receiver, actions);
          break;
        }
        case EV_REQUEST: {
          // QUIRK (simulator.rs:446): the request is answered by `receiver` itself — unless the opt-in variant asks for
          // the node it was sent to.
          SimulatedNode& node = nodes[cfg.true_data_sync ? ev.sender : ev.receiver];
          int p = (int)resp_pool.size();
          resp_pool.push_back(node.node.handle_request(req_pool[ev.payload]));
          schedule_network_event(EV_RESPONSE, ev.receiver, ev.sender, p);
          break;
        }
        case EV_RESPONSE: {
          SimulatedNode& node = nodes[ev.receiver];
          node.node.handle_response(node.context, resp_pool[ev.payload], to_node_time(clk, node.startup_time));
          if (payload_free) resp_pool[ev.payload] = DataSyncResponse();
          NodeUpdateActions actions = node.node.update_node(node.context, to_node_time(clk, node.startup_time));
          process_node_actions(clk, ev.receiver, actions);
          break;
        }
      }
    }
  }
  uint64_t max_active_round() const {
    uint64_t r = 0;
    for (auto& n : nodes) r = std::max<uint64_t>(r, n.node.active_round());
    return r;
  }
};

}  // namespace lbft_oracle
