// host_setup.hpp — host-side preparation of a batched run: configuration validation, capacity
// selection and the tables whose arithmetic must come from the host libm so that it matches what
// the reference's Rust computes through the same libm (ln/sqrt/exp/pow), namely
//   * RandomDelay::new mu/sigma ............................. bft-lib/src/simulator.rs:99-106
//   * the rand_distr 0.4.0 ziggurat layer tables ............ (crate literals, "%.18f"-rounded)
//   * PacemakerState::leader(round) for every round ......... librabft-v2/src/pacemaker.rs:100-109
//                                                             + bft-lib/src/configuration.rs:65-75
//   * PacemakerState::duration / query-all period per n ..... librabft-v2/src/pacemaker.rs:111-124,196
// Pure C++ (no CUDA) so the CPU debugging harness in tests/hostcore can share it.  Written
// independently of oracle/ (the oracle is the checker, not a dependency).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/lbft.h"
#include "sim_params.h"

namespace lbft {

inline uint64_t host_rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }

// SipHash-1-3 (zero key) of one little-endian u64: `round.hash(&mut DefaultHasher::new())`.
inline uint64_t siphash13_u64(uint64_t mword) {
  uint64_t v0 = 0x736f6d6570736575ULL, v1 = 0x646f72616e646f6dULL, v2 = 0x6c7967656e657261ULL, v3 = 0x7465646279746573ULL;
  auto rnd = [&]() {
    v0 += v1; v1 = host_rotl(v1, 13); v1 ^= v0; v0 = host_rotl(v0, 32);
    v2 += v3; v3 = host_rotl(v3, 16); v3 ^= v2;
    v0 += v3; v3 = host_rotl(v3, 21); v3 ^= v0;
    v2 += v1; v1 = host_rotl(v1, 17); v1 ^= v2; v2 = host_rotl(v2, 32);
  };
  v3 ^= mword; rnd(); v0 ^= mword;
  uint64_t b = 8ULL << 56;
  v3 ^= b; rnd(); v0 ^= b;
  v2 ^= 0xff;
  rnd(); rnd(); rnd();
  return v0 ^ v1 ^ v2 ^ v3;
}

// EpochConfiguration::pick_author (configuration.rs:65-75): Xoshiro256** seeded through SplitMix64,
// one rand-0.8 `gen_range(0..total_votes)` (widening-multiply rejection), weighted linear scan.
inline uint32_t pick_author(const std::vector<uint32_t>& weights, uint64_t total, uint64_t seed) {
  uint64_t s[4], x = seed;
  for (int i = 0; i < 4; i++) {
    x += 0x9e3779b97f4a7c15ULL;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    s[i] = z ^ (z >> 31);
  }
  uint64_t zone = (total << __builtin_clzll(total)) - 1, target;
  for (;;) {
    uint64_t v = host_rotl(s[1] * 5, 7) * 9, t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = host_rotl(s[3], 45);
    unsigned __int128 mm = (unsigned __int128)v * total;
    if ((uint64_t)mm <= zone) { target = (uint64_t)(mm >> 64); break; }
  }
  for (uint32_t a = 0; a < weights.size(); a++) {
    if (weights[a] > target) return a;
    target -= weights[a];
  }
  return 0;  // unreachable
}

inline uint32_t pow2_ceil(uint32_t v) {
  uint32_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

constexpr uint32_t kThrSmem = 256;  // doubles: delay thresholds held in shared memory when they fit

// The kernel instantiation a handle launches (kernels.cuh), decided once by HostSetup::build.
struct KernelSel {
  bool wide;   // lbft_wide_kernel instead of lbft_event_loop_kernel
  bool smem;   // wide kernel: instance state in shared memory
  int group;   // wide kernel: lanes per instance (8 / 32)
  bool epochs; // Layout::epochs > 1: the instantiation with the epoch machinery (plain kernels only)
  bool tds;    // LBFT_FLAG_TRUE_DATA_SYNC (plain single-epoch thread kernels only)
  int tile;    // instances per warp tile, the lane interleaving of the state (thread kernel: 32, or 8 / 16 = sparse tiles on
               // plain calendar-queue kernels; wide kernel: 1)
  int nmax;    // 16 / 32 / 64: width of the author masks
  int qmode;   // Layout::queue_scan
  int fixed;   // FX_* (sim_params.h): the instantiation with that compile-time layout; FX_NONE = generic
  bool rec, res;
  bool sweep;  // a sweep handle: lbft_sweep_event_loop_kernel / lbft_sweep_wide_kernel (per-instance parameter sets)
  bool ct;     // LBFT_FLAG_COMMIT_TIMES: the commit-times twin (lbft_ct_*_kernel) of the kernel the other fields name
};

// The kernel's name, spelled like the symbol cuobjdump shows (lbft_kernel_info).
inline std::string kernel_name(const KernelSel& k) {
  char buf[96];
  if (k.ct && k.sweep && k.wide)
    snprintf(buf, sizeof buf, "lbft_ct_sweep_wide_kernel<%d,%d,%s,%d>", k.nmax, k.qmode, k.smem ? "true" : "false", k.group);
  else if (k.ct && k.sweep)
    snprintf(buf, sizeof buf, "lbft_ct_sweep_event_loop_kernel<%d,%d,%d>", k.nmax, k.qmode, k.tile);
  else if (k.ct && k.wide)
    snprintf(buf, sizeof buf, "lbft_ct_wide_kernel<%d,%d,%s,%d,%d>", k.nmax, k.qmode, k.smem ? "true" : "false", k.group, k.fixed);
  else if (k.ct)
    snprintf(buf, sizeof buf, "lbft_ct_event_loop_kernel<%d,%d,%d,%d>", k.nmax, k.qmode, k.fixed, k.tile);
  else if (k.sweep && k.wide)
    snprintf(buf, sizeof buf, "lbft_sweep_wide_kernel<%d,%d,%s,%d>", k.nmax, k.qmode, k.smem ? "true" : "false", k.group);
  else if (k.sweep)
    snprintf(buf, sizeof buf, "lbft_sweep_event_loop_kernel<%d,%d,%d>", k.nmax, k.qmode, k.tile);
  else if (k.wide)
    snprintf(buf, sizeof buf, "lbft_wide_kernel<%d,%d,%s,%d,%s,%d>", k.nmax, k.qmode, k.smem ? "true" : "false", k.group, k.epochs ? "true" : "false", k.fixed);
  else
    snprintf(buf, sizeof buf, "lbft_event_loop_kernel<%d,%d,%d,%s,%s,%s,%s,%d>", k.nmax, k.qmode, k.fixed, k.rec ? "true" : "false",
             k.res ? "true" : "false", k.epochs ? "true" : "false", k.tds ? "true" : "false", k.tile);
  return buf;
}
// Whether two selections name the same kernel (the fields kernel_name prints).
constexpr bool same_kernel(const KernelSel& a, const KernelSel& b) {
  return a.ct == b.ct && a.sweep == b.sweep && a.wide == b.wide && a.nmax == b.nmax && a.qmode == b.qmode && a.epochs == b.epochs && a.fixed == b.fixed &&
         (a.wide ? a.smem == b.smem && a.group == b.group
                 : a.rec == b.rec && a.res == b.res && a.tds == b.tds && a.tile == b.tile);
}

// The compile-time layout (sim_params.h fixed_layout) a configuration matches: its layout is bit-identical to the constant
// (which also pins the queue mode and a single-epoch, non-data-sync handle), it neither records nor resumes, and the delay
// model is the reference's (LogNormal served by the threshold table; FX_DEFAULT4 / FX_PART7 also need the table in shared
// memory and no silent nodes).  The kernel family, tile and lane-group conditions are the product's: HostSetup::build.
inline int fixed_shape_of(const Params& P) {
  constexpr Layout kDefault4 = fixed_layout(FX_DEFAULT4), kPart7 = fixed_layout(FX_PART7), kCommittee64 = fixed_layout(FX_COMMITTEE64);
  const bool table_delay = P.delay_kind == LBFT_DELAY_LOGNORMAL && !P.delay_const && P.delay_kmax != 0;
  const bool plain_model = table_delay && P.delay_kmax + 2 <= kThrSmem && P.silent_mask == 0;
  if (P.record_rs || P.resumable) return FX_NONE;
  if (plain_model && memcmp(&P.L, &kDefault4, sizeof(Layout)) == 0) return FX_DEFAULT4;
  if (plain_model && memcmp(&P.L, &kPart7, sizeof(Layout)) == 0) return FX_PART7;
  if (table_delay && memcmp(&P.L, &kCommittee64, sizeof(Layout)) == 0) return FX_COMMITTEE64;
  return FX_NONE;
}

// The delay model's mean: what the stamp-width and queue-mode tests are sized by.
inline double mean_delay(const lbft_config& c) {
  return c.delay_kind == LBFT_DELAY_UNIFORM ? 0.5 * (double)(c.delay_lo + c.delay_hi) : c.delay_mean;
}

// Round capacity per epoch: round_cap, or enough for the horizon, in whole bitset words.
inline uint32_t round_cap_of(const lbft_config& c) {
  uint32_t rcap = c.round_cap ? c.round_cap : (uint32_t)(c.max_clock / 12 + 40);
  rcap = (rcap + 31) / 32 * 32;
  return rcap < 32 ? 32 : rcap;
}

// Epochs (node.rs:329-348): a node commits at most one command per round, so commands_per_epoch >= round_cap can never be
// reached and the layout stays single-epoch (every BASELINE configuration).  Otherwise the per-round tables get `epochs` spans
// of round_cap rounds each (global round id = epoch * rspan + round).
inline uint32_t epochs_of(const lbft_config& c, uint32_t rcap) {
  if (c.commands_per_epoch >= rcap) return 1;
  uint32_t epochs = (uint32_t)(rcap / c.commands_per_epoch) + 2;
  if (epochs > MAX_EPOCHS) epochs = MAX_EPOCHS;
  while (epochs > 2 && (uint64_t)epochs * rcap > 32768) epochs--;
  return epochs;
}

// The delay model of a configuration (simulator.rs:101-102) into the fields a sweep keeps per set; the error text if it is
// not valid.
inline const char* delay_model(const lbft_config& c, SweepSet& s) {
  s.delay_kind = c.delay_kind;
  if (c.delay_kind == LBFT_DELAY_LOGNORMAL) {
    if (!(c.delay_mean > 0.0) || !(c.delay_variance >= 0.0)) return "LogNormal delay needs mean > 0 and variance >= 0";
    s.mu = std::log(c.delay_mean / std::sqrt(1.0 + c.delay_variance / (c.delay_mean * c.delay_mean)));
    s.sigma = std::sqrt(std::log(1.0 + c.delay_variance / (c.delay_mean * c.delay_mean)));
    s.delay_const = s.sigma == 0.0;
    s.delay_const_value = s.delay_const ? (int64_t)std::exp(s.mu) : 0;
    if (s.delay_const && (s.delay_const_value < 0 || s.delay_const_value > (1 << 29))) return "constant delay out of range";
  } else if (c.delay_kind == LBFT_DELAY_UNIFORM) {
    if (c.delay_lo < 0 || c.delay_hi < c.delay_lo || c.delay_hi > (1 << 29)) return "uniform delay needs 0 <= lo <= hi < 2^29";
    s.uni_lo = (uint64_t)c.delay_lo;
    s.uni_span = (uint64_t)(c.delay_hi - c.delay_lo + 1);
  } else return "unknown delay_kind";
  return nullptr;
}

// Why `c` cannot make a handle (the first failing check), or null.
inline const char* config_error(const lbft_config& c) {
  if (c.struct_size != sizeof(lbft_config)) return "lbft_config.struct_size does not match this library (ABI mismatch)";
  if (c.num_instances == 0) return "num_instances must be > 0";
  if (c.num_nodes < 1 || c.num_nodes > 64) return "num_nodes must be in 1..64";
  if (!c.seeds) return "seeds must not be NULL";
  if (c.max_clock < 0 || c.max_clock >= (1 << 29)) return "max_clock must be in [0, 2^29)";
  if (c.flags & ~(uint32_t)(LBFT_FLAG_ROUND_SWITCHES | LBFT_FLAG_RESUMABLE | LBFT_FLAG_TRUE_DATA_SYNC | LBFT_FLAG_COMMIT_TIMES))
    return "unknown bits in flags";
  const bool tds = (c.flags & LBFT_FLAG_TRUE_DATA_SYNC) != 0;
  if (tds && (c.flags & (LBFT_FLAG_ROUND_SWITCHES | LBFT_FLAG_RESUMABLE)))
    return "LBFT_FLAG_TRUE_DATA_SYNC cannot be combined with recording / resumable runs";
  if (c.commands_per_epoch == 0) return "commands_per_epoch must be > 0";
  if (c.delta < 0 || c.target_commit_interval < 0) return "delta and target_commit_interval must be >= 0";
  // delta == 0 makes round durations 0: a node can then create a timeout and propose in the same update (SURVEY App.
  // C.1b), which the round-id form does not represent (the device would flag every instance LBFT_ST_INVARIANT after
  // running the whole batch).  Refuse it up front.
  if (c.delta == 0) return "delta = 0 is not supported: a timeout and a proposal in the same update (SURVEY App. C.1b)";
  SweepSet s{};
  if (const char* e = delay_model(c, s)) return e;
  uint64_t total = 0;
  for (uint32_t i = 0; i < c.num_nodes; i++) {
    if (c.voting_rights && c.voting_rights[i] > (1u << 24)) return "voting_rights entries must be <= 2^24";
    total += c.voting_rights ? c.voting_rights[i] : 1;
  }
  if (total == 0) return "total voting rights must be > 0";
  if (c.partition_windows > 64) return "partition_windows must be <= 64";
  if (round_cap_of(c) > 32768) return "round_cap must be <= 32768";
  if (c.queue_cap > (1u << 20)) return "queue_cap too large";
  if (c.payload_cap > 0xfff0u) return "payload_cap must be < 65520";
  if (tds && c.commands_per_epoch < round_cap_of(c))
    return "LBFT_FLAG_TRUE_DATA_SYNC needs commands_per_epoch >= round_cap (single-epoch runs)";
  // commit times: the twins of the one-shot single-epoch kernels only (their table is indexed by round id)
  if ((c.flags & LBFT_FLAG_COMMIT_TIMES) && (c.flags & (LBFT_FLAG_ROUND_SWITCHES | LBFT_FLAG_RESUMABLE | LBFT_FLAG_TRUE_DATA_SYNC)))
    return "LBFT_FLAG_COMMIT_TIMES (commit times) cannot be combined with recording, resumable or true data-sync runs";
  if ((c.flags & LBFT_FLAG_COMMIT_TIMES) && epochs_of(c, round_cap_of(c)) > 1)
    return "LBFT_FLAG_COMMIT_TIMES (commit times) needs commands_per_epoch >= round_cap (single-epoch runs)";
  return nullptr;
}

// Kernel family.  One thread per instance needs tens of thousands of instances to fill an H100 (65 536 x 4 authors is one wave
// of warps) and serialises the 32 instances of a warp through every fan-out; one WARP per instance (lbft_wide_kernel) has no
// cross-instance divergence, splits fan-outs, queue scans and per-author vectors over its lanes, and for committees of <= 16
// keeps the whole instance in shared memory: committees of <= 5 switch below ~4 K instances, larger ones always profit (H100:
// 1 024 x 4 takes 2.5 ms wide against 9.2 ms on the thread kernel, 65 536 x 4 49.5 ms on the thread kernel against 68.4 ms
// wide).  Recording / resumable handles stay on the thread kernel (the wide one has no save area).
// LBFT_FORCE_KERNEL=wide|thread is a test seam, read here only: it runs one configuration through both families (and any
// value turns off the sparse tiles below).
// Returns KernelSel::tile: 1 = the wide kernel, else the thread kernel's instances per warp tile.  (Decided before the queue: the
// wide kernel has a shared-memory queue of its own.)
inline int kernel_family(const lbft_config& c, uint32_t rcap) {
  const uint32_t N = c.num_nodes, I = c.num_instances;
  const char* force = std::getenv("LBFT_FORCE_KERNEL");
  if (c.flags & (LBFT_FLAG_ROUND_SWITCHES | LBFT_FLAG_RESUMABLE | LBFT_FLAG_TRUE_DATA_SYNC)) return 32;
  if (force && !strcmp(force, "thread")) return 32;
  if (force && !strcmp(force, "wide")) return 1;
  if (N < 6 && I > 4096) return 32;
  // Sparse warp tiles of the thread kernel (kernels.cuh TILE: 8 or 16 instances per warp, the other lanes retire at once):
  // the instances of a warp serialise through each other's code paths, so as long as the batch does not fill the machine
  // with full warps (2 112 warps of <= 128 registers = one wave on 132 SMs), fewer instances per warp finish sooner.
  // Measured on BASELINE configs[4] (16 384 x 7, H100): 8 per warp 42.0 ms, full tiles 77.7, the wide kernel (8 lanes per
  // instance) 60.4.  So for committees of 6..16 (calendar queue, plain
  // single-epoch handles): about one wave of 8-instance warps -> tile 8, of 16-instance warps -> tile 16, more -> full
  // tiles; below that the wide kernel.
  if (force || N < 6 || N > 16 || c.max_clock > 4095 || I <= 12288 || c.commands_per_epoch < rcap || c.queue_cap > 0xfff0u) return 1;
  const uint32_t tile = I <= 24576 ? 8u : (I <= 49152 ? 16u : 32u);
  // (these handles get the calendar queue: the sparse-tile kernels keep the occupancy words of their instances in shared
  // memory, sim_core.cuh KS — ((max_clock + 8) / 8) x tile words per warp: horizons up to ~3 500 ms at 8 per warp, ~1 750
  // at 16)
  return (uint64_t)(((uint32_t)c.max_clock + 8) / 8) * tile > 3584 ? 32 : (int)tile;
}

// The layout, with the queue mode (queue_scan) and the queue / payload capacities decided here.
inline Layout choose_layout(const lbft_config& c, uint32_t rcap, uint32_t epochs, int tile) {
  const uint32_t N = c.num_nodes;
  const bool wide = tile == 1, tds = (c.flags & LBFT_FLAG_TRUE_DATA_SYNC) != 0;
  // (recording round switches queues the duplicate timers the normal path elides — measured high-water marks
  // roughly double, 46 -> 64+ at N = 4 — so the smallest committees get 128 entries and the HBM scan queue)
  // (resumable runs queue them too: the event dropped at a stop must be the one the reference drops)
  const bool record = (c.flags & (LBFT_FLAG_ROUND_SWITCHES | LBFT_FLAG_RESUMABLE)) != 0;
  uint32_t pcap = c.payload_cap ? c.payload_cap : (N <= 4 ? 32u : (N <= 8 ? 64u : pow2_ceil(8 * N)));
  // (true data-sync keeps a snapshot per request and per response in flight as well)
  if (tds && !c.payload_cap) pcap = N <= 4 ? 128u : (N <= 8 ? 192u : 4 * pcap);
  // The shortest horizons run on the compact entries: 32-bit keys (time:14 | kind:2 | stamp:16) + 16-bit payload words.
  // (16-bit stamps: ~0.14 N^2 events are created per simulated ms at the reference's 10 ms mean delay, and proportionally
  // more with shorter delays; stay well inside 65 536 — an overflow would be flagged, not silent)
  const double mean = mean_delay(c), events_per_ms = 0.14 * N * N * (10.0 / (mean < 1.0 ? 1.0 : mean));
  const bool compact = c.max_clock < (1 << 14) - 64 && pcap <= 255 && events_per_ms * (double)c.max_clock < 32768.0;
  // Small committees use the scan queue (64-bit entries: time:24 | 3-kind:2 | stamp:22 | slot:8 | sender:4 |
  // receiver:4, O(1) append, linear min-scan); larger ones the binary heap with 3-word entries.
  // (explicit capacities beyond what the scan queue can encode / scan efficiently select the heap.)
  uint32_t scan = N <= 5 && c.max_clock < (1 << 24) - 64 && c.payload_cap <= 255 && c.queue_cap <= 512 ? 1u : 0u;
  uint32_t cap = c.queue_cap ? c.queue_cap : (scan ? (N <= 4 ? (record ? 128u : 64u) : 8 * N * N) : pow2_ceil(6 * N * N + 32));
  if (cap < readout_queue_floor(scan, rcap)) cap = readout_queue_floor(scan, rcap);
  if (scan && compact && cap <= 64) scan = 2;  // queue in shared memory
  // the HBM scan queue hands out 22-bit creation stamps: long horizons / very short delays go to the heap or calendar
  // queue (30-bit / 32-bit stamps) instead of aborting with LBFT_ST_QUEUE_OVERFLOW half-way through
  if (scan == 1 && events_per_ms * (double)c.max_clock > 2.0e6) scan = 0;
  // The wide kernel scans its (single) shared-memory queue with all 32 lanes, so the same compact entries serve committees
  // up to 16 (4-bit sender/receiver) and queues up to 1 024 entries.
  if (wide && N <= 16 && compact) {
    const uint32_t want = c.queue_cap ? c.queue_cap : (N <= 4 ? 64u : 8 * N * N);
    if (want <= 1024) {
      scan = 2;
      cap = want < readout_queue_floor(2, rcap) ? readout_queue_floor(2, rcap) : want;
    }
  }
  // everything else with a moderate horizon: calendar queue (O(1) push/pop, exact: FIFO order inside a (time, kind)
  // list is creation-stamp order); the binary heap remains for long horizons
  if (scan == 0 && c.max_clock <= 4095 && cap <= 0xfff0u) scan = 3;
  // epochs: the read-out floor of the global round ids, for the mode as it stands; then a shared-memory queue that outgrew
  // shared memory moves to the HBM scan, calendar or heap queue (keeping the floor it got)
  if (epochs > 1) {
    const uint32_t floor = readout_queue_floor(scan, epochs * rcap);
    if (cap < floor) cap = scan ? floor : pow2_ceil(floor);
    if (scan == 2 && cap > (wide ? 1024u : 64u)) scan = N <= 5 ? 1u : (c.max_clock <= 4095 ? 3u : 0u);
  }
  return make_layout(N, rcap, cap, pcap, c.partition_windows, scan, (uint32_t)c.max_clock, (c.flags & LBFT_FLAG_ROUND_SWITCHES) != 0,
                     (c.flags & LBFT_FLAG_RESUMABLE) != 0, epochs, tds);
}

// The kernel a handle launches, once its layout is known.
inline KernelSel select_kernel(const lbft_config& c, int tile, const Params& p, bool sweep) {
  KernelSel k{};
  const uint32_t N = c.num_nodes, qscan = p.L.queue_scan;
  k.wide = tile == 1;
  k.tile = tile;
  // lanes per instance: enough for the committee's fan-out, few enough that a warp carries several instances
  // (8 lanes per instance — four instances per warp — win once the batch fills the machine with warps, committees of 64
  // included: on an H100 8 192 x 64 takes 0.86 s against 1.32 s with a warp per instance; below ~4 K instances a whole warp
  // per instance has the lower latency)
  k.group = c.num_instances > 4096 && p.L.epochs == 1 ? 8 : 32;
  // wide kernel: the whole instance lives in shared memory when the instances of 16 resident warps (32 / group each) fit on
  // an SM
  const size_t smem_bytes = sizeof(uint32_t) * (size_t)p.L.total_words + 6u * (size_t)p.L.queue_cap + 1024u;
  k.smem = k.wide && qscan == 2 && p.L.epochs == 1 && smem_bytes * (128u / k.group) <= 56u * 1024u;
  k.qmode = (int)qscan;
  k.nmax = (qscan == 1 || qscan == 2) ? 16 : (N <= 16 ? 16 : (N <= 32 ? 32 : 64));
  k.epochs = p.L.epochs > 1;
  k.tds = p.L.tds != 0;
  k.rec = p.record_rs != 0;
  k.res = p.resumable != 0;
  // compile-time layouts: FX_DEFAULT4 on the thread kernel, FX_PART7 on its 8-instance warp tiles, FX_COMMITTEE64 on the wide
  // kernel with 8 lanes per instance (sweep handles run the generic layout)
  const int fx = fixed_shape_of(p);
  k.fixed = !sweep && ((fx == FX_DEFAULT4 && !k.wide) || (fx == FX_PART7 && !k.wide && k.tile == 8) ||
                       (fx == FX_COMMITTEE64 && k.wide && k.group == 8))
                ? fx : FX_NONE;
  k.sweep = sweep;
  k.ct = (c.flags & LBFT_FLAG_COMMIT_TIMES) != 0;  // (the flag changes nothing above: the twin of the flag-off kernel)
  return k;
}

// `c` with the fields of one parameter set of a sweep substituted.
inline lbft_config with_set(const lbft_config& c, const lbft_param_set& q) {
  lbft_config cs = c;
  cs.delay_kind = q.delay_kind;
  cs.delay_mean = q.delay_mean;
  cs.delay_variance = q.delay_variance;
  cs.delay_lo = q.delay_lo;
  cs.delay_hi = q.delay_hi;
  cs.target_commit_interval = q.target_commit_interval;
  cs.delta = q.delta;
  cs.gamma = q.gamma;
  cs.lambda = q.lambda;
  return cs;
}

// `c` with the fault model of one parameter set of a fault sweep substituted: `silent` (num_nodes entries) receives the
// mask's nodes and must outlive the result.
inline lbft_config with_faults(const lbft_config& c, const lbft_fault_set& f, uint8_t (&silent)[64]) {
  lbft_config cs = c;
  for (uint32_t n = 0; n < 64; n++) silent[n] = (uint8_t)((f.silent_mask >> n) & 1);
  cs.silent = f.silent_mask ? silent : nullptr;
  cs.partition_windows = f.partition_windows;
  cs.partition_max_len = f.partition_max_len;
  return cs;
}

struct HostSetup {
  Params params{};  // pointer members are left null; the runtime fills in device addresses
  std::vector<double> zig_x, zig_f;
  std::vector<uint8_t> leader;
  std::vector<int32_t> duration, period;
  std::vector<uint32_t> weights;
  std::vector<double> delay_thr;  // see build_delay_table()
  std::vector<SweepSet> sets;     // sweep handles: one record per parameter set (build_sweep); empty otherwise
  std::vector<uint32_t> set_of;   // sweep handles: [num_instances] the set of each instance
  std::vector<SweepFaults> faults;  // fault and rights sweeps: one record per parameter set (build_sweep_faults / _rights); empty otherwise
  std::vector<SweepRights> rights;  // rights sweeps: one record per parameter set (build_sweep_rights); empty otherwise
  bool committees = false;          // a committee sweep (build_sweep_committees): each set's fault record carries its committee size
  std::vector<uint16_t> links;      // links sweeps: the distinct N x N link-latency matrices of the sets (build_sweep_links)
  std::vector<uint32_t> link_off;   // links sweeps: one record per parameter set, where its matrix starts in `links`; empty otherwise
  std::string error;
  KernelSel sel{};

  bool build(const lbft_config& c) {
    if (const char* e = config_error(c)) return fail(e);
    const uint32_t rcap = round_cap_of(c);
    const int tile = kernel_family(c, rcap);
    build_shared(c, choose_layout(c, rcap, epochs_of(c, rcap), tile));
    SweepSet s{};
    add_set(c, rcap, s);
    use_set(s);
    sel = select_kernel(c, tile, params, false);
    return true;
  }

  // A sweep handle (lbft_create_sweep): `c` with each set's delay / NodeConfig fields substituted must be a valid plain
  // configuration.  Layout and kernel are what build() picks for the set with the highest event rate (the shortest mean
  // delay: the one the stamp-width and queue-mode tests are sized by), on the sweep kernels; per set, the delay model, the
  // threshold table and the duration / period tables are built as build() builds them and concatenated.
  //
  // A fault sweep (lbft_create_sweep_faults, `fs` not null): each set's fault model is substituted as well, the shared
  // configuration carries none, and the layout and kernel are what a sweep picks with the largest window count of any set in
  // the configuration; `faults` gets each set's record, and Params::silent_mask the union of the sets' silent nodes (the
  // kernels' launch-uniform test for whether any node can be silent: sim_core.cuh Core::any_silent).
  //
  // A rights sweep (lbft_create_sweep_rights, `vr` not null: [num_sets][num_nodes]): each set's voting rights are substituted
  // as well and the configuration carries none.  Layout and kernel do not depend on the rights.  `rights` gets each set's
  // record, with one leader table per distinct row of `vr` appended to `leader` (set 0's first, where a plain handle has its
  // own); `faults` gets each set's fault record, the configuration's shared faults when `fs` is null; and weights, Params'
  // quorum and c_weights are set 0's.
  //
  // A committee sweep (lbft_create_sweep_committees, `sizes` not null: [num_sets], with `vr`): a rights sweep whose set s runs a
  // committee of sizes[s] <= num_nodes nodes, validated as a plain configuration of that many nodes.  c.num_nodes stays the
  // layout's committee, so layout and kernel are the rights sweep's; each row of `vr` is 0 past its set's committee, and each
  // set's fault record carries the size.
  //
  // A links sweep (lbft_create_sweep_links, `lk` not null: [num_sets][num_nodes][num_nodes]): a rights sweep (a committee sweep
  // when `sizes` is not null) whose set s adds lk[s][a][b] to the time of every network event from a to b.  With `vr` null each
  // set gets the configuration's shared rights (1 per node of its committee when it has none).  Layout and kernel do not depend
  // on the matrices: the stamp-width and queue-mode tests are sized by the shortest mean delay, which over-estimates the event
  // rate of a network slowed by its links, so they stay safe (and an overrun still surfaces as LBFT_ERR_CAPACITY).  `links` gets
  // one matrix per distinct one, `link_off` each set's.
  bool build_sweep(const lbft_config& c, const lbft_param_set* ps, uint32_t num_sets, const uint32_t* set_of_instance,
                   const lbft_fault_set* fs = nullptr, const uint64_t* vr = nullptr, const uint32_t* sizes = nullptr,
                   const uint32_t* lk = nullptr) {
    if (c.struct_size != sizeof(lbft_config)) return fail("lbft_config.struct_size does not match this library (ABI mismatch)");
    if (!ps || !set_of_instance) return fail("sets and set_of_instance must not be NULL");
    if (num_sets == 0 || num_sets > c.num_instances || num_sets > 65536u) return fail("num_sets must be in 1..min(num_instances, 65536)");
    if (c.flags & ~(uint32_t)LBFT_FLAG_COMMIT_TIMES) return fail("sweep handles take no flags (recording, resumable and true data-sync runs are plain handles only)");
    for (uint32_t i = 0; i < c.num_instances; i++)
      if (set_of_instance[i] >= num_sets) return fail("set_of_instance has an index >= num_sets");
    if (fs && (c.silent || c.partition_windows || c.partition_max_len))
      return fail("a fault sweep takes its silent nodes and partitions per set only: lbft_config.silent must be NULL and "
                  "partition_windows / partition_max_len 0");
    if ((vr || sizes) && c.voting_rights)
      return fail("a rights sweep takes its voting rights per set only: lbft_config.voting_rights must be NULL");
    uint32_t fastest = 0, windows = 0;
    for (uint32_t s = 0; s < num_sets; s++) {
      uint8_t silent[64];
      lbft_config cs = fs ? with_faults(with_set(c, ps[s]), fs[s], silent) : with_set(c, ps[s]);
      if (vr) cs.voting_rights = vr + (size_t)s * c.num_nodes;
      const char* e = sizes ? committee_error(c, cs, sizes[s]) : nullptr;
      if (!e && sizes) cs.num_nodes = sizes[s];
      if (!e) e = config_error(cs);
      if (!e && fs && cs.num_nodes < 64 && (fs[s].silent_mask >> cs.num_nodes)) e = "silent_mask has a bit at or above num_nodes";
      if (!e && lk) e = links_error(lk + (size_t)s * c.num_nodes * c.num_nodes, c.num_nodes, cs.num_nodes);
      if (e || ps[s].reserved)
        return fail(("parameter set " + std::to_string(s) + ": " + (ps[s].reserved ? "reserved must be 0" : e)).c_str());
      if (mean_delay(cs) < mean_delay(with_set(c, ps[fastest]))) fastest = s;
      if (fs && fs[s].partition_windows > windows) windows = fs[s].partition_windows;
    }
    // a committee or links sweep without rights: the shared rights, or 1, for each node of a set's committee (validated above)
    std::vector<uint64_t> ones;
    if ((sizes || lk) && !vr) {
      ones.assign((size_t)num_sets * c.num_nodes, 0);
      for (uint32_t s = 0; s < num_sets; s++)
        for (uint32_t n = 0; n < (sizes ? sizes[s] : c.num_nodes); n++)
          ones[(size_t)s * c.num_nodes + n] = c.voting_rights ? c.voting_rights[n] : 1;
      vr = ones.data();
    }
    lbft_config cf = with_set(c, ps[fastest]);
    if (fs) cf.partition_windows = windows;
    if (vr) cf.voting_rights = vr;  // (set 0's: build_shared's weights, quorum and first leader table; no decision reads them)
    const uint32_t rcap = round_cap_of(cf);
    if (c.commands_per_epoch < rcap)
      return fail("sweep handles need commands_per_epoch >= round_cap (single-epoch runs: epochs are plain handles only)");
    const int tile = kernel_family(cf, rcap);
    build_shared(cf, choose_layout(cf, rcap, 1, tile));
    sets.resize(num_sets);
    for (uint32_t s = 0; s < num_sets; s++) add_set(with_set(c, ps[s]), rcap, sets[s]);
    use_set(sets[fastest]);
    set_of.assign(set_of_instance, set_of_instance + c.num_instances);
    if (fs) {
      faults.resize(num_sets);
      for (uint32_t s = 0; s < num_sets; s++) {
        faults[s] = SweepFaults{fs[s].silent_mask, (uint16_t)fs[s].partition_windows, 0, fs[s].partition_max_len};
        params.silent_mask |= fs[s].silent_mask;  // the union: the kernels' launch-uniform "any silent node" test
      }
    } else if (vr) {
      faults.assign(num_sets, SweepFaults{params.silent_mask, (uint16_t)params.L.part_windows, 0, params.part_max_len});
    }
    if (sizes)
      for (uint32_t s = 0; s < num_sets; s++) faults[s].num_nodes = (uint16_t)sizes[s];
    if (vr) add_rights(vr, num_sets);
    if (lk) add_links(lk, num_sets);
    committees = sizes != nullptr;
    sel = select_kernel(cf, tile, params, true);
    return true;
  }

  // A fault sweep (lbft_create_sweep_faults): build_sweep with each set's fault model.
  bool build_sweep_faults(const lbft_config& c, const lbft_param_set* ps, const lbft_fault_set* fs, uint32_t num_sets,
                          const uint32_t* set_of_instance) {
    if (!fs) return fail("faults must not be NULL");
    return build_sweep(c, ps, num_sets, set_of_instance, fs);
  }

  // A rights sweep (lbft_create_sweep_rights): build_sweep with each set's voting rights, and its faults when `fs` is not null.
  bool build_sweep_rights(const lbft_config& c, const lbft_param_set* ps, const lbft_fault_set* fs, const uint64_t* vr,
                          uint32_t num_sets, const uint32_t* set_of_instance) {
    if (!vr) return fail("voting_rights must not be NULL");
    return build_sweep(c, ps, num_sets, set_of_instance, fs, vr);
  }

  // A committee sweep (lbft_create_sweep_committees): build_sweep_rights with each set's committee size, its voting rights
  // (row s of `vr`, or 1 for each of its nodes when `vr` is null) and its faults when `fs` is not null.
  bool build_sweep_committees(const lbft_config& c, const lbft_param_set* ps, const lbft_fault_set* fs, const uint64_t* vr,
                              const uint32_t* sizes, uint32_t num_sets, const uint32_t* set_of_instance) {
    if (!sizes) return fail("committee_sizes must not be NULL");
    return build_sweep(c, ps, num_sets, set_of_instance, fs, vr, sizes);
  }

  // A links sweep (lbft_create_sweep_links): build_sweep with each set's link-latency matrix (lk[s], [num_nodes][num_nodes]),
  // its voting rights (row s of `vr`, or the shared ones when `vr` is null), its faults when `fs` is not null and its committee
  // size when `sizes` is not null.
  bool build_sweep_links(const lbft_config& c, const lbft_param_set* ps, const lbft_fault_set* fs, const uint64_t* vr,
                         const uint32_t* sizes, const uint32_t* lk, uint32_t num_sets, const uint32_t* set_of_instance) {
    if (!lk) return fail("link_latency must not be NULL");
    return build_sweep(c, ps, num_sets, set_of_instance, fs, vr, sizes, lk);
  }

  // Which records follow each set in the sweep's device table (sim_core.cuh sweep_set_at): bit 0 faults, bit 1 rights, bit 2 on
  // a committee sweep, whose fault records carry the committee sizes (the entries are those of a rights sweep), and bit 3 the
  // links records of a links sweep.
  uint32_t records() const {
    return (faults.empty() ? 0u : 1u) | (rights.empty() ? 0u : 2u) | (committees ? 4u : 0u) | (link_off.empty() ? 0u : 8u);
  }

  // A sweep's device table of parameter sets, the bytes the runtime uploads: `sets`, each followed by its fault record, its
  // rights record and its links record where records() has them (SweepSet, SweepSetFaults, SweepSetRights or SweepSetLinks
  // entries).
  std::vector<uint64_t> set_table() const {
    const uint32_t rec = records();
    const size_t pitch = (rec & 8)   ? sizeof(SweepSetLinks)
                         : (rec & 2) ? sizeof(SweepSetRights)
                                     : ((rec & 1) ? sizeof(SweepSetFaults) : sizeof(SweepSet));
    static_assert(sizeof(SweepSet) % 8 == 0 && sizeof(SweepSetFaults) % 8 == 0 && sizeof(SweepSetRights) % 8 == 0 &&
                      sizeof(SweepSetLinks) % 8 == 0, "whole words");
    std::vector<uint64_t> t(sets.size() * pitch / 8);
    for (size_t k = 0; k < sets.size(); k++) {
      char* e = reinterpret_cast<char*>(t.data()) + k * pitch;
      memcpy(e, &sets[k], sizeof(SweepSet));
      if (rec & 1) memcpy(e + offsetof(SweepSetFaults, faults), &faults[k], sizeof(SweepFaults));
      if (rec & 2) memcpy(e + offsetof(SweepSetRights, rights), &rights[k], sizeof(SweepRights));
      if (rec & 8) {
        const SweepLinks l{link_off[k], 0};
        memcpy(e + offsetof(SweepSetLinks, links), &l, sizeof(SweepLinks));
      }
    }
    return t;
  }

 private:
  // Everything but the per-set part: the launch-uniform fields of Params, the voting rights, the leader table and the ziggurat.
  void build_shared(const lbft_config& c, const Layout& L) {
    const uint32_t N = c.num_nodes;
    Params& p = params;
    p.num_instances = c.num_instances;
    p.max_clock = (int32_t)c.max_clock;
    p.commands_per_epoch = c.commands_per_epoch > 0xffffffffULL ? 0xffffffffu : (uint32_t)c.commands_per_epoch;
    // voting rights / quorum (configuration.rs:29-56; simulated_context.rs:209-216 = all 1)
    weights.assign(N, 1);
    uint64_t total = 0;
    for (uint32_t i = 0; i < N; i++) {
      if (c.voting_rights) weights[i] = (uint32_t)c.voting_rights[i];
      total += weights[i];
    }
    p.quorum = quorum_of(total);
    for (uint32_t i = 0; i < 64; i++) p.c_weights[i] = i < N ? weights[i] : 0;
    if (c.silent)
      for (uint32_t i = 0; i < N; i++)
        if (c.silent[i]) p.silent_mask |= 1ULL << i;
    p.part_max_len = c.partition_max_len;
    // loop_until(.., Some(csv_path)) simulator.rs:380-381: keep DataWriter's round-switch table (the compile-time-layout
    // kernel never records: its layout has no table, so the generic instantiation is selected)
    p.record_rs = (c.flags & LBFT_FLAG_ROUND_SWITCHES) ? 1u : 0u;
    p.resumable = (c.flags & LBFT_FLAG_RESUMABLE) ? 1u : 0u;
    p.stop_clock = p.max_clock;
    p.L = L;
    leader.clear();
    add_leader_table(weights, total);
    build_ziggurat();
  }

  static uint32_t quorum_of(uint64_t total) { return (uint32_t)(2 * total / 3 + 1); }

  // leader(round) under voting rights `w` for every representable round (+1: the pacemaker looks at active_round <= round_cap),
  // appended to `leader`; returns where it starts.
  uint32_t add_leader_table(const std::vector<uint32_t>& w, uint64_t total) {
    const uint32_t off = (uint32_t)leader.size(), rspan = params.L.rspan;
    leader.resize((size_t)off + rspan + 1);
    for (uint32_t r = 0; r <= rspan; r++) leader[(size_t)off + r] = (uint8_t)pick_author(w, total, siphash13_u64(r));
    return off;
  }

  // A rights sweep's records (`vr`: [num_sets][num_nodes], checked by config_error): per set its weights and quorum, and one
  // leader table per distinct row.  Set 0's table is the one build_shared made.  A committee sweep's rows are 0 past each set's
  // committee, which pick_author's scan never reaches: each table is the set's plain committee's.
  void add_rights(const uint64_t* vr, uint32_t num_sets) {
    const uint32_t N = params.L.num_nodes;
    std::map<std::vector<uint32_t>, uint32_t> table_of;
    table_of.emplace(weights, 0u);
    rights.assign(num_sets, SweepRights{});
    std::vector<uint32_t> row(N);
    for (uint32_t s = 0; s < num_sets; s++) {
      uint64_t total = 0;
      for (uint32_t n = 0; n < N; n++) total += row[n] = (uint32_t)vr[(size_t)s * N + n];
      auto it = table_of.find(row);
      if (it == table_of.end()) it = table_of.emplace(row, add_leader_table(row, total)).first;
      SweepRights& r = rights[s];
      r.quorum = quorum_of(total);
      r.leader_off = it->second;
      for (uint32_t n = 0; n < N; n++) r.weights[n] = row[n];
    }
  }

  // A links sweep's records (`lk`: [num_sets][N][N], checked by links_error): one matrix of u16 per distinct one in `links`, and
  // where each set's starts in `link_off`.
  void add_links(const uint32_t* lk, uint32_t num_sets) {
    const size_t NN = (size_t)params.L.num_nodes * params.L.num_nodes;
    std::map<std::vector<uint16_t>, uint32_t> off_of;
    link_off.assign(num_sets, 0);
    std::vector<uint16_t> m(NN);
    for (uint32_t s = 0; s < num_sets; s++) {
      for (size_t k = 0; k < NN; k++) m[k] = (uint16_t)lk[s * NN + k];
      auto it = off_of.find(m);
      if (it == off_of.end()) {
        it = off_of.emplace(m, (uint32_t)links.size()).first;
        links.insert(links.end(), m.begin(), m.end());
      }
      link_off[s] = it->second;
    }
  }

  // The part of a configuration a sweep varies per parameter set (lbft_param_set): its delay model and tci into `s`, its delay
  // thresholds and its duration / period tables appended to delay_thr / duration / period, where `s` records their offsets.
  void add_set(const lbft_config& c, uint32_t rcap, SweepSet& s) {
    delay_model(c, s);  // (valid: config_error() has checked it)
    s.tci = (int32_t)(c.target_commit_interval > (1 << 30) ? (1 << 30) : c.target_commit_interval);
    s.thr_off = (uint32_t)delay_thr.size();
    build_delay_table(s);
    // duration(n) = (delta as f64 * (n as f64).powf(gamma)) as i64; period = (lambda * duration as f64) as i64
    s.rt_off = (uint32_t)duration.size();
    for (uint32_t n = 0; n <= rcap; n++) {
      double dv = (double)c.delta * std::pow((double)n, c.gamma);
      int64_t dur = std::isnan(dv) ? 0 : (dv >= 9.2e18 ? INT64_MAX : (dv <= -9.2e18 ? INT64_MIN : (int64_t)dv));
      double pv = c.lambda * (double)dur;
      int64_t per = std::isnan(pv) ? 0 : (pv >= 9.2e18 ? INT64_MAX : (pv <= -9.2e18 ? INT64_MIN : (int64_t)pv));
      const int64_t CL = 1 << 30;  // any deadline beyond max_clock (< 2^29) behaves identically
      duration.push_back((int32_t)(dur > CL ? CL : (dur < -CL ? -CL : dur)));
      period.push_back((int32_t)(per > CL ? CL : (per < -CL ? -CL : per)));
    }
  }

  // The launch-uniform copy of a set's delay model and tci (a sweep's kernels read each instance's set instead).
  void use_set(const SweepSet& s) {
    Params& p = params;
    p.delay_kind = s.delay_kind;
    p.delay_const = s.delay_const;
    p.delay_const_value = s.delay_const_value;
    p.mu = s.mu;
    p.sigma = s.sigma;
    p.uni_lo = s.uni_lo;
    p.uni_span = s.uni_span;
    p.tci = s.tci;
    p.delay_kmax = s.delay_kmax;
  }

  // LogNormal delay without a device-side exp(): the reference truncates exp(mu + sigma*z) to an integer
  // (simulator.rs:115-117), so only the integer part matters.  thr[k] is the smallest double z with
  // (exp(mu + sigma*z) as i64) >= k, found by bisection over the doubles with the HOST libm — the very
  // function the Rust reference calls — so the device result is bit-identical to the host's by
  // construction (no last-ulp dependence on the CUDA math library).  Table: thr[0] = -inf,
  // thr[1..kmax], thr[kmax+1] = +inf, where kmax = delay at the largest deviate the ziggurat can emit.
  // Appended to delay_thr; s.delay_kmax = 0 (and nothing appended) keeps the exp() path.
  void build_delay_table(SweepSet& s) {
    s.delay_kmax = 0;
    if (s.delay_kind != LBFT_DELAY_LOGNORMAL || s.delay_const) return;
    const double mu = s.mu, sigma = s.sigma;
    auto D = [mu, sigma](double z) -> int64_t {
      double v = std::exp(mu + sigma * z);
      return v >= 9.0e18 ? INT64_MAX : (int64_t)v;
    };
    // |z| <= 12.2254 for the 256-layer ziggurat: the tail returns R - ln(a)/R only once -2 ln(b) >= (ln(a)/R)^2, and
    // -2 ln(b) <= 106 ln(2) for an Open01 b >= 2^-53 (tests/rng_support.py largest_deviate)
    const double ZMAX = 14.0;
    int64_t kmax = D(ZMAX);
    if (kmax < 1 || kmax > 4096) return;  // too wide: keep the exp() path
    auto key = [](double d) { int64_t b; memcpy(&b, &d, 8); return b < 0 ? INT64_MIN - b : b; };  // monotone map
    auto unkey = [](int64_t k) { int64_t b = k < 0 ? INT64_MIN - k : k; double d; memcpy(&d, &b, 8); return d; };
    std::vector<double> thr((size_t)kmax + 2, 0.0);
    thr[0] = -INFINITY;
    thr[kmax + 1] = INFINITY;
    for (int64_t k = 1; k <= kmax; k++) {
      if (D(-ZMAX) >= k) { thr[k] = -INFINITY; continue; }
      int64_t lo = key(-ZMAX), hi = key(ZMAX);  // D(lo) < k <= D(hi)
      while ((__int128)hi - lo > 1) {
        int64_t mid = (int64_t)(((__int128)lo + hi) >> 1);
        if (D(unkey(mid)) >= k) hi = mid; else lo = mid;
      }
      thr[k] = unkey(hi);
      // exp() must be monotone across the threshold for the table to be exact: check a few ulps either side
      for (int j = 1; j <= 4; j++)
        if (D(unkey(hi + j)) < k || D(unkey(hi - j)) >= k) return;
    }
    delay_thr.insert(delay_thr.end(), thr.begin(), thr.end());
    s.delay_kmax = (uint32_t)kmax;
  }

  // rand_distr 0.4.0 ziggurat_tables.rs (ZIG_NORM_X / ZIG_NORM_F / ZIG_NORM_R): regenerated with the
  // crate's generator recurrence and passed through the "%.18f" decimal literals it ships.
  void build_ziggurat() {
    const double R = 3.6541528853610088, V = 0.00492867323399;
    std::vector<double> xs(257);
    auto f = [](double t) { return std::exp(-t * t / 2.0); };
    xs[0] = V / f(R);
    xs[1] = R;
    for (int i = 2; i < 256; i++) xs[i] = std::sqrt(-2.0 * std::log(V / xs[i - 1] + f(xs[i - 1])));
    xs[256] = 0.0;
    auto lit = [](double v) {
      char buf[64];
      snprintf(buf, sizeof buf, "%.18f", v);
      return strtod(buf, nullptr);
    };
    zig_x.resize(257);
    zig_f.resize(257);
    for (int i = 0; i <= 256; i++) {
      zig_x[i] = lit(xs[i]);
      zig_f[i] = lit(f(xs[i]));
    }
    params.zig_r = lit(R);
  }

  // A committee sweep's checks on set s beyond those of a plain configuration of its size n (`cs`: the set's configuration with
  // the layout's num_nodes): null when valid.
  static const char* committee_error(const lbft_config& c, const lbft_config& cs, uint32_t n) {
    if (c.num_nodes > 64) return "num_nodes must be in 1..64";
    if (n < 1 || n > c.num_nodes) return "committee size must be in 1..lbft_config.num_nodes (the layout's committee)";
    for (uint32_t k = n; k < c.num_nodes; k++) {
      if (cs.voting_rights && cs.voting_rights[k]) return "voting_rights has a non-zero entry at or past the set's committee size";
      if (cs.silent && cs.silent[k]) return "a silent node is at or past the set's committee size";
    }
    return nullptr;
  }

  // A links sweep's checks on set s's matrix `m` ([N][N]) for a committee of n nodes: null when valid.
  static const char* links_error(const uint32_t* m, uint32_t N, uint32_t n) {
    for (uint32_t a = 0; a < N; a++)
      for (uint32_t b = 0; b < N; b++) {
        const uint32_t v = m[(size_t)a * N + b];
        if (v > 65535u) return "link_latency entries must be <= 65535";
        if (v && (a >= n || b >= n)) return "link_latency has a non-zero entry in a row or column at or past the set's committee size";
      }
    return nullptr;
  }

  bool fail(const char* msg) {
    error = msg;
    return false;
  }
};

// lbft_latency_stats: the groups of a handle (its parameter sets, or one), and the checks on its spec (null when it is valid).
inline uint32_t latency_groups(const HostSetup& hs) { return hs.sets.empty() ? 1u : (uint32_t)hs.sets.size(); }
inline const char* latency_spec_error(const HostSetup& hs, const lbft_latency_spec& spec) {
  if (spec.struct_size != sizeof(lbft_latency_spec)) return "lbft_latency_spec.struct_size does not match this library (ABI mismatch)";
  if (spec.num_bins < 1 || spec.num_bins > 65536u) return "num_bins must be in 1..65536";
  if (spec.bin_width < 1) return "bin_width must be >= 1";
  if (spec.proposed_from > spec.proposed_until) return "proposed_from must be <= proposed_until";
  if ((uint64_t)latency_groups(hs) * spec.num_bins > (1u << 24)) return "num_groups * num_bins must be <= 2^24";
  // every sample is at most max_clock and an instance has fewer than round_cap rows per node: this bounds sum
  const Params& p = hs.params;
  const unsigned __int128 bound = (unsigned __int128)p.num_instances * p.L.num_nodes * p.L.round_cap * (uint64_t)p.max_clock;
  if (bound >> 64) return "num_instances * num_nodes * round_cap * max_clock must fit in 64 bits (the bound on sum)";
  return nullptr;
}

// lbft_block_latency_stats: the total voting rights of group g of a handle (on a rights sweep its parameter set's, on every
// other handle the one committee's), and the checks on one threshold for every group (lbft_block_latency_stats) and on a
// threshold per group (lbft_block_latency_stats_groups, thresholds[latency_groups(hs)]): null when valid.  A message that
// names a group lives until the next check on this thread.
inline uint64_t total_voting_rights(const HostSetup& hs, uint32_t g = 0) {
  uint64_t total = 0;
  if (!hs.rights.empty()) {
    for (uint32_t w : hs.rights[g].weights) total += w;  // (0 past num_nodes)
    return total;
  }
  for (uint32_t w : hs.weights) total += w;
  return total;
}
inline const char* group_threshold_message(const char* what, uint32_t g, uint64_t total) {
  static thread_local std::string msg;
  msg = std::string(what) + " must be in 1..total voting rights of group " + std::to_string(g) + " (" + std::to_string(total) + ")";
  return msg.c_str();
}
inline const char* block_latency_threshold_error(const HostSetup& hs, uint64_t threshold) {
  if (hs.rights.empty()) {
    if (threshold < 1 || threshold > total_voting_rights(hs)) return "threshold must be in 1..total voting rights of the handle";
    return nullptr;
  }
  for (uint32_t g = 0; g < latency_groups(hs); g++)
    if (threshold < 1 || threshold > total_voting_rights(hs, g)) return group_threshold_message("threshold", g, total_voting_rights(hs, g));
  return nullptr;
}
inline const char* block_latency_thresholds_error(const HostSetup& hs, const uint64_t* thresholds) {
  for (uint32_t g = 0; g < latency_groups(hs); g++)
    if (thresholds[g] < 1 || thresholds[g] > total_voting_rights(hs, g))
      return group_threshold_message(("thresholds[" + std::to_string(g) + "]").c_str(), g, total_voting_rights(hs, g));
  return nullptr;
}

}  // namespace lbft
