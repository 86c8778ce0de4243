// hostcore.cpp — TEST INFRASTRUCTURE: compiles the device state machine (csrc/sim_core.cuh) with g++
// so that its logic can be checked against the oracle in the CPU-only container.  It is never part
// of, linked into, or reachable from the product library (librabft_simulator_b200/csrc/liblbft_b200.so).
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../librabft_simulator_b200/csrc/host_setup.hpp"
#include "../../librabft_simulator_b200/csrc/sim_core.cuh"

using namespace lbft;
static thread_local std::string g_err;

template <int NMAX, int QMODE, bool REC, bool RES, bool EP, bool TDS = false>
static void run_all_ep(const Params& P, std::vector<uint32_t>& state, const double* zx, const double* zf) {
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * P.L.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, false, REC, RES, 1, EP, TDS> core(P, mem, zx, zf, P.delay_thr, sk.data() + lane, sd.data() + lane);
    // QMODE 2: the stand-in for the shared-memory queue is per call, like shared memory is per launch
    if (RES && (P.run_flags & 1u)) core.restore_regs();
    else core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
    if (RES) core.save_regs();
  }
}

// (the host harness instantiates the epoch machinery for every mode, so that the CPU tests cover epochs x recording x staged
// runs; the product library has it for plain kernels only)
template <int NMAX, int QMODE, bool REC, bool RES>
static void run_all(const Params& P, std::vector<uint32_t>& state, const double* zx, const double* zf) {
  if (P.L.tds) {
    if (!REC && !RES) run_all_ep<NMAX, QMODE, false, false, false, true>(P, state, zx, zf);  // (HostSetup refuses the other combinations)
  } else if (P.L.epochs > 1) run_all_ep<NMAX, QMODE, REC, RES, true>(P, state, zx, zf);
  else run_all_ep<NMAX, QMODE, REC, RES, false>(P, state, zx, zf);
}

// The instantiations with a compile-time layout (sim_core.cuh FX, sim_params.h fixed_layout) on the host: selected by the
// product's fixed_shape_of (host_setup.hpp; the kernel family / tile / lane-group conditions do not exist here), so that the
// CPU tests of those shapes exercise the very state machine the BASELINE configurations run on the GPU.
template <int NMAX, int QMODE, int FX>
static void run_all_fx(const Params& P, std::vector<uint32_t>& state, const double* zx, const double* zf) {
  for (uint32_t inst = 0; inst < P.num_instances; inst++) {
    uint32_t tile = inst / 32, lane = inst % 32;
    TileMem<32> mem{state.data() + (size_t)tile * P.L.total_words * 32, lane};
    std::vector<uint32_t> sk(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    std::vector<uint16_t> sd(QMODE == 2 ? (size_t)P.L.queue_cap * 32 : 1);
    // (calendar queue: with the occupancy words in a stand-in for shared memory, as the sparse-tile kernels hold them)
    constexpr bool KS = QMODE == 3;
    std::vector<uint32_t> km(KS ? (size_t)((P.L.cal_times + 7) / 8) * 32 : 1);
    Core<TileMem<32>, NMAX, QMODE, FX, false, false, 1, false, false, KS> core(P, mem, zx, zf, P.delay_thr, sk.data() + lane, sd.data() + lane);
    core.km = km.data() + lane;
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
  }
}
static int run_impl(const lbft_config* c, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                    uint32_t* counters, uint32_t* status, uint32_t* words_per_instance, std::vector<uint32_t>& state,
                    Params& P, const int64_t* stops = nullptr, size_t nstops = 0, bool generic = false);

// The FX_DEFAULT4 instantiation (the compact node / slot encoding, Core::PACK) as run_all_fx runs it, and the generic one
// that the same layout takes without its compile-time shape (run_all_ep<16, 2, false, false, false>).
using PackedCore = Core<TileMem<32>, 16, 2, FX_DEFAULT4, false, false, 1, false, false, false>;
using GenericCore = Core<TileMem<32>, 16, 2, FX_NONE, false, false, 1, false, false, false>;
static_assert(PackedCore::PACK && !GenericCore::PACK, "the two encodings of the four-author layout");

// Words per (instance, node) of hostcore_final_state's decoded output: the F_NSCALAR scalars, vmask, tmask, tcmask, the
// timeout hcbr of authors 0..3 and the TC hcbr of authors 0..3.
constexpr uint32_t kDecodedWords = F_NSCALAR + 3 + 4 + 4;

// Node n of the instance in `mem`, read back through C's own accessors: node_ld for the scalars, load_node for the masks,
// hcbr_of on the node's timeout / TC hcbr vectors.  An hcbr entry is reported only for the authors of tmask / tcmask (0
// otherwise): the other entries are left over from earlier rounds by design and nothing reads them.
template <class C>
static void decode_node(C& core, uint32_t n, uint32_t* out) {
  const uint32_t b = core.nbase(n);
  for (uint32_t f = 0; f < F_NSCALAR; f++) out[f] = core.node_ld(b, f);
  typename C::NodeRegs d;
  core.win = 0;  // (the bitset word load_node speculates on: any valid index)
  core.load_node(n, d);
  out[F_NSCALAR] = (uint32_t)d.vmask;
  out[F_NSCALAR + 1] = (uint32_t)d.tmask;
  out[F_NSCALAR + 2] = (uint32_t)d.tcmask;
  const uint32_t th = C::PACK ? C::kPackedTimeoutHcbr : core.L.n_thcbr, tch = C::PACK ? C::kPackedTcHcbr : core.L.n_tchcbr;
  for (uint32_t a = 0; a < 4; a++) {
    out[F_NSCALAR + 3 + a] = ((d.tmask >> a) & 1) ? C::hcbr_of(core.m.at(b + th), a) : 0u;
    out[F_NSCALAR + 7 + a] = ((d.tcmask >> a) & 1) ? C::hcbr_of(core.m.at(b + tch), a) : 0u;
  }
}

static size_t read_round_switches(const Layout& L, const std::vector<uint32_t>& state, uint32_t num_nodes, uint32_t instance,
                                  lbft_round_switch* out, size_t cap) {
  const uint32_t row = L.round_cap + 1, tile = instance >> 5, lane = instance & 31;
  size_t k = 0;
  for (uint32_t node = 0; node < num_nodes; node++)
    for (uint32_t r = 1; r < row; r++) {  // slot 0 is the per-node maximum, not a switch
      const uint32_t w = state[((size_t)tile * L.total_words + rs_table_base(L) + (size_t)node * row + r) * 32 + lane];
      if (!w) continue;
      if (k < cap) out[k] = lbft_round_switch{node, r, (int64_t)(w - 1u)};
      k++;
    }
  return k;
}

// FNV-1a over a byte range; over a host table, its length and then its bytes (hostcore_setup_digest)
static uint64_t fnv1a(uint64_t h, const void* p, size_t n) {
  for (size_t i = 0; i < n; i++) h = (h ^ ((const uint8_t*)p)[i]) * 0x100000001b3ULL;
  return h;
}
template <class T>
static uint64_t fnv1a(uint64_t h, const std::vector<T>& v) {
  const uint64_t n = v.size();
  return fnv1a(fnv1a(h, &n, sizeof n), v.data(), n * sizeof(T));
}

extern "C" {
const char* hostcore_last_error(void) { return g_err.c_str(); }

// What the host setup decided for a configuration: [0] delay_kmax (0 = exp() fallback), [1] scan queue,
// [2] round_cap, [3] queue_cap, [4] payload_cap, [5] words per instance.
int hostcore_setup_info(const lbft_config* c, uint32_t* out6) {
  HostSetup hs;
  if (!hs.build(*c)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  out6[0] = hs.params.delay_kmax;
  out6[1] = hs.params.L.queue_scan;
  out6[2] = hs.params.L.round_cap;
  out6[3] = hs.params.L.queue_cap;
  out6[4] = hs.params.L.payload_cap;
  out6[5] = hs.params.L.total_words;
  return LBFT_OK;
}

// Which compile-time-layout instantiation (sim_params.h FX_*) hostcore_run takes for this configuration; 0 = generic.
int hostcore_fixed_shape(const lbft_config* c) {
  HostSetup hs;
  if (!hs.build(*c)) { g_err = hs.error; return -1; }
  return getenv("HOSTCORE_NO_FIXED") ? (int)FX_NONE : fixed_shape_of(hs.params);
}

// The product's lbft_kernel_info for this configuration: the kernel HostSetup selects (LBFT_FORCE_KERNEL included).
int hostcore_kernel_info(const lbft_config* c, char* buf, size_t cap) {
  HostSetup hs;
  if (!hs.build(*c)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  if (!buf || cap == 0) { g_err = "NULL argument"; return LBFT_ERR_INVALID; }
  snprintf(buf, cap, "%s", kernel_name(hs.sel).c_str());
  return LBFT_OK;
}

// One 64-bit digest (FNV-1a) of everything the host setup built for a configuration: the Params bytes before the device
// pointers, padding included, then each host table with its length.  *epochs receives Layout::epochs.
int hostcore_setup_digest(const lbft_config* c, uint64_t* digest, uint32_t* epochs) {
  HostSetup hs;
  if (!hs.build(*c)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  uint64_t h = fnv1a(0xcbf29ce484222325ULL, &hs.params, offsetof(Params, seeds));
  h = fnv1a(fnv1a(fnv1a(fnv1a(h, hs.zig_x), hs.zig_f), hs.leader), hs.duration);
  *digest = fnv1a(fnv1a(fnv1a(h, hs.period), hs.weights), hs.delay_thr);
  *epochs = hs.params.L.epochs;
  return LBFT_OK;
}

// Same outputs as the product's lbft_* getters; chain_out (optional) receives, per instance,
// round_cap * 2 words of the chain table and leader_out (optional) the leader table.
int hostcore_run(const lbft_config* c, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                 uint32_t* counters, uint32_t* status, uint32_t* words_per_instance) {
  std::vector<uint32_t> state;
  Params P;
  return run_impl(c, commit_counts, last_states, lc_round, counters, status, words_per_instance, state, P);
}

// Same contract as the product's lbft_round_switches (include/lbft.h): runs the batch with the configuration's
// flags (LBFT_FLAG_ROUND_SWITCHES required) and reads one instance's table out of the tile layout.
int hostcore_round_switches(const lbft_config* c, uint32_t instance, lbft_round_switch* out, size_t cap, size_t* n) {
  if (!(c->flags & LBFT_FLAG_ROUND_SWITCHES)) { g_err = "LBFT_FLAG_ROUND_SWITCHES not set"; return LBFT_ERR_STATE; }
  if (instance >= c->num_instances) { g_err = "instance out of range"; return LBFT_ERR_INVALID; }
  const size_t IN = (size_t)c->num_instances * c->num_nodes;
  std::vector<uint32_t> cc(IN), lc(IN), counters((size_t)c->num_instances * 12), status(c->num_instances), state;
  std::vector<uint64_t> ls(IN);
  Params P;
  int rc = run_impl(c, cc.data(), ls.data(), lc.data(), counters.data(), status.data(), nullptr, state, P);
  if (rc != LBFT_OK) return rc;
  if (n) *n = read_round_switches(P.L, state, c->num_nodes, instance, out, cap);
  return LBFT_OK;
}
// lbft_run_until called once per stop (LBFT_FLAG_RESUMABLE required); outputs describe the state at the last stop.
int hostcore_run_staged(const lbft_config* c, const int64_t* stops, size_t nstops, uint32_t* commit_counts,
                        uint64_t* last_states, uint32_t* lc_round, uint32_t* counters, uint32_t* status) {
  std::vector<uint32_t> state;
  Params P;
  return run_impl(c, commit_counts, last_states, lc_round, counters, status, nullptr, state, P, stops, nstops);
}

int hostcore_round_switches_staged(const lbft_config* c, uint32_t instance, const int64_t* stops, size_t nstops,
                                   lbft_round_switch* out, size_t cap, size_t* n) {
  if (!(c->flags & LBFT_FLAG_ROUND_SWITCHES)) { g_err = "LBFT_FLAG_ROUND_SWITCHES not set"; return LBFT_ERR_STATE; }
  if (instance >= c->num_instances) { g_err = "instance out of range"; return LBFT_ERR_INVALID; }
  const size_t IN = (size_t)c->num_instances * c->num_nodes;
  std::vector<uint32_t> cc(IN), lc(IN), counters((size_t)c->num_instances * 12), status(c->num_instances), state;
  std::vector<uint64_t> ls(IN);
  Params P;
  int rc = run_impl(c, cc.data(), ls.data(), lc.data(), counters.data(), status.data(), nullptr, state, P, stops, nstops);
  if (rc != LBFT_OK) return rc;
  if (n) *n = read_round_switches(P.L, state, c->num_nodes, instance, out, cap);
  return LBFT_OK;
}

// The compact encoding of FX_DEFAULT4 (sim_core.cuh Core::PACK) as the core defines it: [0] F_NSCALAR, [1] kPackedScalarWords,
// [2] kPackedWords, [3] kPackedTimeoutHcbr, [4] kPackedTcHcbr; then word, shift, mask of packed_field(f) for f = 0 ..
// F_NSCALAR + 2 (the scalars, then the vote / timeout / TC author masks); then the layout's node_base, node_words, n_hasblk,
// rset_words, created_base, qcmade_base, chain_base, round_cap, pay_base, pay_words, payload_cap, total_words.  Returns the
// number of words written, or -1 if `cap` is too small.
int hostcore_packed_fields(uint32_t* out, size_t cap) {
  constexpr Layout L = fixed_layout(FX_DEFAULT4);
  const uint32_t head[] = {F_NSCALAR, PackedCore::kPackedScalarWords, PackedCore::kPackedWords, PackedCore::kPackedTimeoutHcbr,
                           PackedCore::kPackedTcHcbr};
  const uint32_t tail[] = {L.node_base, L.node_words, L.n_hasblk, L.rset_words, L.created_base, L.qcmade_base, L.chain_base,
                           L.round_cap, L.pay_base, L.pay_words, L.payload_cap, L.total_words};
  const size_t need = 5 + 3 * (F_NSCALAR + 3) + 12;
  if (!out || cap < need) { g_err = "output too small"; return -1; }
  size_t k = 0;
  for (uint32_t v : head) out[k++] = v;
  for (uint32_t f = 0; f < F_NSCALAR + 3; f++) {
    const auto pf = PackedCore::packed_field(f);
    out[k++] = pf.word;
    out[k++] = pf.shift;
    out[k++] = pf.mask;
  }
  for (uint32_t v : tail) out[k++] = v;
  return (int)k;
}

// One node block through the compact encoding's writers and readers, in a tile of fixed_layout(FX_DEFAULT4).total_words x 32
// words that the caller has filled (`tile`, updated in place).  vals: the F_NSCALAR scalars, vmask, tmask, tcmask, the
// timeout hcbr of authors 0..3, the TC hcbr of authors 0..3.  Node `node` of lane `lane` is loaded (which leaves the bitset
// words clean), given the scalars and masks and stored; the TC hcbr goes in through put_timeout_hcbr and
// copy_timeout_hcbr_to_tc, then the timeout hcbr through put_timeout_hcbr.  out: the scalars and masks as load_node reads
// them back, the same through node_ld, the timeout hcbr and the TC hcbr through hcbr_of (62 words).
int hostcore_packed_roundtrip(const uint32_t* vals, uint32_t node, uint32_t lane, uint32_t* tile, uint32_t* out) {
  if (!vals || !tile || !out) { g_err = "NULL argument"; return LBFT_ERR_INVALID; }
  if (node >= 4 || lane >= 32) { g_err = "node or lane out of range"; return LBFT_ERR_INVALID; }
  const Params P{};
  PackedCore core(P, TileMem<32>{tile, lane}, nullptr, nullptr, nullptr);
  PackedCore::NodeRegs d;
  core.win = 0;  // (the bitset word load_node speculates on: any valid index)
  core.load_node(node, d);
  for (uint32_t f = 0; f < F_NSCALAR; f++) d.f[f] = vals[f];
  d.vmask = vals[F_NSCALAR];
  d.tmask = vals[F_NSCALAR + 1];
  d.tcmask = vals[F_NSCALAR + 2];
  core.store_node(d);
  for (uint32_t a = 0; a < 4; a++) core.put_timeout_hcbr(d, a, vals[F_NSCALAR + 7 + a]);
  core.copy_timeout_hcbr_to_tc(d);
  for (uint32_t a = 0; a < 4; a++) core.put_timeout_hcbr(d, a, vals[F_NSCALAR + 3 + a]);
  PackedCore::NodeRegs e;
  core.load_node(node, e);
  uint32_t k = 0;
  for (uint32_t f = 0; f < F_NSCALAR; f++) out[k++] = e.f[f];
  out[k++] = e.vmask;
  out[k++] = e.tmask;
  out[k++] = e.tcmask;
  const uint32_t b = core.nbase(node);
  for (uint32_t f = 0; f < F_NSCALAR + 3; f++) out[k++] = core.node_ld(b, f);
  for (uint32_t a = 0; a < 4; a++) out[k++] = PackedCore::hcbr_of(core.m.at(b + PackedCore::kPackedTimeoutHcbr), a);
  for (uint32_t a = 0; a < 4; a++) out[k++] = PackedCore::hcbr_of(core.m.at(b + PackedCore::kPackedTcHcbr), a);
  return LBFT_OK;
}

// A configuration of the FX_DEFAULT4 layout run through the compact-encoding instantiation (generic == 0) or the generic one
// on the same layout (generic == 1), in a state buffer filled with 0xdeadbeef.  The outputs are hostcore_run's; `decoded`
// (optional) receives kDecodedWords words per (instance, node) as decode_node reads them, and `raw` (optional) the state
// buffer: ceil(num_instances / 32) warp tiles of total_words x 32 words.
int hostcore_final_state(const lbft_config* c, int generic, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                         uint32_t* counters, uint32_t* status, uint32_t* decoded, uint32_t* raw) {
  HostSetup hs;
  if (!hs.build(*c)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  if (fixed_shape_of(hs.params) != FX_DEFAULT4) { g_err = "not the FX_DEFAULT4 layout"; return LBFT_ERR_INVALID; }
  if (!generic && getenv("HOSTCORE_NO_FIXED")) { g_err = "HOSTCORE_NO_FIXED is set: no compact-encoding run"; return LBFT_ERR_STATE; }
  std::vector<uint32_t> state;
  Params P;
  int rc = run_impl(c, commit_counts, last_states, lc_round, counters, status, nullptr, state, P, nullptr, 0, generic != 0);
  if (rc != LBFT_OK) return rc;
  for (uint32_t inst = 0; decoded && inst < c->num_instances; inst++) {
    const TileMem<32> mem{state.data() + (size_t)(inst / 32) * P.L.total_words * 32, inst % 32};
    for (uint32_t n = 0; n < 4; n++) {
      uint32_t* o = decoded + ((size_t)inst * 4 + n) * kDecodedWords;
      if (generic) {
        GenericCore core(P, mem, nullptr, nullptr, nullptr);
        decode_node(core, n, o);
      } else {
        PackedCore core(P, mem, nullptr, nullptr, nullptr);
        decode_node(core, n, o);
      }
    }
  }
  if (raw) memcpy(raw, state.data(), state.size() * sizeof(uint32_t));
  return LBFT_OK;
}
}  // extern "C"

static int run_impl(const lbft_config* c, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                    uint32_t* counters, uint32_t* status, uint32_t* words_per_instance, std::vector<uint32_t>& state,
                    Params& P, const int64_t* stops, size_t nstops, bool generic) {
  HostSetup hs;
  if (!hs.build(*c)) { g_err = hs.error; return LBFT_ERR_INVALID; }
  P = hs.params;
  P.seeds = c->seeds;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.leader = hs.leader.data();
  P.duration = hs.duration.data();
  P.period = hs.period.data();
  P.weights = hs.weights.data();
  P.delay_thr = hs.delay_thr.empty() ? nullptr : hs.delay_thr.data();
  uint32_t tiles = (c->num_instances + 31) / 32;
  state.assign((size_t)tiles * P.L.total_words * 32, 0xdeadbeefu);
  P.state = state.data();
  P.out_commit_counts = commit_counts;
  P.out_last_state = last_states;
  P.out_lc_round = lc_round;
  P.out_counters = counters;
  P.out_status = status;
  if (words_per_instance) *words_per_instance = P.L.total_words;
  if (stops && !P.resumable) { g_err = "LBFT_FLAG_RESUMABLE not set"; return LBFT_ERR_STATE; }
  const int64_t one_stop[1] = {P.max_clock};
  if (!stops) { stops = one_stop; nstops = 1; }
  // one launch per stop over the same state, like lbft_run_until
  for (size_t stage = 0; stage < nstops; stage++) {
    if (stops[stage] < 0 || stops[stage] > P.max_clock) { g_err = "stop_clock out of range"; return LBFT_ERR_INVALID; }
    P.stop_clock = (int32_t)stops[stage];
    P.run_flags = stage > 0 ? 1u : 0u;
#define RUN(NMAX, QS)                                                                                             \
  (P.resumable ? (P.record_rs ? run_all<NMAX, QS, true, true>(P, state, P.zig_x, P.zig_f)                           \
                              : run_all<NMAX, QS, false, true>(P, state, P.zig_x, P.zig_f))                          \
               : (P.record_rs ? run_all<NMAX, QS, true, false>(P, state, P.zig_x, P.zig_f)                          \
                              : run_all<NMAX, QS, false, false>(P, state, P.zig_x, P.zig_f)))
  const int fx = (generic || getenv("HOSTCORE_NO_FIXED")) ? (int)FX_NONE : fixed_shape_of(P);
  if (fx == FX_DEFAULT4) run_all_fx<16, 2, FX_DEFAULT4>(P, state, P.zig_x, P.zig_f);
  else if (fx == FX_PART7) run_all_fx<16, 3, FX_PART7>(P, state, P.zig_x, P.zig_f);
  else if (fx == FX_COMMITTEE64) run_all_fx<64, 3, FX_COMMITTEE64>(P, state, P.zig_x, P.zig_f);
  else if (P.L.queue_scan == 2) RUN(16, 2);
  else if (P.L.queue_scan == 1) RUN(16, 1);
  else if (P.L.queue_scan == 3) {
    if (c->num_nodes <= 16) RUN(16, 3);
    else if (c->num_nodes <= 32) RUN(32, 3);
    else RUN(64, 3);
  } else if (c->num_nodes <= 16) RUN(16, 0);
  else if (c->num_nodes <= 32) RUN(32, 0);
  else RUN(64, 0);
#undef RUN
  }
  return LBFT_OK;
}
