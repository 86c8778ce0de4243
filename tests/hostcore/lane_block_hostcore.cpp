// lane_block_hostcore.cpp — TEST INFRASTRUCTURE for the lane-block form of the compact encoding (sim_core.cuh TileMem LB): the
// FX_DEFAULT4 core the bench kernel and its commit-times twin run, with its node words and slots in lane blocks, compiled with
// g++ over the product's host setup, so that it can be compared with the lane-interleaved form hostcore.cpp runs.  Never part
// of, linked into, or reachable from the product library.
#include <cstring>
#include <string>
#include <vector>

#include "../../librabft_simulator_b200/csrc/host_setup.hpp"
#include "../../librabft_simulator_b200/csrc/sim_core.cuh"

using namespace lbft;
static thread_local std::string g_lb_err;

using LaneMem = TileMem<32, true>;
using LaneCore = Core<LaneMem, 16, 2, FX_DEFAULT4, false, false, 1, false, false, false>;
static_assert(LaneCore::PACK && LaneCore::PS == 1, "the compact encoding in lane blocks");

// Per (instance, node), as hostcore.cpp's decode_node: the F_NSCALAR scalars (node_ld), vmask, tmask, tcmask (load_node), the
// timeout and TC hcbr of authors 0..3 (hcbr_of; 0 for authors outside tmask / tcmask).
constexpr uint32_t kDecodedWords = F_NSCALAR + 3 + 4 + 4;
static void decode_node(LaneCore& core, uint32_t n, uint32_t* out) {
  const uint32_t b = core.nbase(n);
  for (uint32_t f = 0; f < F_NSCALAR; f++) out[f] = core.node_ld(b, f);
  LaneCore::NodeRegs d;
  core.win = 0;
  core.load_node(n, d);
  out[F_NSCALAR] = d.vmask;
  out[F_NSCALAR + 1] = d.tmask;
  out[F_NSCALAR + 2] = d.tcmask;
  for (uint32_t a = 0; a < 4; a++) {
    out[F_NSCALAR + 3 + a] = ((d.tmask >> a) & 1) ? LaneCore::hcbr_of(d.pk + LaneCore::kPackedTimeoutHcbr, a) : 0u;
    out[F_NSCALAR + 7 + a] = ((d.tcmask >> a) & 1) ? LaneCore::hcbr_of(d.pk + LaneCore::kPackedTcHcbr, a) : 0u;
  }
}

extern "C" {
const char* lane_block_last_error(void) { return g_lb_err.c_str(); }

// TileMem<32, true>::block_word: the tile offset of word k of `lane`'s block in the region of K-word blocks at word `base`.
uint64_t lane_block_word(uint32_t base, uint32_t K, uint32_t k, uint32_t lane) { return LaneMem::block_word(base, K, k, lane); }

// hostcore_packed_roundtrip (hostcore.cpp) through the lane-block core: the same values, writers, readers and 62 outputs.
int lane_block_roundtrip(const uint32_t* vals, uint32_t node, uint32_t lane, uint32_t* tile, uint32_t* out) {
  if (!vals || !tile || !out) { g_lb_err = "NULL argument"; return LBFT_ERR_INVALID; }
  if (node >= 4 || lane >= 32) { g_lb_err = "node or lane out of range"; return LBFT_ERR_INVALID; }
  const Params P{};
  LaneCore core(P, LaneMem{tile, lane}, nullptr, nullptr, nullptr);
  LaneCore::NodeRegs d;
  core.win = 0;
  core.load_node(node, d);
  for (uint32_t f = 0; f < F_NSCALAR; f++) d.f[f] = vals[f];
  d.vmask = vals[F_NSCALAR];
  d.tmask = vals[F_NSCALAR + 1];
  d.tcmask = vals[F_NSCALAR + 2];
  core.store_node(d);
  for (uint32_t a = 0; a < 4; a++) core.put_timeout_hcbr(d, a, vals[F_NSCALAR + 7 + a]);
  core.copy_timeout_hcbr_to_tc(d);
  for (uint32_t a = 0; a < 4; a++) core.put_timeout_hcbr(d, a, vals[F_NSCALAR + 3 + a]);
  LaneCore::NodeRegs e;
  core.load_node(node, e);
  uint32_t k = 0;
  for (uint32_t f = 0; f < F_NSCALAR; f++) out[k++] = e.f[f];
  out[k++] = e.vmask;
  out[k++] = e.tmask;
  out[k++] = e.tcmask;
  const uint32_t b = core.nbase(node);
  for (uint32_t f = 0; f < F_NSCALAR + 3; f++) out[k++] = core.node_ld(b, f);
  for (uint32_t a = 0; a < 4; a++) out[k++] = LaneCore::hcbr_of(core.pk_at(b) + LaneCore::kPackedTimeoutHcbr, a);
  for (uint32_t a = 0; a < 4; a++) out[k++] = LaneCore::hcbr_of(core.pk_at(b) + LaneCore::kPackedTcHcbr, a);
  return LBFT_OK;
}

// hostcore_final_state (hostcore.cpp, generic == 0) through the lane-block core: a configuration of the FX_DEFAULT4 layout in a
// state buffer filled with 0xdeadbeef; the outputs, `decoded` (kDecodedWords per instance and node, optional) and `raw`
// (the state buffer, optional).
int lane_block_final_state(const lbft_config* c, uint32_t* commit_counts, uint64_t* last_states, uint32_t* lc_round,
                           uint32_t* counters, uint32_t* status, uint32_t* decoded, uint32_t* raw) {
  HostSetup hs;
  if (!hs.build(*c)) { g_lb_err = hs.error; return LBFT_ERR_INVALID; }
  if (fixed_shape_of(hs.params) != FX_DEFAULT4) { g_lb_err = "not the FX_DEFAULT4 layout"; return LBFT_ERR_INVALID; }
  Params P = hs.params;
  P.seeds = c->seeds;
  P.zig_x = hs.zig_x.data();
  P.zig_f = hs.zig_f.data();
  P.leader = hs.leader.data();
  P.duration = hs.duration.data();
  P.period = hs.period.data();
  P.weights = hs.weights.data();
  P.delay_thr = hs.delay_thr.empty() ? nullptr : hs.delay_thr.data();
  std::vector<uint32_t> state((size_t)((c->num_instances + 31) / 32) * P.L.total_words * 32, 0xdeadbeefu);
  P.state = state.data();
  P.out_commit_counts = commit_counts;
  P.out_last_state = last_states;
  P.out_lc_round = lc_round;
  P.out_counters = counters;
  P.out_status = status;
  P.stop_clock = (int32_t)P.max_clock;
  P.run_flags = 0;
  for (uint32_t inst = 0; inst < c->num_instances; inst++) {
    const LaneMem mem{state.data() + (size_t)(inst / 32) * P.L.total_words * 32, inst % 32};
    std::vector<uint32_t> sk((size_t)P.L.queue_cap * 32);  // stands in for the shared-memory queue
    std::vector<uint16_t> sd((size_t)P.L.queue_cap * 32);
    LaneCore core(P, mem, P.zig_x, P.zig_f, P.delay_thr, sk.data() + mem.lane, sd.data() + mem.lane);
    core.init(P.seeds[inst]);
    core.run();
    core.finalize(inst);
  }
  for (uint32_t inst = 0; decoded && inst < c->num_instances; inst++) {
    LaneCore core(P, LaneMem{state.data() + (size_t)(inst / 32) * P.L.total_words * 32, inst % 32}, nullptr, nullptr, nullptr);
    for (uint32_t n = 0; n < 4; n++) decode_node(core, n, decoded + ((size_t)inst * 4 + n) * kDecodedWords);
  }
  if (raw) memcpy(raw, state.data(), state.size() * sizeof(uint32_t));
  return LBFT_OK;
}
}  // extern "C"
