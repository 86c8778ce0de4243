// lbft_api.cu — the C ABI of include/lbft.h over the sm_90a event-loop kernel.
//
// Replaces, for a whole batch of instances at once, the reference call sequence
//   Simulator::new(seed, nodes, RandomDelay::new(mean, variance), context_factory)   simulator.rs:200-250
//   sim.loop_until(GlobalTime(max_clock), None)                                      simulator.rs:380-475
//   contexts[i].committed_history() / last_committed_state()                         simulated_context.rs:98-100,194-196
// (callers: librabft-v2/src/main.rs:36-53, librabft-v2/tests/simulated_run.rs:19-94).
// There is no CPU fallback: without a usable CUDA device every entry point fails with LBFT_ERR_CUDA.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/lbft.h"
#include "host_setup.hpp"
#include "kernels.cuh"

using namespace lbft;

#define LBFT_SAME(a, b) ((uint32_t)(a) == (uint32_t)(b))
static_assert(LBFT_SAME(ST_DONE, LBFT_ST_DONE) && LBFT_SAME(ST_ROUND_OVERFLOW, LBFT_ST_ROUND_OVERFLOW) &&
                  LBFT_SAME(ST_QUEUE_OVERFLOW, LBFT_ST_QUEUE_OVERFLOW) && LBFT_SAME(ST_PAYLOAD_OVERFLOW, LBFT_ST_PAYLOAD_OVERFLOW) &&
                  LBFT_SAME(ST_INVARIANT, LBFT_ST_INVARIANT) && LBFT_SAME(ST_EPOCH_CHANGE, LBFT_ST_EPOCH_CHANGE) &&
                  LBFT_SAME(ST_DELAY_NEAR_INT, LBFT_ST_DELAY_NEAR_INT) && LBFT_SAME(ST_TIME_OVERFLOW, LBFT_ST_TIME_OVERFLOW),
              "status bits out of sync with include/lbft.h");
static_assert(sizeof(lbft_instance_counters) == 12 * sizeof(uint32_t), "counter layout");
static_assert(sizeof(lbft_latency_summary) == 6 * sizeof(uint64_t), "latency summary layout (64-bit atomics on every field)");
static_assert(LBFT_SAME(ST_ERROR_BITS, LBFT_ST_ERROR_MASK), "error mask out of sync with include/lbft.h");

// ---------------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static int set_error(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t e_ = (expr);                                                                             \
    if (e_ != cudaSuccess)                                                                               \
      return set_error(LBFT_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));             \
  } while (0)

// The owners of a handle's CUDA resources: each frees what it holds when it is destroyed.  Memory is the only code that
// allocates or frees the handle's memory: on the device (Pinned false) or pinned on the host (true).
template <bool Pinned>
class Memory {
 public:
  Memory() = default;
  Memory(const Memory&) = delete;
  Memory& operator=(const Memory&) = delete;
  ~Memory() { release(); }
  // Replaces what it holds by `bytes` of new memory; holds nothing when that fails.  A failed allocation is reported by the
  // return value alone: the runtime's record of it is cleared, so that the next launch's error check does not see it.
  cudaError_t alloc(size_t bytes) {
    release();
    void* p = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return e;
    }
    p_ = static_cast<unsigned char*>(p);
    bytes_ = bytes;
    return cudaSuccess;
  }
  size_t bytes() const { return bytes_; }
  template <class T = unsigned char>
  T* at(size_t offset = 0) const { return reinterpret_cast<T*>(p_ + offset); }

 private:
  void release() {
    if (Pinned) cudaFreeHost(p_);
    else cudaFree(p_);
    p_ = nullptr;
    bytes_ = 0;
  }
  unsigned char* p_ = nullptr;
  size_t bytes_ = 0;
};
using DeviceMemory = Memory<false>;
using PinnedMemory = Memory<true>;

// A stream or an event, created into `h` and destroyed with its owner.
template <class H, cudaError_t (*Destroy)(H)>
struct Owned {
  H h = nullptr;
  Owned() = default;
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() {
    if (h) Destroy(h);
  }
  operator H() const { return h; }
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;

// The per-run results, in the order of the outputs block and of its pinned host mirrors.  The first three regions are
// lbft_device_buffer(5) (include/lbft.h).  Only the first holds 8-byte words, so no region needs padding.
enum Output { OUT_LAST_STATE, OUT_COMMIT_COUNTS, OUT_ROUNDS, OUT_LC_ROUND, OUT_COUNTERS, OUT_STATUS, OUT_ERROR, OUT_END };
class OutputLayout {
 public:
  OutputLayout(size_t I = 0, size_t N = 0) {
    const size_t bytes[OUT_END] = {I * N * sizeof(uint64_t), I * N * sizeof(uint32_t), I * sizeof(uint32_t),
                                   I * N * sizeof(uint32_t), I * 12 * sizeof(uint32_t), I * sizeof(uint32_t),
                                   sizeof(uint32_t)};  // (error: the OR of the status words with an error bit)
    for (int r = 0; r < OUT_END; r++) at_[r + 1] = at_[r] + bytes[r];
  }
  size_t offset(Output r) const { return at_[r]; }
  size_t bytes(Output r) const { return at_[r + 1] - at_[r]; }
  size_t total() const { return at_[OUT_END]; }

 private:
  size_t at_[OUT_END + 1] = {};
};

struct lbft_sim {
  HostSetup hs;
  Params P{};  // its device pointers point into `inputs`, `state` and `outputs`
  int device = 0;
  uint32_t I = 0, N = 0;
  uint32_t stride = 32;  // instances per tile (the lane-interleaving factor of the state layout)
  Stream stream;
  Event ev[6];
  // Device memory counted in lbft_memory_info:
  //  * inputs: the seeds, then the launch-invariant tables (create_on_device);
  //  * outputs: the per-run results (regions);
  //  * state: the instance state, an allocation of its own, which the bench kernel's 128-bit lane-block accesses rely on;
  //  * times: LBFT_FLAG_COMMIT_TIMES' commit-time table [I][N + 1][round_cap] (sim_core.cuh Core CT), never cleared.
  DeviceMemory inputs, outputs, state, times;
  OutputLayout regions;
  const uint64_t* sets = nullptr;    // sweep handles only, in `inputs`: HostSetup::set_table
  const uint32_t* set_of = nullptr;  // sweep handles only, in `inputs`
  const uint16_t* links = nullptr;   // links sweeps only, in `inputs`: HostSetup::links
  const SweepOutage* outages = nullptr;  // outage sweeps only, in `inputs`: HostSetup::outages
  // the read-out buffers, allocated on first use and grown by grow_buffer
  DeviceMemory logs;       // lbft_commit_logs: [I][cap]
  DeviceMemory times_out;  // lbft_commit_times: [I][N][cap] committed, then [I][cap] proposed
  DeviceMemory lat;        // lbft_latency_stats / lbft_block_latency_stats: summaries, unreached counts and bins
  uint64_t device_bytes = 0;
  // pinned host staging: two seed buffers (lbft_set_seeds never writes the one an in-flight upload reads) and two mirrors
  // of `outputs` (an asynchronous run fills the one the getters are not reading, so the results of run k stay readable while
  // run k+1 is in flight: lbft_run_async / lbft_wait)
  PinnedMemory h_seeds[2];
  int seed_set = 0;        // buffer holding the most recently set seeds
  int seed_inflight = -1;  // buffer an in-flight upload is reading, -1 if none
  PinnedMemory res[2];
  int done = 0;            // result set the getters read
  bool pending = false;    // an lbft_run_async has not been waited for
  bool uploaded = false, ran = false, downloaded = false;
  bool started = false;     // resumable handles: a staged run is in progress, the next launch restores the instances
  int64_t next_stop = 0;    // stop clock of the next launch (max_clock unless set by lbft_run_until)
  int64_t last_stop = -1;   // stop clock of the last launch
  lbft_timing timing{};

  // The members free their resources after this, with the handle's device current.  (One process may drive several GPUs.)
  ~lbft_sim() {
    if (!stream) return;  // nothing was created on the device
    cudaSetDevice(device);
    cudaStreamSynchronize(stream);  // an lbft_run_async may still be in flight
  }
  // Allocates one of the four blocks above, counted in device_bytes.
  cudaError_t dev_alloc(DeviceMemory& m, size_t bytes) {
    const cudaError_t e = m.alloc(bytes);
    if (e == cudaSuccess) device_bytes += bytes;
    return e;
  }
  // Region r of the finished run's results, in the host mirror the getters read.
  template <class T>
  const T* result(Output r) const { return res[done].at<T>(regions.offset(r)); }
};

// The three phases of a run, enqueued on the handle's stream without waiting.
static int enqueue_upload(lbft_sim* s) {
  CUDA_TRY(cudaEventRecord(s->ev[0], s->stream));
  CUDA_TRY(cudaMemcpyAsync(s->inputs.at(), s->h_seeds[s->seed_set].at(), s->I * sizeof(uint64_t), cudaMemcpyHostToDevice, s->stream));
  CUDA_TRY(cudaEventRecord(s->ev[1], s->stream));
  s->seed_inflight = s->seed_set;
  return LBFT_OK;
}
static int enqueue_kernel(lbft_sim* s);
static int enqueue_download(lbft_sim* s, PinnedMemory& r) {
  CUDA_TRY(cudaEventRecord(s->ev[4], s->stream));
  CUDA_TRY(cudaMemcpyAsync(r.at(), s->outputs.at(), s->regions.total(), cudaMemcpyDeviceToHost, s->stream));
  CUDA_TRY(cudaEventRecord(s->ev[5], s->stream));
  return LBFT_OK;
}
// After the stream has drained: timings, and the one-word error check (the per-instance statuses are only scanned
// to name the first offender when the device-side OR says there is one).
static int finish_upload(lbft_sim* s) {
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, s->ev[0], s->ev[1]));
  s->timing.h2d_ms = ms;
  s->timing.h2d_bytes = s->I * sizeof(uint64_t);
  s->seed_inflight = -1;
  s->uploaded = true;
  return LBFT_OK;
}
static int finish_kernel(lbft_sim* s) {
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, s->ev[2], s->ev[3]));
  s->timing.init_ms = 0;
  s->timing.sim_ms = ms;
  s->timing.finalize_ms = 0;
  s->timing.kernel_launches = 1;
  s->ran = true;
  s->downloaded = false;
  s->started = s->P.resumable != 0;
  s->last_stop = s->P.stop_clock;
  return LBFT_OK;
}
static int finish_download(lbft_sim* s, int set) {
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, s->ev[4], s->ev[5]));
  s->timing.d2h_ms = ms;
  s->timing.d2h_bytes = s->regions.total();
  s->done = set;
  s->downloaded = true;
  const uint32_t* status = s->result<uint32_t>(OUT_STATUS);
  if (*s->result<uint32_t>(OUT_ERROR) & LBFT_ST_ERROR_MASK) {
    for (size_t i = 0; i < s->I; i++)
      if (status[i] & LBFT_ST_ERROR_MASK) {
        char buf[360];
        snprintf(buf, sizeof buf, "instance %zu ended with status 0x%x (see lbft_status; raise round_cap/queue_cap/payload_cap%s)", i,
                 status[i], (status[i] & LBFT_ST_QUEUE_OVERFLOW) ? "; QUEUE_OVERFLOW also means the queue mode ran out of creation "
                 "stamps: queue_cap > 512 selects a queue with wider stamps" : "");
        return set_error(LBFT_ERR_CAPACITY, buf);
      }
  }
  return LBFT_OK;
}
static int need_idle(lbft_sim* s) {
  if (!s) return set_error(LBFT_ERR_INVALID, "sim must not be NULL");
  if (s->pending) return set_error(LBFT_ERR_STATE, "an lbft_run_async is in flight: call lbft_wait first");
  return LBFT_OK;
}

static int create_on_device(std::unique_ptr<lbft_sim> s, const lbft_config* config, lbft_sim** out_sim);

// The body of the lbft_create* entry points: build(hs) fills the host setup of a new handle, or returns false with hs.error set;
// then the device half.  (The host tables can be large: a rights sweep keeps a leader table per distinct row of rights.)
template <class Build>
static int create_handle(const lbft_config* config, lbft_sim** out_sim, Build build) {
  if (!config || !out_sim) return set_error(LBFT_ERR_INVALID, "config and out_sim must not be NULL");
  *out_sim = nullptr;
  std::unique_ptr<lbft_sim> s(new (std::nothrow) lbft_sim());
  if (!s) return set_error(LBFT_ERR_NOMEM, "out of host memory");
  bool built = false;
  try {
    built = build(s->hs);
  } catch (const std::bad_alloc&) {
    return set_error(LBFT_ERR_NOMEM, "out of host memory for the handle's host tables");
  }
  if (!built) return set_error(LBFT_ERR_INVALID, s->hs.error);
  return create_on_device(std::move(s), config, out_sim);
}

extern "C" {

uint32_t lbft_abi_version(void) { return LBFT_ABI_VERSION; }
const char* lbft_last_error(void) { return g_last_error.c_str(); }

int lbft_create(const lbft_config* config, lbft_sim** out_sim) {
  return create_handle(config, out_sim, [&](HostSetup& hs) {
    if (!hs.build(*config)) return false;
    if (hs.params.L.epochs > 1 && (hs.params.record_rs || hs.params.resumable)) {
      hs.error = "recording / resumable handles need commands_per_epoch >= round_cap: the kernels with the epoch machinery "
                 "(node.rs:329-348) are built for plain runs only";
      return false;
    }
    return true;
  });
}

int lbft_create_sweep(const lbft_config* config, const lbft_param_set* sets, uint32_t num_sets, const uint32_t* set_of_instance,
                      lbft_sim** out_sim) {
  return create_handle(config, out_sim, [&](HostSetup& hs) { return hs.build_sweep(*config, sets, num_sets, set_of_instance); });
}

int lbft_create_sweep_faults(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults, uint32_t num_sets,
                             const uint32_t* set_of_instance, lbft_sim** out_sim) {
  return create_handle(config, out_sim,
                       [&](HostSetup& hs) { return hs.build_sweep_faults(*config, sets, faults, num_sets, set_of_instance); });
}

int lbft_create_sweep_rights(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                             const uint64_t* voting_rights, uint32_t num_sets, const uint32_t* set_of_instance, lbft_sim** out_sim) {
  return create_handle(config, out_sim,
                       [&](HostSetup& hs) { return hs.build_sweep_rights(*config, sets, faults, voting_rights, num_sets, set_of_instance); });
}

int lbft_create_sweep_committees(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                                 const uint64_t* voting_rights, const uint32_t* committee_sizes, uint32_t num_sets,
                                 const uint32_t* set_of_instance, lbft_sim** out_sim) {
  return create_handle(config, out_sim, [&](HostSetup& hs) {
    return hs.build_sweep_committees(*config, sets, faults, voting_rights, committee_sizes, num_sets, set_of_instance);
  });
}

int lbft_create_sweep_links(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                            const uint64_t* voting_rights, const uint32_t* committee_sizes, const uint32_t* link_latency,
                            uint32_t num_sets, const uint32_t* set_of_instance, lbft_sim** out_sim) {
  return create_handle(config, out_sim, [&](HostSetup& hs) {
    return hs.build_sweep_links(*config, sets, faults, voting_rights, committee_sizes, link_latency, num_sets, set_of_instance);
  });
}

int lbft_create_sweep_outages(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                              const uint64_t* voting_rights, const uint32_t* committee_sizes, const uint32_t* link_latency,
                              const lbft_outage* outages, uint32_t num_sets, const uint32_t* set_of_instance, lbft_sim** out_sim) {
  return create_handle(config, out_sim, [&](HostSetup& hs) {
    return hs.build_sweep_outages(*config, sets, faults, voting_rights, committee_sizes, link_latency, outages, num_sets,
                                  set_of_instance);
  });
}

}  // extern "C"

// The device half of the lbft_create* entry points, once the host setup `s->hs` is built.  On failure the partial handle is
// deleted, and its owners free what it holds.
static int create_on_device(std::unique_ptr<lbft_sim> s, const lbft_config* config, lbft_sim** out_sim) {
  s->I = config->num_instances;
  s->N = config->num_nodes;
  s->device = config->device;
  s->stride = (uint32_t)s->hs.sel.tile;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return set_error(LBFT_ERR_CUDA, std::string("no usable CUDA device (there is no CPU fallback): ") + cudaGetErrorString(e));
  if (s->device < 0 || s->device >= ndev) return set_error(LBFT_ERR_INVALID, "device ordinal out of range");
#define CREATE_TRY(expr)                                                                                         \
  do {                                                                                                           \
    cudaError_t e2_ = (expr);                                                                                    \
    if (e2_ != cudaSuccess)                                                                                      \
      return set_error(e2_ == cudaErrorMemoryAllocation ? LBFT_ERR_NOMEM : LBFT_ERR_CUDA,                        \
                       std::string(#expr) + ": " + cudaGetErrorString(e2_));                                     \
  } while (0)
  CREATE_TRY(cudaSetDevice(s->device));
  CREATE_TRY(cudaStreamCreateWithFlags(&s->stream.h, cudaStreamNonBlocking));
  for (auto& evt : s->ev) CREATE_TRY(cudaEventCreate(&evt.h));
  const HostSetup& hs = s->hs;
  const size_t I = s->I, N = s->N, tiles = (I + s->stride - 1) / s->stride;
  // The inputs block: the seeds (uploaded by every run), then the launch-invariant tables, uploaded here in one copy.  The
  // regions are ordered by element size, so none needs padding; a table that is empty has no region and a null pointer.
  const std::vector<uint64_t> set_table = hs.set_table();  // (empty on a plain handle)
  const size_t seeds_bytes = I * sizeof(uint64_t);
  std::vector<unsigned char> tables;
  auto stage = [&](const auto& v) {  // -> the region's offset in the block
    const size_t at = seeds_bytes + tables.size();
    const unsigned char* b = reinterpret_cast<const unsigned char*>(v.data());
    tables.insert(tables.end(), b, b + v.size() * sizeof(v[0]));
    return at;
  };
  const size_t zig_x = stage(hs.zig_x), zig_f = stage(hs.zig_f), delay_thr = stage(hs.delay_thr), sets = stage(set_table),
               outages = stage(hs.outages), duration = stage(hs.duration), period = stage(hs.period), weights = stage(hs.weights), set_of = stage(hs.set_of),
               links = stage(hs.links), leader = stage(hs.leader);
  CREATE_TRY(s->dev_alloc(s->inputs, seeds_bytes + tables.size()));
  CREATE_TRY(cudaMemcpy(s->inputs.at(seeds_bytes), tables.data(), tables.size(), cudaMemcpyHostToDevice));
  s->regions = OutputLayout(I, N);
  CREATE_TRY(s->dev_alloc(s->outputs, s->regions.total()));
  CREATE_TRY(s->dev_alloc(s->state, tiles * hs.params.L.total_words * s->stride * sizeof(uint32_t)));
  if (hs.sel.ct) CREATE_TRY(s->dev_alloc(s->times, I * (N + 1) * hs.params.L.round_cap * sizeof(int32_t)));
  for (int b = 0; b < 2; b++) {
    CREATE_TRY(s->h_seeds[b].alloc(seeds_bytes));
    CREATE_TRY(s->res[b].alloc(s->regions.total()));
  }
#undef CREATE_TRY
  memcpy(s->h_seeds[0].at(), config->seeds, seeds_bytes);
  Params& P = s->P;
  P = hs.params;
  const DeviceMemory& in = s->inputs;
  P.seeds = in.at<uint64_t>();
  P.zig_x = in.at<double>(zig_x);
  P.zig_f = in.at<double>(zig_f);
  P.delay_thr = hs.delay_thr.empty() ? nullptr : in.at<double>(delay_thr);
  P.duration = in.at<int32_t>(duration);
  P.period = in.at<int32_t>(period);
  P.weights = in.at<uint32_t>(weights);
  P.leader = in.at<uint8_t>(leader);
  if (!set_table.empty()) {
    s->sets = in.at<uint64_t>(sets);
    s->set_of = in.at<uint32_t>(set_of);
  }
  if (!hs.links.empty()) s->links = in.at<uint16_t>(links);
  if (!hs.outages.empty()) s->outages = in.at<SweepOutage>(outages);
  P.state = s->state.at<uint32_t>();
  const DeviceMemory& out = s->outputs;
  const OutputLayout& at = s->regions;
  P.out_last_state = out.at<uint64_t>(at.offset(OUT_LAST_STATE));
  P.out_commit_counts = out.at<uint32_t>(at.offset(OUT_COMMIT_COUNTS));
  P.out_rounds = out.at<uint32_t>(at.offset(OUT_ROUNDS));
  P.out_lc_round = out.at<uint32_t>(at.offset(OUT_LC_ROUND));
  P.out_counters = out.at<uint32_t>(at.offset(OUT_COUNTERS));
  P.out_status = out.at<uint32_t>(at.offset(OUT_STATUS));
  P.out_error = out.at<uint32_t>(at.offset(OUT_ERROR));
  *out_sim = s.release();
  return LBFT_OK;
}

extern "C" {

int lbft_set_seeds(lbft_sim* s, const uint64_t* seeds) {
  if (!s || !seeds) return set_error(LBFT_ERR_INVALID, "NULL argument");
  // never the buffer an in-flight upload is reading (lbft_run_async): the caller may stage run k+1 while run k runs
  const int b = s->seed_set != s->seed_inflight ? s->seed_set : 1 - s->seed_set;
  memcpy(s->h_seeds[b].at(), seeds, (size_t)s->I * sizeof(uint64_t));
  s->seed_set = b;
  s->uploaded = false;
  s->started = false;
  return LBFT_OK;
}

int lbft_device_buffer(lbft_sim* s, uint32_t which, void** device_ptr, size_t* bytes) {
  if (!s || !device_ptr || !bytes) return set_error(LBFT_ERR_INVALID, "NULL argument");
  if (which > 5) return set_error(LBFT_ERR_INVALID, "unknown buffer id");
  if (which == 5) {  // the first three regions
    *device_ptr = s->outputs.at();
    *bytes = s->regions.offset(OUT_LC_ROUND);
    return LBFT_OK;
  }
  static const Output ids[5] = {OUT_COMMIT_COUNTS, OUT_LAST_STATE, OUT_COUNTERS, OUT_STATUS, OUT_ROUNDS};
  const Output r = ids[which];
  *device_ptr = s->outputs.at(s->regions.offset(r));
  *bytes = s->regions.bytes(r);
  return LBFT_OK;
}

int lbft_upload(lbft_sim* s) {
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  if (int r = enqueue_upload(s)) return r;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  if (int r = finish_upload(s)) return r;
  s->started = false;  // fresh seeds: the next launch is Simulator::new
  s->next_stop = s->P.max_clock;
  return LBFT_OK;
}

int lbft_run_device(lbft_sim* s) {
  if (int r = need_idle(s)) return r;
  if (!s->uploaded) return set_error(LBFT_ERR_STATE, "lbft_upload must be called before lbft_run_device");
  CUDA_TRY(cudaSetDevice(s->device));
  if (int r = enqueue_kernel(s)) return r;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  return finish_kernel(s);
}

int lbft_download(lbft_sim* s) {
  if (int r = need_idle(s)) return r;
  if (!s->ran) return set_error(LBFT_ERR_STATE, "nothing has been run yet");
  CUDA_TRY(cudaSetDevice(s->device));
  const int set = 1 - s->done;
  if (int r = enqueue_download(s, s->res[set])) return r;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  return finish_download(s, set);
}

// lbft_run = lbft_run_async + lbft_wait.
int lbft_run_async(lbft_sim* s) {
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  s->next_stop = s->P.max_clock;
  s->started = false;
  if (int r = enqueue_upload(s)) return r;
  s->uploaded = true;
  if (int r = enqueue_kernel(s)) return r;
  if (int r = enqueue_download(s, s->res[1 - s->done])) return r;
  s->pending = true;
  return LBFT_OK;
}

int lbft_wait(lbft_sim* s) {
  if (!s) return set_error(LBFT_ERR_INVALID, "sim must not be NULL");
  if (!s->pending) return set_error(LBFT_ERR_STATE, "no lbft_run_async is in flight");
  CUDA_TRY(cudaSetDevice(s->device));
  s->pending = false;
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  if (int r = finish_upload(s)) return r;
  if (int r = finish_kernel(s)) return r;
  return finish_download(s, 1 - s->done);
}

int lbft_run(lbft_sim* s) {
  if (int r = lbft_run_async(s)) return r;
  return lbft_wait(s);
}

int lbft_run_until(lbft_sim* s, int64_t stop_clock) {
  if (int r = need_idle(s)) return r;
  if (!s->P.resumable) return set_error(LBFT_ERR_STATE, "not a resumable handle: set LBFT_FLAG_RESUMABLE in lbft_config.flags");
  if (stop_clock < 0 || stop_clock > s->P.max_clock)
    return set_error(LBFT_ERR_INVALID, "stop_clock must be in [0, lbft_config.max_clock] (the horizon the device tables are sized for)");
  if (!s->started) {
    int r = lbft_upload(s);  // Simulator::new on the next launch
    if (r != LBFT_OK) return r;
  }
  s->next_stop = stop_clock;
  int r = lbft_run_device(s);
  if (r != LBFT_OK) return r;
  return lbft_download(s);
}

}  // extern "C"

// A rights sweep's device table (lbft_create_sweep_rights), or null: the read-outs take each instance's leaders and weights from
// it, set g's entry at sweep_set_at(table, g, records) (a links sweep's entries carry their links record too).
static const SweepSet* rights_table(const lbft_sim* s) {
  return s->hs.rights.empty() ? nullptr : reinterpret_cast<const SweepSet*>(s->sets);
}
__device__ __forceinline__ const SweepRights& rights_of(const SweepSet* table, uint32_t g, uint32_t records) {
  return reinterpret_cast<const SweepSetRights*>(sweep_set_at(table, g, records))->rights;
}

static int enqueue_kernel(lbft_sim* s) {
  s->P.stop_clock = (int32_t)(s->P.resumable ? s->next_stop : (int64_t)s->P.max_clock);
  s->P.run_flags = (s->P.resumable && s->started) ? 1u : 0u;
  CUDA_TRY(cudaMemsetAsync(s->P.out_error, 0, sizeof(uint32_t), s->stream));
  CUDA_TRY(cudaEventRecord(s->ev[2], s->stream));
  const KernelSel& k = s->hs.sel;
  const uint32_t records = s->hs.records();
  const SweepParams sp{s->P,      s->set_of,  reinterpret_cast<const SweepSet*>(s->sets), records & 1u, (records >> 1) & 3u,
                       s->links, s->outages, s->hs.down_mask};
  const CtParams<Params> cp{s->P, s->times.at<int32_t>()};
  const CtParams<SweepParams> csp{sp, s->times.at<int32_t>()};
  cudaError_t e = k.ct ? (k.sweep ? (k.wide ? launch_ct_sweep_wide(k, csp, s->stream) : launch_ct_sweep_thread(k, csp, s->stream))
                                  : (k.wide ? launch_ct_wide(k, cp, s->stream) : launch_ct_thread(k, cp, s->stream)))
                  : k.sweep ? (k.wide ? launch_sweep_wide(k, sp, s->stream) : launch_sweep_thread(k, sp, s->stream))
                  : k.wide ? launch_wide(k, s->P, s->stream)
                  : k.fixed == FX_DEFAULT4 ? launch_fixed(k, s->P, s->stream)
                  : (k.qmode == 1 || k.qmode == 2) ? launch_scan(k, s->P, s->stream)
                  : k.qmode == 3 ? launch_calendar(k, s->P, s->stream)
                                 : launch_heap(k, s->P, s->stream);
  if (e != cudaSuccess) return set_error(LBFT_ERR_CUDA, std::string("kernel launch (") + kernel_name(k) + "): " + cudaGetErrorString(e));
  CUDA_TRY(cudaEventRecord(s->ev[3], s->stream));
  return LBFT_OK;
}

extern "C" {

// ---- snapshots: header + the state tiles (which hold the save areas of a resumable handle) ----
namespace {
struct SnapshotHeader {
  uint64_t magic;  // "LBFTSNP1"
  uint32_t abi, num_instances, num_nodes, total_words;
  int64_t max_clock, last_stop;
  uint64_t config_digest;
};
constexpr uint64_t kSnapMagic = 0x31504e535446424cULL;
uint64_t fnv1a(uint64_t h, const void* p, size_t n) {
  const unsigned char* b = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001b3ULL; }
  return h;
}
// Everything that shapes the simulation except the seeds: the scalar part of Params (layout, delay model, quorum,
// voting rights, ...) and the host tables.
uint64_t config_digest(const lbft_sim* s) {
  Params q = s->P;
  q.stop_clock = 0; q.run_flags = 0;
  uint64_t h = fnv1a(0xcbf29ce484222325ULL, &q, offsetof(Params, seeds));
  h = fnv1a(h, s->hs.leader.data(), s->hs.leader.size());
  h = fnv1a(h, s->hs.duration.data(), s->hs.duration.size() * sizeof(int32_t));
  h = fnv1a(h, s->hs.period.data(), s->hs.period.size() * sizeof(int32_t));
  if (!s->hs.delay_thr.empty()) h = fnv1a(h, s->hs.delay_thr.data(), s->hs.delay_thr.size() * sizeof(double));
  return h;
}
}  // namespace

int lbft_snapshot_size(lbft_sim* s, size_t* bytes) {
  if (!s || !bytes) return set_error(LBFT_ERR_INVALID, "NULL argument");
  if (!s->P.resumable) return set_error(LBFT_ERR_STATE, "not a resumable handle: set LBFT_FLAG_RESUMABLE in lbft_config.flags");
  *bytes = sizeof(SnapshotHeader) + s->state.bytes();
  return LBFT_OK;
}

int lbft_snapshot_save(lbft_sim* s, void* buf, size_t cap) {
  size_t need = 0;
  if (int r = lbft_snapshot_size(s, &need)) return r;
  if (!buf || cap < need) return set_error(LBFT_ERR_INVALID, "snapshot buffer too small (see lbft_snapshot_size)");
  if (!s->started) return set_error(LBFT_ERR_STATE, "nothing to snapshot: call lbft_run_until first");
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  SnapshotHeader h{kSnapMagic, LBFT_ABI_VERSION, s->I, s->N, s->P.L.total_words, s->P.max_clock, s->last_stop, config_digest(s)};
  memcpy(buf, &h, sizeof h);
  CUDA_TRY(cudaMemcpy(static_cast<char*>(buf) + sizeof h, s->P.state, s->state.bytes(), cudaMemcpyDeviceToHost));
  return LBFT_OK;
}

int lbft_snapshot_load(lbft_sim* s, const void* buf, size_t bytes) {
  size_t need = 0;
  if (int r = lbft_snapshot_size(s, &need)) return r;
  if (!buf || bytes < sizeof(SnapshotHeader)) return set_error(LBFT_ERR_INVALID, "not a snapshot");
  SnapshotHeader h;
  memcpy(&h, buf, sizeof h);
  if (h.magic != kSnapMagic || h.abi != LBFT_ABI_VERSION) return set_error(LBFT_ERR_INVALID, "not a snapshot of this library version");
  if (bytes != need || h.num_instances != s->I || h.num_nodes != s->N || h.total_words != s->P.L.total_words ||
      h.max_clock != s->P.max_clock || h.config_digest != config_digest(s))
    return set_error(LBFT_ERR_INVALID, "the snapshot was taken from a differently configured simulator");
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  CUDA_TRY(cudaMemcpy(s->P.state, static_cast<const char*>(buf) + sizeof h, s->state.bytes(), cudaMemcpyHostToDevice));
  s->started = true;   // the next lbft_run_until restores the instances from their save areas
  s->uploaded = true;  // the seeds are not needed any more
  s->ran = false;
  s->downloaded = false;
  s->last_stop = h.last_stop;
  return LBFT_OK;
}

static int need_results(lbft_sim* s, const void* out) {
  if (!s || !out) return set_error(LBFT_ERR_INVALID, "NULL argument");
  // (while an lbft_run_async is in flight the getters keep serving the previous run's results: they live in the
  // other set of host mirrors)
  if (!s->downloaded) return set_error(LBFT_ERR_STATE, "results are not available: call lbft_run (or lbft_download) first");
  return LBFT_OK;
}
// Copies region r of the finished run's results to `out`.
static int read_result(lbft_sim* s, Output r, void* out) {
  if (int e = need_results(s, out)) return e;
  memcpy(out, s->result<unsigned char>(r), s->regions.bytes(r));
  return LBFT_OK;
}
int lbft_commit_counts(lbft_sim* s, uint32_t* out) { return read_result(s, OUT_COMMIT_COUNTS, out); }
int lbft_last_states(lbft_sim* s, uint64_t* out) { return read_result(s, OUT_LAST_STATE, out); }
int lbft_counters(lbft_sim* s, lbft_instance_counters* out) { return read_result(s, OUT_COUNTERS, out); }
int lbft_active_rounds(lbft_sim* s, uint32_t* out) { return read_result(s, OUT_ROUNDS, out); }  // == counters' max_active_round
int lbft_status(lbft_sim* s, uint32_t* out) { return read_result(s, OUT_STATUS, out); }
int lbft_timing_info(lbft_sim* s, lbft_timing* out) {
  if (!s || !out) return set_error(LBFT_ERR_INVALID, "NULL argument");
  *out = s->timing;
  return LBFT_OK;
}
int lbft_kernel_info(lbft_sim* s, char* buf, size_t cap) {
  if (!s || !buf || cap == 0) return set_error(LBFT_ERR_INVALID, "NULL argument");
  snprintf(buf, cap, "%s", kernel_name(s->hs.sel).c_str());
  return LBFT_OK;
}
int lbft_memory_info(lbft_sim* s, uint64_t* device_bytes, uint32_t* words_per_instance) {
  if (!s) return set_error(LBFT_ERR_INVALID, "NULL argument");
  if (device_bytes) *device_bytes = s->device_bytes;
  if (words_per_instance) *words_per_instance = s->P.L.total_words;
  return LBFT_OK;
}

// committed_history() of one node: walk the instance's chain table backwards from the node's last
// committed round (every commit extends the previous one by exactly one block,
// simulated_context.rs:172-174, so the log is the ancestor chain of the last committed block).
int lbft_commit_log(lbft_sim* s, uint32_t instance, uint32_t node, lbft_commit* out, size_t cap, size_t* n) {
  if (!s || !n) return set_error(LBFT_ERR_INVALID, "NULL argument");
  if (!s->downloaded) return set_error(LBFT_ERR_STATE, "results are not available: call lbft_run first");
  if (instance >= s->I || node >= s->N) return set_error(LBFT_ERR_INVALID, "instance/node out of range");
  if (cap && !out) return set_error(LBFT_ERR_INVALID, "out must not be NULL when cap > 0");
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  const Layout& L = s->P.L;
  std::vector<uint32_t> chain(2 * (size_t)L.round_cap);
  const uint32_t S = s->stride, tile = instance / S, lane = instance % S;
  const uint32_t* src = s->P.state + ((size_t)tile * L.total_words + L.chain_base) * S + lane;
  CUDA_TRY(cudaMemcpy2D(chain.data(), sizeof(uint32_t), src, S * sizeof(uint32_t), sizeof(uint32_t), chain.size(), cudaMemcpyDeviceToHost));
  uint32_t lc = s->result<uint32_t>(OUT_LC_ROUND)[(size_t)instance * s->N + node];
  uint32_t count = s->result<uint32_t>(OUT_COMMIT_COUNTS)[(size_t)instance * s->N + node];
  // epochs > 1: the parent of an epoch's first block is the block whose state is the epoch's initial state
  std::vector<uint32_t> einit(L.epochs, 0);
  if (L.epochs > 1)
    CUDA_TRY(cudaMemcpy2D(einit.data(), sizeof(uint32_t), s->P.state + ((size_t)tile * L.total_words + L.einit_base) * S + lane,
                          S * sizeof(uint32_t), sizeof(uint32_t), L.epochs, cudaMemcpyDeviceToHost));
  std::vector<lbft_commit> log(count);
  const uint32_t leaders = rights_table(s) ? s->hs.rights[s->hs.set_of[instance]].leader_off : 0u;  // the instance's leader table
  uint32_t i = count;
  for (uint32_t r = lc; r != 0 && i > 0;) {
    if (r >= L.round_cap) return set_error(LBFT_ERR_STATE, "corrupt chain table");
    --i;
    log[i].proposer = s->hs.leader[leaders + r % L.rspan];
    log[i].index = chain[2 * r] >> 16;
    log[i].time = (int64_t)(int32_t)chain[2 * r + 1];
    const uint32_t p = chain[2 * r] & 0xffffu, e = r / L.rspan;
    r = p ? e * L.rspan + p : einit[e];
  }
  if (i != 0) return set_error(LBFT_ERR_STATE, "chain shorter than the commit count");
  *n = count;
  for (size_t k = 0; k < count && k < cap; k++) out[k] = log[k];
  return LBFT_OK;
}

}  // extern "C"

// A read-out buffer grown to at least `bytes` on first use (its contents are not kept); `label` names it in the error.
static int grow_buffer(DeviceMemory& buf, size_t bytes, const char* label) {
  if (bytes <= buf.bytes()) return LBFT_OK;
  cudaError_t e = buf.alloc(bytes);
  if (e != cudaSuccess) return set_error(LBFT_ERR_NOMEM, std::string(label) + ": " + cudaGetErrorString(e));
  return LBFT_OK;
}

// The end of a bulk read-out, once its copies are enqueued: waits for them and fails the call if the kernel counted, in
// out_error, instances whose node logs are not prefixes of one chain.
static int finish_chain_check(lbft_sim* s) {
  uint32_t bad = 0;
  CUDA_TRY(cudaMemcpyAsync(&bad, s->P.out_error, sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  if (!bad) return LBFT_OK;
  char buf[160];
  snprintf(buf, sizeof buf, "%u instance(s) have node logs that are not prefixes of one chain: read them with lbft_commit_log", bad);
  return set_error(LBFT_ERR_STATE, buf);
}

// ---------------------------------------------------------------------------------------------
// Bulk read-out of the commit logs: one device pass + one device->host copy for the whole batch
// (committed_history() of every context, simulated_context.rs:98-100; lbft_commit_log does one strided copy per
// (instance, node) and is meant for spot checks).
// Every commit extends the previous one by exactly one block (simulated_context.rs:172-174), so a node's log is the
// ancestor chain of its last committed block; the kernel lays out the LONGEST log of each instance in commit order
// (sim_core.cuh walk_commit_chain, which also verifies that every other node's last committed block lies on it at
// depth == its commit count, SURVEY App. C.3).  Instances where that does not hold are counted in *bad.
// The proposer of round r is leader(r) of the instance's leader table: on a rights sweep (`rights` not null) its set's.
// ---------------------------------------------------------------------------------------------
__global__ void lbft_commit_logs_kernel(const __grid_constant__ Params P, uint32_t stride, const uint32_t* set_of, const SweepSet* rights,
                                        uint32_t records, lbft_commit* out, uint32_t cap, uint32_t* bad) {
  const uint32_t inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= P.num_instances) return;
  const Layout& L = P.L;
  const uint32_t N = L.num_nodes, tile = inst / stride, lane = inst % stride;
  const uint32_t* tb = P.state + (size_t)tile * L.total_words * stride + lane;
  const uint8_t* leader = P.leader + (rights ? rights_of(rights, set_of[inst], records).leader_off : 0u);
  lbft_commit* row = out + (size_t)inst * cap;
  if (!walk_commit_chain(L, tb, stride, P.out_commit_counts + (size_t)inst * N, P.out_lc_round + (size_t)inst * N,
                         [&](uint32_t k, uint32_t r, uint32_t c0) {
                           if (k >= cap) return;
                           lbft_commit e;
                           e.proposer = leader[r % L.rspan];
                           e.index = c0 >> 16;
                           e.time = (int64_t)(int32_t)tb[(size_t)(L.chain_base + 2 * r + 1) * stride];
                           row[k] = e;
                         }))
    atomicAdd(bad, 1u);
}

int lbft_commit_logs(lbft_sim* s, lbft_commit* out, size_t cap, uint32_t* lens) {
  if (!s || !out || cap == 0) return set_error(LBFT_ERR_INVALID, "out must not be NULL and cap must be > 0");
  if (!s->downloaded) return set_error(LBFT_ERR_STATE, "results are not available: call lbft_run first");
  if (cap > 0xffffu) return set_error(LBFT_ERR_INVALID, "cap must be <= 65535 rows per instance");
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  const size_t bytes = (size_t)s->I * cap * sizeof(lbft_commit);
  if (int r = grow_buffer(s->logs, bytes, "commit-log buffer")) return r;
  // rows beyond a log's length are zero
  CUDA_TRY(cudaMemsetAsync(s->logs.at(), 0, bytes, s->stream));
  CUDA_TRY(cudaMemsetAsync(s->P.out_error, 0, sizeof(uint32_t), s->stream));
  lbft_commit_logs_kernel<<<(s->I + 127) / 128, 128, 0, s->stream>>>(s->P, s->stride, s->set_of, rights_table(s), s->hs.records(),
                                                                       s->logs.at<lbft_commit>(),
                                                                       (uint32_t)cap, s->P.out_error);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(out, s->logs.at(), bytes, cudaMemcpyDeviceToHost, s->stream));
  const int r = finish_chain_check(s);  // (the lengths are returned when the chain check fails too)
  if (lens && r != LBFT_ERR_CUDA) memcpy(lens, s->result<uint32_t>(OUT_COMMIT_COUNTS), s->regions.bytes(OUT_COMMIT_COUNTS));
  return r;
}

// Bulk read-out of the commit-time table (LBFT_FLAG_COMMIT_TIMES), aligned with lbft_commit_logs: one thread per instance
// walks its chain (sim_core.cuh commit_times_of).  Instances whose logs are not prefixes of one chain are counted in *bad.
__global__ void lbft_commit_times_kernel(const __grid_constant__ Params P, uint32_t stride, const int32_t* times, uint32_t cap,
                                         int64_t* committed, int64_t* proposed, uint32_t* bad) {
  const uint32_t inst = blockIdx.x * blockDim.x + threadIdx.x;
  if (inst >= P.num_instances) return;
  const Layout& L = P.L;
  const uint32_t N = L.num_nodes, tile = inst / stride, lane = inst % stride;
  if (!commit_times_of(L, P.state + (size_t)tile * L.total_words * stride + lane, stride, P.out_commit_counts + (size_t)inst * N,
                       P.out_lc_round + (size_t)inst * N, times + (size_t)inst * (N + 1) * L.round_cap, cap,
                       committed + (size_t)inst * N * cap, proposed + (size_t)inst * cap))
    atomicAdd(bad, 1u);
}

// lbft_latency_stats: the accumulators before the reduction — every field 0, min INT64_MAX (turned into -1 for an empty group on
// the host), max -1.
__global__ void lbft_latency_init_kernel(lbft_latency_summary* sum, uint32_t groups, unsigned long long* hist, size_t hist_len) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < hist_len || i < groups; i += (size_t)gridDim.x * blockDim.x) {
    if (i < groups) sum[i] = lbft_latency_summary{0, 0, 0, 0, INT64_MAX, -1};
    if (i < hist_len) hist[i] = 0;
  }
}

// The per-group reduction of both overloads of lbft_latency_stats_kernel, one object per thread: the instance it counts, the
// samples it adds, then the block's share of the totals (finish).  Integer atomics only, so every value is exact and
// independent of launch shape and atomic order.  The path is picked from what the block sees:
//  * all instances of the block in one group (a plain handle, or a sweep laid out set by set as SweepSimulator.grid does) and
//    num_bins <= kLatSharedBins: the histogram is built in shared memory (u32: a block holds at most 128 instances x 64 nodes x
//    32 768 rows = 2^28 samples) and added to the group's with one atomic per non-zero bin;
//  * otherwise every sample adds to its group's histogram in global memory.
// The summary fields are summed over each warp whose lanes share a group (shuffles, then one atomic per field), else per thread.
// kUnreached: the count of blocks that never reach the threshold, which only the threshold overload has (the per-sample one
// compiles no shuffle or atomic for it).
constexpr uint32_t kLatSharedBins = 8192;
constexpr uint32_t kLatBlock = 128;
extern __shared__ uint32_t lat_sh_bins[];
template <bool kUnreached>
struct LatencyReduction {
  int64_t width;
  uint32_t bins, g;          // g: the group of this thread's instance
  bool shared_hist;
  unsigned long long* gh;    // the group's histogram in global memory
  unsigned long long clean = 0, excluded = 0, samples = 0, total = 0, unreached = 0;
  long long lo = INT64_MAX, hi = -1;

  // Every thread of the block constructs one.  first: the block's first instance; inst: this thread's, live if in the batch.
  __device__ __forceinline__ LatencyReduction(const uint32_t* set_of, uint32_t first, uint32_t inst, bool live, int64_t width,
                                              uint32_t bins, unsigned long long* hist)
      : width(width), bins(bins) {
    const uint32_t g0 = set_of ? set_of[first] : 0u;
    g = live && set_of ? set_of[inst] : g0;
    gh = hist + (size_t)g * bins;  // (with shared_hist, the same for every thread: g == g0)
    shared_hist = __syncthreads_and(g == g0) && bins <= kLatSharedBins;
    if (shared_hist) {
      for (uint32_t b = threadIdx.x; b < bins; b += blockDim.x) lat_sh_bins[b] = 0;
      __syncthreads();
    }
  }
  // Counts a live instance as clean, or as excluded when its status has an error bit; lead: whether this thread counts it.
  // Returns whether its chain is walked.
  __device__ __forceinline__ bool admit(uint32_t status, bool lead) {
    if (status & ST_ERROR_BITS) {
      excluded = lead;
      return false;
    }
    clean = lead;
    return true;
  }
  __device__ __forceinline__ void add(int64_t lat) {
    samples++;
    total += (unsigned long long)lat;
    lo = lat < lo ? lat : lo;
    hi = lat > hi ? lat : hi;
    const uint32_t b = latency_bin(lat, width, bins);
    if (shared_hist) atomicAdd(&lat_sh_bins[b], 1u);
    else atomicAdd(&gh[b], 1ull);
  }
  // Every thread of the block calls this.  unreached_out: [groups], with kUnreached only.
  __device__ __forceinline__ void finish(lbft_latency_summary* sum, unsigned long long* unreached_out) {
    lbft_latency_summary* gs = sum + g;
    const uint32_t full = 0xffffffffu;
    if (__all_sync(full, g == __shfl_sync(full, g, 0))) {
      for (int o = 16; o > 0; o >>= 1) {
        clean += __shfl_down_sync(full, clean, o);
        excluded += __shfl_down_sync(full, excluded, o);
        samples += __shfl_down_sync(full, samples, o);
        total += __shfl_down_sync(full, total, o);
        if constexpr (kUnreached) unreached += __shfl_down_sync(full, unreached, o);
        lo = min(lo, __shfl_down_sync(full, lo, o));
        hi = max(hi, __shfl_down_sync(full, hi, o));
      }
      if ((threadIdx.x & 31) != 0) clean = excluded = samples = unreached = 0;  // (lane 0 holds the warp's totals)
    }
    if (clean) atomicAdd((unsigned long long*)&gs->instances, clean);
    if (excluded) atomicAdd((unsigned long long*)&gs->excluded, excluded);
    if constexpr (kUnreached)
      if (unreached) atomicAdd(&unreached_out[g], unreached);
    if (samples) {
      atomicAdd((unsigned long long*)&gs->samples, samples);
      atomicAdd((unsigned long long*)&gs->sum, total);
      atomicMin((long long*)&gs->min, lo);
      atomicMax((long long*)&gs->max, hi);
    }
    if (shared_hist) {
      __syncthreads();
      for (uint32_t b = threadIdx.x; b < bins; b += blockDim.x)
        if (lat_sh_bins[b]) atomicAdd(&gh[b], (unsigned long long)lat_sh_bins[b]);
    }
  }
};

// Per-group commit-latency statistics: one thread per instance walks its chain (sim_core.cuh latency_samples_of) unless its
// status has an error bit, and adds every sample.
__global__ void __launch_bounds__(kLatBlock) lbft_latency_stats_kernel(const __grid_constant__ Params P, uint32_t stride,
                                                                       const int32_t* times, const uint32_t* set_of, int64_t width,
                                                                       uint32_t bins, int64_t from, int64_t until,
                                                                       lbft_latency_summary* sum, unsigned long long* hist,
                                                                       uint32_t* bad) {
  const uint32_t inst = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = inst < P.num_instances;
  LatencyReduction<false> red(set_of, blockIdx.x * blockDim.x, inst, live, width, bins, hist);
  if (live && red.admit(P.out_status[inst], true)) {
    const Layout& L = P.L;
    const uint32_t N = L.num_nodes, tile = inst / stride, lane = inst % stride;
    if (!latency_samples_of(L, P.state + (size_t)tile * L.total_words * stride + lane, stride, P.out_commit_counts + (size_t)inst * N,
                            P.out_lc_round + (size_t)inst * N, times + (size_t)inst * (N + 1) * L.round_cap, from, until,
                            [&](int64_t lat) { red.add(lat); }))
      atomicAdd(bad, 1u);
  }
  red.finish(sum, nullptr);
}

// lbft_block_latency_stats / lbft_block_latency_stats_groups: per-group block-latency statistics at a voting-rights threshold
// W[g] per group g (sim_core.cuh block_latency_samples_of).  An overload of the per-sample kernel above: the same reduction over other samples, so tools that
// list the library's kernels by name see it as the latency reduction it is.  A group of G lanes per instance, G the smallest
// power of two >= min(N, 32), so lane j holds nodes j and, when N > 32, j + 32.  Every lane of the group walks the chain (same
// addresses: broadcast loads).  Per block, lane j loads its nodes' commit times (+inf where the node did not commit it) and
// sums, over G width-G shuffles under the group's mask, the voting rights (P.c_weights, or on a rights sweep its set's,
// indexed by the source lane) of the nodes with a time <= each of its own; the group then takes the least time whose sum reaches W (sim_core.cuh
// block_threshold_time_lanes: block_threshold_time without a per-node array), and lane 0 of the group accumulates the sample or
// the unreached block into the reduction of the per-sample kernel (LatencyReduction).
__global__ void __launch_bounds__(kLatBlock) lbft_latency_stats_kernel(const __grid_constant__ Params P, uint32_t stride,
                                                                       const int32_t* times, const uint32_t* set_of,
                                                                       const SweepSet* rights, uint32_t records, uint32_t G,
                                                                       const uint32_t* W,
                                                                       int64_t width, uint32_t bins,
                                                                       int64_t from, int64_t until, lbft_latency_summary* sum,
                                                                       unsigned long long* unreached_out,
                                                                       unsigned long long* hist, uint32_t* bad) {
  const uint32_t per_block = kLatBlock / G;
  const uint32_t j = threadIdx.x & (G - 1);  // the lane within the group
  const uint32_t inst = blockIdx.x * per_block + threadIdx.x / G;
  const bool live = inst < P.num_instances;
  LatencyReduction<true> red(set_of, blockIdx.x * per_block, inst, live, width, bins, hist);
  if (live && red.admit(P.out_status[inst], j == 0)) {
    const Layout& L = P.L;
    const uint32_t N = L.num_nodes, tile = inst / stride, lane = inst % stride;
    const uint32_t* cc = P.out_commit_counts + (size_t)inst * N;
    const int32_t* t_inst = times + (size_t)inst * (N + 1) * L.round_cap;
    const uint32_t warp_lane = threadIdx.x & 31;
    const uint32_t gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1u) << (warp_lane & ~(G - 1));
    const uint32_t n0 = j, n1 = j + 32;  // (n1 < N only when N > 32, i.e. G == 32)
    const uint32_t cc0 = n0 < N ? cc[n0] : 0u, cc1 = n1 < N ? cc[n1] : 0u;
    const uint32_t* w = rights ? rights_of(rights, red.g, records).weights : P.c_weights;  // (red.g: the instance's set on a sweep)
    const uint32_t Wg = W[red.g];
    auto time_of = [&](uint32_t k, uint32_t r) -> int64_t {
      return block_threshold_time_lanes(L, G, gmask, j, cc0, cc1, t_inst, w, k, r, Wg);
    };
    const bool ok = block_latency_samples_of(
        L, P.state + (size_t)tile * L.total_words * stride + lane, stride, cc, P.out_lc_round + (size_t)inst * N, t_inst, from, until,
        time_of,
        [&](int64_t lat) {
          if (j == 0) red.add(lat);
        },
        [&]() { red.unreached += j == 0; });
    if (!ok && j == 0) atomicAdd(bad, 1u);
  }
  red.finish(sum, unreached_out);
}

// The state checks of the read-outs of the commit-time table, after their NULL checks: the flag, then a finished run.
static int need_commit_times(lbft_sim* s) {
  if (!s->hs.sel.ct) return set_error(LBFT_ERR_STATE, "commit times were not recorded: set LBFT_FLAG_COMMIT_TIMES in lbft_config.flags");
  if (!s->downloaded) return set_error(LBFT_ERR_STATE, "results are not available: call lbft_run first");
  return LBFT_OK;
}

// lbft_latency_stats (thresholds NULL: the per-sample overload of lbft_latency_stats_kernel) and lbft_block_latency_stats /
// lbft_block_latency_stats_groups (the threshold overload, thresholds[groups]), once their arguments are checked.  The buffer
// holds [groups] summaries, [groups] unreached counts and the [groups][num_bins] bins, which lbft_latency_init_kernel sets in
// one pass, then the [groups] thresholds; unreached is NULL for a per-sample call.
static int latency_stats(lbft_sim* s, const lbft_latency_spec* spec, const uint64_t* thresholds, lbft_latency_summary* out,
                         uint64_t* unreached, uint64_t* hist) {
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  const uint32_t groups = latency_groups(s->hs), bins = spec->num_bins;
  const size_t hist_len = (size_t)groups * bins, counts_bytes = groups * sizeof(lbft_latency_summary) + (groups + hist_len) * sizeof(uint64_t);
  if (int r = grow_buffer(s->lat, counts_bytes + groups * sizeof(uint32_t), "latency-statistics buffer")) return r;
  lbft_latency_summary* d_sum = s->lat.at<lbft_latency_summary>();
  unsigned long long* d_unreached = s->lat.at<unsigned long long>(groups * sizeof(lbft_latency_summary));
  unsigned long long* d_hist = d_unreached + groups;
  uint32_t* d_thresholds = s->lat.at<uint32_t>(counts_bytes);
  const size_t init_blocks = (groups + hist_len + 255) / 256;
  lbft_latency_init_kernel<<<(unsigned)(init_blocks < 4096 ? init_blocks : 4096), 256, 0, s->stream>>>(d_sum, groups, d_unreached,
                                                                                                       groups + hist_len);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemsetAsync(s->P.out_error, 0, sizeof(uint32_t), s->stream));
  const uint32_t* set_of = s->hs.sel.sweep ? s->set_of : nullptr;
  const size_t smem = bins <= kLatSharedBins ? bins * sizeof(uint32_t) : 0;
  std::vector<uint32_t> W;  // (lives until finish_chain_check has synchronised the stream)
  if (!thresholds) {
    lbft_latency_stats_kernel<<<(s->I + kLatBlock - 1) / kLatBlock, kLatBlock, smem, s->stream>>>(
        s->P, s->stride, s->times.at<int32_t>(), set_of, spec->bin_width, bins, spec->proposed_from, spec->proposed_until, d_sum, d_hist,
        s->P.out_error);
  } else {
    uint32_t G = 1;  // lanes per instance: the smallest power of two >= min(N, 32)
    while (G < s->N && G < 32) G <<= 1;
    const uint32_t per_block = kLatBlock / G;
    W.assign(thresholds, thresholds + groups);  // (checked: each at most 64 * 2^24)
    CUDA_TRY(cudaMemcpyAsync(d_thresholds, W.data(), groups * sizeof(uint32_t), cudaMemcpyHostToDevice, s->stream));
    lbft_latency_stats_kernel<<<(s->I + per_block - 1) / per_block, kLatBlock, smem, s->stream>>>(
        s->P, s->stride, s->times.at<int32_t>(), set_of, rights_table(s), s->hs.records(), G, d_thresholds, spec->bin_width, bins, spec->proposed_from,
        spec->proposed_until, d_sum, d_unreached, d_hist, s->P.out_error);
  }
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(out, d_sum, groups * sizeof(lbft_latency_summary), cudaMemcpyDeviceToHost, s->stream));
  if (unreached) CUDA_TRY(cudaMemcpyAsync(unreached, d_unreached, groups * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
  if (hist) CUDA_TRY(cudaMemcpyAsync(hist, d_hist, hist_len * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
  if (int r = finish_chain_check(s)) return r;
  for (uint32_t g = 0; g < groups; g++)
    if (out[g].samples == 0) out[g].min = -1;
  return LBFT_OK;
}

extern "C" {

int lbft_commit_times(lbft_sim* s, int64_t* committed, int64_t* proposed, size_t cap) {
  if (!s || !committed) return set_error(LBFT_ERR_INVALID, "sim and committed must not be NULL");
  if (int r = need_commit_times(s)) return r;
  if (cap == 0 || cap > 0xffffu) return set_error(LBFT_ERR_INVALID, "cap must be in 1..65535 rows per instance");
  if (int r = need_idle(s)) return r;
  CUDA_TRY(cudaSetDevice(s->device));
  const size_t I = s->I, N = s->N;
  if (int r = grow_buffer(s->times_out, I * (N + 1) * cap * sizeof(int64_t), "commit-time buffer")) return r;
  int64_t* d_committed = s->times_out.at<int64_t>();
  int64_t* d_proposed = d_committed + I * N * cap;
  CUDA_TRY(cudaMemsetAsync(s->P.out_error, 0, sizeof(uint32_t), s->stream));
  lbft_commit_times_kernel<<<(s->I + 127) / 128, 128, 0, s->stream>>>(s->P, s->stride, s->times.at<int32_t>(), (uint32_t)cap, d_committed,
                                                                        d_proposed, s->P.out_error);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(committed, d_committed, I * N * cap * sizeof(int64_t), cudaMemcpyDeviceToHost, s->stream));
  if (proposed) CUDA_TRY(cudaMemcpyAsync(proposed, d_proposed, I * cap * sizeof(int64_t), cudaMemcpyDeviceToHost, s->stream));
  return finish_chain_check(s);
}

int lbft_latency_stats(lbft_sim* s, const lbft_latency_spec* spec, lbft_latency_summary* out, uint64_t* hist) {
  if (!s || !spec || !out) return set_error(LBFT_ERR_INVALID, "sim, spec and out must not be NULL");
  if (int r = need_commit_times(s)) return r;
  if (const char* e = latency_spec_error(s->hs, *spec)) return set_error(LBFT_ERR_INVALID, e);
  return latency_stats(s, spec, nullptr, out, nullptr, hist);
}

int lbft_block_latency_stats(lbft_sim* s, const lbft_latency_spec* spec, uint64_t threshold, lbft_latency_summary* out,
                             uint64_t* unreached, uint64_t* hist) {
  if (!s || !spec || !out) return set_error(LBFT_ERR_INVALID, "sim, spec and out must not be NULL");
  if (int r = need_commit_times(s)) return r;
  if (const char* e = latency_spec_error(s->hs, *spec)) return set_error(LBFT_ERR_INVALID, e);
  if (const char* e = block_latency_threshold_error(s->hs, threshold)) return set_error(LBFT_ERR_INVALID, e);
  const std::vector<uint64_t> thresholds(latency_groups(s->hs), threshold);
  return latency_stats(s, spec, thresholds.data(), out, unreached, hist);
}

int lbft_block_latency_stats_groups(lbft_sim* s, const lbft_latency_spec* spec, const uint64_t* thresholds, lbft_latency_summary* out,
                                    uint64_t* unreached, uint64_t* hist) {
  if (!s || !spec || !out || !thresholds) return set_error(LBFT_ERR_INVALID, "sim, spec, thresholds and out must not be NULL");
  if (int r = need_commit_times(s)) return r;
  if (const char* e = latency_spec_error(s->hs, *spec)) return set_error(LBFT_ERR_INVALID, e);
  if (const char* e = block_latency_thresholds_error(s->hs, thresholds)) return set_error(LBFT_ERR_INVALID, e);
  return latency_stats(s, spec, thresholds, out, unreached, hist);
}

int lbft_round_switches(lbft_sim* s, uint32_t instance, lbft_round_switch* out, size_t cap, size_t* n) {
  if (!s || !n) return set_error(LBFT_ERR_INVALID, "NULL argument");
  if (!s->P.record_rs) return set_error(LBFT_ERR_STATE, "round switches were not recorded: set LBFT_FLAG_ROUND_SWITCHES in lbft_config.flags");
  if (!s->downloaded) return set_error(LBFT_ERR_STATE, "results are not available: call lbft_run first");
  if (instance >= s->I) return set_error(LBFT_ERR_INVALID, "instance out of range");
  if (cap && !out) return set_error(LBFT_ERR_INVALID, "out must not be NULL when cap > 0");
  CUDA_TRY(cudaSetDevice(s->device));
  const Layout& L = s->P.L;
  const uint32_t row = L.round_cap + 1;
  std::vector<uint32_t> table((size_t)s->N * row);
  const uint32_t S = s->stride, tile = instance / S, lane = instance % S;
  const uint32_t* src = s->P.state + ((size_t)tile * L.total_words + rs_table_base(L)) * S + lane;
  CUDA_TRY(cudaMemcpy2D(table.data(), sizeof(uint32_t), src, S * sizeof(uint32_t), sizeof(uint32_t), table.size(), cudaMemcpyDeviceToHost));
  size_t k = 0;
  for (uint32_t node = 0; node < s->N; node++)
    for (uint32_t r = 1; r < row; r++) {  // slot 0 is the per-node maximum, not a switch
      const uint32_t w = table[(size_t)node * row + r];
      if (!w) continue;
      if (k < cap) out[k] = lbft_round_switch{node, r, (int64_t)(w - 1u)};
      k++;
    }
  *n = k;
  return LBFT_OK;
}

void lbft_destroy(lbft_sim* s) { delete s; }

}  // extern "C"
