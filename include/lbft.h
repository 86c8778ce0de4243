/* lbft.h — C ABI of the H100-native batched LibraBFTv2 discrete-event simulator.
 *
 * Drop-in boundary for the ONE hot path of novifinancial/librabft_simulator (reference checkout
 * /root/reference @ cc2ec64d): the discrete-event loop `Simulator::new` + `Simulator::loop_until`
 * (bft-lib/src/simulator.rs:200-250, 380-475) driving librabft-v2's NodeState / RecordStore /
 * Pacemaker / data-sync handlers over bft-lib's SimulatedContext.  The reference has no FFI seam
 * (it is generic Rust, simulator.rs:284-295); this header is the seam a Rust shim would bind with
 * `extern "C"` (see INTEGRATION.md).  One handle runs `num_instances` independent simulator
 * instances (instance i == `Simulator::new(seeds[i], num_nodes, RandomDelay::new(mean, variance),
 * context_factory)`) in lockstep on one GPU and exposes what the reference's callers read back:
 * `committed_history()` (simulated_context.rs:98-100) and `last_committed_state()` (:194-196).
 *
 * Conventions: plain C types only; every function returns LBFT_OK (0) or a negative error code and
 * never throws or aborts across the boundary; `lbft_last_error()` gives the thread-local message.
 * A handle is not thread-safe; distinct handles are independent.  There is NO CPU fallback: if no
 * CUDA device is usable, lbft_create fails with LBFT_ERR_CUDA.
 */
#ifndef LBFT_H_
#define LBFT_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LBFT_ABI_VERSION 1

enum {
  LBFT_OK = 0,
  LBFT_ERR_INVALID = -1,    /* bad argument / unsupported configuration                        */
  LBFT_ERR_CUDA = -2,       /* CUDA runtime error or no usable device                           */
  LBFT_ERR_STATE = -3,      /* call sequence error (e.g. results requested before lbft_run)     */
  LBFT_ERR_CAPACITY = -4,   /* some instance overflowed a device table; see lbft_status         */
  LBFT_ERR_NOMEM = -5
};

/* RandomDelay (simulator.rs:39-43, 99-118).  LOGNORMAL is the reference's only model.
 * UNIFORM is an extension (BASELINE.json config 2): integer uniform on [delay_lo, delay_hi]. */
enum { LBFT_DELAY_LOGNORMAL = 0, LBFT_DELAY_UNIFORM = 1 };

/* Per-instance status bits returned by lbft_status(). */
enum {
  LBFT_ST_DONE = 1u << 0,             /* event loop reached max_clock (or drained)               */
  LBFT_ST_ROUND_OVERFLOW = 1u << 1,   /* a round number reached round_cap                         */
  LBFT_ST_QUEUE_OVERFLOW = 1u << 2,   /* pending-event queue reached queue_cap                    */
  LBFT_ST_PAYLOAD_OVERFLOW = 1u << 3, /* in-flight notification pool reached payload_cap          */
  LBFT_ST_INVARIANT = 1u << 4,        /* a layout invariant (SURVEY App. C) was violated          */
  LBFT_ST_EPOCH_CHANGE = 1u << 5,     /* advisory: the instance went through an epoch change      */
                                      /* (commands_per_epoch reached, node.rs:329-348)            */
  LBFT_ST_DELAY_NEAR_INT = 1u << 6,   /* a LogNormal sample landed within 1e-9 of an integer: the */
                                      /* truncation may depend on the libm's last ulp (advisory)  */
  LBFT_ST_TIME_OVERFLOW = 1u << 7     /* a time left the 31-bit range of the device encoding      */
};
#define LBFT_ST_ERROR_MASK                                                                       \
  (LBFT_ST_ROUND_OVERFLOW | LBFT_ST_QUEUE_OVERFLOW | LBFT_ST_PAYLOAD_OVERFLOW | LBFT_ST_INVARIANT | \
   LBFT_ST_TIME_OVERFLOW)

/* One row of SimulatedContext::committed_history(): (Command{proposer,index}, NodeTime)
 * (simulated_context.rs:31-35, 98-100). */
typedef struct lbft_commit {
  uint32_t proposer;
  uint32_t index;
  int64_t time;
} lbft_commit;

/* One entry of DataWriter::nodes_round_switch (data_writer.rs:14, 34-50): at the pop of an event with
 * scheduled time `time`, node `node` was seen with ActiveRound::active_round() == `round`, larger than
 * at any earlier pop (simulator.rs:393-394: sampled after the max_clock test, before the clock max()). */
typedef struct lbft_round_switch {
  uint32_t node;
  uint32_t round;
  int64_t time;
} lbft_round_switch;

/* lbft_config.flags */
#define LBFT_FLAG_ROUND_SWITCHES 1u /* record round switches = loop_until(.., Some(csv_path)) simulator.rs:380-381 */
#define LBFT_FLAG_RESUMABLE 2u      /* lbft_run_until / snapshots: loop_until may be called again with a larger clock   */
/* NON-PARITY variant: a data-sync request is answered by the node it was SENT TO, from that node's records, and the requester
 * inserts the records of the response (what librabft-v2/src/data_sync.rs:183-240 is written for).  The reference simulator
 * dispatches the request to the requester itself (bft-lib/src/simulator.rs:446), which makes every round trip a no-op; that
 * behaviour is the default here, as its golden tests pin it.  Plain runs only (no other flag, commands_per_epoch >= round_cap). */
#define LBFT_FLAG_TRUE_DATA_SYNC 4u
/* Record commit latency: the global clock (Simulator.clock) at which each block is proposed and at which each node commits it,
 * read back with lbft_commit_times.  Plain and sweep handles; not with recording, resumable or true data-sync runs, nor with
 * commands_per_epoch < round_cap (LBFT_ERR_INVALID).  (Bit 8 is unassigned.) */
#define LBFT_FLAG_COMMIT_TIMES 16u

/* Per-instance event counters (simulator.rs:31 event_count; data_writer.rs message counter). */
typedef struct lbft_instance_counters {
  uint32_t processed[4];      /* popped events by Event::kind(): 0 notify 1 request 2 response 3 timer */
  uint32_t timers_cancelled;  /* timer pops skipped by ignore_scheduled_updates_until (:406-410)       */
  uint32_t scheduled;         /* Simulator.event_count: creation stamps handed out                     */
  uint32_t max_active_round;  /* max over nodes of ActiveRound::active_round() (simulator.rs:86-88)     */
  uint32_t rng_draws;         /* Xoshiro256** next_u64 calls on the instance stream                    */
  uint32_t max_queue;         /* high-water mark of the device event queue: the smallest queue_cap     *
                               * with which the instance completes (the read-out floor aside)         */
  uint32_t scheduled_notify;  /* DataSyncNotifyEvents handed a creation stamp (simulator.rs:348-354)    */
  uint32_t max_payloads;      /* high-water mark of in-flight notification snapshots: the smallest     *
                               * payload_cap with which the instance completes                        */
  uint32_t timers_elided;     /* duplicate timers accounted as cancelled without being queued (impl.)  */
} lbft_instance_counters;

/* Device timing of the last lbft_run / lbft_run_device, measured with CUDA events on the stream the
 * kernels are launched on. */
typedef struct lbft_timing {
  double init_ms;        /* state-initialisation kernel                         */
  double sim_ms;         /* event-loop kernel(s)                                */
  double finalize_ms;    /* read-out kernel (commit counts + state keys)        */
  double h2d_ms, d2h_ms; /* host<->device copies inside lbft_run                */
  uint64_t h2d_bytes, d2h_bytes;
  uint32_t kernel_launches; /* kernels launched by the last run                 */
  uint32_t reserved;
} lbft_timing;

/* Batched equivalent of the arguments of `Simulator::new` + `NodeConfig` + `SimulatedContext::new`
 * + `loop_until` (simulator.rs:200-208,380; node.rs:76-81; simulated_context.rs:86; main.rs:57-172). */
typedef struct lbft_config {
  uint32_t struct_size;   /* = sizeof(lbft_config); ABI guard                                          */
  uint32_t num_instances; /* independent simulator instances                                           */
  uint32_t num_nodes;     /* main.rs --nodes (1..64)                                                   */
  uint32_t delay_kind;    /* LBFT_DELAY_*                                                              */
  const uint64_t* seeds;  /* [num_instances] host pointer; main.rs --seed, simulator.rs:212            */
  int64_t max_clock;      /* loop_until(GlobalTime(max_clock)); main.rs --max_clock                    */
  double delay_mean;      /* RandomDelay::new(mean, variance), simulator.rs:99-106                     */
  double delay_variance;
  int64_t delay_lo, delay_hi;     /* LBFT_DELAY_UNIFORM only                                           */
  int64_t target_commit_interval; /* NodeConfig, node.rs:76-81                                         */
  int64_t delta;                  /* > 0 (delta = 0 is refused: SURVEY App. C.1b)                      */
  double gamma;
  double lambda;
  uint64_t commands_per_epoch;    /* SimulatedContext::new(_, _, max_command_per_epoch)                */
  /* ---- extensions (NULL / 0 = reference behaviour; SURVEY Appendix D) ---- */
  const uint64_t* voting_rights;  /* [num_nodes] EpochConfiguration weights (configuration.rs:29-43)   */
  const uint8_t* silent;          /* [num_nodes] non-zero = silent (crashed) node                      */
  uint32_t partition_windows;     /* per-instance random partition plan: number of windows             */
  uint32_t partition_max_len;     /* maximal window length in ms                                       */
  /* ---- device / capacity tuning (0 = auto) ---- */
  int32_t device;                 /* CUDA device ordinal                                               */
  uint32_t round_cap;             /* rounds representable per instance                                 */
  uint32_t queue_cap;             /* pending events per instance                                       */
  uint32_t payload_cap;           /* in-flight notifications per instance                              */
  uint32_t flags;                 /* LBFT_FLAG_* bits; unknown bits are rejected                       */
  uint32_t reserved;
} lbft_config;

typedef struct lbft_sim lbft_sim;

/* Validate the configuration, precompute the host tables (ziggurat layers, leader per round, round
 * durations — all libm calls stay on the host), allocate device state.  Does not run anything. */
int lbft_create(const lbft_config* config, lbft_sim** out_sim);

/* The per-instance part of lbft_config for a parameter sweep: the network delay (main.rs --mean / --variance, or the
 * uniform extension) and NodeConfig (--delta, --gamma, --lambda, --target_commit_interval). */
typedef struct lbft_param_set {
  uint32_t delay_kind;            /* LBFT_DELAY_*                                                      */
  uint32_t reserved;              /* 0                                                                 */
  double delay_mean, delay_variance;
  int64_t delay_lo, delay_hi;
  int64_t target_commit_interval, delta;
  double gamma, lambda;
} lbft_param_set;

/* A sweep handle: one batch whose instances run under num_sets parameter sets — instance i under
 * sets[set_of_instance[i]] — and share everything else of `config` (committee, voting rights, silent nodes, partition
 * plan, commands_per_epoch, max_clock, capacities, device); the delay / NodeConfig fields of `config` are ignored.
 * Every output of instance i is what lbft_create + lbft_run give it with that set's fields substituted into `config`
 * (as long as neither run reports LBFT_ERR_CAPACITY: the sweep's layout is the one the set with the shortest mean delay
 * would get).  Each set is validated like lbft_create validates those fields.  Refused (LBFT_ERR_INVALID, before any device
 * work): num_sets == 0 or > min(num_instances, 65536), NULL sets / set_of_instance, an index >= num_sets, any flags bit
 * but LBFT_FLAG_COMMIT_TIMES, and commands_per_epoch < round_cap (sweeps are plain single-epoch runs).  Every other entry point works on the handle
 * as on a plain one; lbft_set_seeds keeps the set assignment, and lbft_run_until / snapshots return LBFT_ERR_STATE. */
int lbft_create_sweep(const lbft_config* config, const lbft_param_set* sets, uint32_t num_sets,
                      const uint32_t* set_of_instance, lbft_sim** out_sim);

/* The fault model of one parameter set of a fault sweep: what lbft_config.silent / partition_windows / partition_max_len
 * give a plain handle. */
typedef struct lbft_fault_set {
  uint64_t silent_mask;           /* bit n: node n is silent (lbft_config.silent[n] != 0); bits >= num_nodes must be 0 */
  uint32_t partition_windows;     /* 0..64, as lbft_config.partition_windows                                        */
  uint32_t partition_max_len;     /* as lbft_config.partition_max_len                                               */
} lbft_fault_set;

/* A fault sweep: lbft_create_sweep with the fault model per parameter set as well.  Every output of instance i (but the
 * implementation counters max_queue / max_payloads / timers_elided, and runs with a capacity error) is what lbft_create +
 * lbft_run give it with sets[s] and faults[s] substituted into `config`, s = set_of_instance[i].  The layout and kernel are
 * what lbft_create_sweep picks with partition_windows set to the largest window count of any set.  Refused (LBFT_ERR_INVALID,
 * before any device work): whatever lbft_create_sweep refuses, NULL faults, a silent_mask bit >= num_nodes, a set whose
 * substituted configuration lbft_create refuses (the error names the set), and config->silent != NULL or non-zero
 * config->partition_windows / partition_max_len (a fault sweep takes its faults per set only).  Flags, and every other entry
 * point, as for lbft_create_sweep. */
int lbft_create_sweep_faults(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                             uint32_t num_sets, const uint32_t* set_of_instance, lbft_sim** out_sim);

/* A rights sweep: lbft_create_sweep / lbft_create_sweep_faults with the voting rights per parameter set as well.
 * voting_rights[s * num_nodes + n] is node n's voting right in set s.  faults may be NULL: then the configuration's shared
 * silent nodes / partition plan apply to every set, as in lbft_create_sweep; otherwise the rules of lbft_create_sweep_faults.
 * Every output of instance i (with the exceptions of lbft_create_sweep_faults) is what lbft_create + lbft_run give it with
 * sets[s], faults[s] (or the shared faults) and row s of voting_rights substituted into `config`, s = set_of_instance[i]; the
 * proposers of lbft_commit_log(s) and the state keys come from the set's own leaders.  The layout and kernel are what
 * lbft_create_sweep / lbft_create_sweep_faults pick for the same call: voting rights enter no kernel choice.  One leader table
 * of round_cap + 1 bytes is kept per distinct row (lbft_memory_info counts them).  Refused (LBFT_ERR_INVALID, before any device
 * work): whatever the corresponding sweep entry point refuses, NULL voting_rights, config->voting_rights != NULL (a rights sweep
 * takes its rights per set only), and a row with an entry above 2^24 or a total of 0 (the error names the set).  Every other
 * entry point as for a sweep; lbft_block_latency_stats / lbft_block_latency_stats_groups weigh each group with its set's rights. */
int lbft_create_sweep_rights(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                             const uint64_t* voting_rights, uint32_t num_sets, const uint32_t* set_of_instance,
                             lbft_sim** out_sim);

/* A committee sweep: lbft_create_sweep_rights with the committee size per parameter set as well.  config->num_nodes is the
 * layout's committee, and the stride of every per-node output; set s runs committee_sizes[s] (1..config->num_nodes) nodes.
 * voting_rights[s * num_nodes + n] is node n's voting right in set s, 0 for n >= committee_sizes[s]; voting_rights may be NULL:
 * then each node of a set's committee holds 1.  For its nodes 0..n_s-1 (n_s = committee_sizes[set_of_instance[i]]) every output
 * of instance i (with the exceptions of lbft_create_sweep_faults) is what lbft_create + lbft_run give it with num_nodes = n_s,
 * sets[s], faults[s] (or the shared faults) and row s of voting_rights truncated to n_s substituted into `config`.  Its other
 * nodes are absent: commit count, last committed round and state key 0, lbft_commit_logs length 0 and lbft_commit_log 0 rows,
 * lbft_commit_times entries -1.  The layout and kernel are what lbft_create_sweep_rights picks for the same call.  Refused
 * (LBFT_ERR_INVALID, before any device work; the error names the set): whatever lbft_create_sweep_rights refuses (but a NULL
 * voting_rights), NULL committee_sizes, a size of 0 or above num_nodes, a row with a non-zero entry at or past its set's size,
 * a silent node (a set's silent_mask bit, or with faults NULL a config->silent entry) at or past a set's size, and a set whose
 * substituted configuration lbft_create refuses.  lbft_block_latency_stats(_groups) weigh each group with its set's rights,
 * so "all" and "quorum" are per committee. */
int lbft_create_sweep_committees(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                                 const uint64_t* voting_rights, const uint32_t* committee_sizes, uint32_t num_sets,
                                 const uint32_t* set_of_instance, lbft_sim** out_sim);

/* A links sweep: the most general sweep, with a matrix of link latencies per parameter set as well.  link_latency[(s * N + a)
 * * N + b] (N = config->num_nodes, the layout's committee) is M_s[a][b], whole milliseconds in 0..65535: every network event
 * (notification, request, response) an instance of set s schedules from sender a to receiver b (the event's sender and receiver,
 * the pair its partition test looks at) is due at clock + delay + M_s[a][b], where delay is drawn from the set's delay model
 * exactly as without links.  The partition test, the silent-receiver elision and the drop past max_clock see that time.  The
 * startup delay of Simulator::new and the timers get no link term.  faults, voting_rights and committee_sizes may each be NULL;
 * the rules are those of lbft_create_sweep_faults, lbft_create_sweep_rights and lbft_create_sweep_committees, and where faults
 * or voting_rights is NULL the configuration's shared value applies to every set.  A set whose matrix is all zero computes what
 * the same set computes without links, counters included.  The layout and kernel are what the same call without link_latency
 * picks: the matrices enter no kernel choice.  Sets with equal matrices share one device table of N x N u16 (lbft_memory_info
 * counts them).  Refused (LBFT_ERR_INVALID, before any device work; the error names the set): whatever the corresponding sweep
 * refuses, NULL link_latency, an entry above 65535, and a non-zero entry in a row or column at or past the set's committee
 * size. */
int lbft_create_sweep_links(const lbft_config* config, const lbft_param_set* sets, const lbft_fault_set* faults,
                            const uint64_t* voting_rights, const uint32_t* committee_sizes, const uint32_t* link_latency,
                            uint32_t num_sets, const uint32_t* set_of_instance, lbft_sim** out_sim);

/* Simulator::new for every instance followed by loop_until(max_clock) (simulator.rs:200-250,
 * 380-475): copies the seeds host->device, runs the event-loop kernel to completion, copies the
 * per-node summaries (commit counts, last-committed-state keys, counters, status) device->host.
 * Returns LBFT_ERR_CAPACITY if any instance has a bit of LBFT_ST_ERROR_MASK set. */
int lbft_run(lbft_sim* sim);

/* Replace the seeds of the batch (a fresh `Simulator::new(seed, ..)` per instance on the next run);
 * `seeds` is a host array of num_instances entries, copied into the handle's pinned staging buffer. */
int lbft_set_seeds(lbft_sim* sim, const uint64_t* seeds);

/* The same three phases separately, for callers that keep inputs resident in HBM (bench.py `value`). */
int lbft_upload(lbft_sim* sim);     /* seeds host -> device                                  */
int lbft_run_device(lbft_sim* sim); /* init + event loop + read-out kernels, no host copies  */
int lbft_download(lbft_sim* sim);   /* summaries device -> host                              */

/* lbft_run split in two so that one host thread can drive several handles (one per GPU) at once and overlap its own
 * work with the device: lbft_run_async enqueues seeds host->device, the kernel and the summaries device->host on the
 * handle's stream and returns at once; lbft_wait blocks until they are done and reports like lbft_run
 * (lbft_run == lbft_run_async + lbft_wait).  Host staging is double-buffered: while a run is in flight the getters keep
 * serving the previous run's results, and lbft_set_seeds stages the next run's seeds without touching the buffer the
 * in-flight upload reads.  Every other entry point that touches the device returns LBFT_ERR_STATE until lbft_wait. */
int lbft_run_async(lbft_sim* sim);
int lbft_wait(lbft_sim* sim);

/* committed_history().len() per node (main.rs:47-53): out[instance * num_nodes + node]. */
int lbft_commit_counts(lbft_sim* sim, uint32_t* out);
/* last_committed_state() per node (simulated_context.rs:194-196): SipHash-1-3 key of the log. */
int lbft_last_states(lbft_sim* sim, uint64_t* out);
/* committed_history() of one node; writes min(*n, cap) rows, *n = full length. */
int lbft_commit_log(lbft_sim* sim, uint32_t instance, uint32_t node, lbft_commit* out, size_t cap, size_t* n);
/* committed_history() of EVERY context of the batch in one device pass and one copy (simulated_context.rs:98-100):
 * out[instance * cap + k], k < cap, is row k of the instance's longest log, and every node's committed_history() is
 * its first lens[instance * num_nodes + node] rows — the logs of one instance are prefixes of one chain because a
 * commit extends the previous one by exactly one block (simulated_context.rs:172-174); the device verifies it and
 * the call fails with LBFT_ERR_STATE if it does not hold for some instance (then read that instance with
 * lbft_commit_log).  Rows past a log's end are zero; logs longer than cap are truncated (lens tells).  lens may be
 * NULL. */
int lbft_commit_logs(lbft_sim* sim, lbft_commit* out, size_t cap, uint32_t* lens);
/* Commit latency of EVERY context of the batch (needs LBFT_FLAG_COMMIT_TIMES), aligned row for row with lbft_commit_logs and
 * read the same way (one device pass, one copy).  committed[(instance * num_nodes + node) * cap + k] is the global clock of
 * the event at which the node committed row k of its committed_history(); proposed[instance * cap + k] is the global clock
 * of the event at which row k of the instance's longest log was proposed (= the row's NodeTime + the proposer's startup
 * time).  Entries past a log's end (or past cap) are -1; proposed may be NULL.  LBFT_ERR_STATE without the flag, before a
 * run has finished, while an lbft_run_async is in flight, or when the logs of an instance are not prefixes of one chain;
 * LBFT_ERR_INVALID if cap is 0 or > 65535. */
int lbft_commit_times(lbft_sim* sim, int64_t* committed, int64_t* proposed, size_t cap);
/* Round switches of one instance (needs LBFT_FLAG_ROUND_SWITCHES, else LBFT_ERR_STATE): node-major,
 * rounds ascending within a node; writes min(*n, cap) rows, *n = full length.  Replaces the data behind
 * DataWriter::write_to_file's round_switches.txt (data_writer.rs:61-86); number_of_messages.txt is
 * processed[0] + processed[1] + processed[2] of lbft_counters. */
int lbft_round_switches(lbft_sim* sim, uint32_t instance, lbft_round_switch* out, size_t cap, size_t* n);
/* max over nodes of ActiveRound::active_round() per instance (simulator.rs:86-88): out[num_instances].  The same
 * number as lbft_instance_counters.max_active_round, without copying the whole counter table — it is the unit of
 * the throughput metric (simulated consensus rounds). */
int lbft_active_rounds(lbft_sim* sim, uint32_t* out);
/* Per-instance counters and status flags: out[num_instances]. */
int lbft_counters(lbft_sim* sim, lbft_instance_counters* out);
int lbft_status(lbft_sim* sim, uint32_t* out);
int lbft_timing_info(lbft_sim* sim, lbft_timing* out);
/* Name of the kernel instantiation this handle launches, spelled like the symbol ncu and cuobjdump show (the host picks
 * it from the configuration: committee size, horizon, capacities, flags); NUL-terminated, truncated to cap. */
int lbft_kernel_info(lbft_sim* sim, char* buf, size_t cap);
/* Bytes of device memory held by the handle, and the per-instance state footprint. */
int lbft_memory_info(lbft_sim* sim, uint64_t* device_bytes, uint32_t* words_per_instance);

/* Resumable runs (needs LBFT_FLAG_RESUMABLE, else LBFT_ERR_STATE).  lbft_config.max_clock is the FINAL horizon the
 * device tables are sized for; lbft_run_until(sim, t), 0 <= t <= max_clock, is loop_until(GlobalTime(t), ..)
 * (simulator.rs:380-475) on every instance: the first call is Simulator::new + loop_until, each later call continues
 * where the previous one stopped — including the reference's own exit behaviour: the first event beyond t is popped
 * and dropped (simulator.rs:383-391), so a staged run is NOT the same simulation as a one-shot run to the same
 * clock.  Results (all getters) describe the state at the stop.  lbft_run / lbft_upload / lbft_set_seeds start over. */
int lbft_run_until(lbft_sim* sim, int64_t stop_clock);
/* Checkpoint of the whole batch between two lbft_run_until calls (the batched analogue of
 * ConsensusNode::save_node / load_node, librabft-v2/src/node.rs:211-238, plus the simulator's own queue, clock and
 * RNG): save after a lbft_run_until, load into a handle created from the same configuration (verified by a digest;
 * LBFT_ERR_INVALID otherwise), then continue with lbft_run_until. */
int lbft_snapshot_size(lbft_sim* sim, size_t* bytes);
int lbft_snapshot_save(lbft_sim* sim, void* buf, size_t cap);
int lbft_snapshot_load(lbft_sim* sim, const void* buf, size_t bytes);

/* Device address of a result buffer, for callers that consume results on the GPU (e.g. an NCCL
 * all-gather of per-instance commit counts): which = 0 commit counts [I][N] u32, 1 last states [I][N]
 * u64, 2 counters [I][12] u32, 3 status [I] u32, 4 active rounds [I] u32, 5 = buffers 1, 0 and 4 as the one contiguous block they are
 * allocated in (last states, commit counts, active rounds — in this order): the summaries of a shard in a single collective.
 * Valid until lbft_destroy. */
int lbft_device_buffer(lbft_sim* sim, uint32_t which, void** device_ptr, size_t* bytes);

void lbft_destroy(lbft_sim* sim);
const char* lbft_last_error(void);
uint32_t lbft_abi_version(void);

/* Commit-latency statistics (lbft_latency_stats).  A sample is one latency committed - proposed of row k of node n's
 * committed_history(), with the times of lbft_commit_times; it counts when the row's proposed time p lies in
 * [proposed_from, proposed_until).  Bin b of a histogram counts latencies in [b * bin_width, (b + 1) * bin_width); the last
 * bin also counts every latency above it. */
typedef struct lbft_latency_spec {
  uint32_t struct_size;           /* = sizeof(lbft_latency_spec)                                       */
  uint32_t num_bins;              /* 1..65536                                                          */
  int64_t bin_width;              /* >= 1 (ms of global clock)                                         */
  int64_t proposed_from, proposed_until;  /* window on the proposed time, from <= until                */
} lbft_latency_spec;

/* One group's statistics: instances without an error bit, instances with one (LBFT_ST_ERROR_MASK: they add nothing), the
 * number of samples, their sum, and their minimum and maximum (-1 when samples == 0). */
typedef struct lbft_latency_summary {
  uint64_t instances, excluded, samples, sum;
  int64_t min, max;
} lbft_latency_summary;

/* Commit-latency statistics of the last run (needs LBFT_FLAG_COMMIT_TIMES), reduced on the device per group: a parameter set
 * of a sweep handle (num_sets groups, instance i in group set_of_instance[i]) or the whole batch of a plain handle (one
 * group).  out[num_groups]; hist[group * num_bins + b], or NULL (then not copied).  Every row of every log counts (there is no
 * cap), and every value is an exact integer that does not depend on launch shape.  The chain of an instance with an error
 * bit is not walked.  LBFT_ERR_STATE without the flag, before a run has finished, while an lbft_run_async is in flight, or
 * when the logs of an instance without an error bit are not prefixes of one chain; LBFT_ERR_INVALID for NULL sim / spec /
 * out, a wrong struct_size, num_bins outside 1..65536, bin_width < 1, proposed_from > proposed_until,
 * num_groups * num_bins > 2^24, or a handle whose num_instances * num_nodes * round_cap * max_clock does not fit in 64 bits
 * (the bound on sum). */
int lbft_latency_stats(lbft_sim* sim, const lbft_latency_spec* spec, lbft_latency_summary* out, uint64_t* hist);

/* Block-latency statistics at a voting-rights threshold (lbft_block_latency_stats).  The blocks of an instance are the rows k
 * of its longest log (the chain every log is a prefix of) whose proposed time p lies in [proposed_from, proposed_until); node n
 * has committed row k iff k < its commit count, at the time t_n of lbft_commit_times, and holds the voting right w_n
 * (lbft_config.voting_rights).  The threshold time of a block is the least t_n at which the voting rights of the nodes that
 * committed it at or before t_n sum to at least `threshold`; it does not depend on the order of ties.  A block has one sample,
 * T - p, or is unreached when the committed weight stays below the threshold to the end of the run.  Blocks that no node
 * committed are on no log and are not counted.  Common thresholds, with total the sum of the voting rights: 1 (the first node
 * to commit), (total + 2) / 3 (f + 1: a client can trust the block), 2 * total / 3 + 1 (a quorum), total (every node).
 *
 * Groups, exclusion of instances with an error bit, histogram bins, the window and the exactness of every value are those of
 * lbft_latency_stats: out[num_groups] (samples counts the reached blocks; sum / min / max / hist cover their latencies),
 * unreached[num_groups] the blocks that never reached the threshold, or NULL (then not copied), hist[group * num_bins + b] or
 * NULL.  Refusals: those of lbft_latency_stats, with its messages, and LBFT_ERR_INVALID for a threshold of 0 or above the
 * handle's total voting rights.  On a rights sweep (lbft_create_sweep_rights) each group is weighed with its set's voting
 * rights, and a threshold above any group's total is refused (the error names the group). */
int lbft_block_latency_stats(lbft_sim* sim, const lbft_latency_spec* spec, uint64_t threshold, lbft_latency_summary* out,
                             uint64_t* unreached, uint64_t* hist);

/* lbft_block_latency_stats with one threshold per group: thresholds[num_groups], each in 1..that group's total voting rights.
 * Works on every handle with LBFT_FLAG_COMMIT_TIMES (a plain handle has one group).  Everything else, refusals and their
 * messages included, is that of lbft_block_latency_stats; with the same threshold W for every group it returns what
 * lbft_block_latency_stats(W) returns. */
int lbft_block_latency_stats_groups(lbft_sim* sim, const lbft_latency_spec* spec, const uint64_t* thresholds,
                                    lbft_latency_summary* out, uint64_t* unreached, uint64_t* hist);

#ifdef __cplusplus
}
#endif
#endif /* LBFT_H_ */
