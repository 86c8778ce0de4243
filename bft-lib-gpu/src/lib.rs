//! `bft-lib-gpu` — the reference's simulator call shape over the H100 library.
//!
//! Replaces, for the LibraBFTv2 + `SimulatedContext` instantiation, `bft_lib::simulator::Simulator`
//! (bft-lib/src/simulator.rs:26-33): `Simulator::new(seed, nodes, RandomDelay::new(mean, variance), context_factory)`
//! (:200-208) and `loop_until(GlobalTime(max_clock), csv_path)` (:380).  The two call sites of the hot path,
//! librabft-v2/src/main.rs:36-53 and librabft-v2/tests/simulated_run.rs:19-43, switch to `GpuSimulator` and keep
//! reading `committed_history()` / `last_committed_state()` (bft-lib/src/simulated_context.rs:98-100, 194-196).
//!
//! `ffi` mirrors include/lbft.h item by item (checked by tests/test_rust_shim.py in this repository).
use std::os::raw::{c_char, c_int};

use bft_lib::base_types::NodeTime;
use bft_lib::simulated_context::{Author, Command, State};
use bft_lib::simulator::GlobalTime;
use librabft_v2::node::NodeConfig;

pub mod ffi {
    use super::{c_char, c_int};

    /// include/lbft.h `lbft_config`
    #[repr(C)]
    pub struct LbftConfig {
        pub struct_size: u32,
        pub num_instances: u32,
        pub num_nodes: u32,
        pub delay_kind: u32,
        pub seeds: *const u64,
        pub max_clock: i64,
        pub delay_mean: f64,
        pub delay_variance: f64,
        pub delay_lo: i64,
        pub delay_hi: i64,
        pub target_commit_interval: i64,
        pub delta: i64,
        pub gamma: f64,
        pub lambda: f64,
        pub commands_per_epoch: u64,
        pub voting_rights: *const u64,
        pub silent: *const u8,
        pub partition_windows: u32,
        pub partition_max_len: u32,
        pub device: i32,
        pub round_cap: u32,
        pub queue_cap: u32,
        pub payload_cap: u32,
        pub flags: u32,
        pub reserved: u32,
    }

    /// include/lbft.h `lbft_param_set`: one parameter set of a sweep handle (`lbft_create_sweep`) — the network delay
    /// and `NodeConfig` of the instances assigned to it
    #[repr(C)]
    #[derive(Clone, Copy, Default, Debug, PartialEq)]
    pub struct LbftParamSet {
        pub delay_kind: u32,
        pub reserved: u32,
        pub delay_mean: f64,
        pub delay_variance: f64,
        pub delay_lo: i64,
        pub delay_hi: i64,
        pub target_commit_interval: i64,
        pub delta: i64,
        pub gamma: f64,
        pub lambda: f64,
    }
    /// The header's spelling of `LbftParamSet`, as the `extern "C"` block names it.
    #[allow(non_camel_case_types)]
    pub type lbft_param_set = LbftParamSet;

    /// include/lbft.h `lbft_fault_set`: the fault model of one parameter set of a fault sweep (`lbft_create_sweep_faults`) —
    /// bit n of `silent_mask` makes node n silent; the partition plan as `LbftConfig::partition_windows` / `partition_max_len`
    #[repr(C)]
    #[derive(Clone, Copy, Default, Debug, PartialEq)]
    pub struct LbftFaultSet {
        pub silent_mask: u64,
        pub partition_windows: u32,
        pub partition_max_len: u32,
    }
    /// The header's spelling of `LbftFaultSet`, as the `extern "C"` block names it.
    #[allow(non_camel_case_types)]
    pub type lbft_fault_set = LbftFaultSet;

    /// include/lbft.h `lbft_commit`: one row of `committed_history()`
    #[repr(C)]
    #[derive(Clone, Copy, Default, Debug, PartialEq)]
    pub struct LbftCommit {
        pub proposer: u32,
        pub index: u32,
        pub time: i64,
    }

    /// include/lbft.h `lbft_round_switch`: one entry of `DataWriter::nodes_round_switch`
    #[repr(C)]
    #[derive(Clone, Copy, Default, Debug, PartialEq)]
    pub struct LbftRoundSwitch {
        pub node: u32,
        pub round: u32,
        pub time: i64,
    }

    /// include/lbft.h `lbft_instance_counters`
    #[repr(C)]
    #[derive(Clone, Copy, Default, Debug)]
    pub struct LbftInstanceCounters {
        pub processed: [u32; 4],
        pub timers_cancelled: u32,
        pub scheduled: u32,
        pub max_active_round: u32,
        pub rng_draws: u32,
        pub max_queue: u32,
        pub scheduled_notify: u32,
        pub max_payloads: u32,
        pub timers_elided: u32,
    }

    /// include/lbft.h `lbft_latency_spec`: the histogram and proposal-time window of `lbft_latency_stats`
    #[repr(C)]
    #[derive(Clone, Copy, Debug, PartialEq)]
    pub struct LbftLatencySpec {
        pub struct_size: u32,
        pub num_bins: u32,
        pub bin_width: i64,
        pub proposed_from: i64,
        pub proposed_until: i64,
    }
    /// The header's spelling of `LbftLatencySpec`, as the `extern "C"` block names it.
    #[allow(non_camel_case_types)]
    pub type lbft_latency_spec = LbftLatencySpec;

    /// include/lbft.h `lbft_latency_summary`: one group's commit-latency statistics (`min` / `max` are -1 when `samples == 0`)
    #[repr(C)]
    #[derive(Clone, Copy, Default, Debug, PartialEq)]
    pub struct LbftLatencySummary {
        pub instances: u64,
        pub excluded: u64,
        pub samples: u64,
        pub sum: u64,
        pub min: i64,
        pub max: i64,
    }
    /// The header's spelling of `LbftLatencySummary`, as the `extern "C"` block names it.
    #[allow(non_camel_case_types)]
    pub type lbft_latency_summary = LbftLatencySummary;

    pub const LBFT_OK: c_int = 0;
    pub const LBFT_ERR_CAPACITY: c_int = -4;
    pub const LBFT_FLAG_ROUND_SWITCHES: u32 = 1;
    pub const LBFT_FLAG_RESUMABLE: u32 = 2;
    pub const LBFT_FLAG_TRUE_DATA_SYNC: u32 = 4;
    pub const LBFT_FLAG_COMMIT_TIMES: u32 = 16;

    pub enum LbftSim {}

    #[link(name = "lbft_b200")]
    extern "C" {
        pub fn lbft_abi_version() -> u32;
        pub fn lbft_last_error() -> *const c_char;
        pub fn lbft_create(config: *const LbftConfig, out_sim: *mut *mut LbftSim) -> c_int;
        pub fn lbft_create_sweep(config: *const LbftConfig, sets: *const lbft_param_set, num_sets: u32, set_of_instance: *const u32,
                                 out_sim: *mut *mut LbftSim) -> c_int;
        pub fn lbft_create_sweep_faults(config: *const LbftConfig, sets: *const lbft_param_set, faults: *const lbft_fault_set, num_sets: u32,
                                        set_of_instance: *const u32, out_sim: *mut *mut LbftSim) -> c_int;
        pub fn lbft_create_sweep_rights(config: *const LbftConfig, sets: *const lbft_param_set, faults: *const lbft_fault_set,
                                        voting_rights: *const u64, num_sets: u32, set_of_instance: *const u32,
                                        out_sim: *mut *mut LbftSim) -> c_int;
        pub fn lbft_create_sweep_committees(config: *const LbftConfig, sets: *const lbft_param_set, faults: *const lbft_fault_set,
                                            voting_rights: *const u64, committee_sizes: *const u32, num_sets: u32,
                                            set_of_instance: *const u32, out_sim: *mut *mut LbftSim) -> c_int;
        pub fn lbft_create_sweep_links(config: *const LbftConfig, sets: *const lbft_param_set, faults: *const lbft_fault_set,
                                       voting_rights: *const u64, committee_sizes: *const u32, link_latency: *const u32,
                                       num_sets: u32, set_of_instance: *const u32, out_sim: *mut *mut LbftSim) -> c_int;
        pub fn lbft_destroy(sim: *mut LbftSim);
        pub fn lbft_set_seeds(sim: *mut LbftSim, seeds: *const u64) -> c_int;
        pub fn lbft_run(sim: *mut LbftSim) -> c_int;
        pub fn lbft_run_async(sim: *mut LbftSim) -> c_int;
        pub fn lbft_wait(sim: *mut LbftSim) -> c_int;
        pub fn lbft_run_until(sim: *mut LbftSim, stop_clock: i64) -> c_int;
        pub fn lbft_commit_counts(sim: *mut LbftSim, out: *mut u32) -> c_int;
        pub fn lbft_last_states(sim: *mut LbftSim, out: *mut u64) -> c_int;
        pub fn lbft_active_rounds(sim: *mut LbftSim, out: *mut u32) -> c_int;
        pub fn lbft_status(sim: *mut LbftSim, out: *mut u32) -> c_int;
        pub fn lbft_counters(sim: *mut LbftSim, out: *mut LbftInstanceCounters) -> c_int;
        pub fn lbft_commit_log(sim: *mut LbftSim, instance: u32, node: u32, out: *mut LbftCommit, cap: usize, n: *mut usize) -> c_int;
        pub fn lbft_commit_logs(sim: *mut LbftSim, out: *mut LbftCommit, cap: usize, lens: *mut u32) -> c_int;
        pub fn lbft_commit_times(sim: *mut LbftSim, committed: *mut i64, proposed: *mut i64, cap: usize) -> c_int;
        pub fn lbft_latency_stats(sim: *mut LbftSim, spec: *const lbft_latency_spec, out: *mut lbft_latency_summary, hist: *mut u64) -> c_int;
        pub fn lbft_block_latency_stats(sim: *mut LbftSim, spec: *const lbft_latency_spec, threshold: u64,
                                        out: *mut lbft_latency_summary, unreached: *mut u64, hist: *mut u64) -> c_int;
        pub fn lbft_block_latency_stats_groups(sim: *mut LbftSim, spec: *const lbft_latency_spec, thresholds: *const u64,
                                               out: *mut lbft_latency_summary, unreached: *mut u64, hist: *mut u64) -> c_int;
        pub fn lbft_round_switches(sim: *mut LbftSim, instance: u32, out: *mut LbftRoundSwitch, cap: usize, n: *mut usize) -> c_int;
        pub fn lbft_snapshot_size(sim: *mut LbftSim, bytes: *mut usize) -> c_int;
        pub fn lbft_snapshot_save(sim: *mut LbftSim, buf: *mut u8, cap: usize) -> c_int;
        pub fn lbft_snapshot_load(sim: *mut LbftSim, buf: *const u8, bytes: usize) -> c_int;
    }
}

fn last_error() -> String {
    unsafe { std::ffi::CStr::from_ptr(ffi::lbft_last_error()).to_string_lossy().into_owned() }
}

fn check(code: c_int, what: &str) {
    // the reference panics on its own invariant violations (simulated_context.rs:163-174, pacemaker.rs:118-121);
    // the library reports them as codes, and this shim turns them back into panics for its callers
    assert!(code == ffi::LBFT_OK, "{} failed with {}: {}", what, code, last_error());
}

/// What `loop_until` hands back per node: the two things the reference's callers read from `&SimulatedContext`.
pub struct ContextView {
    history: Vec<(Command, NodeTime)>,
    state: u64,
}

impl ContextView {
    /// `SimulatedContext::committed_history()` (simulated_context.rs:98-100)
    pub fn committed_history(&self) -> &Vec<(Command, NodeTime)> {
        &self.history
    }
    /// `StateFinalizer::last_committed_state()` (simulated_context.rs:194-196)
    pub fn last_committed_state(&self) -> State {
        State(self.state)
    }
}

/// One handle of the library per GPU; a batch is sharded contiguously over the handles (SURVEY §8e).
struct Shard {
    sim: *mut ffi::LbftSim,
    first: usize,
    count: usize,
}

/// Drop-in for `bft_lib::simulator::Simulator` (one seed) and its batched form (many seeds, one or several GPUs).
pub struct GpuSimulator {
    seeds: Vec<u64>,
    nodes: usize,
    mean: f64,
    variance: f64,
    config: NodeConfig,
    commands_per_epoch: usize,
    horizon: Option<i64>,
    devices: Vec<i32>,
    record_round_switches: bool,
    commit_times: bool,
    shards: Vec<Shard>,
}

impl GpuSimulator {
    /// `Simulator::new(rng_seed, num_nodes, RandomDelay::new(mean, variance), context_factory)` (simulator.rs:200-208).
    /// What the reference's `context_factory` closure captures (main.rs:23-34, simulated_run.rs:29-42) is passed as values.
    pub fn new(rng_seed: u64, num_nodes: usize, mean: f64, variance: f64, config: NodeConfig, commands_per_epoch: usize) -> Self {
        Self::new_batch(vec![rng_seed], num_nodes, mean, variance, config, commands_per_epoch)
    }

    /// One independent `Simulator` per seed, advanced in lockstep on the GPU.
    pub fn new_batch(seeds: Vec<u64>, num_nodes: usize, mean: f64, variance: f64, config: NodeConfig, commands_per_epoch: usize) -> Self {
        GpuSimulator {
            seeds,
            nodes: num_nodes,
            mean,
            variance,
            config,
            commands_per_epoch,
            horizon: None,
            devices: vec![0],
            record_round_switches: false,
            commit_times: false,
            shards: Vec::new(),
        }
    }

    /// Record when each block is proposed and when each node commits it (`LBFT_FLAG_COMMIT_TIMES`), for `latency_stats`.
    pub fn with_commit_times(mut self) -> Self {
        self.commit_times = true;
        self
    }

    /// Shard the batch over these CUDA devices (contiguous instance ranges, no data-path communication); one host
    /// thread drives them all through `lbft_run_async` / `lbft_wait`.
    pub fn on_devices(mut self, devices: Vec<i32>) -> Self {
        assert!(!devices.is_empty());
        self.devices = devices;
        self
    }

    /// For callers that call `loop_until` more than once on one simulator: `horizon` is the largest clock they will pass.
    pub fn with_horizon(mut self, horizon: GlobalTime) -> Self {
        self.horizon = Some(horizon.0);
        self
    }

    fn create(&mut self, max_clock: i64) {
        let world = self.devices.len().min(self.seeds.len()).max(1);
        for g in 0..world {
            let first = g * self.seeds.len() / world;
            let end = (g + 1) * self.seeds.len() / world;
            let mut flags = 0u32;
            if self.horizon.is_some() {
                flags |= ffi::LBFT_FLAG_RESUMABLE;
            }
            if self.record_round_switches {
                flags |= ffi::LBFT_FLAG_ROUND_SWITCHES;
            }
            if self.commit_times {
                flags |= ffi::LBFT_FLAG_COMMIT_TIMES;
            }
            let c = ffi::LbftConfig {
                struct_size: std::mem::size_of::<ffi::LbftConfig>() as u32,
                num_instances: (end - first) as u32,
                num_nodes: self.nodes as u32,
                delay_kind: 0,
                seeds: self.seeds[first..end].as_ptr(),
                max_clock: self.horizon.unwrap_or(max_clock),
                delay_mean: self.mean,
                delay_variance: self.variance,
                delay_lo: 0,
                delay_hi: 0,
                target_commit_interval: self.config.target_commit_interval.0,
                delta: self.config.delta.0,
                gamma: self.config.gamma,
                lambda: self.config.lambda,
                commands_per_epoch: self.commands_per_epoch as u64,
                voting_rights: std::ptr::null(),
                silent: std::ptr::null(),
                partition_windows: 0,
                partition_max_len: 0,
                device: self.devices[g],
                round_cap: 0,
                queue_cap: 0,
                payload_cap: 0,
                flags,
                reserved: 0,
            };
            let mut sim: *mut ffi::LbftSim = std::ptr::null_mut();
            check(unsafe { ffi::lbft_create(&c, &mut sim) }, "lbft_create");
            self.shards.push(Shard { sim, first, count: end - first });
        }
    }

    /// Run every instance to `max_clock` (`Simulator::new` + `loop_until` on the first call).
    fn run(&mut self, max_clock: i64) {
        if self.shards.is_empty() {
            self.create(max_clock);
        } else {
            assert!(self.horizon.is_some(), "loop_until called again: build the simulator with_horizon(..)");
        }
        if self.horizon.is_some() {
            for s in &self.shards {
                check(unsafe { ffi::lbft_run_until(s.sim, max_clock) }, "lbft_run_until");
            }
        } else {
            // all GPUs at once from this one thread
            for s in &self.shards {
                check(unsafe { ffi::lbft_run_async(s.sim) }, "lbft_run_async");
            }
            for s in &self.shards {
                check(unsafe { ffi::lbft_wait(s.sim) }, "lbft_wait");
            }
        }
    }

    /// `loop_until(GlobalTime(max_clock), None)` (simulator.rs:380) — the contexts of instance 0, as the reference's
    /// callers expect for a single simulator.
    pub fn loop_until(&mut self, max_clock: GlobalTime) -> Vec<ContextView> {
        self.run(max_clock.0);
        self.contexts(0)
    }

    /// Batched form: run, then `committed_history().len()` for every (instance, node) — what main.rs:47-53 prints.
    pub fn loop_until_batch(&mut self, max_clock: GlobalTime) -> Vec<Vec<usize>> {
        self.run(max_clock.0);
        let mut out = Vec::with_capacity(self.seeds.len());
        for s in &self.shards {
            let mut counts = vec![0u32; s.count * self.nodes];
            check(unsafe { ffi::lbft_commit_counts(s.sim, counts.as_mut_ptr()) }, "lbft_commit_counts");
            for i in 0..s.count {
                out.push(counts[i * self.nodes..(i + 1) * self.nodes].iter().map(|&c| c as usize).collect());
            }
        }
        out
    }

    fn shard_of(&self, instance: usize) -> (&Shard, usize) {
        let s = self.shards.iter().find(|s| instance >= s.first && instance < s.first + s.count).expect("instance out of range");
        (s, instance - s.first)
    }

    /// The `Vec<&Context>` of one instance of the batch.
    pub fn contexts(&self, instance: usize) -> Vec<ContextView> {
        let (s, local) = self.shard_of(instance);
        let mut states = vec![0u64; s.count * self.nodes];
        check(unsafe { ffi::lbft_last_states(s.sim, states.as_mut_ptr()) }, "lbft_last_states");
        (0..self.nodes)
            .map(|n| {
                let mut len = 0usize;
                check(unsafe { ffi::lbft_commit_log(s.sim, local as u32, n as u32, std::ptr::null_mut(), 0, &mut len) }, "lbft_commit_log");
                let mut buf = vec![ffi::LbftCommit::default(); len];
                check(unsafe { ffi::lbft_commit_log(s.sim, local as u32, n as u32, buf.as_mut_ptr(), len, &mut len) }, "lbft_commit_log");
                ContextView {
                    history: buf
                        .iter()
                        .map(|e| (Command { proposer: Author(e.proposer as usize), index: e.index as usize }, NodeTime(e.time)))
                        .collect(),
                    state: states[local * self.nodes + n],
                }
            })
            .collect()
    }

    /// Every commit log of the batch with one device pass and one copy per GPU (`lbft_commit_logs`): row k of
    /// `rows[instance]` is entry k of the instance's longest log; node n's `committed_history()` is its first
    /// `lens[instance][n]` rows.
    pub fn commit_logs(&self, cap: usize) -> (Vec<Vec<ffi::LbftCommit>>, Vec<Vec<u32>>) {
        let (mut rows, mut lens) = (Vec::new(), Vec::new());
        for s in &self.shards {
            let mut r = vec![ffi::LbftCommit::default(); s.count * cap];
            let mut l = vec![0u32; s.count * self.nodes];
            check(unsafe { ffi::lbft_commit_logs(s.sim, r.as_mut_ptr(), cap, l.as_mut_ptr()) }, "lbft_commit_logs");
            for i in 0..s.count {
                rows.push(r[i * cap..(i + 1) * cap].to_vec());
                lens.push(l[i * self.nodes..(i + 1) * self.nodes].to_vec());
            }
        }
        (rows, lens)
    }

    /// Commit-latency statistics of the whole batch (`lbft_latency_stats`; build the simulator `with_commit_times()`), reduced
    /// on each GPU and merged over them: the summary and `num_bins` histogram counts, bin b holding latencies in
    /// `[b * bin_width, (b + 1) * bin_width)` and the last bin everything above.  Only rows proposed in
    /// `[proposed_from, proposed_until)` count.
    pub fn latency_stats(&self, num_bins: u32, bin_width: i64, proposed_from: i64, proposed_until: i64) -> (ffi::LbftLatencySummary, Vec<u64>) {
        let spec = ffi::LbftLatencySpec {
            struct_size: std::mem::size_of::<ffi::LbftLatencySpec>() as u32,
            num_bins,
            bin_width,
            proposed_from,
            proposed_until,
        };
        let mut total = ffi::LbftLatencySummary { min: i64::MAX, max: -1, ..Default::default() };
        let mut hist = vec![0u64; num_bins as usize];
        for s in &self.shards {
            let mut part = ffi::LbftLatencySummary::default();
            let mut h = vec![0u64; num_bins as usize];
            check(unsafe { ffi::lbft_latency_stats(s.sim, &spec, &mut part, h.as_mut_ptr()) }, "lbft_latency_stats");
            total.instances += part.instances;
            total.excluded += part.excluded;
            total.samples += part.samples;
            total.sum += part.sum;
            if part.samples > 0 {
                total.min = total.min.min(part.min);
                total.max = total.max.max(part.max);
            }
            for (a, b) in hist.iter_mut().zip(h) {
                *a += b;
            }
        }
        if total.samples == 0 {
            total.min = -1;
        }
        (total, hist)
    }

    /// Block-latency statistics of the whole batch at a voting-rights threshold (`lbft_block_latency_stats`; build the
    /// simulator `with_commit_times()`), reduced on each GPU and merged over them: one sample per block of each instance's
    /// chain proposed in `[proposed_from, proposed_until)`, the time from its proposal until the nodes that committed it hold
    /// `threshold` voting rights (1 ..= the total; e.g. `2 * total / 3 + 1` for a quorum).  Returns the summary, the number
    /// of blocks that never reached the threshold, and the `num_bins` histogram counts.
    pub fn block_latency_stats(&self, threshold: u64, num_bins: u32, bin_width: i64, proposed_from: i64, proposed_until: i64)
                               -> (ffi::LbftLatencySummary, u64, Vec<u64>) {
        let spec = ffi::LbftLatencySpec {
            struct_size: std::mem::size_of::<ffi::LbftLatencySpec>() as u32,
            num_bins,
            bin_width,
            proposed_from,
            proposed_until,
        };
        let mut total = ffi::LbftLatencySummary { min: i64::MAX, max: -1, ..Default::default() };
        let mut unreached = 0u64;
        let mut hist = vec![0u64; num_bins as usize];
        for s in &self.shards {
            let mut part = ffi::LbftLatencySummary::default();
            let mut part_unreached = 0u64;
            let mut h = vec![0u64; num_bins as usize];
            check(unsafe { ffi::lbft_block_latency_stats(s.sim, &spec, threshold, &mut part, &mut part_unreached, h.as_mut_ptr()) },
                  "lbft_block_latency_stats");
            total.instances += part.instances;
            total.excluded += part.excluded;
            total.samples += part.samples;
            total.sum += part.sum;
            if part.samples > 0 {
                total.min = total.min.min(part.min);
                total.max = total.max.max(part.max);
            }
            unreached += part_unreached;
            for (a, b) in hist.iter_mut().zip(h) {
                *a += b;
            }
        }
        if total.samples == 0 {
            total.min = -1;
        }
        (total, unreached, hist)
    }
}

impl Drop for GpuSimulator {
    fn drop(&mut self) {
        for s in &self.shards {
            unsafe { ffi::lbft_destroy(s.sim) }
        }
    }
}
