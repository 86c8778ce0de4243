"""Host-side mirror of the reference's simulator interface over the C ABI.

Reference surface being mirrored (novifinancial/librabft_simulator):

* ``bft_lib::simulator::RandomDelay::new(mean, variance)``                     simulator.rs:99-106
* ``librabft_v2::node::NodeConfig {target_commit_interval, delta, gamma, lambda}``  node.rs:76-81
* ``bft_lib::simulator::Simulator::new(seed, num_nodes, delay, context_factory)``   simulator.rs:200-208
* ``Simulator::loop_until(GlobalTime(max_clock), csv_path) -> Vec<&Context>``       simulator.rs:380
* ``SimulatedContext::committed_history()`` / ``last_committed_state()``            simulated_context.rs:98-100,194-196

``BatchSimulator`` is the batched form (one handle = many independent ``Simulator`` instances, one per seed,
advanced in lockstep on one H100); ``Simulator`` is the single-instance spelling of the reference.  All the
simulation work happens in the CUDA library; this module only marshals arguments and results.
"""
import ctypes
import os
from dataclasses import dataclass
from fractions import Fraction

import numpy as np

from . import _lib

DELAY_LOGNORMAL, DELAY_UNIFORM = 0, 1
# one row of committed_history(): include/lbft.h lbft_commit
COMMIT_DTYPE = np.dtype([("proposer", np.uint32), ("index", np.uint32), ("time", np.int64)])
# one group's commit-latency statistics: include/lbft.h lbft_latency_summary
LATENCY_SUMMARY_DTYPE = np.dtype([("instances", np.uint64), ("excluded", np.uint64), ("samples", np.uint64), ("sum", np.uint64),
                                  ("min", np.int64), ("max", np.int64)])


class LatencyStats:
    """Commit-latency statistics per group (``BatchResult.latency_stats``), every value an exact integer: arrays
    ``instances`` (clean instances), ``excluded`` (instances with an error bit), ``samples``, ``sum``, ``min`` and ``max``
    (-1 for an empty group) of shape ``[groups]``, and ``hist[groups, num_bins]``, where bin b counts the latencies in
    ``[b * bin_width, (b + 1) * bin_width)`` and the last bin also every latency above it."""

    def __init__(self, summary, hist, bin_width):
        for f in LATENCY_SUMMARY_DTYPE.names:
            setattr(self, f, np.ascontiguousarray(summary[f]))
        self.hist = hist
        self.bin_width = int(bin_width)
        self.num_bins = hist.shape[1]

    def mean(self):
        """Mean latency per group (float64), nan where a group has no samples."""
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(self.samples > 0, self.sum.astype(np.float64) / self.samples, np.nan)

    def percentile(self, q):
        """The q-th percentile (0 <= q <= 100) per group: the lower edge ``b * bin_width`` of the first bin whose cumulative
        count reaches rank ``max(1, ceil(q * samples / 100))``, with the rank computed exactly; +inf when that bin is the
        last (it holds every latency above), nan for an empty group.  With ``bin_width = 1`` and an empty last bin this is
        ``np.percentile(latencies, q, method="inverted_cdf")``."""
        qf = Fraction(q)
        if not 0 <= qf <= 100:
            raise ValueError("q must be in [0, 100]")
        n = self.samples.astype(object)
        rank = np.maximum(1, -((-(n * qf.numerator)) // (100 * qf.denominator))).astype(np.uint64)  # ceil, in Python ints
        b = (np.cumsum(self.hist, axis=1) < rank[:, None]).sum(axis=1)
        out = b.astype(np.float64) * self.bin_width
        out[b >= self.num_bins - 1] = np.inf
        out[self.samples == 0] = np.nan
        return out


class BlockLatencyStats(LatencyStats):
    """Block-latency statistics per group at a voting-rights threshold (``BatchResult.block_latency_stats``): the fields of
    ``LatencyStats``, where a sample is one block's latency from its proposal to the time the nodes that committed it reach
    the group's threshold in voting rights, plus ``unreached[groups]``, the blocks that never reached it, the resolved integer
    ``thresholds[groups]``, and ``threshold``: their common value, or None when the groups' thresholds differ (a named
    threshold on a sweep whose sets carry different voting rights)."""

    def __init__(self, summary, unreached, hist, bin_width, threshold):
        super().__init__(summary, hist, bin_width)
        self.unreached = unreached
        t = np.asarray(threshold, dtype=np.int64).reshape(-1)
        self.thresholds = np.broadcast_to(t, (len(unreached),)).copy() if t.size == 1 else t
        self.threshold = int(t[0]) if (t == t[0]).all() else None


def resolve_threshold(threshold, total):
    """A threshold of ``block_latency_stats`` as an integer weight, with ``total`` the sum of the voting rights: an int as it
    is, or ``"first"`` (1), ``"validity"`` (f + 1: ``(total + 2) // 3``), ``"quorum"`` (``2 * total // 3 + 1``) or ``"all"``
    (``total``)."""
    if isinstance(threshold, str):
        names = {"first": 1, "validity": (total + 2) // 3, "quorum": 2 * total // 3 + 1, "all": total}
        if threshold not in names:
            raise ValueError("threshold must be an int or one of %s, not %r" % (", ".join(map(repr, names)), threshold))
        return names[threshold]
    return int(threshold)


@dataclass(frozen=True)
class RandomDelay:
    """``RandomDelay`` (simulator.rs:39-43).  ``new`` is the reference's LogNormal; ``uniform`` is an extension."""
    kind: int = DELAY_LOGNORMAL
    mean: float = 10.0
    variance: float = 4.0
    lo: int = 0
    hi: int = 0

    @staticmethod
    def new(mean, variance):
        return RandomDelay(DELAY_LOGNORMAL, float(mean), float(variance))

    @staticmethod
    def uniform(lo, hi):
        return RandomDelay(DELAY_UNIFORM, 0.0, 0.0, int(lo), int(hi))


@dataclass(frozen=True)
class NodeConfig:
    """``NodeConfig`` (node.rs:76-81) with the CLI defaults of main.rs:72-172."""
    target_commit_interval: int = 100000
    delta: int = 20
    gamma: float = 2.0
    lambda_: float = 0.5


@dataclass(frozen=True)
class GlobalTime:
    """``GlobalTime(i64)`` (simulator.rs:35-37)."""
    value: int

    def __int__(self):
        return int(self.value)


@dataclass(frozen=True)
class Command:
    """``Command {proposer, index}`` (simulated_context.rs:31-35)."""
    proposer: int
    index: int


class SimulatedContextView:
    """Read-only view of one node's ``SimulatedContext`` after the run (simulated_context.rs:74-100)."""

    def __init__(self, batch, instance, author):
        self._batch, self._instance, self.author = batch, instance, author

    def committed_history(self):
        """``committed_history()`` -> list of ``(Command, NodeTime)`` (simulated_context.rs:98-100)."""
        return [(Command(p, i), t) for (p, i, t) in self._batch.commit_log(self._instance, self.author)]

    def last_committed_state(self):
        """``StateFinalizer::last_committed_state()`` -> the ``State(u64)`` key (simulated_context.rs:194-196)."""
        return int(self._batch.last_committed_states[self._instance, self.author])

    def num_commits(self):
        return int(self._batch.commit_counts[self._instance, self.author])

    def commit_times(self):
        """Aligned with ``committed_history()``: ``(proposed, committed)`` global clocks per row — when the block was proposed
        and when this node committed it (needs ``commit_times=True``; include/lbft.h lbft_commit_times)."""
        n = self.num_commits()
        committed, proposed = self._batch.commit_times()  # (the whole batch once per result, shared by its contexts)
        return [(int(proposed[self._instance, k]), int(committed[self._instance, self.author, k])) for k in range(n)]


class BatchResult:
    """Results of ``BatchSimulator.loop_until``: what the reference's callers read from ``Vec<&Context>``.

    The summary arrays (commit counts, state keys, status, rounds) are copied out of the library's pinned result
    buffers when the result is created, so a ``BatchResult`` keeps describing ITS run after the handle has been
    re-run, re-seeded or closed.  Counters and commit logs are read on demand and are only available until the
    handle runs again (a stale read raises instead of returning another run's data)."""

    def __init__(self, sim):
        self._sim = sim
        self._generation = sim._generation
        I, N = sim.num_instances, sim.num_nodes
        #: ``committed_history().len()`` per node: [instance, node]
        self.commit_counts = sim._fetch("lbft_commit_counts", np.uint32, (I, N))
        #: ``last_committed_state()`` per node (SipHash-1-3 key of the commit log): [instance, node]
        self.last_committed_states = sim._fetch("lbft_last_states", np.uint64, (I, N))
        #: max over nodes of ``ActiveRound::active_round()`` per instance (simulator.rs:86-88)
        self.active_rounds = sim._fetch("lbft_active_rounds", np.uint32, (I,))
        self.status = sim._fetch("lbft_status", np.uint32, (I,))
        self._counters = None
        self._commit_times = {}  # cap -> (committed, proposed), read on first use

    @property
    def counters(self):
        """lbft_instance_counters per instance, [instance, 12] (fetched on first use; 48 bytes per instance)."""
        if self._counters is None:
            self._check_current("counters")
            self._counters = self._sim._fetch("lbft_counters", np.uint32, (self._sim.num_instances, 12))
        return self._counters

    def _check_current(self, what):
        if self._sim._handle is None or self._generation != self._sim._generation:
            raise RuntimeError("the %s of this result are gone: the simulator has been run again (or closed) since; read "
                               "them before the next run" % what)

    # lbft_instance_counters columns
    @property
    def events_processed(self):
        return self.counters[:, 0:4].sum(axis=1)

    def commit_log(self, instance, author):
        self._check_current("commit logs")
        return self._sim.commit_log(instance, author)

    def commit_logs(self, cap=None):
        """All commit logs of the batch in one device pass (``lbft_commit_logs``): ``(rows[instance, cap], lens[instance,
        node])``; node n's ``committed_history()`` is ``rows[instance, :lens[instance, n]]``."""
        self._check_current("commit logs")
        return self._sim.commit_logs(cap)

    def commit_times(self, cap=None):
        """Commit latency of the whole batch in one device pass (``lbft_commit_times``; needs ``commit_times=True``):
        ``(committed[instance, node, cap], proposed[instance, cap])`` as int64 global clocks, aligned row for row with
        ``commit_logs(cap)`` — ``committed[i, n, k]`` is when node n committed row k of its ``committed_history()``,
        ``proposed[i, k]`` when row k of the instance's longest log was proposed; -1 past each log's end.  ``cap`` defaults to
        the longest log of the batch.  Read from the handle once per ``cap``; the arrays are shared, do not modify them."""
        cap = max(1, int(self.commit_counts.max())) if cap is None else int(cap)
        if cap not in self._commit_times:
            self._check_current("commit times")
            self._commit_times[cap] = self._sim.commit_times(cap)
        return self._commit_times[cap]

    def commit_latencies(self, cap=None):
        """``committed - proposed`` per ``[instance, node, row]`` (int64), -1 where the node committed nothing."""
        committed, proposed = self.commit_times(cap)
        return np.where(committed >= 0, committed - proposed[:, None, :], -1)

    def latency_stats(self, num_bins=1024, bin_width=1, proposed_from=0, proposed_until=None):
        """Commit-latency statistics per group, reduced on the device (``lbft_latency_stats``; needs ``commit_times=True``): a
        group is a parameter set of a sweep (``param_sets`` order) or the whole batch of a plain simulator.  The samples are
        the non-negative entries of ``commit_latencies()`` at full cap whose row was proposed in ``[proposed_from,
        proposed_until)`` (``None``: no upper bound); instances with an error bit in ``status`` add nothing and are counted
        in ``excluded``.  Returns a ``LatencyStats``."""
        self._check_current("latency statistics")
        return self._sim.latency_stats(num_bins, bin_width, proposed_from, proposed_until)

    def block_latency_stats(self, threshold="quorum", num_bins=1024, bin_width=1, proposed_from=0, proposed_until=None):
        """Block-latency statistics per group, reduced on the device (``lbft_block_latency_stats``; needs
        ``commit_times=True``): one sample per block of each instance's chain (a row of its longest log) proposed in
        ``[proposed_from, proposed_until)``, the time from its proposal until the nodes that committed it hold ``threshold``
        voting rights.  ``threshold``: an int in 1..total voting rights, or ``"first"``, ``"validity"`` (f + 1), ``"quorum"``
        or ``"all"`` (see ``resolve_threshold``).  Blocks that never reach it are counted in ``unreached``.  Groups, windows,
        bins and excluded instances are those of ``latency_stats``.  Returns a ``BlockLatencyStats``."""
        self._check_current("block latency statistics")
        return self._sim.block_latency_stats(threshold, num_bins, bin_width, proposed_from, proposed_until)

    def contexts(self, instance=0):
        """The ``Vec<&Context>`` that ``loop_until`` returns for one instance."""
        return [SimulatedContextView(self, instance, a) for a in range(self._sim.num_nodes)]


class BatchSimulator:
    """Many independent ``Simulator`` instances (one per seed) on one GPU."""

    def __init__(self, seeds, num_nodes, network_delay=RandomDelay(), node_config=NodeConfig(),
                 commands_per_epoch=30000, voting_rights=None, silent=None, partition_windows=0,
                 partition_max_len=0, device=0, round_cap=0, queue_cap=0, payload_cap=0, record_round_switches=False, resumable=False,
                 true_data_sync=False, commit_times=False):
        self._lib = _lib.load()
        self.record_round_switches = bool(record_round_switches)  # LBFT_FLAG_ROUND_SWITCHES (DataWriter, data_writer.rs)
        self.resumable = bool(resumable)  # LBFT_FLAG_RESUMABLE: run_until / snapshot / restore
        # LBFT_FLAG_TRUE_DATA_SYNC: NON-PARITY variant — requests are answered by the node they were sent to (the reference
        # simulator dispatches them to the requester itself, simulator.rs:446)
        self.true_data_sync = bool(true_data_sync)
        # LBFT_FLAG_COMMIT_TIMES: record when each block is proposed and when each node commits it (commit_times())
        self.commit_times_enabled = bool(commit_times)
        self.seeds = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).reshape(-1))
        self.num_instances = int(self.seeds.shape[0])
        self.num_nodes = int(num_nodes)
        self.network_delay, self.node_config = network_delay, node_config
        self.commands_per_epoch = int(commands_per_epoch)
        self.voting_rights = None if voting_rights is None else np.ascontiguousarray(voting_rights, dtype=np.uint64)
        self.silent = None if silent is None else np.ascontiguousarray(silent, dtype=np.uint8)
        self.partition_windows, self.partition_max_len = int(partition_windows), int(partition_max_len)
        self.device, self.round_cap, self.queue_cap, self.payload_cap = int(device), int(round_cap), int(queue_cap), int(payload_cap)
        self._handle = None
        self._generation = 0   # bumped by every run: results of an older run know they are stale
        self.timing = None

    # -- lifetime -------------------------------------------------------------------------------
    def make_config(self, max_clock):
        c = _lib.LbftConfig()
        c.struct_size = ctypes.sizeof(_lib.LbftConfig)
        c.num_instances, c.num_nodes = self.num_instances, self.num_nodes
        c.delay_kind = self.network_delay.kind
        c.seeds = self.seeds.ctypes.data
        c.max_clock = int(max_clock)
        c.delay_mean, c.delay_variance = self.network_delay.mean, self.network_delay.variance
        c.delay_lo, c.delay_hi = self.network_delay.lo, self.network_delay.hi
        c.target_commit_interval, c.delta = self.node_config.target_commit_interval, self.node_config.delta
        c.gamma, c.lambda_ = self.node_config.gamma, self.node_config.lambda_
        c.commands_per_epoch = self.commands_per_epoch
        c.voting_rights = None if self.voting_rights is None else self.voting_rights.ctypes.data
        c.silent = None if self.silent is None else self.silent.ctypes.data
        c.partition_windows, c.partition_max_len = self.partition_windows, self.partition_max_len
        c.device, c.round_cap, c.queue_cap, c.payload_cap = self.device, self.round_cap, self.queue_cap, self.payload_cap
        c.flags = ((_lib.FLAG_ROUND_SWITCHES if self.record_round_switches else 0) | (_lib.FLAG_RESUMABLE if self.resumable else 0) |
                   (_lib.FLAG_TRUE_DATA_SYNC if self.true_data_sync else 0) | (_lib.FLAG_COMMIT_TIMES if self.commit_times_enabled else 0))
        return c

    def create(self, max_clock):
        """``lbft_create``: validate, build the host tables, allocate device state."""
        self.close()
        handle = ctypes.c_void_p()
        cfg = self.make_config(max_clock)
        _lib.check(self._lib.lbft_create(ctypes.byref(cfg), ctypes.byref(handle)))
        self._handle = handle
        return self

    def close(self):
        if self._handle is not None:
            self._lib.lbft_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- running --------------------------------------------------------------------------------
    def loop_until(self, max_clock, csv_path=None, strict=True):
        """``Simulator::new`` + ``loop_until(max_clock)`` for every instance; host buffers in, host results out."""
        if csv_path is not None:
            # simulator.rs:380-381, 470-472: a DataWriter is kept during the loop and written at the end
            if self.num_instances != 1:
                raise ValueError("csv_path names ONE simulator's output directory: for a batch pass record_round_switches=True "
                                 "and call write_data_files(path, instance)")
            self.record_round_switches = True
        self.create(int(max_clock))
        self._generation += 1
        code = self._lib.lbft_run(self._handle)
        _lib.check(code, allow=() if strict else (_lib.LBFT_ERR_CAPACITY,))
        self._read_timing()
        if csv_path is not None:
            self.write_data_files(csv_path, 0)
        return BatchResult(self)

    def run_until(self, stop_clock, strict=True):
        """``lbft_run_until``: ``loop_until(GlobalTime(stop_clock), ..)`` on every instance of a resumable handle created
        with the final horizon (``create(horizon)``); the first call is ``Simulator::new`` + ``loop_until``, later calls
        continue — and, like the reference, each call drops the first event beyond its clock (simulator.rs:383-391)."""
        self._generation += 1
        code = self._lib.lbft_run_until(self._handle, int(stop_clock))
        _lib.check(code, allow=() if strict else (_lib.LBFT_ERR_CAPACITY,))
        self._read_timing()
        return BatchResult(self)

    def snapshot(self):
        """``lbft_snapshot_save``: the whole batch between two ``run_until`` calls, as a ``numpy.uint8`` array."""
        n = ctypes.c_size_t(0)
        _lib.check(self._lib.lbft_snapshot_size(self._handle, ctypes.byref(n)))
        buf = np.empty(n.value, dtype=np.uint8)
        _lib.check(self._lib.lbft_snapshot_save(self._handle, ctypes.c_void_p(buf.ctypes.data), n.value))
        return buf

    def restore(self, snapshot):
        """``lbft_snapshot_load`` into a handle created from the same configuration; continue with ``run_until``."""
        buf = np.ascontiguousarray(snapshot, dtype=np.uint8)
        self._generation += 1
        _lib.check(self._lib.lbft_snapshot_load(self._handle, ctypes.c_void_p(buf.ctypes.data), buf.nbytes))

    def set_seeds(self, seeds):
        """Re-seed the batch: the next run is a fresh ``Simulator::new(seed, ..)`` per instance."""
        seeds = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).reshape(-1))
        if seeds.shape[0] != self.num_instances:
            raise ValueError("expected %d seeds" % self.num_instances)
        self.seeds = seeds
        _lib.check(self._lib.lbft_set_seeds(self._handle, ctypes.c_void_p(seeds.ctypes.data)))

    def run(self, strict=True):
        """``lbft_run`` on the existing handle: seeds host->device, event-loop kernel, summaries device->host."""
        self._generation += 1
        code = self._lib.lbft_run(self._handle)
        _lib.check(code, allow=() if strict else (_lib.LBFT_ERR_CAPACITY,))
        self._read_timing()
        return BatchResult(self)

    def run_async(self):
        """``lbft_run_async``: enqueue upload + kernel + download on the handle's stream and return at once; the previous
        run's ``BatchResult`` stays valid, and ``set_seeds`` may stage the next batch meanwhile.  Finish with ``wait()``."""
        _lib.check(self._lib.lbft_run_async(self._handle))

    def wait(self, strict=True, relaunch=False, before_relaunch=None):
        """``lbft_wait``: block until the run started by ``run_async`` is done; returns its ``BatchResult``.

        ``relaunch=True`` starts the next run (``lbft_run_async`` on the seeds staged by ``set_seeds`` meanwhile) BEFORE the
        finished run's summaries are copied out of the pinned mirrors, so that the host-side copies overlap the next
        kernel: the library keeps two sets of mirrors and the getters serve the finished run while the next one is in
        flight.  ``before_relaunch()`` runs between the two (the multi-GPU all-gather reads the device buffers there)."""
        self._generation += 1
        code = self._lib.lbft_wait(self._handle)
        _lib.check(code, allow=() if strict else (_lib.LBFT_ERR_CAPACITY,))
        self._read_timing()
        if before_relaunch is not None:
            before_relaunch()
        if relaunch:
            self.run_async()
        return BatchResult(self)

    def run_stream(self, batches, strict=True):
        """Run a sequence of seed batches with one run always in flight: yields one ``BatchResult`` per batch, in order.
        Batch k + 1 is staged (pinned seed buffer) while batch k runs and launched the moment batch k's results have
        landed; each step still copies its seeds host->device and its summaries device->host."""
        it = iter(batches)
        first = next(it, None)
        if first is None:
            return
        self.set_seeds(first)
        self.run_async()
        inflight = True
        try:
            for nxt in it:
                self.set_seeds(nxt)
                inflight = False
                res = self.wait(strict=strict, relaunch=True)
                inflight = True
                yield res
            inflight = False
            yield self.wait(strict=strict)
        finally:
            if inflight:  # the consumer stopped early (or a batch failed to stage): drain the run that is still in flight
                self.drain()

    def drain(self):
        """Wait for an in-flight ``run_async`` and discard its result, leaving the handle idle (no-op if there is none)."""
        if self._handle is not None and self._lib.lbft_wait(self._handle) == _lib.LBFT_OK:
            self._generation += 1

    def device_buffer(self, which):
        """(device pointer, bytes) of a result buffer: 0 commit counts, 1 last states, 2 counters, 3 status."""
        ptr, nbytes = ctypes.c_void_p(), ctypes.c_size_t()
        _lib.check(self._lib.lbft_device_buffer(self._handle, which, ctypes.byref(ptr), ctypes.byref(nbytes)))
        return int(ptr.value), int(nbytes.value)

    def upload(self):
        _lib.check(self._lib.lbft_upload(self._handle))

    def run_device(self):
        self._generation += 1
        _lib.check(self._lib.lbft_run_device(self._handle))
        self._read_timing()

    def download(self, strict=True):
        _lib.check(self._lib.lbft_download(self._handle), allow=() if strict else (_lib.LBFT_ERR_CAPACITY,))
        self._read_timing()
        return BatchResult(self)

    def _read_timing(self):
        t = _lib.LbftTiming()
        _lib.check(self._lib.lbft_timing_info(self._handle, ctypes.byref(t)))
        self.timing = t

    def kernel_info(self):
        """Name of the kernel instantiation the handle launches (as ncu / cuobjdump spell it)."""
        buf = ctypes.create_string_buffer(128)
        _lib.check(self._lib.lbft_kernel_info(self._handle, buf, 128))
        return buf.value.decode()

    def memory_info(self):
        b, w = ctypes.c_uint64(), ctypes.c_uint32()
        _lib.check(self._lib.lbft_memory_info(self._handle, ctypes.byref(b), ctypes.byref(w)))
        return int(b.value), int(w.value)

    # -- results --------------------------------------------------------------------------------
    def _fetch(self, fn, dtype, shape):
        if self._handle is None:
            raise RuntimeError("the simulator has been closed (or not created): results are fetched from the handle on first "
                               "access, so read them before close() / before leaving the `with` block")
        out = np.empty(shape, dtype=dtype)
        _lib.check(getattr(self._lib, fn)(self._handle, ctypes.c_void_p(out.ctypes.data)))
        return out

    def commit_log(self, instance, author):
        """``committed_history()`` of one node as a list of ``(proposer, index, time)``."""
        n = ctypes.c_size_t(0)
        _lib.check(self._lib.lbft_commit_log(self._handle, instance, author, None, 0, ctypes.byref(n)))
        buf = (_lib.LbftCommit * max(1, n.value))()
        _lib.check(self._lib.lbft_commit_log(self._handle, instance, author, buf, n.value, ctypes.byref(n)))
        return [(int(buf[i].proposer), int(buf[i].index), int(buf[i].time)) for i in range(n.value)]

    def commit_logs(self, cap=None):
        """``lbft_commit_logs``: every ``committed_history()`` of the batch with one device pass and one copy.  Returns
        ``(rows, lens)``: ``rows[instance, k]`` (fields ``proposer``, ``index``, ``time``) is row k of the instance's longest
        log and node n's log is ``rows[instance, :lens[instance, n]]``."""
        lens = np.empty((self.num_instances, self.num_nodes), dtype=np.uint32)
        if cap is None:
            cap = max(1, int(self._fetch("lbft_commit_counts", np.uint32, (self.num_instances, self.num_nodes)).max()))
        rows = np.empty((self.num_instances, int(cap)), dtype=COMMIT_DTYPE)
        _lib.check(self._lib.lbft_commit_logs(self._handle, ctypes.c_void_p(rows.ctypes.data), int(cap), ctypes.c_void_p(lens.ctypes.data)))
        return rows, lens

    def commit_times(self, cap=None):
        """``lbft_commit_times``: ``(committed[instance, node, cap], proposed[instance, cap])``, int64 global clocks with -1
        padding (see ``BatchResult.commit_times``); ``cap`` defaults to the longest log of the batch."""
        if cap is None:
            cap = max(1, int(self._fetch("lbft_commit_counts", np.uint32, (self.num_instances, self.num_nodes)).max()))
        committed = np.empty((self.num_instances, self.num_nodes, int(cap)), dtype=np.int64)
        proposed = np.empty((self.num_instances, int(cap)), dtype=np.int64)
        _lib.check(self._lib.lbft_commit_times(self._handle, ctypes.c_void_p(committed.ctypes.data), ctypes.c_void_p(proposed.ctypes.data),
                                               int(cap)))
        return committed, proposed

    def _latency_buffers(self, num_bins, bin_width, proposed_from, proposed_until):
        spec = _lib.LbftLatencySpec(struct_size=ctypes.sizeof(_lib.LbftLatencySpec), num_bins=int(num_bins), bin_width=int(bin_width),
                                    proposed_from=int(proposed_from),
                                    proposed_until=np.iinfo(np.int64).max if proposed_until is None else int(proposed_until))
        groups = len(self.param_sets) if isinstance(self, SweepSimulator) else 1
        summary = np.zeros(groups, dtype=LATENCY_SUMMARY_DTYPE)
        # (a histogram the library refuses, num_bins out of range or num_groups * num_bins > 2^24, is not allocated here)
        hist = np.zeros((groups, spec.num_bins if 1 <= spec.num_bins and groups * spec.num_bins <= 1 << 24 else 0), dtype=np.uint64)
        return spec, summary, hist

    def latency_stats(self, num_bins=1024, bin_width=1, proposed_from=0, proposed_until=None):
        """``lbft_latency_stats``: per-group commit-latency statistics as a ``LatencyStats`` (see
        ``BatchResult.latency_stats``)."""
        spec, summary, hist = self._latency_buffers(num_bins, bin_width, proposed_from, proposed_until)
        _lib.check(self._lib.lbft_latency_stats(self._handle, ctypes.byref(spec), ctypes.c_void_p(summary.ctypes.data),
                                                ctypes.c_void_p(hist.ctypes.data) if hist.size else None))
        return LatencyStats(summary, hist, spec.bin_width)

    def total_voting_rights(self):
        """The sum of the voting rights of the committee (each node holds 1 unless ``voting_rights`` says otherwise)."""
        return self.num_nodes if self.voting_rights is None else int(self.voting_rights.sum())

    def group_voting_rights(self):
        """The total voting rights of each group of ``latency_stats`` / ``block_latency_stats``, as an int64 array: the one
        group of a plain simulator holds ``total_voting_rights()``."""
        return np.full(1, self.total_voting_rights(), dtype=np.int64)

    def block_latency_stats(self, threshold="quorum", num_bins=1024, bin_width=1, proposed_from=0, proposed_until=None):
        """``lbft_block_latency_stats``: per-group block-latency statistics at a voting-rights threshold as a
        ``BlockLatencyStats`` (see ``BatchResult.block_latency_stats``).  A named threshold is resolved per group, with the
        group's total voting rights; where the groups' totals differ it goes through ``lbft_block_latency_stats_groups``."""
        spec, summary, hist = self._latency_buffers(num_bins, bin_width, proposed_from, proposed_until)
        unreached = np.zeros(summary.shape[0], dtype=np.uint64)
        totals = self.group_voting_rights()
        out = (ctypes.c_void_p(summary.ctypes.data), ctypes.c_void_p(unreached.ctypes.data),
               ctypes.c_void_p(hist.ctypes.data) if hist.size else None)
        if isinstance(threshold, str) and (totals != totals[0]).any():
            w = np.array([resolve_threshold(threshold, int(t)) for t in totals], dtype=np.uint64)
            _lib.check(self._lib.lbft_block_latency_stats_groups(self._handle, ctypes.byref(spec), ctypes.c_void_p(w.ctypes.data), *out))
        else:
            w = resolve_threshold(threshold, int(totals[0]))
            _lib.check(self._lib.lbft_block_latency_stats(self._handle, ctypes.byref(spec), ctypes.c_uint64(min(max(w, 0), (1 << 64) - 1)), *out))
        return BlockLatencyStats(summary, unreached, hist, spec.bin_width, w)

    def round_switches(self, instance):
        """``DataWriter::nodes_round_switch`` of one instance as ``[(node, round, time)]``, node-major
        (needs ``record_round_switches=True``)."""
        n = ctypes.c_size_t(0)
        _lib.check(self._lib.lbft_round_switches(self._handle, instance, None, 0, ctypes.byref(n)))
        buf = (_lib.LbftRoundSwitch * max(1, n.value))()
        _lib.check(self._lib.lbft_round_switches(self._handle, instance, buf, n.value, ctypes.byref(n)))
        return [(int(buf[i].node), int(buf[i].round), int(buf[i].time)) for i in range(n.value)]

    def write_data_files(self, path, instance=0):
        """``DataWriter::new`` + ``write_to_file`` (data_writer.rs:20-33, 61-96) for one instance:
        ``<path>/round_switches.txt`` and ``<path>/number_of_messages.txt``."""
        counters = self._fetch("lbft_counters", np.uint32, (self.num_instances, 12))[instance]
        write_data_files(path, self.num_nodes, self.round_switches(instance), int(counters[0]) + int(counters[1]) + int(counters[2]))


@dataclass(frozen=True)
class FaultSet:
    """The fault model of one point of a sweep: the silent (crashed) nodes, by index, and the random partition plan — what
    ``BatchSimulator``'s ``silent`` / ``partition_windows`` / ``partition_max_len`` give a whole batch — and the timed outages:
    ``((node, down_from, down_until), ...)``, at most one per node, in ms of global clock.  The node is down at clock t iff
    ``down_from <= t < down_until`` (``down_until`` None: it never recovers).  While down it handles no event and answers no
    request; it keeps its state and acts again at the first event addressed to it after the window
    (``lbft_create_sweep_outages``)."""
    silent: tuple = ()
    partition_windows: int = 0
    partition_max_len: int = 0
    outages: tuple = ()

    def __post_init__(self):
        object.__setattr__(self, "silent", tuple(int(n) for n in self.silent))  # (a list or array compares, and hashes, as a tuple)
        out = []
        for w in self.outages:
            node, start, end = w
            out.append((int(node), int(start), None if end is None else int(end)))
        nodes = [w[0] for w in out]
        if len(set(nodes)) != len(nodes):
            raise ValueError("FaultSet.outages takes at most one window per node")
        object.__setattr__(self, "outages", tuple(out))

    def has_fault_model(self):
        """Whether the silent nodes or the partition plan differ from none (what ``lbft_fault_set`` carries; the outages are
        passed apart)."""
        return bool(self.silent) or bool(self.partition_windows) or bool(self.partition_max_len)

    def to_c(self):
        mask = 0
        for n in self.silent:
            if not 0 <= int(n) < 64:
                raise ValueError("silent node index %r is not in 0..63" % (n,))
            mask |= 1 << int(n)
        return _lib.LbftFaultSet(silent_mask=mask, partition_windows=int(self.partition_windows),
                                 partition_max_len=int(self.partition_max_len))


@dataclass(frozen=True)
class ParamSet:
    """One point of a parameter sweep: the network delay and ``NodeConfig`` of the instances assigned to it
    (main.rs --mean / --variance and --delta / --gamma / --lambda / --target_commit_interval), its fault model, its
    voting rights: a tuple of one int per node of the set, or None for 1 per node (``BatchSimulator``'s ``voting_rights``),
    its committee size: None for the simulator's ``num_nodes``, and its link latencies: an ``n x n`` nested sequence of whole
    milliseconds (``n`` the set's committee size), entry ``[a][b]`` added to the time of every message from node a to node b
    (see ``regional_latency``), or None for none."""
    network_delay: RandomDelay = RandomDelay()
    node_config: NodeConfig = NodeConfig()
    faults: FaultSet = FaultSet()
    voting_rights: tuple = None
    num_nodes: int = None
    link_latency: tuple = None

    def __post_init__(self):
        if self.voting_rights is not None:  # (a list or array compares, and hashes, as a tuple)
            object.__setattr__(self, "voting_rights", tuple(int(w) for w in self.voting_rights))
        if self.link_latency is not None:  # (likewise, a tuple of tuples)
            object.__setattr__(self, "link_latency", tuple(tuple(int(v) for v in row) for row in self.link_latency))

    def to_c(self):
        d, n = self.network_delay, self.node_config
        return _lib.LbftParamSet(delay_kind=d.kind, reserved=0, delay_mean=d.mean, delay_variance=d.variance, delay_lo=d.lo,
                                 delay_hi=d.hi, target_commit_interval=n.target_commit_interval, delta=n.delta, gamma=n.gamma,
                                 lambda_=n.lambda_)


def regional_latency(region_of_node, latency_between_regions):
    """The link-latency matrix (``ParamSet.link_latency``) of a committee placed in regions: ``region_of_node[a]`` is node a's
    region, ``latency_between_regions[r][q]`` the latency in ms of a message from region r to region q (its diagonal the
    latency within a region).  Entry ``[a][b]`` is ``latency_between_regions[region_of_node[a]][region_of_node[b]]``."""
    regions = np.asarray(region_of_node, dtype=np.int64).reshape(-1)
    between = np.asarray(latency_between_regions, dtype=np.int64)
    if between.ndim != 2 or between.shape[0] != between.shape[1]:
        raise ValueError("latency_between_regions must be a square matrix, one row and column per region")
    if regions.size and (regions.min() < 0 or regions.max() >= between.shape[0]):
        raise ValueError("region_of_node has a region outside 0..%d" % (between.shape[0] - 1))
    return tuple(tuple(int(v) for v in row) for row in between[regions[:, None], regions[None, :]])


class SweepSimulator(BatchSimulator):
    """A parameter sweep as ONE batch (``lbft_create_sweep``): instance i runs ``Simulator::new(seeds[i], ..)`` under
    ``param_sets[set_of_instance[i]]``; everything else (committee, voting rights, ``commands_per_epoch``, capacities,
    device) is shared and passed as for ``BatchSimulator``.  Silent nodes and partitions are shared too, unless a set carries
    a ``FaultSet`` of its own: then every set has its own (``lbft_create_sweep_faults``) and the shared ``silent`` /
    ``partition_*`` arguments must be left unset.  Likewise the voting rights: when a set carries its own
    (``lbft_create_sweep_rights``), every set has its own (1 per node where left None) and ``voting_rights`` must be left
    unset.  And the committee size: when a set has its own (``ParamSet.num_nodes``, ``lbft_create_sweep_committees``),
    ``num_nodes`` is the size of the layout every instance gets and must be at least every set's; the per-node arrays keep
    ``num_nodes`` columns, and an instance's nodes past its set's committee read as nodes that never committed (mask them with
    ``nodes_of_instance()``).  Every result of instance i (of its committee's nodes) is what a ``BatchSimulator`` with that
    set's delay, node config, faults, voting rights and committee size computes for it.  And the link latencies: when a set
    carries a matrix (``ParamSet.link_latency``, ``lbft_create_sweep_links``), every network message from node a to node b of
    an instance of that set arrives ``link_latency[a][b]`` ms later than its drawn delay says; sets without one get zeros.
    And the outages: when a set's ``FaultSet`` carries timed outages (``lbft_create_sweep_outages``), each of its nodes with a
    window handles nothing while it is down; sets without any get none.
    Running, re-seeding (the set assignment stays), streaming and reading results work as on a ``BatchSimulator``."""

    def __init__(self, seeds, num_nodes, param_sets, set_of_instance, **shared):
        super().__init__(seeds, num_nodes, **shared)
        self.param_sets = list(param_sets)
        self.set_of_instance = np.ascontiguousarray(np.asarray(set_of_instance, dtype=np.uint32).reshape(-1))
        if self.set_of_instance.shape[0] != self.num_instances:
            raise ValueError("set_of_instance needs one entry per seed (%d)" % self.num_instances)
        for s, p in enumerate(self.param_sets):
            if p.num_nodes is not None and not 1 <= int(p.num_nodes) <= self.num_nodes:
                raise ValueError("parameter set %d: num_nodes (%r) must be in 1..num_nodes of the simulator (%d), the layout's "
                                 "committee" % (s, p.num_nodes, self.num_nodes))
        if self._committees() and self.voting_rights is not None:
            raise ValueError("a sweep whose sets have their own committee sizes takes voting rights per set only (ParamSet.voting_rights)")

    @classmethod
    def grid(cls, seeds_per_point, delays, node_configs, num_nodes=4, faults=None, voting_rights=None, link_latency=None, **shared):
        """The Cartesian product ``delays x node_configs`` (point p = i * len(node_configs) + j), each point run over the
        same seeds (``seeds_per_point``: a sequence of seeds, or a count k for seeds 0..k-1) in a contiguous block of
        instances: point p holds instances [p * k, (p + 1) * k).  ``set_of_instance`` and ``param_sets`` say which is which.
        ``faults``, a list of ``FaultSet``, adds a third, fastest-varying axis: point p = (i * len(node_configs) + j) *
        len(faults) + f, so ``latency_stats().mean().reshape(len(delays), len(node_configs), len(faults))`` is the cube.
        ``voting_rights``, a list of rows of one voting right per node, adds a fastest-varying axis after that (after
        ``node_configs`` when ``faults`` is None): ``block_latency_stats("quorum").mean().reshape(len(delays),
        len(node_configs), len(faults), len(voting_rights))``.  ``num_nodes``, a list of committee sizes instead of one,
        likewise adds a fastest-varying axis of committees, in a layout of the largest (it cannot be combined with a
        ``voting_rights`` list, whose rows have a fixed length).  ``link_latency``, a list of ``num_nodes x num_nodes`` matrices
        (``regional_latency``), adds the fastest-varying axis after all of those (not with a list of committee sizes: the
        matrices have a fixed size)."""
        seeds = np.arange(seeds_per_point, dtype=np.uint64) if np.isscalar(seeds_per_point) else \
            np.asarray(seeds_per_point, dtype=np.uint64).reshape(-1)
        sets = [ParamSet(d, n) for d in delays for n in node_configs] if faults is None else \
            [ParamSet(d, n, f) for d in delays for n in node_configs for f in faults]
        if link_latency is not None and not np.isscalar(num_nodes):
            raise ValueError("a grid takes a list of committee sizes (num_nodes) or a list of link-latency matrices, not both")
        if voting_rights is not None:
            if not np.isscalar(num_nodes):
                raise ValueError("a grid takes a list of committee sizes (num_nodes) or a list of voting-rights rows, not both")
            sets = [ParamSet(p.network_delay, p.node_config, p.faults, v) for p in sets for v in voting_rights]
        if not np.isscalar(num_nodes):
            sizes = [int(n) for n in num_nodes]
            sets = [ParamSet(p.network_delay, p.node_config, p.faults, None, n) for p in sets for n in sizes]
            num_nodes = max(sizes)
        if link_latency is not None:
            sets = [ParamSet(p.network_delay, p.node_config, p.faults, p.voting_rights, None, m) for p in sets for m in link_latency]
        k = seeds.shape[0]
        return cls(np.tile(seeds, len(sets)), num_nodes, sets, np.repeat(np.arange(len(sets), dtype=np.uint32), k), **shared)

    def create(self, max_clock):
        """``lbft_create_sweep``, or ``lbft_create_sweep_faults`` when some set has faults, or ``lbft_create_sweep_rights``
        when some set has voting rights, or ``lbft_create_sweep_committees`` when some set has its own committee size, or
        ``lbft_create_sweep_links`` when some set has link latencies, or ``lbft_create_sweep_outages`` when some set's faults
        carry outages: validate every set, build the per-set host tables, allocate device state."""
        per_set = any(p.faults.has_fault_model() for p in self.param_sets)
        if per_set and (self.silent is not None or self.partition_windows or self.partition_max_len):
            raise ValueError("a sweep takes silent nodes and partitions either per set (ParamSet.faults) or shared (silent / "
                             "partition_windows / partition_max_len), not both")
        rights = self._rights_table()
        if rights is not None and self.voting_rights is not None:
            raise ValueError("a sweep takes voting rights either per set (ParamSet.voting_rights) or shared (voting_rights), not both")
        self.close()
        handle = ctypes.c_void_p()
        cfg = self.make_config(max_clock)
        sets = (_lib.LbftParamSet * max(1, len(self.param_sets)))(*[p.to_c() for p in self.param_sets])
        so = ctypes.c_void_p(self.set_of_instance.ctypes.data)
        faults = (_lib.LbftFaultSet * len(self.param_sets))(*[p.faults.to_c() for p in self.param_sets]) if per_set else None
        links = self._link_table()
        outages = self._outage_table()
        if outages is not None:
            sizes = np.ascontiguousarray(self._committee_sizes(), dtype=np.uint32) if self._committees() else None
            _lib.check(self._lib.lbft_create_sweep_outages(
                ctypes.byref(cfg), sets, faults, None if rights is None else ctypes.c_void_p(rights.ctypes.data),
                None if sizes is None else ctypes.c_void_p(sizes.ctypes.data),
                None if links is None else ctypes.c_void_p(links.ctypes.data), outages, len(self.param_sets), so,
                ctypes.byref(handle)))
        elif links is not None:
            sizes = np.ascontiguousarray(self._committee_sizes(), dtype=np.uint32) if self._committees() else None
            _lib.check(self._lib.lbft_create_sweep_links(
                ctypes.byref(cfg), sets, faults, None if rights is None else ctypes.c_void_p(rights.ctypes.data),
                None if sizes is None else ctypes.c_void_p(sizes.ctypes.data), ctypes.c_void_p(links.ctypes.data),
                len(self.param_sets), so, ctypes.byref(handle)))
        elif self._committees():
            sizes = np.ascontiguousarray(self._committee_sizes(), dtype=np.uint32)
            _lib.check(self._lib.lbft_create_sweep_committees(
                ctypes.byref(cfg), sets, faults, None if rights is None else ctypes.c_void_p(rights.ctypes.data),
                ctypes.c_void_p(sizes.ctypes.data), len(self.param_sets), so, ctypes.byref(handle)))
        elif rights is not None:
            _lib.check(self._lib.lbft_create_sweep_rights(ctypes.byref(cfg), sets, faults, ctypes.c_void_p(rights.ctypes.data),
                                                          len(self.param_sets), so, ctypes.byref(handle)))
        elif per_set:
            _lib.check(self._lib.lbft_create_sweep_faults(ctypes.byref(cfg), sets, faults, len(self.param_sets), so, ctypes.byref(handle)))
        else:
            _lib.check(self._lib.lbft_create_sweep(ctypes.byref(cfg), sets, len(self.param_sets), so, ctypes.byref(handle)))
        self._handle = handle
        return self

    def _committees(self):
        """Whether some set has its own committee size (a committee sweep)."""
        return any(p.num_nodes is not None for p in self.param_sets)

    def _committee_sizes(self):
        """Each set's committee size."""
        return np.array([self.num_nodes if p.num_nodes is None else int(p.num_nodes) for p in self.param_sets], dtype=np.int64)

    def _rights_table(self):
        """The [num_sets][num_nodes] voting rights of a rights or committee sweep (1 per node of its committee where a set
        leaves them None, 0 past it), or None when no set carries any."""
        if all(p.voting_rights is None for p in self.param_sets):
            return None
        sizes = self._committee_sizes()
        rows = np.zeros((len(self.param_sets), self.num_nodes), dtype=np.uint64)
        for s, p in enumerate(self.param_sets):
            row = (1,) * int(sizes[s]) if p.voting_rights is None else p.voting_rights
            if len(row) != sizes[s]:
                raise ValueError("ParamSet.voting_rights needs one entry per node of the set (%d)" % sizes[s])
            rows[s, :len(row)] = row
        return rows

    def _link_table(self):
        """The [num_sets][num_nodes][num_nodes] link latencies of a links sweep (each set's matrix in the top-left corner of its
        committee, 0 elsewhere and for sets without one), or None when no set carries any."""
        if all(p.link_latency is None for p in self.param_sets):
            return None
        sizes = self._committee_sizes()
        out = np.zeros((len(self.param_sets), self.num_nodes, self.num_nodes), dtype=np.uint32)
        for s, p in enumerate(self.param_sets):
            if p.link_latency is None:
                continue
            m = np.asarray(p.link_latency, dtype=np.int64)
            n = int(sizes[s])
            if m.shape != (n, n):
                raise ValueError("parameter set %d: link_latency must be %d x %d (the set's committee)" % (s, n, n))
            if (m < 0).any() or (m > 65535).any():
                raise ValueError("parameter set %d: link_latency entries must be in 0..65535 ms" % s)
            out[s, :n, :n] = m
        return out

    def _outage_table(self):
        """The [num_sets * num_nodes] ``lbft_outage`` windows of an outage sweep (empty ones for nodes without a window, and
        ``down_until`` None as the largest int64), or None when no set carries any."""
        if all(not p.faults.outages for p in self.param_sets):
            return None
        N = self.num_nodes
        out = (_lib.LbftOutage * (len(self.param_sets) * N))()
        for s, p in enumerate(self.param_sets):
            for node, start, end in p.faults.outages:
                if not 0 <= node < N:
                    raise ValueError("parameter set %d: outage node %d is not in 0..%d" % (s, node, N - 1))
                out[s * N + node] = _lib.LbftOutage(start, _lib.INT64_MAX if end is None else end)
        return out

    def nodes_of_instance(self):
        """The committee size of each instance, as an int64 array [num_instances]: its set's, where the per-node arrays have
        ``num_nodes`` columns.  ``np.arange(sim.num_nodes) < sim.nodes_of_instance()[:, None]`` masks the nodes an instance
        has."""
        return self._committee_sizes()[self.set_of_instance]

    def total_voting_rights(self):
        """The sum of the voting rights of the committee; on a sweep whose sets carry their own voting rights, their common
        total (``ValueError`` when the sets' totals differ: see ``group_voting_rights``)."""
        totals = self.group_voting_rights()
        if (totals != totals[0]).any():
            raise ValueError("the parameter sets of this sweep have different total voting rights: use group_voting_rights()")
        return int(totals[0])

    def group_voting_rights(self):
        """The total voting rights of each parameter set (a group of the latency statistics), as an int64 array: its own
        row's total on a rights sweep, its committee's on a committee sweep, the shared committee's otherwise."""
        rights = self._rights_table()
        if rights is not None:
            return rights.sum(axis=1).astype(np.int64)
        if self._committees():
            return self._committee_sizes()
        return np.full(len(self.param_sets), super().total_voting_rights(), dtype=np.int64)


def format_round_switches_csv(num_nodes, switches):
    """Text of ``round_switches.txt`` (data_writer.rs:61-86) from ``[(node, round, time)]``.

    A header ``node 0,node 1,..`` then one row per round in ``0..max_round`` — EXCLUSIVE of the largest round any
    node reached, as the reference's ``for round_num in 0..max_round`` has it — holding, per node, the time at which
    that round was first seen, or nothing.  Text conventions are the ``csv`` crate's defaults (bft-lib/Cargo.toml:23
    ``csv = "1.1"``: ``,`` delimiter, ``\n`` terminator, quotes only when needed; a record that is a single empty field
    is written as ``""``).  FORMAT UNPINNED: neither the crate nor a Rust toolchain is available here, so the bytes
    are a restatement; the values are checked bit-exactly against the oracle, and the file is checked to read back
    through the steps of the reference's own consumer (visualization/round_switch/round_plotter.py:11-14, 52-53).
    """
    first = {}
    max_round = 0
    for node, rnd, time in switches:
        first.setdefault((node, rnd), time)  # `.find(..)`: the first entry of that round
        max_round = max(max_round, rnd)
    lines = [",".join("node %d" % n for n in range(num_nodes))]
    for rnd in range(max_round):
        fields = ["" if (n, rnd) not in first else str(first[(n, rnd)]) for n in range(num_nodes)]
        lines.append('""' if fields == [""] else ",".join(fields))
    return "\n".join(lines) + "\n"


def write_data_files(path, num_nodes, switches, message_count):
    if not os.path.exists(path):
        os.mkdir(path)  # fs::create_dir: not recursive (data_writer.rs:28-30)
    with open(os.path.join(path, "round_switches.txt"), "w", newline="") as f:
        f.write(format_round_switches_csv(num_nodes, switches))
    with open(os.path.join(path, "number_of_messages.txt"), "w", newline="") as f:
        f.write("%d\n" % message_count)  # wtr.serialize(Some(message_counter)) data_writer.rs:88-95


class Simulator:
    """Single-instance spelling of ``bft_lib::simulator::Simulator`` (simulator.rs:200-208, 380).

    ``context_factory`` is accepted for signature compatibility with the reference's callers
    (main.rs:23-34, simulated_run.rs:29-42); it may be ``None`` or a ``NodeConfig`` /
    ``(NodeConfig, commands_per_epoch)`` describing what the reference's closure would build.
    """

    def __init__(self, rng_seed, num_nodes, network_delay, context_factory=None, horizon=None, **kw):
        node_config, cpe = NodeConfig(), 30000
        # horizon: the largest clock any later loop_until will be given.  The reference needs no such thing (its heap is
        # unbounded); the device tables are sized for it.  Without it loop_until is one-shot, as before.
        self._horizon = None if horizon is None else int(horizon)
        self._ran = False
        if horizon is not None:
            kw["resumable"] = True
        if isinstance(context_factory, NodeConfig):
            node_config = context_factory
        elif isinstance(context_factory, tuple):
            node_config, cpe = context_factory
        elif context_factory is not None:
            raise TypeError("context_factory must be None, a NodeConfig or (NodeConfig, commands_per_epoch)")
        self._batch = BatchSimulator([rng_seed], num_nodes, network_delay, node_config, cpe, **kw)

    @staticmethod
    def new(rng_seed, num_nodes, network_delay, context_factory=None, horizon=None, **kw):
        return Simulator(rng_seed, num_nodes, network_delay, context_factory, horizon, **kw)

    def loop_until(self, max_clock, csv_path=None):
        if self._horizon is None:
            if self._ran:
                raise RuntimeError("loop_until was already run: pass horizon=<largest clock> to Simulator.new to call it again "
                                   "(the device tables are sized for a horizon, include/lbft.h lbft_run_until)")
            res = self._batch.loop_until(int(max_clock), csv_path)
        else:
            # simulator.rs:380 called repeatedly on one Simulator.  A DataWriter lives for ONE call (:381, :470-472), the
            # device keeps one table per run: csv_path is only supported on one-shot simulators.
            if csv_path is not None:
                raise ValueError("csv_path on a resumable Simulator is not supported")
            if not self._ran:
                self._batch.create(self._horizon)
            res = self._batch.run_until(int(max_clock))
        self._ran = True
        self.result = res
        return res.contexts(0)
