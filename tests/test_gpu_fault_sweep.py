"""Fault sweeps (lbft_create_sweep_faults) on the GPU: BASELINE config 5's shape with per-set partition plans and config 4's
shape with per-set silent authors, each against the oracle (strided subsets) and against one plain handle per set (every
instance), through both kernel families; a 65 536-instance grid of delays x deltas x fault sets against 64 plain handles; the
equivalence with a sweep whose configuration carries uniform faults; commit times and latency statistics; re-seeded and
streamed handles."""
import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator
from tests.fault_support import oracle_per_set
from tests.latency_support import assert_same_stats, numpy_stats
from tests.support import assert_same

pytestmark = pytest.mark.gpu

W64 = [1 + (i % 3) for i in range(64)]                       # BASELINE config 4's voting rights
SILENT64 = [i for i in range(64) if i % 3 == 0 and i <= 60]  # ... and its 21 silent authors
OUTPUTS = ("commit_counts", "last_committed_states", "active_rounds", "status")


class Rows:
    """The rows `keep` of a result, with the attribute names of tests.support.Result."""

    def __init__(self, res, keep):
        self.commit_counts, self.last_states = res.commit_counts[keep], res.last_committed_states[keep]
        self.counters = res.counters[keep]


def plain_per_set(sim, max_clock, **shared):
    """Each set of a sweep run as a plain handle over its instances: the results gathered in instance order."""
    out = {f: np.zeros_like(getattr(sim.last, f)) for f in OUTPUTS}
    out["counters"] = np.zeros_like(sim.last.counters)
    for s, ps in enumerate(sim.param_sets):
        idx = np.nonzero(sim.set_of_instance == s)[0]
        f = ps.faults
        silent = None
        if f.silent:
            silent = np.zeros(sim.num_nodes, np.uint8)
            silent[list(f.silent)] = 1
        p = BatchSimulator(sim.seeds[idx], sim.num_nodes, ps.network_delay, ps.node_config, silent=silent,
                           partition_windows=f.partition_windows, partition_max_len=f.partition_max_len, **shared)
        r = p.loop_until(max_clock, strict=False)
        for k in OUTPUTS:
            out[k][idx] = getattr(r, k)
        out["counters"][idx] = r.counters
        p.close()
    return out


def check_against_plain(sim, res, max_clock, **shared):
    """Every instance that neither run flags equals the plain handle of its set (counters 0..7: the implementation counters
    max_queue / max_payloads / timers_elided may differ with the layout)."""
    want = plain_per_set(sim, max_clock, **shared)
    ok = ((res.status & ~np.uint32(64)) == 1) & ((want["status"] & ~np.uint32(64)) == 1)
    assert ok.mean() > 0.99, ok.mean()
    for k in ("commit_counts", "last_committed_states"):
        np.testing.assert_array_equal(getattr(res, k)[ok], want[k][ok], err_msg=k)
    np.testing.assert_array_equal(res.counters[ok, :8], want["counters"][ok, :8])
    np.testing.assert_array_equal(res.active_rounds[ok], want["active_rounds"][ok])


def run(sim, max_clock):
    sim.last = sim.loop_until(max_clock, strict=False)
    return sim.last


def test_config5_shape_with_partition_plans_per_set(oracle, kernel_choice):
    """16 384 x 7: sets with no partition, config 5's plan (4 x 150 ms), 2 x 400 ms and 8 x 100 ms."""
    fl = [FaultSet(), FaultSet((), 4, 150), FaultSet((), 2, 400), FaultSet((), 8, 100)]
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), f) for f in fl]
    seeds = np.arange(1, 16385, dtype=np.uint64)
    sim = SweepSimulator(seeds, 7, sets, np.arange(16384) % 4)
    res = run(sim, 1000)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    keep = np.arange(0, 16384, 61)
    o = oracle_per_set(oracle, seeds[keep], 7, 1000, sets, sim.set_of_instance[keep])
    assert_same(o, Rows(res, keep), "config 5 shape on the %s kernel" % kernel_choice)
    check_against_plain(sim, res, 1000)
    sim.close()


def test_config4_shape_with_silent_authors_per_set(oracle, kernel_choice):
    """8 192 x 64 with config 4's voting rights: 0, 7, 14 and 21 of its silent authors per set."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet(tuple(SILENT64[:k]))) for k in (0, 7, 14, 21)]
    seeds = np.arange(52, 52 + 8192, dtype=np.uint64)
    sim = SweepSimulator(seeds, 64, sets, np.arange(8192) // 2048, voting_rights=W64)
    res = run(sim, 1000)
    keep = np.arange(0, 8192, 97)
    o = oracle_per_set(oracle, seeds[keep], 64, 1000, sets, sim.set_of_instance[keep], voting_rights=W64)
    assert_same(o, Rows(res, keep), "config 4 shape on the %s kernel" % kernel_choice)
    check_against_plain(sim, res, 1000, voting_rights=W64)
    sim.close()


GRID_FAULTS = [FaultSet(), FaultSet((3,)), FaultSet((), 4, 150), FaultSet((0,), 2, 400)]


def test_grid_65536_equals_64_plain_handles():
    """4 delays x 4 deltas x 4 fault sets x 1 024 seeds, 4 authors, in one handle."""
    delays = [RandomDelay.new(m, 4.0) for m in (6.0, 8.0, 10.0, 14.0)]
    configs = [NodeConfig(delta=d) for d in (20, 30, 40, 60)]
    sim = SweepSimulator.grid(np.arange(1, 1025), delays, configs, num_nodes=4, faults=GRID_FAULTS)
    assert sim.num_instances == 65536 and len(sim.param_sets) == 64
    res = run(sim, 1000)
    check_against_plain(sim, res, 1000)
    sim.close()


@pytest.mark.parametrize("nodes,count,uniform", [(7, 16384, FaultSet((), 4, 150)), (4, 65536, FaultSet((1,), 2, 400)),
                                                 (64, 2048, FaultSet(tuple(SILENT64)))])
def test_uniform_faults_equal_a_sweep_with_shared_faults(nodes, count, uniform):
    """Every set carrying F: the kernel and every output, counters included, of lbft_create_sweep with F in the configuration."""
    base = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig()), ParamSet(RandomDelay.new(8.0, 2.0), NodeConfig(delta=30))]
    seeds = np.arange(5, 5 + count, dtype=np.uint64)
    set_of = np.arange(count) % 2
    a = SweepSimulator(seeds, nodes, [ParamSet(p.network_delay, p.node_config, uniform) for p in base], set_of)
    silent = None
    if uniform.silent:
        silent = np.zeros(nodes, np.uint8)
        silent[list(uniform.silent)] = 1
    b = SweepSimulator(seeds, nodes, base, set_of, silent=silent, partition_windows=uniform.partition_windows,
                       partition_max_len=uniform.partition_max_len)
    ra, rb = a.loop_until(1000, strict=False), b.loop_until(1000, strict=False)
    assert a.kernel_info() == b.kernel_info()
    assert a.memory_info()[1] == b.memory_info()[1]
    for k in OUTPUTS:
        np.testing.assert_array_equal(getattr(ra, k), getattr(rb, k), err_msg=k)
    np.testing.assert_array_equal(ra.counters, rb.counters)
    a.close()
    b.close()


def test_commit_times_and_latency_stats_on_a_fault_grid():
    """commit_times() of a fault grid against plain commit-times handles per set, and latency_stats() against numpy."""
    delays = [RandomDelay.new(10.0, 4.0), RandomDelay.new(6.0, 2.0)]
    sim = SweepSimulator.grid(np.arange(1, 513), delays, [NodeConfig()], num_nodes=4, faults=GRID_FAULTS, commit_times=True)
    res = sim.loop_until(1000)
    committed, proposed = res.commit_times(cap=160)
    for s, ps in enumerate(sim.param_sets):
        rows = slice(s * 512, (s + 1) * 512)
        f = ps.faults
        silent = None
        if f.silent:
            silent = np.zeros(4, np.uint8)
            silent[list(f.silent)] = 1
        p = BatchSimulator(sim.seeds[rows], 4, ps.network_delay, ps.node_config, silent=silent, partition_windows=f.partition_windows,
                           partition_max_len=f.partition_max_len, commit_times=True)
        c2, p2 = p.loop_until(1000).commit_times(cap=160)
        np.testing.assert_array_equal(committed[rows], c2, err_msg="set %d" % s)
        np.testing.assert_array_equal(proposed[rows], p2, err_msg="set %d" % s)
        p.close()
    stats = res.latency_stats(num_bins=256, bin_width=2, proposed_from=100, proposed_until=900)
    want = numpy_stats(committed, proposed, res.status, sim.set_of_instance, len(sim.param_sets), 256, 2, 100, 900)
    assert_same_stats(stats, want)
    assert stats.mean().reshape(2, 1, 4).shape == (2, 1, 4)
    sim.close()


def test_reseeded_and_streamed_handles_keep_their_faults():
    """set_seeds and run_stream keep each instance's set, faults included: equal to fresh handles over the new seeds."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), f) for f in GRID_FAULTS]
    set_of = np.arange(4096) % 4
    sim = SweepSimulator(np.arange(4096), 4, sets, set_of).create(1000)
    batches = [np.arange(k * 4096, (k + 1) * 4096, dtype=np.uint64) + 77 for k in range(3)]
    results = [(r.commit_counts.copy(), r.last_committed_states.copy()) for r in sim.run_stream(batches, strict=False)]
    sim.set_seeds(batches[1])
    again = sim.run(strict=False)
    for b, (cc, ls) in zip(batches, results):
        fresh = SweepSimulator(b, 4, sets, set_of)
        r = fresh.loop_until(1000, strict=False)
        np.testing.assert_array_equal(cc, r.commit_counts)
        np.testing.assert_array_equal(ls, r.last_committed_states)
        fresh.close()
    np.testing.assert_array_equal(again.commit_counts, results[1][0])
    sim.close()
