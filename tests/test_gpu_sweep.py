"""Sweep handles (lbft_create_sweep) on the GPU: every instance against the oracle run with its set's settings, through both
kernel families; a full 65 536-instance sweep of 256 sets against the same sets run as 256 plain handles; bulk commit logs;
streamed re-seeding; and the kernel each handle launches against the picks the CPU tests pin."""
import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, NodeConfig, RandomDelay, SweepSimulator
from tests.support import assert_same
from tests.sweep_support import KERNEL_CASES, SETS, SWEEP_PICKS, oracle_per_set, set_kwargs

pytestmark = pytest.mark.gpu


class GpuResult:
    """Adapter giving the product's BatchResult the attribute names of tests.support.Result."""

    def __init__(self, res):
        self.commit_counts, self.last_states = res.commit_counts, res.last_committed_states
        self.counters, self.status = res.counters, res.status


class Rows:
    """The rows `keep` of a result, with the attribute names of tests.support.Result."""

    def __init__(self, commit_counts, last_states, counters, keep):
        self.commit_counts, self.last_states, self.counters = commit_counts[keep], last_states[keep], counters[keep]


CASES = [
    # (first seed, instances, nodes, max_clock, shared)
    (200, 48, 4, 1000, {"round_cap": 256}),
    (400, 36, 7, 1000, {"round_cap": 256}),
    (500, 24, 40, 600, {}),
]


@pytest.mark.parametrize("seed0,count,nodes,max_clock,shared", CASES)
def test_sweep_matches_the_oracle(oracle, kernel_choice, seed0, count, nodes, max_clock, shared):
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(SETS)
    sim = SweepSimulator(seeds, nodes, SETS, set_of, **shared)
    res = sim.loop_until(max_clock)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    o = oracle_per_set(oracle, seeds, nodes, max_clock, SETS, set_of, **shared)
    assert ((res.status & ~np.uint32(64)) == 1).all(), res.status
    assert_same(o, GpuResult(res), "sweep N=%d on the %s kernel" % (nodes, kernel_choice))
    sim.close()


def grid_256():
    """256 points: 16 LogNormal delays (mean x variance) x 16 NodeConfigs (delta x gamma)."""
    delays = [RandomDelay.new(m, v) for m in (6.0, 8.0, 10.0, 14.0) for v in (0.0, 2.0, 4.0, 8.0)]
    configs = [NodeConfig(delta=d, gamma=g) for d in (20, 30, 40, 60) for g in (1.5, 2.0, 2.5, 3.0)]
    return delays, configs


def test_full_sweep_equals_plain_handles():
    """65 536 instances x 4 authors over 256 sets in one handle against the same 256 sets as 256 plain handles of 256 seeds."""
    delays, configs = grid_256()
    seeds = np.arange(9000, 9256, dtype=np.uint64)
    sim = SweepSimulator.grid(seeds, delays, configs, num_nodes=4)
    assert sim.num_instances == 65536
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info() == "lbft_sweep_event_loop_kernel<16,2,32>"
    counters = res.counters
    clean = 0
    for p, ps in enumerate(sim.param_sets):
        rows = slice(p * 256, (p + 1) * 256)
        plain = BatchSimulator(seeds, 4, ps.network_delay, ps.node_config)
        r = plain.loop_until(1000, strict=False)
        ok = ((r.status & ~np.uint32(64)) == 1) & ((res.status[rows] & ~np.uint32(64)) == 1)
        clean += int(ok.sum())
        a, b = Rows(r.commit_counts, r.last_committed_states, r.counters, ok), Rows(
            res.commit_counts[rows], res.last_committed_states[rows], counters[rows], ok)
        assert_same(a, b, "point %d" % p)
        np.testing.assert_array_equal(r.active_rounds[ok], res.active_rounds[rows][ok])
        plain.close()
    assert clean >= 65536 * 0.99, clean
    sim.close()


def test_commit_logs_match_the_oracle(oracle):
    seeds = np.arange(3100, 3124, dtype=np.uint64)
    set_of = (np.arange(24) * 5) % len(SETS)
    sim = SweepSimulator(seeds, 4, SETS, set_of, round_cap=256)
    res = sim.loop_until(1000)
    rows, lens = res.commit_logs()
    for i in range(24):
        kw = set_kwargs(SETS[set_of[i]])
        kw["round_cap"] = 256
        for node in (0, 3):
            want = oracle.commit_log([seeds[i]], 4, 0, node, 1000, **kw)
            got = [(int(r["proposer"]), int(r["index"]), int(r["time"])) for r in rows[i, :lens[i, node]]]
            assert got == want, (i, node)
            assert got == sim.commit_log(i, node)
    sim.close()


def test_run_stream_reseeds_and_keeps_the_assignment(oracle):
    set_of = np.arange(24) % len(SETS)
    batches = [np.arange(s, s + 24, dtype=np.uint64) for s in (10, 500, 4000)]
    sim = SweepSimulator(batches[0], 4, SETS, set_of, round_cap=256)
    sim.create(1000)
    outs = list(sim.run_stream(batches))
    assert len(outs) == 3
    for seeds, res in zip(batches, outs):
        o = oracle_per_set(oracle, seeds, 4, 1000, SETS, set_of, round_cap=256)
        np.testing.assert_array_equal(o.commit_counts, res.commit_counts)
        np.testing.assert_array_equal(o.last_states, res.last_committed_states)
        np.testing.assert_array_equal(o.status & ~np.uint32(64), res.status & ~np.uint32(64))
    assert_same(o, GpuResult(outs[-1]), "last streamed batch")  # (counters are read from the handle: the last run's only)
    sim.close()


def test_kernel_info_matches_the_cpu_picks(monkeypatch):
    for family, want in SWEEP_PICKS.items():
        if family:
            monkeypatch.setenv("LBFT_FORCE_KERNEL", family)
        else:
            monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
        for name, count, nodes, kw in KERNEL_CASES:
            kw = dict(kw)
            max_clock = kw.pop("max_clock", 1000)
            sim = SweepSimulator(np.arange(1, count + 1, dtype=np.uint64), nodes, [SETS[0]], np.zeros(count), **kw)
            sim.create(max_clock)
            assert sim.kernel_info() == want[name], (family, name)
            sim.close()
