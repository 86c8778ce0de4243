"""Outage sweeps (lbft_create_sweep_outages) on the GPU: BASELINE config 5's shape (7 nodes, partition plans) and config 4's (64
nodes, weights, 21 silent), each with a crash-stop, a crash-recovery and an empty schedule, through both kernel families, against
the test oracle with the set's windows; every sweep kernel of tests/kernel_matrix.py and its commit-times twin as an outage sweep,
empty and non-empty schedules alternating between neighbouring instances; a 65 536-instance grid whose [0, inf) schedules equal a
silent-node fault sweep and whose empty schedules equal the plain sweep; per-set block_latency_stats("quorum") against numpy over
the commit times; the shared device table of equal schedules."""
import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _lib
from tests.block_latency_support import assert_same_block_stats, numpy_block_stats
from tests.fault_support import fault_kwargs
from tests.kernel_matrix import CT, MATRIX
from tests.outage_support import OutageOracle, oracle_per_set, set_with_outages
from tests.support import assert_same

pytestmark = pytest.mark.gpu

W64 = tuple(1 + (i % 3) for i in range(64))  # BASELINE config 4's voting rights
SILENT21 = tuple(range(0, 63, 3))  # 21 of 64 authors silent (config 4)
OUTPUTS = ("commit_counts", "last_committed_states", "active_rounds", "counters", "status")
# The counters a window moves in the other sets of its launch: a node with a window in any set has its duplicate timers queued
# rather than elided at push (DESIGN §6l), which moves the implementation counters max_queue and timers_elided, and nothing else.
REF_COUNTERS = [c for c in range(12) if c not in (8, 11)]


def same_outputs(a, b, idx_a, idx_b, what, counters=REF_COUNTERS):
    for field in OUTPUTS:
        x, y = getattr(a, field)[idx_a], getattr(b, field)[idx_b]
        if field == "counters":
            x, y = x[:, counters], y[:, counters]
        np.testing.assert_array_equal(x, y, err_msg="%s %s" % (what, field))


@pytest.fixture(scope="module")
def outage_oracle():
    return OutageOracle()


class Rows:
    def __init__(self, res, keep):
        self.commit_counts, self.last_states = res.commit_counts[keep], res.last_committed_states[keep]
        self.counters = res.counters[keep]


def clean(status):
    return (status & np.uint32(_lib.ST_ERROR_MASK)) == 0


def three_schedules(base, node):
    """`base` with node `node` crashing at 500 ms for good, down over [500, 800), and never down."""
    return [set_with_outages(base, w) for w in (((node, 500, None),), ((node, 500, 800),), ())]


def test_config5_shape_with_three_schedules(outage_oracle, kernel_choice):
    """16 384 instances of 7 nodes with config 5's partition plan (4 x 150 ms): node 0 crash-stop at 500 ms, down over [500,
    800), and never down."""
    sets = three_schedules(ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet((), 4, 150)), 0)
    seeds = np.arange(1, 16385, dtype=np.uint64)
    sim = SweepSimulator(seeds, 7, sets, np.arange(16384) % 3, payload_cap=128)
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    assert clean(res.status).mean() > 0.99
    keep = np.arange(0, 16384, 37)
    keep = keep[clean(res.status[keep])]
    o = oracle_per_set(outage_oracle, seeds[keep], 7, 1000, sets, sim.set_of_instance[keep])
    assert_same(o, Rows(res, keep), kernel_choice)
    np.testing.assert_array_equal(o.status, res.status[keep])
    sim.close()


def test_config4_shape_with_three_schedules(outage_oracle, kernel_choice):
    """8 192 instances of 64 nodes with config 4's weights and 21 silent authors: node 1 (live, weight 2) crash-stop at 500 ms,
    down over [500, 800), and never down."""
    sets = three_schedules(ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet(SILENT21), W64), 1)
    seeds = np.arange(1, 8193, dtype=np.uint64)
    sim = SweepSimulator(seeds, 64, sets, np.arange(8192) % 3)
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    assert clean(res.status).mean() > 0.99
    keep = np.arange(0, 8192, 1021)
    keep = keep[clean(res.status[keep])]
    assert_same(oracle_per_set(outage_oracle, seeds[keep], 64, 1000, sets, sim.set_of_instance[keep]), Rows(res, keep), kernel_choice)
    sim.close()


SWEEP_KERNELS = sorted(n for n in MATRIX if MATRIX[n].kind != "plain")  # the 28 sweep kernels and their 28 commit-times twins


def live_node(p, N, shared_silent):
    """A node of set `p` that is neither silent in it nor in the shared configuration, or None."""
    silent = set(p.faults.silent) | {k for k in range(N) if shared_silent is not None and shared_silent[k]}
    live = [k for k in range(N) if k not in silent]
    return live[-1] if live else None


@pytest.mark.parametrize("name", SWEEP_KERNELS)
def test_every_sweep_kernel_as_an_outage_sweep(name, monkeypatch, outage_oracle):
    """Each sweep entry of tests/kernel_matrix.py, and its commit-times twin, run as an outage sweep whose even sets carry an
    empty schedule and odd sets a crash-recovery window over the middle third of the run, interleaved across neighbouring
    instances: the entry's kernel runs; the even sets' instances equal the same sweep without outages in every output (commit
    logs and, on the twins, commit times included) but max_queue and timers_elided (REF_COUNTERS); the others equal the test
    oracle with their set's window."""
    e = MATRIX[name]
    if e.force:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", e.force)
    else:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    kw = dict(e.kw)
    ct = bool(kw.pop("flags", 0) & CT)
    sets = []
    for k, p in enumerate(e.sets):
        node = live_node(p, e.N, kw.get("silent"))
        w = ((node, e.max_clock // 3, 2 * e.max_clock // 3),) if k % 2 and node is not None else ()
        sets.append(set_with_outages(p, w))
    assert any(p.faults.outages for p in sets)
    sim = SweepSimulator(e.seeds, e.N, sets, e.set_of, commit_times=ct, **kw)
    ref = SweepSimulator(e.seeds, e.N, list(e.sets), e.set_of, commit_times=ct, **kw)
    try:
        res = sim.loop_until(e.max_clock, strict=False)
        r = ref.loop_until(e.max_clock, strict=False)
        assert sim.kernel_info() == name == ref.kernel_info()
        ok = clean(res.status)
        assert ok.mean() > 0.5 and res.commit_counts.max() >= 3, np.unique(res.status)
        z = (np.asarray(e.set_of) % 2 == 0) & ok & clean(r.status)
        assert z.any()
        same_outputs(res, r, z, z, "empty")
        rows_s, _ = res.commit_logs()
        rows_r, _ = r.commit_logs(rows_s.shape[1])
        np.testing.assert_array_equal(rows_s[z], rows_r[z])
        if ct:
            cs, ps = res.commit_times(rows_s.shape[1])
            cr, pr = r.commit_times(rows_s.shape[1])
            np.testing.assert_array_equal(cs[z], cr[z])
            np.testing.assert_array_equal(ps[z], pr[z])
        # the windowed sets against the test oracle, on the entry's sample of instances
        odd = np.nonzero((np.asarray(e.set_of) % 2 == 1) & ok)[0]
        pick = np.intersect1d(e.oracle_instances(), odd)
        if len(pick) == 0:
            pick = odd[:2]
        assert len(pick) > 0
        shared = {k: v for k, v in kw.items() if k in ("voting_rights", "silent", "partition_windows", "partition_max_len",
                                                       "commands_per_epoch")}
        for s in sorted(set(e.set_of[pick].tolist())):
            idx = pick[e.set_of[pick] == s]
            p = sets[s]
            fk = fault_kwargs(p.faults, e.N) if e.kind == "faults" else {}
            o = oracle_per_set(outage_oracle, e.seeds[idx], e.N, e.max_clock, [p], np.zeros(len(idx), np.int64), faults=False,
                               **dict(shared, **fk))
            assert_same(o, Rows(res, idx), "set %d" % s)
    finally:
        sim.close()
        ref.close()


def test_grid_of_65536_instances(outage_oracle):
    """4 delays x 4 deltas x 4 outage scenarios (none; node 2 down from 0 for good; node 0 down over [500, 800); node 0 crash-stop
    at 500) x 1 024 seeds, 7 nodes: a sample against the test oracle; the empty schedules byte-equal to the plain sweep but for
    max_queue and timers_elided (REF_COUNTERS); the [0,
    inf) schedules byte-equal to the same grid with node 2 silent (but for the implementation counters max_queue, max_payloads
    and the count of duplicate timers elided at push: a silent node's incoming events are elided at send, a down node's queued
    and dropped at their pop, and a node with a window in any set has its duplicate timers queued); block_latency_stats("quorum")
    equals numpy over the commit times."""
    delays = [RandomDelay.new(m, 4.0) for m in (5.0, 10.0, 15.0, 20.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30, 40)]
    scen = [FaultSet(), FaultSet(outages=((2, 0, None),)), FaultSet(outages=((0, 500, 800),)), FaultSet(outages=((0, 500, None),))]
    sim = SweepSimulator.grid(1024, delays, configs, num_nodes=7, faults=scen, commit_times=True, payload_cap=128)
    assert sim.num_instances == 65536 and len(sim.param_sets) == 64
    res = sim.loop_until(1000, strict=False)
    ok = clean(res.status)
    assert ok.mean() > 0.95
    keep = np.arange(0, 65536, 97)
    keep = keep[ok[keep]]
    assert_same(oracle_per_set(outage_oracle, sim.seeds[keep], 7, 1000, sim.param_sets, sim.set_of_instance[keep]), Rows(res, keep))
    committed, proposed = res.commit_times()
    rows, _ = res.commit_logs()
    scenario = sim.set_of_instance % 4
    # empty schedules: the plain sweep (lbft_create_sweep), every output
    plain = SweepSimulator.grid(1024, delays, configs, num_nodes=7, commit_times=True, payload_cap=128)
    r = plain.loop_until(1000, strict=False)
    rc, rp = r.commit_times()
    rr, _ = r.commit_logs(rows.shape[1])
    idx = np.nonzero(scenario == 0)[0]
    idx_p = (idx // 4096) * 1024 + idx % 1024  # plain point q is the grid's point 4q: instances [q * 1024, (q + 1) * 1024)
    np.testing.assert_array_equal(sim.seeds[idx], plain.seeds[idx_p])
    same_outputs(res, r, idx, idx_p, "empty")
    np.testing.assert_array_equal(rows[idx], rr[idx_p])
    np.testing.assert_array_equal(committed[idx], rc[idx_p])
    np.testing.assert_array_equal(proposed[idx], rp[idx_p])
    plain.close()
    # [0, inf) schedules: a fault sweep with node 2 silent in the same sets
    silent = SweepSimulator.grid(1024, delays, configs, num_nodes=7, faults=[FaultSet(), FaultSet((2,)), FaultSet(), FaultSet()],
                                 commit_times=True, payload_cap=128)
    s = silent.loop_until(1000, strict=False)
    sc, sp = s.commit_times()
    sr, _ = s.commit_logs(rows.shape[1])
    idx = np.nonzero(scenario == 1)[0]
    np.testing.assert_array_equal(sim.seeds, silent.seeds)
    same_outputs(res, s, idx, idx, "forever", [c for c in REF_COUNTERS if c != 10])
    np.testing.assert_array_equal(rows[idx], sr[idx])
    np.testing.assert_array_equal(committed[idx], sc[idx])
    np.testing.assert_array_equal(proposed[idx], sp[idx])
    silent.close()
    # per-set block latency at the quorum, on the device, against numpy over the commit times
    got = res.block_latency_stats("quorum")
    want = numpy_block_stats(committed, proposed, res.status, sim.set_of_instance, 64, np.ones(7, np.int64), 5)
    assert_same_block_stats(got, want, "quorum")
    for lo, hi in ((200, 500), (500, 800), (800, 1000)):
        got = res.block_latency_stats("quorum", proposed_from=lo, proposed_until=hi)
        want = numpy_block_stats(committed, proposed, res.status, sim.set_of_instance, 64, np.ones(7, np.int64), 5,
                                 proposed_from=lo, proposed_until=hi)
        assert_same_block_stats(got, want, "quorum [%d, %d)" % (lo, hi))
    assert got.samples.sum() > 0
    sim.close()


def test_equal_schedules_share_one_device_table():
    """lbft_memory_info: a sweep over two distinct schedules holds one more table of N windows (8 bytes each) than a sweep over
    one."""
    base = ParamSet(RandomDelay.new(10.0, 4.0))
    one = SweepSimulator(np.arange(64), 7, [set_with_outages(base, ((1, 100, 300),))] * 4, np.arange(64) % 4).create(1000)
    two = SweepSimulator(np.arange(64), 7, [set_with_outages(base, ((1, 100, 300),) if k % 2 else ((2, 0, None),)) for k in range(4)],
                         np.arange(64) % 4).create(1000)
    assert two.memory_info()[0] - one.memory_info()[0] == 7 * 8
    one.close()
    two.close()
