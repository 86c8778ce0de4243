"""Links sweeps (lbft_create_sweep_links) on the GPU: BASELINE config 5's shape (7 nodes, partition plans) and config 4's (64
nodes, weights, 21 silent) with three matrices each, through both kernel families, against the oracle with the set's link
latencies; every sweep kernel of tests/kernel_matrix.py and its commit-times twin as a links sweep, zero and non-zero matrices
alternating between neighbouring instances; a 65 536-instance grid of delays x deltas x matrices; re-seeded and streamed
handles."""
import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _lib, regional_latency
from tests.block_latency_support import assert_same_block_stats, numpy_block_stats
from tests.fault_support import fault_kwargs
from tests.kernel_matrix import CT, MATRIX
from tests.link_support import LinkOracle, matrices, oracle_per_set
from tests.support import assert_same

pytestmark = pytest.mark.gpu

W64 = tuple(1 + (i % 3) for i in range(64))  # BASELINE config 4's voting rights
SILENT21 = tuple(range(0, 63, 3))  # 21 of 64 authors silent (config 4)


@pytest.fixture(scope="module")
def link_oracle():
    return LinkOracle()


class Rows:
    def __init__(self, res, keep):
        self.commit_counts, self.last_states = res.commit_counts[keep], res.last_committed_states[keep]
        self.counters = res.counters[keep]


def clean(status):
    return (status & np.uint32(_lib.ST_ERROR_MASK)) == 0


def test_config5_shape_with_three_matrices(link_oracle, kernel_choice):
    """16 384 instances of 7 nodes with config 5's partition plan (4 x 150 ms) under a regional, an asymmetric and a zero matrix."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet((), 4, 150), None, None, m)
            for _, m in (matrices(7)[0], matrices(7)[1], matrices(7)[3])]
    seeds = np.arange(1, 16385, dtype=np.uint64)
    sim = SweepSimulator(seeds, 7, sets, np.arange(16384) % 3, payload_cap=128)
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    assert clean(res.status).mean() > 0.95  # (the slow links outgrow the default queue of a few instances: a capacity status)
    keep = np.arange(0, 16384, 37)
    keep = keep[clean(res.status[keep])]
    o = oracle_per_set(link_oracle, seeds[keep], 7, 1000, sets, sim.set_of_instance[keep])
    assert_same(o, Rows(res, keep), kernel_choice)
    np.testing.assert_array_equal(o.status, res.status[keep])
    sim.close()


def test_config4_shape_with_three_matrices(link_oracle, kernel_choice):
    """8 192 instances of 64 nodes with config 4's weights and 21 silent authors under three matrices."""
    far = tuple(tuple(0 if a == b else (30 if 63 in (a, b) else 2) for b in range(64)) for a in range(64))
    mats = [regional_latency([k % 4 for k in range(64)], [[1, 20, 35, 50], [20, 1, 25, 40], [35, 25, 1, 15], [50, 40, 15, 1]]), far,
            ((0,) * 64,) * 64]
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet(SILENT21), W64, None, m) for m in mats]
    seeds = np.arange(1, 8193, dtype=np.uint64)
    sim = SweepSimulator(seeds, 64, sets, np.arange(8192) % 3)
    res = sim.loop_until(1000, strict=False)
    assert clean(res.status).mean() > 0.99
    keep = np.arange(0, 8192, 1021)
    keep = keep[clean(res.status[keep])]
    assert_same(oracle_per_set(link_oracle, seeds[keep], 64, 1000, sets, sim.set_of_instance[keep]), Rows(res, keep), kernel_choice)
    sim.close()


SWEEP_KERNELS = sorted(n for n in MATRIX if MATRIX[n].kind != "plain")  # the 28 sweep kernels and their 28 commit-times twins


def small_matrix(n):
    """A non-zero n x n matrix of 0..4 ms, different in each direction (small: the entries' queue and payload capacities hold)."""
    return tuple(tuple((a + 2 * b) % 5 for b in range(n)) for a in range(n))


@pytest.mark.parametrize("name", SWEEP_KERNELS)
def test_every_sweep_kernel_as_a_links_sweep(name, monkeypatch, link_oracle):
    """Each sweep entry of tests/kernel_matrix.py, and its commit-times twin, run as a links sweep whose even sets carry an all-zero
    matrix and odd sets a non-zero one, interleaved across neighbouring instances: the entry's kernel runs; the zero sets' instances
    equal the same sweep without links in every output (commit logs and, on the twins, commit times included); the others equal
    the oracle with their set's matrix."""
    e = MATRIX[name]
    if e.force:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", e.force)
    else:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    kw = dict(e.kw)
    ct = bool(kw.pop("flags", 0) & CT)
    zero = ((0,) * e.N,) * e.N
    sets = [ParamSet(p.network_delay, p.node_config, p.faults, None, None, small_matrix(e.N) if k % 2 else zero) for k, p in enumerate(e.sets)]
    sim = SweepSimulator(e.seeds, e.N, sets, e.set_of, commit_times=ct, **kw)
    ref = SweepSimulator(e.seeds, e.N, list(e.sets), e.set_of, commit_times=ct, **kw)
    try:
        res = sim.loop_until(e.max_clock, strict=False)
        r = ref.loop_until(e.max_clock, strict=False)
        assert sim.kernel_info() == name == ref.kernel_info()
        ok = clean(res.status)
        assert ok.mean() > 0.5 and res.commit_counts.max() >= 3, np.unique(res.status)
        z = (np.asarray(e.set_of) % 2 == 0) & ok & clean(r.status)
        for field in ("commit_counts", "last_committed_states", "active_rounds", "counters", "status"):
            np.testing.assert_array_equal(getattr(res, field)[z], getattr(r, field)[z], err_msg=field)
        rows_s, _ = res.commit_logs()
        rows_r, _ = r.commit_logs(rows_s.shape[1])
        np.testing.assert_array_equal(rows_s[z], rows_r[z])
        if ct:
            cs, ps = res.commit_times(rows_s.shape[1])
            cr, pr = r.commit_times(rows_s.shape[1])
            np.testing.assert_array_equal(cs[z], cr[z])
            np.testing.assert_array_equal(ps[z], pr[z])
        # the non-zero sets against the oracle, on the entry's sample of instances
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
            o = oracle_per_set(link_oracle, e.seeds[idx], e.N, e.max_clock, [p], np.zeros(len(idx), np.int64), faults=False,
                               **dict(shared, **fk))
            assert_same(o, Rows(res, idx), "set %d" % s)
    finally:
        sim.close()
        ref.close()


def test_grid_of_65536_instances(link_oracle):
    """4 delays x 4 deltas x 4 matrices (regional, asymmetric, one far node, zero) x 1 024 seeds, 7 nodes: a sample of each set
    against the oracle; the zero sets equal a sweep without links; block_latency_stats("quorum") equals numpy over the commit
    times."""
    delays = [RandomDelay.new(m, 4.0) for m in (5.0, 10.0, 15.0, 20.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30, 40)]
    mats = [m for _, m in matrices(7)]
    sim = SweepSimulator.grid(1024, delays, configs, num_nodes=7, link_latency=mats, commit_times=True, payload_cap=128)
    assert sim.num_instances == 65536 and len(sim.param_sets) == 64
    res = sim.loop_until(1000, strict=False)
    ok = clean(res.status)
    assert ok.mean() > 0.9  # (the 5 ms delays under the slowest matrices outgrow the default queue in a few per cent)
    keep = np.arange(0, 65536, 97)
    keep = keep[ok[keep]]
    assert_same(oracle_per_set(link_oracle, sim.seeds[keep], 7, 1000, sim.param_sets, sim.set_of_instance[keep]), Rows(res, keep))
    plain = SweepSimulator.grid(1024, delays, configs, num_nodes=7, commit_times=True, payload_cap=128)
    r = plain.loop_until(1000, strict=False)
    zero_sets = np.arange(64)[np.arange(64) % 4 == 3]
    for k, s in enumerate(zero_sets):
        idx = np.nonzero(sim.set_of_instance == s)[0]
        idx_p = np.nonzero(plain.set_of_instance == k)[0]
        np.testing.assert_array_equal(sim.seeds[idx], plain.seeds[idx_p])
        for field in ("commit_counts", "last_committed_states", "active_rounds", "counters", "status"):
            np.testing.assert_array_equal(getattr(res, field)[idx], getattr(r, field)[idx_p], err_msg="set %d %s" % (s, field))
    plain.close()
    committed, proposed = res.commit_times()
    got = res.block_latency_stats("quorum")
    want = numpy_block_stats(committed, proposed, res.status, sim.set_of_instance, 64, np.ones(7, np.int64), 5)
    assert_same_block_stats(got, want, "quorum")
    assert got.samples.sum() > 0
    q = got.mean().reshape(len(delays), len(configs), len(mats))
    assert (np.where(np.isnan(q[:, :, 0]), np.inf, q[:, :, 0]) > q[:, :, 3]).all()  # the regional links slow the quorum at every point
    sim.close()


def test_reseeded_and_streamed_handles():
    """set_seeds and run_stream on a links sweep keep the set assignment and the matrices: what fresh handles give."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), link_latency=m) for m in (small_matrix(4), matrices(4)[1][1])]
    a = np.arange(1, 4097, dtype=np.uint64)
    b = a + 100000
    sim = SweepSimulator(a, 4, sets, np.arange(4096) % 2, payload_cap=64, queue_cap=256)
    sim.create(1000)
    first = [(r.last_committed_states.copy(), r.commit_counts.copy()) for r in sim.run_stream([a, b, a])]
    sim.set_seeds(b)
    again = sim.run()
    for seeds, (keys, counts) in ((a, first[0]), (b, first[1]), (a, first[2]), (b, (again.last_committed_states, again.commit_counts))):
        fresh = SweepSimulator(seeds, 4, sets, np.arange(4096) % 2, payload_cap=64, queue_cap=256)
        r = fresh.loop_until(1000)
        np.testing.assert_array_equal(keys, r.last_committed_states)
        np.testing.assert_array_equal(counts, r.commit_counts)
        fresh.close()
    sim.close()


def test_equal_matrices_share_one_device_table():
    """lbft_memory_info: a sweep over two distinct matrices holds one more N x N u16 table than a sweep over one."""
    m = matrices(7)
    one = SweepSimulator(np.arange(64), 7, [ParamSet(RandomDelay.new(10.0, 4.0), link_latency=m[0][1])] * 4, np.arange(64) % 4).create(1000)
    two = SweepSimulator(np.arange(64), 7, [ParamSet(RandomDelay.new(10.0, 4.0), link_latency=m[k % 2][1]) for k in range(4)],
                         np.arange(64) % 4).create(1000)
    assert two.memory_info()[0] - one.memory_info()[0] == 7 * 7 * 2
    one.close()
    two.close()
