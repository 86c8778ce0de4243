"""Committee sweeps (lbft_create_sweep_committees) on the GPU: BASELINE config 5's and config 4's shapes with two committee sizes in
one layout (partitions, and silent authors per set), through both kernel families, against the oracle (strided subsets) and against
one plain handle per set (every instance); every sweep kernel of tests/kernel_matrix.py and its commit-times twin with committee
sizes alternating between neighbouring instances, against a plain handle per size; a 65 536-instance grid of delays x deltas x
committee sizes against one sweep handle per size; re-seeded and streamed handles."""
import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _lib
from tests.block_latency_support import THRESHOLD_NAMES
from tests.committee_support import oracle_per_committee
from tests.kernel_matrix import CT, MATRIX
from tests.support import assert_same

pytestmark = pytest.mark.gpu

W64 = tuple(1 + (i % 3) for i in range(64))  # BASELINE config 4's voting rights
OUTPUTS = ("commit_counts", "last_committed_states", "active_rounds", "status")


class Rows:
    def __init__(self, res, keep):
        self.commit_counts, self.last_states = res.commit_counts[keep], res.last_committed_states[keep]
        self.counters = res.counters[keep]


def size(sim, ps):
    return sim.num_nodes if ps.num_nodes is None else ps.num_nodes


def plain_handle(seeds, n, ps, max_clock, **kw):
    """A plain handle of committee n with the set's delay, NodeConfig, faults and voting rights."""
    f = ps.faults
    silent = None
    if f.silent:
        silent = np.zeros(n, np.uint8)
        silent[list(f.silent)] = 1
    p = BatchSimulator(seeds, n, ps.network_delay, ps.node_config, voting_rights=ps.voting_rights, silent=silent,
                       partition_windows=f.partition_windows, partition_max_len=f.partition_max_len, **kw)
    return p, p.loop_until(max_clock, strict=False)


def assert_absent_zero(sim, res):
    """The nodes past each instance's committee: commit count, state key 0, and a commit log of no rows."""
    absent = np.arange(sim.num_nodes)[None, :] >= sim.nodes_of_instance()[:, None]
    assert (res.commit_counts[absent] == 0).all() and (res.last_committed_states[absent] == 0).all()
    return absent


def check_against_plain(sim, res, max_clock, clean=0.99):
    """Every instance that neither run flags equals the plain handle of its set's committee (counters 0..7); at least `clean`."""
    assert_absent_zero(sim, res)
    ok_all = []
    for s, ps in enumerate(sim.param_sets):
        idx = np.nonzero(sim.set_of_instance == s)[0]
        n = size(sim, ps)
        p, r = plain_handle(sim.seeds[idx], n, ps, max_clock, queue_cap=sim.queue_cap)
        ok = ((res.status[idx] & ~np.uint32(64)) == 1) & ((r.status & ~np.uint32(64)) == 1)
        ok_all.append(ok)
        np.testing.assert_array_equal(res.commit_counts[idx][ok][:, :n], r.commit_counts[ok], err_msg="set %d" % s)
        np.testing.assert_array_equal(res.last_committed_states[idx][ok][:, :n], r.last_committed_states[ok], err_msg="set %d" % s)
        np.testing.assert_array_equal(res.active_rounds[idx][ok], r.active_rounds[ok], err_msg="set %d" % s)
        np.testing.assert_array_equal(res.counters[idx][ok][:, :8], r.counters[ok][:, :8], err_msg="set %d" % s)
        p.close()
    assert np.concatenate(ok_all).mean() > clean


def test_config5_shape_with_two_committees(oracle, kernel_choice):
    """16 384 instances in a layout of 7: committees of 4 and 7, each with and without config 5's partition plan (4 x 150 ms)."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), f, None, n) for n in (4, 7) for f in (FaultSet(), FaultSet((), 4, 150))]
    seeds = np.arange(1, 16385, dtype=np.uint64)
    sim = SweepSimulator(seeds, 7, sets, np.arange(16384) % 4)
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    keep = np.arange(0, 16384, 61)
    assert_same(oracle_per_committee(oracle, seeds[keep], 7, 1000, sets, sim.set_of_instance[keep]), Rows(res, keep), kernel_choice)
    check_against_plain(sim, res, 1000)
    sim.close()


def test_config4_shape_with_two_committees_and_silent_authors(oracle, kernel_choice):
    """8 192 instances in a layout of 64: committees of 16 and 64 with config 4's weights, each with none and with a third of its
    authors (less one) silent."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), f, W64[:n], n) for n in (16, 64)
            for f in (FaultSet(), FaultSet(tuple(i for i in range(n) if i % 3 == 0 and i < n - 4)))]
    seeds = np.arange(1, 8193, dtype=np.uint64)
    sim = SweepSimulator(seeds, 64, sets, np.arange(8192) % len(sets))
    res = sim.loop_until(1000, strict=False)
    keep = np.arange(0, 8192, 1021)
    assert_same(oracle_per_committee(oracle, seeds[keep], 64, 1000, sets, sim.set_of_instance[keep]), Rows(res, keep), kernel_choice)
    check_against_plain(sim, res, 1000)
    sim.close()


def test_grid_of_65536_instances():
    """4 delays x 4 deltas x committees of 4, 7, 10 and 16 x 1 024 seeds against one sweep handle per committee size, instance by
    instance.  (The 5 ms delays outgrow the default queue in a few per cent of the instances on either side: outside the contract.)"""
    delays = [RandomDelay.new(m, 4.0) for m in (5.0, 10.0, 15.0, 20.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30, 40)]
    sizes = [4, 7, 10, 16]
    sim = SweepSimulator.grid(1024, delays, configs, num_nodes=sizes)
    assert sim.num_instances == 65536
    res = sim.loop_until(1000, strict=False)
    assert_absent_zero(sim, res)
    ok_all = []
    for k, n in enumerate(sizes):
        one = SweepSimulator.grid(1024, delays, configs, num_nodes=n)
        r = one.loop_until(1000, strict=False)
        idx = np.nonzero(sim.nodes_of_instance() == n)[0]
        assert len(idx) == one.num_instances
        np.testing.assert_array_equal(sim.seeds[idx], one.seeds)
        ok = ((res.status[idx] & ~np.uint32(64)) == 1) & ((r.status & ~np.uint32(64)) == 1)
        ok_all.append(ok)
        for field in ("commit_counts", "last_committed_states"):
            np.testing.assert_array_equal(getattr(res, field)[idx][ok][:, :n], getattr(r, field)[ok], err_msg="n=%d %s" % (n, field))
        np.testing.assert_array_equal(res.active_rounds[idx][ok], r.active_rounds[ok])
        np.testing.assert_array_equal(res.counters[idx][ok][:, :8], r.counters[ok][:, :8])
        one.close()
    assert np.concatenate(ok_all).mean() > 0.9
    sim.close()


SWEEP_KERNELS = sorted(n for n in MATRIX if MATRIX[n].kind != "plain")  # the 28 sweep kernels and their 28 commit-times twins


def committee_entry(e):
    """The matrix entry as a committee sweep: set k takes the entry's committee N when k is even and N - 1 when odd (N where a
    silent node of the set, or of the shared configuration, is the last), so the sizes alternate between neighbouring instances
    (Entry.set_of interleaves the sets).  The entry's shared voting rights become each set's, truncated to its committee."""
    kw = dict(e.kw)
    flags = kw.pop("flags", 0)
    base = kw.pop("voting_rights", None)
    shared_silent = [i for i, v in enumerate(kw.get("silent") or []) if v]
    sets = []
    for k, p in enumerate(e.sets):
        n = e.N - 1 if k % 2 and e.N > 1 else e.N
        if any(i >= n for i in list(p.faults.silent) + shared_silent):
            n = e.N
        row = None if base is None else tuple(int(w) for w in base[:n])
        if row is not None and sum(row) == 0:
            n, row = e.N, tuple(int(w) for w in base)
        sets.append(ParamSet(p.network_delay, p.node_config, p.faults, row, n))
    return sets, kw, bool(flags & CT)


@pytest.mark.parametrize("name", SWEEP_KERNELS)
def test_every_sweep_kernel_as_a_committee_sweep(name, monkeypatch):
    """Each sweep entry of tests/kernel_matrix.py, and its commit-times twin, run as a committee sweep with two sizes interleaved
    across neighbouring instances: the entry's kernel runs, the absent nodes read 0 and log nothing, and every instance's commit
    counts, state keys and commit-log rows (proposers included) equal the plain handle of its set's committee; on the twins also
    its commit times (-1 for absent nodes) and block_latency_stats at each set's named thresholds."""
    e = MATRIX[name]
    if e.force:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", e.force)
    else:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    sets, kw, ct = committee_entry(e)
    sim = SweepSimulator(e.seeds, e.N, sets, e.set_of, commit_times=ct, **kw)
    res = sim.loop_until(e.max_clock, strict=False)
    try:
        assert sim.kernel_info() == name
        assert len({p.num_nodes for p in sets}) == 2 or e.N == 1
        clean = (res.status & np.uint32(_lib.ST_ERROR_MASK)) == 0
        assert clean.mean() > 0.5 and res.commit_counts.max() >= 3, np.unique(res.status)
        absent = assert_absent_zero(sim, res)
        rows_s, lens_s = res.commit_logs()
        assert (lens_s[absent] == 0).all()
        cap = rows_s.shape[1]
        if ct:
            committed_s, proposed_s = res.commit_times(cap)
            assert (committed_s[absent] == -1).all()
            stats = {t: res.block_latency_stats(t) for t in THRESHOLD_NAMES}
        compared = 0
        for s, ps in enumerate(sets):
            idx = np.nonzero(e.set_of == s)[0]
            n = ps.num_nodes
            faults = ps if e.kind == "faults" else ParamSet(ps.network_delay, ps.node_config, FaultSet(), ps.voting_rights)
            shared = dict(kw)
            if shared.get("silent") is not None:
                shared["silent"] = np.asarray(shared["silent"])[:n]
            p, r = plain_handle(e.seeds[idx], n, faults, e.max_clock, commit_times=ct, **shared)
            try:
                ok = ((res.status[idx] & ~np.uint32(64)) == 1) & ((r.status & ~np.uint32(64)) == 1)
                for field in ("commit_counts", "last_committed_states"):
                    np.testing.assert_array_equal(getattr(res, field)[idx][ok][:, :n], getattr(r, field)[ok], err_msg="set %d %s" % (s, field))
                np.testing.assert_array_equal(res.active_rounds[idx][ok], r.active_rounds[ok], err_msg="set %d rounds" % s)
                rows_p, _ = r.commit_logs(cap)
                np.testing.assert_array_equal(rows_s[idx][ok], rows_p[ok], err_msg="set %d commit logs" % s)
                if ct and ok.all():
                    committed_p, proposed_p = r.commit_times(cap)
                    np.testing.assert_array_equal(committed_s[idx][:, :n], committed_p, err_msg="set %d committed" % s)
                    np.testing.assert_array_equal(proposed_s[idx], proposed_p, err_msg="set %d proposed" % s)
                    for t in THRESHOLD_NAMES:
                        want, got = r.block_latency_stats(t), stats[t]
                        assert got.thresholds[s] == want.threshold, (s, t)
                        for fld in ("instances", "excluded", "samples", "sum", "min", "max", "unreached"):
                            assert getattr(got, fld)[s] == getattr(want, fld)[0], (s, t, fld)
                        np.testing.assert_array_equal(got.hist[s], want.hist[0], err_msg="set %d %s hist" % (s, t))
                    compared += 1
                if ok.any():
                    i = idx[np.nonzero(ok)[0][0]]
                    assert res.commit_log(i, e.N - 1) == ([] if n < e.N else r.commit_log(int(np.nonzero(ok)[0][0]), e.N - 1))
            finally:
                p.close()
        if ct:
            assert compared > 0, "no set compared its statistics"
    finally:
        sim.close()


def test_reseeded_and_streamed_handles():
    """set_seeds and run_stream on a committee sweep keep the set assignment and the absent nodes' zeros: what fresh handles give."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), num_nodes=n) for n in (2, 4)]
    a = np.arange(1, 4097, dtype=np.uint64)
    b = a + 100000
    sim = SweepSimulator(a, 4, sets, np.arange(4096) % 2)
    sim.create(1000)
    first = [(r.last_committed_states.copy(), r.commit_counts.copy()) for r in sim.run_stream([a, b, a])]
    sim.set_seeds(b)
    again = sim.run()
    absent = np.arange(4)[None, :] >= sim.nodes_of_instance()[:, None]
    for seeds, (keys, counts) in ((a, first[0]), (b, first[1]), (a, first[2]), (b, (again.last_committed_states, again.commit_counts))):
        assert (counts[absent] == 0).all() and (keys[absent] == 0).all()
        fresh = SweepSimulator(seeds, 4, sets, np.arange(4096) % 2)
        r = fresh.loop_until(1000)
        np.testing.assert_array_equal(keys, r.last_committed_states)
        np.testing.assert_array_equal(counts, r.commit_counts)
        fresh.close()
    sim.close()
