"""Rights sweeps (lbft_create_sweep_rights) on the GPU: BASELINE config 5's and config 4's shapes with per-set voting rights (and
per-set silent authors), through both kernel families, against the oracle (strided subsets) and against one plain handle per set
(every instance); a 65 536-instance grid of delays x deltas x stake rows against 64 plain handles; commit logs, commit times and
block-latency statistics per set at each set's named thresholds, on every sweep kernel of tests/kernel_matrix.py and its
commit-times twin, with stake rows interleaved between neighbouring instances; sets whose first
leaders differ, read through lbft_commit_logs and lbft_commit_log; re-seeded and streamed handles."""
import ctypes

import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, BlockLatencyStats, FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _lib
from tests.block_latency_support import THRESHOLD_NAMES, assert_same_block_stats
from tests.kernel_matrix import CT, MATRIX
from tests.rights_support import oracle_per_set
from tests.support import assert_same

pytestmark = pytest.mark.gpu

W64 = tuple(1 + (i % 3) for i in range(64))                  # BASELINE config 4's voting rights
SILENT64 = tuple(i for i in range(64) if i % 3 == 0 and i <= 60)  # ... and its 21 silent authors
OUTPUTS = ("commit_counts", "last_committed_states", "active_rounds", "status")


def zipf(n, s=1.0, scale=1000):
    return tuple(max(1, int(scale / (k + 1) ** s)) for k in range(n))


def near_third(n):
    """Node 0 holds just under a third of the total."""
    return (n - 2,) + (2,) * (n - 1)


class Rows:
    def __init__(self, res, keep):
        self.commit_counts, self.last_states = res.commit_counts[keep], res.last_committed_states[keep]
        self.counters = res.counters[keep]


def plain_per_set(sim, max_clock, commit_times=False):
    """Each set of a sweep run as a plain handle over its instances (its delay, NodeConfig, faults and voting rights)."""
    handles = []
    for s, ps in enumerate(sim.param_sets):
        idx = np.nonzero(sim.set_of_instance == s)[0]
        f = ps.faults
        silent = None
        if f.silent:
            silent = np.zeros(sim.num_nodes, np.uint8)
            silent[list(f.silent)] = 1
        p = BatchSimulator(sim.seeds[idx], sim.num_nodes, ps.network_delay, ps.node_config, voting_rights=ps.voting_rights, silent=silent,
                           partition_windows=f.partition_windows, partition_max_len=f.partition_max_len, commit_times=commit_times,
                           queue_cap=sim.queue_cap)
        handles.append((idx, p, p.loop_until(max_clock, strict=False)))
    return handles


def check_against_plain(sim, res, max_clock, clean=0.99):
    """Every instance that neither run flags equals the plain handle of its set (counters 0..7); at least `clean` of them."""
    want = {k: np.zeros_like(getattr(res, k)) for k in OUTPUTS}
    want["counters"] = np.zeros_like(res.counters)
    for idx, p, r in plain_per_set(sim, max_clock):
        for k in OUTPUTS:
            want[k][idx] = getattr(r, k)
        want["counters"][idx] = r.counters
        p.close()
    ok = ((res.status & ~np.uint32(64)) == 1) & ((want["status"] & ~np.uint32(64)) == 1)
    assert ok.mean() > clean, ok.mean()
    for k in ("commit_counts", "last_committed_states", "active_rounds"):
        np.testing.assert_array_equal(getattr(res, k)[ok], want[k][ok], err_msg=k)
    np.testing.assert_array_equal(res.counters[ok, :8], want["counters"][ok, :8])


def test_config5_shape_with_stake_rows(oracle, kernel_choice):
    """16 384 x 7 with four stake rows: uniform, [3, 1, ...], node 0 just under a third, Zipf."""
    rows = [(1,) * 7, (3,) + (1,) * 6, near_third(7), zipf(7)]
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet(), r) for r in rows]
    seeds = np.arange(1, 16385, dtype=np.uint64)
    sim = SweepSimulator(seeds, 7, sets, np.arange(16384) % 4)
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info().startswith("lbft_sweep_wide_kernel" if kernel_choice == "wide" else "lbft_sweep_event_loop_kernel")
    keep = np.arange(0, 16384, 61)
    assert_same(oracle_per_set(oracle, seeds[keep], 7, 1000, sets, sim.set_of_instance[keep]), Rows(res, keep), kernel_choice)
    check_against_plain(sim, res, 1000)
    sim.close()


def test_config4_shape_with_stake_rows_and_silent_authors(oracle, kernel_choice):
    """8 192 x 64: config 4's weights, uniform, one holder near a third, Zipf; each with none and with 21 silent authors."""
    rows = [W64, (1,) * 64, near_third(64), zipf(64, 1.0, 200)]
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), f, r) for r in rows for f in (FaultSet(), FaultSet(SILENT64))]
    seeds = np.arange(1, 8193, dtype=np.uint64)
    sim = SweepSimulator(seeds, 64, sets, np.arange(8192) % len(sets))
    res = sim.loop_until(1000, strict=False)
    keep = np.arange(0, 8192, 1021)
    assert_same(oracle_per_set(oracle, seeds[keep], 64, 1000, sets, sim.set_of_instance[keep]), Rows(res, keep), kernel_choice)
    check_against_plain(sim, res, 1000)
    sim.close()


def test_grid_of_65536_instances():
    """4 delays x 4 deltas x 4 stake rows x 1 024 seeds at N = 4 against 64 plain handles.  (The 5 ms delays outgrow the
    default queue in a few per cent of the instances, on both sides alike: those capacity errors are outside the contract.)"""
    rows = [(1, 1, 1, 1), (3, 1, 1, 1), (1, 1, 1, 0), (1 << 24, 1, 1 << 24, 7)]
    delays = [RandomDelay.new(m, 4.0) for m in (5.0, 10.0, 15.0, 20.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30, 40)]
    sim = SweepSimulator.grid(1024, delays, configs, num_nodes=4, voting_rights=rows)
    assert sim.num_instances == 65536
    res = sim.loop_until(1000, strict=False)
    check_against_plain(sim, res, 1000, clean=0.9)
    sim.close()


SWEEP_KERNELS = sorted(n for n in MATRIX if MATRIX[n].kind != "plain")  # the 28 sweep kernels and their 28 commit-times twins


def rights_entry(e):
    """The matrix entry as a rights sweep: set k takes stake row k % 2 (the entry's shared rights, or 1 per node; then the last
    node at 2), so the rows alternate between neighbouring instances (Entry.set_of interleaves the sets).  Shared keywords other
    than the rights stay shared (silent nodes and partitions included, where a sweep entry has them)."""
    kw = dict(e.kw)
    flags = kw.pop("flags", 0)
    base = tuple(int(w) for w in kw.pop("voting_rights", [1] * e.N))
    rows = (base, (1,) * (e.N - 1) + (2,))
    sets = [ParamSet(p.network_delay, p.node_config, p.faults, rows[k % 2]) for k, p in enumerate(e.sets)]
    return sets, kw, bool(flags & CT)


def groups_stats(sim, thresholds, **spec):
    """lbft_block_latency_stats_groups called directly, with one threshold per group."""
    spec_c, summary, hist = sim._latency_buffers(spec.get("num_bins", 1024), spec.get("bin_width", 1), spec.get("proposed_from", 0),
                                                  spec.get("proposed_until"))
    unreached = np.zeros(summary.shape[0], np.uint64)
    w = np.ascontiguousarray(thresholds, np.uint64)
    _lib.check(sim._lib.lbft_block_latency_stats_groups(sim._handle, ctypes.byref(spec_c), ctypes.c_void_p(w.ctypes.data),
                                                        ctypes.c_void_p(summary.ctypes.data), ctypes.c_void_p(unreached.ctypes.data),
                                                        ctypes.c_void_p(hist.ctypes.data)))
    return BlockLatencyStats(summary, unreached, hist, spec_c.bin_width, w)


@pytest.mark.parametrize("name", SWEEP_KERNELS)
def test_every_sweep_kernel_as_a_rights_sweep(name, monkeypatch):
    """Each sweep entry of tests/kernel_matrix.py, and its commit-times twin, run as a rights sweep with two stake rows interleaved
    across neighbouring instances: the entry's kernel runs, and every instance's commit counts, state keys and commit-log rows
    (proposers included) equal the plain handle of its set; on the twins also its commit times and block_latency_stats at each
    set's named thresholds, and the scalar entry point at the least group total against the per-group one."""
    e = MATRIX[name]
    if e.force:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", e.force)
    else:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    sets, kw, ct = rights_entry(e)
    sim = SweepSimulator(e.seeds, e.N, sets, e.set_of, commit_times=ct, **kw)
    res = sim.loop_until(e.max_clock, strict=False)
    try:
        assert sim.kernel_info() == name
        # (a set whose silent node holds more than a third of its row stalls, and on the smallest shared-memory queues its
        # timeouts can outgrow the queue: a capacity error, outside the contract, on the plain handle alike)
        clean = (res.status & np.uint32(_lib.ST_ERROR_MASK)) == 0
        assert clean.mean() > 0.5 and res.commit_counts.max() >= 3, np.unique(res.status)
        rows_s, lens_s = res.commit_logs()
        cap = rows_s.shape[1]
        if ct:
            committed_s, proposed_s = res.commit_times(cap)
            stats = {t: res.block_latency_stats(t) for t in THRESHOLD_NAMES}
        compared = 0
        for s, ps in enumerate(sets):
            idx = np.nonzero(e.set_of == s)[0]
            f = ps.faults
            faults = {}
            if e.kind == "faults":
                silent = np.zeros(e.N, np.uint8)
                silent[list(f.silent)] = 1
                faults = dict(silent=silent if f.silent else None, partition_windows=f.partition_windows,
                              partition_max_len=f.partition_max_len)
            p = BatchSimulator(e.seeds[idx], e.N, ps.network_delay, ps.node_config, voting_rights=ps.voting_rights, commit_times=ct,
                               **kw, **faults)
            try:
                r = p.loop_until(e.max_clock, strict=False)
                ok = ((res.status[idx] & ~np.uint32(64)) == 1) & ((r.status & ~np.uint32(64)) == 1)
                for field in ("commit_counts", "last_committed_states", "active_rounds"):
                    np.testing.assert_array_equal(getattr(res, field)[idx][ok], getattr(r, field)[ok], err_msg="set %d %s" % (s, field))
                rows_p, _ = r.commit_logs(cap)
                np.testing.assert_array_equal(rows_s[idx][ok], rows_p[ok], err_msg="set %d commit logs" % s)
                if ct and ok.all():
                    committed_p, proposed_p = r.commit_times(cap)
                    np.testing.assert_array_equal(committed_s[idx], committed_p, err_msg="set %d committed" % s)
                    np.testing.assert_array_equal(proposed_s[idx], proposed_p, err_msg="set %d proposed" % s)
                    for t in THRESHOLD_NAMES:
                        want, got = r.block_latency_stats(t), stats[t]
                        assert got.thresholds[s] == want.threshold, (s, t)
                        for fld in ("instances", "excluded", "samples", "sum", "min", "max", "unreached"):
                            assert getattr(got, fld)[s] == getattr(want, fld)[0], (s, t, fld)
                        np.testing.assert_array_equal(got.hist[s], want.hist[0], err_msg="set %d %s hist" % (s, t))
                    compared += 1
            finally:
                p.close()
        if ct:
            assert compared > 0, "no set compared its statistics"
            # one W for every group: the scalar entry point and the per-group one with equal thresholds, field by field
            totals = sim.group_voting_rights()
            for w in (1, int(totals.min())):
                assert_same_block_stats(res.block_latency_stats(w), groups_stats(sim, [w] * len(sets)), "W=%d" % w)
    finally:
        sim.close()


def test_sets_with_different_first_leaders():
    """Rows whose weighted draws elect different leaders from round 1 on: the proposer column of both commit-log read-outs and the
    state keys follow each set's own table."""
    rows = [(50, 1, 1, 1), (1, 1, 1, 50), (1, 50, 1, 1)]
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet(), r) for r in rows]
    seeds = np.arange(1, 97, dtype=np.uint64)
    sim = SweepSimulator(seeds, 4, sets, np.arange(96) % 3, queue_cap=512)  # (one leader for every round outgrows the default queue)
    res = sim.loop_until(1000)
    rows_s, lens_s = res.commit_logs()
    live = np.arange(rows_s.shape[1])[None, :] < lens_s.max(axis=1)[:, None]  # (rows past an instance's longest log are zero)
    heavy = [np.bincount(rows_s["proposer"][(np.arange(96) % 3 == s)[:, None] & live], minlength=4) for s in range(3)]
    assert [int(np.argmax(h)) for h in heavy] == [0, 3, 1], heavy
    for s, (idx, p, r) in enumerate(plain_per_set(sim, 1000)):
        np.testing.assert_array_equal(res.last_committed_states[idx], r.last_committed_states)
        rows_p, _ = r.commit_logs(rows_s.shape[1])
        np.testing.assert_array_equal(rows_s[idx], rows_p)
        for k, i in enumerate(idx[:4]):
            assert res.commit_log(i, 2) == r.commit_log(k, 2)
        p.close()
    sim.close()


def test_reseeded_and_streamed_handles():
    """set_seeds and run_stream on a rights sweep give what fresh handles give."""
    rows = [(1, 1, 1, 1), (3, 1, 1, 1)]
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), FaultSet(), r) for r in rows]
    a = np.arange(1, 4097, dtype=np.uint64)
    b = a + 100000
    sim = SweepSimulator(a, 4, sets, np.arange(4096) % 2)
    sim.create(1000)
    first = [r.last_committed_states.copy() for r in sim.run_stream([a, b, a])]
    sim.set_seeds(b)
    again = sim.run()
    for seeds, got in ((a, first[0]), (b, first[1]), (a, first[2]), (b, again.last_committed_states)):
        fresh = SweepSimulator(seeds, 4, sets, np.arange(4096) % 2)
        np.testing.assert_array_equal(got, fresh.loop_until(1000).last_committed_states)
        fresh.close()
    sim.close()
