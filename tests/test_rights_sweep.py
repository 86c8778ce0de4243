"""Rights sweeps (lbft_create_sweep_rights) without a GPU: the SW and SW + CT device cores compiled for the host
(tests/hostcore/rights_hostcore.cpp) against the oracle run once per set with that set's voting rights, the equivalence with a sweep
whose configuration carries uniform rights, the deduplicated leader tables, block-latency statistics per group against numpy, the
refusals of both new entry points, SweepSimulator.grid's rights axis, and the signatures in all three bindings."""
import ctypes

import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _build, _lib
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE, BlockLatencyStats, resolve_threshold
from tests.block_latency_support import THRESHOLD_NAMES, assert_same_block_stats, numpy_block_stats
from tests.fault_support import c_faults, fault_kwargs
from tests.latency_support import make_spec
from tests.rights_support import FLAGS_CT, RightsHarness, cross_rights, oracle_per_set, rights_of, stake_rows
from tests.support import assert_same, make_config
from tests.sweep_support import KERNEL_CASES, SETS, c_sets


@pytest.fixture(scope="module")
def rights():
    return RightsHarness()


@pytest.fixture(scope="module")
def lib():
    _build.build_product()
    return _lib.load()


SHAPES = [
    # (first seed, nodes, max_clock, shared, queue mode of the sweep's layout)
    (100, 4, 1000, {"round_cap": 256}, 2),  # shared-memory scan queue
    (200, 7, 1500, {"round_cap": 256}, 3),  # calendar queue
    (300, 40, 600, {}, 3),
    (400, 7, 5000, {"round_cap": 768}, 0),  # beyond the calendar's horizon: binary heap
]


@pytest.mark.parametrize("seed0,nodes,max_clock,shared,qmode", SHAPES)
@pytest.mark.parametrize("with_faults", [False, True])
def test_rights_sweep_matches_the_oracle_per_instance(oracle, rights, seed0, nodes, max_clock, shared, qmode, with_faults):
    """The 12 parameter sets crossed with the stake rows (with_faults: and with no fault, the heaviest node silent and a
    zero-weight node silent, on a third of the sets), instance i on set i % num_sets: every instance equals the oracle run with its
    set's delay, NodeConfig, faults and voting rights; the proposer column is each set's own leader table."""
    rows = stake_rows(nodes)
    sets = cross_rights(SETS[::3] if with_faults else SETS, rows, with_faults)
    count = 2 * len(sets)
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    name = rights.kernel_info(seeds, nodes, max_clock, sets, set_of, faults=with_faults, **shared)[0]
    assert ",%d," % qmode in name and name.startswith("lbft_sweep_"), name
    h = rights.run(seeds, nodes, max_clock, sets, set_of, faults=with_faults, **shared)
    o = oracle_per_set(oracle, seeds, nodes, max_clock, sets, set_of, faults=with_faults, **shared)
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert_same(o, h, "rights sweep N=%d" % nodes)
    assert h.commit_counts.sum() > 0
    # the proposers: what a one-set rights sweep of the same set (its table at offset 0) gives each instance
    for s in range(0, len(sets), 7):
        idx = np.nonzero(set_of == s)[0]
        one = rights.run(seeds[idx], nodes, max_clock, [sets[s]], np.zeros(len(idx)), faults=with_faults, **shared)
        np.testing.assert_array_equal(h.proposers[idx], one.proposers, err_msg="set %d proposers" % s)
        np.testing.assert_array_equal(h.last_states[idx], one.last_states)
    # a silent node that holds more than a third blocks every quorum; a silent zero-weight node changes no leader
    if with_faults:
        heavy = np.array([len(p.faults.silent) == 1 and p.voting_rights[p.faults.silent[0]] * 3 >= sum(p.voting_rights) for p in sets])
        assert (h.commit_counts[heavy[set_of]] == 0).all()


def test_uniform_rights_are_a_sweep_with_shared_rights(rights, monkeypatch):
    """Every set carrying the rights V: the kernel and words per instance of lbft_create_sweep(_faults) with V in the configuration
    (each tests/sweep_support.KERNEL_CASES shape, automatic and forced to each family), and identical outputs, counters included."""
    for family in (None, "thread", "wide"):
        if family:
            monkeypatch.setenv("LBFT_FORCE_KERNEL", family)
        else:
            monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
        for name, count, nodes, kw in KERNEL_CASES:
            kw = dict(kw)
            max_clock = kw.pop("max_clock", 1000)
            seeds = np.arange(1, count + 1, dtype=np.uint64)
            set_of = np.arange(count) % 2
            for v in ([1] * nodes, [3] + [1] * (nodes - 1)):
                sets = [ParamSet(SETS[k].network_delay, SETS[k].node_config, voting_rights=v) for k in (0, 1)]
                got = rights.kernel_info(seeds, nodes, max_clock, sets, set_of, **kw)[:2]
                want = rights.kernel_info(seeds, nodes, max_clock, sets, set_of, rights=False, voting_rights=v, **kw)[:2]
                assert got == want, (family, name, got, want)
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    for name, count, nodes, kw in KERNEL_CASES:  # the outputs, on a batch small enough for the host core
        max_clock = kw.get("max_clock", 1000)
        shared = {k: v for k, v in kw.items() if k != "max_clock"}
        seeds = np.arange(11, 11 + 24, dtype=np.uint64)
        set_of = np.arange(24) % 3
        for v in ([1] * nodes, [3] + [1] * (nodes - 1)):
            sets = [ParamSet(p.network_delay, p.node_config, voting_rights=v) for p in SETS[:3]]
            a = rights.run(seeds, nodes, max_clock, sets, set_of, flags=FLAGS_CT, **shared)
            b = rights.run(seeds, nodes, max_clock, sets, set_of, rights=False, voting_rights=v, flags=FLAGS_CT, **shared)
            for field in ("commit_counts", "last_states", "counters", "status", "lc_round", "proposers", "committed", "proposed"):
                np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="%s %s" % (name, field))
    # per-set faults as well: against lbft_create_sweep_faults with the rights in the configuration
    sets = [ParamSet(p.network_delay, p.node_config, f, (3, 1, 1, 1)) for p in SETS[:2] for f in (FaultSet((1,)), FaultSet((), 4, 150))]
    seeds = np.arange(5, 5 + 32, dtype=np.uint64)
    set_of = np.arange(32) % 4
    a = rights.run(seeds, 4, 1000, sets, set_of, faults=True)
    b = rights.run(seeds, 4, 1000, sets, set_of, faults=True, rights=False, voting_rights=[3, 1, 1, 1])
    for field in ("commit_counts", "last_states", "counters", "status", "proposers"):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)


def test_leader_tables_are_deduplicated(rights):
    """A grid of 4 stake rows x 64 other points holds 4 leader tables of round_cap + 1 bytes, not 256."""
    rows = [r for _, r in stake_rows(7)[:4]]
    delays = [RandomDelay.new(m, v) for m in (5.0, 10.0, 15.0, 20.0) for v in (1.0, 4.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30, 40, 50, 60, 70, 80)]
    sets = [ParamSet(d, n, voting_rights=tuple(r)) for d in delays for n in configs for r in rows]
    assert len(sets) == 256
    seeds = np.arange(1, 513, dtype=np.uint64)
    set_of = np.arange(512) % 256
    _, _, table = rights.kernel_info(seeds, 7, 1000, sets, set_of, round_cap=256)
    _, _, one = rights.kernel_info(seeds, 7, 1000, sets, set_of, rights=False, round_cap=256)
    assert one == 257 and table == 4 * one


def test_block_latency_per_group_matches_numpy(rights):
    """lbft_block_latency_stats_groups over a rights sweep (the product's checks, per-group weights and serial threshold time on
    the host) against numpy over the same commit times, at each set's named thresholds and at one threshold for all."""
    rows = stake_rows(7)
    sets = cross_rights(SETS[:3], rows, with_faults=True)
    count = 3 * len(sets)
    seeds = np.arange(50, 50 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    totals = rights_of(sets, 7).sum(axis=1).astype(np.int64)
    weights = rights_of(sets, 7).astype(np.int64)
    spec = make_spec(1024, 1, 0, None)
    for name in THRESHOLD_NAMES + [1]:
        W = np.array([resolve_threshold(name, int(t)) for t in totals])
        h = rights.run(seeds, 7, 1000, sets, set_of, faults=True, cap=256, spec=spec, thresholds=W, flags=FLAGS_CT)
        want = _per_group_numpy(h, set_of, weights, W, len(sets))
        assert_same_block_stats(h.stats, want, str(name))
        assert h.stats.samples.sum() > 0
        assert (h.stats.thresholds == W).all() and h.stats.threshold == (W[0] if (W == W[0]).all() else None)


def _per_group_numpy(h, set_of, weights, W, groups):
    """numpy_block_stats with each group's weights and threshold, group by group."""
    parts = [numpy_block_stats(h.committed[set_of == g], h.proposed[set_of == g], h.status[set_of == g],
                               np.zeros((set_of == g).sum(), np.int64), 1, weights[g], int(W[g])) for g in range(groups)]
    cat = lambda f: np.concatenate([getattr(p, f) for p in parts])  # noqa: E731
    summary = np.zeros(groups, LATENCY_SUMMARY_DTYPE)
    for f in LATENCY_SUMMARY_DTYPE.names:
        summary[f] = cat(f)
    return BlockLatencyStats(summary, cat("unreached"), np.concatenate([p.hist for p in parts]), 1, W)


def _create(lib, cfg, sets, faults, vr, num_sets, set_of):
    h = ctypes.c_void_p()
    rc = lib.lbft_create_sweep_rights(ctypes.byref(cfg), sets, faults, None if vr is None else ctypes.c_void_p(vr.ctypes.data), num_sets,
                                      None if set_of is None else ctypes.c_void_p(set_of.ctypes.data), ctypes.byref(h))
    assert h.value is None
    return rc, lib.lbft_last_error().decode()


def test_rights_sweep_refusals(lib):
    """Everything lbft_create_sweep_rights refuses, with LBFT_ERR_INVALID and before any device work (so without a GPU too)."""
    cfg, keep = make_config(np.arange(1, 9, dtype=np.uint64), 4)
    ok = np.arange(8, dtype=np.uint32) % 4
    good = cross_rights(SETS[:2], stake_rows(4)[:2])
    sets, vr = c_sets(good), rights_of(good, 4)
    # what lbft_create_sweep refuses, with its messages
    for num_sets, set_of, want in ((0, ok, "num_sets"), (9, np.arange(8, dtype=np.uint32), "num_sets"), (4, None, "NULL"),
                                   (4, np.full(8, 4, np.uint32), "index >= num_sets")):
        rc, msg = _create(lib, cfg, sets, None, vr, num_sets, set_of)
        assert rc == -1 and want in msg, msg
    assert _create(lib, cfg, None, None, vr, 4, ok) == (-1, "sets and set_of_instance must not be NULL")
    bad = ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=0))
    rc, msg = _create(lib, cfg, c_sets([good[0], good[1], bad, good[3]]), None, vr, 4, ok)
    assert rc == -1 and "parameter set 2" in msg, msg
    # what lbft_create_sweep_faults refuses when faults are given
    faulty = [ParamSet(p.network_delay, p.node_config, FaultSet((4,)), p.voting_rights) for p in good]
    rc, msg = _create(lib, cfg, sets, c_faults(faulty), vr, 4, ok)
    assert rc == -1 and msg.startswith("parameter set 0: silent_mask has a bit at or above num_nodes"), msg
    cfg_s, keep_s = make_config(np.arange(1, 9, dtype=np.uint64), 4, silent=[0, 1, 0, 0])
    assert "per set only" in _create(lib, cfg_s, sets, c_faults(good), vr, 4, ok)[1]
    # rights must be given, per set only
    assert _create(lib, cfg, sets, None, None, 4, ok) == (-1, "voting_rights must not be NULL")
    cfg_v, keep_v = make_config(np.arange(1, 9, dtype=np.uint64), 4, voting_rights=[1, 1, 1, 1])
    rc, msg = _create(lib, cfg_v, sets, None, vr, 4, ok)
    assert rc == -1 and msg == "a rights sweep takes its voting rights per set only: lbft_config.voting_rights must be NULL", msg
    # a row config_error refuses, named by its set
    for row, want in (([1, 1 << 24 | 1, 1, 1], "voting_rights entries must be <= 2^24"), ([0, 0, 0, 0], "total voting rights must be > 0")):
        bad_vr = vr.copy()
        bad_vr[2] = row
        rc, msg = _create(lib, cfg, sets, None, bad_vr, 4, ok)
        assert rc == -1 and msg == "parameter set 2: " + want, msg
    assert lib.lbft_create_sweep_rights(None, sets, None, None, 4, None, ctypes.byref(ctypes.c_void_p())) == -1


def test_threshold_checks_per_group(rights):
    """The product's threshold checks on a rights sweep: one W above any group's total names the group; a threshold per group is
    checked against that group's total."""
    sets = [ParamSet(SETS[0].network_delay, SETS[0].node_config, voting_rights=r) for r in ((1, 1, 1, 1), (5, 1, 1, 1))]
    seeds = np.arange(1, 5, dtype=np.uint64)
    set_of = np.arange(4) % 2
    spec = make_spec()
    run = lambda W: rights.run(seeds, 4, 500, sets, set_of, spec=spec, thresholds=W, flags=FLAGS_CT)  # noqa: E731
    run([4, 8])
    with pytest.raises(RuntimeError, match=r"thresholds\[0\] must be in 1..total voting rights of group 0 \(4\)"):
        run([5, 8])
    with pytest.raises(RuntimeError, match=r"thresholds\[1\] must be in 1..total voting rights of group 1 \(8\)"):
        run([4, 9])
    with pytest.raises(RuntimeError, match=r"thresholds\[1\]"):
        run([1, 0])
    # the spec checks come first, with lbft_latency_stats' messages, through the per-group path too
    for bad, msg in ((make_spec(0), "num_bins must be in 1..65536"), (make_spec(8, 0), "bin_width must be >= 1"),
                     (make_spec(8, 1, 10, 5), "proposed_from must be <= proposed_until")):
        with pytest.raises(RuntimeError, match=msg):
            rights.run(seeds, 4, 500, sets, set_of, spec=bad, thresholds=[4, 8], flags=FLAGS_CT)
        with pytest.raises(RuntimeError, match=msg):
            rights.threshold_check(seeds, 4, 500, sets, set_of, bad, 1, flags=FLAGS_CT)
    # one W for every group: accepted up to the least total, refused above it naming that group
    rights.threshold_check(seeds, 4, 500, sets, set_of, spec, 4, flags=FLAGS_CT)
    with pytest.raises(RuntimeError, match=r"^-1: threshold must be in 1..total voting rights of group 0 \(4\)$"):
        rights.threshold_check(seeds, 4, 500, sets, set_of, spec, 5, flags=FLAGS_CT)
    with pytest.raises(RuntimeError, match=r"threshold must be in 1..total voting rights of group 0 \(4\)"):
        rights.threshold_check(seeds, 4, 500, sets, set_of, spec, 0, flags=FLAGS_CT)
    swapped = sets[::-1]  # the group named is the one whose total is exceeded
    with pytest.raises(RuntimeError, match=r"group 1 \(4\)"):
        rights.threshold_check(seeds, 4, 500, swapped, set_of, spec, 5, flags=FLAGS_CT)


def test_groups_entry_point_checks_arguments_without_a_device(lib):
    """lbft_block_latency_stats_groups refuses NULL arguments before looking at the handle, as lbft_block_latency_stats does."""
    spec = make_spec()
    out = (_lib.LbftLatencySummary * 1)()
    w = np.ones(1, np.uint64)
    args = (ctypes.byref(spec), ctypes.c_void_p(w.ctypes.data), ctypes.cast(out, ctypes.c_void_p))
    assert lib.lbft_block_latency_stats_groups(None, *args, None, None) == -1
    assert lib.lbft_last_error() == b"sim, spec, thresholds and out must not be NULL"
    assert lib.lbft_block_latency_stats_groups(None, None, None, None, None, None) == -1
    assert lib.lbft_block_latency_stats(None, ctypes.byref(spec), 1, ctypes.cast(out, ctypes.c_void_p), None, None) == -1
    assert lib.lbft_last_error() == b"sim, spec and out must not be NULL"


def test_grid_rights_axis_and_shared_rights_refusal():
    """SweepSimulator.grid(voting_rights=...): the fastest axis, after faults; per-set and shared voting rights do not mix; the
    totals per group."""
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30)]
    fl = [FaultSet(), FaultSet((3,))]
    vr = [(1, 1, 1, 1), (3, 1, 1, 1), (0, 2, 2, 2)]
    sim = SweepSimulator.grid([5, 6], delays, configs, num_nodes=4, faults=fl, voting_rights=vr)
    assert sim.num_instances == 72 and len(sim.param_sets) == 36
    for i, d in enumerate(delays):
        for j, n in enumerate(configs):
            for f, fs in enumerate(fl):
                for v, row in enumerate(vr):
                    assert sim.param_sets[((i * len(configs) + j) * len(fl) + f) * len(vr) + v] == ParamSet(d, n, fs, row)
    no_faults = SweepSimulator.grid([5], delays, configs, num_nodes=4, voting_rights=vr)
    assert no_faults.param_sets == [ParamSet(d, n, FaultSet(), row) for d in delays for n in configs for row in vr]
    np.testing.assert_array_equal(sim.group_voting_rights(), np.tile([4, 6, 6], 12))
    with pytest.raises(ValueError, match="group_voting_rights"):
        sim.total_voting_rights()
    same = SweepSimulator.grid([5], delays, configs, num_nodes=4, voting_rights=[(3, 1, 1, 1), (2, 2, 1, 1)])
    assert same.total_voting_rights() == 6
    plain = SweepSimulator.grid([5], delays, configs, num_nodes=4)
    assert plain.total_voting_rights() == 4 and (plain.group_voting_rights() == 4).all()
    assert ParamSet(voting_rights=[1, 2]) == ParamSet(voting_rights=(1, 2)) and ParamSet().voting_rights is None
    s = SweepSimulator(np.arange(4), 4, [ParamSet(voting_rights=(1, 1, 1, 1)), ParamSet()], [0, 1, 0, 1], voting_rights=[1, 1, 1, 1])
    with pytest.raises(ValueError, match="per set"):
        s.create(1000)
    with pytest.raises(ValueError, match="one entry per node"):
        SweepSimulator(np.arange(4), 4, [ParamSet(voting_rights=(1, 1, 1))], [0, 0, 0, 0]).create(1000)
    t = BlockLatencyStats(np.zeros(2, LATENCY_SUMMARY_DTYPE), np.zeros(2, np.uint64), np.zeros((2, 1), np.uint64), 1, [3, 5])
    assert t.threshold is None and list(t.thresholds) == [3, 5]


def test_rights_signatures_match_the_header():
    """lbft_create_sweep_rights and lbft_block_latency_stats_groups: the extern declarations of the Rust shim and the ctypes
    bindings against include/lbft.h."""
    from tests.test_rust_shim import c_functions, rust_functions
    c = c_functions()
    assert c["lbft_create_sweep_rights"][0] == ["ptr:lbft_config", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "u32", "ptr:u32",
                                                "ptr:lbft_sim"]
    assert c["lbft_block_latency_stats_groups"][0] == ["ptr:lbft_sim", "ptr:lbft_latency_spec", "ptr:u64", "ptr:lbft_latency_summary",
                                                       "ptr:u64", "ptr:u64"]
    r = rust_functions()
    assert r["lbft_create_sweep_rights"][0] == ["ptr:LbftConfig", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "u32", "ptr:u32",
                                                "ptr:*mut LbftSim"], r["lbft_create_sweep_rights"]
    assert r["lbft_block_latency_stats_groups"][0][2] == "ptr:u64"
    lib = _lib.load()
    assert len(lib.lbft_create_sweep_rights.argtypes) == 7 and len(lib.lbft_block_latency_stats_groups.argtypes) == 6
    assert {"lbft_create_sweep_rights", "lbft_block_latency_stats_groups"} <= set(_lib.EXPORTS)
