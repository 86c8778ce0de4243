"""Committee sweeps (lbft_create_sweep_committees) without a GPU: the SW and SW + CT device cores compiled for the host
(tests/hostcore/committee_hostcore.cpp) against the oracle run once per set as a plain configuration of that set's committee size,
instance by instance; the outputs of the absent nodes; each set's leader table against the plain handle of its size and their
deduplication; the equivalence of full-size committees with rights and plain sweeps; block-latency statistics per group against
numpy; every refusal and its message; SweepSimulator.grid's committee axis; and the signatures in all three bindings."""
import ctypes

import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _build, _lib
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE, BlockLatencyStats, resolve_threshold
from tests.block_latency_support import THRESHOLD_NAMES, assert_same_block_stats, numpy_block_stats
from tests.committee_support import FLAGS_CT, CommitteeHarness, cross_sizes, oracle_per_committee, rights_rows, size_of
from tests.fault_support import c_faults
from tests.latency_support import make_spec
from tests.support import assert_same, make_config
from tests.sweep_support import KERNEL_CASES, SETS, c_sets


@pytest.fixture(scope="module")
def harness():
    return CommitteeHarness()


@pytest.fixture(scope="module")
def lib():
    _build.build_product()
    return _lib.load()


SHAPES = [
    # (first seed, layout's committee, committee sizes, max_clock, shared, queue mode of the sweep's layout, partition plans)
    # shared-memory scan queue (a committee of one starts a round about every millisecond: room for 1 000 rounds)
    (100, 4, (1, 2, 3, 4), 1000, {"round_cap": 1024, "payload_cap": 64}, 2, False),
    (200, 7, (3, 4, 7), 1500, {"round_cap": 256}, 3, True),  # calendar queue; the plan's author masks drawn over 3, 4 and 7 nodes
    (300, 16, (4, 5, 6, 16), 800, {}, 3, False),  # 5 / 6: where a plain handle's queue and kernel family change
    (400, 40, (32, 33, 40), 600, {}, 3, False),  # the author masks widen past 32
    (500, 64, (4, 64), 600, {}, 3, False),
    (600, 7, (2, 5, 7), 5000, {"round_cap": 768}, 0, False),  # beyond the calendar's horizon: binary heap
]


def plain_of(ps, n):
    """Set `ps` as a full-size set of a layout of its own committee n (its rights truncated to n)."""
    return ParamSet(ps.network_delay, ps.node_config, ps.faults, ps.voting_rights)


@pytest.mark.parametrize("seed0,nodes,sizes,max_clock,shared,qmode,partitions", SHAPES)
@pytest.mark.parametrize("ct", [False, True])
def test_committee_sweep_matches_the_oracle_per_instance(oracle, harness, seed0, nodes, sizes, max_clock, shared, qmode, partitions, ct):
    """The 12 parameter sets crossed with the committee sizes (each with no fault, a silent node or a zero-weight node), instance
    i on set i % num_sets: every instance equals the oracle run as a plain configuration of its set's size, the absent nodes read
    0; the proposers, commit times and state keys equal a sweep of that set alone in a layout of its own size."""
    sets = cross_sizes(SETS, sizes, partitions)
    count = 2 * len(sets)
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    flags = FLAGS_CT if ct else 0
    name = harness.kernel_info(seeds, nodes, max_clock, sets, set_of, faults=True, flags=flags, **shared)[0]
    assert ",%d," % qmode in name and name.startswith("lbft_ct_sweep_" if ct else "lbft_sweep_"), name
    h = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, flags=flags, **shared)
    o = oracle_per_committee(oracle, seeds, nodes, max_clock, sets, set_of, **shared)
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert_same(o, h, "committee sweep layout %d" % nodes)
    n_of = np.array([size_of(p, nodes) for p in sets])[set_of]
    absent = np.arange(nodes)[None, :] >= n_of[:, None]
    assert (h.lc_round[absent] == 0).all() and (h.commit_counts[absent] == 0).all() and (h.last_states[absent] == 0).all()
    assert h.commit_counts.sum() > 0
    if ct:
        assert (h.committed[absent] == -1).all()
    for s in range(0, len(sets), 5):
        idx = np.nonzero(set_of == s)[0]
        n = size_of(sets[s], nodes)
        one = harness.run(seeds[idx], n, max_clock, [plain_of(sets[s], n)], np.zeros(len(idx)), faults=True, mode="rights", flags=flags,
                          **shared)
        np.testing.assert_array_equal(h.proposers[idx], one.proposers, err_msg="set %d proposers" % s)
        np.testing.assert_array_equal(h.last_states[idx][:, :n], one.last_states)
        np.testing.assert_array_equal(h.counters[idx][:, :8], one.counters[:, :8])
        if ct:
            np.testing.assert_array_equal(h.committed[idx][:, :n], one.committed, err_msg="set %d committed" % s)
            np.testing.assert_array_equal(h.proposed[idx], one.proposed, err_msg="set %d proposed" % s)


def test_absent_nodes_are_written(harness):
    """Committees of 1 and 2 in a layout of 4, over outputs filled with garbage before the run: commit count, last committed
    round and state key 0, commit times -1, and the active round of the present nodes only."""
    sets = [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(), num_nodes=n) for n in (1, 2)]
    seeds = np.arange(1, 17, dtype=np.uint64)
    set_of = np.arange(16) % 2
    h = harness.run(seeds, 4, 1000, sets, set_of, flags=FLAGS_CT, round_cap=256)
    for s, n in enumerate((1, 2)):
        idx = set_of == s
        assert (h.commit_counts[idx][:, n:] == 0).all() and (h.lc_round[idx][:, n:] == 0).all() and (h.last_states[idx][:, n:] == 0).all()
        assert (h.committed[idx][:, n:] == -1).all()
        assert (h.commit_counts[idx][:, :n] > 0).all()
        one = harness.run(seeds[idx], n, 1000, [ParamSet(sets[s].network_delay)], np.zeros(idx.sum()), mode="plain", flags=FLAGS_CT,
                          round_cap=256)
        np.testing.assert_array_equal(h.counters[idx][:, 6], one.counters[:, 6])  # (the largest active round)


def test_leader_tables_are_the_plain_committees_and_deduplicated(harness):
    """Each set's leader table equals that of the plain handle of its committee and rights (a row padded with zeros draws the
    leaders of the n-node row); equal (size, rights) pairs share one table."""
    rows = {4: [None, (3, 1, 1, 1)], 7: [None, (1, 1, 1, 1, 1, 1, 5)], 16: [None]}
    sets = [ParamSet(SETS[k % 3].network_delay, SETS[k % 3].node_config, voting_rights=r, num_nodes=n) for k in range(3)
            for n, rs in rows.items() for r in rs]
    seeds = np.arange(1, 1 + 2 * len(sets), dtype=np.uint64)
    set_of = np.arange(len(seeds)) % len(sets)
    name, words, leader_bytes, records, tables = harness.kernel_info(seeds, 16, 1000, sets, set_of, leaders=True, round_cap=256)
    assert records == 0b111
    span = 257
    assert leader_bytes == 5 * span  # 5 distinct (size, rights) pairs of 15 sets
    for s, p in enumerate(sets):
        n = size_of(p, 16)
        plain = harness.kernel_info(seeds[:2], n, 1000, [ParamSet(p.network_delay, p.node_config)], [0, 0], mode="plain", leaders=True,
                                    round_cap=256, voting_rights=p.voting_rights)[4]
        np.testing.assert_array_equal(tables[s * span:(s + 1) * span], plain[:span], err_msg="set %d (n = %d)" % (s, n))
        assert tables[s * span:(s + 1) * span].max() < n


def test_full_size_committees_are_rights_and_plain_sweeps(harness, monkeypatch):
    """Every set at the layout's size: the kernel and words per instance of lbft_create_sweep_rights with all-ones rows and of
    lbft_create_sweep (each tests/sweep_support.KERNEL_CASES shape, automatic and forced to each family), and identical outputs."""
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
            sets = [ParamSet(SETS[k].network_delay, SETS[k].node_config, num_nodes=nodes) for k in (0, 1)]
            got = harness.kernel_info(seeds, nodes, max_clock, sets, set_of, **kw)
            assert got[:2] == harness.kernel_info(seeds, nodes, max_clock, sets, set_of, mode="rights", **kw)[:2], (family, name)
            assert got[:2] == harness.kernel_info(seeds, nodes, max_clock, sets, set_of, mode="plain", **kw)[:2], (family, name)
            assert got[3] == 0b111
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    fields = ("commit_counts", "last_states", "counters", "status", "lc_round", "proposers", "committed", "proposed")
    for name, count, nodes, kw in KERNEL_CASES:  # the outputs, on a batch small enough for the host core
        max_clock = kw.get("max_clock", 1000)
        shared = {k: v for k, v in kw.items() if k != "max_clock"}
        seeds = np.arange(11, 11 + 24, dtype=np.uint64)
        set_of = np.arange(24) % 3
        for row in (None, (3,) + (1,) * (nodes - 1)):
            sets = [ParamSet(p.network_delay, p.node_config, voting_rights=row, num_nodes=nodes) for p in SETS[:3]]
            a = harness.run(seeds, nodes, max_clock, sets, set_of, flags=FLAGS_CT, **shared)
            b = harness.run(seeds, nodes, max_clock, sets, set_of, mode="rights", flags=FLAGS_CT, **shared)
            for field in fields:
                np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="%s %s" % (name, field))
            if row is None:
                c = harness.run(seeds, nodes, max_clock, sets, set_of, mode="plain", flags=FLAGS_CT, **shared)
                for field in fields:
                    np.testing.assert_array_equal(getattr(a, field), getattr(c, field), err_msg="%s %s" % (name, field))
    # per-set faults as well: against lbft_create_sweep_faults
    sets = [ParamSet(p.network_delay, p.node_config, f, num_nodes=4) for p in SETS[:2] for f in (FaultSet((1,)), FaultSet((), 4, 150))]
    seeds = np.arange(5, 5 + 32, dtype=np.uint64)
    set_of = np.arange(32) % 4
    a = harness.run(seeds, 4, 1000, sets, set_of, faults=True)
    b = harness.run(seeds, 4, 1000, sets, set_of, faults=True, mode="plain")
    for field in ("commit_counts", "last_states", "counters", "status", "proposers"):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)


def test_block_latency_per_group_matches_numpy(harness):
    """lbft_block_latency_stats_groups over a committee sweep (the product's checks, each group's weights, the serial threshold
    time) against numpy over the same commit times, at each set's named thresholds: "all" and "quorum" are per committee."""
    sets = cross_sizes(SETS[:3], (3, 4, 7), partitions=True)
    count = 3 * len(sets)
    seeds = np.arange(50, 50 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    rows = rights_rows(sets, 7)
    totals = rows.sum(axis=1).astype(np.int64)
    assert sorted(set(totals.tolist())) == [3, 4, 6]
    spec = make_spec(1024, 1, 0, None)
    for name in THRESHOLD_NAMES:
        W = np.array([resolve_threshold(name, int(t)) for t in totals])
        h = harness.run(seeds, 7, 1000, sets, set_of, faults=True, cap=256, spec=spec, thresholds=W, flags=FLAGS_CT)
        parts = [numpy_block_stats(h.committed[set_of == g], h.proposed[set_of == g], h.status[set_of == g],
                                   np.zeros((set_of == g).sum(), np.int64), 1, rows[g].astype(np.int64), int(W[g])) for g in range(len(sets))]
        cat = lambda f: np.concatenate([getattr(p, f) for p in parts])  # noqa: E731
        summary = np.zeros(len(sets), LATENCY_SUMMARY_DTYPE)
        for f in LATENCY_SUMMARY_DTYPE.names:
            summary[f] = cat(f)
        want = BlockLatencyStats(summary, cat("unreached"), np.concatenate([p.hist for p in parts]), 1, W)
        assert_same_block_stats(h.stats, want, name)
        assert h.stats.samples.sum() > 0
    # one W for every group is refused above the least committee's total, naming that group
    with pytest.raises(RuntimeError, match=r"thresholds\[0\] must be in 1..total voting rights of group 0 \(3\)"):
        harness.run(seeds, 7, 1000, sets, set_of, faults=True, spec=spec, thresholds=[4] * len(sets), flags=FLAGS_CT)


def _create(lib, cfg, sets, faults, vr, sizes, num_sets, set_of):
    h = ctypes.c_void_p()
    rc = lib.lbft_create_sweep_committees(ctypes.byref(cfg), sets, faults, None if vr is None else ctypes.c_void_p(vr.ctypes.data),
                                          None if sizes is None else ctypes.c_void_p(sizes.ctypes.data), num_sets,
                                          None if set_of is None else ctypes.c_void_p(set_of.ctypes.data), ctypes.byref(h))
    assert h.value is None
    return rc, lib.lbft_last_error().decode()


def test_committee_sweep_refusals(lib):
    """Everything lbft_create_sweep_committees refuses, with LBFT_ERR_INVALID and before any device work (so without a GPU too)."""
    cfg, keep = make_config(np.arange(1, 9, dtype=np.uint64), 7)
    ok = np.arange(8, dtype=np.uint32) % 4
    sizes = np.array([3, 4, 7, 5], np.uint32)
    good = [ParamSet(SETS[k].network_delay, SETS[k].node_config) for k in range(4)]
    sets = c_sets(good)
    # what lbft_create_sweep / _rights refuse, with their messages
    for num_sets, set_of, want in ((0, ok, "num_sets"), (9, np.arange(8, dtype=np.uint32), "num_sets"), (4, None, "NULL"),
                                   (4, np.full(8, 4, np.uint32), "index >= num_sets")):
        rc, msg = _create(lib, cfg, sets, None, None, sizes, num_sets, set_of)
        assert rc == -1 and want in msg, msg
    assert _create(lib, cfg, None, None, None, sizes, 4, ok) == (-1, "sets and set_of_instance must not be NULL")
    bad = ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=0))
    rc, msg = _create(lib, cfg, c_sets([good[0], good[1], bad, good[3]]), None, None, sizes, 4, ok)
    assert rc == -1 and msg.startswith("parameter set 2: delta = 0"), msg
    cfg_v, keep_v = make_config(np.arange(1, 9, dtype=np.uint64), 7, voting_rights=[1] * 7)
    rc, msg = _create(lib, cfg_v, sets, None, None, sizes, 4, ok)
    assert msg == "a rights sweep takes its voting rights per set only: lbft_config.voting_rights must be NULL", msg
    cfg_s, keep_s = make_config(np.arange(1, 9, dtype=np.uint64), 7, silent=[0, 1, 0, 0, 0, 0, 0])
    assert "per set only" in _create(lib, cfg_s, sets, c_faults(good), None, sizes, 4, ok)[1]
    cfg_f, keep_f = make_config(np.arange(1, 9, dtype=np.uint64), 7, flags=_lib.FLAG_RESUMABLE)
    assert "sweep handles take no flags" in _create(lib, cfg_f, sets, None, None, sizes, 4, ok)[1]
    # the sizes
    assert _create(lib, cfg, sets, None, None, None, 4, ok) == (-1, "committee_sizes must not be NULL")
    for s, n in ((1, 0), (3, 8)):
        bad_sizes = sizes.copy()
        bad_sizes[s] = n
        rc, msg = _create(lib, cfg, sets, None, None, bad_sizes, 4, ok)
        assert (rc, msg) == (-1, "parameter set %d: committee size must be in 1..lbft_config.num_nodes (the layout's committee)" % s)
    # the rights rows: 0 past the set's size, a total > 0 within it, entries <= 2^24
    vr = np.zeros((4, 7), np.uint64)
    for s, n in enumerate(sizes):
        vr[s, :n] = 1
    for s, col, val, want in ((0, 3, 1, "voting_rights has a non-zero entry at or past the set's committee size"),
                              (3, 6, 2, "voting_rights has a non-zero entry at or past the set's committee size"),
                              (1, 0, 1 << 25, "voting_rights entries must be <= 2^24")):
        bad_vr = vr.copy()
        bad_vr[s, col] = val
        assert _create(lib, cfg, sets, None, bad_vr, sizes, 4, ok) == (-1, "parameter set %d: %s" % (s, want))
    zero = vr.copy()
    zero[0, :3] = 0
    assert _create(lib, cfg, sets, None, zero, sizes, 4, ok) == (-1, "parameter set 0: total voting rights must be > 0")
    # silent nodes at or past a set's size: per set, and shared
    faulty = [ParamSet(p.network_delay, p.node_config, FaultSet((n - 1,) if s != 1 else (4,))) for s, (p, n) in enumerate(zip(good, sizes))]
    assert _create(lib, cfg, sets, c_faults(faulty), None, sizes, 4, ok) == (-1, "parameter set 1: a silent node is at or past the set's committee size")
    faulty[1] = ParamSet(good[1].network_delay, good[1].node_config, FaultSet((7,)))  # (past the layout as well)
    assert _create(lib, cfg, sets, c_faults(faulty), None, sizes, 4, ok) == (-1, "parameter set 1: silent_mask has a bit at or above num_nodes")
    cfg_s3, keep_s3 = make_config(np.arange(1, 9, dtype=np.uint64), 7, silent=[0, 0, 0, 1, 0, 0, 0])
    assert _create(lib, cfg_s3, sets, None, None, sizes, 4, ok) == (-1, "parameter set 0: a silent node is at or past the set's committee size")
    # a layout of more than 64 nodes
    cfg_b, keep_b = make_config(np.arange(1, 9, dtype=np.uint64), 65)
    assert _create(lib, cfg_b, sets, None, None, sizes, 4, ok) == (-1, "parameter set 0: num_nodes must be in 1..64")
    assert lib.lbft_create_sweep_committees(None, sets, None, None, None, 4, None, ctypes.byref(ctypes.c_void_p())) == -1


def test_refusals_reach_the_host_setup(harness):
    """The same checks through the host harness (the product's HostSetup), where a valid call builds: a set whose committee of 1
    carries a partition plan (its author masks are empty), and the largest committee's silent node on a set of that size."""
    sets = [ParamSet(SETS[0].network_delay, SETS[0].node_config, FaultSet((), 2, 100), num_nodes=1),
            ParamSet(SETS[1].network_delay, SETS[1].node_config, FaultSet((6,)), num_nodes=7)]
    harness.check(np.arange(1, 5, dtype=np.uint64), 7, 1000, sets, [0, 1, 0, 1], faults=True)
    with pytest.raises(RuntimeError, match="parameter set 0: a silent node is at or past the set's committee size"):
        harness.check(np.arange(1, 5, dtype=np.uint64), 7, 1000, sets[::-1], [0, 1, 0, 1], faults=True, sizes=[1, 7])


def test_grid_committee_axis_and_python_refusals():
    """SweepSimulator.grid(num_nodes=[...]): the fastest axis, after faults, in a layout of the largest size; no voting-rights list
    with it; sizes above the layout's and shared rights refused; totals per group and each instance's committee."""
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30)]
    fl = [FaultSet(), FaultSet((0,))]
    sizes = [4, 7, 10, 16]
    sim = SweepSimulator.grid([5, 6], delays, configs, num_nodes=sizes, faults=fl)
    assert sim.num_nodes == 16 and sim.num_instances == 2 * 48 and len(sim.param_sets) == 48
    for i, d in enumerate(delays):
        for j, n in enumerate(configs):
            for f, fs in enumerate(fl):
                for k, size in enumerate(sizes):
                    assert sim.param_sets[((i * len(configs) + j) * len(fl) + f) * len(sizes) + k] == ParamSet(d, n, fs, None, size)
    no_faults = SweepSimulator.grid([5], delays, configs, num_nodes=sizes)
    assert no_faults.param_sets == [ParamSet(d, n, FaultSet(), None, k) for d in delays for n in configs for k in sizes]
    np.testing.assert_array_equal(sim.group_voting_rights(), np.tile(sizes, 12))
    np.testing.assert_array_equal(sim.nodes_of_instance(), np.repeat(np.tile(sizes, 12), 2))
    with pytest.raises(ValueError, match="group_voting_rights"):
        sim.total_voting_rights()
    with pytest.raises(ValueError, match="not both"):
        SweepSimulator.grid([5], delays, configs, num_nodes=sizes, voting_rights=[(1,) * 4])
    with pytest.raises(ValueError, match="parameter set 1: num_nodes"):
        SweepSimulator(np.arange(4), 4, [ParamSet(num_nodes=4), ParamSet(num_nodes=5)], [0, 1, 0, 1])
    with pytest.raises(ValueError, match="parameter set 0: num_nodes"):
        SweepSimulator(np.arange(4), 4, [ParamSet(num_nodes=0)], [0, 0, 0, 0])
    mixed = SweepSimulator(np.arange(4), 7, [ParamSet(voting_rights=(3, 1, 1), num_nodes=3), ParamSet()], [0, 1, 0, 1])
    np.testing.assert_array_equal(mixed.group_voting_rights(), [5, 7])
    np.testing.assert_array_equal(mixed.nodes_of_instance(), [3, 7, 3, 7])
    np.testing.assert_array_equal(mixed._rights_table(), [[3, 1, 1, 0, 0, 0, 0], [1] * 7])
    with pytest.raises(ValueError, match="one entry per node of the set"):
        SweepSimulator(np.arange(4), 7, [ParamSet(voting_rights=(1,) * 4, num_nodes=3)], [0, 0, 0, 0]).create(1000)
    with pytest.raises(ValueError, match="per set only"):
        SweepSimulator(np.arange(4), 4, [ParamSet(num_nodes=3)], [0, 0, 0, 0], voting_rights=[1, 1, 1, 1])
    plain = SweepSimulator.grid([5], delays, configs, num_nodes=4)
    assert (plain.nodes_of_instance() == 4).all() and (plain.group_voting_rights() == 4).all()


def test_committee_signatures_match_the_header():
    """lbft_create_sweep_committees: the extern declarations of the Rust shim and the ctypes bindings against include/lbft.h."""
    from tests.test_rust_shim import c_functions, rust_functions
    c = c_functions()
    assert c["lbft_create_sweep_committees"][0] == ["ptr:lbft_config", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "ptr:u32",
                                                    "u32", "ptr:u32", "ptr:lbft_sim"]
    r = rust_functions()
    assert r["lbft_create_sweep_committees"][0] == ["ptr:LbftConfig", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "ptr:u32",
                                                    "u32", "ptr:u32", "ptr:*mut LbftSim"], r["lbft_create_sweep_committees"]
    lib = _lib.load()
    assert len(lib.lbft_create_sweep_committees.argtypes) == 8
    assert "lbft_create_sweep_committees" in _lib.EXPORTS
