"""Links sweeps (lbft_create_sweep_links) without a GPU: the SW and SW + CT device cores compiled for the host
(tests/hostcore/link_hostcore.cpp) against the oracle run once per set with its link latencies, instance by instance, in every
queue mode, with faults, voting rights and committee sizes; all-zero matrices against the same sweep through the existing entry
points; the deduplication of equal matrices; every refusal and its message; the link oracle's term on its own, and the link
oracle without links against the oracle; and
SweepSimulator.grid's link axis, regional_latency and the Python refusals."""
import ctypes

import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _build, _lib, regional_latency
from tests.committee_support import cross_sizes, size_of
from tests.link_support import LinkHarness, LinkOracle, link_table, matrices, oracle_per_set, set_config
from tests.support import assert_same, make_config
from tests.sweep_support import KERNEL_CASES, SETS, c_sets

FLAGS_CT = _lib.FLAG_COMMIT_TIMES


@pytest.fixture(scope="module")
def harness():
    return LinkHarness()


@pytest.fixture(scope="module")
def link_oracle():
    return LinkOracle()


@pytest.fixture(scope="module")
def lib():
    _build.build_product()
    return _lib.load()


def with_variants(sets, n, partitions):
    """Set k with variant k % 3: no fault; a silent node (node k % n); a zero-weight node 0; every other set with a partition
    plan when `partitions`."""
    out = []
    for k, p in enumerate(sets):
        plan = (2, 200) if partitions and k % 2 else (0, 0)
        silent = (k % n,) if k % 3 == 1 else ()
        rights = (0,) + (1,) * (n - 1) if k % 3 == 2 else None
        out.append(ParamSet(p.network_delay, p.node_config, FaultSet(silent, *plan), rights))
    return out


def crossed(nodes, sizes, partitions):
    """The 12 sets of tests/sweep_support.SETS with fault / rights variants (and committee sizes), each crossed with the four
    matrices of its committee."""
    base = cross_sizes(SETS, sizes, partitions) if sizes else with_variants(SETS, nodes, partitions)
    return [ParamSet(p.network_delay, p.node_config, p.faults, p.voting_rights, p.num_nodes, m)
            for p in base for _, m in matrices(size_of(p, nodes))]


SHAPES = [
    # (first seed, layout's committee, committee sizes or None, max_clock, shared, queue mode, partition plans)
    (100, 4, None, 1000, {"round_cap": 256, "payload_cap": 64}, 2, False),  # shared-memory scan queue (slow links: more in flight)
    (200, 5, None, 1000, {"round_cap": 256, "payload_cap": 128, "queue_cap": 400, "force": "thread"}, 1, True),  # HBM scan queue (the thread kernel's)
    (300, 7, None, 1500, {"round_cap": 256, "payload_cap": 128}, 3, True),  # calendar queue
    (400, 7, None, 5000, {"round_cap": 768, "payload_cap": 128}, 0, False),  # beyond the calendar's horizon: binary heap
    (500, 7, (3, 4, 7), 1500, {"round_cap": 256, "payload_cap": 128}, 3, True),  # committee sizes: each matrix in its committee's corner
]


@pytest.mark.parametrize("seed0,nodes,sizes,max_clock,shared,qmode,partitions", SHAPES)
@pytest.mark.parametrize("ct", [False, True])
def test_link_sweep_matches_the_oracle_per_instance(harness, link_oracle, monkeypatch, seed0, nodes, sizes, max_clock, shared, qmode,
                                                    partitions, ct):
    """Every instance equals the oracle run as a plain configuration of its set (delay, NodeConfig, faults, rights, committee
    size) with its set's link latencies: commit counts, state keys, the counters the reference has (events processed by kind,
    cancelled timers, creation stamps, largest active round, RNG draws, scheduled notifications), commit logs and commit
    times."""
    shared = dict(shared)
    if "force" in shared:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", shared.pop("force"))
    sets = crossed(nodes, sizes, partitions)
    count = 2 * len(sets)
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    flags = FLAGS_CT if ct else 0
    name, _, _, records = harness.kernel_info(seeds, nodes, max_clock, sets, set_of, faults=True, flags=flags, **shared)
    assert ",%d," % qmode in name and name.startswith("lbft_ct_sweep_" if ct else "lbft_sweep_"), name
    assert records & 0b1011 == 0b1011 and bool(records & 4) == bool(sizes)
    h = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, flags=flags, **shared)
    o = oracle_per_set(link_oracle, seeds, nodes, max_clock, sets, set_of, **shared)
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert_same(o, h, "links sweep layout %d" % nodes)
    assert h.commit_counts.sum() > 0
    for i in range(0, count, 7):  # commit logs, and with CT commit times, of a sample of instances
        ps = sets[set_of[i]]
        n, kw, m = set_config(ps, nodes)
        kw.update(shared)
        log = link_oracle.commit_log(seeds[i:i + 1], n, 0, int(np.argmax(h.commit_counts[i, :n])), max_clock, m, **kw)
        assert [p for p, _, _ in log][:128] == h.proposers[i, :len(log)].tolist(), i
        if ct:
            committed, proposed, counts = harness.oracle_commit_times(seeds[i:i + 1], n, max_clock, m, **kw)
            np.testing.assert_array_equal(counts[0], h.commit_counts[i, :n])
            np.testing.assert_array_equal(committed[0], h.committed[i, :n], err_msg="instance %d committed" % i)
            np.testing.assert_array_equal(proposed[0], h.proposed[i], err_msg="instance %d proposed" % i)


def test_links_change_the_run(harness):
    """The same seeds under a non-zero matrix and under zeros differ (the term is applied), and a larger uniform term delays the
    first commit of every instance."""
    base = ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig())
    n = 4
    zero = ParamSet(base.network_delay, base.node_config, link_latency=((0,) * n,) * n)
    slow = ParamSet(base.network_delay, base.node_config, link_latency=((40,) * n,) * n)
    seeds = np.arange(1, 33, dtype=np.uint64)
    set_of = np.arange(32) % 2
    h = harness.run(seeds, n, 1000, [zero, slow], set_of, flags=FLAGS_CT, round_cap=256)
    a, b = h.committed[set_of == 0][:, :, 0], h.committed[set_of == 1][:, :, 0]
    assert (b[b >= 0].min() > a[a >= 0].min()) and (h.commit_counts[set_of == 1].sum() < h.commit_counts[set_of == 0].sum())


def test_all_zero_matrices_equal_the_sweep_without_links(harness, monkeypatch):
    """A links sweep whose matrices are all zero: the kernel and words per instance of the same call through the existing entry
    points (each tests/sweep_support.KERNEL_CASES shape, automatic and forced to each family), and every output identical,
    counters included, with faults, rights and committee sizes."""
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
            zero = ((0,) * nodes,) * nodes
            sets = [ParamSet(SETS[k].network_delay, SETS[k].node_config, voting_rights=(1,) * nodes, link_latency=zero) for k in (0, 1)]
            got = harness.kernel_info(seeds, nodes, max_clock, sets, set_of, **kw)
            assert got[:2] == harness.kernel_info(seeds, nodes, max_clock, sets, set_of, links=False, **kw)[:2], (family, name)
            assert got[3] == 0b1011
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    fields = ("commit_counts", "last_states", "counters", "status", "lc_round", "proposers", "committed", "proposed")
    for seed0, nodes, sizes, max_clock, shared, _, partitions in SHAPES:
        shared = {k: v for k, v in shared.items() if k != "force"}
        base = cross_sizes(SETS[:4], sizes, partitions) if sizes else with_variants(SETS[:6], nodes, partitions)
        sets = [ParamSet(p.network_delay, p.node_config, p.faults, p.voting_rights, p.num_nodes, matrices(size_of(p, nodes))[3][1])
                for p in base]
        seeds = np.arange(seed0, seed0 + 3 * len(sets), dtype=np.uint64)
        set_of = np.arange(len(seeds)) % len(sets)
        a = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, flags=FLAGS_CT, **shared)
        b = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, links=False, flags=FLAGS_CT, **shared)
        for field in fields:
            np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="layout %d %s" % (nodes, field))
    # shared faults and shared voting rights (faults and voting_rights NULL): the configuration's apply to every set
    sets = [ParamSet(p.network_delay, p.node_config, link_latency=((0,) * 7,) * 7) for p in SETS[:3]]
    seeds = np.arange(70, 94, dtype=np.uint64)
    set_of = np.arange(24) % 3
    shared = dict(voting_rights=[3, 1, 1, 1, 1, 1, 2], silent=[0, 0, 1, 0, 0, 0, 0], partition_windows=2, partition_max_len=100)
    a = harness.run(seeds, 7, 1000, sets, set_of, flags=FLAGS_CT, **shared)
    b = harness.run(seeds, 7, 1000, sets, set_of, links=False, flags=FLAGS_CT, **shared)
    for field in fields:
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="shared " + field)


def test_equal_matrices_share_one_table(harness):
    """One device table of N x N u16 per distinct matrix, whatever the sets' other fields."""
    mats = matrices(7)
    sets = [ParamSet(SETS[k % 4].network_delay, SETS[k % 4].node_config, link_latency=mats[k % 3][1]) for k in range(10)]
    seeds = np.arange(1, 21, dtype=np.uint64)
    set_of = np.arange(20) % 10
    assert harness.kernel_info(seeds, 7, 1000, sets, set_of)[2] == 3 * 49 * 2
    sets = [ParamSet(p.network_delay, p.node_config, link_latency=mats[0][1]) for p in SETS[:5]]
    assert harness.kernel_info(seeds[:10], 7, 1000, sets, np.arange(10) % 5)[2] == 49 * 2


def _create(lib, cfg, sets, faults, vr, sizes, links, num_sets, set_of):
    h = ctypes.c_void_p()
    ptr = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib.lbft_create_sweep_links(ctypes.byref(cfg), sets, faults, ptr(vr), ptr(sizes), ptr(links), num_sets, ptr(set_of),
                                     ctypes.byref(h))
    assert h.value is None
    return rc, lib.lbft_last_error().decode()


def test_link_sweep_refusals(lib):
    """Everything lbft_create_sweep_links refuses, with LBFT_ERR_INVALID and before any device work (so without a GPU too)."""
    cfg, keep = make_config(np.arange(1, 9, dtype=np.uint64), 7)
    ok = np.arange(8, dtype=np.uint32) % 4
    good = [ParamSet(SETS[k].network_delay, SETS[k].node_config) for k in range(4)]
    sets = c_sets(good)
    links = np.zeros((4, 7, 7), np.uint32)
    links[:, :3, :3] = 5
    # what the other sweeps refuse, with their messages
    assert _create(lib, cfg, sets, None, None, None, links, 0, ok)[1].startswith("num_sets")
    assert _create(lib, cfg, None, None, None, None, links, 4, ok) == (-1, "sets and set_of_instance must not be NULL")
    bad = ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=0))
    rc, msg = _create(lib, cfg, c_sets([good[0], bad, good[2], good[3]]), None, None, None, links, 4, ok)
    assert rc == -1 and msg.startswith("parameter set 1: delta = 0"), msg
    sizes = np.array([3, 4, 7, 5], np.uint32)
    vr = np.ones((4, 7), np.uint64)
    assert _create(lib, cfg, sets, None, vr, sizes, links, 4, ok) == (
        -1, "parameter set 0: voting_rights has a non-zero entry at or past the set's committee size")
    cfg_v, keep_v = make_config(np.arange(1, 9, dtype=np.uint64), 7, voting_rights=[1] * 7)
    assert "per set only" in _create(lib, cfg_v, sets, None, vr, None, links, 4, ok)[1]
    assert "per set only" in _create(lib, cfg_v, sets, None, None, sizes, links, 4, ok)[1]
    # the matrices
    assert _create(lib, cfg, sets, None, None, None, None, 4, ok) == (-1, "link_latency must not be NULL")
    big = links.copy()
    big[2, 1, 0] = 65536
    assert _create(lib, cfg, sets, None, None, None, big, 4, ok) == (-1, "parameter set 2: link_latency entries must be <= 65535")
    for s, a, b in ((0, 3, 0), (1, 0, 4), (3, 6, 6)):  # a row, a column and the diagonal at or past the set's size
        past = links.copy()
        past[s, a, b] = 1
        assert _create(lib, cfg, sets, None, None, sizes, past, 4, ok) == (
            -1, "parameter set %d: link_latency has a non-zero entry in a row or column at or past the set's committee size" % s)
    full = links.copy()
    full[2, 6, 6] = 65535  # set 2's committee is the layout's: its whole matrix is in range
    cfg_b, keep_b = make_config(np.arange(1, 9, dtype=np.uint64), 65)
    assert _create(lib, cfg_b, sets, None, None, None, np.zeros((4, 65, 65), np.uint32), 4, ok)[1] == "parameter set 0: num_nodes must be in 1..64"
    assert lib.lbft_create_sweep_links(None, sets, None, None, None, None, 4, None, ctypes.byref(ctypes.c_void_p())) == -1


def test_refusals_reach_the_host_setup(harness):
    """The same checks through the host harness (the product's HostSetup), where a valid call builds: entries of 65535 and a
    non-zero diagonal, with committee sizes, faults and no rights."""
    seeds = np.arange(1, 5, dtype=np.uint64)
    m = np.full((2, 7, 7), 65535, np.uint32)
    m[0, 3:, :] = 0
    m[0, :, 3:] = 0
    sets = [ParamSet(SETS[0].network_delay, SETS[0].node_config, FaultSet((1,)), num_nodes=3),
            ParamSet(SETS[1].network_delay, SETS[1].node_config, FaultSet((), 2, 100), num_nodes=7)]
    harness.check(seeds, 7, 1000, sets, [0, 1, 0, 1], faults=True, table=m)
    m[0, 2, 5] = 1
    with pytest.raises(RuntimeError, match="parameter set 0: link_latency has a non-zero entry"):
        harness.check(seeds, 7, 1000, sets, [0, 1, 0, 1], faults=True, table=m)


def test_oracle_schedules_each_network_event_after_its_link(link_oracle):
    """The oracle's extension on its own: under a variance-0 delay model every delay is d = 10, so each network event of the
    trace (notifications, requests and responses, partitioned ones included) is due at its send clock + 10 +
    M[sender][receiver], and without links at its send clock + 10."""
    n = 5
    m = np.array(matrices(n)[1][1], np.uint32)  # asymmetric, with a non-zero diagonal
    kw = dict(delay_mean=10.0, delay_variance=0.0, partition_windows=2, partition_max_len=200)
    seeds = np.arange(3, 6, dtype=np.uint64)
    for inst in range(len(seeds)):
        rows = link_oracle.trace(seeds, n, inst, 1000, m, **kw)
        kinds, recv, send, sent, due = rows.T
        assert set(kinds.tolist()) == {0, 1, 2}, "notifications, requests and responses"
        np.testing.assert_array_equal(due, sent + 10 + m[send, recv])
        plain = link_oracle.trace(seeds, n, inst, 1000, None, **kw)
        np.testing.assert_array_equal(plain[:, 4], plain[:, 3] + 10)
    # a zero matrix leaves the trace as it is without one
    np.testing.assert_array_equal(link_oracle.trace(seeds, n, 0, 1000, np.zeros((n, n), np.uint32), **kw),
                                  link_oracle.trace(seeds, n, 0, 1000, None, **kw))


def test_link_oracle_without_links_is_the_oracle(oracle, link_oracle):
    """The link oracle restates the oracle's send path: with an all-zero matrix every output of every instance (commit counts,
    state keys, all counters, status) is the oracle's own, over the 12 sets with silent nodes, partition plans and rights."""
    n = 7
    for k, p in enumerate(with_variants(SETS, n, True)):
        _, kw, m = set_config(p, n)
        seeds = np.arange(40 * k, 40 * k + 12, dtype=np.uint64)
        a = link_oracle.run(seeds, n, 1200, np.zeros((n, n), np.uint32), round_cap=256, **kw)
        b = oracle.run(seeds, n, 1200, round_cap=256, **kw)
        for field in ("commit_counts", "last_states", "counters", "status"):
            np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="set %d %s" % (k, field))
        assert a.commit_counts.sum() > 0


def test_regional_latency():
    """regional_latency expands a region map and a region-to-region matrix (diagonal: within a region) into the node matrix,
    directions kept; refusals."""
    between = [[1, 50, 80], [45, 2, 60], [85, 65, 3]]
    m = regional_latency([2, 0, 0, 1], between)
    assert m == ((3, 85, 85, 65), (80, 1, 1, 50), (80, 1, 1, 50), (60, 45, 45, 2))
    assert isinstance(m, tuple) and all(isinstance(r, tuple) for r in m)
    assert ParamSet(link_latency=m) == ParamSet(link_latency=np.array(m))  # stored as a tuple of tuples: hashable, comparable
    hash(ParamSet(link_latency=m))
    with pytest.raises(ValueError, match="square"):
        regional_latency([0, 1], [[1, 2, 3]])
    with pytest.raises(ValueError, match="region outside 0..2"):
        regional_latency([0, 3], between)


def test_grid_link_axis_and_python_refusals():
    """SweepSimulator.grid(link_latency=[...]): the fastest axis, after faults and after the voting-rights axis; not with a list
    of committee sizes; matrices of the wrong size or range refused; the table passed to the C ABI."""
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30)]
    fl = [FaultSet(), FaultSet((0,))]
    stake = [(1,) * 7, (3, 1, 1, 1, 1, 1, 1)]
    mats = [m for _, m in matrices(7)[:3]]
    sim = SweepSimulator.grid([5, 6], delays, configs, num_nodes=7, faults=fl, voting_rights=stake, link_latency=mats)
    assert sim.num_instances == 2 * 72 and len(sim.param_sets) == 72
    for i, d in enumerate(delays):
        for j, n in enumerate(configs):
            for f, fs in enumerate(fl):
                for v, row in enumerate(stake):
                    for k, m in enumerate(mats):
                        p = (((i * len(configs) + j) * len(fl) + f) * len(stake) + v) * len(mats) + k
                        assert sim.param_sets[p] == ParamSet(d, n, fs, row, None, m)
    no_faults = SweepSimulator.grid([5], delays, configs, num_nodes=7, link_latency=mats)
    assert no_faults.param_sets == [ParamSet(d, n, FaultSet(), None, None, m) for d in delays for n in configs for m in mats]
    np.testing.assert_array_equal(no_faults._link_table(), link_table(no_faults.param_sets, 7))
    with pytest.raises(ValueError, match="not both"):
        SweepSimulator.grid([5], delays, configs, num_nodes=[4, 7], link_latency=mats)
    mixed = SweepSimulator(np.arange(4), 7, [ParamSet(num_nodes=3, link_latency=matrices(3)[0][1]), ParamSet()], [0, 1, 0, 1])
    t = mixed._link_table()
    assert t.shape == (2, 7, 7) and (t[1] == 0).all() and (t[0, 3:] == 0).all() and (t[0, :, 3:] == 0).all()
    np.testing.assert_array_equal(t[0, :3, :3], matrices(3)[0][1])
    assert SweepSimulator.grid([5], delays, configs, num_nodes=7)._link_table() is None
    with pytest.raises(ValueError, match="parameter set 0: link_latency must be 3 x 3"):
        SweepSimulator(np.arange(2), 7, [ParamSet(num_nodes=3, link_latency=matrices(7)[0][1])], [0, 0]).create(1000)
    with pytest.raises(ValueError, match="parameter set 0: link_latency entries must be in 0..65535"):
        SweepSimulator(np.arange(2), 2, [ParamSet(link_latency=((0, 65536), (0, 0)))], [0, 0]).create(1000)


def test_link_signatures_match_the_header():
    """lbft_create_sweep_links: the extern declarations of the Rust shim and the ctypes bindings against include/lbft.h."""
    from tests.test_rust_shim import c_functions, rust_functions
    c = c_functions()
    assert c["lbft_create_sweep_links"][0] == ["ptr:lbft_config", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "ptr:u32",
                                               "ptr:u32", "u32", "ptr:u32", "ptr:lbft_sim"]
    r = rust_functions()
    assert r["lbft_create_sweep_links"][0] == ["ptr:LbftConfig", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "ptr:u32",
                                               "ptr:u32", "u32", "ptr:u32", "ptr:*mut LbftSim"], r["lbft_create_sweep_links"]
    lib = _lib.load()
    assert len(lib.lbft_create_sweep_links.argtypes) == 9
    assert "lbft_create_sweep_links" in _lib.EXPORTS
