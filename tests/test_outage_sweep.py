"""Outage sweeps (lbft_create_sweep_outages) without a GPU: the SW and SW + CT device cores compiled for the host
(tests/hostcore/outage_hostcore.cpp) against the oracle run once per set with its outage windows (tests/hostcore/outage_oracle.hpp),
instance by instance, in every queue mode, with partitions, voting rights, committee sizes and link matrices; the test oracle
pinned on pop traces (no window is the oracle, an empty window is no window, [0, > max_clock) is a silent node); empty schedules
against the same sweep through the existing entry points; [0, inf) schedules against silent nodes; the edges of a window (from
clock 0, at a node's startup, ending at max_clock, max_clock + 1 and never), the sync-request addressee, and duplicate timers
inside a window; every refusal and its message; the lbft_outage layout; block latency over windows of proposal time; and
FaultSet.outages through SweepSimulator."""
import ctypes

import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _build, _lib
from librabft_simulator_b200._lib import INT64_MAX, LbftOutage
from tests.block_latency_support import assert_same_block_stats, numpy_block_stats
from tests.committee_support import cross_sizes, size_of
from tests.link_support import LinkOracle, matrices
from tests.outage_support import (EV_REQUEST, EV_TIMER, POP_CANCELLED, POP_HANDLED, POP_RECEIVER_DOWN, POP_RECEIVER_SILENT,
                                  POP_SENDER_DOWN, POP_SENDER_SILENT, OutageHarness, OutageOracle, c_windows, oracle_per_set,
                                  schedules, set_config, set_with_outages)
from tests.support import assert_same, make_config
from tests.sweep_support import KERNEL_CASES, SETS, c_sets

FLAGS_CT = _lib.FLAG_COMMIT_TIMES
FIELDS = ("commit_counts", "last_states", "counters", "status", "lc_round", "proposers", "committed", "proposed")


@pytest.fixture(scope="module")
def harness():
    return OutageHarness()


@pytest.fixture(scope="module")
def outage_oracle():
    return OutageOracle()


@pytest.fixture(scope="module")
def lib():
    _build.build_product()
    return _lib.load()


def variants(sets, n, partitions):
    """Set k with variant k % 3: no fault; a silent node (node k % n); a zero-weight node 0; every other set with a partition plan
    when `partitions`."""
    out = []
    for k, p in enumerate(sets):
        plan = (2, 200) if partitions and k % 2 else (0, 0)
        silent = (k % n,) if k % 3 == 1 else ()
        rights = (0,) + (1,) * (n - 1) if k % 3 == 2 else None
        out.append(ParamSet(p.network_delay, p.node_config, FaultSet(silent, *plan), rights))
    return out


def crossed(nodes, sizes, partitions, links, max_clock):
    """The sets of tests/sweep_support.SETS with fault / rights variants (and committee sizes), with every other set carrying a
    link matrix when `links`, each crossed with the outage schedules of its committee (schedules)."""
    base = cross_sizes(SETS, sizes, partitions) if sizes else variants(SETS, nodes, partitions)
    out = []
    for k, p in enumerate(base):
        n = size_of(p, nodes)
        m = matrices(n)[k % 3][1] if links and k % 2 else None
        p = ParamSet(p.network_delay, p.node_config, p.faults, p.voting_rights, p.num_nodes, m)
        out += [set_with_outages(p, w) for _, w in schedules(n, max_clock, p.faults.silent)]
    return out


SHAPES = [
    # (first seed, layout's committee, committee sizes or None, max_clock, shared, queue mode, partition plans, link matrices)
    (100, 4, None, 1000, {"round_cap": 256, "payload_cap": 64}, 2, False, False),  # shared-memory scan queue
    (200, 5, None, 1000, {"round_cap": 256, "payload_cap": 128, "queue_cap": 400, "force": "thread"}, 1, True, True),  # HBM scan queue
    (300, 7, None, 1500, {"round_cap": 256, "payload_cap": 128}, 3, True, True),  # calendar queue
    (400, 7, None, 5000, {"round_cap": 768, "payload_cap": 128}, 0, False, False),  # beyond the calendar's horizon: binary heap
    (500, 7, (3, 4, 7), 1500, {"round_cap": 256, "payload_cap": 128}, 3, True, True),  # committee sizes
]


@pytest.mark.parametrize("seed0,nodes,sizes,max_clock,shared,qmode,partitions,links", SHAPES)
@pytest.mark.parametrize("ct", [False, True])
def test_outage_sweep_matches_the_oracle_per_instance(harness, outage_oracle, monkeypatch, seed0, nodes, sizes, max_clock, shared,
                                                      qmode, partitions, links, ct):
    """Every instance equals the test oracle run as a plain configuration of its set (delay, NodeConfig, faults, rights,
    committee size, link latencies) with its set's outage windows: commit counts, state keys, the counters the reference has
    (events processed by kind, cancelled timers, creation stamps, largest active round, RNG draws, scheduled notifications),
    commit logs and commit times."""
    shared = dict(shared)
    if "force" in shared:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", shared.pop("force"))
    sets = crossed(nodes, sizes, partitions, links, max_clock)
    count = 2 * len(sets)
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    flags = FLAGS_CT if ct else 0
    name, _, _, records, mask = harness.kernel_info(seeds, nodes, max_clock, sets, set_of, faults=True, links=links, flags=flags,
                                                    **shared)
    assert ",%d," % qmode in name and name.startswith("lbft_ct_sweep_" if ct else "lbft_sweep_"), name
    assert records & 0b10011 == 0b10011 and bool(records & 8) == links and bool(records & 4) == bool(sizes)
    assert mask == sum(1 << k for k in {k for p in sets for k, a, b in p.faults.outages if a < min(max_clock + 1, b or INT64_MAX)})
    h = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, links=links, flags=flags, **shared)
    o = oracle_per_set(outage_oracle, seeds, nodes, max_clock, sets, set_of, **shared)
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert_same(o, h, "outage sweep layout %d" % nodes)
    assert h.commit_counts.sum() > 0
    for i in range(0, count, 5):  # commit logs, and with CT commit times, of a sample of instances
        ps = sets[set_of[i]]
        n, kw, m, w = set_config(ps, nodes)
        kw.update(shared)
        log = outage_oracle.commit_log(seeds[i:i + 1], n, 0, int(np.argmax(h.commit_counts[i, :n])), max_clock, m, w, **kw)
        assert [p for p, _, _ in log][:128] == h.proposers[i, :len(log)].tolist(), i
        if ct:
            committed, proposed, counts = outage_oracle.commit_times(seeds[i:i + 1], n, max_clock, m, w, **kw)
            np.testing.assert_array_equal(counts[0], h.commit_counts[i, :n])
            np.testing.assert_array_equal(committed[0], h.committed[i, :n], err_msg="instance %d committed" % i)
            np.testing.assert_array_equal(proposed[0], h.proposed[i], err_msg="instance %d proposed" % i)


def test_no_window_is_the_oracle(oracle, outage_oracle):
    """The test oracle restates the oracle's loop: without windows, and with only empty windows, every output of every instance
    (commit counts, state keys, all counters, status) is the oracle's and the link oracle's own, over sets with silent nodes,
    partition plans and rights; and the pop trace of an empty window is that of no window, with no pop dropped by an outage."""
    n = 7
    link_oracle = LinkOracle()
    for k, p in enumerate(variants(SETS, n, True)[::2]):
        _, kw, _, _ = set_config(p, n)
        seeds = np.arange(40 * k, 40 * k + 8, dtype=np.uint64)
        a = outage_oracle.run(seeds, n, 1200, None, None, round_cap=256, **kw)
        empty = c_windows(((1, 300, 300), (3, 0, 0), (5, 1100, 1100)), n)
        b = outage_oracle.run(seeds, n, 1200, None, empty, round_cap=256, **kw)
        c = oracle.run(seeds, n, 1200, round_cap=256, **kw)
        d = link_oracle.run(seeds, n, 1200, np.zeros((n, n), np.uint32), round_cap=256, **kw)
        for field in ("commit_counts", "last_states", "counters", "status"):
            for other, what in ((b, "empty windows"), (c, "oracle"), (d, "link oracle")):
                np.testing.assert_array_equal(getattr(a, field), getattr(other, field), err_msg="set %d %s %s" % (k, field, what))
        assert a.commit_counts.sum() > 0
        t0 = outage_oracle.trace(seeds, n, 0, 1200, None, None, round_cap=256, **kw)
        t1 = outage_oracle.trace(seeds, n, 0, 1200, None, empty, round_cap=256, **kw)
        np.testing.assert_array_equal(t0, t1)
        assert set(np.unique(t0[:, 4]).tolist()) <= {POP_HANDLED, POP_CANCELLED, POP_RECEIVER_SILENT, POP_SENDER_SILENT}
        assert len(t0) == int(a.counters[0, :4].sum())


@pytest.mark.parametrize("down", [(0,), (2,), (1, 4)])
def test_forever_window_is_a_silent_node(oracle, outage_oracle, down):
    """[0, > max_clock) on a node set S gives the oracle with silent = S, on every output including all counters, and its pop
    trace is the silent run's with each "silent" fate read as "down"."""
    n = 7
    silent = np.zeros(n, np.uint8)
    silent[list(down)] = 1
    for k, p in enumerate(SETS[:6]):
        ps = ParamSet(p.network_delay, p.node_config, FaultSet((), 2 if k % 2 else 0, 200))
        _, kw, _, _ = set_config(ps, n)
        seeds = np.arange(10 * k, 10 * k + 10, dtype=np.uint64)
        for end in (1201, 5000, INT64_MAX):
            w = c_windows([(d, 0, end) for d in down], n)
            a = outage_oracle.run(seeds, n, 1200, None, w, round_cap=256, **kw)
            b = oracle.run(seeds, n, 1200, round_cap=256, silent=silent, **{k2: v for k2, v in kw.items() if k2 != "silent"})
            for field in ("commit_counts", "last_states", "counters", "status"):
                np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="set %d %s" % (k, field))
        t0 = outage_oracle.trace(seeds, n, 1, 1200, None, w, round_cap=256, **kw)
        kw_s = dict(kw)
        kw_s["silent"] = silent
        t1 = outage_oracle.trace(seeds, n, 1, 1200, None, None, round_cap=256, **kw_s)
        t1[t1[:, 4] == POP_RECEIVER_SILENT, 4] = POP_RECEIVER_DOWN
        t1[t1[:, 4] == POP_SENDER_SILENT, 4] = POP_SENDER_DOWN
        np.testing.assert_array_equal(t0, t1)


def _one_set(harness, outage_oracle, ps, n, max_clock, seeds, **shared):
    """The harness over one set (CT), checked against the test oracle on every output including commit times; returns the
    harness's result."""
    set_of = np.zeros(len(seeds), np.uint32)
    h = harness.run(seeds, n, max_clock, [ps], set_of, faults=True, flags=FLAGS_CT, **shared)
    o = oracle_per_set(outage_oracle, seeds, n, max_clock, [ps], set_of, **shared)
    assert_same(o, h, str(ps.faults.outages))
    _, kw, m, w = set_config(ps, n)
    kw.update(shared)
    committed, proposed, counts = outage_oracle.commit_times(seeds, n, max_clock, m, w, **kw)
    np.testing.assert_array_equal(committed, h.committed)
    np.testing.assert_array_equal(proposed, h.proposed)
    return h


def test_window_edges(harness, outage_oracle):
    """Windows from clock 0; from a node's startup time, so that its startup timer pops inside (a variance-0 delay model: every
    node starts at the same time); ending at max_clock (an event at max_clock is still dropped), at max_clock + 1 and never (the same run)."""
    n, max_clock = 7, 1000
    base = ParamSet(RandomDelay.new(10.0, 0.0), NodeConfig())
    seeds = np.arange(1, 17, dtype=np.uint64)
    _one_set(harness, outage_oracle, set_with_outages(base, ((2, 0, 200),)), n, max_clock, seeds, round_cap=256)
    rows = outage_oracle.trace(seeds, n, 0, max_clock, None, None, round_cap=256)
    startup = int(rows[(rows[:, 0] == EV_TIMER) & (rows[:, 1] == 3)][0, 3])
    rows = outage_oracle.trace(seeds, n, 0, max_clock, None, c_windows(((3, startup, 300),), n), round_cap=256)
    first = rows[(rows[:, 0] == EV_TIMER) & (rows[:, 1] == 3)][0]
    assert first[3] == startup and first[4] == POP_RECEIVER_DOWN, first
    _one_set(harness, outage_oracle, set_with_outages(base, ((3, startup, 300),)), n, max_clock, seeds, round_cap=256)
    ends = {}
    for end in (max_clock, max_clock + 1, INT64_MAX):
        ps = set_with_outages(ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig()), ((4, 600, None if end == INT64_MAX else end),))
        ends[end] = _one_set(harness, outage_oracle, ps, n, max_clock, seeds, round_cap=256)
    for field in FIELDS:
        np.testing.assert_array_equal(getattr(ends[max_clock + 1], field), getattr(ends[INT64_MAX], field), err_msg=field)


def test_requests_to_a_down_node_are_dropped(harness, outage_oracle):
    """A window on a node that sync requests are addressed to: the trace shows requests dropped because their sender (the node
    they were sent to) is down, and those instances are among the ones compared with the harness."""
    n, max_clock = 4, 1500
    ps = set_with_outages(ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig()), ((1, 500, 800),))
    seeds = np.arange(1, 33, dtype=np.uint64)
    _one_set(harness, outage_oracle, ps, n, max_clock, seeds, round_cap=256)
    hits = 0
    for i in range(len(seeds)):
        rows = outage_oracle.trace(seeds, n, i, max_clock, None, c_windows(ps.faults.outages, n), round_cap=256)
        req = rows[(rows[:, 0] == EV_REQUEST) & (rows[:, 4] == POP_SENDER_DOWN)]
        assert (req[:, 2] == 1).all() and ((req[:, 3] >= 500) & (req[:, 3] < 800)).all()
        hits += len(req)
    assert hits > 0


def test_duplicate_timers_inside_a_window(harness, outage_oracle):
    """The push-time elision of a duplicate timer: where the trace shows two timer pops of one (node, time) both dropped by a
    window, the harness's timers_cancelled is the oracle's (the duplicate counts as popped, not as cancelled), and such an
    instance is among those compared."""
    n, max_clock = 4, 1500
    found = []
    for k, p in enumerate(SETS[:4]):
        ps = set_with_outages(ParamSet(p.network_delay, p.node_config), ((k % n, 300, 700),))
        seeds = np.arange(100 * k, 100 * k + 24, dtype=np.uint64)
        h = _one_set(harness, outage_oracle, ps, n, max_clock, seeds, round_cap=256)
        for i in range(len(seeds)):
            rows = outage_oracle.trace(seeds, n, i, max_clock, None, c_windows(ps.faults.outages, n), round_cap=256)
            t = rows[(rows[:, 0] == EV_TIMER) & (rows[:, 4] == POP_RECEIVER_DOWN)]
            keys, counts = np.unique(t[:, 1] * (1 << 32) + t[:, 3], return_counts=True)
            if (counts >= 2).any():
                found.append((k, i, int(h.counters[i, 4])))
    assert found, "no instance with a duplicate timer inside a window"


def test_empty_schedules_equal_the_sweep_without_outages(harness, monkeypatch):
    """An outage sweep whose windows are all empty (or past max_clock): the kernel and words per instance of the same call
    through the existing entry points (each tests/sweep_support.KERNEL_CASES shape, automatic and forced to each family), and
    every output identical, counters included, with faults, rights, committee sizes and link matrices."""
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
            sets = [ParamSet(SETS[k].network_delay, SETS[k].node_config, voting_rights=(1,) * nodes) for k in (0, 1)]
            got = harness.kernel_info(seeds, nodes, max_clock, sets, set_of, **kw)
            assert got[:2] == harness.kernel_info(seeds, nodes, max_clock, sets, set_of, outages=False, **kw)[:2], (family, name)
            assert got[3] == 0b10011 and got[4] == 0
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    for seed0, nodes, sizes, max_clock, shared, _, partitions, links in SHAPES:
        shared = {k: v for k, v in shared.items() if k != "force"}
        base = cross_sizes(SETS[:4], sizes, partitions) if sizes else variants(SETS[:6], nodes, partitions)
        sets = []
        for k, p in enumerate(base):
            n = size_of(p, nodes)
            m = matrices(n)[k % 3][1] if links else None
            live = [x for x in range(n) if x not in p.faults.silent]
            w = ((live[0], 300, 300),) if k % 3 == 0 else (((live[-1], max_clock + 1, None),) if k % 3 == 1 else ())
            sets.append(set_with_outages(ParamSet(p.network_delay, p.node_config, p.faults, p.voting_rights, p.num_nodes, m), w))
        seeds = np.arange(seed0, seed0 + 3 * len(sets), dtype=np.uint64)
        set_of = np.arange(len(seeds)) % len(sets)
        assert harness.kernel_info(seeds, nodes, max_clock, sets, set_of, faults=True, links=links, **shared)[4] == 0
        a = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, links=links, flags=FLAGS_CT, **shared)
        b = harness.run(seeds, nodes, max_clock, sets, set_of, faults=True, links=links, outages=False, flags=FLAGS_CT, **shared)
        for field in FIELDS:
            np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="layout %d %s" % (nodes, field))
    # shared faults and shared voting rights (faults and voting_rights NULL): the configuration's apply to every set
    sets = [set_with_outages(ParamSet(p.network_delay, p.node_config), ((0, 500, 500),)) for p in SETS[:3]]
    seeds = np.arange(70, 94, dtype=np.uint64)
    set_of = np.arange(24) % 3
    shared = dict(voting_rights=[3, 1, 1, 1, 1, 1, 2], silent=[0, 0, 1, 0, 0, 0, 0], partition_windows=2, partition_max_len=100)
    a = harness.run(seeds, 7, 1000, sets, set_of, flags=FLAGS_CT, **shared)
    b = harness.run(seeds, 7, 1000, sets, set_of, outages=False, flags=FLAGS_CT, **shared)
    for field in FIELDS:
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="shared " + field)


def test_forever_schedules_equal_a_silent_node_sweep(harness):
    """[0, inf) schedules through the product's setup equal a FaultSet(silent=...) sweep of the same sets on every output but the
    implementation counters max_queue, max_payloads and the count of duplicate timers elided at push (a silent node's incoming
    events are elided at send, a down node's are queued and dropped at their pop; a node with a window in any set has its
    duplicate timers queued)."""
    n, max_clock = 7, 1200
    down = [(0,), (3,), (2, 5), ()]
    sets_o, sets_s = [], []
    for k, p in enumerate(SETS[:8]):
        d = down[k % 4]
        plan = (2, 200) if k % 2 else (0, 0)
        sets_o.append(ParamSet(p.network_delay, p.node_config, FaultSet((), *plan, tuple((x, 0, None) for x in d))))
        sets_s.append(ParamSet(p.network_delay, p.node_config, FaultSet(d, *plan)))
    seeds = np.arange(1, 1 + 4 * len(sets_o), dtype=np.uint64)
    set_of = np.arange(len(seeds)) % len(sets_o)
    a = harness.run(seeds, n, max_clock, sets_o, set_of, faults=True, flags=FLAGS_CT, round_cap=256)
    b = harness.run(seeds, n, max_clock, sets_s, set_of, faults=True, outages=False, flags=FLAGS_CT, round_cap=256)
    keep = [c for c in range(12) if c not in (8, 10, 11)]
    for field in FIELDS:
        x, y = getattr(a, field), getattr(b, field)
        if field == "counters":
            x, y = x[:, keep], y[:, keep]
        np.testing.assert_array_equal(x, y, err_msg=field)


def test_equal_schedules_share_one_table(harness):
    """One device table of N windows per distinct schedule (after clamping), whatever the sets' other fields."""
    ws = [((1, 100, 400),), ((2, 0, None),), ()]
    sets = [set_with_outages(ParamSet(SETS[k % 4].network_delay, SETS[k % 4].node_config), ws[k % 3]) for k in range(10)]
    seeds = np.arange(1, 21, dtype=np.uint64)
    set_of = np.arange(20) % 10
    info = harness.kernel_info(seeds, 7, 1000, sets, set_of)
    assert info[2] == 3 * 7 * 8 and info[4] == 0b110
    # a window reaching past max_clock and one that never ends clamp to the same window; so do all empty ones
    sets = [set_with_outages(ParamSet(SETS[0].network_delay, SETS[0].node_config), w)
            for w in (((1, 100, 1001),), ((1, 100, None),), ((1, 100, 5000),), ((2, 7, 7),), ((3, 1500, 2000),), ())]
    info = harness.kernel_info(seeds[:12], 7, 1000, sets, np.arange(12) % 6)
    assert info[2] == 2 * 7 * 8 and info[4] == 0b10


def _create(lib, cfg, sets, faults, vr, sizes, links, outages, num_sets, set_of):
    h = ctypes.c_void_p()
    ptr = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib.lbft_create_sweep_outages(ctypes.byref(cfg), sets, faults, ptr(vr), ptr(sizes), ptr(links), outages, num_sets, ptr(set_of),
                                       ctypes.byref(h))
    assert h.value is None
    return rc, lib.lbft_last_error().decode()


def test_outage_sweep_refusals(lib):
    """Everything lbft_create_sweep_outages refuses, with LBFT_ERR_INVALID and before any device work (so without a GPU too)."""
    cfg, keep = make_config(np.arange(1, 9, dtype=np.uint64), 7)
    ok = np.arange(8, dtype=np.uint32) % 4
    good = [ParamSet(SETS[k].network_delay, SETS[k].node_config) for k in range(4)]
    sets = c_sets(good)

    def table(*entries):
        t = (LbftOutage * 28)()
        for s, node, a, b in entries:
            t[s * 7 + node] = LbftOutage(a, b)
        return t

    w = table((0, 1, 100, 200))
    # what the other sweeps refuse, with their messages
    assert _create(lib, cfg, sets, None, None, None, None, w, 0, ok)[1].startswith("num_sets")
    assert _create(lib, cfg, None, None, None, None, None, w, 4, ok) == (-1, "sets and set_of_instance must not be NULL")
    bad = ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=0))
    rc, msg = _create(lib, cfg, c_sets([good[0], bad, good[2], good[3]]), None, None, None, None, w, 4, ok)
    assert rc == -1 and msg.startswith("parameter set 1: delta = 0"), msg
    big = np.zeros((4, 7, 7), np.uint32)
    big[2, 1, 0] = 65536
    assert _create(lib, cfg, sets, None, None, None, big, w, 4, ok) == (-1, "parameter set 2: link_latency entries must be <= 65535")
    cfg_t, keep_t = make_config(np.arange(1, 9, dtype=np.uint64), 7, flags=_lib.FLAG_TRUE_DATA_SYNC)
    assert "take no flags" in _create(lib, cfg_t, sets, None, None, None, None, w, 4, ok)[1]
    # the windows
    assert _create(lib, cfg, sets, None, None, None, None, None, 4, ok) == (-1, "outages must not be NULL")
    assert _create(lib, cfg, sets, None, None, None, None, table((1, 2, -1, 5)), 4, ok) == (
        -1, "parameter set 1: outages: down_from must be >= 0")
    assert _create(lib, cfg, sets, None, None, None, None, table((3, 0, 50, 49)), 4, ok) == (
        -1, "parameter set 3: outages: down_until must be >= down_from")
    sizes = np.array([3, 4, 7, 5], np.uint32)
    assert _create(lib, cfg, sets, None, None, sizes, None, table((1, 4, 10, 20)), 4, ok) == (
        -1, "parameter set 1: outages has a non-empty window on a node at or past the set's committee size")
    faults = (_lib.LbftFaultSet * 4)(*[FaultSet((k,)).to_c() for k in range(4)])
    assert _create(lib, cfg, sets, faults, None, None, None, table((2, 2, 0, 1)), 4, ok) == (
        -1, "parameter set 2: outages has a non-empty window on a silent node")
    cfg_s, keep_s = make_config(np.arange(1, 9, dtype=np.uint64), 7, silent=[0, 0, 0, 0, 0, 1, 0])
    assert _create(lib, cfg_s, sets, None, None, None, None, table((3, 5, 0, INT64_MAX)), 4, ok) == (
        -1, "parameter set 3: outages has a non-empty window on a silent node")
    assert lib.lbft_create_sweep_outages(None, sets, None, None, None, None, w, 4, None, ctypes.byref(ctypes.c_void_p())) == -1


def test_refusals_reach_the_host_setup(harness):
    """The same checks through the host harness (the product's HostSetup), where a valid call builds: empty windows on a silent
    node and past a set's committee, with committee sizes and faults."""
    seeds = np.arange(1, 5, dtype=np.uint64)
    sets = [ParamSet(SETS[0].network_delay, SETS[0].node_config, FaultSet((1,)), num_nodes=3),
            ParamSet(SETS[1].network_delay, SETS[1].node_config, FaultSet((), 2, 100), num_nodes=7)]
    t = (LbftOutage * 14)()
    t[1] = LbftOutage(40, 40)  # empty, on set 0's silent node
    t[5] = LbftOutage(0, 0)    # empty, past set 0's committee
    t[7 + 6] = LbftOutage(0, INT64_MAX)
    harness.check(seeds, 7, 1000, sets, [0, 1, 0, 1], faults=True, table=t)
    t[4] = LbftOutage(3, 4)
    with pytest.raises(RuntimeError, match="parameter set 0: outages has a non-empty window on a node at or past"):
        harness.check(seeds, 7, 1000, sets, [0, 1, 0, 1], faults=True, table=t)


def test_block_latency_over_windows_of_proposal_time(harness, outage_oracle):
    """Quorum latency of blocks proposed before, during and after a leader's crash-recovery window: the numpy reduction
    (tests/block_latency_support.py) over the harness's commit times equals the reduction over the test oracle's, per window,
    and commits resume after the window."""
    n, max_clock = 7, 1800
    sets = [set_with_outages(ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig()), w) for w in ((), ((0, 500, 800),), ((0, 500, None),))]
    seeds = np.arange(1, 1 + 8 * len(sets), dtype=np.uint64)
    set_of = np.arange(len(seeds)) % len(sets)
    h = harness.run(seeds, n, max_clock, sets, set_of, flags=FLAGS_CT, round_cap=512, cap=256)
    committed = np.zeros_like(h.committed)
    proposed = np.zeros_like(h.proposed)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        _, kw, m, w = set_config(ps, n)
        c, p, _ = outage_oracle.commit_times(seeds[idx], n, max_clock, m, w, cap=256, round_cap=512, **kw)
        committed[idx], proposed[idx] = c, p
    weights = np.ones(n, np.int64)
    for lo, hi in ((200, 500), (500, 800), (800, 1800)):
        a = numpy_block_stats(h.committed, h.proposed, h.status, set_of, len(sets), weights, 5, proposed_from=lo, proposed_until=hi)
        b = numpy_block_stats(committed, proposed, h.status, set_of, len(sets), weights, 5, proposed_from=lo, proposed_until=hi)
        assert_same_block_stats(a, b, "[%d, %d)" % (lo, hi))
        if lo == 800:
            assert (a.samples > 0).all()  # commits resume after a recovery, and go on without the crashed node


def test_faultset_outages_through_the_sweep_simulator():
    """FaultSet(outages=...): stored as a tuple, None kept for "never recovers", one window per node; to_c() unchanged; the
    table SweepSimulator passes to lbft_create_sweep_outages; grid's faults axis carries the scenarios; refusals."""
    f = FaultSet(outages=[(0, 500, None), (3, 100, 200)])
    assert f.outages == ((0, 500, None), (3, 100, 200)) and f != FaultSet() and hash(f)
    assert bytes(f.to_c()) == bytes(FaultSet().to_c())
    assert FaultSet() == FaultSet((), 0, 0, ())
    with pytest.raises(ValueError, match="at most one window per node"):
        FaultSet(outages=((1, 0, 10), (1, 20, 30)))
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20)]
    scen = [FaultSet(), FaultSet(outages=((0, 500, None),)), FaultSet(outages=((0, 500, 800),))]
    sim = SweepSimulator.grid([5, 6], delays, configs, num_nodes=7, faults=scen)
    assert [p.faults for p in sim.param_sets] == scen * 4
    t = sim._outage_table()
    assert len(t) == 12 * 7
    assert (t[7].down_from, t[7].down_until) == (500, INT64_MAX) and (t[14].down_from, t[14].down_until) == (500, 800)
    assert all((t[k].down_from, t[k].down_until) == (0, 0) for k in range(84) if k not in range(7, 84, 21) and k not in range(14, 84, 21))
    assert SweepSimulator.grid([5], delays, configs, num_nodes=7)._outage_table() is None
    assert not any(p.faults.has_fault_model() for p in sim.param_sets)
    with pytest.raises(ValueError, match="parameter set 0: outage node 7 is not in 0..6"):
        SweepSimulator(np.arange(2), 7, [ParamSet(faults=FaultSet(outages=((7, 0, 1),)))], [0, 0])._outage_table()


def test_outage_layout_and_signatures_match_the_header():
    """lbft_outage: its fields in the header, the Rust shim and ctypes; lbft_create_sweep_outages: the extern declarations of the
    Rust shim and the ctypes bindings against include/lbft.h."""
    from tests.test_rust_shim import c_functions, c_struct_fields, rust_functions, rust_struct_fields
    assert c_struct_fields("lbft_outage") == [("down_from", "i64"), ("down_until", "i64")]
    assert rust_struct_fields("LbftOutage") == [("down_from", "i64"), ("down_until", "i64")]
    assert ctypes.sizeof(LbftOutage) == 16 and LbftOutage.down_from.offset == 0 and LbftOutage.down_until.offset == 8
    c = c_functions()
    assert c["lbft_create_sweep_outages"][0] == ["ptr:lbft_config", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "ptr:u32",
                                                 "ptr:u32", "ptr:lbft_outage", "u32", "ptr:u32", "ptr:lbft_sim"]
    r = rust_functions()
    assert r["lbft_create_sweep_outages"][0] == ["ptr:LbftConfig", "ptr:lbft_param_set", "ptr:lbft_fault_set", "ptr:u64", "ptr:u32",
                                                 "ptr:u32", "ptr:lbft_outage", "u32", "ptr:u32", "ptr:*mut LbftSim"], r["lbft_create_sweep_outages"]
    lib = _lib.load()
    assert len(lib.lbft_create_sweep_outages.argtypes) == 10
    assert "lbft_create_sweep_outages" in _lib.EXPORTS
