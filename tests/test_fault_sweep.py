"""Fault sweeps (lbft_create_sweep_faults) without a GPU: the SW and SW + CT device cores compiled for the host
(tests/hostcore/fault_hostcore.cpp) against the oracle run once per set with that set's faults, the equivalence with a sweep whose
configuration carries uniform faults, commit times and latency statistics per set, the refusals of the C ABI, SweepSimulator.grid's
third axis, and the struct layouts of the bindings."""
import ctypes
import re

import numpy as np
import pytest

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _build, _lib
from tests.ct_support import CtHarness
from tests.fault_support import FaultHarness, c_faults, cross, fault_kwargs, fault_sets, oracle_per_set
from tests.latency_support import assert_same_stats, make_spec, numpy_stats
from tests.support import FLAG_RESUMABLE, FLAG_ROUND_SWITCHES, assert_same, make_config
from tests.sweep_support import KERNEL_CASES, SETS, c_sets, set_kwargs


@pytest.fixture(scope="module")
def faults():
    return FaultHarness()


@pytest.fixture(scope="module")
def lib():
    _build.build_product()
    return _lib.load()


SHAPES = [
    # (first seed, nodes, max_clock, shared, queue mode of the sweep's layout)
    (100, 4, 1000, {"round_cap": 256}, 2),  # shared-memory scan queue
    (200, 7, 1500, {"round_cap": 256}, 3),  # calendar queue (the fastest set's event rate leaves the compact entries)
    (300, 40, 600, {}, 3),
    (400, 7, 5000, {"round_cap": 768}, 0),  # beyond the calendar's horizon: binary heap
]


@pytest.mark.parametrize("seed0,nodes,max_clock,shared,qmode", SHAPES)
def test_fault_sweep_matches_the_oracle_per_instance(oracle, faults, seed0, nodes, max_clock, shared, qmode):
    """The 12 parameter sets crossed with 7 fault sets, instance i on set i % 84: every instance equals the oracle run with its
    set's delay, NodeConfig, silent nodes and partition plan."""
    sets = cross(SETS, fault_sets(nodes))
    count = 2 * len(sets)
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    name, windows = faults.kernel_info(seeds, nodes, max_clock, sets, set_of, **shared)
    assert ",%d," % qmode in name and windows == 64, name
    h = faults.run(seeds, nodes, max_clock, sets, set_of, **shared)
    o = oracle_per_set(oracle, seeds, nodes, max_clock, sets, set_of, **shared)
    assert (o.status & ~np.uint32(64) == 1).all(), o.status
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert_same(o, h, "fault sweep N=%d" % nodes)
    # f + 1 silent nodes leave no quorum: nothing commits; the other fault sets commit something
    nf = len(fault_sets(nodes))
    stuck = (set_of % nf) == 3
    assert (h.commit_counts[stuck] == 0).all()
    assert h.commit_counts[~stuck].sum() > 0


UNIFORM = [FaultSet((1,)), FaultSet((), 4, 150), FaultSet((0,), 2, 400)]


def test_uniform_faults_are_a_sweep_with_shared_faults(faults, monkeypatch):
    """Every set carrying the faults F: the kernel and layout of lbft_create_sweep with F in the configuration (each
    tests/sweep_support.KERNEL_CASES shape, automatic and forced to each family), and identical outputs, counters included."""
    for family in (None, "thread", "wide"):
        if family:
            monkeypatch.setenv("LBFT_FORCE_KERNEL", family)
        else:
            monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
        for name, count, nodes, kw in KERNEL_CASES:
            kw = dict(kw)
            max_clock = kw.pop("max_clock", 1000)
            kw.pop("partition_windows", None), kw.pop("partition_max_len", None)
            seeds = np.arange(1, count + 1, dtype=np.uint64)
            set_of = np.arange(count) % 2
            for f in UNIFORM:
                sets = [ParamSet(SETS[0].network_delay, SETS[0].node_config, f), ParamSet(SETS[1].network_delay, SETS[1].node_config, f)]
                got = faults.kernel_info(seeds, nodes, max_clock, sets, set_of, **kw)
                want = faults.kernel_info(seeds, nodes, max_clock, sets, set_of, faults=False, **kw, **fault_kwargs(f, nodes))
                assert got == want, (family, name, f, got, want)
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    for name, count, nodes, kw in KERNEL_CASES:  # the outputs, on a batch small enough for the host core
        max_clock = kw.get("max_clock", 1000)
        seeds = np.arange(11, 11 + 24, dtype=np.uint64)
        set_of = np.arange(24) % 3
        for f in UNIFORM:
            sets = [ParamSet(p.network_delay, p.node_config, f) for p in SETS[:3]]
            a = faults.run(seeds, nodes, max_clock, sets, set_of)
            b = faults.run(seeds, nodes, max_clock, sets, set_of, faults=False, **fault_kwargs(f, nodes))
            for field in ("commit_counts", "last_states", "counters", "status", "lc_round"):
                np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg="%s %s %s" % (name, f, field))


def test_silent_mask_bits_follow_the_committee(faults):
    """Bit 63 is a node of a 64-author committee: accepted there, refused (naming the set) below it."""
    seeds = np.arange(1, 9, dtype=np.uint64)
    sets = [ParamSet(p.network_delay, p.node_config, FaultSet((63,))) for p in SETS[:2]]
    assert faults.kernel_info(seeds, 64, 1000, sets, np.arange(8) % 2)[0].startswith("lbft_sweep_")
    with pytest.raises(RuntimeError, match="parameter set 0: silent_mask has a bit at or above num_nodes"):
        faults.kernel_info(seeds, 63, 1000, sets, np.arange(8) % 2)


def test_layout_takes_the_largest_window_count(faults):
    """Sets with 0, 2 and 4 windows: the layout and kernel of a sweep with partition_windows = 4 in its configuration."""
    seeds = np.arange(1, 16385, dtype=np.uint64)
    set_of = np.arange(16384) % 3
    sets = [ParamSet(SETS[0].network_delay, SETS[0].node_config, FaultSet((), w, 150)) for w in (0, 2, 4)]
    name, windows = faults.kernel_info(seeds, 7, 1000, sets, set_of)
    assert windows == 4
    assert (name, windows) == faults.kernel_info(seeds, 7, 1000, sets, set_of, faults=False, partition_windows=4, partition_max_len=150)


@pytest.mark.parametrize("nodes,max_clock,shared", [(4, 1000, {"round_cap": 256}), (7, 1000, {}), (40, 600, {})])
def test_commit_times_match_plain_handles_per_set(faults, nodes, max_clock, shared):
    """The SW + CT core of a fault sweep against the plain commit-times core run once per set with that set's faults."""
    ct = CtHarness()
    sets = cross(SETS[:4], fault_sets(nodes))
    count = 2 * len(sets)
    seeds = np.arange(900, 900 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    h = faults.run_ct(seeds, nodes, max_clock, sets, set_of, cap=128, **shared)
    assert h.commit_counts.max() > 0
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        kw = dict(shared)
        kw.update(set_kwargs(ps))
        kw.update(fault_kwargs(ps.faults, nodes))
        g = ct.run(seeds[idx], nodes, max_clock, cap=128, **kw)
        for field in ("commit_counts", "last_states", "status", "committed", "proposed"):
            np.testing.assert_array_equal(getattr(h, field)[idx], getattr(g, field), err_msg="set %d %s" % (s, field))


def test_latency_statistics_per_set_match_numpy(faults):
    """lbft_latency_stats grouped by set (the product's spec check and walk on the host) against numpy over the commit times."""
    sets = cross(SETS[:3], fault_sets(7))
    count = 3 * len(sets)
    seeds = np.arange(50, 50 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(sets)
    for bins, width, lo, hi in ((1024, 1, 0, None), (5, 7, 200, 800)):
        h = faults.run_ct(seeds, 7, 1000, sets, set_of, cap=256, spec=make_spec(bins, width, lo, hi))
        want = numpy_stats(h.committed, h.proposed, h.status, set_of, len(sets), bins, width, lo, hi)
        assert_same_stats(h.stats, want, "bins %d" % bins)
        assert (h.stats.samples[3::len(fault_sets(7))] == 0).all()  # f + 1 silent: no commit, no sample


def _create(lib, cfg, sets, faults, num_sets, set_of):
    h = ctypes.c_void_p()
    rc = lib.lbft_create_sweep_faults(ctypes.byref(cfg), sets, faults, num_sets,
                                      None if set_of is None else ctypes.c_void_p(set_of.ctypes.data), ctypes.byref(h))
    assert h.value is None
    return rc, lib.lbft_last_error().decode()


def test_fault_sweep_refusals(lib):
    """Everything lbft_create_sweep_faults refuses, with LBFT_ERR_INVALID and before any device work (so without a GPU too)."""
    cfg, keep = make_config(np.arange(1, 9, dtype=np.uint64), 4)
    ok = np.arange(8, dtype=np.uint32) % 4
    good = cross(SETS[:2], [FaultSet(), FaultSet((1,), 2, 100)])
    sets, fsets = c_sets(good), c_faults(good)
    # what lbft_create_sweep refuses, with its messages
    for num_sets, set_of, want in ((0, ok, "num_sets"), (9, np.arange(8, dtype=np.uint32), "num_sets"), (4, None, "NULL"),
                                   (4, np.full(8, 4, np.uint32), "index >= num_sets")):
        rc, msg = _create(lib, cfg, sets, fsets, num_sets, set_of)
        assert rc == -1 and want in msg, msg
    assert _create(lib, cfg, None, fsets, 4, ok) == (-1, "sets and set_of_instance must not be NULL")
    for flags in (FLAG_ROUND_SWITCHES, FLAG_RESUMABLE):
        cfg_f, keep_f = make_config(np.arange(1, 9, dtype=np.uint64), 4, flags=flags)
        rc, msg = _create(lib, cfg_f, sets, fsets, 4, ok)
        assert rc == -1 and "flags" in msg
    cfg_e, keep_e = make_config(np.arange(1, 9, dtype=np.uint64), 4, commands_per_epoch=5)
    assert "commands_per_epoch" in _create(lib, cfg_e, sets, fsets, 4, ok)[1]
    bad = ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=0))
    rc, msg = _create(lib, cfg, c_sets([good[0], good[1], bad, good[3]]), fsets, 4, ok)
    assert rc == -1 and "parameter set 2" in msg, msg
    cfg_s, keep_s = make_config(np.arange(1, 9, dtype=np.uint64), 4)
    cfg_s.struct_size = 12
    assert "struct_size" in _create(lib, cfg_s, sets, fsets, 4, ok)[1]
    # faults must be given, per set only
    assert _create(lib, cfg, sets, None, 4, ok) == (-1, "faults must not be NULL")
    for shared in ({"silent": [0, 1, 0, 0]}, {"partition_windows": 2}, {"partition_max_len": 100}):
        cfg_x, keep_x = make_config(np.arange(1, 9, dtype=np.uint64), 4, **shared)
        rc, msg = _create(lib, cfg_x, sets, fsets, 4, ok)
        assert rc == -1 and "per set only" in msg, (shared, msg)
    # each set's substituted configuration, named by the set
    for f, want in ((FaultSet((4,)), "silent_mask has a bit at or above num_nodes"), (FaultSet((63,)), "silent_mask"),
                    (FaultSet((), 65, 10), "partition_windows must be <= 64")):
        bad_sets = good[:2] + [ParamSet(good[2].network_delay, good[2].node_config, f), good[3]]
        rc, msg = _create(lib, cfg, c_sets(bad_sets), c_faults(bad_sets), 4, ok)
        assert rc == -1 and msg.startswith("parameter set 2: ") and want in msg, msg
    assert lib.lbft_create_sweep_faults(None, sets, fsets, 4, None, ctypes.byref(ctypes.c_void_p())) == -1


def test_grid_fault_axis_and_shared_fault_refusal():
    """SweepSimulator.grid(faults=...): a third, fastest-varying axis; per-set faults and shared faults do not mix."""
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20, 30)]
    fl = [FaultSet(), FaultSet((3,)), FaultSet((), 4, 150), FaultSet((0, 1))]
    sim = SweepSimulator.grid([5, 6], delays, configs, num_nodes=4, faults=fl)
    assert sim.num_instances == 48 and len(sim.param_sets) == 24
    for i, d in enumerate(delays):
        for j, n in enumerate(configs):
            for f, fs in enumerate(fl):
                assert sim.param_sets[(i * len(configs) + j) * len(fl) + f] == ParamSet(d, n, fs)
    np.testing.assert_array_equal(sim.set_of_instance, np.repeat(np.arange(24), 2))
    plain = SweepSimulator.grid([5, 6], delays, configs, num_nodes=4)
    assert plain.param_sets == [ParamSet(d, n) for d in delays for n in configs]
    assert all(p.faults == FaultSet() for p in plain.param_sets)
    for shared in ({"silent": [0, 0, 0, 1]}, {"partition_windows": 2}, {"partition_max_len": 10}):
        s = SweepSimulator.grid([5, 6], delays, configs, num_nodes=4, faults=fl, **shared)
        with pytest.raises(ValueError, match="per set"):
            s.create(1000)
    assert FaultSet((0, 5), 3, 7).to_c().silent_mask == 0x21
    assert FaultSet([3]) == FaultSet((3,)) and FaultSet([]) == FaultSet()  # (SweepSimulator.create tests sets against FaultSet())
    with pytest.raises(ValueError):
        FaultSet((64,)).to_c()


def test_fault_set_layouts_match_the_header():
    """lbft_fault_set: the ctypes structure and the Rust shim's #[repr(C)] struct, field by field against include/lbft.h, and
    the extern declaration of lbft_create_sweep_faults."""
    from tests.test_rust_shim import RUST, c_functions, c_struct_fields, rust_functions, rust_struct_fields
    c = c_struct_fields("lbft_fault_set")
    assert c == [("silent_mask", "u64"), ("partition_windows", "u32"), ("partition_max_len", "u32")]
    assert c == rust_struct_fields("LbftFaultSet")
    assert "#[repr(C)]" in RUST.split("pub struct LbftFaultSet")[0][-200:]
    kinds = {"u32": ctypes.c_uint32, "u64": ctypes.c_uint64}
    assert [(n, kinds[t]) for n, t in c] == list(_lib.LbftFaultSet._fields_)
    assert ctypes.sizeof(_lib.LbftFaultSet) == 16 and _lib.LbftFaultSet.partition_max_len.offset == 12
    assert c_functions()["lbft_create_sweep_faults"][0] == ["ptr:lbft_config", "ptr:lbft_param_set", "ptr:lbft_fault_set", "u32", "ptr:u32",
                                                            "ptr:lbft_sim"]
    r = rust_functions()["lbft_create_sweep_faults"][0]
    assert r == ["ptr:LbftConfig", "ptr:lbft_param_set", "ptr:lbft_fault_set", "u32", "ptr:u32", "ptr:*mut LbftSim"], r
    assert "lbft_create_sweep_faults" in _lib.EXPORTS
    assert re.search(r"lbft_create_sweep_faults", open(_lib.__file__.replace("_lib.py", "simulator.py")).read())
