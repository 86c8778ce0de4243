"""Sweep handles (lbft_create_sweep) without a GPU: the SW device core compiled for the host (tests/hostcore) against the
oracle instance by instance, the one-set sweep against the plain run, the refusals of the C ABI, the kernel picks, and the
struct layouts of the bindings."""
import ctypes
import re

import numpy as np
import pytest

from librabft_simulator_b200 import NodeConfig, ParamSet, RandomDelay, SweepSimulator, _build, _lib
from tests.support import FLAG_RESUMABLE, FLAG_ROUND_SWITCHES, FLAG_TRUE_DATA_SYNC, assert_same, make_config
from tests.sweep_support import KERNEL_CASES, SETS, SWEEP_PICKS, SweepHostCore, c_sets, oracle_per_set, set_kwargs


@pytest.fixture(scope="module")
def sweep():
    return SweepHostCore()


@pytest.fixture(scope="module")
def lib():
    _build.build_product()
    return _lib.load()


CASES = [
    # (first seed, instances, nodes, max_clock, shared, queue mode of the sweep's layout)
    (100, 48, 3, 1000, {"round_cap": 256}, 2),  # shared-memory scan queue
    (200, 48, 4, 1000, {"round_cap": 256}, 2),
    (300, 24, 4, 4000, {"round_cap": 768}, 1),  # the fastest set's event rate needs the 22-bit stamps of the HBM scan queue
    (400, 36, 7, 1000, {"round_cap": 256}, 2),  # (a small batch: the wide kernel's shared-memory queue)
    (500, 24, 40, 600, {}, 3),                  # calendar queue
    (600, 12, 7, 5000, {"round_cap": 768}, 0),  # beyond the calendar's horizon: binary heap
]


@pytest.mark.parametrize("seed0,count,nodes,max_clock,shared,qmode", CASES)
def test_sweep_matches_the_oracle_per_instance(oracle, hostcore, sweep, seed0, count, nodes, max_clock, shared, qmode):
    """Interleaved assignment (instance i runs set i % 12): every instance equals the oracle run with its set's settings."""
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    set_of = np.arange(count) % len(SETS)
    # the set with the shortest mean delay (uniform on 1..4) is the one whose plain layout the sweep takes
    kw = dict(shared)
    kw.update(set_kwargs(SETS[6]))
    assert hostcore.setup_info(nodes, max_clock, **kw)["queue_scan"] == qmode
    h = sweep.run(seeds, nodes, max_clock, SETS, set_of, **shared)
    o = oracle_per_set(oracle, seeds, nodes, max_clock, SETS, set_of, **shared)
    assert (o.status & ~np.uint32(64) == 1).all(), o.status
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert h.words_per_instance == hostcore.setup_info(nodes, max_clock, **kw)["words"]
    assert_same(o, h, "sweep N=%d" % nodes)


def test_one_set_sweep_is_the_plain_run(hostcore, sweep):
    """One set over the whole batch: bit for bit the plain run of that configuration, every counter included."""
    for nodes, max_clock, ps in ((4, 1000, SETS[0]), (7, 1000, SETS[5]), (3, 1000, SETS[6])):
        seeds = np.arange(7000, 7040, dtype=np.uint64)
        h = sweep.run(seeds, nodes, max_clock, [ps], np.zeros(len(seeds)))
        g = hostcore.run(seeds, nodes, max_clock, **set_kwargs(ps))
        assert_same(g, h, "one-set sweep")
        np.testing.assert_array_equal(g.counters, h.counters)
        np.testing.assert_array_equal(g.status, h.status)
        np.testing.assert_array_equal(g.lc_round, h.lc_round)
        assert g.words_per_instance == h.words_per_instance


def test_sweep_kernel_choice(sweep, monkeypatch):
    """The sweep twin of the kernel a plain handle picks, automatically and forced to each family (LBFT_FORCE_KERNEL)."""
    for family, want in SWEEP_PICKS.items():
        if family:
            monkeypatch.setenv("LBFT_FORCE_KERNEL", family)
        else:
            monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
        for name, count, nodes, kw in KERNEL_CASES:
            kw = dict(kw)
            max_clock = kw.pop("max_clock", 1000)
            seeds = np.arange(1, count + 1, dtype=np.uint64)
            got = sweep.kernel_info(seeds, nodes, max_clock, [SETS[0]], np.zeros(count), **kw)
            assert got == want[name], (family, name, got)
    # the layout and kernel follow the set with the shortest mean delay: at 8 authors and 1 000 instances the reference delay
    # fits the wide kernel's shared-memory queue, a 1 ms uniform delay needs the wider stamps of the calendar queue
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    seeds = np.arange(1, 1001, dtype=np.uint64)
    fast = ParamSet(RandomDelay.uniform(1, 1), NodeConfig())
    assert sweep.kernel_info(seeds, 8, 1000, [SETS[0]], np.zeros(1000)) == "lbft_sweep_wide_kernel<16,2,true,32>"
    assert sweep.kernel_info(seeds, 8, 1000, [SETS[0], fast], np.arange(1000) % 2) == "lbft_sweep_wide_kernel<16,3,false,32>"


def _create_sweep(lib, cfg, sets, num_sets, set_of):
    h = ctypes.c_void_p()
    rc = lib.lbft_create_sweep(ctypes.byref(cfg), sets, num_sets, None if set_of is None else ctypes.c_void_p(set_of.ctypes.data),
                               ctypes.byref(h))
    assert h.value is None
    return rc, lib.lbft_last_error().decode()


def test_sweep_refusals(lib):
    """Everything lbft_create_sweep refuses, with LBFT_ERR_INVALID and before any device work (so without a GPU too)."""
    cfg, keep = make_config(np.arange(1, 9, dtype=np.uint64), 4)
    sets, ok = c_sets(SETS[:4]), np.arange(8, dtype=np.uint32) % 4
    for num_sets, set_of in ((0, ok), (9, np.arange(8, dtype=np.uint32)), (4, None), (4, np.full(8, 4, np.uint32))):
        rc, msg = _create_sweep(lib, cfg, sets, num_sets, set_of)
        assert rc == -1, (num_sets, msg)
    assert _create_sweep(lib, cfg, None, 4, ok)[0] == -1
    # more than 65 536 sets even when there are that many instances
    big, keep_big = make_config(np.arange(65537, dtype=np.uint64), 4)
    many = c_sets([SETS[0]] * 65537)
    rc, msg = _create_sweep(lib, big, many, 65537, np.arange(65537, dtype=np.uint32))
    assert rc == -1 and "65536" in msg
    for flags in (FLAG_ROUND_SWITCHES, FLAG_RESUMABLE, FLAG_TRUE_DATA_SYNC):
        cfg_f, keep_f = make_config(np.arange(1, 9, dtype=np.uint64), 4, flags=flags)
        rc, msg = _create_sweep(lib, cfg_f, sets, 4, ok)
        assert rc == -1 and "flags" in msg
    cfg_e, keep_e = make_config(np.arange(1, 9, dtype=np.uint64), 4, commands_per_epoch=5)
    rc, msg = _create_sweep(lib, cfg_e, sets, 4, ok)
    assert rc == -1 and "commands_per_epoch" in msg
    # each set is validated like lbft_create validates those fields, and the message names the set
    for bad in (ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=0)), ParamSet(RandomDelay.new(-1.0, 4.0), NodeConfig()),
                ParamSet(RandomDelay.uniform(5, 2), NodeConfig()), ParamSet(RandomDelay(kind=7), NodeConfig())):
        rc, msg = _create_sweep(lib, cfg, c_sets([SETS[0], SETS[1], bad, SETS[3]]), 4, ok)
        assert rc == -1 and "parameter set 2" in msg, msg
    # the shared part is validated too (the struct_size ABI guard first)
    cfg_s, keep_s = make_config(np.arange(1, 9, dtype=np.uint64), 4)
    cfg_s.struct_size = 12
    assert _create_sweep(lib, cfg_s, sets, 4, ok)[0] == -1
    assert lib.lbft_create_sweep(None, sets, 4, None, ctypes.byref(ctypes.c_void_p())) == -1


def test_param_set_layouts_match_the_header():
    """lbft_param_set: the ctypes structure and the Rust shim's #[repr(C)] struct, field by field against include/lbft.h."""
    from tests.test_rust_shim import RUST, c_struct_fields, rust_struct_fields
    c = c_struct_fields("lbft_param_set")
    assert c == rust_struct_fields("LbftParamSet")
    assert "#[repr(C)]" in RUST.split("pub struct LbftParamSet")[0][-200:]
    kinds = {"u32": ctypes.c_uint32, "i64": ctypes.c_int64, "f64": ctypes.c_double}
    assert [(n, kinds[t]) for n, t in c] == [("lambda" if n == "lambda_" else n, t) for n, t in _lib.LbftParamSet._fields_]
    assert ctypes.sizeof(_lib.LbftParamSet) == 72 and _lib.LbftParamSet.delay_mean.offset == 8 and _lib.LbftParamSet.lambda_.offset == 64
    rust = re.search(r"pub fn lbft_create_sweep\(([^)]*)\)", RUST).group(1)
    assert "*const lbft_param_set" in rust and "num_sets: u32" in rust


def test_grid_lays_out_contiguous_blocks_per_point():
    """SweepSimulator.grid: the Cartesian product of delays and node configs, one block of the same seeds per point."""
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0, 16.0)]
    configs = [NodeConfig(delta=d) for d in (10, 20)]
    sim = SweepSimulator.grid([5, 6, 7, 8], delays, configs, num_nodes=4)
    assert sim.num_instances == 24 and len(sim.param_sets) == 6
    np.testing.assert_array_equal(sim.set_of_instance, np.repeat(np.arange(6), 4))
    np.testing.assert_array_equal(sim.seeds, np.tile([5, 6, 7, 8], 6))
    assert sim.param_sets[3] == ParamSet(delays[1], configs[1])
    assert SweepSimulator.grid(3, delays[:1], configs[:1]).seeds.tolist() == [0, 1, 2]
    with pytest.raises(ValueError, match="one entry per seed"):
        SweepSimulator([1, 2, 3], 4, SETS[:2], [0, 1])
    cfg = sim.make_config(1000)
    assert cfg.flags == 0 and cfg.num_instances == 24 and cfg.struct_size == 152
