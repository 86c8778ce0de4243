"""GPU parity tests proper: the sm_90a kernel, called through the C ABI (ctypes -> liblbft_b200.so), against
the CPU oracle on the same seeded inputs; plus size-independent properties at BASELINE.json's full sizes.
Bit-exact: commit counts, SipHash state keys of the full commit logs, the logs themselves, and the event /
RNG counters."""
import numpy as np
import pytest

from tests.support import assert_same

pytestmark = pytest.mark.gpu


class GpuResult:
    """Adapter giving the product's BatchResult the attribute names of tests.support.Result."""

    def __init__(self, res):
        self.commit_counts, self.last_states = res.commit_counts, res.last_committed_states
        self.last_committed_states = self.last_states
        self.counters, self.status = res.counters, res.status


def make_sim(seeds, nodes, **kw):
    """A BatchSimulator from the keyword form of an lbft_config used by tests.support / tests.fuzz_configs."""
    from librabft_simulator_b200 import BatchSimulator, NodeConfig, RandomDelay
    kw = dict(kw)
    delay = RandomDelay.new(kw.pop("delay_mean", 10.0), kw.pop("delay_variance", 4.0))
    if "delay_lo" in kw:
        delay = RandomDelay.uniform(kw.pop("delay_lo"), kw.pop("delay_hi"))
        kw.pop("delay_kind", None)
    nc = NodeConfig(kw.pop("target_commit_interval", 100000), kw.pop("delta", 20), kw.pop("gamma", 2.0), kw.pop("lambda_", 0.5))
    return BatchSimulator(seeds, nodes, delay, nc, kw.pop("commands_per_epoch", 30000), **kw)


def gpu_run(seeds, nodes, max_clock=1000, strict=True, **kw):
    sim = make_sim(seeds, nodes, **kw)
    res = sim.loop_until(max_clock, strict=strict)
    return sim, GpuResult(res)


def test_native_library_is_loaded():
    from librabft_simulator_b200 import _lib
    lib = _lib.load()
    assert lib.lbft_abi_version() == 1


def test_golden_3_nodes_on_gpu():
    # librabft-v2/tests/simulated_run.rs:45-66, read through the reference-shaped interface
    from librabft_simulator_b200 import GlobalTime, RandomDelay, Simulator
    sim = Simulator.new(52, 3, RandomDelay.new(10.0, 4.0), None)
    contexts = sim.loop_until(GlobalTime(1000).value, None)
    assert [len(c.committed_history()) for c in contexts] == [27, 27, 27]
    assert [c.last_committed_state() for c in contexts] == [11134312813757838303] * 3


def test_golden_8_nodes_on_gpu():
    # librabft-v2/tests/simulated_run.rs:68-94
    from librabft_simulator_b200 import RandomDelay, Simulator
    contexts = Simulator.new(48, 8, RandomDelay.new(10.0, 4.0), None).loop_until(1000)
    assert [len(c.committed_history()) for c in contexts] == [28] * 7 + [30]
    assert [c.last_committed_state() for c in contexts] == [12785928431398617538] * 7 + [4890275890002623733]


CASES = [
    (1, 1024, 4, 1000, {}),   # BASELINE config 2 (LogNormal leg): 1 024 instances x 4 authors
    (1000, 96, 3, 1000, {}),
    (5, 64, 7, 1000, {}),
    (9, 33, 8, 1000, {}),     # ragged: not a multiple of the 32-instance tile
    (77, 5, 16, 600, {}),
    (3, 40, 2, 1000, {}),
    (52, 1, 3, 3000, {"delay_variance": 0.0}),  # BASELINE config 1: fixed 10 ms, > 100 rounds
    (11, 64, 4, 2500, {}),
    (21, 64, 4, 1000, {"delay_mean": 25.0, "delay_variance": 200.0}),
    (31, 32, 5, 1500, {"delta": 5, "gamma": 1.5, "lambda_": 0.25, "queue_cap": 4096, "payload_cap": 1024}),
    (41, 16, 4, 4000, {"target_commit_interval": 300, "delta": 400}),
    (61, 64, 4, 1000, {"queue_cap": 128}),   # 64-bit-key scan queue in HBM (QMODE 1)
    (62, 40, 6, 1000, {}),                   # calendar queue (QMODE 3)
    (63, 8, 6, 4200, {}),                    # binary heap (QMODE 0): horizon beyond the calendar's range
    (64, 12, 9, 700, {"delay_kind": 1, "delay_lo": 0, "delay_hi": 3, "round_cap": 256}),  # calendar queue with zero delays
]


@pytest.mark.parametrize("seed0,count,nodes,max_clock,extra", CASES)
def test_gpu_matches_oracle(oracle, kernel_choice, seed0, count, nodes, max_clock, extra):
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    o = oracle.run(seeds, nodes, max_clock, **extra)
    sim, g = gpu_run(seeds, nodes, max_clock, **dict(extra))
    assert sim.kernel_info().startswith("lbft_wide_kernel" if kernel_choice == "wide" else "lbft_event_loop_kernel")
    assert ((g.status & ~np.uint32(64)) == 1).all(), np.unique(g.status)
    assert_same(o, g, "N=%d" % nodes)
    # the commit logs themselves, for a few (instance, node) pairs
    for inst in sorted({0, count // 2, count - 1}):
        for node in (0, nodes - 1):
            assert sim.commit_log(inst, node) == oracle.commit_log(seeds, nodes, inst, node, max_clock, **extra)


def test_full_size_properties_65536_instances(oracle):
    # BASELINE config 3 at full size.  The oracle checks a sample; everything is checked through
    # size-independent properties: state key == SipHash of the returned log, logs prefix-consistent,
    # determinism (same seeds -> same results) and seed-locality (results depend only on the own seed).
    I, N = 65536, 4
    seeds = np.arange(52, 52 + I, dtype=np.uint64)
    sim, g = gpu_run(seeds, N, 1000)
    assert ((g.status & ~np.uint32(64)) == 1).all()
    assert g.commit_counts.min() >= 10 and g.commit_counts.max() <= 60
    # EVERY instance against the oracle (it does the 65 536 x 4 batch in a few seconds on the box's cores)
    assert_same(oracle.run(seeds, N, 1000), g, "BASELINE configs[2], all 65 536 instances")
    sample = [0, 1, 31, 32, 4095, 32768, 65535]
    for inst in sample:
        logs = [sim.commit_log(inst, n) for n in range(N)]
        longest = max(logs, key=len)
        for n, lg in enumerate(logs):
            assert lg == longest[: len(lg)]
            assert oracle.state_key(lg) == int(g.last_committed_states[inst, n])
    # seed-locality: a different batch containing some of the same seeds gives the same per-seed results
    sub = seeds[1000:1064][::-1].copy()
    sim2, g2 = gpu_run(sub, N, 1000)
    np.testing.assert_array_equal(g2.commit_counts[::-1], g.commit_counts[1000:1064])
    np.testing.assert_array_equal(g2.last_committed_states[::-1], g.last_committed_states[1000:1064])


def full_size_properties(oracle, I, N, sample, kw, active_nodes, sub=slice(1000, 1032), compare=None):
    """Checks of a BASELINE configuration at its full size: the oracle on `compare` (default: every instance) plus
    size-independent properties."""
    seeds = np.arange(52, 52 + I, dtype=np.uint64)
    sim, g = gpu_run(seeds, N, 1000, **dict(kw))
    assert ((g.status & ~np.uint32(64)) == 1).all(), np.unique(g.status)
    compare = np.arange(I) if compare is None else np.asarray(compare)
    o = oracle.run(seeds[compare], N, 1000, **kw)
    np.testing.assert_array_equal(o.commit_counts, g.commit_counts[compare])
    np.testing.assert_array_equal(o.last_states, g.last_committed_states[compare])
    np.testing.assert_array_equal(o.counters[:, :8], g.counters[compare, :8])
    np.testing.assert_array_equal(o.counters[:, 9], g.counters[compare, 9])
    for inst in sample[:3]:
        logs = {n: sim.commit_log(inst, n) for n in active_nodes}
        longest = max(logs.values(), key=len)   # may be empty: a partitioned instance can commit nothing in the horizon
        for n, lg in logs.items():
            assert lg == longest[: len(lg)]                                   # one chain: every log is a prefix of the longest
            assert oracle.state_key(lg) == int(g.last_committed_states[inst, n])
    # seed-locality: a different batch holding some of the same seeds, in another order and tile position
    part = seeds[sub][::-1].copy()
    sim2, g2 = gpu_run(part, N, 1000, **dict(kw))
    np.testing.assert_array_equal(g2.commit_counts[::-1], g.commit_counts[sub])
    np.testing.assert_array_equal(g2.last_committed_states[::-1], g.last_committed_states[sub])
    return g


def test_full_size_properties_16384_instances_7_authors_partitions(oracle):
    # BASELINE configs[4]: 16 384 instances x 7 authors, a random partition plan per instance
    g = full_size_properties(oracle, 16384, 7, [0, 1, 31, 32, 8191, 16383], {"partition_windows": 4, "partition_max_len": 150},
                             active_nodes=range(7))
    # no per-instance lower bound exists: the oracle has 8.6 % of such instances commit nothing (2 048 seeds; median 9, max 30)
    best = g.commit_counts.max(axis=1)
    assert best.max() <= 60 and (best > 0).mean() > 0.5 and np.median(best) >= 5


def test_full_size_properties_8192_instances_64_authors_weighted_silent(oracle):
    # BASELINE configs[3]: 8 192 instances x 64 authors, weighted voting rights, 21 silent nodes
    silent = [n for n in range(64) if SILENT64[n]]
    # the oracle needs ~1 s per 64-author instance and core: a strided sample of 64 instances here; bench.py compares as many
    # as fit its budget on every run ("parity": checked N of 8192)
    g = full_size_properties(oracle, 8192, 64, [0, 4095, 8191], {"voting_rights": W64, "silent": SILENT64},
                             active_nodes=[n for n in range(64) if not SILENT64[n]][::9], sub=slice(1000, 1008),
                             compare=np.unique(np.linspace(0, 8191, 64).astype(np.int64)))
    assert len(silent) == 21 and (g.commit_counts[:, silent] == 0).all()       # a silent node never handles an event
    # 43 live authors hold a quorum: every instance makes progress (oracle, 48 seeds: 13..17 commits)
    assert (g.commit_counts[:, [n for n in range(64) if not SILENT64[n]]].max(axis=1) >= 1).all()


def test_capacity_overflow_is_reported_not_hidden():
    from librabft_simulator_b200 import _lib
    with pytest.raises(_lib.LbftError) as e:
        gpu_run([9, 10], 8, 1000, queue_cap=32, round_cap=32)
    assert e.value.code == _lib.LBFT_ERR_CAPACITY
    sim, g = gpu_run([9, 10], 8, 1000, strict=False, queue_cap=32, round_cap=32)
    assert (g.status & _lib.ST_ERROR_MASK).all()


# ---- BASELINE configs 2, 4, 5: extension features (semantics fixed by the oracle, SURVEY App. D) ----
W64 = [1 + (i % 3) for i in range(64)]
SILENT64 = [1 if i % 3 == 0 and i <= 60 else 0 for i in range(64)]

EXT_CASES = [
    ("config2_uniform_delay", 1, 1024, 4, 1000, {"delay_kind": 1, "delay_lo": 5, "delay_hi": 15}),
    ("weighted", 7, 32, 5, 1000, {"voting_rights": [1, 2, 5, 1, 3]}),
    ("silent_f1", 100, 32, 4, 2000, {"silent": [0, 0, 0, 1]}),
    ("silent_no_quorum", 100, 8, 4, 1000, {"silent": [0, 1, 1, 0]}),
    ("config4_64_authors_weighted_silent", 1, 4, 64, 400, {"voting_rights": W64, "silent": SILENT64}),
    ("n33", 5, 3, 33, 300, {}),
    ("config5_partitions", 1000, 96, 7, 1000, {"partition_windows": 4, "partition_max_len": 150}),
]


@pytest.mark.parametrize("name,seed0,count,nodes,max_clock,extra", EXT_CASES)
def test_gpu_extensions_match_oracle(oracle, kernel_choice, name, seed0, count, nodes, max_clock, extra):
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    o = oracle.run(seeds, nodes, max_clock, **extra)
    sim, g = gpu_run(seeds, nodes, max_clock, **dict(extra))
    assert (o.status == 1).all()
    assert ((g.status & ~np.uint32(64)) == 1).all(), np.unique(g.status)
    assert_same(o, g, name)
    assert sim.commit_log(count - 1, nodes - 2 if nodes > 1 else 0) == oracle.commit_log(
        seeds, nodes, count - 1, nodes - 2 if nodes > 1 else 0, max_clock, **extra)


@pytest.mark.parametrize("nodes,count,seed0", [(3, 4096, 10_000), (4, 8192, 20_000), (5, 2048, 30_000), (7, 1024, 40_000)])
def test_wide_seed_sweep_matches_oracle(oracle, kernel_choice, nodes, count, seed0):
    # every instance of a few thousand seeds, compared in full (the oracle needs ~1 ms per instance and core)
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    o = oracle.run(seeds, nodes, 1000)
    sim, g = gpu_run(seeds, nodes, 1000)
    assert (o.status == 1).all() and ((g.status & ~np.uint32(64)) == 1).all()
    assert_same(o, g, "sweep N=%d" % nodes)
