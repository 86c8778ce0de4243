"""Block-latency statistics (lbft_block_latency_stats) without a GPU: the product's spec and threshold checks and per-instance
walk (block_latency_samples_of with block_threshold_time) on the host-compiled CT cores of plain handles, sweeps and fault sweeps,
bit for bit against numpy over the oracle's commit times; the invariants across thresholds; the refusals; the Python threshold
names; and the declarations in the header and the Rust shim."""
import ctypes
import os
import re

import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, FaultSet, SweepSimulator, _lib
from librabft_simulator_b200.simulator import resolve_threshold
from tests.block_latency_support import (BlockLatencyHarness, assert_same_block_stats, numpy_block_stats, thresholds,
                                         threshold_times)
from tests.ct_support import CtHarness
from tests.fault_support import cross, fault_kwargs
from tests.latency_support import BIN_SETTINGS, WINDOWS, make_spec
from tests.sweep_support import SETS, set_kwargs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, first seed, instances, nodes, max_clock, config keywords)
CASES = [
    ("n3", 1, 48, 3, 1000, {}),
    ("n4", 100, 64, 4, 1000, {}),
    ("n7", 400, 32, 7, 1000, dict(partition_windows=4, partition_max_len=150)),
    ("n40", 700, 6, 40, 600, {}),
    # a weighted committee: a zero-weight node, two silent nodes (total 13, quorum 9, the silent nodes hold 2)
    ("n7_weighted", 900, 32, 7, 1000, dict(voting_rights=[3, 1, 0, 2, 5, 1, 1], silent=[0, 0, 0, 0, 0, 1, 1])),
]


@pytest.fixture(scope="module")
def blk():
    return BlockLatencyHarness()


@pytest.fixture(scope="module")
def ct():
    return CtHarness()


def oracle_times(ct, seeds, nodes, max_clock, cap=256, **kw):
    committed, proposed, counts = ct.oracle(seeds, nodes, max_clock, cap=cap, **kw)
    assert counts.max() < cap  # full cap: every row
    return committed, proposed


def weights_of(nodes, kw):
    return np.ones(nodes, np.int64) if kw.get("voting_rights") is None else np.asarray(kw["voting_rights"], np.int64)


def check_against_numpy(blk, seeds, nodes, max_clock, want_times, group_of, groups, weights, msg, **run_kw):
    """Every threshold of ``thresholds`` x BIN_SETTINGS x WINDOWS; returns {threshold: stats at the widest window}."""
    committed, proposed = want_times
    seen, widest = 0, {}
    for w in thresholds(int(weights.sum())):
        for bins, width in BIN_SETTINGS:
            for lo, hi in WINDOWS:
                stats, status, h_committed, h_proposed = blk.run(seeds, nodes, max_clock, w, make_spec(bins, width, lo, hi), **run_kw)
                clean = (status & np.uint32(_lib.ST_ERROR_MASK)) == 0
                np.testing.assert_array_equal(h_committed[clean], committed[clean], err_msg=msg)
                np.testing.assert_array_equal(h_proposed[clean], proposed[clean], err_msg=msg)
                want = numpy_block_stats(committed, proposed, status, group_of, groups, weights, w, bins, width, lo, hi)
                assert_same_block_stats(stats, want, "%s W=%d bins=%d w=%d [%s, %s)" % (msg, w, bins, width, lo, hi))
                np.testing.assert_array_equal(stats.hist.sum(axis=1), stats.samples)
                seen += int(stats.samples.sum())
                if lo == hi:
                    assert (stats.samples == 0).all() and (stats.unreached == 0).all() and (stats.min == -1).all()
                if (bins, width, lo, hi) == (1024, 1, 0, None):
                    widest[w] = stats
    assert seen > 0, msg
    return widest


def assert_threshold_invariants(widest, msg=""):
    """samples + unreached is the same at every threshold (the blocks), and samples does not increase with the threshold."""
    ws = sorted(widest)
    blocks = widest[ws[0]].samples + widest[ws[0]].unreached
    for a, b in zip(ws, ws[1:]):
        np.testing.assert_array_equal(widest[b].samples + widest[b].unreached, blocks, err_msg=msg)
        assert (widest[b].samples <= widest[a].samples).all(), (msg, a, b)
    assert (widest[ws[0]].unreached == 0).all(), msg  # threshold 1: every block some node committed is reached


@pytest.mark.parametrize("name,seed0,count,nodes,max_clock,kw", CASES, ids=[c[0] for c in CASES])
def test_plain_handles_match_numpy_over_the_oracle(blk, ct, name, seed0, count, nodes, max_clock, kw):
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    times = oracle_times(ct, seeds, nodes, max_clock, **kw)
    widest = check_against_numpy(blk, seeds, nodes, max_clock, times, np.zeros(count, np.int64), 1, weights_of(nodes, kw), name, **kw)
    assert_threshold_invariants(widest, name)
    assert widest[max(widest)].instances[0] + widest[max(widest)].excluded[0] == count
    if name == "n7_weighted":  # the silent nodes never commit: "all" is never reached, a quorum is
        total = int(weights_of(nodes, kw).sum())
        assert widest[total].samples[0] == 0 and widest[total].unreached[0] > 0
        assert widest[resolve_threshold("quorum", total)].samples[0] > 0


def test_sweep_of_twelve_sets_matches_numpy_over_the_oracle(blk, ct):
    seeds = np.arange(2000, 2048, dtype=np.uint64)
    set_of = np.arange(48) % len(SETS)
    committed = np.zeros((48, 4, 256), np.int64)
    proposed = np.zeros((48, 256), np.int64)
    for s, ps in enumerate(SETS):
        idx = np.nonzero(set_of == s)[0]
        committed[idx], proposed[idx] = oracle_times(ct, seeds[idx], 4, 1000, round_cap=256, **set_kwargs(ps))
    widest = check_against_numpy(blk, seeds, 4, 1000, (committed, proposed), set_of, len(SETS), np.ones(4, np.int64), "12 sets",
                                 sets=SETS, set_of=set_of, round_cap=256)
    assert_threshold_invariants(widest, "12 sets")


def test_fault_sweep_matches_numpy_over_the_oracle(blk, ct):
    """7 nodes (f = 2): no faults, f silent, f + 1 silent (a quorum is never reached) and 4 x 150 ms partitions, crossed with two
    of the twelve sets."""
    faults = [FaultSet(), FaultSet((0, 1)), FaultSet((4, 5, 6)), FaultSet((), 4, 150)]
    sets = cross(SETS[:2], faults)
    seeds = np.arange(5000, 5064, dtype=np.uint64)
    set_of = np.arange(64) % len(sets)
    committed = np.zeros((64, 7, 256), np.int64)
    proposed = np.zeros((64, 256), np.int64)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        kw = dict(round_cap=256)
        kw.update(set_kwargs(ps))
        kw.update(fault_kwargs(ps.faults, 7))
        committed[idx], proposed[idx] = oracle_times(ct, seeds[idx], 7, 1000, **kw)
    widest = check_against_numpy(blk, seeds, 7, 1000, (committed, proposed), set_of, len(sets), np.ones(7, np.int64), "faults",
                                 sets=sets, set_of=set_of, faults=True, round_cap=256)
    assert_threshold_invariants(widest, "faults")
    quorum = widest[resolve_threshold("quorum", 7)]
    f1 = np.array([ps.faults == faults[2] for ps in sets])
    assert (quorum.samples[f1] == 0).all() and (quorum.unreached[f1] == 0).all()  # f + 1 silent: nothing is ever committed
    assert (quorum.samples[~f1] > 0).all()


def test_threshold_times_are_independent_of_tie_order():
    """Two nodes commit at the same time: T is that time whichever of them comes first, and a zero-weight node changes nothing."""
    committed = np.array([[[5], [3], [3], [-1], [9]]], np.int64)  # [I=1, N=5, cap=1]; node 3 did not commit
    for weights in ([1, 1, 1, 1, 1], [1, 0, 1, 1, 1], [1, 1, 0, 1, 1]):
        for perm in ([0, 1, 2, 3, 4], [4, 3, 2, 1, 0], [2, 0, 4, 1, 3]):
            c, w = committed[:, perm, :], np.asarray(weights)[perm]
            T, reached = threshold_times(c, w, 2)
            want = 3 if weights[1] and weights[2] else 5
            assert reached[0, 0] and T[0, 0] == want, (weights, perm)
            T, reached = threshold_times(c, w, int(w.sum()))
            assert not reached[0, 0]  # node 3 holds a voting right and never commits


def test_error_instances_are_excluded(blk, ct):
    """A queue_cap at the median of the uncapped run's max_queue makes some instances overflow: they are counted in excluded,
    and the others equal a run over just them."""
    seeds = np.arange(3000, 3064, dtype=np.uint64)
    cap = int(np.median(ct.run(seeds, 7, 1000).counters[:, 8]))
    stats, status, _, _ = blk.run(seeds, 7, 1000, 5, queue_cap=cap)
    bad = (status & np.uint32(_lib.ST_ERROR_MASK)) != 0
    assert 0 < bad.sum() < len(seeds)
    assert stats.excluded[0] == bad.sum() and stats.instances[0] == (~bad).sum()
    clean, clean_status, _, _ = blk.run(seeds[~bad], 7, 1000, 5)
    assert not (clean_status & np.uint32(_lib.ST_ERROR_MASK)).any()
    for f in ("instances", "samples", "sum", "min", "max", "hist", "unreached"):
        np.testing.assert_array_equal(getattr(stats, f), getattr(clean, f), err_msg=f)


def test_refusals(blk):
    seeds = np.arange(8, dtype=np.uint64)
    # the spec refusals of lbft_latency_stats, with its messages
    cases = [
        (dict(num_bins=0), "num_bins must be in 1..65536"),
        (dict(num_bins=65537), "num_bins must be in 1..65536"),
        (dict(bin_width=0), "bin_width must be >= 1"),
        (dict(proposed_from=10, proposed_until=9), "proposed_from must be <= proposed_until"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match="^-1: " + re.escape(msg)):
            blk.run(seeds, 4, 1000, 1, make_spec(**kw))
    spec = make_spec()
    spec.struct_size = 8
    with pytest.raises(RuntimeError, match="^-1: lbft_latency_spec.struct_size does not match"):
        blk.run(seeds, 4, 1000, 1, spec)
    sets = [SETS[i % len(SETS)] for i in range(257)]
    with pytest.raises(RuntimeError, match=r"^-1: num_groups \* num_bins must be <= 2\^24"):
        blk.run(np.arange(257, dtype=np.uint64), 4, 1000, 1, make_spec(65536), sets=sets, set_of=np.arange(257), round_cap=128)
    with pytest.raises(RuntimeError, match=r"^-1: num_instances \* num_nodes \* round_cap \* max_clock must fit in 64 bits"):
        blk.run(np.arange(1 << 16, dtype=np.uint64), 64, (1 << 29) - 1, 1, round_cap=32768, commands_per_epoch=32768)
    with pytest.raises(RuntimeError, match="^-3: commit times were not recorded"):
        blk.run(seeds, 4, 1000, 1, flags=0)
    # the threshold: 1..total voting rights (4 here; 13 for the weighted committee)
    msg = "^-1: " + re.escape("threshold must be in 1..total voting rights of the handle")
    for w in (0, 5, 1 << 63, (1 << 64) - 1):
        with pytest.raises(RuntimeError, match=msg):
            blk.run(seeds, 4, 1000, w)
    with pytest.raises(RuntimeError, match=msg):
        blk.run(seeds, 7, 1000, 14, voting_rights=[3, 1, 0, 2, 5, 1, 1])
    blk.run(seeds, 7, 1000, 13, voting_rights=[3, 1, 0, 2, 5, 1, 1])
    blk.run(seeds, 4, 1000, 4)


def test_c_abi_checks_arguments_without_a_device():
    lib = _lib.load()
    spec = make_spec()
    out = (_lib.LbftLatencySummary * 1)()
    assert lib.lbft_block_latency_stats(None, ctypes.byref(spec), 1, ctypes.cast(out, ctypes.c_void_p), None, None) == -1
    assert b"must not be NULL" in lib.lbft_last_error()
    assert lib.lbft_block_latency_stats(None, None, 1, None, None, None) == -1


@pytest.mark.parametrize("total", [1, 2, 3, 4, 5, 6, 7, 10, 13, 40, 64, 100, 127, 1 << 20])
def test_threshold_names_follow_the_reference_formulas(total):
    """configuration.rs:52-62: quorum_threshold = 2 * total / 3 + 1, validity_threshold = (total + 2) / 3."""
    assert resolve_threshold("first", total) == 1
    assert resolve_threshold("validity", total) == (total + 2) // 3
    assert resolve_threshold("quorum", total) == 2 * total // 3 + 1
    assert resolve_threshold("all", total) == total
    assert resolve_threshold(7, total) == 7
    for N in (1, 4, 7, 10, 40, 64):  # with equal weights: f + 1 and N - f, N = 3f + 1 + k
        f = (N - 1) // 3
        assert resolve_threshold("validity", N) == f + 1
        assert resolve_threshold("quorum", N) == N - f


def test_threshold_name_errors_and_totals():
    for bad in ("Quorum", "", "f+1", "majority"):
        with pytest.raises(ValueError, match="threshold must be an int or one of"):
            resolve_threshold(bad, 4)
    assert BatchSimulator([1, 2], 4).total_voting_rights() == 4
    assert BatchSimulator([1, 2], 7, voting_rights=[3, 1, 0, 2, 5, 1, 1]).total_voting_rights() == 13
    weights = 1 + np.arange(64) % 3
    assert BatchSimulator([1], 64, voting_rights=weights).total_voting_rights() == 127
    assert resolve_threshold("quorum", 127) == 85
    sweep = SweepSimulator.grid(2, [SETS[0].network_delay], [SETS[0].node_config], num_nodes=7, faults=[FaultSet(), FaultSet((0,))])
    assert sweep.total_voting_rights() == 7 and hasattr(sweep, "block_latency_stats")
    with pytest.raises(ValueError):  # raised before the handle is touched
        sweep.block_latency_stats("nope")


def test_header_python_and_rust_declarations():
    header = open(os.path.join(ROOT, "include", "lbft.h")).read()
    assert re.search(r"int lbft_block_latency_stats\(lbft_sim\* sim, const lbft_latency_spec\* spec, uint64_t threshold, "
                     r"lbft_latency_summary\* out,\s+uint64_t\* unreached, uint64_t\* hist\);", header)
    assert re.search(r"#define LBFT_ABI_VERSION 1\b", header)
    rust = open(os.path.join(ROOT, "bft-lib-gpu", "src", "lib.rs")).read()
    assert re.search(r"pub fn lbft_block_latency_stats\(sim: \*mut LbftSim, spec: \*const lbft_latency_spec, threshold: u64,\s+"
                     r"out: \*mut lbft_latency_summary, unreached: \*mut u64, hist: \*mut u64\) -> c_int;", rust)
    assert "pub fn block_latency_stats(&self" in rust
    assert "lbft_block_latency_stats" in _lib.EXPORTS
    lib = _lib.load()
    assert lib.lbft_block_latency_stats.argtypes[2] is ctypes.c_uint64
