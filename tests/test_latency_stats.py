"""Commit-latency statistics (lbft_latency_stats) without a GPU: the product's spec check and per-instance walk
(latency_samples_of) on the host-compiled CT core, bit for bit against numpy over the oracle's commit times; the refusals; the
arithmetic of LatencyStats; and the new structs between the header, the Python binding and the Rust shim."""
import ctypes
import os
import re

import numpy as np
import pytest

from librabft_simulator_b200 import LatencyStats, _lib
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE
from tests.ct_support import CtHarness
from tests.latency_support import BIN_SETTINGS, WINDOWS, LatencyHarness, assert_same_stats, make_spec, numpy_stats
from tests.sweep_support import SETS, set_kwargs
from tests.test_rust_shim import c_struct_fields, rust_struct_fields

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, first seed, instances, nodes, max_clock, config keywords)
CASES = [
    ("n3", 1, 48, 3, 1000, {}),
    ("n4", 100, 64, 4, 1000, {}),
    ("n7", 400, 32, 7, 1000, dict(partition_windows=4, partition_max_len=150)),
    ("n40", 700, 6, 40, 600, {}),
]


@pytest.fixture(scope="module")
def lat():
    return LatencyHarness()


@pytest.fixture(scope="module")
def ct():
    return CtHarness()


def oracle_times(ct, seeds, nodes, max_clock, cap=256, **kw):
    committed, proposed, counts = ct.oracle(seeds, nodes, max_clock, cap=cap, **kw)
    assert counts.max() < cap  # full cap: every row
    return committed, proposed


@pytest.mark.parametrize("name,seed0,count,nodes,max_clock,kw", CASES, ids=[c[0] for c in CASES])
def test_plain_handles_match_numpy_over_the_oracle(lat, ct, name, seed0, count, nodes, max_clock, kw):
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    committed, proposed = oracle_times(ct, seeds, nodes, max_clock, **kw)
    seen_samples = 0
    for bins, width in BIN_SETTINGS:
        for lo, hi in WINDOWS:
            stats, status = lat.run(seeds, nodes, max_clock, make_spec(bins, width, lo, hi), **kw)
            want = numpy_stats(committed, proposed, status, np.zeros(count, np.int64), 1, bins, width, lo, hi)
            assert_same_stats(stats, want, "%s bins=%d w=%d [%s, %s)" % (name, bins, width, lo, hi))
            assert int(stats.hist.sum()) == int(stats.samples[0])
            seen_samples += int(stats.samples[0])
            if lo == hi:
                assert stats.samples[0] == 0 and stats.min[0] == -1 and stats.max[0] == -1
    assert seen_samples > 0
    assert stats.instances[0] + stats.excluded[0] == count


def test_sweep_of_twelve_sets_matches_numpy_over_the_oracle(lat, ct):
    seeds = np.arange(2000, 2048, dtype=np.uint64)
    set_of = np.arange(48) % len(SETS)
    committed = np.zeros((48, 4, 256), np.int64)
    proposed = np.zeros((48, 256), np.int64)
    for s, ps in enumerate(SETS):
        idx = np.nonzero(set_of == s)[0]
        committed[idx], proposed[idx] = oracle_times(ct, seeds[idx], 4, 1000, round_cap=256, **set_kwargs(ps))
    overflow_filled = False
    for bins, width in BIN_SETTINGS:
        for lo, hi in WINDOWS:
            stats, status = lat.run(seeds, 4, 1000, make_spec(bins, width, lo, hi), sets=SETS, set_of=set_of, round_cap=256)
            want = numpy_stats(committed, proposed, status, set_of, len(SETS), bins, width, lo, hi)
            assert_same_stats(stats, want, "bins=%d w=%d [%s, %s)" % (bins, width, lo, hi))
            np.testing.assert_array_equal(stats.hist.sum(axis=1), stats.samples)
            if bins == 5:
                overflow_filled |= bool((stats.hist[:, -1] > 0).any())
    assert overflow_filled
    assert (stats.instances + stats.excluded == 4).all()


def test_error_instances_are_excluded_and_not_walked(lat, ct):
    """A queue_cap at the median of the uncapped run's max_queue makes some instances overflow: they are counted in excluded,
    and the others equal a run over just them."""
    seeds = np.arange(3000, 3064, dtype=np.uint64)
    cap = int(np.median(ct.run(seeds, 7, 1000).counters[:, 8]))
    stats, status = lat.run(seeds, 7, 1000, queue_cap=cap)
    bad = (status & np.uint32(_lib.ST_ERROR_MASK)) != 0
    assert 0 < bad.sum() < len(seeds)
    assert stats.excluded[0] == bad.sum() and stats.instances[0] == (~bad).sum()
    clean, clean_status = lat.run(seeds[~bad], 7, 1000)
    assert not (clean_status & np.uint32(_lib.ST_ERROR_MASK)).any()
    assert clean.excluded[0] == 0
    for f in ("instances", "samples", "sum", "min", "max", "hist"):
        np.testing.assert_array_equal(getattr(stats, f), getattr(clean, f), err_msg=f)


def test_refusals(lat):
    seeds = np.arange(8, dtype=np.uint64)
    cases = [
        (dict(num_bins=0), "num_bins must be in 1..65536"),
        (dict(num_bins=65537), "num_bins must be in 1..65536"),
        (dict(bin_width=0), "bin_width must be >= 1"),
        (dict(proposed_from=10, proposed_until=9), "proposed_from must be <= proposed_until"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match="^-1: " + re.escape(msg)):
            lat.run(seeds, 4, 1000, make_spec(**kw))
    spec = make_spec()
    spec.struct_size = 8
    with pytest.raises(RuntimeError, match="^-1: lbft_latency_spec.struct_size does not match"):
        lat.run(seeds, 4, 1000, spec)
    # num_groups * num_bins: 257 sets x 65536 bins is one bin too many per set; 256 x 65536 = 2^24 is accepted
    sets = [SETS[i % len(SETS)] for i in range(257)]
    with pytest.raises(RuntimeError, match=r"^-1: num_groups \* num_bins must be <= 2\^24"):
        lat.run(np.arange(257, dtype=np.uint64), 4, 1000, make_spec(65536), sets=sets, set_of=np.arange(257), round_cap=128)
    # the bound on sum: I * N * round_cap * max_clock >= 2^64 (checked before anything runs)
    with pytest.raises(RuntimeError, match=r"^-1: num_instances \* num_nodes \* round_cap \* max_clock must fit in 64 bits"):
        lat.run(np.arange(1 << 16, dtype=np.uint64), 64, (1 << 29) - 1, round_cap=32768, commands_per_epoch=32768)
    with pytest.raises(RuntimeError, match="^-3: commit times were not recorded"):
        lat.run(seeds, 4, 1000, flags=0)


def test_largest_grouping_is_accepted(lat):
    sets = [SETS[i % len(SETS)] for i in range(256)]
    stats, _ = lat.run(np.arange(256, dtype=np.uint64), 4, 300, make_spec(65536), sets=sets, set_of=np.arange(256), round_cap=64)
    assert stats.hist.shape == (256, 65536)
    np.testing.assert_array_equal(stats.hist.sum(axis=1), stats.samples)


def test_c_abi_checks_arguments_without_a_device():
    lib = _lib.load()
    spec = make_spec()
    out = (_lib.LbftLatencySummary * 1)()
    assert lib.lbft_latency_stats(None, ctypes.byref(spec), ctypes.cast(out, ctypes.c_void_p), None) == -1
    assert b"must not be NULL" in lib.lbft_last_error()
    assert lib.lbft_latency_stats(None, None, None, None) == -1


def synthetic(hists, bin_width=1):
    hist = np.asarray(hists, dtype=np.uint64)
    out = np.zeros(hist.shape[0], LATENCY_SUMMARY_DTYPE)
    out["samples"] = hist.sum(axis=1)
    centres = np.arange(hist.shape[1]) * bin_width
    out["sum"] = (hist * centres.astype(np.uint64)).sum(axis=1)
    return LatencyStats(out, hist, bin_width)


@pytest.mark.parametrize("q", [0, 1, 50, 90, 99, 100])
def test_percentile_equals_numpy_inverted_cdf(q):
    rng = np.random.default_rng(7)
    for n in (1, 2, 3, 7, 10, 99, 100, 101, 1000, 4099):
        lat = rng.integers(0, 60, size=n)
        hist = np.bincount(lat, minlength=64)  # bin width 1, last bin (63) empty
        stats = synthetic([hist])
        assert stats.percentile(q)[0] == np.percentile(lat, q, method="inverted_cdf"), (q, n)
    # with a wider bin: the lower edge of the bin that holds numpy's answer
    lat = rng.integers(0, 60, size=777)
    stats = synthetic([np.bincount(lat // 5, minlength=13)], bin_width=5)
    assert stats.percentile(q)[0] == np.percentile(lat, q, method="inverted_cdf") // 5 * 5


def test_percentile_empty_group_and_overflow_bin():
    stats = synthetic([[0, 0, 0, 0], [3, 0, 0, 1], [0, 0, 0, 5]], bin_width=10)
    np.testing.assert_array_equal(stats.mean()[1:], [30 / 4, 30.0])
    assert np.isnan(stats.mean()[0])
    p = stats.percentile(75)
    assert np.isnan(p[0]) and p[1] == 0.0 and p[2] == np.inf
    p = stats.percentile(76)
    assert p[1] == np.inf
    assert stats.percentile(0)[1] == 0.0
    with pytest.raises(ValueError):
        stats.percentile(100.5)


def test_percentile_rank_is_exact():
    """In floating point, 7 / 100 * 100 is 7.000000000000001, whose ceiling would make the rank 8; the exact rank is 7."""
    assert np.ceil(7 / 100 * 100) == 8
    hist = np.zeros((1, 200), np.uint64)
    hist[0, :100] = 1  # latencies 0..99, one each
    stats = synthetic(hist)
    assert stats.percentile(7)[0] == 6.0
    assert stats.percentile(7.5)[0] == 7.0


def test_structs_match_the_header_python_and_the_rust_shim():
    py = {"lbft_latency_spec": _lib.LbftLatencySpec, "lbft_latency_summary": _lib.LbftLatencySummary}
    kinds = {ctypes.c_uint32: "u32", ctypes.c_uint64: "u64", ctypes.c_int64: "i64"}
    for cname, rname in (("lbft_latency_spec", "LbftLatencySpec"), ("lbft_latency_summary", "LbftLatencySummary")):
        c = c_struct_fields(cname)
        assert c == rust_struct_fields(rname), cname
        assert c == [(n, kinds[t]) for n, t in py[cname]._fields_], cname
    assert ctypes.sizeof(_lib.LbftLatencySpec) == 32 and ctypes.sizeof(_lib.LbftLatencySummary) == 48
    assert [(n, t) for n, t in c_struct_fields("lbft_latency_summary")] == [
        (n, "i64" if LATENCY_SUMMARY_DTYPE[n] == np.int64 else "u64") for n in LATENCY_SUMMARY_DTYPE.names]
    header = open(os.path.join(ROOT, "include", "lbft.h")).read()
    assert re.search(r"int lbft_latency_stats\(lbft_sim\* sim, const lbft_latency_spec\* spec, lbft_latency_summary\* out, "
                     r"uint64_t\* hist\);", header)
    assert re.search(r"#define LBFT_ABI_VERSION 1\b", header)
    rust = open(os.path.join(ROOT, "bft-lib-gpu", "src", "lib.rs")).read()
    assert re.search(r"pub fn lbft_latency_stats\(sim: \*mut LbftSim, spec: \*const lbft_latency_spec, out: \*mut lbft_latency_summary, "
                     r"hist: \*mut u64\) -> c_int;", rust)
    assert "pub fn latency_stats(&self" in rust
    assert "lbft_latency_stats" in _lib.EXPORTS
