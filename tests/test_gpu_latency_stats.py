"""Commit-latency statistics (lbft_latency_stats) on the GPU, bit for bit against numpy over the same handle's commit_times() at
full cap: the BASELINE shapes through both kernel families; the 256 x 256 grid sweep, the same instances under a random
permutation of 1 000 sets, and 65 536 one-instance sets; a batch with error instances; re-seeded and streamed handles; long logs;
repeated calls; the state errors."""
import numpy as np
import pytest

from bench import CONFIGS, make_sim
from librabft_simulator_b200 import BatchSimulator, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _lib
from tests.latency_support import BIN_SETTINGS, WINDOWS, assert_same_stats, numpy_stats
from tests.test_gpu_sweep import grid_256

pytestmark = pytest.mark.gpu

SETTINGS = [dict(num_bins=b, bin_width=w, proposed_from=lo, proposed_until=hi) for (b, w), (lo, hi) in zip(BIN_SETTINGS, WINDOWS[::-1])]


def check_against_numpy(res, group_of, groups, settings=SETTINGS, msg=""):
    committed, proposed = res.commit_times()  # full cap: the longest log of the batch
    for kw in settings:
        got = res.latency_stats(**kw)
        want = numpy_stats(committed, proposed, res.status, group_of, groups, **kw)
        assert_same_stats(got, want, "%s %s" % (msg, kw))
        np.testing.assert_array_equal(got.hist.sum(axis=1), got.samples)
    return got


@pytest.mark.parametrize("cid", [1, 2, 3, 4, 5], ids=["config%d" % c for c in range(1, 6)])
def test_baseline_shapes(kernel_choice, cid):
    c = CONFIGS[cid]
    seeds = np.arange(c["base_seed"], c["base_seed"] + c["instances"], dtype=np.uint64)
    sim = make_sim(seeds, c["nodes"], commit_times=True, **c["kw"])
    res = sim.loop_until(c["max_clock"], strict=False)
    check_against_numpy(res, np.zeros(len(seeds), np.int64), 1, msg="config %d %s" % (cid, kernel_choice))
    full = res.latency_stats()
    assert full.samples[0] > 0 and full.instances[0] == len(seeds)
    sim.close()


def test_histogram_wider_than_shared_memory_takes_the_global_path():
    """A plain handle with num_bins above the shared-memory histogram's size: every sample adds to global memory."""
    c = CONFIGS[3]
    seeds = np.arange(c["base_seed"], c["base_seed"] + c["instances"], dtype=np.uint64)
    sim = make_sim(seeds, c["nodes"], commit_times=True)
    res = sim.loop_until(c["max_clock"])
    check_against_numpy(res, np.zeros(len(seeds), np.int64), 1, [dict(num_bins=16384), dict(num_bins=65536, bin_width=3)])
    sim.close()


def test_grid_sweep_and_other_groupings_of_the_same_instances():
    delays, configs = grid_256()
    seeds = np.arange(9000, 9256, dtype=np.uint64)
    sim = SweepSimulator.grid(seeds, delays, configs, num_nodes=4, commit_times=True)
    res = sim.loop_until(1000, strict=False)
    check_against_numpy(res, sim.set_of_instance, 256, msg="grid")
    stats = res.latency_stats(num_bins=64)
    assert (stats.instances + stats.excluded == 256).all()
    assert np.isfinite(stats.mean().reshape(len(delays), len(configs))).all()
    sim.close()
    # the same instances (seed and parameter set), grouped into 1 000 sets by a random permutation
    rng = np.random.default_rng(11)
    sets_1000 = [sim.param_sets[i % 256] for i in range(1000)]
    inst = rng.permutation(65536)
    set_of = np.empty(65536, np.uint32)
    # instance j keeps its grid point: set_of[j] is a set equal to point j // 256, chosen at random among its copies
    point = np.arange(65536) // 256
    copies = [np.arange(p, 1000, 256) for p in range(256)]
    set_of[inst] = [copies[point[j]][k % len(copies[point[j]])] for k, j in enumerate(inst)]
    perm = SweepSimulator(np.tile(seeds, 256), 4, sets_1000, set_of, commit_times=True)
    pres = perm.loop_until(1000, strict=False)
    np.testing.assert_array_equal(pres.commit_counts, res.commit_counts)
    check_against_numpy(pres, set_of, 1000, msg="1000 sets")
    # merged per grid point, the 1 000 groups give the grid's statistics
    got = pres.latency_stats(num_bins=64)
    for f in ("instances", "excluded", "samples", "sum"):
        merged = np.zeros(256, np.uint64)
        np.add.at(merged, np.arange(1000) % 256, getattr(got, f))
        np.testing.assert_array_equal(merged, getattr(stats, f), err_msg=f)
    merged = np.zeros((256, 64), np.uint64)
    np.add.at(merged, np.arange(1000) % 256, got.hist)
    np.testing.assert_array_equal(merged, stats.hist)
    perm.close()
    # 65 536 one-instance sets (constant delays keep the host setup of so many sets quick)
    cheap = [ParamSet(RandomDelay.new(m, 0.0), n) for m in (6.0, 8.0, 10.0, 14.0) for n in configs]
    one = SweepSimulator(np.arange(65536, dtype=np.uint64), 4, [cheap[i % 64] for i in range(65536)], np.arange(65536),
                         commit_times=True)
    ores = one.loop_until(1000, strict=False)
    check_against_numpy(ores, np.arange(65536), 65536, [dict(num_bins=256), dict(num_bins=256, bin_width=4, proposed_from=200,
                                                                                  proposed_until=800)], msg="one-instance sets")
    one.close()


def test_error_instances_are_excluded():
    delay = RandomDelay.new(10.0, 4.0)
    seeds = np.arange(100, 4196, dtype=np.uint64)
    free = BatchSimulator(seeds, 7, delay, commit_times=True)
    cap = int(np.median(free.loop_until(1000).counters[:, 8]))
    free.close()
    sim = BatchSimulator(seeds, 7, delay, queue_cap=cap, commit_times=True)
    res = sim.loop_until(1000, strict=False)
    bad = (res.status & np.uint32(_lib.ST_ERROR_MASK)) != 0
    assert 0 < bad.sum() < len(seeds)
    stats = res.latency_stats()
    assert stats.excluded[0] == bad.sum() and stats.instances[0] == (~bad).sum()
    clean_sim = BatchSimulator(seeds[~bad], 7, delay, queue_cap=cap, commit_times=True)
    clean = clean_sim.loop_until(1000).latency_stats()
    assert clean.excluded[0] == 0
    for f in ("instances", "samples", "sum", "min", "max", "hist"):
        np.testing.assert_array_equal(getattr(stats, f), getattr(clean, f), err_msg=f)
    sim.close()
    clean_sim.close()


def test_reseeded_and_streamed_handles_agree_with_fresh_ones(kernel_choice):
    """The commit-time table is not cleared between runs."""
    delay = RandomDelay.new(10.0, 4.0)
    batches = [np.arange(s, s + 512, dtype=np.uint64) for s in (10, 7000, 123456)]
    kw = dict(num_bins=64, bin_width=2, proposed_from=100, proposed_until=900)

    def fresh(seeds):
        sim = BatchSimulator(seeds, 4, delay, commit_times=True)
        out = sim.loop_until(1000).latency_stats(**kw)
        sim.close()
        return out

    want = [fresh(b) for b in batches]
    sim = BatchSimulator(batches[0], 4, delay, commit_times=True)
    sim.create(1000)
    for b, w in zip(batches, want):
        sim.set_seeds(b)
        assert_same_stats(sim.run().latency_stats(**kw), w, "re-seeded")
    results = list(sim.run_stream(batches[::-1]))
    assert_same_stats(results[-1].latency_stats(**kw), want[0], "streamed")
    sim.close()


def test_long_logs_count_every_row():
    seeds = np.arange(300, 428, dtype=np.uint64)
    sim = BatchSimulator(seeds, 7, RandomDelay.new(10.0, 4.0), round_cap=512, commit_times=True)
    res = sim.loop_until(5000)
    assert res.commit_counts.max() > 100
    check_against_numpy(res, np.zeros(len(seeds), np.int64), 1, SETTINGS + [dict(proposed_from=4000)])
    sim.close()


def test_repeated_calls_return_identical_bytes_and_state_errors():
    delay = RandomDelay.new(10.0, 4.0)
    sim = BatchSimulator(np.arange(4096, dtype=np.uint64), 4, delay, commit_times=True)
    res = sim.loop_until(1000)
    a, b = res.latency_stats(num_bins=100), res.latency_stats(num_bins=100)
    for f in ("instances", "excluded", "samples", "sum", "min", "max", "hist"):
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
    sim.run_async()
    with pytest.raises(_lib.LbftError) as e:
        sim.latency_stats()
    assert e.value.code == -3 and "in flight" in str(e.value)
    sim.wait()
    with pytest.raises(RuntimeError, match="latency statistics of this result are gone"):
        res.latency_stats()
    for kw in (dict(num_bins=0), dict(bin_width=0), dict(proposed_from=5, proposed_until=4), dict(num_bins=65537)):
        with pytest.raises(_lib.LbftError) as e:
            sim.latency_stats(**kw)
        assert e.value.code == -1, kw
    sim.close()
    plain = BatchSimulator(np.arange(64, dtype=np.uint64), 4, delay)
    r = plain.loop_until(1000)
    with pytest.raises(_lib.LbftError) as e:
        r.latency_stats()
    assert e.value.code == -3 and "LBFT_FLAG_COMMIT_TIMES" in str(e.value)
    plain.close()
    unrun = BatchSimulator(np.arange(64, dtype=np.uint64), 4, delay, commit_times=True).create(1000)
    with pytest.raises(_lib.LbftError) as e:
        unrun.latency_stats()
    assert e.value.code == -3 and "lbft_run first" in str(e.value)
    unrun.close()


def test_grid_example_reads_like_the_readme():
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0, 16.0, 64.0)]
    configs = [NodeConfig(delta=d) for d in (20, 40, 80, 160)]
    sim = SweepSimulator.grid(range(512), delays, configs, num_nodes=4, commit_times=True)
    stats = sim.loop_until(1000, strict=False).latency_stats(proposed_from=200, proposed_until=800)
    mean, p99 = stats.mean().reshape(4, 4), stats.percentile(99).reshape(4, 4)
    assert mean.shape == p99.shape == (4, 4) and (p99 >= stats.min.reshape(4, 4)).all()
    sim.close()
