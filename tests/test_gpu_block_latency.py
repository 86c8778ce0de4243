"""Block-latency statistics (lbft_block_latency_stats) on the GPU, bit for bit against numpy over the same handle's
commit_times() at full cap: the BASELINE shapes through both kernel families at the named thresholds (config 4: two nodes per
lane, weighted and with silent authors); the 256 x 256 grid sweep and the same instances under a random permutation of 1 000
sets; a histogram wider than shared memory; a fault-sweep grid; a batch with error instances; re-seeded handles; repeated calls;
the state errors."""
import numpy as np
import pytest

from bench import CONFIGS, make_sim
from librabft_simulator_b200 import BatchSimulator, FaultSet, NodeConfig, RandomDelay, SweepSimulator, _lib
from librabft_simulator_b200.simulator import resolve_threshold
from tests.block_latency_support import THRESHOLD_NAMES, assert_same_block_stats, numpy_block_stats
from tests.latency_support import BIN_SETTINGS, WINDOWS
from tests.test_gpu_sweep import grid_256

pytestmark = pytest.mark.gpu

SETTINGS = [dict(num_bins=b, bin_width=w, proposed_from=lo, proposed_until=hi) for (b, w), (lo, hi) in zip(BIN_SETTINGS, WINDOWS[::-1])]


def weights_of(sim):
    return np.ones(sim.num_nodes, np.int64) if sim.voting_rights is None else sim.voting_rights.astype(np.int64)


def check_against_numpy(sim, res, group_of, groups, thresholds=THRESHOLD_NAMES, settings=SETTINGS, msg=""):
    """Returns {threshold name or value: its statistics over the whole run with 1 024 one-ms bins}."""
    committed, proposed = res.commit_times()  # full cap: the longest log of the batch
    total = sim.total_voting_rights()
    out = {}
    for t in thresholds:
        for kw in settings:
            got = res.block_latency_stats(t, **kw)
            assert got.threshold == resolve_threshold(t, total)
            want = numpy_block_stats(committed, proposed, res.status, group_of, groups, weights_of(sim), got.threshold, **kw)
            assert_same_block_stats(got, want, "%s %s %s" % (msg, t, kw))
            np.testing.assert_array_equal(got.hist.sum(axis=1), got.samples)
        out[t] = res.block_latency_stats(t)
    return out


@pytest.mark.parametrize("cid", [1, 2, 3, 4, 5], ids=["config%d" % c for c in range(1, 6)])
def test_baseline_shapes(kernel_choice, cid):
    c = CONFIGS[cid]
    seeds = np.arange(c["base_seed"], c["base_seed"] + c["instances"], dtype=np.uint64)
    sim = make_sim(seeds, c["nodes"], commit_times=True, **c["kw"])
    res = sim.loop_until(c["max_clock"], strict=False)
    out = check_against_numpy(sim, res, np.zeros(len(seeds), np.int64), 1, msg="config %d %s" % (cid, kernel_choice))
    assert out["first"].samples[0] > 0 and out["first"].unreached[0] == 0
    assert out["quorum"].samples[0] > 0
    if cid == 4:  # 64 weighted authors, 21 of them silent: total 127, quorum 85, and "all" is never reached
        assert sim.total_voting_rights() == 127 and out["quorum"].threshold == 85
        assert out["all"].samples[0] == 0 and out["all"].unreached[0] > 0
    sim.close()


def test_grid_sweep_permuted_sets_and_a_global_histogram():
    delays, configs = grid_256()
    seeds = np.arange(9000, 9256, dtype=np.uint64)
    sim = SweepSimulator.grid(seeds, delays, configs, num_nodes=4, commit_times=True)
    res = sim.loop_until(1000, strict=False)
    check_against_numpy(sim, res, sim.set_of_instance, 256, ["quorum", 2], msg="grid")
    check_against_numpy(sim, res, sim.set_of_instance, 256, ["validity"], [dict(num_bins=16384)], msg="grid, 16 384 bins")
    stats = res.block_latency_stats("quorum", num_bins=64)
    assert (stats.instances + stats.excluded == 256).all()
    assert np.isfinite(stats.mean().reshape(len(delays), len(configs))).all()
    sim.close()
    # the same instances (seed and parameter set), grouped into 1 000 sets by a random permutation: warps and blocks mix groups
    rng = np.random.default_rng(11)
    sets_1000 = [sim.param_sets[i % 256] for i in range(1000)]
    inst = rng.permutation(65536)
    set_of = np.empty(65536, np.uint32)
    point = np.arange(65536) // 256
    copies = [np.arange(p, 1000, 256) for p in range(256)]
    set_of[inst] = [copies[point[j]][k % len(copies[point[j]])] for k, j in enumerate(inst)]
    perm = SweepSimulator(np.tile(seeds, 256), 4, sets_1000, set_of, commit_times=True)
    pres = perm.loop_until(1000, strict=False)
    np.testing.assert_array_equal(pres.commit_counts, res.commit_counts)
    check_against_numpy(perm, pres, set_of, 1000, ["quorum"], msg="1000 sets")
    got = pres.block_latency_stats("quorum", num_bins=64)
    for f in ("instances", "excluded", "samples", "sum", "unreached"):
        merged = np.zeros(256, np.uint64)
        np.add.at(merged, np.arange(1000) % 256, getattr(got, f))
        np.testing.assert_array_equal(merged, getattr(stats, f), err_msg=f)
    perm.close()


def test_fault_sweep_grid_of_crashed_nodes():
    """7 nodes (f = 2) with 0, 1 and 2 crashed nodes: the quorum latency of the README's cube."""
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 16.0)]
    configs = [NodeConfig(delta=d) for d in (20, 80)]
    faults = [FaultSet(), FaultSet((6,)), FaultSet((5, 6))]
    sim = SweepSimulator.grid(range(512), delays, configs, num_nodes=7, faults=faults, commit_times=True)
    res = sim.loop_until(1000, strict=False)
    out = check_against_numpy(sim, res, sim.set_of_instance, len(sim.param_sets), THRESHOLD_NAMES + [4], msg="faults")
    quorum = res.block_latency_stats("quorum", proposed_from=200, proposed_until=800)
    cube = quorum.mean().reshape(len(delays), len(configs), len(faults))
    assert np.isfinite(cube[:, :, 0]).all()  # (with crashed nodes and delta = 80, no block proposed in the window commits: nan)
    crashed = np.array([len(ps.faults.silent) > 0 for ps in sim.param_sets])
    blocks = out["first"].samples + out["first"].unreached
    # with a crashed node no block is ever committed by all: every block of those sets is unreached
    assert (out["all"].samples[crashed] == 0).all()
    np.testing.assert_array_equal(out["all"].unreached[crashed], blocks[crashed])
    assert blocks[crashed].sum() > 0 and (out["quorum"].samples[crashed] > 0).any()
    sim.close()


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
    check_against_numpy(sim, res, np.zeros(len(seeds), np.int64), 1, ["quorum"], msg="errors")
    stats = res.block_latency_stats()
    assert stats.excluded[0] == bad.sum() and stats.instances[0] == (~bad).sum()
    sim.close()


def test_reseeded_handles_agree_with_fresh_ones(kernel_choice):
    """The commit-time table is not cleared between runs."""
    delay = RandomDelay.new(10.0, 4.0)
    batches = [np.arange(s, s + 512, dtype=np.uint64) for s in (10, 7000)]
    kw = dict(num_bins=64, bin_width=2, proposed_from=100, proposed_until=900)

    def fresh(seeds):
        sim = BatchSimulator(seeds, 4, delay, commit_times=True)
        out = sim.loop_until(1000).block_latency_stats("quorum", **kw)
        sim.close()
        return out

    want = [fresh(b) for b in batches]
    sim = BatchSimulator(batches[0], 4, delay, commit_times=True)
    sim.create(1000)
    for b, w in zip(batches[::-1], want[::-1]):
        sim.set_seeds(b)
        assert_same_block_stats(sim.run().block_latency_stats("quorum", **kw), w, "re-seeded")
    sim.close()


def test_repeated_calls_return_identical_bytes_and_state_errors():
    delay = RandomDelay.new(10.0, 4.0)
    sim = BatchSimulator(np.arange(4096, dtype=np.uint64), 4, delay, commit_times=True)
    res = sim.loop_until(1000)
    a, b = res.block_latency_stats("validity", num_bins=100), res.block_latency_stats("validity", num_bins=100)
    for f in ("instances", "excluded", "samples", "sum", "min", "max", "hist", "unreached"):
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
    for t in (0, 5, -1):
        with pytest.raises(_lib.LbftError, match="threshold must be in 1..total voting rights") as e:
            res.block_latency_stats(t)
        assert e.value.code == -1
    with pytest.raises(ValueError):
        res.block_latency_stats("most")
    sim.run_async()
    with pytest.raises(_lib.LbftError) as e:
        sim.block_latency_stats()
    assert e.value.code == -3 and "in flight" in str(e.value)
    sim.wait()
    with pytest.raises(RuntimeError, match="block latency statistics of this result are gone"):
        res.block_latency_stats()
    sim.close()
    plain = BatchSimulator(np.arange(64, dtype=np.uint64), 4, delay)
    r = plain.loop_until(1000)
    with pytest.raises(_lib.LbftError) as e:
        r.block_latency_stats()
    assert e.value.code == -3 and "LBFT_FLAG_COMMIT_TIMES" in str(e.value)
    plain.close()
    unrun = BatchSimulator(np.arange(64, dtype=np.uint64), 4, delay, commit_times=True).create(1000)
    with pytest.raises(_lib.LbftError) as e:
        unrun.block_latency_stats()
    assert e.value.code == -3 and "lbft_run first" in str(e.value)
    unrun.close()
