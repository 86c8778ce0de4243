"""The latency reduction on the GPU at every lane-group width and along every reduction path, on purpose.  Both overloads of
lbft_latency_stats_kernel (per-sample and threshold) are compared bit for bit with numpy over the handle's own commit_times():

* lane widths: the threshold overload gives each instance G lanes, G the smallest power of two >= min(N, 32), and at N > 32 a
  lane holds nodes j and j + 32.  N in {1, 2, 3, 5, 8, 9, 16, 17, 31, 32, 33, 47, 63, 64} (G = 1 .. 32, a partly filled warp,
  a partly filled upper half) with zero voting rights (node 0 among them), 2^24 on the top node and node 32, a seeded random
  vector with the top node silent; batches of k * 128 + 1 instances, so the last block of either launch holds one instance;
  and, per width, a small handle against numpy over the oracle's commit times;
* reduction paths: shared (8 192 bins) and global (8 193) histograms; groups of 96 (uniform warps, mixed blocks), 100 (mixed
  warps) and 3 (several groups in one warp of the threshold launch at G = 8 and 16); one instance per group; groups x bins
  at 2^24 and one bin over (refused); error instances inside uniform warps against a run of the clean seeds alone;
* merge identity: a grid's one-instance-per-group statistics merged per point equal the grid's, and a plain handle's equal the
  merge of its seeds split over any grouping;
* the lane form alone (sim_core.cuh block_threshold_time_lanes) through a device probe over synthetic tables at every N from 1
  to 64, against block_threshold_time on the host and numpy."""
import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, NodeConfig, ParamSet, RandomDelay, SweepSimulator, _lib
from tests.block_latency_support import (CAP, BlockLatencyHarness, BlockThresholdProbe, assert_same_block_stats, numpy_block_stats,
                                         numpy_threshold_times, synthetic_cases, synthetic_thresholds, thresholds)
from tests.ct_support import CtHarness
from tests.latency_support import assert_same_stats, numpy_stats

pytestmark = pytest.mark.gpu

INT64_MAX = np.iinfo(np.int64).max
DELAY = RandomDelay.new(10.0, 4.0)
LANE_NS = [1, 2, 3, 5, 8, 9, 16, 17, 31, 32, 33, 47, 63, 64]


def lanes(N):
    G = 1
    while G < N and G < 32:
        G *= 2
    return G


def weights_of(sim):
    return np.ones(sim.num_nodes, np.int64) if sim.voting_rights is None else sim.voting_rights.astype(np.int64)


def lane_weights(N):
    """(name, voting rights, silent) per N: zeros with node 0 among them, the cap on nodes 0, 32 and the top one, and a seeded random
    vector with the top node silent (N >= 4, so that the others still hold a quorum)."""
    out = []
    if N > 1:
        out.append(("zeros", np.array([0 if n % 3 == 0 else 1 + n % 2 for n in range(N)]), None))
    cap = np.ones(N, np.int64)
    cap[[0, N - 1]] = CAP  # (node 0 too, so that no node holds a quorum alone and rounds do not race past the table)
    if N > 32:
        cap[32] = CAP
    out.append(("cap", cap, None))
    if N >= 4:
        w = np.random.default_rng(N).integers(1, 4, N)
        w[N - 1] = 1
        out.append(("random, top silent", w, [0] * (N - 1) + [1]))
    return out


def horizon(N, w, silent):
    """A horizon at which the instances commit and the round table holds: short when one node holds a quorum alone (it commits
    every round), long when a node is silent (the first rounds it leads time out)."""
    if w.max() >= 2 * w.sum() // 3 + 1:
        return 60
    return 1000 if silent is not None else 300 if N > 32 else 400


def run(seeds, N, max_clock, sets=None, set_of=None, **kw):
    sim = (BatchSimulator(seeds, N, DELAY, commit_times=True, **kw) if sets is None else
           SweepSimulator(seeds, N, sets, set_of, commit_times=True, **kw))
    return sim, sim.loop_until(max_clock, strict=False)


def check_both(sim, res, group_of, groups, ws, spec):
    """Both overloads against numpy over the handle's commit times at full cap; returns {W: block statistics}."""
    committed, proposed = res.commit_times()
    assert_same_stats(res.latency_stats(**spec), numpy_stats(committed, proposed, res.status, group_of, groups, **spec), "per-sample")
    out = {}
    for w in ws:
        got = res.block_latency_stats(int(w), **spec)
        want = numpy_block_stats(committed, proposed, res.status, group_of, groups, weights_of(sim), int(w), **spec)
        assert_same_block_stats(got, want, "W=%d %s" % (w, spec))
        out[int(w)] = got
    return out


def has_ties(committed):
    """Whether some block has two nodes committing it at the same clock."""
    t = np.sort(np.where(committed >= 0, committed, INT64_MAX), axis=1)
    return bool(((t[:, 1:, :] == t[:, :-1, :]) & (t[:, 1:, :] < INT64_MAX)).any())


def zero_weight_first(cc, times, weights):
    """Whether some block of a synthetic table is committed by a zero-weight node strictly before every node with a voting right."""
    N = cc.shape[1]
    t = np.where(cc[:, :, None] > np.arange(times.shape[2]), times[:, :N, :], INT64_MAX)
    pos = np.where((weights > 0)[None, :, None], t, INT64_MAX).min(axis=1)
    zero = np.where((weights == 0)[None, :, None], t, INT64_MAX).min(axis=1)
    return bool((zero < pos).any())


@pytest.fixture(scope="module")
def ct():
    return CtHarness()


@pytest.mark.parametrize("N", LANE_NS)
def test_lane_widths(ct, N):
    """257 instances (the last block of the per-sample launch, and of the threshold launch at every G, holds one instance)."""
    seeds = np.arange(7000 + 1000 * N, 7000 + 1000 * N + 257, dtype=np.uint64)
    rng = np.random.default_rng(N)
    spec = dict(num_bins=64, bin_width=2, proposed_from=0, proposed_until=None)
    saw_ties = False
    for name, w, silent in lane_weights(N):
        max_clock = horizon(N, w, silent)
        sim, res = run(seeds, N, max_clock, voting_rights=w, silent=silent)
        try:
            assert not (res.status & np.uint32(_lib.ST_ERROR_MASK)).any()
            assert (res.commit_counts.max(axis=1) > 0).mean() > 0.9, "%s: instances that never committed" % name
            total = int(w.sum())
            ws = set(synthetic_thresholds(w, rng)) | set(thresholds(total)) | {int(w.max()), min(total, int(w.max()) + 1)}
            ws |= {total - 1} if total > 1 else set()
            out = check_both(sim, res, np.zeros(len(seeds), np.int64), 1, sorted(ws), spec)
            blocks = out[1].samples + out[1].unreached
            for t in out:
                np.testing.assert_array_equal(out[t].samples + out[t].unreached, blocks, err_msg="%s W=%d" % (name, t))
            assert out[1].unreached[0] == 0 and blocks[0] > 0
            if silent is not None:
                assert out[total].samples[0] == 0 and out[total].unreached[0] == blocks[0]
            saw_ties |= has_ties(res.commit_times()[0])
        finally:
            sim.close()
    # (a committee of two never ties in these runs, and none commits a block at a zero-weight node strictly first:
    # test_lane_form_on_synthetic_tables asserts both on its tables)
    assert saw_ties or N <= 2, "no block with two nodes committing at one clock"
    # a few instances against numpy over the oracle's commit times: a reference that does not rest on the device read-out
    name, w, silent = lane_weights(N)[0]
    max_clock = horizon(N, w, silent)
    few = seeds[:2 if N > 32 else 4]
    sim, res = run(few, N, max_clock, voting_rights=w, silent=silent)
    try:
        cap = int(res.commit_counts.max()) + 1
        oc, op, counts = ct.oracle(few, N, max_clock, cap=cap, voting_rights=w, silent=silent)
        np.testing.assert_array_equal(counts, res.commit_counts)
        total = int(w.sum())
        for t in thresholds(total):
            want = numpy_block_stats(oc, op, res.status, np.zeros(len(few), np.int64), 1, w.astype(np.int64), t, **spec)
            assert_same_block_stats(res.block_latency_stats(t, **spec), want, "oracle, W=%d" % t)
            assert want.samples[0] > 0 or t == total
    finally:
        sim.close()


def test_shared_and_global_histograms():
    """8 192 bins fit shared memory (a plain handle: every block in one group); 8 193 do not."""
    seeds = np.arange(4097, dtype=np.uint64)
    sim, res = run(seeds, 7, 600)
    try:
        for bins in (8192, 8193):
            out = check_both(sim, res, np.zeros(len(seeds), np.int64), 1, [1, 3, 5, 7], dict(num_bins=bins, bin_width=1))
            assert out[5].samples[0] > 0
    finally:
        sim.close()


SETS = [ParamSet(RandomDelay.new(10.0, 4.0)), ParamSet(RandomDelay.new(20.0, 30.0), NodeConfig(delta=30)),
        ParamSet(RandomDelay.uniform(2, 14)), ParamSet(RandomDelay.new(8.0, 0.0))]


@pytest.mark.parametrize("N,I,size", [(4, 96 * 12, 96), (4, 1000, 100), (7, 385, 3), (12, 385, 3), (33, 193, 3), (4, 513, 1)],
                         ids=["groups_of_96", "groups_of_100", "groups_of_3_G8", "groups_of_3_G16", "groups_of_3_G32", "one_per_group"])
def test_groupings(N, I, size):
    """Contiguous groups of `size` instances (sets cycled), so warps and blocks are uniform or not as the size says."""
    set_of = np.arange(I) // size
    groups = int(set_of.max()) + 1
    sets = [SETS[g % len(SETS)] for g in range(groups)]
    seeds = np.arange(300, 300 + I, dtype=np.uint64)
    sim, res = run(seeds, N, 400, sets, set_of)
    try:
        ws = thresholds(N) + ([N - 1] if N > 1 else [])
        for spec in (dict(num_bins=32, bin_width=3, proposed_from=50, proposed_until=350), dict(num_bins=8193)):
            out = check_both(sim, res, set_of, groups, ws, spec)
        assert (out[1].samples > 0).mean() > 0.9
    finally:
        sim.close()


def test_groups_times_bins_at_the_limit():
    """512 one-instance groups x 32 768 bins = 2^24: accepted and exact; one bin more is refused."""
    I = 512
    sets = [SETS[i % len(SETS)] for i in range(I)]
    sim, res = run(np.arange(I, dtype=np.uint64), 4, 300, sets, np.arange(I))
    try:
        check_both(sim, res, np.arange(I), I, [3], dict(num_bins=1 << 15, bin_width=1))
        for call in (lambda: res.latency_stats(num_bins=(1 << 15) + 1), lambda: res.block_latency_stats(3, num_bins=(1 << 15) + 1)):
            with pytest.raises(_lib.LbftError, match=r"num_groups \* num_bins must be <= 2\^24") as e:
                call()
            assert e.value.code == -1
    finally:
        sim.close()


@pytest.mark.parametrize("sweep", [False, True], ids=["plain", "groups_of_96"])
def test_error_instances_in_uniform_warps(sweep):
    """A queue_cap at the median max_queue of an uncapped run flags about half the instances, among them the first instance of
    some warp of either launch; the statistics equal a run of the clean seeds alone."""
    N, I = 7, 96 * 8
    seeds = np.arange(100, 100 + I, dtype=np.uint64)
    free = BatchSimulator(seeds, N, DELAY, commit_times=True)
    cap = int(np.median(free.loop_until(600).counters[:, 8]))
    free.close()
    set_of = np.arange(I) // 96 if sweep else np.zeros(I, np.int64)
    groups = int(set_of.max()) + 1
    kw = dict(sets=[SETS[0]] * groups, set_of=set_of) if sweep else {}
    sim, res = run(seeds, N, 600, queue_cap=cap, **kw)
    try:
        bad = (res.status & np.uint32(_lib.ST_ERROR_MASK)) != 0
        assert 0 < bad.sum() < I
        assert bad[::32].any() and bad[::128 // lanes(N)].any()  # (lane 0 of a per-sample warp; the first group of a threshold block)
        got = check_both(sim, res, set_of, groups, [1, 5], {})
        clean_seeds = seeds[~bad]
        ckw = dict(sets=[SETS[0]] * groups, set_of=set_of[~bad]) if sweep else {}
        csim, cres = run(clean_seeds, N, 600, **ckw)
        try:
            assert not (cres.status & np.uint32(_lib.ST_ERROR_MASK)).any()
            np.testing.assert_array_equal(cres.commit_counts, res.commit_counts[~bad])
            want_excluded = np.bincount(set_of[bad], minlength=groups)
            for w in (1, 5):
                clean = cres.block_latency_stats(w)
                np.testing.assert_array_equal(got[w].excluded, want_excluded)
                for f in ("instances", "samples", "sum", "min", "max", "unreached"):
                    np.testing.assert_array_equal(getattr(got[w], f), getattr(clean, f), err_msg=f)
            a, b = res.latency_stats(), cres.latency_stats()
            for f in ("instances", "samples", "sum", "min", "max", "hist"):
                np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)
        finally:
            csim.close()
    finally:
        sim.close()


def merge(stats, point_of, points):
    """Per-group statistics merged into `points` groups on the host: sums and counts add, min and max (-1: empty) combine."""
    out = {}
    for f in ("instances", "excluded", "samples", "sum", "unreached"):
        if hasattr(stats, f):
            out[f] = np.zeros(points, np.uint64)
            np.add.at(out[f], point_of, getattr(stats, f))
    lo = np.full(points, INT64_MAX, np.int64)
    np.minimum.at(lo, point_of, np.where(stats.samples > 0, stats.min, INT64_MAX))
    out["min"] = np.where(out["samples"] > 0, lo, -1)
    out["max"] = np.full(points, -1, np.int64)
    np.maximum.at(out["max"], point_of, stats.max)
    out["hist"] = np.zeros((points, stats.hist.shape[1]), np.uint64)
    np.add.at(out["hist"], point_of, stats.hist)
    return out


def assert_merged(stats, merged, msg):
    for f, v in merged.items():
        np.testing.assert_array_equal(getattr(stats, f), v, err_msg="%s %s" % (msg, f))


def test_merge_identity():
    """A grid's one-instance-per-group statistics merged per point equal the grid's own; a plain handle's equal the merge of the
    same seeds split over a random grouping."""
    k = 64
    grid_sim = SweepSimulator.grid(k, [s.network_delay for s in SETS[:2]], [NodeConfig(), NodeConfig(delta=30)], num_nodes=5,
                                   commit_times=True)
    grid = grid_sim.loop_until(500, strict=False)
    point_of, points = grid_sim.set_of_instance.astype(np.int64), len(grid_sim.param_sets)
    one_sim = SweepSimulator(grid_sim.seeds, 5, [grid_sim.param_sets[p] for p in point_of], np.arange(len(point_of)), commit_times=True)
    one = one_sim.loop_until(500, strict=False)
    try:
        spec = dict(num_bins=40, bin_width=2, proposed_from=100)
        assert_merged(grid.latency_stats(**spec), merge(one.latency_stats(**spec), point_of, points), "per-sample grid")
        for w in (1, 3, 4, 5):
            assert_merged(grid.block_latency_stats(w, **spec), merge(one.block_latency_stats(w, **spec), point_of, points), "grid W=%d" % w)
    finally:
        grid_sim.close()
        one_sim.close()
    seeds = np.arange(2000, 2000 + 1025, dtype=np.uint64)
    plain_sim, plain = run(seeds, 9, 400)
    group_of = np.random.default_rng(5).integers(0, 37, len(seeds))
    split_sim, split = run(seeds, 9, 400, [SETS[0]] * 37, group_of)
    try:
        zero = np.zeros(37, np.int64)
        assert_merged(plain.latency_stats(), merge(split.latency_stats(), zero, 1), "per-sample split")
        for w in (1, 4, 7, 9):
            assert_merged(plain.block_latency_stats(w), merge(split.block_latency_stats(w), zero, 1), "split W=%d" % w)
    finally:
        plain_sim.close()
        split_sim.close()


@pytest.fixture(scope="module")
def probe():
    return BlockThresholdProbe()


@pytest.fixture(scope="module")
def blk():
    return BlockLatencyHarness()


@pytest.mark.parametrize("N", range(1, 65))
def test_lane_form_on_synthetic_tables(probe, blk, N):
    """The device function the threshold overload runs, at every N, against block_threshold_time on the host and numpy."""
    rng = np.random.default_rng(1000 + N)
    ties = zero_first = False
    for label, weights, cc, times, W in synthetic_cases(N, rng):
        want = numpy_threshold_times(cc, times, weights, W)
        np.testing.assert_array_equal(blk.threshold_times(cc, times, weights, W), want, err_msg="host " + label)
        np.testing.assert_array_equal(probe.threshold_times(cc, times, weights, W), want, err_msg="device " + label)
        ties |= has_ties(np.where(cc[:, :, None] > np.arange(times.shape[2]), times[:, :N, :].astype(np.int64), -1))
        zero_first |= zero_weight_first(cc, times, weights)
    assert (ties and zero_first) or N == 1
