"""Commit times (LBFT_FLAG_COMMIT_TIMES) on the GPU, through both kernel families: the BASELINE shapes and a small shared-memory
wide batch against the oracle observed event time by event time, with every other output identical to a flag-off handle; a
65 536-instance sweep of 256 sets against plain commit-times handles; re-seeded and streamed handles against fresh ones; the
busy-handle and missing-flag errors; logs longer than cap."""
import numpy as np
import pytest

from bench import CONFIGS, make_sim
from librabft_simulator_b200 import BatchSimulator, RandomDelay, Simulator, SweepSimulator, _lib
from tests.ct_support import CtHarness
from tests.test_commit_times import ct_name
from tests.test_gpu_sweep import grid_256

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ct():
    return CtHarness()


def run_pair(seeds, nodes, max_clock, **kw):
    """The same batch on a flag-off and a commit-times handle: (off, on, simulators)."""
    off_sim, on_sim = make_sim(seeds, nodes, **kw), make_sim(seeds, nodes, commit_times=True, **kw)
    off, on = off_sim.loop_until(max_clock, strict=False), on_sim.loop_until(max_clock, strict=False)
    return off, on, off_sim, on_sim


def assert_other_outputs_identical(off, on, off_sim, on_sim):
    for f in ("commit_counts", "last_committed_states", "active_rounds", "status", "counters"):
        np.testing.assert_array_equal(getattr(off, f), getattr(on, f), err_msg=f)
    assert on_sim.kernel_info() == ct_name(off_sim.kernel_info())
    b_off, w_off = off_sim.memory_info()
    b_on, w_on = on_sim.memory_info()
    assert w_on == w_off
    I, N = on_sim.num_instances, on_sim.num_nodes
    assert (b_on - b_off) % (I * (N + 1) * 4) == 0 and b_on > b_off  # the [I][N + 1][round_cap] int32 table


# (BASELINE config, instance stride of the subset checked against the oracle); every instance is also checked against the host
# core (the CT core through the same host setup, so the same layout and compile-time shape), except for config 4, whose 64-author
# instances are too slow for it
SHAPES = [(1, 1), (2, 16), (3, 512), (4, 256), (5, 128)]
_HOST = {}  # config -> the host core's run; computed once for both families (its times do not depend on the layout)


@pytest.mark.parametrize("cid,stride", SHAPES, ids=["config%d" % c for c, _ in SHAPES])
def test_baseline_shapes_match_the_oracle(ct, kernel_choice, cid, stride):
    c = CONFIGS[cid]
    seeds = np.arange(c["base_seed"], c["base_seed"] + c["instances"], dtype=np.uint64)
    off, on, off_sim, on_sim = run_pair(seeds, c["nodes"], c["max_clock"], **c["kw"])
    assert_other_outputs_identical(off, on, off_sim, on_sim)
    if cid == 3 and kernel_choice == "thread":
        assert on_sim.kernel_info() == "lbft_ct_event_loop_kernel<16,2,1,32>"  # the compact-encoding twin
    committed, proposed = on.commit_times()
    cap = committed.shape[2]
    rows, lens = on.commit_logs(cap)
    np.testing.assert_array_equal(lens, on.commit_counts)
    sub = np.arange(0, len(seeds), stride)
    kw = {k: v for k, v in c["kw"].items()}
    oc, op, counts = ct.oracle(seeds[sub], c["nodes"], c["max_clock"], cap=cap, **kw)
    ok = (on.status[sub] & np.uint32(_lib.ST_ERROR_MASK)) == 0
    assert ok.all()
    np.testing.assert_array_equal(counts, on.commit_counts[sub])
    np.testing.assert_array_equal(oc, committed[sub])
    np.testing.assert_array_equal(op, proposed[sub])
    if cid != 4:
        if cid not in _HOST:
            _HOST[cid] = ct.run(seeds, c["nodes"], c["max_clock"], cap=cap, **kw)
        host = _HOST[cid]
        assert ((host.status & np.uint32(_lib.ST_ERROR_MASK)) == 0).all()
        np.testing.assert_array_equal(host.commit_counts, on.commit_counts)
        np.testing.assert_array_equal(host.committed, committed)
        np.testing.assert_array_equal(host.proposed, proposed)
    # every row: latency >= 0, -1 past each log, committed times non-decreasing
    k = np.arange(cap)
    inside = k[None, None, :] < on.commit_counts[:, :, None]
    assert ((committed >= 0) == inside).all()
    lat = on.commit_latencies(cap)
    assert (lat[inside] >= 0).all() and (lat[~inside] == -1).all()
    assert (np.diff(np.where(inside, committed, np.iinfo(np.int64).max), axis=2) >= 0).all()
    off_sim.close()
    on_sim.close()


def test_small_shared_memory_wide_batch(ct, monkeypatch):
    monkeypatch.setenv("LBFT_FORCE_KERNEL", "wide")
    seeds = np.arange(5000, 5064, dtype=np.uint64)
    off, on, off_sim, on_sim = run_pair(seeds, 4, 1000)
    assert on_sim.kernel_info() == "lbft_ct_wide_kernel<16,2,true,32,0>"
    assert_other_outputs_identical(off, on, off_sim, on_sim)
    committed, proposed = on.commit_times(64)
    oc, op, _ = ct.oracle(seeds, 4, 1000, cap=64)
    np.testing.assert_array_equal(oc, committed)
    np.testing.assert_array_equal(op, proposed)


def test_sweep_of_256_sets_equals_plain_commit_time_handles():
    delays, configs = grid_256()
    seeds = np.arange(9000, 9256, dtype=np.uint64)
    sim = SweepSimulator.grid(seeds, delays, configs, num_nodes=4, commit_times=True)
    res = sim.loop_until(1000, strict=False)
    assert sim.kernel_info() == "lbft_ct_sweep_event_loop_kernel<16,2,32>"
    off = SweepSimulator.grid(seeds, delays, configs, num_nodes=4).loop_until(1000, strict=False)
    for f in ("commit_counts", "last_committed_states", "status", "counters"):
        np.testing.assert_array_equal(getattr(off, f), getattr(res, f), err_msg=f)
    committed, proposed = res.commit_times(96)
    for p in (0, 37, 128, 201, 255):
        ps = sim.param_sets[p]
        rows = slice(p * 256, (p + 1) * 256)
        plain = BatchSimulator(seeds, 4, ps.network_delay, ps.node_config, commit_times=True)
        r = plain.loop_until(1000, strict=False)
        ok = ((r.status | res.status[rows]) & np.uint32(_lib.ST_ERROR_MASK)) == 0
        assert ok.mean() > 0.99
        c, q = r.commit_times(96)
        np.testing.assert_array_equal(c[ok], committed[rows][ok], err_msg="set %d" % p)
        np.testing.assert_array_equal(q[ok], proposed[rows][ok], err_msg="set %d" % p)
        plain.close()
    sim.close()


def test_reseeded_and_streamed_handles_agree_with_fresh_ones(kernel_choice):
    """The commit-time table is not cleared between runs."""
    delay = RandomDelay.new(10.0, 4.0)
    batches = [np.arange(s, s + 512, dtype=np.uint64) for s in (10, 7000, 123456)]

    def fresh(seeds):
        sim = BatchSimulator(seeds, 4, delay, commit_times=True)
        r = sim.loop_until(1000)
        out = (r.commit_counts, r.last_committed_states) + r.commit_times(64)
        sim.close()
        return out

    want = [fresh(b) for b in batches]
    sim = BatchSimulator(batches[0], 4, delay, commit_times=True)
    sim.create(1000)
    for b, w in zip(batches, want):  # re-seeded
        sim.set_seeds(b)
        r = sim.run()
        for a, x in zip(w, (r.commit_counts, r.last_committed_states) + r.commit_times(64)):
            np.testing.assert_array_equal(a, x)
    results = list(sim.run_stream(batches[::-1]))  # streamed: the last result is current once the stream ends
    got = (results[-1].commit_counts, results[-1].last_committed_states) + results[-1].commit_times(64)
    for a, x in zip(want[0], got):
        np.testing.assert_array_equal(a, x)
    sim.close()


def test_busy_handle_and_missing_flag_are_state_errors():
    delay = RandomDelay.new(10.0, 4.0)
    sim = BatchSimulator(np.arange(64, dtype=np.uint64), 4, delay, commit_times=True)
    sim.loop_until(1000)
    sim.run_async()
    with pytest.raises(_lib.LbftError) as e:
        sim.commit_times(16)
    assert e.value.code == -3 and "in flight" in str(e.value)
    r = sim.wait()
    r.commit_times(16)
    for cap in (0, 65536):
        with pytest.raises(_lib.LbftError) as e:
            sim.commit_times(cap)
        assert e.value.code == -1
    sim.close()
    plain = BatchSimulator(np.arange(64, dtype=np.uint64), 4, delay)
    r = plain.loop_until(1000)
    with pytest.raises(_lib.LbftError) as e:
        r.commit_times(16)
    assert e.value.code == -3 and "LBFT_FLAG_COMMIT_TIMES" in str(e.value)
    plain.close()


def test_logs_longer_than_cap_are_cut_like_the_commit_logs():
    seeds = np.arange(300, 428, dtype=np.uint64)
    sim = BatchSimulator(seeds, 7, RandomDelay.new(10.0, 4.0), round_cap=512, commit_times=True)
    res = sim.loop_until(5000)
    assert res.commit_counts.max() > 100
    full_c, full_p = res.commit_times()
    short_c, short_p = res.commit_times(40)
    np.testing.assert_array_equal(short_c, full_c[:, :, :40])
    np.testing.assert_array_equal(short_p, full_p[:, :40])
    rows, lens = res.commit_logs(40)
    k = np.arange(40)
    np.testing.assert_array_equal(short_c >= 0, k[None, None, :] < lens[:, :, None])
    np.testing.assert_array_equal(short_p >= 0, k[None, :] < lens.max(axis=1)[:, None])
    sim.close()


def test_simulator_context_view_rows_align_with_committed_history():
    contexts = Simulator.new(52, 3, RandomDelay.new(10.0, 4.0), None, commit_times=True).loop_until(1000)
    for c in contexts:
        hist, times = c.committed_history(), c.commit_times()
        assert len(hist) == len(times) == 27
        for (cmd, t), (proposed, committed) in zip(hist, times):
            assert proposed > t and committed >= proposed
