"""The compact node / notification encoding of the bench kernel (FX_DEFAULT4 on the thread-per-instance kernel) on the H100,
at the configurations of tests/test_packed_encoding.py that drive its byte-wide fields to their limits: every instance
against the host-compiled compact core, the instances without an error bit against the oracle, and the commit logs
themselves — long ones included — for a sample."""
from types import SimpleNamespace

import numpy as np
import pytest

from tests.support import assert_same
from tests.test_gpu_parity import make_sim
from tests.test_packed_encoding import CONFIGS, subset

pytestmark = pytest.mark.gpu

KERNEL = "lbft_event_loop_kernel<16,2,1,false,false,false,false,32>"  # <NMAX, QMODE, FX_DEFAULT4, ..., 32 instances per tile>


@pytest.fixture
def thread_kernel(monkeypatch):
    # batches of <= 4 096 four-author instances go to the warp-per-instance kernel unless asked otherwise
    monkeypatch.setenv("LBFT_FORCE_KERNEL", "thread")


def run_packed(seeds, name, strict=False):
    max_clock, kw = CONFIGS[name]
    sim = make_sim(seeds, 4, **dict(kw))
    res = sim.loop_until(max_clock, strict=strict)
    assert sim.kernel_info() == KERNEL
    res.counters  # (read now: valid until the handle runs again)
    return sim, res


def check_against_host(oracle, hostcore, seeds, name, res):
    """Every instance against the host-compiled compact core; those without an error bit against the oracle.  Returns the
    mask of the latter and the oracle's results."""
    from librabft_simulator_b200._lib import ST_ERROR_MASK, ST_ROUND_OVERFLOW
    max_clock, kw = CONFIGS[name]
    h = hostcore.run(seeds, 4, max_clock, **kw)
    np.testing.assert_array_equal(res.commit_counts, h.commit_counts)
    np.testing.assert_array_equal(res.last_committed_states, h.last_states)
    np.testing.assert_array_equal(res.counters, h.counters)
    np.testing.assert_array_equal(res.status, h.status)
    np.testing.assert_array_equal(res.active_rounds, h.counters[:, 6])
    o = oracle.run(seeds, 4, max_clock, **kw)
    ok = (res.status & ST_ERROR_MASK) == 0
    g = SimpleNamespace(commit_counts=res.commit_counts[ok], last_states=res.last_committed_states[ok], counters=res.counters[ok])
    assert_same(subset(o, ok), g, name)
    if name != "queue_overflow":
        # every instance whose reference reaches round 128 overflows; one that overflows got at least to round 127
        # (tests/test_packed_encoding.py checks the exact condition on the decoded node states)
        overflow = (res.status & ST_ROUND_OVERFLOW) != 0
        assert overflow[o.counters[:, 6] >= 128].all() and (o.counters[overflow, 6] >= 127).all()
    return ok, o


def check_commit_logs(oracle, sim, res, seeds, name, ok, count=4):
    """The logs of the completed instances with the most commits, and of the first and last one, through lbft_commit_log
    and lbft_commit_logs (cap 128) against the oracle's.  Returns the longest log compared."""
    max_clock, kw = CONFIGS[name]
    idx = np.flatnonzero(ok)
    if len(idx) == 0:
        return 0
    best = idx[np.argsort(-res.commit_counts[idx].max(axis=1), kind="stable")[:count]]
    sample = sorted(set(best.tolist()) | {int(idx[0]), int(idx[-1])})
    rows, lens = sim.commit_logs(128)
    longest = 0
    for inst in sample:
        for node in range(4):
            want = oracle.commit_log(seeds, 4, inst, node, max_clock, **kw)
            assert sim.commit_log(inst, node) == want, (name, inst, node)
            assert lens[inst, node] == len(want)
            got = [(int(r["proposer"]), int(r["index"]), int(r["time"])) for r in rows[inst, :lens[inst, node]]]
            assert got == want, (name, inst, node)
            longest = max(longest, len(want))
    return longest


@pytest.mark.parametrize("name", list(CONFIGS))
def test_edge_configuration_on_gpu(oracle, hostcore, thread_kernel, name):
    seeds = np.arange(1001, 1001 + 320, dtype=np.uint64)
    sim, res = run_packed(seeds, name)
    ok, _ = check_against_host(oracle, hostcore, seeds, name, res)
    longest = check_commit_logs(oracle, sim, res, seeds, name, ok)
    if name in ("horizon_3000", "fast_delays", "commit_tracker"):
        assert longest > 100


def test_boundary_configuration_8192_instances(oracle, hostcore, thread_kernel):
    seeds = np.arange(1, 8193, dtype=np.uint64)
    sim, res = run_packed(seeds, "weighted_boundary")
    ok, o = check_against_host(oracle, hostcore, seeds, "weighted_boundary", res)
    assert 0 < ok.sum() < len(ok) and o.counters[ok, 6].max() == 127
    assert check_commit_logs(oracle, sim, res, seeds, "weighted_boundary", ok) > 100


@pytest.mark.parametrize("name", ["round_overflow_4000", "queue_overflow", "weighted_boundary"])
def test_strict_mode_reports_the_overflow(hostcore, thread_kernel, name):
    from librabft_simulator_b200 import _lib
    seeds = np.arange(1, 65, dtype=np.uint64)
    with pytest.raises(_lib.LbftError) as e:
        run_packed(seeds, name, strict=True)
    assert e.value.code == _lib.LBFT_ERR_CAPACITY
    sim, res = run_packed(seeds, name)
    failing = (res.status & _lib.ST_ERROR_MASK) != 0
    assert failing.any()
    max_clock, kw = CONFIGS[name]
    np.testing.assert_array_equal(res.status, hostcore.run(seeds, 4, max_clock, **kw).status)
    if name != "weighted_boundary":
        assert failing.all()


@pytest.mark.parametrize("count", [1, 33, 4097])
def test_ragged_batch_sizes(oracle, hostcore, thread_kernel, count):
    seeds = np.arange(7001, 7001 + count, dtype=np.uint64)
    sim, res = run_packed(seeds, "weighted_boundary")
    check_against_host(oracle, hostcore, seeds, "weighted_boundary", res)


def summary(res):
    return (res.commit_counts.copy(), res.last_committed_states.copy(), res.counters.copy(), res.status.copy(),
            res.active_rounds.copy())


def assert_same_summary(a, b, what):
    for x, y, field in zip(a, b, ("commit counts", "last states", "counters", "status", "active rounds")):
        np.testing.assert_array_equal(x, y, err_msg="%s: %s" % (what, field))


def test_reused_handle_reads_no_stale_word(thread_kernel):
    """init clears only the words the compact encoding uses: a handle run again with other seeds must compute exactly what a
    fresh handle computes, so no word left over from the earlier batch is ever read."""
    name = "weighted_boundary"
    max_clock, kw = CONFIGS[name]
    a = np.arange(1, 257, dtype=np.uint64)
    b = np.arange(9001, 9257, dtype=np.uint64)
    fresh_sim, fresh = run_packed(b, name)
    want = summary(fresh)
    want_rows, want_lens = fresh_sim.commit_logs(128)
    _, fresh_a = run_packed(a, name)
    want_a = summary(fresh_a)

    sim, res_a = run_packed(a, name)
    sim.set_seeds(b)
    res_b = sim.run(strict=False)
    assert_same_summary(summary(res_b), want, "re-seeded handle")
    rows, lens = sim.commit_logs(128)
    np.testing.assert_array_equal(lens, want_lens)
    np.testing.assert_array_equal(rows, want_rows)  # (rows beyond an instance's longest log are zero)

    got = []
    for res in sim.run_stream([a, b, a, b], strict=False):
        got.append(summary(res))
    for k, g in enumerate(got):
        assert_same_summary(g, want if k % 2 else want_a, "run_stream batch %d" % k)
