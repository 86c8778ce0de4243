"""The capacity edges (tests/capacity_cases.py) on the GPU, one case per table entry.  Run A has generous capacities, run B
the tight capacity C derived from A.  Both run the case's kernel; in B the error bit under test is set exactly on the
instances whose peak in A exceeds C (rounds: reached C), and no other bit is; some clean instance of B uses the last entry;
every clean instance of B is bit-identical to A (commit counts, state keys, all 12 counters, status, the bulk commit logs,
and on commit-times twins the commit times); and every instance of B, flagged ones included, ends with the status and the
12 counters of the host-compiled core at the same configuration: where an overflowing instance stops does not depend on the
queue implementation.  The resumable case runs B as a stop schedule against the staged host core and through a snapshot.
In every run, an instance flagged for the queue whose queue never filled has used up its mode's creation stamps."""
import numpy as np
import pytest

from librabft_simulator_b200 import SweepSimulator, _lib
from tests import sweep_support
from tests.capacity_cases import CLEAN, EDGES, tight
from tests.kernel_matrix import CT, REC, RES
from tests.support import assert_same
from tests.test_capacity_edges import check_edge, check_stamps, effective_caps, host_run, set_force
from tests.test_gpu_parity import make_sim

pytestmark = pytest.mark.gpu
ERR = np.uint32(_lib.ST_ERROR_MASK)
DELAY_NEAR_INT = np.uint32(_lib.ST_DELAY_NEAR_INT)  # (an advisory bit of the device's own)


@pytest.fixture(scope="module")
def sweep_host():
    return sweep_support.SweepHostCore()


class Run:
    """A GPU run's results under tests.support.Result's names, read before the handle runs again."""

    def __init__(self, sim, res, queue_cap):
        self.kernel = sim.kernel_info()
        self.commit_counts, self.last_states = res.commit_counts, res.last_committed_states
        self.counters, self.status = res.counters.copy(), res.status & ~DELAY_NEAR_INT
        self.queue_cap = queue_cap
        self.rows, self.lens = res.commit_logs()
        self.times = res.commit_times() if sim.commit_times_enabled else None
        self.excluded = res.latency_stats().excluded if sim.commit_times_enabled else None


def handle(case, kw):
    kw = dict(kw)
    flags = kw.pop("flags", 0)
    modes = dict(record_round_switches=bool(flags & REC), resumable=bool(flags & RES), commit_times=bool(flags & CT))
    if case.kind == "sweep":
        return SweepSimulator(case.seeds, case.N, case.sets, case.set_of, **kw, **modes)
    return make_sim(case.seeds, case.N, **kw, **modes)


def gpu_run(hostcore, case, kw):
    sim = handle(case, kw)
    try:
        return Run(sim, sim.loop_until(case.max_clock, strict=False), effective_caps(hostcore, case, kw)["queue_cap"])
    finally:
        sim.close()


def same_logs(A, B, idx):
    for i in idx:
        np.testing.assert_array_equal(B.lens[i], A.lens[i])
        k = int(A.lens[i].max())
        np.testing.assert_array_equal(B.rows[i, :k], A.rows[i, :k], err_msg="commit log of instance %d" % i)


def same_end(host, B, what):
    """Every instance, flagged or not: status and all 12 counters as the host-compiled core computes them."""
    np.testing.assert_array_equal(B.status, host.status & ~DELAY_NEAR_INT, err_msg="status against the host core " + what)
    np.testing.assert_array_equal(B.counters, host.counters, err_msg="counters against the host core " + what)


@pytest.mark.parametrize("cid", sorted(EDGES))
def test_tight_capacity_on_the_gpu(hostcore, sweep_host, monkeypatch, cid):
    case = EDGES[cid]
    set_force(monkeypatch, case.force)
    A = gpu_run(hostcore, case, case.kw)
    assert A.kernel == case.name
    C = tight(case, A.counters)
    B = gpu_run(hostcore, case, case.tight_kw(C))
    assert B.kernel == case.name
    flagged = check_edge(case, A, B, C)
    print("%s: C = %d, %d flagged, %d clean" % (cid, C, flagged.sum(), (~flagged).sum()))
    same_logs(A, B, np.nonzero(~flagged)[0])
    if case.kind == "ct":
        for a, b in zip(A.times, B.times):
            k = min(a.shape[-1], b.shape[-1])
            np.testing.assert_array_equal(b[~flagged][..., :k], a[~flagged][..., :k], err_msg="commit times")
        assert int(np.sum(B.excluded)) == int(flagged.sum()) and int(np.sum(A.excluded)) == 0
    same_end(host_run(hostcore, sweep_host, case, case.tight_kw(C)), B, "at C = %d" % C)
    same_end(host_run(hostcore, sweep_host, case, case.kw), A, "at the generous capacities")
    for run in (A, B):
        check_stamps(case.qmode, run)
    if case.kind == "resumable":
        check_stops_and_snapshot(hostcore, case, C, B)


def check_stops_and_snapshot(hostcore, case, C, B):
    """A stop schedule over B (with a repeated stop, and instances flagged after the first) against the staged host core at
    every stop; then a snapshot taken after the first stop, restored into a second handle, continues to the same results.
    (A stop drops the first event beyond it, as the reference's loop_until does, so a schedule is compared with the staged
    host core, not with the one-shot run; its last stop is the one-shot run when no event lies past the first stops.)"""
    mc = case.max_clock
    stops = [mc // 3, mc // 3, 2 * mc // 3, mc]
    kw = case.tight_kw(C)
    sim = handle(case, kw)
    try:
        sim.create(mc)
        for k, stop in enumerate(stops, 1):
            got = sim.run_until(stop, strict=False)
            if k == 1:
                snap = sim.snapshot()
                assert (got.status & ERR).any(), "no instance flagged after the first stop"
            ref = hostcore.run_staged(case.seeds, case.N, stops[:k], mc, **kw)
            np.testing.assert_array_equal(got.status & ~DELAY_NEAR_INT, ref.status)
            np.testing.assert_array_equal(got.counters, ref.counters)
            np.testing.assert_array_equal(got.commit_counts, ref.commit_counts)
            np.testing.assert_array_equal(got.last_committed_states, ref.last_states)
        final = (got.status.copy(), got.counters.copy(), got.commit_counts.copy(), got.last_committed_states.copy())
    finally:
        sim.close()
    second = handle(case, kw)
    try:
        second.create(mc)
        second.restore(snap)
        for stop in stops[1:]:
            cont = second.run_until(stop, strict=False)
        for a, b in zip(final, (cont.status, cont.counters, cont.commit_counts, cont.last_committed_states)):
            np.testing.assert_array_equal(b, a)
    finally:
        second.close()
    assert ((B.status & ERR) != 0).any()


@pytest.mark.parametrize("cid", sorted(CLEAN))
def test_floor_and_horizon_on_the_gpu(hostcore, oracle, monkeypatch, cid):
    case = CLEAN[cid]
    set_force(monkeypatch, case.force)
    run = gpu_run(hostcore, case, case.kw)
    assert run.kernel == case.name
    assert not (run.status & ERR).any(), np.unique(run.status)
    assert_same(oracle.run(case.seeds, case.N, case.max_clock, **case.kw), run, case.id)
    same_end(hostcore.run(case.seeds, case.N, case.max_clock, **case.kw), run, case.id)
    check_stamps(case.qmode, run)
