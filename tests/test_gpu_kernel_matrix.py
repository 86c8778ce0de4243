"""Every event-loop kernel of the library on the GPU, one case per kernel-matrix entry (tests/kernel_matrix.py): the handle
runs the entry's kernel, no instance ends with an error bit, and the oracle agrees bit for bit on commit counts, state keys,
counters, the epoch-change bit and the commit logs of the instances it checks.  Where the oracle checks a sample of a large
batch, the whole batch is compared with the same seeds through another instantiation (results depend on the seed alone).
Recording, resumable, true-data-sync and commit-times kernels are also checked on what only they produce; on the commit-times
twins that includes both latency read-outs, so every lane-group width of the block-latency reduction (N = 1 .. 64) runs here."""
import numpy as np
import pytest

from librabft_simulator_b200 import SweepSimulator, _lib
from tests import fault_support, sweep_support
from tests.block_latency_support import assert_same_block_stats, numpy_block_stats, thresholds
from tests.ct_support import CtHarness
from tests.kernel_matrix import CT, MATRIX, REC, RES, TDS, flag_off
from tests.latency_support import numpy_stats
from tests.support import Result, assert_same
from tests.test_gpu_parity import make_sim

pytestmark = pytest.mark.gpu
EPOCH_CHANGE = np.uint32(_lib.ST_EPOCH_CHANGE)
DELAY_NEAR_INT = np.uint32(_lib.ST_DELAY_NEAR_INT)  # (an advisory bit of the device's own; the oracle has no such bit)


@pytest.fixture(scope="module")
def ct():
    return CtHarness()


def handle(e):
    """The entry's handle (not yet created): a BatchSimulator, or a SweepSimulator over its sets."""
    kw = dict(e.kw)
    flags = kw.pop("flags", 0)
    modes = dict(record_round_switches=bool(flags & REC), resumable=bool(flags & RES), true_data_sync=bool(flags & TDS),
                 commit_times=bool(flags & CT))
    if e.kind == "plain":
        return make_sim(e.seeds, e.N, **kw, **modes)
    return SweepSimulator(e.seeds, e.N, e.sets, e.set_of, **kw, **modes)


def oracle_kw(e, instance=None):
    """The oracle's keywords for the entry (for one instance of a sweep: with its set's delay, NodeConfig and faults)."""
    kw = dict(e.kw)
    kw["flags"] = kw.get("flags", 0) & TDS  # (the modes are the device's; the data-sync variant is the oracle's too)
    if instance is not None and e.kind != "plain":
        ps = e.sets[e.set_of[instance]]
        kw.update(sweep_support.set_kwargs(ps))
        if e.kind == "faults":
            kw.update(fault_support.fault_kwargs(ps.faults, e.N))
    return kw


def oracle_run(oracle, e, idx):
    seeds = e.seeds[idx]
    if e.kind == "plain":
        return oracle.run(seeds, e.N, e.max_clock, **oracle_kw(e))
    shared = {k: v for k, v in e.kw.items() if k != "flags"}
    per_set = sweep_support.oracle_per_set if e.kind == "sweep" else fault_support.oracle_per_set
    return per_set(oracle, seeds, e.N, e.max_clock, e.sets, e.set_of[idx], **shared)


def rows_of(res, idx):
    out = Result(len(idx), res.commit_counts.shape[1])
    out.commit_counts, out.last_states = res.commit_counts[idx], res.last_committed_states[idx]
    out.counters, out.status = res.counters[idx], res.status[idx]
    return out


def assert_outputs_equal(a, b, what):
    for f in ("commit_counts", "last_committed_states", "status"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg="%s: %s" % (what, f))
    np.testing.assert_array_equal(a.counters[:, :8], b.counters[:, :8], err_msg="%s: counters" % what)
    np.testing.assert_array_equal(a.counters[:, 9], b.counters[:, 9], err_msg="%s: scheduled notifications" % what)


def run(e, monkeypatch, force):
    if force is None:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    else:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", force)
    sim = handle(e)
    return sim, sim.loop_until(e.max_clock)


@pytest.mark.parametrize("name", sorted(MATRIX))
def test_kernel_matches_the_oracle(oracle, ct, monkeypatch, name):
    e = MATRIX[name]
    sim, res = run(e, monkeypatch, e.force)
    try:
        assert sim.kernel_info() == name
        assert not (res.status & np.uint32(_lib.ST_ERROR_MASK)).any(), np.unique(res.status)
        idx = e.oracle_instances()
        ref = oracle_run(oracle, e, idx)
        assert_same(ref, rows_of(res, idx), name)
        # (the oracle marks a run in which a data-sync response delivered records with LBFT_ST_INVARIANT: the reference never
        # does that, and the true-data-sync variant is built to; the device flags nothing there)
        want = ref.status & ~(np.uint32(_lib.ST_INVARIANT) if e.flags & TDS else np.uint32(0))
        np.testing.assert_array_equal(res.status[idx] & ~DELAY_NEAR_INT, want, err_msg="status")
        # the checked instances commit: a check of zero commits and empty logs would pass whatever the commit path does
        assert ref.commit_counts.max() >= 3 and (ref.commit_counts.max(axis=1) > 0).mean() >= 0.5, ref.commit_counts.max(axis=1)
        if "commands_per_epoch" in e.kw:
            check_epochs(e, ref)
        check_commit_logs(oracle, e, sim, res, idx)
        if len(idx) < e.I:
            check_whole_batch(e, monkeypatch, res)
        if e.flags & REC:
            for i in idx:
                assert sim.round_switches(int(i)) == oracle.round_switches(e.seeds, e.N, int(i), e.max_clock, **dict(oracle_kw(e), flags=REC))
        if e.flags & RES:
            check_stops_and_snapshot(oracle, e, sim, idx)
        if e.flags & CT:
            check_commit_times(ct, e, monkeypatch, res, idx)
    finally:
        sim.close()


def check_epochs(e, ref):
    """A lone author crosses at least two epoch boundaries; a committee stalls at its first (DESIGN §9), which some checked
    instance reaches (the status parity above pins the device's epoch-change bit to the oracle's)."""
    if e.N == 1:
        assert ref.commit_counts.max() > 2 * e.kw["commands_per_epoch"], "no checked instance crossed two epoch boundaries"
    assert (ref.status & EPOCH_CHANGE).any(), "no checked instance reached an epoch change"


def check_commit_logs(oracle, e, sim, res, idx):
    """The bulk commit logs: their lengths are the commit counts; every node's log of (up to 64) sampled instances hashes to the
    node's state key (the oracle's SipHash of the log); and against the oracle's commit_log row for row (which re-runs the
    instance once per node): one node of every sampled instance, rotating over the committee, and the first and last node of the
    first and last sampled instance."""
    rows, lens = res.commit_logs()
    np.testing.assert_array_equal(lens, res.commit_counts)
    as_list = lambda i, n: [(int(r["proposer"]), int(r["index"]), int(r["time"])) for r in rows[i, :lens[i, n]]]  # noqa: E731
    for i in np.unique(np.concatenate([idx[:32], idx[-32:]])):
        for n in range(e.N):
            assert oracle.state_key(as_list(i, n)) == res.last_committed_states[i, n], (i, n)
    pairs = {(int(i), int(i) % e.N) for i in idx} | {(int(i), n) for i in (idx[0], idx[-1]) for n in (0, e.N - 1)}
    for i, n in sorted(pairs):
        want = oracle.commit_log(e.seeds[i:i + 1], e.N, 0, n, e.max_clock, **oracle_kw(e, i))
        assert as_list(i, n) == want, (i, n)


def check_whole_batch(e, monkeypatch, res):
    """Every instance, through another instantiation: the full-tile thread kernel, or (for that one) the wide kernel."""
    thread32 = "event_loop_kernel" in e.name and e.name.endswith(",32>")
    other, got = run(e, monkeypatch, "wide" if thread32 else "thread")
    try:
        assert other.kernel_info() != e.name
        assert_outputs_equal(got, res, "%s against %s" % (e.name, other.kernel_info()))
    finally:
        other.close()


def check_stops_and_snapshot(oracle, e, sim, idx):
    """A stop schedule with a repeated stop against the staged oracle at every stop, then a snapshot taken after the first stop
    and loaded into a second handle, which continues to the same results."""
    mc = e.max_clock
    stops = [mc // 3, mc // 3, 2 * mc // 3, mc]
    sim.set_seeds(e.seeds)
    for k, stop in enumerate(stops, 1):
        got = sim.run_until(stop)
        if k == 1:
            snap = sim.snapshot()
        ref = oracle.run_staged(e.seeds[idx], e.N, stops[:k], mc, **oracle_kw(e))
        assert_same(ref, rows_of(got, idx), "after stops %s" % stops[:k])
    second = handle(e)
    try:
        second.create(mc)
        second.restore(snap)
        for stop in stops[1:]:
            cont = second.run_until(stop)
        assert_outputs_equal(cont, got, "restored handle")
    finally:
        second.close()


def check_commit_times(ct, e, monkeypatch, res, idx):
    """Commit times against the oracle observed event by event; the per-sample and block latency statistics against numpy over
    the handle's own commit times (a window and an overflowing last bin); every other output as the flag-off kernel's on the
    same seeds."""
    off_entry = flag_off(e)
    off, off_res = run(off_entry, monkeypatch, off_entry.force)
    try:
        assert_outputs_equal(off_res, res, "%s against %s" % (e.name, off.kernel_info()))
    finally:
        off.close()
    committed, proposed = res.commit_times()
    cap = committed.shape[2]
    groups = e.set_of[idx] if e.sets else np.zeros(len(idx), np.int64)
    for g in np.unique(groups):
        sub = idx[groups == g]
        oc, op, counts = ct.oracle(e.seeds[sub], e.N, e.max_clock, cap=cap, **oracle_kw(e, int(sub[0])))
        np.testing.assert_array_equal(counts, res.commit_counts[sub])
        np.testing.assert_array_equal(oc, committed[sub])
        np.testing.assert_array_equal(op, proposed[sub])
    spec = dict(num_bins=8, bin_width=1, proposed_from=e.max_clock // 4, proposed_until=3 * e.max_clock // 4)
    group_of = e.set_of if e.sets else np.zeros(e.I, np.int64)
    ngroups = len(e.sets) or 1
    got = res.latency_stats(**spec)
    want = numpy_stats(committed, proposed, res.status, group_of, ngroups, **spec)
    for f in ("instances", "excluded", "samples", "sum", "min", "max", "hist"):
        np.testing.assert_array_equal(getattr(got, f), getattr(want, f), err_msg=f)
    assert got.samples.sum() > 0, "no commit latency in the window"
    assert got.hist[:, -1].sum() > 0, "no latency overflowed the last bin"
    check_block_latency(e, res, committed, proposed, group_of, ngroups, spec)


def check_block_latency(e, res, committed, proposed, group_of, ngroups, spec):
    """Block latency at the named thresholds, one in between and total - 1, field by field against numpy over the same commit
    times, with the invariants across thresholds; on a single-group entry also with 8 193 bins (the global histogram)."""
    weights = np.asarray(e.kw.get("voting_rights", [1] * e.N), np.int64)
    total = int(weights.sum())
    ws = sorted(set(thresholds(total)) | ({total - 1} if total > 1 else set()))
    stats = {}
    for w in ws:
        got = res.block_latency_stats(w, **spec)
        want = numpy_block_stats(committed, proposed, res.status, group_of, ngroups, weights, w, **spec)
        assert_same_block_stats(got, want, "W=%d" % w)
        stats[w] = got
    blocks = stats[ws[0]].samples + stats[ws[0]].unreached
    for a, b in zip(ws, ws[1:]):
        np.testing.assert_array_equal(stats[b].samples + stats[b].unreached, blocks, err_msg="blocks at W=%d" % b)
        assert (stats[b].samples <= stats[a].samples).all(), (a, b)
    assert ws[0] == 1 and (stats[1].unreached == 0).all()
    assert blocks.sum() > 0, "no block in the window"
    if ngroups == 1:
        wide = dict(spec, num_bins=8193)
        for w in (1, ws[len(ws) // 2], total):
            want = numpy_block_stats(committed, proposed, res.status, group_of, ngroups, weights, w, **wide)
            assert_same_block_stats(res.block_latency_stats(w, **wide), want, "8 193 bins, W=%d" % w)
