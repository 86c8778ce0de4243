"""Commit times (LBFT_FLAG_COMMIT_TIMES) without a GPU: the CT core compiled for the host, through the product's host setup and
read-out, against the oracle observed event time by event time; every other output against the flag-off core; the kernel
picks, the refusals and the bindings."""
import os
import re

import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, NodeConfig, RandomDelay, Simulator, SweepSimulator, _lib
from tests.ct_support import CtHarness
from tests.support import FLAG_RESUMABLE, FLAG_ROUND_SWITCHES, FLAG_TRUE_DATA_SYNC, assert_same
from tests.sweep_support import KERNEL_CASES, SETS, SweepHostCore, set_kwargs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CT = _lib.FLAG_COMMIT_TIMES
W7 = [1, 2, 3, 1, 2, 3, 1]
SILENT7 = [0, 0, 0, 0, 0, 0, 1]

# (name, first seed, instances, nodes, max_clock, config keywords); "thread": the layout of the thread-per-instance family
# (LBFT_FORCE_KERNEL), which a batch this small would not get — the seven-author compile-time layout is one of those
CASES = [
    ("n3", 1, 64, 3, 1000, {}),
    ("n4_default4", 100, 96, 4, 1000, {}),                                   # FX_DEFAULT4: the compact encoding, queue mode 2
    ("n4_uniform", 200, 64, 4, 1000, dict(delay_kind=1, delay_lo=5, delay_hi=15)),
    ("n5_scan", 300, 24, 5, 10000, {}),                                      # queue mode 1
    ("n7_part7", 400, 48, 7, 1000, dict(partition_windows=4, partition_max_len=150, thread=True)),  # FX_PART7, queue mode 3
    ("n7_weights_silent", 500, 48, 7, 1000, dict(voting_rights=W7, silent=SILENT7)),
    ("n7_heap", 600, 16, 7, 5000, dict(round_cap=512)),                      # queue mode 0, logs longer than 128 rows
    ("n40", 700, 8, 40, 600, {}),
]


@pytest.fixture(scope="module")
def ct():
    return CtHarness()


def check_invariants(res, N, cap):
    """proposed - row time = the proposer's startup; latency >= 0; committed times non-decreasing in k; -1 past each log."""
    I = res.commit_counts.shape[0]
    lens = np.minimum(res.commit_counts.astype(np.int64), cap)
    k = np.arange(cap)
    inside = k[None, None, :] < lens[:, :, None]
    assert ((res.committed >= 0) == inside).all()
    longest = lens.max(axis=1)
    assert ((res.proposed >= 0) == (k[None, :] < longest[:, None])).all()
    lat = res.committed - res.proposed[:, None, :]
    assert (lat[inside] >= 0).all()
    c = np.where(inside, res.committed, np.iinfo(np.int64).max)
    assert (np.diff(c, axis=2) >= 0).all()
    return I


@pytest.mark.parametrize("name,seed0,count,nodes,max_clock,kw", CASES, ids=[c[0] for c in CASES])
def test_matches_the_oracle_and_the_flag_off_core(ct, hostcore, oracle, monkeypatch, name, seed0, count, nodes, max_clock, kw):
    kw = dict(kw)
    if kw.pop("thread", False):
        monkeypatch.setenv("LBFT_FORCE_KERNEL", "thread")
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    cap = 256
    res = ct.run(seeds, nodes, max_clock, cap=cap, **kw)
    off = hostcore.run(seeds, nodes, max_clock, **kw)
    # every other output bit for bit the flag-off run's
    for f in ("commit_counts", "last_states", "lc_round", "counters", "status"):
        assert np.array_equal(getattr(res, f), getattr(off, f)), f
    # the oracle observed per event time: the same run (its own outputs unchanged) and the same times
    committed, proposed, counts = ct.oracle(seeds, nodes, max_clock, cap=cap, **kw)
    ref = oracle.run(seeds, nodes, max_clock, **kw)
    assert np.array_equal(counts, ref.commit_counts)
    ok = (res.status & np.uint32(_lib.ST_ERROR_MASK)) == 0
    assert ok.mean() > 0.9, res.status
    assert_same(ref, res, name)
    assert np.array_equal(res.committed[ok], committed[ok]), name
    assert np.array_equal(res.proposed[ok], proposed[ok]), name
    check_invariants(res, nodes, cap)


def test_the_cases_cover_every_queue_mode_and_both_compile_time_layouts(hostcore, monkeypatch):
    modes, shapes = set(), set()
    for _, _, _, n, mc, kw in CASES:
        kw = dict(kw)
        if kw.pop("thread", False):
            monkeypatch.setenv("LBFT_FORCE_KERNEL", "thread")
        else:
            monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
        modes.add(hostcore.setup_info(n, mc, **kw)["queue_scan"])
        shapes.add(hostcore.fixed_shape(n, mc, **kw))
    assert modes == {0, 1, 2, 3}
    assert {1, 2} <= shapes  # FX_DEFAULT4, FX_PART7


def test_proposed_time_is_row_time_plus_proposer_startup(ct, oracle):
    """The cross-check that needs no oracle times: proposed[k] - committed_history()[k].time is the startup time of row k's
    proposer (simulator.rs:120-126), as the core holds it; and every node handles no event before its startup, so none of its
    commits is earlier."""
    seeds = np.arange(800, 864, dtype=np.uint64)
    for nodes, kw in ((4, {}), (7, dict(partition_windows=4, partition_max_len=150))):
        res = ct.run(seeds, nodes, 1000, cap=64, **kw)
        inside = res.committed >= 0
        assert (np.where(inside, res.committed, np.iinfo(np.int64).max) >= res.startup[:, :, None]).all()
        for i in range(0, len(seeds), 7):
            n = int(np.argmax(res.commit_counts[i]))
            log = oracle.commit_log(seeds, nodes, i, n, 1000, **kw)
            assert len(log) == res.commit_counts[i, n]  # (0 when a partition kept every node from committing)
            for k, (proposer, _, t) in enumerate(log[:64]):
                assert int(res.proposed[i, k]) - t == int(res.startup[i, proposer]), (nodes, i, k)


def test_rows_past_cap_are_cut_like_the_commit_logs(ct):
    seeds = np.arange(900, 910, dtype=np.uint64)
    full = ct.run(seeds, 7, 5000, cap=512, round_cap=512)
    short = ct.run(seeds, 7, 5000, cap=40, round_cap=512)
    assert full.commit_counts.max() > 40
    assert np.array_equal(short.committed, full.committed[:, :, :40])
    assert np.array_equal(short.proposed, full.proposed[:, :40])


def test_reseeded_handle_agrees_with_a_fresh_one(ct):
    """The commit-time table is not cleared between runs: a second run over the same table must read only its own entries."""
    seeds = np.arange(1000, 1064, dtype=np.uint64)
    for nodes, kw in ((4, {}), (7, dict(partition_windows=4, partition_max_len=150)), (5, {})):
        fresh = ct.run(seeds, nodes, 1000, **kw)
        reused = ct.run(seeds, nodes, 1000, first_seeds=seeds[::-1] + np.uint64(5000), **kw)
        for f in ("commit_counts", "last_states", "counters", "status", "committed", "proposed"):
            assert np.array_equal(getattr(fresh, f), getattr(reused, f)), (nodes, f)


def test_sweep_matches_the_oracle_per_set(ct, oracle):
    for nodes, seed0 in ((4, 2000), (7, 2100)):
        seeds = np.arange(seed0, seed0 + 48, dtype=np.uint64)
        set_of = np.arange(48) % len(SETS)
        res = ct.run_sweep(seeds, nodes, 1000, SETS, set_of, cap=128, round_cap=256)
        off = SweepHostCore().run(seeds, nodes, 1000, SETS, set_of, round_cap=256)
        for f in ("commit_counts", "last_states", "lc_round", "counters", "status"):
            assert np.array_equal(getattr(res, f), getattr(off, f)), f
        for s, ps in enumerate(SETS):
            idx = np.nonzero(set_of == s)[0]
            kw = set_kwargs(ps)
            committed, proposed, counts = ct.oracle(seeds[idx], nodes, 1000, cap=128, round_cap=256, **kw)
            assert np.array_equal(counts, res.commit_counts[idx])
            assert np.array_equal(committed, res.committed[idx]), (nodes, s)
            assert np.array_equal(proposed, res.proposed[idx]), (nodes, s)
        check_invariants(res, nodes, 128)


def ct_name(name):
    """The commit-times twin of a flag-off kernel name."""
    m = re.match(r"lbft_event_loop_kernel<(\d+),(\d+),(\d+),false,false,false,false,(\d+)>$", name)
    if m:
        return "lbft_ct_event_loop_kernel<%s,%s,%s,%s>" % m.groups()
    m = re.match(r"lbft_wide_kernel<(\d+),(\d+),(true|false),(\d+),false,(\d+)>$", name)
    if m:
        return "lbft_ct_wide_kernel<%s,%s,%s,%s,%s>" % m.groups()
    m = re.match(r"lbft_sweep_(event_loop|wide)_kernel<(.*)>$", name)
    assert m, name
    return "lbft_ct_sweep_%s_kernel<%s>" % m.groups()


@pytest.mark.parametrize("force", [None, "thread", "wide"])
def test_kernel_picks_are_the_twins_of_the_flag_off_picks(hostcore, monkeypatch, force):
    if force:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", force)
    else:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    sweep = SweepHostCore()
    seen = set()
    for name, I, N, kw in KERNEL_CASES:
        kw = dict(kw)
        mc = kw.pop("max_clock", 1000)
        seeds = np.arange(I, dtype=np.uint64)
        off = hostcore.kernel_info(seeds, N, mc, **kw)
        on = hostcore.kernel_info(seeds, N, mc, flags=CT, **kw)
        assert on == ct_name(off), name
        assert hostcore.setup_info(N, mc, flags=CT, **kw) == hostcore.setup_info(N, mc, **kw), name
        set_of = np.zeros(I, np.uint32)
        s_off = sweep.kernel_info(seeds, N, mc, SETS[:1], set_of, **kw)
        s_on = sweep.kernel_info(seeds, N, mc, SETS[:1], set_of, flags=CT, **kw)
        assert s_on == ct_name(s_off), name
        seen |= {on, s_on}
    if force is None:  # the bench shape gets the twin of the compact-encoding kernel
        assert "lbft_ct_event_loop_kernel<16,2,1,32>" in seen


def test_refusals(hostcore):
    for flags in (CT | FLAG_ROUND_SWITCHES, CT | FLAG_RESUMABLE, CT | FLAG_TRUE_DATA_SYNC):
        with pytest.raises(RuntimeError, match="commit times.*recording, resumable or true data-sync"):
            hostcore.setup_info(4, 1000, flags=flags)
    with pytest.raises(RuntimeError, match=r"commit times.*commands_per_epoch >= round_cap"):
        hostcore.setup_info(4, 1000, flags=CT, commands_per_epoch=20)
    hostcore.setup_info(4, 1000, commands_per_epoch=20)  # (epochs without the flag stay accepted)
    for flags in (8, 8 | CT):
        with pytest.raises(RuntimeError, match="unknown bits in flags"):
            hostcore.setup_info(4, 1000, flags=flags)
    sweep, seeds, set_of = SweepHostCore(), np.arange(8, dtype=np.uint64), np.zeros(8, np.uint32)
    for flags in (CT | FLAG_ROUND_SWITCHES, CT | FLAG_RESUMABLE, CT | 8):
        with pytest.raises(RuntimeError, match="sweep handles take no flags"):
            sweep.kernel_info(seeds, 4, 1000, SETS[:1], set_of, flags=flags)


def test_getter_without_the_flag_is_a_state_error(ct):
    with pytest.raises(RuntimeError, match="^-3: commit times were not recorded"):
        ct.run(np.arange(4, dtype=np.uint64), 4, 1000, flags=0)


def test_c_abi_checks_arguments_without_a_device():
    lib = _lib.load()
    assert lib.lbft_commit_times(None, None, None, 16) == -1


def test_bindings_match_the_header_the_rust_shim_and_integration_md():
    header = open(os.path.join(ROOT, "include", "lbft.h")).read()
    assert int(re.search(r"#define LBFT_FLAG_COMMIT_TIMES (\d+)u", header).group(1)) == _lib.FLAG_COMMIT_TIMES == 16
    assert not re.search(r"#define LBFT_FLAG_\w+ 8u", header)  # bit 8 stays unassigned
    assert re.search(r"int lbft_commit_times\(lbft_sim\* sim, int64_t\* committed, int64_t\* proposed, size_t cap\);", header)
    assert "lbft_commit_times" in _lib.EXPORTS
    rust = open(os.path.join(ROOT, "bft-lib-gpu", "src", "lib.rs")).read()
    assert re.search(r"pub const LBFT_FLAG_COMMIT_TIMES: u32 = 16;", rust)
    assert re.search(r"pub fn lbft_commit_times\(sim: \*mut LbftSim, committed: \*mut i64, proposed: \*mut i64, cap: usize\) -> c_int;", rust)
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    row = [ln for ln in doc.splitlines() if "lbft_commit_times" in ln]
    assert row and "new" in row[0].lower()


def test_python_options_map_onto_the_flag():
    delay = RandomDelay.new(10.0, 4.0)
    assert BatchSimulator([1, 2], 4, delay, commit_times=True).make_config(1000).flags == CT
    assert BatchSimulator([1, 2], 4, delay).make_config(1000).flags == 0
    sw = SweepSimulator.grid(4, [delay], [NodeConfig(), NodeConfig(delta=30)], commit_times=True)
    assert sw.make_config(1000).flags == CT
    assert Simulator.new(52, 3, delay, None, commit_times=True)._batch.make_config(1000).flags == CT
