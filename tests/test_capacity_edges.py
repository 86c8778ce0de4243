"""The capacity edges (tests/capacity_cases.py) on the host-compiled core: every case selects its kernel at its generous and
its tight capacity and gets the capacities it asks for; at the tight capacity C the error bit under test is set exactly on
the instances whose peak in the generous run exceeds C, some clean instance uses the last entry, and every clean instance
ends bit for bit as it did in the generous run (and as the oracle says).  Also: the read-out floor the host raises queue_cap
to, and the creation-stamp limits of the configurations the host sends to 16-bit stamps."""
import ctypes
import itertools

import numpy as np
import pytest

from librabft_simulator_b200 import _lib
from tests import sweep_support
from tests.capacity_cases import CAP_FIELD, CASES, CLEAN, EDGES, PEAK_COLUMN, STAMP_LIMIT, readout_queue_floor, tight
from tests.support import P, assert_same, make_config

ERR = np.uint32(_lib.ST_ERROR_MASK)
BIT = {"queue": np.uint32(_lib.ST_QUEUE_OVERFLOW), "payload": np.uint32(_lib.ST_PAYLOAD_OVERFLOW),
       "round": np.uint32(_lib.ST_ROUND_OVERFLOW)}

# The (family, tile or lane group, state in shared memory, QMODE, capacity) combinations the table covers.
COVERED = {
    ("thread", 32, False, 0, "queue"), ("thread", 32, False, 1, "queue"), ("thread", 32, False, 2, "queue"),
    ("thread", 32, False, 3, "queue"), ("thread", 8, False, 3, "queue"), ("thread", 16, False, 3, "queue"),
    ("thread", 32, False, 2, "payload"), ("thread", 32, False, 3, "payload"),
    ("thread", 32, False, 2, "round"), ("thread", 32, False, 3, "round"),
    ("wide", 32, False, 0, "queue"), ("wide", 8, False, 2, "queue"), ("wide", 8, True, 2, "queue"), ("wide", 32, True, 2, "queue"),
    ("wide", 8, False, 3, "queue"), ("wide", 32, False, 3, "queue"), ("wide", 32, False, 3, "payload"),
    ("wide", 32, True, 2, "round"),
    ("sweep thread", 32, False, 3, "queue"), ("sweep wide", 8, False, 2, "queue"),
    ("thread", 32, False, 0, "floor"), ("thread", 32, False, 1, "floor"), ("thread", 32, False, 2, "floor"),
    ("thread", 32, False, 3, "floor"), ("thread", 32, False, 3, "horizon"), ("wide", 32, False, 3, "horizon"),
    ("wide", 32, False, 2, "horizon"),
}


def set_force(monkeypatch, force):
    if force is None:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    else:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", force)


@pytest.fixture(scope="module")
def sweep_host():
    return sweep_support.SweepHostCore()


def host_kernel(hostcore, sweep_host, case, kw):
    if case.kind == "sweep":
        return sweep_host.kernel_info(case.seeds, case.N, case.max_clock, case.sets, case.set_of, **kw)
    return hostcore.kernel_info(case.seeds, case.N, case.max_clock, **kw)


def host_run(hostcore, sweep_host, case, kw):
    if case.kind == "sweep":
        return sweep_host.run(case.seeds, case.N, case.max_clock, case.sets, case.set_of, **kw)
    return hostcore.run(case.seeds, case.N, case.max_clock, **kw)


def effective_caps(hostcore, case, kw):
    """The capacities the host setup gives the case's batch (the batch size picks the kernel family, and with it the queue
    mode and its read-out floor; a sweep's layout is its fastest set's: the host setup of that set)."""
    if case.kind == "sweep":
        fastest = min(case.sets, key=lambda p: p.network_delay.mean if p.network_delay.kind == 0 else
                      0.5 * (p.network_delay.lo + p.network_delay.hi))
        kw = dict(kw, **sweep_support.set_kwargs(fastest))
    cfg, keep = make_config(case.seeds, case.N, case.max_clock, **kw)
    out = np.zeros(6, np.uint32)
    assert hostcore.lib.hostcore_setup_info(ctypes.byref(cfg), P(out.ctypes.data)) == 0
    return dict(zip(("delay_kmax", "queue_scan", "round_cap", "queue_cap", "payload_cap", "words"), out.tolist()))


def check_stamps(qmode, res):
    """A creation stamp past the mode's limit is flagged: stamp-flagged <=> counters[:, 5] >= the limit (the flag fires when
    the counter reaches it, so every stamp handed out is representable)."""
    stamp_out = res.counters[:, 5] >= STAMP_LIMIT[qmode]
    queue_bit = (res.status & BIT["queue"]) != 0
    assert not (stamp_out & ~queue_bit).any(), "stamps past the limit without LBFT_ST_QUEUE_OVERFLOW"
    # a queue flag with the queue never full is a stamp flag
    np.testing.assert_array_equal(queue_bit & (res.counters[:, 8] < res.queue_cap), queue_bit & stamp_out)


def check_edge(case, A, B, C):
    """Properties of a tight run B against the generous run A (both results of the same core)."""
    assert not (A.status & ERR).any(), ("run A is not generous", np.unique(A.status))
    bit = BIT[case.cap]
    flagged = (B.status & ERR) != 0
    if case.cap == "round":
        r = A.counters[:, 6]
        assert flagged[r >= C].all() and (r[flagged] >= C - 1).all()
        last = ~flagged & (A.counters[:, 6] == C - 1)
    else:
        peak = A.counters[:, PEAK_COLUMN[case.cap]]
        np.testing.assert_array_equal(flagged, peak > C, err_msg="flagged <=> peak in A > C")
        last = ~flagged & (peak == C)
    np.testing.assert_array_equal(B.status[flagged] & ERR, np.full(flagged.sum(), bit), err_msg="other error bits")
    assert last.any(), "no clean instance uses the last entry"
    assert flagged.any() and (~flagged).any()
    clean = ~flagged
    np.testing.assert_array_equal(B.commit_counts[clean], A.commit_counts[clean])
    np.testing.assert_array_equal(B.last_states[clean], A.last_states[clean])
    np.testing.assert_array_equal(B.counters[clean], A.counters[clean])
    np.testing.assert_array_equal(B.status[clean], A.status[clean])
    return flagged


def test_the_table_covers_its_combinations():
    assert {c.combination() for c in CASES.values()} == COVERED


@pytest.mark.parametrize("cid", sorted(CASES))
def test_case_selects_its_kernel_and_capacities(hostcore, sweep_host, monkeypatch, cid):
    case = CASES[cid]
    set_force(monkeypatch, case.force)
    runs = [case.kw]
    if case.cap in CAP_FIELD:
        runs.append(case.tight_kw(tight(case, host_run(hostcore, sweep_host, case, case.kw).counters)))
    for kw in runs:
        assert host_kernel(hostcore, sweep_host, case, kw) == case.name, kw
        got = effective_caps(hostcore, case, kw)
        for cap in ("round_cap", "queue_cap", "payload_cap"):
            if cap in kw:
                assert got[cap] == kw[cap], (cap, got)
        assert got["queue_scan"] == case.qmode, got
    if case.cap == "floor":
        assert case.kw["queue_cap"] == readout_queue_floor(case.qmode, case.kw["round_cap"])


@pytest.mark.parametrize("cid", sorted(EDGES))
def test_tight_capacity_flags_exactly_the_overflowing_instances(hostcore, sweep_host, oracle, monkeypatch, cid):
    case = EDGES[cid]
    set_force(monkeypatch, case.force)
    A = host_run(hostcore, sweep_host, case, case.kw)
    C = tight(case, A.counters)
    B = host_run(hostcore, sweep_host, case, case.tight_kw(C))
    A.queue_cap = effective_caps(hostcore, case, case.kw)["queue_cap"]
    B.queue_cap = effective_caps(hostcore, case, case.tight_kw(C))["queue_cap"]
    flagged = check_edge(case, A, B, C)
    check_stamps(case.qmode, A)
    check_stamps(case.qmode, B)
    # the clean instances of a small sample against the oracle
    idx = np.nonzero(~flagged)[0][:24]
    if case.kind == "sweep":
        shared = {k: v for k, v in case.kw.items() if k != "flags"}
        ref = sweep_support.oracle_per_set(oracle, case.seeds[idx], case.N, case.max_clock, case.sets, case.set_of[idx], **shared)
    else:
        ref = oracle.run(case.seeds[idx], case.N, case.max_clock, **dict(case.kw, flags=0))
    sub = type(ref)(len(idx), case.N)
    sub.commit_counts, sub.last_states, sub.counters = B.commit_counts[idx], B.last_states[idx], B.counters[idx]
    assert_same(ref, sub, case.id)


@pytest.mark.parametrize("cid", sorted(CLEAN))
def test_floor_and_horizon_runs_match_the_oracle(hostcore, oracle, monkeypatch, cid):
    case = CLEAN[cid]
    set_force(monkeypatch, case.force)
    res = hostcore.run(case.seeds, case.N, case.max_clock, **case.kw)
    assert not (res.status & ERR).any(), np.unique(res.status)
    assert_same(oracle.run(case.seeds, case.N, case.max_clock, **dict(case.kw, flags=0)), res, case.id)
    if case.cap == "floor":
        # logs close to round_cap rows: the chain scratch finalize() borrows spans (nearly) the whole queue area
        assert res.commit_counts.max() >= case.kw["round_cap"] * 3 // 4, res.commit_counts.max()


@pytest.mark.parametrize("qmode,N,max_clock,kw", [(0, 1, 5000, dict(payload_cap=256)), (1, 1, 3000, {}), (2, 2, 1000, {}),
                                                  (3, 2, 1000, dict(payload_cap=256))])
def test_queue_cap_is_raised_to_the_readout_floor(hostcore, monkeypatch, qmode, N, max_clock, kw):
    set_force(monkeypatch, "thread")
    for rc in (64, 160, 224):
        floor = readout_queue_floor(qmode, rc)
        got = hostcore.setup_info(N, max_clock, round_cap=rc, queue_cap=floor - 1, **kw)
        if got["queue_scan"] != qmode:
            continue
        assert got["queue_cap"] == floor, (rc, got)
        assert hostcore.setup_info(N, max_clock, round_cap=rc, queue_cap=floor, **kw)["queue_cap"] == floor


# ---- 16-bit stamps: every configuration the host sends to the shared-memory scan queue with default capacities ----
STAMP_DELAYS = [{}, dict(delay_kind=1, delay_lo=0, delay_hi=12), dict(delay_variance=0.0), dict(delay_mean=25.0, delay_variance=200.0),
                dict(delay_kind=1, delay_lo=0, delay_hi=2), dict(delay_kind=1, delay_lo=1, delay_hi=4), dict(delay_mean=2.0, delay_variance=1.0),
                dict(target_commit_interval=150, delta=30, gamma=1.5, lambda_=1.0)]
STAMP_HORIZONS = [100, 400, 1000, 2000, 4095, 6000, 9000, 12000, 16319]


def test_sixteen_bit_stamps_suffice_where_the_host_chooses_them(hostcore, monkeypatch):
    """choose_layout sends a configuration to 16-bit stamps from an estimate of its event rate: no instance of such a
    configuration may run out of stamps (a QUEUE_OVERFLOW with no queue capacity exceeded)."""
    scanned = 0
    for force, N, kw, mc in itertools.product((None, "wide"), range(1, 6), STAMP_DELAYS, STAMP_HORIZONS):
        set_force(monkeypatch, force)
        info = hostcore.setup_info(N, mc, **kw)
        if info["queue_scan"] != 2:
            continue
        scanned += 1
        res = hostcore.run(np.arange(1000 * N + mc, 1000 * N + mc + 32, dtype=np.uint64), N, mc, **kw)
        assert res.counters[:, 5].max() < STAMP_LIMIT[2], (force, N, kw, mc, res.counters[:, 5].max())
        res.queue_cap = info["queue_cap"]
        check_stamps(2, res)
    assert scanned > 100
