"""Test support for outage sweeps (lbft_create_sweep_outages): the ctypes wrapper of tests/hostcore/outage_hostcore.cpp (the SW and
SW + CT cores through the product's host setup and set table), the outage schedules the tests cross with tests/sweep_support.SETS,
and the oracle run once per set with that set's delay, NodeConfig, faults, voting rights, committee size, link latencies and
outage windows (tests/hostcore/outage_oracle.hpp), with a trace of every pop and its fate."""
import ctypes

import numpy as np

from librabft_simulator_b200 import FaultSet, ParamSet, _build
from librabft_simulator_b200._lib import INT64_MAX, LbftCommit, LbftConfig, LbftFaultSet, LbftOutage, LbftParamSet
from tests.committee_support import size_of
from tests.fault_support import c_faults, fault_kwargs
from tests.link_support import link_table, rights_rows
from tests.support import P, Result, make_config
from tests.sweep_support import c_sets, set_kwargs

# PopFate of outage_oracle.hpp: what became of a pop
POP_HANDLED, POP_CANCELLED, POP_RECEIVER_SILENT, POP_RECEIVER_DOWN, POP_SENDER_SILENT, POP_SENDER_DOWN = range(6)
EV_NOTIFY, EV_REQUEST, EV_RESPONSE, EV_TIMER = range(4)


def with_outages(fs, outages):
    """`fs` with its outages replaced."""
    return FaultSet(fs.silent, fs.partition_windows, fs.partition_max_len, tuple(outages))


def set_with_outages(ps, outages):
    """Parameter set `ps` with its fault set's outages replaced."""
    return ParamSet(ps.network_delay, ps.node_config, with_outages(ps.faults, outages), ps.voting_rights, ps.num_nodes, ps.link_latency)


def schedules(n, max_clock, silent=()):
    """(name, outages) per committee of n nodes, over nodes that are not silent: none; a crash-stop of the first live node at a
    third of the run; a crash-recovery of the last live node over the middle fifth; two nodes down at once, one of them from
    clock 0 for a while; an empty window; a window past max_clock."""
    live = [k for k in range(n) if k not in silent]
    a, b = live[0], live[-1]
    out = [("none", ()), ("crash-stop", ((a, max_clock // 3, None),)),
           ("crash-recovery", ((b, 2 * max_clock // 5, 3 * max_clock // 5),)),
           ("empty", ((a, 300, 300),)), ("past", ((b, max_clock + 1, max_clock + 500),))]
    if len(live) >= 3:
        out.append(("two", ((live[1], 0, max_clock // 4), (b, max_clock // 2, max_clock // 2 + 150))))
    return out


def c_windows(outages, n):
    """The [n] lbft_outage windows of one set (empty where a node has none; None as INT64_MAX), unclamped."""
    w = (LbftOutage * n)()
    for node, start, end in outages:
        w[node] = LbftOutage(start, INT64_MAX if end is None else end)
    return w


def outage_table(sets, num_nodes):
    """The [num_sets * num_nodes] lbft_outage table lbft_create_sweep_outages takes."""
    t = (LbftOutage * (len(sets) * num_nodes))()
    for s, p in enumerate(sets):
        for node, start, end in p.faults.outages:
            t[s * num_nodes + node] = LbftOutage(start, INT64_MAX if end is None else end)
    return t


def set_config(ps, num_nodes, faults=True):
    """(committee size n, make_config keywords, n x n matrix or None, n windows) of one set run as a plain configuration of its
    committee."""
    n = size_of(ps, num_nodes)
    kw = set_kwargs(ps)
    if faults:
        kw.update(fault_kwargs(ps.faults, n))
    kw["voting_rights"] = None if ps.voting_rights is None else np.asarray(ps.voting_rights, np.uint64)
    m = None if ps.link_latency is None else np.asarray(ps.link_latency, np.uint32)
    return n, kw, m, c_windows(ps.faults.outages, n)


class OutageOracle:
    """The oracle with link latencies and outage windows (tests/hostcore/outage_oracle.hpp, through outage_oracle_* of
    tests/hostcore/outage_hostcore.cpp): runs, commit logs, commit times and a trace of every pop."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_outage_hostcore())
        L = self.lib
        L.outage_hostcore_last_error.restype = ctypes.c_char_p
        L.outage_oracle_run.argtypes = [ctypes.POINTER(LbftConfig), P, P, P, P, P, P]
        L.outage_oracle_commit_log.argtypes = [ctypes.POINTER(LbftConfig), P, P, ctypes.c_uint32, ctypes.c_uint32,
                                               ctypes.POINTER(LbftCommit), ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.outage_oracle_trace.argtypes = [ctypes.POINTER(LbftConfig), P, P, ctypes.c_uint32, P, ctypes.c_size_t,
                                          ctypes.POINTER(ctypes.c_size_t)]
        L.outage_oracle_commit_times.argtypes = [ctypes.POINTER(LbftConfig), P, P, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_size_t,
                                                 P, P, P]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.outage_hostcore_last_error().decode())

    @staticmethod
    def _ptrs(links, windows):
        m = None if links is None else np.ascontiguousarray(links, np.uint32)
        return m, (None if m is None else P(m.ctypes.data)), (None if windows is None else ctypes.cast(windows, P))

    def run(self, seeds, num_nodes, max_clock, links=None, windows=None, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m, mp, wp = self._ptrs(links, windows)
        res = Result(cfg.num_instances, num_nodes)
        self._check(self.lib.outage_oracle_run(ctypes.byref(cfg), mp, wp, P(res.commit_counts.ctypes.data),
                                               P(res.last_states.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data)))
        return res

    def commit_log(self, seeds, num_nodes, instance, node, max_clock, links=None, windows=None, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m, mp, wp = self._ptrs(links, windows)
        n = ctypes.c_size_t()
        buf = (LbftCommit * 65536)()
        self._check(self.lib.outage_oracle_commit_log(ctypes.byref(cfg), mp, wp, instance, node, buf, 65536, ctypes.byref(n)))
        return [(int(buf[i].proposer), int(buf[i].index), int(buf[i].time)) for i in range(n.value)]

    def trace(self, seeds, num_nodes, instance, max_clock, links=None, windows=None, **kw):
        """Every pop of one instance as an int64 array [pops, 5]: kind, receiver, sender, pop clock, fate (POP_*)."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m, mp, wp = self._ptrs(links, windows)
        n = ctypes.c_size_t()
        self._check(self.lib.outage_oracle_trace(ctypes.byref(cfg), mp, wp, instance, None, 0, ctypes.byref(n)))
        rows = np.zeros((n.value, 5), np.int64)
        self._check(self.lib.outage_oracle_trace(ctypes.byref(cfg), mp, wp, instance, P(rows.ctypes.data), n.value, ctypes.byref(n)))
        return rows

    def commit_times(self, seeds, num_nodes, max_clock, links=None, windows=None, cap=128, **kw):
        """(committed [I][N][cap], proposed [I][cap], commit_counts [I][N]) of a run with link latencies and outages."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m, mp, wp = self._ptrs(links, windows)
        I = cfg.num_instances
        committed, proposed = np.zeros((I, num_nodes, cap), np.int64), np.zeros((I, cap), np.int64)
        counts = np.zeros((I, num_nodes), np.uint32)
        self._check(self.lib.outage_oracle_commit_times(ctypes.byref(cfg), mp, wp, 0, I, cap, P(committed.ctypes.data),
                                                        P(proposed.ctypes.data), P(counts.ctypes.data)))
        return committed, proposed, counts


def oracle_per_set(oracle, seeds, num_nodes, max_clock, sets, set_of, faults=True, **shared):
    """The oracle run once per set as a plain configuration of its committee with its link latencies and outage windows, over
    its instances, in [I][num_nodes] arrays whose columns past the committee are 0."""
    seeds, set_of = np.asarray(seeds, dtype=np.uint64), np.asarray(set_of)
    out = Result(len(seeds), num_nodes)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        if len(idx) == 0:
            continue
        n, kw, m, w = set_config(ps, num_nodes, faults)
        kw.update(shared)
        r = oracle.run(seeds[idx], n, max_clock, m, w, **kw)
        out.commit_counts[idx[:, None], np.arange(n)] = r.commit_counts
        out.last_states[idx[:, None], np.arange(n)] = r.last_states
        out.counters[idx], out.status[idx] = r.counters, r.status
    return out


class OutageHarness:
    """outage_hostcore_* of tests/hostcore/outage_hostcore.cpp.  outages=False builds the same sweep without its windows through
    the existing entry points (lbft_create_sweep_links when links=True, else _committees / _rights / _faults / lbft_create_sweep as
    the sets call for): what empty schedules must equal."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_outage_hostcore())
        L = self.lib
        L.outage_hostcore_last_error.restype = ctypes.c_char_p
        head = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.POINTER(LbftFaultSet), P, P, P, P, ctypes.c_uint32, P]
        L.outage_hostcore_kernel_info.argtypes = head + [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32),
                                                         ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32),
                                                         ctypes.POINTER(ctypes.c_uint64)]
        L.outage_hostcore_run.argtypes = head + [P] * 6 + [ctypes.c_size_t, P, P]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.outage_hostcore_last_error().decode()))

    def _args(self, seeds, num_nodes, max_clock, sets, set_of, faults, links, outages, shared, rows="auto", sizes="auto",
              table="auto"):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        if isinstance(rows, str):
            rows = rights_rows(sets, num_nodes)
        if isinstance(sizes, str):
            sizes = None if all(p.num_nodes is None for p in sets) else np.array([size_of(p, num_nodes) for p in sets], np.uint32)
        sizes = None if sizes is None else np.ascontiguousarray(sizes, np.uint32)
        mats = link_table(sets, num_nodes) if links else None
        if isinstance(table, str):
            table = outage_table(sets, num_nodes) if outages else None
        keep += [so, c_sets(sets), c_faults(sets) if faults else None, rows, sizes, mats, table]
        ptr = lambda a: None if a is None else P(a.ctypes.data)  # noqa: E731
        return cfg, keep, (ctypes.byref(cfg), keep[-6], keep[-5], ptr(rows), ptr(sizes), ptr(mats),
                           None if table is None else ctypes.cast(table, P), len(sets), P(so.ctypes.data))

    def kernel_info(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, links=False, outages=True, **shared):
        """(kernel name, words per instance, bytes of outage schedules, records bits, down mask) of the handle's host setup."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, links, outages, shared)
        buf, w, ob, rec, dm = (ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint32(),
                               ctypes.c_uint64())
        self._check(self.lib.outage_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(ob),
                                                         ctypes.byref(rec), ctypes.byref(dm)))
        return buf.value.decode(), w.value, ob.value, rec.value, dm.value

    def check(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, links=False, table="auto", **shared):
        """The host setup's refusal (RuntimeError with the message), given a raw outage table."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, links, True, shared, table=table)
        buf, w, ob, rec, dm = (ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint32(),
                               ctypes.c_uint64())
        self._check(self.lib.outage_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(ob),
                                                         ctypes.byref(rec), ctypes.byref(dm)))

    def run(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, links=False, outages=True, cap=128, **shared):
        """The getters' outputs, ``lc_round`` and ``proposers[I, cap]``; with ``flags=FLAG_COMMIT_TIMES`` also ``committed`` /
        ``proposed``."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, links, outages, shared)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        res.proposers = np.zeros((I, cap), np.uint32)
        res.committed = np.zeros((I, num_nodes, cap), np.int64)
        res.proposed = np.zeros((I, cap), np.int64)
        self._check(self.lib.outage_hostcore_run(
            *head, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data),
            P(res.counters.ctypes.data), P(res.status.ctypes.data), P(res.proposers.ctypes.data), cap, P(res.committed.ctypes.data),
            P(res.proposed.ctypes.data)))
        return res
