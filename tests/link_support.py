"""Test support for links sweeps (lbft_create_sweep_links): the ctypes wrapper of tests/hostcore/link_hostcore.cpp (the SW and
SW + CT cores through the product's host setup and set table), the link-latency matrices the tests cross with
tests/sweep_support.SETS, and the oracle run once per set with that set's delay, NodeConfig, faults, voting rights, committee
size and link latencies (tests/hostcore/link_oracle.hpp)."""
import ctypes

import numpy as np

from librabft_simulator_b200 import ParamSet, _build, regional_latency
from librabft_simulator_b200._lib import LbftCommit, LbftConfig, LbftFaultSet, LbftParamSet
from tests.committee_support import size_of
from tests.fault_support import c_faults, fault_kwargs
from tests.support import P, Result, make_config
from tests.sweep_support import c_sets, set_kwargs


def matrices(n):
    """(name, n x n matrix) per committee size n: nodes in three regions with symmetric latencies between them; an asymmetric
    matrix (every pair its own latency, a -> b differing from b -> a, a non-zero diagonal); one node far from all others; all
    zero."""
    regional = regional_latency([k % 3 for k in range(n)], [[1, 30, 80], [30, 2, 55], [80, 55, 3]])
    asym = tuple(tuple((7 * a + 3 * b) % 23 for b in range(n)) for a in range(n))
    far = tuple(tuple(0 if a == b else (120 if n - 1 in (a, b) else 4) for b in range(n)) for a in range(n))
    zero = tuple(tuple(0 for _ in range(n)) for _ in range(n))
    return [("regional", regional), ("asymmetric", asym), ("far", far), ("zero", zero)]


def cross_links(sets, mats):
    """Every parameter set with every matrix, matrices fastest (each set keeps its faults, rights and committee size)."""
    return [ParamSet(p.network_delay, p.node_config, p.faults, p.voting_rights, p.num_nodes, m) for p in sets for _, m in mats]


def link_table(sets, num_nodes):
    """The [num_sets][num_nodes][num_nodes] table lbft_create_sweep_links takes: each set's matrix in its committee's corner."""
    out = np.zeros((len(sets), num_nodes, num_nodes), np.uint32)
    for s, p in enumerate(sets):
        if p.link_latency is not None:
            m = np.asarray(p.link_latency, np.uint32)
            out[s, :m.shape[0], :m.shape[1]] = m
    return out


def rights_rows(sets, num_nodes):
    """The [num_sets][num_nodes] rights rows (1 per node of a set's committee where it leaves them None), or None if no set
    carries rights or its own committee size."""
    if all(p.voting_rights is None and p.num_nodes is None for p in sets):
        return None
    rows = np.zeros((len(sets), num_nodes), np.uint64)
    for s, p in enumerate(sets):
        n = size_of(p, num_nodes)
        rows[s, :n] = (1,) * n if p.voting_rights is None else p.voting_rights
    return rows


class LinkOracle:
    """The oracle with link latencies (tests/hostcore/link_oracle.hpp, through link_oracle_* of tests/hostcore/link_hostcore.cpp):
    runs, commit logs and a trace of every network event."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_link_hostcore())
        L = self.lib
        L.link_hostcore_last_error.restype = ctypes.c_char_p
        L.link_oracle_run.argtypes = [ctypes.POINTER(LbftConfig), P, P, P, P, P]
        L.link_oracle_commit_log.argtypes = [ctypes.POINTER(LbftConfig), P, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(LbftCommit),
                                             ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.link_oracle_trace.argtypes = [ctypes.POINTER(LbftConfig), P, ctypes.c_uint32, P, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.link_hostcore_last_error().decode())

    def run(self, seeds, num_nodes, max_clock, links, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m = np.ascontiguousarray(links, np.uint32)
        res = Result(cfg.num_instances, num_nodes)
        self._check(self.lib.link_oracle_run(ctypes.byref(cfg), P(m.ctypes.data), P(res.commit_counts.ctypes.data),
                                             P(res.last_states.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data)))
        return res

    def commit_log(self, seeds, num_nodes, instance, node, max_clock, links, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m = np.ascontiguousarray(links, np.uint32)
        n = ctypes.c_size_t()
        buf = (LbftCommit * 65536)()
        self._check(self.lib.link_oracle_commit_log(ctypes.byref(cfg), P(m.ctypes.data), instance, node, buf, 65536, ctypes.byref(n)))
        return [(int(buf[i].proposer), int(buf[i].index), int(buf[i].time)) for i in range(n.value)]

    def trace(self, seeds, num_nodes, instance, max_clock, links=None, **kw):
        """Every network event of one instance as an int64 array [events, 5]: kind, receiver, sender, send clock, due time."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m = None if links is None else np.ascontiguousarray(links, np.uint32)
        ptr = None if m is None else P(m.ctypes.data)
        n = ctypes.c_size_t()
        self._check(self.lib.link_oracle_trace(ctypes.byref(cfg), ptr, instance, None, 0, ctypes.byref(n)))
        rows = np.zeros((n.value, 5), np.int64)
        self._check(self.lib.link_oracle_trace(ctypes.byref(cfg), ptr, instance, P(rows.ctypes.data), n.value, ctypes.byref(n)))
        return rows


def set_config(ps, num_nodes, faults=True):
    """(committee size n, make_config keywords, n x n matrix) of one set run as a plain configuration of its committee."""
    n = size_of(ps, num_nodes)
    kw = set_kwargs(ps)
    if faults:
        kw.update(fault_kwargs(ps.faults, n))
    kw["voting_rights"] = None if ps.voting_rights is None else np.asarray(ps.voting_rights, np.uint64)
    m = np.zeros((n, n), np.uint32) if ps.link_latency is None else np.asarray(ps.link_latency, np.uint32)
    return n, kw, m


def oracle_per_set(oracle, seeds, num_nodes, max_clock, sets, set_of, faults=True, **shared):
    """The oracle run once per set as a plain configuration of its committee with its link latencies, over its instances, in
    [I][num_nodes] arrays whose columns past the committee are 0."""
    seeds, set_of = np.asarray(seeds, dtype=np.uint64), np.asarray(set_of)
    out = Result(len(seeds), num_nodes)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        if len(idx) == 0:
            continue
        n, kw, m = set_config(ps, num_nodes, faults)
        kw.update(shared)
        r = oracle.run(seeds[idx], n, max_clock, m, **kw)
        out.commit_counts[idx[:, None], np.arange(n)] = r.commit_counts
        out.last_states[idx[:, None], np.arange(n)] = r.last_states
        out.counters[idx], out.status[idx] = r.counters, r.status
    return out


class LinkHarness:
    """link_hostcore_* of tests/hostcore/link_hostcore.cpp.  links=False builds the same sweep without its matrices through the
    existing entry points (lbft_create_sweep_committees when a set has its own size, _rights when a set has rights, _faults when
    faults=True, else lbft_create_sweep): what all-zero matrices must equal."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_link_hostcore())
        L = self.lib
        L.link_hostcore_last_error.restype = ctypes.c_char_p
        head = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.POINTER(LbftFaultSet), P, P, P, ctypes.c_uint32, P]
        L.link_hostcore_kernel_info.argtypes = head + [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32),
                                                       ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32)]
        L.link_hostcore_run.argtypes = head + [P] * 6 + [ctypes.c_size_t, P, P]
        L.link_oracle_commit_times.argtypes = [ctypes.POINTER(LbftConfig), P, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_size_t, P, P, P]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.link_hostcore_last_error().decode()))

    def _args(self, seeds, num_nodes, max_clock, sets, set_of, faults, links, shared, rows="auto", sizes="auto", table="auto"):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        if isinstance(rows, str):
            rows = rights_rows(sets, num_nodes)
        if isinstance(sizes, str):
            sizes = None if all(p.num_nodes is None for p in sets) else np.array([size_of(p, num_nodes) for p in sets], np.uint32)
        if isinstance(table, str):
            table = link_table(sets, num_nodes) if links else None
        sizes = None if sizes is None else np.ascontiguousarray(sizes, np.uint32)
        keep += [so, c_sets(sets), c_faults(sets) if faults else None, rows, sizes, table]
        ptr = lambda a: None if a is None else P(a.ctypes.data)  # noqa: E731
        return cfg, keep, (ctypes.byref(cfg), keep[-5], keep[-4], ptr(rows), ptr(sizes), ptr(table), len(sets), P(so.ctypes.data))

    def kernel_info(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, links=True, **shared):
        """(kernel name, words per instance, bytes of link-latency tables, records bits) of the handle's host setup."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, links, shared)
        buf, w, lb, rec = ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint32()
        self._check(self.lib.link_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(lb), ctypes.byref(rec)))
        return buf.value.decode(), w.value, lb.value, rec.value

    def check(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, rows="auto", sizes="auto", table="auto", **shared):
        """The host setup's refusal (RuntimeError with the message), given raw rights rows, sizes and matrices."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, True, shared, rows, sizes, table)
        buf, w, lb, rec = ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint32()
        self._check(self.lib.link_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(lb), ctypes.byref(rec)))

    def run(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, links=True, cap=128, **shared):
        """The getters' outputs, ``lc_round`` and ``proposers[I, cap]``; with ``flags=FLAG_COMMIT_TIMES`` also ``committed`` /
        ``proposed``."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, links, shared)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        res.proposers = np.zeros((I, cap), np.uint32)
        res.committed = np.zeros((I, num_nodes, cap), np.int64)
        res.proposed = np.zeros((I, cap), np.int64)
        self._check(self.lib.link_hostcore_run(
            *head, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data),
            P(res.counters.ctypes.data), P(res.status.ctypes.data), P(res.proposers.ctypes.data), cap, P(res.committed.ctypes.data),
            P(res.proposed.ctypes.data)))
        return res

    def oracle_commit_times(self, seeds, num_nodes, max_clock, links, cap=128, **kw):
        """The oracle's (committed [I][N][cap], proposed [I][cap], commit_counts [I][N]) of a run with link latencies."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        m = np.ascontiguousarray(links, np.uint32)
        I = cfg.num_instances
        committed, proposed = np.zeros((I, num_nodes, cap), np.int64), np.zeros((I, cap), np.int64)
        counts = np.zeros((I, num_nodes), np.uint32)
        self._check(self.lib.link_oracle_commit_times(ctypes.byref(cfg), P(m.ctypes.data), 0, I, cap, P(committed.ctypes.data),
                                                      P(proposed.ctypes.data), P(counts.ctypes.data)))
        return committed, proposed, counts
