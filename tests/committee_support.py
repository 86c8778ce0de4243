"""Test support for committee sweeps (lbft_create_sweep_committees): the ctypes wrapper of tests/hostcore/committee_hostcore.cpp
(the SW and SW + CT cores through the product's host setup and set table), the sets the tests cross with tests/sweep_support.SETS,
and the oracle run once per set as a plain configuration of that set's committee size, padded to the layout's committee."""
import ctypes

import numpy as np

from librabft_simulator_b200 import BlockLatencyStats, FaultSet, ParamSet, _build
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, LbftConfig, LbftFaultSet, LbftLatencySpec, LbftParamSet
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE
from tests.fault_support import c_faults, fault_kwargs
from tests.support import P, Result, make_config
from tests.sweep_support import c_sets, set_kwargs

FLAGS_CT = FLAG_COMMIT_TIMES


def size_of(ps, num_nodes):
    return num_nodes if ps.num_nodes is None else int(ps.num_nodes)


def rights_rows(sets, num_nodes):
    """The [num_sets][num_nodes] table lbft_create_sweep_committees takes (1 per node of the set's committee where a set leaves its
    rights None, 0 past it), or None when no set carries rights."""
    if all(p.voting_rights is None for p in sets):
        return None
    rows = np.zeros((len(sets), num_nodes), np.uint64)
    for s, p in enumerate(sets):
        n = size_of(p, num_nodes)
        rows[s, :n] = (1,) * n if p.voting_rights is None else p.voting_rights
    return rows


def variants(n, k, partitions=False):
    """Variant k % 3 of a set of committee n: no fault and 1 per node; a silent node (node k % n, when n > 1); a zero-weight
    node (node 0, when n > 1).  partitions: every other variant also draws a partition plan."""
    v = k % 3
    plan = (2, 200) if partitions and k % 2 else (0, 0)
    silent = (k % n,) if v == 1 and n > 1 else ()
    rights = (0,) + (1,) * (n - 1) if v == 2 and n > 1 else None
    return FaultSet(silent, *plan), rights


def cross_sizes(sets, sizes, partitions=False):
    """Every parameter set with every committee size, sizes fastest; each with a fault / rights variant (variants)."""
    out = []
    for p in sets:
        for n in sizes:
            f, r = variants(n, len(out), partitions)
            out.append(ParamSet(p.network_delay, p.node_config, f, r, n))
    return out


def oracle_per_committee(oracle, seeds, num_nodes, max_clock, sets, set_of, faults=True, **shared):
    """The oracle run once per set as a plain configuration of the set's committee n (delay, NodeConfig, faults when `faults`,
    and voting rights substituted) over its instances, in [I][num_nodes] arrays whose columns past n are 0."""
    seeds, set_of = np.asarray(seeds, dtype=np.uint64), np.asarray(set_of)
    out = Result(len(seeds), num_nodes)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        if len(idx) == 0:
            continue
        n = size_of(ps, num_nodes)
        kw = dict(shared)
        kw.update(set_kwargs(ps))
        if faults:
            kw.update(fault_kwargs(ps.faults, n))
        kw["voting_rights"] = None if ps.voting_rights is None else np.asarray(ps.voting_rights, np.uint64)
        r = oracle.run(seeds[idx], n, max_clock, **kw)
        out.commit_counts[idx[:, None], np.arange(n)] = r.commit_counts
        out.last_states[idx[:, None], np.arange(n)] = r.last_states
        out.counters[idx], out.status[idx] = r.counters, r.status
    return out


class CommitteeHarness:
    """committee_hostcore_* of tests/hostcore/committee_hostcore.cpp.  mode "committees" builds lbft_create_sweep_committees'
    host setup; "rights" lbft_create_sweep_rights' (rows of 1 where a set leaves its rights None); "plain" lbft_create_sweep(_faults)'
    (faults=True), their rights ignored: the handles a committee sweep of full-size sets must equal."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_committee_hostcore())
        L = self.lib
        L.committee_hostcore_last_error.restype = ctypes.c_char_p
        head = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.POINTER(LbftFaultSet), P, P, ctypes.c_uint32, P]
        L.committee_hostcore_kernel_info.argtypes = head + [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32),
                                                            ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint32), P]
        L.committee_hostcore_run.argtypes = head + [P] * 6 + [ctypes.c_size_t, P, P, ctypes.POINTER(LbftLatencySpec), P, P, P, P]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.committee_hostcore_last_error().decode()))

    def _args(self, seeds, num_nodes, max_clock, sets, set_of, faults, mode, shared, sizes=None, rows="auto"):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        if rows == "auto":
            rows = rights_rows(sets, num_nodes)
            if mode == "rights" and rows is None:
                rows = np.ones((len(sets), num_nodes), np.uint64)
        if mode == "plain":
            rows = None
        if sizes is None and mode == "committees":
            sizes = [size_of(p, num_nodes) for p in sets]
        sz = None if sizes is None or mode != "committees" else np.ascontiguousarray(sizes, np.uint32)
        keep += [so, c_sets(sets), c_faults(sets) if faults else None, rows, sz]
        return cfg, keep, (ctypes.byref(cfg), keep[-4], keep[-3], None if rows is None else P(rows.ctypes.data),
                           None if sz is None else P(sz.ctypes.data), len(sets), P(so.ctypes.data))

    def kernel_info(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, mode="committees", leaders=False, **shared):
        """(kernel name, words per instance, bytes of leader tables, records bits) of the handle's host setup, and with
        leaders=True each set's leader table, one after the other (round_cap + 1 entries each)."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, mode, shared)
        buf, w, lb, rec = ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint32()
        tables = np.zeros(len(sets) * ((1 << 15) + 1), np.uint8) if leaders else None
        self._check(self.lib.committee_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(lb),
                                                            ctypes.byref(rec), None if tables is None else P(tables.ctypes.data)))
        out = (buf.value.decode(), w.value, lb.value, rec.value)
        return out + (tables,) if leaders else out

    def check(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, sizes=None, rows="auto", **shared):
        """The host setup's refusal (RuntimeError with the message), given raw sizes / rights rows."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, "committees", shared, sizes, rows)
        buf, w, lb, rec = ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64(), ctypes.c_uint32()
        self._check(self.lib.committee_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(lb),
                                                            ctypes.byref(rec), None))

    def run(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, mode="committees", cap=128, spec=None, thresholds=None, **shared):
        """The getters' outputs, ``lc_round`` and ``proposers[I, cap]``; with ``flags=FLAG_COMMIT_TIMES`` also ``committed`` /
        ``proposed``, and with thresholds (one per set) ``stats``, the BlockLatencyStats of lbft_block_latency_stats_groups."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, mode, shared)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        res.proposers = np.zeros((I, cap), np.uint32)
        res.committed = np.zeros((I, num_nodes, cap), np.int64)
        res.proposed = np.zeros((I, cap), np.int64)
        groups = len(sets)
        out, unreached = np.zeros(groups, LATENCY_SUMMARY_DTYPE), np.zeros(groups, np.uint64)
        hist = np.zeros((groups, spec.num_bins if spec is not None else 0), np.uint64)
        W = None if thresholds is None else np.ascontiguousarray(thresholds, np.uint64)
        self._check(self.lib.committee_hostcore_run(
            *head, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data),
            P(res.counters.ctypes.data), P(res.status.ctypes.data), P(res.proposers.ctypes.data), cap, P(res.committed.ctypes.data),
            P(res.proposed.ctypes.data), None if spec is None else ctypes.byref(spec), None if W is None else P(W.ctypes.data),
            P(out.ctypes.data), P(unreached.ctypes.data), P(hist.ctypes.data) if spec is not None else None))
        if W is not None:
            res.stats = BlockLatencyStats(out, unreached, hist, spec.bin_width, W)
        return res
