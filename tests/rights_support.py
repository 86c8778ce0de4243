"""Test support for rights sweeps (lbft_create_sweep_rights): the ctypes wrapper of tests/hostcore/rights_hostcore.cpp (the SW and
SW + CT cores through the product's host setup and set table), the stake rows the tests cross with tests/sweep_support.SETS, and
the oracle run once per set with that set's delay, NodeConfig, faults and voting rights."""
import ctypes

import numpy as np

from librabft_simulator_b200 import BlockLatencyStats, FaultSet, ParamSet, _build
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, LbftConfig, LbftFaultSet, LbftLatencySpec, LbftParamSet
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE
from tests.fault_support import c_faults, fault_kwargs
from tests.support import P, Result, make_config
from tests.sweep_support import c_sets, set_kwargs

CAP = 1 << 24  # the largest voting right a node may hold


def stake_rows(n):
    """(name, row) per committee size n: all ones; [3, 1, 1, ...]; node 0 at exactly a third of the total, and just above it (no
    quorum forms without it either way); zero-weight nodes (0 and n - 1); entries of 2^24."""
    third = [n - 1] + [2] * (n - 1)  # total 3 (n - 1)
    above = [n] + [2] * (n - 1)
    zero = [0] + [1] * (n - 2) + [0] if n > 2 else [0, 1][:n]
    big = [CAP] * n
    big[1 % n] = 1
    return [("ones", [1] * n), ("skew", [3] + [1] * (n - 1)), ("third", third), ("above_third", above), ("zero", zero), ("cap", big)]


def rights_faults(row):
    """No faults, the heaviest node silent, and (where the row has one) a zero-weight node silent."""
    row = np.asarray(row)
    out = [FaultSet(), FaultSet((int(np.argmax(row)),))]
    if (row == 0).any():
        out.append(FaultSet((int(np.nonzero(row == 0)[0][-1]),)))
    return out


def rights_of(sets, num_nodes):
    """The [num_sets][num_nodes] table lbft_create_sweep_rights takes (1 per node where a set leaves its rights None)."""
    return np.ascontiguousarray([(1,) * num_nodes if p.voting_rights is None else p.voting_rights for p in sets], dtype=np.uint64)


def oracle_per_set(oracle, seeds, num_nodes, max_clock, sets, set_of, faults=True, **shared):
    """The oracle run once per set (delay, NodeConfig, faults when `faults`, and voting rights substituted) over its instances."""
    seeds, set_of = np.asarray(seeds, dtype=np.uint64), np.asarray(set_of)
    out = Result(len(seeds), num_nodes)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        if len(idx) == 0:
            continue
        kw = dict(shared)
        kw.update(set_kwargs(ps))
        if faults:
            kw.update(fault_kwargs(ps.faults, num_nodes))
        kw["voting_rights"] = None if ps.voting_rights is None else np.asarray(ps.voting_rights, np.uint64)
        r = oracle.run(seeds[idx], num_nodes, max_clock, **kw)
        out.commit_counts[idx], out.last_states[idx], out.counters[idx], out.status[idx] = r.commit_counts, r.last_states, r.counters, r.status
    return out


class RightsHarness:
    """rights_hostcore_* of tests/hostcore/rights_hostcore.cpp.  rights=False runs the same sets through lbft_create_sweep_faults
    (faults=True) or lbft_create_sweep's host setup, their voting rights ignored, for the equivalence with shared rights."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_rights_hostcore())
        L = self.lib
        L.rights_hostcore_last_error.restype = ctypes.c_char_p
        head = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.POINTER(LbftFaultSet), P, ctypes.c_uint32, P]
        L.rights_hostcore_kernel_info.argtypes = head + [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32),
                                                         ctypes.POINTER(ctypes.c_uint64)]
        L.rights_hostcore_run.argtypes = head + [P] * 6 + [ctypes.c_size_t, P, P, ctypes.POINTER(LbftLatencySpec), P, P, P, P]
        L.rights_hostcore_threshold_check.argtypes = head + [ctypes.POINTER(LbftLatencySpec), ctypes.c_uint64]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.rights_hostcore_last_error().decode()))

    def _args(self, seeds, num_nodes, max_clock, sets, set_of, faults, rights, shared):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        vr = rights_of(sets, num_nodes) if rights else None
        keep += [so, c_sets(sets), c_faults(sets) if faults else None, vr]
        return cfg, keep, (ctypes.byref(cfg), keep[-3], keep[-2], None if vr is None else P(vr.ctypes.data), len(sets), P(so.ctypes.data))

    def kernel_info(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, rights=True, **shared):
        """(kernel name, words per instance, bytes of leader tables) of the handle's host setup."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, rights, shared)
        buf, w, lb = ctypes.create_string_buffer(128), ctypes.c_uint32(), ctypes.c_uint64()
        self._check(self.lib.rights_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w), ctypes.byref(lb)))
        return buf.value.decode(), w.value, lb.value

    def threshold_check(self, seeds, num_nodes, max_clock, sets, set_of, spec, threshold, faults=False, **shared):
        """lbft_block_latency_stats' checks of its spec and scalar threshold on the handle (RuntimeError with the message)."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, True, shared)
        self._check(self.lib.rights_hostcore_threshold_check(*head, ctypes.byref(spec), threshold))

    def run(self, seeds, num_nodes, max_clock, sets, set_of, faults=False, rights=True, cap=128, spec=None, thresholds=None, **shared):
        """The getters' outputs, ``lc_round`` and ``proposers[I, cap]``; with ``flags=FLAG_COMMIT_TIMES`` also ``committed`` /
        ``proposed``, and with thresholds (one per set) ``stats``, the BlockLatencyStats of lbft_block_latency_stats_groups."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, rights, shared)
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
        self._check(self.lib.rights_hostcore_run(
            *head, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data),
            P(res.counters.ctypes.data), P(res.status.ctypes.data), P(res.proposers.ctypes.data), cap, P(res.committed.ctypes.data),
            P(res.proposed.ctypes.data), None if spec is None else ctypes.byref(spec), None if W is None else P(W.ctypes.data),
            P(out.ctypes.data), P(unreached.ctypes.data), P(hist.ctypes.data) if spec is not None else None))
        if W is not None:
            res.stats = BlockLatencyStats(out, unreached, hist, spec.bin_width, W)
        return res


def cross_rights(sets, rows, with_faults=False):
    """Every parameter set with every stake row (and, with_faults, every fault set of rights_faults(row)), faults fastest."""
    return [ParamSet(p.network_delay, p.node_config, f, tuple(r)) for p in sets for _, r in rows
            for f in (rights_faults(r) if with_faults else [FaultSet()])]


FLAGS_CT = FLAG_COMMIT_TIMES
