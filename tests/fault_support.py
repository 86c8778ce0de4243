"""Test support for fault sweeps (lbft_create_sweep_faults): the ctypes wrapper of tests/hostcore/fault_hostcore.cpp (the SW and
SW + CT cores through the product's host setup), the fault sets the tests cross with tests/sweep_support.SETS, and the oracle
run once per set with that set's delay, NodeConfig, silent nodes and partition plan."""
import ctypes

import numpy as np

from librabft_simulator_b200 import FaultSet, ParamSet, _build
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, LbftConfig, LbftFaultSet, LbftLatencySpec, LbftParamSet
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE, LatencyStats
from tests.support import P, Result, make_config
from tests.sweep_support import c_sets, set_kwargs


def fault_sets(num_nodes):
    """No faults; one silent node; f silent nodes; f + 1 silent nodes (nothing commits); BASELINE config 5's plan (4 windows x
    150 ms); 2 windows x 400 ms with a silent node; 64 windows."""
    f = (num_nodes - 1) // 3
    return [FaultSet(), FaultSet((num_nodes - 1,)), FaultSet(tuple(range(f))), FaultSet(tuple(range(num_nodes - f - 1, num_nodes))),
            FaultSet((), 4, 150), FaultSet((1,), 2, 400), FaultSet((), 64, 50)]


def cross(sets, faults):
    """Every parameter set with every fault set, faults fastest."""
    return [ParamSet(p.network_delay, p.node_config, f) for p in sets for f in faults]


def fault_kwargs(fs, num_nodes):
    """The lbft_config fields (tests.support.make_config keywords) a fault set stands for."""
    silent = None
    if fs.silent:
        silent = np.zeros(num_nodes, np.uint8)
        silent[list(fs.silent)] = 1
    return dict(silent=silent, partition_windows=fs.partition_windows, partition_max_len=fs.partition_max_len)


def c_faults(sets):
    return (LbftFaultSet * max(1, len(sets)))(*[p.faults.to_c() for p in sets])


def oracle_per_set(oracle, seeds, num_nodes, max_clock, sets, set_of, **shared):
    """The oracle run once per set (delay, NodeConfig and faults substituted) over its instances, in instance order."""
    seeds, set_of = np.asarray(seeds, dtype=np.uint64), np.asarray(set_of)
    out = Result(len(seeds), num_nodes)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        if len(idx) == 0:
            continue
        kw = dict(shared)
        kw.update(set_kwargs(ps))
        kw.update(fault_kwargs(ps.faults, num_nodes))
        r = oracle.run(seeds[idx], num_nodes, max_clock, **kw)
        out.commit_counts[idx], out.last_states[idx], out.counters[idx], out.status[idx] = r.commit_counts, r.last_states, r.counters, r.status
    return out


class FaultHarness:
    """fault_hostcore_* of tests/hostcore/fault_hostcore.cpp.  faults=False runs the same sets through lbft_create_sweep's host
    setup (their FaultSet ignored), for the equivalence with a sweep whose configuration carries the faults."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_fault_hostcore())
        L = self.lib
        L.fault_hostcore_last_error.restype = ctypes.c_char_p
        head = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.POINTER(LbftFaultSet), ctypes.c_uint32, P]
        L.fault_hostcore_kernel_info.argtypes = head + [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32)]
        L.fault_hostcore_run.argtypes = head + [P] * 5
        L.fault_hostcore_run_ct.argtypes = head + [P] * 7 + [ctypes.c_size_t, ctypes.POINTER(LbftLatencySpec), P, P]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.fault_hostcore_last_error().decode()))

    def _args(self, seeds, num_nodes, max_clock, sets, set_of, faults, shared):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        keep += [so, c_sets(sets), c_faults(sets) if faults else None]
        return cfg, keep, (ctypes.byref(cfg), keep[-2], keep[-1], len(sets), P(so.ctypes.data))

    def kernel_info(self, seeds, num_nodes, max_clock, sets, set_of, faults=True, **shared):
        """(kernel name, Layout::part_windows) of the handle's host setup."""
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, shared)
        buf, w = ctypes.create_string_buffer(128), ctypes.c_uint32()
        self._check(self.lib.fault_hostcore_kernel_info(*head, buf, ctypes.sizeof(buf), ctypes.byref(w)))
        return buf.value.decode(), w.value

    def run(self, seeds, num_nodes, max_clock, sets, set_of, faults=True, **shared):
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, shared)
        res = Result(cfg.num_instances, num_nodes)
        res.lc_round = np.zeros((cfg.num_instances, num_nodes), np.uint32)
        self._check(self.lib.fault_hostcore_run(*head, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data),
                                                P(res.lc_round.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data)))
        return res

    def run_ct(self, seeds, num_nodes, max_clock, sets, set_of, cap=128, spec=None, faults=True, **shared):
        """The SW + CT core: the getters' outputs, ``committed`` / ``proposed`` (lbft_commit_times at ``cap``) and, with a spec,
        ``stats`` (lbft_latency_stats grouped by set)."""
        shared.setdefault("flags", FLAG_COMMIT_TIMES)
        cfg, keep, head = self._args(seeds, num_nodes, max_clock, sets, set_of, faults, shared)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        res.committed = np.zeros((I, num_nodes, cap), np.int64)
        res.proposed = np.zeros((I, cap), np.int64)
        out = np.zeros(len(sets), LATENCY_SUMMARY_DTYPE)
        hist = np.zeros((len(sets), spec.num_bins if spec is not None else 0), np.uint64)
        self._check(self.lib.fault_hostcore_run_ct(*head, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data),
                                                   P(res.lc_round.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data),
                                                   P(res.committed.ctypes.data), P(res.proposed.ctypes.data), cap,
                                                   None if spec is None else ctypes.byref(spec), P(out.ctypes.data),
                                                   P(hist.ctypes.data) if spec is not None else None))
        if spec is not None:
            res.stats = LatencyStats(out, hist, spec.bin_width)
        return res
