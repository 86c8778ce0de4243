"""Test support for commit times (LBFT_FLAG_COMMIT_TIMES): ctypes wrappers of tests/hostcore/ct_hostcore.cpp — the CT core on
the host through the product's host setup, and the oracle observed one event time at a time."""
import ctypes

import numpy as np

from librabft_simulator_b200 import _build
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, LbftConfig, LbftParamSet
from tests.support import P, Result, make_config
from tests.sweep_support import c_sets


class CtHarness:
    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_ct_hostcore())
        self.lib.ct_hostcore_last_error.restype = ctypes.c_char_p
        self.lib.ct_hostcore_run.argtypes = [ctypes.POINTER(LbftConfig)] + [P] * 8 + [ctypes.c_size_t, P]
        self.lib.ct_hostcore_run_sweep.argtypes = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.c_uint32] + \
            [P] * 8 + [ctypes.c_size_t]
        self.lib.ct_oracle_commit_times.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_size_t,
                                                    P, P, P]

    def _outputs(self, I, N, cap):
        res = Result(I, N)
        res.lc_round = np.zeros((I, N), np.uint32)
        res.committed = np.zeros((I, N, cap), np.int64)
        res.proposed = np.zeros((I, cap), np.int64)
        return res

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.ct_hostcore_last_error().decode()))

    def run(self, seeds, num_nodes, max_clock=1000, cap=128, first_seeds=None, **kw):
        """The CT core over a plain handle's host setup, then lbft_commit_times(cap); flags default to COMMIT_TIMES.  Also
        ``startup[instance, node]``, each node's startup time as the core holds it."""
        kw.setdefault("flags", FLAG_COMMIT_TIMES)
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        res = self._outputs(cfg.num_instances, num_nodes, cap)
        res.startup = np.zeros((cfg.num_instances, num_nodes), np.uint32)
        fs = None if first_seeds is None else np.ascontiguousarray(first_seeds, dtype=np.uint64)
        self._check(self.lib.ct_hostcore_run(ctypes.byref(cfg), None if fs is None else P(fs.ctypes.data), P(res.commit_counts.ctypes.data),
                                             P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data), P(res.counters.ctypes.data),
                                             P(res.status.ctypes.data), P(res.committed.ctypes.data), P(res.proposed.ctypes.data), cap,
                                             P(res.startup.ctypes.data)))
        return res

    def run_sweep(self, seeds, num_nodes, max_clock, sets, set_of, cap=128, **shared):
        shared.setdefault("flags", FLAG_COMMIT_TIMES)
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        res = self._outputs(cfg.num_instances, num_nodes, cap)
        self._check(self.lib.ct_hostcore_run_sweep(ctypes.byref(cfg), c_sets(sets), len(sets), P(so.ctypes.data), P(res.commit_counts.ctypes.data),
                                                   P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data), P(res.counters.ctypes.data),
                                                   P(res.status.ctypes.data), P(res.committed.ctypes.data), P(res.proposed.ctypes.data),
                                                   cap))
        return res

    def oracle(self, seeds, num_nodes, max_clock=1000, cap=128, first=0, count=None, **kw):
        """The oracle's commit times, laid out like lbft_commit_times; instances outside [first, first + count) stay 0."""
        kw.pop("flags", None)
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        I = cfg.num_instances
        count = I - first if count is None else count
        committed = np.zeros((I, num_nodes, cap), np.int64)
        proposed = np.zeros((I, cap), np.int64)
        counts = np.zeros((I, num_nodes), np.uint32)
        rc = self.lib.ct_oracle_commit_times(ctypes.byref(cfg), first, count, cap, P(committed.ctypes.data), P(proposed.ctypes.data),
                                             P(counts.ctypes.data))
        self._check(rc)
        return committed, proposed, counts
