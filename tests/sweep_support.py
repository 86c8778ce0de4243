"""Test support for sweep handles (lbft_create_sweep): the host-compiled SW core (tests/hostcore) and the oracle run once per
parameter set over that set's instances, which is what a sweep must reproduce instance by instance."""
import ctypes

import numpy as np

from librabft_simulator_b200 import NodeConfig, ParamSet, RandomDelay, _build
from librabft_simulator_b200._lib import LbftConfig, LbftParamSet
from tests.support import P, Result, make_config

# Twelve parameter sets: LogNormal delays of several means and variances (variance 0 = the host-evaluated constant delay;
# LogNormal(25, 200) is too wide for a threshold table and takes the exp() path; LogNormal(15, 30) has ~2 000 thresholds, more
# than a thread kernel keeps in shared memory), two uniform delays, and varied delta / gamma / lambda / target_commit_interval.
SETS = [
    ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig()),
    ParamSet(RandomDelay.new(5.0, 2.0), NodeConfig()),
    ParamSet(RandomDelay.new(20.0, 10.0), NodeConfig()),
    ParamSet(RandomDelay.new(10.0, 0.0), NodeConfig()),
    ParamSet(RandomDelay.new(25.0, 200.0), NodeConfig()),
    ParamSet(RandomDelay.new(15.0, 30.0), NodeConfig()),
    ParamSet(RandomDelay.uniform(1, 4), NodeConfig()),
    ParamSet(RandomDelay.uniform(5, 15), NodeConfig()),
    ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(delta=15, gamma=1.5, lambda_=1.0)),
    ParamSet(RandomDelay.new(8.0, 3.0), NodeConfig(target_commit_interval=300, delta=100)),
    ParamSet(RandomDelay.new(4.0, 1.0), NodeConfig(delta=30, gamma=1.0)),
    ParamSet(RandomDelay.new(12.0, 6.0), NodeConfig(delta=10, lambda_=2.0)),
]


def set_kwargs(ps):
    """The lbft_config fields (tests.support.make_config keywords) a parameter set stands for."""
    d, n = ps.network_delay, ps.node_config
    return dict(delay_kind=d.kind, delay_mean=d.mean, delay_variance=d.variance, delay_lo=d.lo, delay_hi=d.hi,
                target_commit_interval=n.target_commit_interval, delta=n.delta, gamma=n.gamma, lambda_=n.lambda_)


def c_sets(sets):
    return (LbftParamSet * max(1, len(sets)))(*[p.to_c() for p in sets])


def oracle_per_set(oracle, seeds, num_nodes, max_clock, sets, set_of, **shared):
    """The oracle run once per set over the instances assigned to it, gathered back into instance order."""
    seeds, set_of = np.asarray(seeds, dtype=np.uint64), np.asarray(set_of)
    out = Result(len(seeds), num_nodes)
    for s, ps in enumerate(sets):
        idx = np.nonzero(set_of == s)[0]
        if len(idx) == 0:
            continue
        kw = dict(shared)
        kw.update(set_kwargs(ps))
        r = oracle.run(seeds[idx], num_nodes, max_clock, **kw)
        out.commit_counts[idx], out.last_states[idx], out.counters[idx], out.status[idx] = r.commit_counts, r.last_states, r.counters, r.status
    return out


class SweepHostCore:
    """hostcore_run_sweep / hostcore_kernel_info_sweep of tests/hostcore/sweep_hostcore.cpp (the SW core through the
    product's host setup)."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_sweep_hostcore())
        self.lib.hostcore_sweep_last_error.restype = ctypes.c_char_p
        self.lib.hostcore_run_sweep.argtypes = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.c_uint32, P,
                                                P, P, P, P, P, ctypes.POINTER(ctypes.c_uint32)]
        self.lib.hostcore_kernel_info_sweep.argtypes = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.c_uint32, P,
                                                        ctypes.c_char_p, ctypes.c_size_t]

    def run(self, seeds, num_nodes, max_clock, sets, set_of, **shared):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        w = ctypes.c_uint32()
        rc = self.lib.hostcore_run_sweep(ctypes.byref(cfg), c_sets(sets), len(sets), P(so.ctypes.data), P(res.commit_counts.ctypes.data),
                                         P(res.last_states.ctypes.data), P(res.lc_round.ctypes.data), P(res.counters.ctypes.data),
                                         P(res.status.ctypes.data), ctypes.byref(w))
        if rc != 0:
            raise RuntimeError(self.lib.hostcore_sweep_last_error().decode())
        res.words_per_instance = w.value
        return res

    def kernel_info(self, seeds, num_nodes, max_clock, sets, set_of, **shared):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **shared)
        so = np.ascontiguousarray(set_of, dtype=np.uint32)
        buf = ctypes.create_string_buffer(128)
        if self.lib.hostcore_kernel_info_sweep(ctypes.byref(cfg), c_sets(sets), len(sets), P(so.ctypes.data), buf, ctypes.sizeof(buf)) != 0:
            raise RuntimeError(self.lib.hostcore_sweep_last_error().decode())
        return buf.value.decode()


# The kernel a sweep handle of each tests/test_hostcore_parity.py::test_kernel_choice case runs (one set with the reference
# delay; the recording / resumable cases are plain handles only): automatic, and forced to each family.
KERNEL_CASES = (("config2", 1024, 4, {}), ("config3", 65536, 4, {}), ("config5", 16384, 7, {}),
                ("config5p", 16384, 7, {"partition_windows": 4, "partition_max_len": 150}),
                ("mid7", 8192, 7, {}), ("full7", 65536, 7, {}), ("big64", 8192, 64, {}),
                ("small64", 64, 64, {}), ("mid4", 8192, 4, {}), ("long7", 64, 7, {"max_clock": 20000}))
SWEEP_PICKS = {
    None: {"config2": "lbft_sweep_wide_kernel<16,2,true,32>", "config3": "lbft_sweep_event_loop_kernel<16,2,32>",
           "config5": "lbft_sweep_event_loop_kernel<16,3,8>", "config5p": "lbft_sweep_event_loop_kernel<16,3,8>",
           "mid7": "lbft_sweep_wide_kernel<16,2,false,8>", "full7": "lbft_sweep_event_loop_kernel<16,3,32>",
           "big64": "lbft_sweep_wide_kernel<64,3,false,8>", "small64": "lbft_sweep_wide_kernel<64,3,false,32>",
           "mid4": "lbft_sweep_event_loop_kernel<16,2,32>", "long7": "lbft_sweep_wide_kernel<16,0,false,32>"},
    "thread": {"config2": "lbft_sweep_event_loop_kernel<16,2,32>", "config3": "lbft_sweep_event_loop_kernel<16,2,32>",
               "config5": "lbft_sweep_event_loop_kernel<16,3,32>", "config5p": "lbft_sweep_event_loop_kernel<16,3,32>",
               "mid7": "lbft_sweep_event_loop_kernel<16,3,32>", "full7": "lbft_sweep_event_loop_kernel<16,3,32>",
               "big64": "lbft_sweep_event_loop_kernel<64,3,32>", "small64": "lbft_sweep_event_loop_kernel<64,3,32>",
               "mid4": "lbft_sweep_event_loop_kernel<16,2,32>", "long7": "lbft_sweep_event_loop_kernel<16,0,32>"},
    "wide": {"config2": "lbft_sweep_wide_kernel<16,2,true,32>", "config3": "lbft_sweep_wide_kernel<16,2,false,8>",
             "config5": "lbft_sweep_wide_kernel<16,2,false,8>", "config5p": "lbft_sweep_wide_kernel<16,2,false,8>",
             "mid7": "lbft_sweep_wide_kernel<16,2,false,8>", "full7": "lbft_sweep_wide_kernel<16,2,false,8>",
             "big64": "lbft_sweep_wide_kernel<64,3,false,8>", "small64": "lbft_sweep_wide_kernel<64,3,false,32>",
             "mid4": "lbft_sweep_wide_kernel<16,2,false,8>", "long7": "lbft_sweep_wide_kernel<16,0,false,32>"},
}
