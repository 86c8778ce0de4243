"""Test support for block-latency statistics (lbft_block_latency_stats): the ctypes wrapper of the host harness's
block_latency_hostcore_stats (tests/hostcore/block_latency_hostcore.cpp) and the same statistics computed with numpy from
commit times, by sorting each block's node times and finding where the cumulative voting rights reach the threshold."""
import ctypes

import numpy as np

from librabft_simulator_b200 import BlockLatencyStats, _build
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, ST_ERROR_MASK, LbftConfig, LbftFaultSet, LbftLatencySpec, LbftParamSet
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE, resolve_threshold
from tests.fault_support import c_faults
from tests.latency_support import INT64_MAX, assert_same_stats, make_spec
from tests.support import P, make_config
from tests.sweep_support import c_sets

THRESHOLD_NAMES = ["first", "validity", "quorum", "all"]


def thresholds(total):
    """The named thresholds and one arbitrary value strictly between validity and quorum (or next to one of them when the
    committee is too small for that), as integers."""
    named = [resolve_threshold(t, total) for t in THRESHOLD_NAMES]
    between = max(1, min(total, (named[1] + named[2]) // 2 + (1 if named[2] - named[1] > 2 else 0)))
    return named + [between]


class BlockLatencyHarness:
    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_block_latency_hostcore())
        self.lib.ct_hostcore_last_error.restype = ctypes.c_char_p
        self.lib.block_latency_hostcore_stats.argtypes = [
            ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.POINTER(LbftFaultSet), ctypes.c_uint32, P,
            ctypes.POINTER(LbftLatencySpec), ctypes.c_uint64, P, P, P, ctypes.c_size_t, P, P, P]

    def run(self, seeds, num_nodes, max_clock=1000, threshold=1, spec=None, sets=None, set_of=None, faults=False, cap=256, **kw):
        """(BlockLatencyStats, status, committed[I, N, cap], proposed[I, cap]) of the CT core over a plain (sets=None), sweep or
        (faults=True: each set's FaultSet) fault-sweep handle's host setup; flags default to COMMIT_TIMES."""
        kw.setdefault("flags", FLAG_COMMIT_TIMES)
        spec = make_spec() if spec is None else spec
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        I = cfg.num_instances
        groups = 1 if sets is None else len(sets)
        so = None if set_of is None else np.ascontiguousarray(set_of, dtype=np.uint32)
        status = np.zeros(I, np.uint32)
        committed = np.zeros((I, num_nodes, cap), np.int64)
        proposed = np.zeros((I, cap), np.int64)
        out = np.zeros(groups, LATENCY_SUMMARY_DTYPE)
        unreached = np.zeros(groups, np.uint64)
        valid = 1 <= spec.num_bins <= 1 << 16 and groups * spec.num_bins <= 1 << 24  # (else the harness refuses: no histogram)
        hist = np.zeros((groups, spec.num_bins if valid else 0), np.uint64)
        rc = self.lib.block_latency_hostcore_stats(
            ctypes.byref(cfg), None if sets is None else c_sets(sets), c_faults(sets) if faults else None, 0 if sets is None else len(sets),
            None if so is None else P(so.ctypes.data), ctypes.byref(spec), threshold, P(status.ctypes.data), P(committed.ctypes.data),
            P(proposed.ctypes.data), cap, P(out.ctypes.data), P(unreached.ctypes.data), P(hist.ctypes.data) if valid else None)
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.ct_hostcore_last_error().decode()))
        return BlockLatencyStats(out, unreached, hist, spec.bin_width, threshold), status, committed, proposed


def threshold_times(committed, weights, threshold):
    """(T[I, cap], reached[I, cap]): per block (row k of each instance), the least commit time at which the voting rights of the
    nodes that committed it at or before that time reach the threshold; committed[I, N, cap] is -1 where a node did not commit."""
    never = np.iinfo(np.int64).max
    t = np.where(committed >= 0, committed, never)
    order = np.argsort(t, axis=1, kind="stable")
    ts = np.take_along_axis(t, order, axis=1)
    cum = np.cumsum(np.asarray(weights, dtype=np.int64)[order], axis=1)
    hit = (cum >= threshold) & (ts < never)
    first = np.argmax(hit, axis=1)
    return np.take_along_axis(ts, first[:, None, :], axis=1)[:, 0, :], hit.any(axis=1)


def numpy_block_stats(committed, proposed, status, group_of, groups, weights, threshold, num_bins=1024, bin_width=1, proposed_from=0,
                      proposed_until=None):
    """The statistics of lbft_block_latency_stats from full-cap commit times (committed[I, N, cap], proposed[I, cap])."""
    until = INT64_MAX if proposed_until is None else proposed_until
    group_of = np.asarray(group_of, dtype=np.int64)
    clean = (status & np.uint32(ST_ERROR_MASK)) == 0
    on_chain = (committed >= 0).any(axis=1)  # a row some node committed
    blocks = on_chain & clean[:, None] & (proposed >= proposed_from) & (proposed < until)
    T, reached = threshold_times(committed, weights, threshold)
    g_all = np.broadcast_to(group_of[:, None], blocks.shape)
    ok = blocks & reached
    g, x = g_all[ok], (T - proposed)[ok]
    out = np.zeros(groups, LATENCY_SUMMARY_DTYPE)
    out["instances"] = np.bincount(group_of[clean], minlength=groups)
    out["excluded"] = np.bincount(group_of[~clean], minlength=groups)
    out["samples"] = np.bincount(g, minlength=groups)
    s = np.zeros(groups, np.uint64)
    np.add.at(s, g, x.astype(np.uint64))
    out["sum"] = s
    lo = np.full(groups, INT64_MAX, np.int64)
    hi = np.full(groups, -1, np.int64)
    np.minimum.at(lo, g, x)
    np.maximum.at(hi, g, x)
    out["min"] = np.where(out["samples"] > 0, lo, -1)
    out["max"] = hi
    unreached = np.bincount(g_all[blocks & ~reached], minlength=groups).astype(np.uint64)
    b = np.minimum(x // bin_width, num_bins - 1)
    hist = np.bincount(g * num_bins + b, minlength=groups * num_bins).astype(np.uint64).reshape(groups, num_bins)
    return BlockLatencyStats(out, unreached, hist, bin_width, threshold)


def assert_same_block_stats(a, b, msg=""):
    assert_same_stats(a, b, msg)
    np.testing.assert_array_equal(a.unreached, b.unreached, err_msg="%s unreached" % msg)
    assert a.threshold == b.threshold, msg
