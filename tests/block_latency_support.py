"""Test support for block-latency statistics (lbft_block_latency_stats): the ctypes wrapper of the host harness's
block_latency_hostcore_stats (tests/hostcore/block_latency_hostcore.cpp) and the same statistics computed with numpy from
commit times, by sorting each block's node times and finding where the cumulative voting rights reach the threshold.  Also the
threshold time alone over synthetic commit-time tables: adversarial tables (synthetic_cases), the serial block_threshold_time
on the host (BlockLatencyHarness.threshold_times) and its lane form on the device (BlockThresholdProbe,
tests/gpuprobe/block_threshold_probe.cu)."""
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
        self.lib.block_threshold_hostcore_times.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, P, P, P, P, P]

    def threshold_times(self, cc, times, weights, W):
        """block_threshold_time over a synthetic table (see synthetic_cases): T[I, round_cap], INT64_MAX where unreached."""
        I, N = cc.shape
        R = times.shape[2]
        cc, times = np.ascontiguousarray(cc, np.uint32), np.ascontiguousarray(times, np.int32)
        w, W = np.ascontiguousarray(weights, np.uint32), np.ascontiguousarray(W, np.uint64)
        T = np.zeros((I, R), np.int64)
        rc = self.lib.block_threshold_hostcore_times(N, I, R, P(cc.ctypes.data), P(times.ctypes.data), P(w.ctypes.data), P(W.ctypes.data),
                                                     P(T.ctypes.data))
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.ct_hostcore_last_error().decode()))
        return T

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


class BlockThresholdProbe:
    """The lane form of the threshold time (sim_core.cuh block_threshold_time_lanes) on the device, over the same synthetic
    tables as BlockLatencyHarness.threshold_times; needs a GPU to run, not to load."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_block_threshold_probe())
        self.lib.block_threshold_probe_last_error.restype = ctypes.c_char_p
        self.lib.block_threshold_probe.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, P, P, P, P, P]

    def threshold_times(self, cc, times, weights, W):
        I, N = cc.shape
        R = times.shape[2]
        cc, times = np.ascontiguousarray(cc, np.uint32), np.ascontiguousarray(times, np.int32)
        w, W = np.ascontiguousarray(weights, np.uint32), np.ascontiguousarray(W, np.uint32)
        T = np.zeros((I, R), np.int64)
        rc = self.lib.block_threshold_probe(N, I, R, P(cc.ctypes.data), P(times.ctypes.data), P(w.ctypes.data), P(W.ctypes.data),
                                            P(T.ctypes.data))
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.block_threshold_probe_last_error().decode()))
        return T


def numpy_threshold_times(cc, times, weights, W):
    """The reference of both: threshold_times per instance's threshold, row r committed by node n iff cc[i, n] > r."""
    I, N = cc.shape
    R = times.shape[2]
    committed = np.where(cc[:, :, None] > np.arange(R), times[:, :N, :].astype(np.int64), -1)
    T = np.full((I, R), INT64_MAX, np.int64)
    for w in np.unique(W):
        sel = W == w
        t, reached = threshold_times(committed[sel], weights, int(w))
        T[sel] = np.where(reached, t, INT64_MAX)
    return T


CAP = 1 << 24  # the largest voting right a node may hold


def synthetic_weights(N, rng):
    """(name, weights) per N: equal, random 0..3 with node 0 at zero, all at the 2^24 cap, and the cap on the top node and node 32
    over zeros and small weights."""
    small = rng.integers(0, 4, N)
    small[0] = 0
    if small.sum() == 0:
        small[-1] = 1
    top = np.where(np.arange(N) % 3 == 0, 0, 1 + np.arange(N) % 2)
    top[N - 1] = CAP
    if N > 32:
        top[32] = CAP
    return [("equal", np.ones(N, np.int64)), ("small", small.astype(np.int64)), ("cap", np.full(N, CAP, np.int64)), ("top", top)]


def synthetic_thresholds(weights, rng, sample=12):
    """Every threshold from 1 to total for N <= 8 with small weights; otherwise the named ones, total - 1, the heaviest weight and
    that + 1, the sums of the heaviest 1..N nodes and their neighbours, and a seeded sample."""
    total = int(weights.sum())
    if len(weights) <= 8 and total <= 64:
        return np.arange(1, total + 1)
    heavy = int(weights.max())
    prefix = np.cumsum(np.sort(weights)[::-1])
    cand = set(thresholds(total)) | {total - 1, heavy, heavy + 1}
    cand |= set(int(x) for x in rng.choice(np.concatenate([prefix - 1, prefix, prefix + 1]), min(sample, 3 * len(prefix)), replace=False))
    cand |= set(int(x) for x in rng.integers(1, total + 1, sample))
    return np.array(sorted(t for t in cand if 1 <= t <= total))


TIME_KINDS = ("tiny", "pairs", "one_clock", "wide")
CC_KINDS = ("full", "cut", "zero_weight_only", "only_node_32")


def synthetic_table(N, R, weights, time_kind, cc_kind, I, rng):
    """cc[I, N], times[I, N + 1, R] (row N, the proposed times, is zero).  time_kind: drawn from 0..1 (ties everywhere), 0..3, all
    nodes at one clock, or 0..9 999; cc_kind: every node commits every row, each node cut off at its own k in 0..R, only the
    zero-weight nodes commit (every row unreached), or only node 32 commits."""
    hi = {"tiny": 2, "pairs": 4, "one_clock": 1, "wide": 10000}[time_kind]
    times = np.zeros((I, N + 1, R), np.int32)
    times[:, :N, :] = rng.integers(0, hi, (I, N, R)) + (rng.integers(0, 1000, (I, 1, R)) if time_kind == "one_clock" else 0)
    if cc_kind == "full":
        cc = np.full((I, N), R)
    elif cc_kind == "cut":
        cc = rng.integers(0, R + 1, (I, N))
    elif cc_kind == "zero_weight_only":
        cc = np.where(weights == 0, R, 0)[None, :].repeat(I, axis=0)
    else:
        cc = np.where(np.arange(N) == 32, R, 0)[None, :].repeat(I, axis=0)
    return cc.astype(np.uint32), times


def synthetic_cases(N, rng, R=6, per_threshold=2):
    """(label, weights, cc, times, W) for every weight vector of synthetic_weights and every time and commit-count kind that
    applies at N; each threshold of synthetic_thresholds on per_threshold instances of each table kind."""
    out = []
    for wname, weights in synthetic_weights(N, rng):
        W = np.repeat(synthetic_thresholds(weights, rng), per_threshold)
        for time_kind in TIME_KINDS:
            for cc_kind in CC_KINDS:
                if (cc_kind == "zero_weight_only" and not (weights == 0).any()) or (cc_kind == "only_node_32" and N <= 32):
                    continue
                cc, times = synthetic_table(N, R, weights, time_kind, cc_kind, len(W), rng)
                out.append(("N=%d %s %s %s" % (N, wname, time_kind, cc_kind), weights, cc, times, W))
    return out
