"""Test support for commit-latency statistics (lbft_latency_stats): the ctypes wrapper of the host harness's
latency_hostcore_stats (tests/hostcore/latency_hostcore.cpp) and the same statistics computed with numpy from commit times."""
import ctypes

import numpy as np

from librabft_simulator_b200 import _build
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, ST_ERROR_MASK, LbftConfig, LbftLatencySpec, LbftParamSet
from librabft_simulator_b200.simulator import LATENCY_SUMMARY_DTYPE, LatencyStats
from tests.support import P, make_config
from tests.sweep_support import c_sets

INT64_MAX = np.iinfo(np.int64).max
# (num_bins, bin_width): one-ms bins, an overflow bin that fills, a single bin
BIN_SETTINGS = [(1024, 1), (5, 7), (1, 1)]
# (proposed_from, proposed_until): empty, everything, and a middle window that leaves out warm-up and the truncated tail
WINDOWS = [(500, 500), (0, None), (200, 800)]


def make_spec(num_bins=1024, bin_width=1, proposed_from=0, proposed_until=None):
    return LbftLatencySpec(struct_size=ctypes.sizeof(LbftLatencySpec), num_bins=num_bins, bin_width=bin_width,
                           proposed_from=proposed_from, proposed_until=INT64_MAX if proposed_until is None else proposed_until)


class LatencyHarness:
    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_latency_hostcore())
        self.lib.ct_hostcore_last_error.restype = ctypes.c_char_p
        self.lib.latency_hostcore_stats.argtypes = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.c_uint32, P,
                                                       ctypes.POINTER(LbftLatencySpec), P, P, P]

    def run(self, seeds, num_nodes, max_clock=1000, spec=None, sets=None, set_of=None, **kw):
        """(LatencyStats, status) of the CT core over a plain (sets=None) or sweep handle's host setup; flags default to
        COMMIT_TIMES."""
        kw.setdefault("flags", FLAG_COMMIT_TIMES)
        spec = make_spec() if spec is None else spec
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        groups = 1 if sets is None else len(sets)
        so = None if set_of is None else np.ascontiguousarray(set_of, dtype=np.uint32)
        status = np.zeros(cfg.num_instances, np.uint32)
        out = np.zeros(groups, LATENCY_SUMMARY_DTYPE)
        valid = 1 <= spec.num_bins <= 1 << 16 and groups * spec.num_bins <= 1 << 24  # (else the harness refuses: no histogram)
        hist = np.zeros((groups, spec.num_bins if valid else 0), np.uint64)
        rc = self.lib.latency_hostcore_stats(ctypes.byref(cfg), None if sets is None else c_sets(sets), 0 if sets is None else len(sets),
                                                None if so is None else P(so.ctypes.data), ctypes.byref(spec), P(status.ctypes.data),
                                                P(out.ctypes.data), P(hist.ctypes.data) if valid else None)
        if rc != 0:
            raise RuntimeError("%d: %s" % (rc, self.lib.ct_hostcore_last_error().decode()))
        return LatencyStats(out, hist, spec.bin_width), status


def numpy_stats(committed, proposed, status, group_of, groups, num_bins=1024, bin_width=1, proposed_from=0, proposed_until=None):
    """The statistics of lbft_latency_stats from full-cap commit times (committed[I, N, cap], proposed[I, cap]) with numpy."""
    until = INT64_MAX if proposed_until is None else proposed_until
    group_of = np.asarray(group_of, dtype=np.int64)
    clean = (status & np.uint32(ST_ERROR_MASK)) == 0
    lat = committed - proposed[:, None, :]
    in_window = (proposed >= proposed_from) & (proposed < until)
    valid = (committed >= 0) & clean[:, None, None] & in_window[:, None, :]
    g = np.broadcast_to(group_of[:, None, None], lat.shape)[valid]
    x = lat[valid]
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
    b = np.minimum(x // bin_width, num_bins - 1)
    hist = np.bincount(g * num_bins + b, minlength=groups * num_bins).astype(np.uint64).reshape(groups, num_bins)
    return LatencyStats(out, hist, bin_width)


def assert_same_stats(a, b, msg=""):
    for f in LATENCY_SUMMARY_DTYPE.names + ("hist",):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg="%s %s" % (msg, f))
    assert a.bin_width == b.bin_width
