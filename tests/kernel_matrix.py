"""The kernel matrix: one entry per event-loop kernel instantiation of the library (csrc/k_*.cu), keyed by the name
lbft_kernel_info gives it (host_setup.hpp kernel_name), with a configuration the product's own host setup sends to that
kernel.  tests/test_kernel_matrix.py checks on the CPU that the table names exactly the kernels the library carries and that
each entry selects its kernel; tests/test_gpu_kernel_matrix.py runs every entry on the GPU against the oracle.  This table is
the record of which kernels the GPU suite runs: a kernel added to a k_*.cu list needs an entry here.

The entries sit at the edges where these kernels go wrong: committees at the limits of the author-mask width (N = 16 on
NMAX 16, N = 17 / 32 on NMAX 32, N = 33 / 64 on NMAX 64, and N = 1 / 2), 8-lane groups over committees that are not a multiple
of 8, ragged batches (never a whole number of warps or tiles), a silent node on the top bit of the mask, and the extensions
(voting rights, partitions, uniform delays from 0, the constant delay, the exp() fallback of a wide LogNormal, a finite
target_commit_interval with other delta / gamma / lambda) rotated over the families and queue modes.

Epochs: the reference stalls at its first epoch change for committees of two or more (DESIGN §9: the leader that completes
the epoch swaps stores before its QC is broadcast), so only a lone author crosses several boundaries; the NMAX 16 epoch
entries run N = 1, the others reach the first boundary.
"""
import itertools
import re
from dataclasses import dataclass, field, replace

import numpy as np

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay
from librabft_simulator_b200._lib import FLAG_COMMIT_TIMES, FLAG_RESUMABLE, FLAG_ROUND_SWITCHES, FLAG_TRUE_DATA_SYNC

REC, RES, TDS, CT = FLAG_ROUND_SWITCHES, FLAG_RESUMABLE, FLAG_TRUE_DATA_SYNC, FLAG_COMMIT_TIMES
BIG_QUEUE = 0x10000  # an explicit queue_cap above the calendar queue's 0xfff0: the binary heap at any horizon


# ---- the extensions, in tests.support.make_config keywords ----
def weights(n):
    return dict(voting_rights=[1 + (i % 3) for i in range(n)])


def silent_top(n):
    """Node n - 1 silent: the top bit of the author mask at n = 16, 32, 64."""
    return dict(silent=[0] * (n - 1) + [1])


PART = dict(partition_windows=3, partition_max_len=120)
UNI0 = dict(delay_kind=1, delay_lo=0, delay_hi=12)
CONST = dict(delay_variance=0.0)
EXP = dict(delay_mean=25.0, delay_variance=200.0)  # too wide for a threshold table: the device evaluates exp()
TCI = dict(target_commit_interval=150, delta=30, gamma=1.5, lambda_=1.0)
TCI2 = dict(target_commit_interval=400, delta=12, gamma=1.0, lambda_=2.0)

# Parameter sets of the sweep entries: a finite target_commit_interval, the exp() fallback, uniform delays from 0 and the
# constant delay.  FAST_SETS makes the uniform set the fastest (mean 1 ms), which sizes a sweep's layout (host_setup.hpp
# build_sweep): the events per ms then rule out the compact queue entries.
SETS = (ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(200, 30, 1.5, 1.0)), ParamSet(RandomDelay.new(25.0, 200.0)),
        ParamSet(RandomDelay.uniform(0, 20)), ParamSet(RandomDelay.new(12.0, 0.0), NodeConfig(400, 12, 1.0, 2.0)))
# Sets that fit the tiny tables of TINY for 400 ms at N = 2.
TINY_SETS = (ParamSet(RandomDelay.new(10.0, 0.0)), ParamSet(RandomDelay.new(25.0, 200.0)),
             ParamSet(RandomDelay.uniform(5, 15), NodeConfig(300, 30, 1.5, 1.0)))
FAST_SETS = (ParamSet(RandomDelay.new(25.0, 200.0)), ParamSet(RandomDelay.uniform(0, 2)),
             ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig(150, 30, 1.5, 1.0)))


def fault_sets(n):
    """No faults, the top node silent, a partition plan with the first node silent."""
    return (FaultSet(), FaultSet((n - 1,)), FaultSet((0,), 3, 100))


@dataclass
class Entry:
    name: str
    kind: str                 # "plain", "sweep" or "faults" (a fault sweep)
    N: int
    I: int
    max_clock: int
    kw: dict = field(default_factory=dict)  # lbft_config fields (tests.support.make_config keywords), flags included
    force: str = None         # LBFT_FORCE_KERNEL, or None
    sets: tuple = ()          # sweeps: ParamSet per set (a fault sweep's carry their FaultSet)
    seed: int = 0             # seeds seed .. seed + I - 1

    @property
    def seeds(self):
        return np.arange(self.seed, self.seed + self.I, dtype=np.uint64)

    @property
    def set_of(self):
        """Sweeps: the set of each instance, interleaved rather than in blocks."""
        return (np.arange(self.I) * 7 // 3) % len(self.sets) if self.sets else None

    @property
    def flags(self):
        return self.kw.get("flags", 0)

    @property
    def per_warp(self):
        """Instances per warp of the entry's kernel: the thread kernel's tile, or 32 / lanes per instance."""
        m = re.search(r"wide_kernel<\d+,\d+,(?:true|false),(\d+)", self.name)
        return 32 // int(m.group(1)) if m else int(re.search(r"(\d+)>$", self.name).group(1))

    def oracle_cost(self):
        """Rough single-thread oracle seconds per instance (about 1 s per 64-author instance at 1 000 ms, DESIGN §6)."""
        return (self.N / 64.0) ** 2 * max(self.max_clock, 100) / 1000.0

    def oracle_instances(self, budget=3.0):
        """The instances the oracle checks: all of them when that fits `budget` single-thread seconds, else every instance of
        the first two warps (each lane position and group slot), the last, ragged warp, and a stride through the middle."""
        if self.I * self.oracle_cost() <= budget:
            return np.arange(self.I)
        w = self.per_warp
        last = (self.I - 1) // w * w
        middle = np.linspace(min(2 * w, last), last, num=max(2, min(24, int(budget / self.oracle_cost()) - 3 * w)), dtype=np.int64)
        return np.unique(np.concatenate([np.arange(min(2 * w, self.I)), middle, np.arange(last, self.I)]))


def ct_name(name):
    """The commit-times twin of a flag-off kernel name (None: the kernel has none)."""
    m = re.match(r"lbft_event_loop_kernel<(\d+),(\d+),(\d+),false,false,false,false,(\d+)>$", name)
    if m:
        return "lbft_ct_event_loop_kernel<%s,%s,%s,%s>" % m.groups()
    m = re.match(r"lbft_wide_kernel<(\d+),(\d+),(true|false),(\d+),false,(\d+)>$", name)
    if m:
        return "lbft_ct_wide_kernel<%s,%s,%s,%s,%s>" % m.groups()
    m = re.match(r"lbft_sweep_(event_loop|wide)_kernel<(.*)>$", name)
    return "lbft_ct_sweep_%s_kernel<%s>" % m.groups() if m else None


def _t(nmax, qm, rec=False, res=False, ep=False, tds=False, tile=32, fx=0):
    b = lambda v: "true" if v else "false"  # noqa: E731
    return "lbft_event_loop_kernel<%d,%d,%d,%s,%s,%s,%s,%d>" % (nmax, qm, fx, b(rec), b(res), b(ep), b(tds), tile)


def _w(nmax, qm, group, smem=False, ep=False, fx=0):
    return "lbft_wide_kernel<%d,%d,%s,%d,%s,%d>" % (nmax, qm, "true" if smem else "false", group, "true" if ep else "false", fx)


def _p(name, N, I, max_clock, force=None, **kw):
    return Entry(name, "plain", N, I, max_clock, kw, force)


def _s(name, N, I, max_clock, force=None, sets=SETS, faults=False, **kw):
    if faults:
        sets = tuple(ParamSet(p.network_delay, p.node_config, f) for p, f in zip(sets, itertools.cycle(fault_sets(N))))
    return Entry(name, "faults" if faults else "sweep", N, I, max_clock, kw, force, sets)


# The tiny tables that put a whole 8-lane instance in shared memory (host_setup.hpp select_kernel: 16 instances' state per SM);
# a committee of two commits several blocks in 400 ms within them.
TINY = dict(round_cap=32, queue_cap=32, payload_cap=12)

_BASE = [
    # ---- thread kernels, shared-memory scan queue (QMODE 2): committees of <= 5 ----
    _p(_t(16, 2, fx=1), 4, 4097, 700, **weights(4)),                                     # the bench kernel's compile-time layout
    _p(_t(16, 2), 2, 4097, 1000, **UNI0),
    _p(_t(16, 2, rec=True), 3, 65, 1000, queue_cap=64, flags=REC, **CONST),
    _p(_t(16, 2, res=True), 3, 70, 1000, queue_cap=64, flags=RES, **EXP),
    _p(_t(16, 2, rec=True, res=True), 2, 33, 1000, queue_cap=64, flags=REC | RES, **TCI),
    _p(_t(16, 2, ep=True), 1, 4097, 50, round_cap=32, queue_cap=16, commands_per_epoch=11, **PART),
    _p(_t(16, 2, tds=True), 3, 97, 1000, flags=TDS, **weights(3)),
    # ---- thread kernels, HBM scan queue (QMODE 1) ----
    _p(_t(16, 1), 5, 4127, 400, **PART),
    _p(_t(16, 1, rec=True), 4, 33, 1000, flags=REC, **UNI0),
    _p(_t(16, 1, res=True), 5, 40, 1000, flags=RES, **weights(5)),
    _p(_t(16, 1, rec=True, res=True), 2, 35, 1000, flags=REC | RES, **CONST),
    _p(_t(16, 1, ep=True), 1, 65, 60, "thread", queue_cap=200, commands_per_epoch=5, **EXP),
    _p(_t(16, 1, tds=True), 5, 65, 1000, flags=TDS, **TCI),
    # ---- thread kernels, calendar queue (QMODE 3): sparse tiles, then full tiles at NMAX 16 / 32 / 64 ----
    _p(_t(16, 3, tile=8), 9, 12289, 200, **TCI2),
    _p(_t(16, 3, tile=16), 16, 24577, 400, **CONST, **silent_top(16)),
    _p(_t(16, 3, tile=8, fx=2), 7, 16385, 1000, partition_windows=4, partition_max_len=150, **weights(7)),
    _p(_t(16, 3), 6, 49153, 150, **UNI0),
    _p(_t(16, 3, rec=True), 16, 33, 300, flags=REC, **PART),
    _p(_t(16, 3, res=True), 6, 40, 500, flags=RES, **CONST),
    _p(_t(16, 3, rec=True, res=True), 9, 33, 400, flags=REC | RES, **EXP),
    _p(_t(16, 3, ep=True), 1, 40, 60, "thread", queue_cap=600, commands_per_epoch=5, **TCI),
    _p(_t(16, 3, tds=True), 16, 40, 300, flags=TDS, **weights(16), **silent_top(16)),
    _p(_t(32, 3), 17, 65, 400, "thread", **PART),
    _p(_t(32, 3, rec=True), 32, 33, 300, flags=REC, **weights(32), **silent_top(32)),
    _p(_t(32, 3, res=True), 17, 34, 200, flags=RES, **UNI0),
    _p(_t(32, 3, rec=True, res=True), 20, 33, 300, flags=REC | RES, **CONST),
    _p(_t(32, 3, ep=True), 17, 33, 400, "thread", commands_per_epoch=4, **UNI0),
    _p(_t(32, 3, tds=True), 32, 33, 150, flags=TDS, **TCI),
    _p(_t(64, 3), 64, 33, 400, "thread", **weights(64), **silent_top(64)),
    _p(_t(64, 3, rec=True), 33, 33, 400, flags=REC, **PART),
    _p(_t(64, 3, res=True), 64, 33, 100, flags=RES, **UNI0),
    _p(_t(64, 3, rec=True, res=True), 33, 33, 400, flags=REC | RES, **CONST),
    _p(_t(64, 3, ep=True), 33, 33, 250, "thread", commands_per_epoch=3, **TCI),
    _p(_t(64, 3, tds=True), 33, 33, 600, flags=TDS, **EXP),
    # ---- thread kernels, binary heap (QMODE 0): horizons past 4 095 ms, or a queue_cap above the calendar's ----
    _p(_t(16, 0), 7, 33, 4200, "thread", **UNI0),
    _p(_t(16, 0, rec=True), 16, 33, 4100, flags=REC, **weights(16), **silent_top(16)),
    _p(_t(16, 0, res=True), 3, 40, 4500, queue_cap=600, flags=RES, **PART),
    _p(_t(16, 0, rec=True, res=True), 8, 33, 4096, flags=REC | RES, **CONST),
    _p(_t(16, 0, ep=True), 1, 40, 60, "thread", queue_cap=BIG_QUEUE, commands_per_epoch=5, **EXP),
    _p(_t(16, 0, tds=True), 5, 33, 4200, queue_cap=1024, flags=TDS, **TCI),
    _p(_t(32, 0), 17, 33, 4100, "thread", **weights(17)),
    _p(_t(32, 0, rec=True), 32, 33, 400, queue_cap=BIG_QUEUE, flags=REC, **PART, **silent_top(32)),
    _p(_t(32, 0, res=True), 20, 33, 300, queue_cap=BIG_QUEUE, flags=RES, **UNI0),
    _p(_t(32, 0, rec=True, res=True), 17, 9, 4100, flags=REC | RES, **CONST),
    _p(_t(32, 0, ep=True), 24, 33, 400, "thread", queue_cap=BIG_QUEUE, commands_per_epoch=5, **UNI0),
    _p(_t(32, 0, tds=True), 32, 33, 150, queue_cap=BIG_QUEUE, flags=TDS, **TCI),
    _p(_t(64, 0), 33, 5, 4100, "thread", **weights(33)),
    _p(_t(64, 0, rec=True), 64, 33, 400, queue_cap=BIG_QUEUE, flags=REC, **PART, **silent_top(64)),
    _p(_t(64, 0, res=True), 40, 33, 120, queue_cap=BIG_QUEUE, flags=RES, **UNI0),
    _p(_t(64, 0, rec=True, res=True), 64, 33, 400, queue_cap=BIG_QUEUE, flags=REC | RES, **CONST),
    _p(_t(64, 0, ep=True), 33, 33, 250, "thread", queue_cap=BIG_QUEUE, commands_per_epoch=3, **TCI),
    _p(_t(64, 0, tds=True), 48, 33, 600, queue_cap=BIG_QUEUE, payload_cap=8192, flags=TDS, **EXP),
    # ---- wide kernels: the instance in shared memory, the compile-time 64-author layout ----
    _p(_w(16, 2, 8, smem=True), 2, 4097, 400, "wide", **TINY),
    _p(_w(16, 2, 32, smem=True), 4, 1000, 1000, **UNI0),
    _p(_w(64, 3, 8, fx=3), 64, 4097, 1000, **weights(64), **silent_top(64)),
    # ---- wide kernels, state in HBM: 8 / 32 lanes and the epoch variant per queue mode and mask width ----
    _p(_w(16, 2, 8), 7, 4097, 400, **PART, **CONST),
    _p(_w(16, 2, 32), 9, 300, 500, **EXP),
    _p(_w(16, 2, 32, ep=True), 1, 64, 60, commands_per_epoch=5, **TCI, **weights(1)),
    _p(_w(16, 1, 8), 5, 4097, 16400, "wide", **CONST, **weights(5)),
    _p(_w(16, 1, 32), 4, 200, 16400, **EXP, **PART),
    _p(_w(16, 1, 32, ep=True), 5, 40, 1000, delay_kind=1, delay_lo=0, delay_hi=2, commands_per_epoch=4, **TCI),
    _p(_w(16, 3, 8), 12, 4097, 200, **TCI),
    _p(_w(16, 3, 32), 16, 100, 300, **CONST, **silent_top(16)),
    _p(_w(16, 3, 32, ep=True), 1, 40, 60, queue_cap=1100, commands_per_epoch=5, **UNI0, **PART),
    _p(_w(32, 3, 8), 17, 4097, 100, **UNI0),
    _p(_w(32, 3, 32), 32, 64, 150, **weights(32), **silent_top(32)),
    _p(_w(32, 3, 32, ep=True), 25, 33, 600, commands_per_epoch=4, **CONST),
    _p(_w(64, 3, 8), 33, 4097, 400, **CONST),
    _p(_w(64, 3, 32), 64, 20, 600, **EXP, **silent_top(64)),
    _p(_w(64, 3, 32, ep=True), 40, 17, 200, commands_per_epoch=3, **TCI),
    _p(_w(16, 0, 8), 9, 4097, 600, queue_cap=BIG_QUEUE, **EXP, **PART),
    _p(_w(16, 0, 32), 8, 33, 4200, **TCI),
    _p(_w(16, 0, 32, ep=True), 1, 34, 60, queue_cap=BIG_QUEUE, commands_per_epoch=5, **CONST),
    _p(_w(32, 0, 8), 20, 4097, 400, queue_cap=BIG_QUEUE, **TCI2),
    _p(_w(32, 0, 32), 32, 3, 4100, **CONST, **silent_top(32)),
    _p(_w(32, 0, 32, ep=True), 18, 33, 300, queue_cap=BIG_QUEUE, commands_per_epoch=4, **weights(18)),
    _p(_w(64, 0, 8), 33, 4097, 80, queue_cap=BIG_QUEUE, **UNI0),
    _p(_w(64, 0, 32), 64, 9, 600, queue_cap=BIG_QUEUE, **EXP, **silent_top(64)),
    _p(_w(64, 0, 32, ep=True), 33, 17, 400, queue_cap=BIG_QUEUE, commands_per_epoch=3, **CONST),
    # ---- sweep thread kernels ----
    _s("lbft_sweep_event_loop_kernel<16,3,8>", 10, 12289, 200),
    _s("lbft_sweep_event_loop_kernel<16,3,16>", 16, 24577, 400, faults=True),
    _s("lbft_sweep_event_loop_kernel<16,2,32>", 3, 4097, 1000, sets=SETS[:3], **weights(3)),
    _s("lbft_sweep_event_loop_kernel<16,1,32>", 5, 4097, 300, faults=True),
    _s("lbft_sweep_event_loop_kernel<16,3,32>", 16, 65, 300, "thread", faults=True),
    _s("lbft_sweep_event_loop_kernel<32,3,32>", 17, 33, 200, "thread", **weights(17)),
    _s("lbft_sweep_event_loop_kernel<64,3,32>", 64, 33, 400, "thread", faults=True),
    _s("lbft_sweep_event_loop_kernel<16,0,32>", 7, 33, 4200, "thread"),
    _s("lbft_sweep_event_loop_kernel<32,0,32>", 32, 33, 400, "thread", queue_cap=BIG_QUEUE, faults=True),
    _s("lbft_sweep_event_loop_kernel<64,0,32>", 33, 33, 400, "thread", queue_cap=BIG_QUEUE),
    # ---- sweep wide kernels ----
    _s("lbft_sweep_wide_kernel<16,2,true,8>", 2, 4097, 400, "wide", sets=TINY_SETS, **TINY),
    _s("lbft_sweep_wide_kernel<16,2,true,32>", 4, 1000, 1000, faults=True),
    _s("lbft_sweep_wide_kernel<16,2,false,8>", 7, 4097, 400, faults=True),
    _s("lbft_sweep_wide_kernel<16,2,false,32>", 9, 300, 500),
    _s("lbft_sweep_wide_kernel<16,1,false,8>", 5, 4097, 1000, "wide", sets=FAST_SETS, round_cap=512),
    _s("lbft_sweep_wide_kernel<16,1,false,32>", 4, 200, 16400, faults=True),
    _s("lbft_sweep_wide_kernel<16,3,false,8>", 12, 4097, 200, faults=True),
    _s("lbft_sweep_wide_kernel<16,3,false,32>", 16, 100, 300, faults=True),
    _s("lbft_sweep_wide_kernel<32,3,false,8>", 17, 4097, 400),
    _s("lbft_sweep_wide_kernel<32,3,false,32>", 32, 64, 400, faults=True),
    _s("lbft_sweep_wide_kernel<64,3,false,8>", 33, 4097, 400, **weights(33)),
    _s("lbft_sweep_wide_kernel<64,3,false,32>", 64, 20, 400, faults=True),
    _s("lbft_sweep_wide_kernel<16,0,false,8>", 9, 4097, 200, queue_cap=BIG_QUEUE),
    _s("lbft_sweep_wide_kernel<16,0,false,32>", 8, 33, 4200, faults=True),
    _s("lbft_sweep_wide_kernel<32,0,false,8>", 20, 4097, 400, queue_cap=BIG_QUEUE, faults=True),
    _s("lbft_sweep_wide_kernel<32,0,false,32>", 32, 5, 4100),
    _s("lbft_sweep_wide_kernel<64,0,false,8>", 33, 4097, 400, queue_cap=BIG_QUEUE),
    _s("lbft_sweep_wide_kernel<64,0,false,32>", 64, 9, 400, queue_cap=BIG_QUEUE, faults=True),
]


def _twins(base):
    """The commit-times twin of every entry whose kernel has one: the same configuration with LBFT_FLAG_COMMIT_TIMES."""
    out = []
    for e in base:
        name = ct_name(e.name)
        if name:
            out.append(replace(e, name=name, kw=dict(e.kw, flags=e.flags | CT)))
    return out


def _seeded(entries):
    """Distinct seeds per entry (a twin keeps its flag-off entry's, so that their outputs can be compared)."""
    seeds, out = {}, []
    for e in entries:
        key = ct_name(e.name) or e.name
        seeds.setdefault(key, 1000 + 7919 * len(seeds))
        out.append(replace(e, seed=seeds[key]))
    return out


_ENTRIES = _seeded(_BASE + _twins(_BASE))
MATRIX = {e.name: e for e in _ENTRIES}
assert len(MATRIX) == len(_ENTRIES), "duplicate kernel name in the matrix"


def flag_off(entry):
    """The flag-off entry a commit-times twin is the twin of."""
    return next(e for e in _ENTRIES if ct_name(e.name) == entry.name)
