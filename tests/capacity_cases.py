"""The capacity-edge cases: one entry per (kernel, capacity) whose run at a tight capacity C puts some instances exactly at C
and others one past it.  tests/test_capacity_edges.py checks the table and runs it on the host-compiled core;
tests/test_gpu_capacity_edges.py runs every case on the GPU.

Each case is run twice: A with the generous capacities of `kw`, then B with the capacity under test set to a C derived from
A (tight()): for the queue and the payload pool a peak (counters[:, 8] max_queue / counters[:, 10] max_payloads) that some
instance of A reaches exactly, with at least 15 % of the instances on each side of it; for the round tables a multiple of 32
that some instance of A completes at active round C - 1 while others reach C.  Two payload cases pin C instead: 32, the top
of the register bitmask allocator, and 33, the first free-list capacity.  Every case selects its named kernel at both
capacities, and the capacities it gets are the ones requested (no read-out floor raises them).

Two kinds of case run clean at one capacity and are compared with the oracle instead: the read-out floor (queue_cap equal
to sim_params.h readout_queue_floor for each queue mode, with commit logs close to round_cap rows, so finalize()'s chain
scratch spans the whole queue area it borrows) and the horizon edges (max_clock 4 095 on the calendar queue: events at
t == max_clock take the last time slot and occupancy word; max_clock 16 319 on the wide kernel's compact keys, the top of
their 14-bit time field).
"""
import re
from dataclasses import dataclass, field

import numpy as np

from librabft_simulator_b200 import NodeConfig, ParamSet, RandomDelay
from tests.kernel_matrix import CT, REC, RES, _t, _w, ct_name

CAP_FIELD = {"queue": "queue_cap", "payload": "payload_cap", "round": "round_cap"}
PEAK_COLUMN = {"queue": 8, "payload": 10}  # lbft_instance_counters max_queue, max_payloads
# the creation-stamp limit of each queue mode (sim_core.cuh kStampLimit): 0 heap, 1 HBM scan, 2 shared-memory scan, 3 calendar
STAMP_LIMIT = {0: 1 << 30, 1: 1 << 22, 2: 1 << 16, 3: 0xfffffff0}


def readout_queue_floor(qmode, round_cap):
    """The smallest queue_cap the host setup gives a queue mode (sim_params.h readout_queue_floor: finalize() borrows the
    queue area as chain scratch of round_cap words).  The calendar queue gets the heap's floor: host_setup.hpp choose_layout
    raises queue_cap before it moves a heap layout to the calendar."""
    return (round_cap + 1) // 2 if qmode in (1, 2) else round_cap


@dataclass
class Case:
    name: str                 # the kernel, as lbft_kernel_info names it
    cap: str                  # "queue", "payload", "round", or "floor" / "horizon" (clean runs against the oracle)
    kind: str                 # "plain", "sweep", "ct" (a commit-times twin) or "resumable"
    N: int
    I: int
    max_clock: int
    kw: dict = field(default_factory=dict)  # run A: tests.support.make_config keywords, generous capacities included
    force: str = None         # LBFT_FORCE_KERNEL, or None
    sets: tuple = ()          # sweeps: ParamSet per set
    pin: int = None           # a C fixed by the case rather than derived from run A
    seed: int = 0

    @property
    def id(self):
        return "%s-%s-N%d%s" % (self.cap, self.name, self.N, "" if self.pin is None else "-C%d" % self.pin)

    @property
    def seeds(self):
        return np.arange(self.seed, self.seed + self.I, dtype=np.uint64)

    @property
    def set_of(self):
        return (np.arange(self.I) * 7 // 3) % len(self.sets) if self.sets else None

    @property
    def flags(self):
        return self.kw.get("flags", 0)

    @property
    def qmode(self):
        return int(re.search(r"kernel<\d+,(\d+),", self.name).group(1))

    def tight_kw(self, C):
        """Run B's keywords: A's with the capacity under test set to C."""
        return dict(self.kw, **{CAP_FIELD[self.cap]: int(C)})

    def combination(self):
        """(family, tile or lane group, state in shared memory, QMODE, capacity) of the case."""
        m = re.match(r"lbft_(?:ct_)?(sweep_)?(event_loop|wide)_kernel<(.*)>$", self.name)
        args = m.group(3).split(",")
        family = ("sweep " if m.group(1) else "") + ("thread" if m.group(2) == "event_loop" else "wide")
        if m.group(2) == "wide":
            return family, int(args[3]), args[2] == "true", int(args[1]), self.cap
        return family, int(args[-1]), False, int(args[1]), self.cap


def tight(case, counters):
    """C for `case` from run A's counters [instance, 12]."""
    if case.cap == "round":
        r = counters[:, 6].astype(np.int64)
        for C in range(32, int(r.max()) + 1, 32):
            if (r == C - 1).any() and (r >= C).mean() >= 0.05:
                return C
        raise AssertionError("%s: no multiple of 32 splits the active rounds %s" % (case.id, np.unique(r)))
    peaks = counters[:, PEAK_COLUMN[case.cap]].astype(np.int64)
    if case.pin is not None:
        assert (peaks == case.pin).any() and (peaks > case.pin).any() and (peaks < case.pin).any(), (case.id, np.unique(peaks))
        return case.pin
    ok = [v for v in np.unique(peaks) if (peaks > v).mean() >= 0.15 and (peaks <= v).mean() >= 0.15]
    assert ok, "%s: no peak splits the instances: %s" % (case.id, np.unique(peaks))
    return int(min(ok, key=lambda v: abs((peaks <= v).mean() - 0.5)))


UNI0 = dict(delay_kind=1, delay_lo=0, delay_hi=12)
# sweep sets with different delays, so their peaks differ: the fastest set sizes the layout (host_setup.hpp build_sweep)
SWEEP_SETS = (ParamSet(RandomDelay.new(10.0, 4.0)), ParamSet(RandomDelay.new(25.0, 200.0)), ParamSet(RandomDelay.uniform(2, 10)),
              ParamSet(RandomDelay.new(14.0, 2.0), NodeConfig(300, 30, 1.5, 1.0)))


def _c(name, cap, N, I, max_clock, force=None, kind="plain", sets=(), pin=None, **kw):
    return Case(name, cap, kind, N, I, max_clock, kw, force, sets, pin)


_CASES = [
    # ---- thread kernels, full tiles: the queue on every mode (the calendar at each mask width) ----
    _c(_t(16, 0), "queue", 12, 97, 4200, "thread", queue_cap=2048, round_cap=160),
    # (recording queues the duplicate timers the others elide: peaks past 64, so the HBM scan queue keeps the compact horizon)
    _c(_t(16, 1, rec=True), "queue", 5, 257, 1000, queue_cap=256, flags=REC),
    _c(_t(16, 2), "queue", 4, 1025, 1000, "thread", round_cap=64, queue_cap=64),  # (round_cap: off the FX_DEFAULT4 layout)
    _c(_t(16, 3), "queue", 9, 513, 200, "thread", queue_cap=1024),
    _c(_t(32, 3), "queue", 17, 65, 200, "thread", queue_cap=4096),
    _c(_t(64, 3), "queue", 33, 33, 120, "thread", queue_cap=8192),
    # ---- thread kernels, the payload pool: the bitmask below 32, at 32 (from a free-list run A), 33, and a large free list ----
    _c(_t(16, 2), "payload", 4, 1025, 1000, "thread", payload_cap=24),
    _c(_t(32, 3), "payload", 17, 129, 200, "thread", pin=32, payload_cap=64),
    _c(_t(32, 3), "payload", 17, 257, 200, "thread", pin=33, payload_cap=64),
    _c(_t(64, 3), "payload", 33, 65, 150, "thread", payload_cap=256),
    # ---- thread kernels, the round tables at NMAX 16 / 32 / 64 ----
    _c(_t(16, 2), "round", 4, 1025, 800, "thread", round_cap=64),
    _c(_t(32, 3), "round", 17, 129, 880, "thread", round_cap=64),
    _c(_t(64, 3), "round", 33, 33, 900, "thread", round_cap=64),
    # ---- thread kernels, sparse tiles (calendar queue, occupancy words in shared memory) ----
    _c(_t(16, 3, tile=8), "queue", 9, 12289, 200, queue_cap=1024),
    _c(_t(16, 3, tile=16), "queue", 6, 24577, 300, queue_cap=512, round_cap=64),
    # ---- wide kernels ----
    _c(_w(16, 0, 32), "queue", 12, 33, 4200, "wide", queue_cap=2048, round_cap=160),
    _c(_w(16, 2, 8), "queue", 7, 4097, 400, queue_cap=1024),
    _c(_w(16, 2, 8, smem=True), "queue", 3, 4097, 400, "wide", round_cap=32, queue_cap=32, payload_cap=12),
    _c(_w(16, 2, 32, smem=True), "queue", 4, 1000, 1000, round_cap=64, queue_cap=64),
    _c(_w(32, 3, 8), "queue", 17, 4097, 100, queue_cap=2048),
    _c(_w(32, 3, 32), "queue", 32, 64, 150, queue_cap=8192),
    _c(_w(16, 3, 32), "payload", 16, 100, 300, payload_cap=256),
    _c(_w(16, 2, 32, smem=True), "round", 4, 1000, 800, round_cap=64),
    # ---- sweeps, commit-times twins, a resumable kernel ----
    _c("lbft_sweep_event_loop_kernel<16,3,32>", "queue", 9, 257, 300, "thread", kind="sweep", sets=SWEEP_SETS, queue_cap=1024),
    _c("lbft_sweep_wide_kernel<16,2,false,8>", "queue", 7, 4097, 400, kind="sweep", sets=SWEEP_SETS, queue_cap=1024),
    _c(ct_name(_t(16, 3)), "queue", 9, 513, 200, "thread", kind="ct", queue_cap=1024, flags=CT),
    _c(ct_name(_w(16, 2, 8)), "queue", 7, 4097, 400, kind="ct", queue_cap=1024, flags=CT),
    _c(_t(16, 1, res=True), "queue", 5, 97, 1000, kind="resumable", queue_cap=256, flags=RES),
    # ---- the read-out floor: queue_cap = readout_queue_floor(mode, round_cap), commit logs near round_cap rows ----
    # (a lone author runs about a round per ms; the heap takes horizons past 4 095 ms)
    _c(_t(16, 0), "floor", 1, 65, 4100, "thread", round_cap=4128, queue_cap=4128, payload_cap=256),
    _c(_t(16, 1), "floor", 1, 65, 150, "thread", round_cap=160, queue_cap=80),
    _c(_t(16, 2), "floor", 2, 65, 1300, "thread", round_cap=64, queue_cap=32),
    _c(_t(16, 3), "floor", 2, 65, 1300, "thread", round_cap=64, queue_cap=64, payload_cap=256),
    # ---- the horizon edges ----
    _c(_t(16, 3), "horizon", 6, 65, 4095, "thread"),
    _c(_w(16, 3, 32), "horizon", 9, 40, 4095),
    _c(_w(16, 2, 32), "horizon", 3, 40, 16319, "wide"),
]


def _seeded(cases):
    return [Case(**dict(c.__dict__, seed=5000 + 7919 * k)) for k, c in enumerate(cases)]


CASES = {c.id: c for c in _seeded(_CASES)}
assert len(CASES) == len(_CASES), "duplicate case id"
EDGES = {k: c for k, c in CASES.items() if c.cap in CAP_FIELD}
CLEAN = {k: c for k, c in CASES.items() if c.cap not in CAP_FIELD}
