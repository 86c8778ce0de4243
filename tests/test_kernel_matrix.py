"""The kernel matrix (tests/kernel_matrix.py) on the CPU: it names exactly the event-loop kernels the library carries, each
entry's configuration makes the product's host setup select its kernel, and every configuration the host setup accepts, over
a grid across every threshold of the kernel choice, names a kernel the library carries (the one refusal lbft_create adds on
top of the host setup's checks, epochs x recording / resumable runs, spelled out as that rule)."""
import ctypes
import itertools
import re
import subprocess

import numpy as np
import pytest

from librabft_simulator_b200 import ParamSet, RandomDelay, _build
from tests.fault_support import FaultHarness
from tests.kernel_matrix import BIG_QUEUE, CT, MATRIX, REC, RES, TDS, ct_name, fault_sets
from tests.support import P, make_config
from tests.sweep_support import SweepHostCore

# the kernels of the library that are not event loops: the bulk read-outs of commit logs / commit times and the latency reduction
NOT_EVENT_LOOPS = {"lbft_commit_logs_kernel", "lbft_commit_times_kernel", "lbft_latency_init_kernel", "lbft_latency_stats_kernel"}


def library_kernels(path):
    """The kernels of a shared library, as cuobjdump lists its functions, demangled and spelled like kernel_name."""
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"Function : (\S+)", out)
    names = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    spelled = set()
    for n in filter(None, names):
        n = re.sub(r"\(.*$", "", n)                # the parameter list
        n = re.sub(r"^void |^lbft::|\s", "", n).replace("lbft::", "")
        spelled.add(n)
    return spelled


@pytest.fixture(scope="module")
def kernels():
    names = library_kernels(_build.build_product())
    other = {n for n in names if n in NOT_EVENT_LOOPS}
    assert other == NOT_EVENT_LOOPS, "the read-out and latency kernels are not where this test expects them"
    return names - other


class Harnesses:
    """The product's host setup for plain handles, sweeps and fault sweeps (the host-compiled harnesses of tests/hostcore)."""

    def __init__(self, hostcore):
        self.plain, self.sweep, self.faults = hostcore, SweepHostCore(), FaultHarness()
        self.plain.lib.hostcore_setup_digest.argtypes = [ctypes.c_void_p, P, P]
        self._epochs = {}

    def kernel_info(self, kind, seeds, N, max_clock, sets, set_of, kw):
        if kind == "plain":
            return self.plain.kernel_info(seeds, N, max_clock, **kw)
        if kind == "sweep":
            return self.sweep.kernel_info(seeds, N, max_clock, sets, set_of, **kw)
        return self.faults.kernel_info(seeds, N, max_clock, sets, set_of, **kw)[0]

    def epochs(self, seeds, N, max_clock, kw):
        """Layout::epochs of a plain handle's host setup (a function of the horizon, round_cap and commands_per_epoch alone,
        host_setup.hpp epochs_of: computed once per such triple)."""
        key = (max_clock, kw.get("round_cap", 0), kw.get("commands_per_epoch"))
        if key not in self._epochs:
            self._epochs[key] = self._layout_epochs(seeds, N, max_clock, kw)
        return self._epochs[key]

    def _layout_epochs(self, seeds, N, max_clock, kw):
        cfg, keep = make_config(seeds, N, max_clock, **kw)
        digest, epochs = np.zeros(1, np.uint64), np.zeros(1, np.uint32)
        assert self.plain.lib.hostcore_setup_digest(ctypes.byref(cfg), P(digest.ctypes.data), P(epochs.ctypes.data)) == 0
        return int(epochs[0])


@pytest.fixture(scope="module")
def harnesses(hostcore):
    return Harnesses(hostcore)


def set_force(monkeypatch, force):
    if force is None:
        monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    else:
        monkeypatch.setenv("LBFT_FORCE_KERNEL", force)


def test_the_matrix_names_every_event_loop_kernel_of_the_library(kernels):
    missing, stale = sorted(kernels - set(MATRIX)), sorted(set(MATRIX) - kernels)
    assert not missing, "kernels of the library without a kernel-matrix entry: %s" % missing
    assert not stale, "kernel-matrix entries whose kernel the library does not carry: %s" % stale


@pytest.mark.parametrize("name", sorted(MATRIX))
def test_each_entry_selects_its_kernel(harnesses, monkeypatch, name):
    e = MATRIX[name]
    set_force(monkeypatch, e.force)
    assert harnesses.kernel_info(e.kind, e.seeds, e.N, e.max_clock, e.sets, e.set_of, e.kw) == name


def test_the_entries_sit_at_the_edges():
    entries = list(MATRIX.values())
    # committees at the limits of the mask width; generic layouts at N = 64 (the compile-time one is a kernel of its own)
    for nmax, qm, committees in ((16, 3, {16}), (16, 0, {16}), (32, 3, {17, 32}), (32, 0, {17, 32}), (64, 3, {33, 64}), (64, 0, {33, 64})):
        got = {e.N for e in entries if re.search(r"kernel<%d,%d," % (nmax, qm), e.name) and not e.name.endswith(",3>")}
        assert got >= committees, (nmax, qm, got)
    assert {1, 2} <= {e.N for e in entries}
    for e in entries:
        wide8 = re.search(r"wide_kernel<\d+,\d+,(true|false),8\b", e.name)
        if wide8 and e.N > 8 and not e.name.endswith(",3>"):  # (the compile-time 64-author layout is N = 64 by definition)
            assert e.N % 8, "%s: an 8-lane group over a committee that is a multiple of 8" % e.name
        if e.per_warp > 1:
            assert e.I % e.per_warp, "%s: %d instances fill whole warps" % (e.name, e.I)
        if "commands_per_epoch" in e.kw:
            # epochs cross after 2..10 commands; the thread kernel with its queue in shared memory keeps that queue only while
            # epochs * 32 rounds <= 128 (host_setup.hpp choose_layout), which takes commands_per_epoch >= 11
            smem_queue_thread = re.match(r"lbft_event_loop_kernel<\d+,2,", e.name)
            assert e.kw["commands_per_epoch"] == 11 if smem_queue_thread else 2 <= e.kw["commands_per_epoch"] <= 10, e.name
        if e.kind != "plain":
            assert len(e.sets) >= 3 and set(e.set_of) == set(range(len(e.sets))) and (np.diff(e.set_of) != 0).mean() > 0.5
            kinds = [(p.network_delay.kind, p.network_delay.mean, p.network_delay.variance) for p in e.sets]
            assert (0, 25.0, 200.0) in kinds and any(k[0] == 1 for k in kinds), e.name
    # a silent node on the top bit of every mask width
    for nmax in (16, 32, 64):
        tops = [e for e in entries if re.search(r"kernel<%d," % nmax, e.name) and e.N == nmax and
                (e.kw.get("silent") is not None and e.kw["silent"][-1] or any(e.N - 1 in p.faults.silent for p in e.sets))]
        assert tops, nmax
    # every extension on each family and queue mode, among the plain kernels (a sweep's sets do not stand in for them)
    extensions = {
        "weights": lambda e: e.kw.get("voting_rights") is not None,
        "partitions": lambda e: e.kw.get("partition_windows", 0) > 0 or any(p.faults.partition_windows for p in e.sets),
        "uniform from 0": lambda e: e.kw.get("delay_kind") == 1 and e.kw.get("delay_lo") == 0 or
        any(p.network_delay.kind == 1 and p.network_delay.lo == 0 for p in e.sets),
        "constant delay": lambda e: e.kw.get("delay_variance") == 0.0 or any(p.network_delay.variance == 0.0 and p.network_delay.kind == 0 for p in e.sets),
        "exp() fallback": lambda e: e.kw.get("delay_variance") == 200.0 or any(p.network_delay.variance == 200.0 for p in e.sets),
        "finite tci": lambda e: e.kw.get("target_commit_interval", 100000) < 100000 or
        any(p.node_config.target_commit_interval < 100000 for p in e.sets),
    }
    for family, qm in itertools.product(("wide", "event_loop"), range(4)):
        group = [e for e in entries if re.match(r"lbft_%s_kernel<\d+,%d," % (family, qm), e.name)]
        for ext, has in extensions.items():
            assert any(has(e) for e in group), "%s kernels, QMODE %d: no entry with %s" % (family, qm, ext)


# ---- every accepted configuration names a kernel of the library ----
COMMITTEES = [1, 2, 4, 5, 6, 8, 16, 17, 32, 33, 64]
# both sides of every batch-size threshold of kernel_family / select_kernel
BATCHES = [4096, 4097, 12288, 12289, 24576, 24577, 49152, 49153]
# both sides of 4 095 / 4 096 (calendar / heap), of the sparse tiles' horizon limits (1 791 / 1 792 at 16 per warp, 3 583 / 3 584
# at 8) and of the compact entries' 16 320
HORIZONS = [1791, 1792, 3583, 3584, 4095, 4096, 16319, 16320]
CAPS = [{}, dict(round_cap=32, queue_cap=16, payload_cap=4), dict(queue_cap=BIG_QUEUE, payload_cap=300)]
PLAIN_FLAGS = [0, REC, RES, REC | RES, TDS, CT]
EPOCHS = [30000, 5]          # one epoch; several
FORCES = [None, "thread", "wide"]


def test_every_accepted_configuration_names_a_kernel_of_the_library(harnesses, kernels, monkeypatch):
    seeds = {I: np.arange(I, dtype=np.uint64) for I in BATCHES}
    sets = [ParamSet(RandomDelay.new(10.0, 4.0)), ParamSet(RandomDelay.new(25.0, 200.0)), ParamSet(RandomDelay.uniform(0, 20))]
    set_of = {I: np.arange(I) % len(sets) for I in BATCHES}
    unknown, refused, named = [], 0, 0
    for force in FORCES:
        set_force(monkeypatch, force)
        for N, I, mc, caps in itertools.product(COMMITTEES, BATCHES, HORIZONS, CAPS):
            runs = [("plain", None, dict(caps, flags=f, commands_per_epoch=cpe)) for f in PLAIN_FLAGS for cpe in EPOCHS
                    # the recording / resumable / data-sync kernels are never a family choice: once is enough
                    if force is None or not f & (REC | RES | TDS)]
            fsets = tuple(ParamSet(p.network_delay, p.node_config, f) for p, f in zip(sets, fault_sets(N)))
            # (a fault sweep picks its kernel as a sweep does, with its largest window count: once, flag off)
            runs += [(kind, s, dict(caps, flags=f)) for kind, s in (("sweep", sets), ("faults", fsets)) for f in (0, CT)
                     if kind == "sweep" or (force is None and not f)]
            for kind, s, kw in runs:
                try:
                    name = harnesses.kernel_info(kind, seeds[I], N, mc, s, set_of[I], kw)
                except RuntimeError:
                    continue  # the host setup refuses the configuration: lbft_create does too
                if kind == "plain" and kw["flags"] & (REC | RES) and harnesses.epochs(seeds[I], N, mc, kw) > 1:
                    refused += 1  # lbft_create refuses epochs x recording / resumable runs after the host setup
                    continue
                named += 1
                if name not in kernels:
                    unknown.append((name, kind, N, I, mc, force, kw))
    assert named > 10000 and refused > 0
    assert not unknown, "accepted configurations name kernels the library does not carry: %s; e.g. %s" % (
        sorted({u[0] for u in unknown}), unknown[:3])


def test_commit_time_twins_share_their_entry_with_the_flag_off_kernel():
    for name, e in MATRIX.items():
        if e.flags & CT:
            off = [o for o in MATRIX.values() if ct_name(o.name) == name]
            assert len(off) == 1 and off[0].seed == e.seed and off[0].I == e.I and off[0].N == e.N, name
