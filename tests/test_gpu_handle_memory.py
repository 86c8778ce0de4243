"""A handle's memory on the GPU: what lbft_memory_info and a run's transfer sizes report for five handle shapes, pinned to the
values of commit 08fb4de (before the handle's tables and results became one allocation each), and a create that runs out of
device memory, after which the same device makes and runs a normal handle."""
import numpy as np
import pytest

from librabft_simulator_b200 import BatchSimulator, FaultSet, NodeConfig, RandomDelay, SweepSimulator, _lib

pytestmark = pytest.mark.gpu

LBFT_ERR_NOMEM = -5
DELAYS = [RandomDelay.new(10.0, 4.0), RandomDelay.new(20.0, 4.0)]
FAULTS = [FaultSet(), FaultSet(silent=(1,))]


def plain(nodes=4, instances=1024, **kw):
    return BatchSimulator(np.arange(1, instances + 1, dtype=np.uint64), nodes, RandomDelay.new(10.0, 4.0), **kw)


# name -> (simulator, kernel family it must get)
CASES = {
    "plain_1024x4": (lambda: plain(), "lbft_wide_kernel"),
    "plain_1024x4_commit_times": (lambda: plain(commit_times=True), "lbft_ct_wide_kernel"),
    "fault_sweep": (lambda: SweepSimulator.grid(256, DELAYS, [NodeConfig()], faults=FAULTS), "lbft_sweep_wide_kernel"),
    "rights_sweep_commit_times": (lambda: SweepSimulator.grid(128, DELAYS, [NodeConfig()], faults=FAULTS,
                                                              voting_rights=[(1, 1, 1, 1), (3, 1, 1, 1)], commit_times=True),
                                  "lbft_ct_sweep_wide_kernel"),
    "wide_128x64": (lambda: plain(nodes=64, instances=128), "lbft_wide_kernel"),
}

# (lbft_memory_info device_bytes, words_per_instance, timing.h2d_bytes, timing.d2h_bytes) after one run to max_clock 1000, as
# commit 08fb4de reports them on an H100 80GB HBM3
PINNED = {
    "plain_1024x4": (3627421, 852, 8192, 122884),
    "plain_1024x4_commit_times": (6248861, 852, 8192, 122884),
    "fault_sweep": (3637509, 852, 8192, 122884),
    "rights_sweep_commit_times": (6269478, 852, 8192, 122884),
    "wide_128x64": (58035853, 113066, 1024, 138244),
}


def measure(name):
    make, family = CASES[name]
    sim = make()
    sim.create(1000)
    sim.run(strict=False)
    got = sim.memory_info() + (int(sim.timing.h2d_bytes), int(sim.timing.d2h_bytes))
    kernel = sim.kernel_info()
    sim.close()
    return got, kernel


@pytest.mark.parametrize("name", sorted(CASES))
def test_memory_and_transfer_sizes_are_pinned(name):
    got, kernel = measure(name)
    assert kernel.startswith(CASES[name][1] + "<"), kernel
    assert got == PINNED[name]


def test_create_that_cannot_fit_fails_and_the_device_stays_usable(oracle):
    """64 nodes with round_cap 32 768: a batch whose state is at least twice the card's memory is refused with LBFT_ERR_NOMEM (an
    ordinary error return); then a normal handle on the same device is created, runs and matches the oracle."""
    import torch
    big = dict(round_cap=32768, commands_per_epoch=32768)
    one = plain(nodes=64, instances=1, **big).create(1000)
    words = one.memory_info()[1]
    one.close()
    instances = -(-2 * torch.cuda.get_device_properties(0).total_memory // (words * 4))
    assert instances < 2 ** 32
    with pytest.raises(_lib.LbftError) as e:
        plain(nodes=64, instances=int(instances), **big).create(1000)
    assert e.value.code == LBFT_ERR_NOMEM, str(e.value)
    seeds = np.arange(1, 65, dtype=np.uint64)
    res = plain(instances=64).loop_until(1000)
    ref = oracle.run(seeds, 4, 1000)
    np.testing.assert_array_equal(res.commit_counts, ref.commit_counts)
    np.testing.assert_array_equal(res.last_committed_states, ref.last_states)
    np.testing.assert_array_equal(res.counters[:, :8], ref.counters[:, :8])
