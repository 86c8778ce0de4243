"""The threshold time of a block without a GPU: the serial block_threshold_time (sim_core.cuh), compiled for the host, against
numpy over adversarial synthetic commit-time tables at every N from 1 to 64 — ties everywhere, all nodes at one clock, blocks
only zero-weight nodes committed, a lone node 32, weights at the 2^24 cap, commit counts that cut each node off at its own row.
Also the device probe of its lane form (tests/gpuprobe/block_threshold_probe.cu) cross-compiled for sm_90a, so that a change
that breaks it fails here before the GPU run (tests/test_gpu_latency_reduction.py runs it)."""
import subprocess

import numpy as np
import pytest

from librabft_simulator_b200 import _build
from tests.block_latency_support import BlockLatencyHarness, numpy_threshold_times, synthetic_cases

INT64_MAX = np.iinfo(np.int64).max


@pytest.fixture(scope="module")
def blk():
    return BlockLatencyHarness()


@pytest.mark.parametrize("N", range(1, 65))
def test_serial_threshold_time_matches_numpy_on_synthetic_tables(blk, N):
    rng = np.random.default_rng(1000 + N)
    ties = zero_first = unreached = 0
    for label, weights, cc, times, W in synthetic_cases(N, rng):
        want = numpy_threshold_times(cc, times, weights, W)
        np.testing.assert_array_equal(blk.threshold_times(cc, times, weights, W), want, err_msg=label)
        committed = cc[:, :, None] > np.arange(times.shape[2])
        t = np.where(committed, times[:, :N, :], INT64_MAX)
        first = t.min(axis=1)
        ties += int(((t == first[:, None, :]) & committed).sum(axis=1).max() > 1)
        zero_first += int(((t == first[:, None, :]) & committed & (weights == 0)[None, :, None]).any())
        unreached += int((want == INT64_MAX).any())
    assert unreached
    assert (ties and zero_first) or N == 1  # (a committee of one has no tie, and holds a voting right)


def test_probe_cross_compiles_for_sm_90a():
    path = _build.build_block_threshold_probe(force=True)
    elves = subprocess.run(["cuobjdump", "--list-elf", path], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in elves
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    assert "block_threshold_probe_kernel" in sass and "SHFL.IDX" in sass and "SHFL.BFLY" in sass
