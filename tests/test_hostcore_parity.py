"""CPU-side check of the DEVICE state machine: csrc/sim_core.cuh compiled with g++ (tests/hostcore) must
reproduce the oracle bit-for-bit — commit counts, SipHash state keys, events processed by kind, cancelled
timers, creation stamps, active rounds and RNG draw counts.  This validates the round-id layout and every
protocol rule of the kernel source before it reaches a GPU."""
import numpy as np
import pytest

from tests.support import assert_same

CASES = [
    # (first seed, instances, nodes, max_clock, extra)
    (52, 1, 3, 1000, {}),     # golden 1 (simulated_run.rs:45-66)
    (48, 1, 8, 1000, {}),     # golden 2 (simulated_run.rs:68-94)
    (1, 96, 4, 1000, {}),     # BASELINE config 2/3 shape
    (1000, 40, 3, 1000, {}),
    (5, 24, 7, 1000, {}),     # config 5 shape without partitions
    (77, 4, 16, 600, {}),
    (3, 16, 2, 1000, {}),
    (52, 2, 3, 3000, {"delay_variance": 0.0}),  # config 1: fixed 10 ms, >100 rounds
    (11, 16, 4, 2500, {}),    # longer horizon
    (21, 16, 4, 1000, {"delay_mean": 25.0, "delay_variance": 200.0}),  # heavy jitter -> timeouts/TCs
    (31, 16, 5, 1500, {"delta": 5, "gamma": 1.5, "lambda_": 0.25, "queue_cap": 4096, "payload_cap": 1024}),   # tight pacemaker -> many timeouts, query-all
    (41, 8, 4, 4000, {"target_commit_interval": 300, "delta": 400}),  # commit tracker query-all path
    (61, 16, 4, 1000, {"queue_cap": 128}),   # forces the 64-bit-key scan queue in HBM (QMODE 1)
    (62, 8, 6, 1000, {}),                    # calendar queue (QMODE 3)
    (63, 4, 6, 4200, {}),                    # binary heap (QMODE 0): horizon beyond the calendar's range
    (64, 6, 9, 700, {"delay_kind": 1, "delay_lo": 0, "delay_hi": 3, "round_cap": 256}),  # calendar queue, zero delays (same-slot pushes)
]


@pytest.mark.parametrize("seed0,count,nodes,max_clock,extra", CASES)
def test_hostcore_matches_oracle(oracle, hostcore, seed0, count, nodes, max_clock, extra):
    seeds = np.arange(seed0, seed0 + count, dtype=np.uint64)
    o = oracle.run(seeds, nodes, max_clock, **extra)
    h = hostcore.run(seeds, nodes, max_clock, **extra)
    assert (o.status == 1).all()
    assert ((h.status & ~np.uint32(64)) == 1).all(), h.status
    assert_same(o, h, "N=%d" % nodes)


def test_goldens_through_hostcore(hostcore):
    r = hostcore.run([52], 3, 1000)
    assert r.commit_counts.tolist() == [[27, 27, 27]]
    assert r.last_states.tolist() == [[11134312813757838303] * 3]
    r = hostcore.run([48], 8, 1000)
    assert r.commit_counts.tolist() == [[28] * 7 + [30]]
    assert r.last_states.tolist() == [[12785928431398617538] * 7 + [4890275890002623733]]


def test_round_overflow_is_flagged(hostcore):
    # a single node makes a round per millisecond: the default round_cap cannot hold 1000 rounds
    r = hostcore.run([3], 1, 1000)
    assert r.status[0] & 2
    r = hostcore.run([3], 1, 1000, round_cap=1056)
    assert r.status[0] == 1 and r.commit_counts[0, 0] > 900


def test_queue_overflow_is_flagged(hostcore):
    r = hostcore.run([9], 8, 1000, queue_cap=16, round_cap=0)
    assert r.status[0] & (4 | 2 | 8)


def test_fast_paths_are_selected_for_the_benchmark_config(hostcore):
    # BASELINE config 3 (N=4, LogNormal(10,4), max_clock=1000) must run on the exact delay-threshold table
    # (no device exp) and the scan queue
    info = hostcore.setup_info(4, 1000)
    assert info["delay_kmax"] > 100 and info["queue_scan"] == 2 and info["round_cap"] == 128
    assert hostcore.setup_info(4, 20000)["queue_scan"] == 1                         # long horizon: 64-bit keys in HBM
    assert hostcore.setup_info(4, 1000, delay_variance=0.0)["delay_kmax"] == 0      # constant delay: host-evaluated
    assert hostcore.setup_info(16, 1000)["queue_scan"] == 3                         # big committees: calendar queue
    assert hostcore.setup_info(16, 5000)["queue_scan"] == 0                         # long horizons: binary heap


def test_delay_table_equals_libm_exp_path(oracle, hostcore):
    # wider LogNormal (sigma ~ 0.35): ~2000 thresholds; results must still equal the oracle's exp()
    seeds = np.arange(900, 916, dtype=np.uint64)
    kw = {"delay_mean": 15.0, "delay_variance": 30.0}
    assert hostcore.setup_info(4, 1000, **kw)["delay_kmax"] > 1000
    assert_same(oracle.run(seeds, 4, 1000, **kw), hostcore.run(seeds, 4, 1000, **kw))
    kw = {"delay_mean": 25.0, "delay_variance": 200.0}  # too wide for a table -> exp() fallback path
    assert hostcore.setup_info(4, 1000, **kw)["delay_kmax"] == 0
    o, h = oracle.run(seeds, 4, 1500, **kw), hostcore.run(seeds, 4, 1500, **kw)
    assert_same(o, h)


def test_epoch_end_stalls_like_the_reference_semantics(oracle, hostcore):
    # commands_per_epoch = 5: in the reference semantics (oracle) the first node to finish the epoch swaps its record
    # store before broadcasting the final QC and nobody else can fetch it (DESIGN.md §9): commits freeze near 5.
    seeds = np.arange(1, 9, dtype=np.uint64)
    o = oracle.run(seeds, 4, 1000, commands_per_epoch=5)
    assert (o.status & 32).all()
    assert o.commit_counts.max() <= 5 and o.commit_counts.min() >= 3
    # the device core reproduces it (tests/test_epochs.py has the matrix); the status bit is advisory
    h = hostcore.run(seeds, 4, 1000, commands_per_epoch=5)
    assert (h.status == 33).all()
    assert_same(o, h, "epoch stall")


W64 = [1 + (i % 3) for i in range(64)]
SILENT64 = [1 if i % 3 == 0 and i <= 60 else 0 for i in range(64)]


def test_compile_time_shapes_match_the_oracle_and_the_generic_instantiation(oracle, hostcore, monkeypatch):
    """The instantiations with a compile-time layout (sim_params.h FX_*: BASELINE configs 1-3, configs[4], configs[3])
    are selected for exactly those shapes and compute what the oracle and the generic instantiation compute."""
    shapes = [
        (1, 4, 24, {}),                                                              # FX_DEFAULT4
        (2, 7, 24, {"partition_windows": 4, "partition_max_len": 150}),              # FX_PART7 (BASELINE configs[4])
        (3, 64, 2, {"voting_rights": W64, "silent": SILENT64}),                      # FX_COMMITTEE64 (BASELINE configs[3])
        (3, 64, 1, {}),                                                              # ... voting rights / silent nodes are run-time
    ]
    # (the layout of a handle depends on the kernel family the host picks for the batch size: the seven-author shape is the
    # thread kernel's, which 16 384 instances select on their own — tests/test_gpu_wide.py — and small batches only when asked)
    monkeypatch.setenv("LBFT_FORCE_KERNEL", "thread")
    for fx, nodes, count, kw in shapes:
        assert hostcore.fixed_shape(nodes, 1000, **kw) == fx
        seeds = np.arange(31000, 31000 + count, dtype=np.uint64)
        o, h = oracle.run(seeds, nodes, 1000, **kw), hostcore.run(seeds, nodes, 1000, **kw)
        assert (h.status == 1).all()
        assert_same(o, h, "compile-time shape %d" % fx)
        monkeypatch.setenv("HOSTCORE_NO_FIXED", "1")
        g = hostcore.run(seeds, nodes, 1000, **kw)
        monkeypatch.delenv("HOSTCORE_NO_FIXED")
        assert_same(g, h, "generic vs compile-time shape %d" % fx)
        np.testing.assert_array_equal(g.counters, h.counters)
    # neighbouring configurations stay generic
    assert hostcore.fixed_shape(7, 1000) == 0                                                   # no partition windows
    assert hostcore.fixed_shape(7, 1200, partition_windows=4, partition_max_len=150) == 0     # another horizon
    assert hostcore.fixed_shape(7, 1000, partition_windows=4, partition_max_len=150, delay_kind=1, delay_lo=5, delay_hi=15) == 0
    assert hostcore.fixed_shape(7, 1000, partition_windows=4, partition_max_len=150, silent=[1, 0, 0, 0, 0, 0, 0]) == 0
    assert hostcore.fixed_shape(48, 1000) == 0
    assert hostcore.fixed_shape(4, 1000, flags=1) == 0                                          # recording


def test_kernel_choice(hostcore, monkeypatch):
    """The kernel the host selects (lbft_kernel_info, through the host setup the product runs): the automatic picks that
    tests/test_gpu_wide.py::test_automatic_choice asserts on the GPU, and what LBFT_FORCE_KERNEL makes of the same cases."""
    cases = (("config2", 1024, 4, {}), ("config3", 65536, 4, {}), ("config5", 16384, 7, {}),
             ("config5p", 16384, 7, {"partition_windows": 4, "partition_max_len": 150}),
             ("mid7", 8192, 7, {}), ("full7", 65536, 7, {}), ("big64", 8192, 64, {}),
             ("small64", 64, 64, {}), ("resumable", 64, 4, {"flags": 2}),
             ("recording", 64, 7, {"flags": 1}), ("mid4", 8192, 4, {}),
             ("long7", 64, 7, {"max_clock": 20000}))

    def picks(family):
        if family:
            monkeypatch.setenv("LBFT_FORCE_KERNEL", family)
        else:
            monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
        out = {}
        for name, count, nodes, kw in cases:
            kw = dict(kw)
            max_clock = kw.pop("max_clock", 1000)
            out[name] = hostcore.kernel_info(np.arange(1, count + 1, dtype=np.uint64), nodes, max_clock, **kw)
        return out

    # <NMAX, QMODE, SMEM, lanes per instance, EP, FX> / <NMAX, QMODE, FX, REC, RES, EP, TDS, instances per warp tile>
    auto = picks(None)
    assert auto["config2"] == "lbft_wide_kernel<16,2,true,32,false,0>"    # a warp per instance, whole instance in shared memory
    assert auto["config3"] == auto["mid4"] == "lbft_event_loop_kernel<16,2,1,false,false,false,false,32>"
    assert auto["config5"] == "lbft_event_loop_kernel<16,3,0,false,false,false,false,8>"  # one wave of 8-instance warp tiles
    assert auto["config5p"] == "lbft_event_loop_kernel<16,3,2,false,false,false,false,8>"  # ... BASELINE configs[4]: its compile-time shape
    assert auto["mid7"] == "lbft_wide_kernel<16,2,false,8,false,0>"       # 8 lanes per instance, four instances per warp
    assert auto["full7"] == "lbft_event_loop_kernel<16,3,0,false,false,false,false,32>"
    assert auto["small64"] == "lbft_wide_kernel<64,3,false,32,false,0>"
    assert auto["big64"] == "lbft_wide_kernel<64,3,false,8,false,3>"      # BASELINE configs[3]: compile-time shape, 8 lanes per instance
    assert auto["long7"] == "lbft_wide_kernel<16,0,false,32,false,0>"     # beyond the 14-bit times of the compact queue
    assert auto["resumable"] == "lbft_event_loop_kernel<16,1,0,false,true,false,false,32>"
    assert auto["recording"] == "lbft_event_loop_kernel<16,3,0,true,false,false,false,32>"

    # forced to one thread per instance: full warp tiles; the compile-time layout only where it is the thread kernel's
    thread = picks("thread")
    assert thread["config2"] == thread["config3"] == thread["mid4"] == "lbft_event_loop_kernel<16,2,1,false,false,false,false,32>"
    for name in ("config5", "config5p", "mid7", "full7"):
        assert thread[name] == "lbft_event_loop_kernel<16,3,0,false,false,false,false,32>", name
    assert thread["big64"] == thread["small64"] == "lbft_event_loop_kernel<64,3,0,false,false,false,false,32>"
    assert thread["long7"] == "lbft_event_loop_kernel<16,0,0,false,false,false,false,32>"

    # forced to the wide kernel: the shared-memory queue up to 16 authors; recording / resumable handles stay on the thread kernel
    wide = picks("wide")
    assert wide["config2"] == "lbft_wide_kernel<16,2,true,32,false,0>"
    for name in ("config3", "mid4", "config5", "config5p", "mid7", "full7"):
        assert wide[name] == "lbft_wide_kernel<16,2,false,8,false,0>", name
    assert wide["big64"] == auto["big64"] and wide["small64"] == auto["small64"] and wide["long7"] == auto["long7"]
    assert thread["resumable"] == wide["resumable"] == auto["resumable"]
    assert thread["recording"] == wide["recording"] == auto["recording"]
