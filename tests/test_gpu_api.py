"""C-ABI behaviour on a real device: call-sequence errors, re-seeding, determinism, timing/memory info and the
device-buffer view used for the NCCL all-gather."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def make(seeds, nodes=4, **kw):
    from librabft_simulator_b200 import BatchSimulator, RandomDelay
    return BatchSimulator(seeds, nodes, RandomDelay.new(10.0, 4.0), **kw)


def test_results_before_run_are_an_error():
    from librabft_simulator_b200 import _lib
    sim = make(np.arange(1, 33, dtype=np.uint64)).create(1000)
    out = np.zeros((32, 4), np.uint32)
    rc = sim._lib.lbft_commit_counts(sim._handle, ctypes.c_void_p(out.ctypes.data))
    assert rc == -3 and b"lbft_run" in sim._lib.lbft_last_error()
    with pytest.raises(_lib.LbftError):
        sim.run_device()          # upload must come first
    sim.upload()
    sim.run_device()
    rc = sim._lib.lbft_commit_counts(sim._handle, ctypes.c_void_p(out.ctypes.data))
    assert rc == -3               # still not downloaded
    res = sim.download()
    assert res.commit_counts.min() > 5
    sim.close()


def test_rerun_is_deterministic_and_reseeding_changes_results(oracle):
    seeds = np.arange(700, 764, dtype=np.uint64)
    sim = make(seeds).create(1000)
    a = sim.run()
    a_states = a.last_committed_states.copy()
    b = sim.run()
    np.testing.assert_array_equal(a_states, b.last_committed_states)
    seeds2 = seeds + np.uint64(5000)
    sim.set_seeds(seeds2)
    c = sim.run()
    assert (c.last_committed_states != a_states).any()
    ref = oracle.run(seeds2, 4, 1000)
    np.testing.assert_array_equal(ref.last_states, c.last_committed_states)
    np.testing.assert_array_equal(ref.commit_counts, c.commit_counts)
    assert sim.timing.kernel_launches == 1 and sim.timing.sim_ms > 0
    assert sim.timing.h2d_bytes == 64 * 8 and sim.timing.d2h_bytes > 0
    dev_bytes, words = sim.memory_info()
    assert dev_bytes > 64 * words * 4 * 0.9 and words > 100
    sim.close()


def test_device_buffer_view_matches_host_results():
    """Every id of lbft_device_buffer views the finished run's results: 0 commit counts, 1 last states, 2 counters, 3 status,
    4 active rounds, and 5 the block of 1, 0 and 4, decoded by ShardedResult as the all-gather's receiver decodes it."""
    import torch
    from librabft_simulator_b200.distributed import ShardedResult, _DeviceView
    seeds = np.arange(40, 104, dtype=np.uint64)
    sim = make(seeds).create(1000)
    res = sim.run()

    def view(which, nbytes_want):
        ptr, nbytes = sim.device_buffer(which)
        assert nbytes == nbytes_want, which
        return torch.as_tensor(_DeviceView(ptr, (nbytes,), "|u1"), device="cuda:0").cpu().numpy()
    np.testing.assert_array_equal(view(0, 64 * 4 * 4).view(np.uint32).reshape(64, 4), res.commit_counts)
    np.testing.assert_array_equal(view(1, 64 * 4 * 8).view(np.uint64).reshape(64, 4), res.last_committed_states)
    np.testing.assert_array_equal(view(2, 64 * 12 * 4).view(np.uint32).reshape(64, 12), res.counters)
    np.testing.assert_array_equal(view(3, 64 * 4).view(np.uint32), res.status)
    np.testing.assert_array_equal(view(4, 64 * 4).view(np.uint32), res.active_rounds)
    block = ShardedResult(None, view(5, 64 * 4 * 12 + 64 * 4), 64, 4, 0, 64)
    np.testing.assert_array_equal(block.commit_counts, res.commit_counts)
    np.testing.assert_array_equal(block.last_committed_states, res.last_committed_states)
    np.testing.assert_array_equal(block.active_rounds, res.active_rounds)
    sim.close()


def test_two_handles_are_independent():
    s1 = make(np.arange(1, 33, dtype=np.uint64)).create(1000)
    s2 = make(np.arange(1, 33, dtype=np.uint64), nodes=7).create(500)
    r2 = s2.run()
    r1 = s1.run()
    assert r1.commit_counts.shape == (32, 4) and r2.commit_counts.shape == (32, 7)
    assert r1.commit_counts.min() > 10
    s1.close(); s2.close()


def test_commit_log_truncation_and_bounds():
    from librabft_simulator_b200 import _lib
    sim = make(np.arange(52, 84, dtype=np.uint64), nodes=3).create(1000)
    res = sim.run()
    n = ctypes.c_size_t()
    buf = (_lib.LbftCommit * 5)()
    assert sim._lib.lbft_commit_log(sim._handle, 0, 0, buf, 5, ctypes.byref(n)) == 0
    assert n.value == 27                      # seed 52 / 3 nodes: the reference golden (simulated_run.rs:53)
    full = sim.commit_log(0, 0)
    assert [(buf[i].proposer, buf[i].index, buf[i].time) for i in range(5)] == full[:5]
    assert sim._lib.lbft_commit_log(sim._handle, 32, 0, buf, 5, ctypes.byref(n)) == -1   # instance out of range
    assert sim._lib.lbft_commit_log(sim._handle, 0, 3, buf, 5, ctypes.byref(n)) == -1    # node out of range
    sim.close()


def test_active_rounds_getter_is_the_counter_column():
    seeds = np.arange(900, 900 + 70, dtype=np.uint64)
    sim = make(seeds).create(1000)
    res = sim.run()
    assert res.active_rounds.shape == (70,) and res.active_rounds.dtype == np.uint32
    np.testing.assert_array_equal(res.active_rounds, res.counters[:, 6])
    assert res.active_rounds.min() > 20
    sim.close()


def test_async_run_keeps_previous_results_readable(oracle):
    """lbft_run_async / lbft_wait: the previous run's results live in the other set of host mirrors, the next batch's seeds
    are staged while a run is in flight, and every device-touching call is refused until lbft_wait."""
    from librabft_simulator_b200 import _lib
    s0, s1 = np.arange(100, 196, dtype=np.uint64), np.arange(5100, 5196, dtype=np.uint64)
    sim = make(s0).create(1000)
    first = sim.run()
    sim.set_seeds(s1)
    sim.run_async()
    with pytest.raises(_lib.LbftError) as e:
        sim.run()
    assert e.value.code == -3
    out = np.zeros((96, 4), np.uint64)                      # read run 0 through the C getter WHILE run 1 is in flight
    assert sim._lib.lbft_last_states(sim._handle, ctypes.c_void_p(out.ctypes.data)) == 0
    np.testing.assert_array_equal(out, first.last_committed_states)
    second = sim.wait()
    np.testing.assert_array_equal(first.last_committed_states, oracle.run(s0, 4, 1000).last_states)   # eager copy: still run 0
    np.testing.assert_array_equal(second.last_committed_states, oracle.run(s1, 4, 1000).last_states)
    with pytest.raises(RuntimeError, match="run again"):
        first.counters                                       # lazily fetched data of an older run is refused, not wrong
    sim.close()


@pytest.mark.parametrize("nodes,count,kw", [(4, 200, {}), (3, 33, {}), (7, 64, dict(partition_windows=3, partition_max_len=200)),
                                            (4, 40, dict(silent=[0, 0, 0, 1]))])
def test_bulk_commit_logs_match_the_per_node_reader(oracle, nodes, count, kw):
    seeds = np.arange(3000, 3000 + count, dtype=np.uint64)
    sim = make(seeds, nodes, **kw).create(1000)
    res = sim.run()
    rows, lens = res.commit_logs()
    np.testing.assert_array_equal(lens, res.commit_counts)
    assert rows.shape == (count, max(1, int(lens.max())))
    for i in sorted({0, 1, count // 2, count - 1}):
        for n in range(nodes):
            got = [(int(r["proposer"]), int(r["index"]), int(r["time"])) for r in rows[i, :lens[i, n]]]
            assert got == sim.commit_log(i, n) == oracle.commit_log(seeds, nodes, i, n, 1000, **kw)
    # state key == SipHash of the returned rows, for EVERY instance and node (simulated_context.rs:51-55)
    for i in range(count):
        for n in range(nodes):
            log = [(int(r["proposer"]), int(r["index"]), int(r["time"])) for r in rows[i, :lens[i, n]]]
            assert oracle.state_key(log) == int(res.last_committed_states[i, n])
    small, lens2 = sim.commit_logs(cap=3)                    # truncation: lens still tells the full length
    np.testing.assert_array_equal(lens2, lens)
    np.testing.assert_array_equal(small, rows[:, :3])
    sim.close()


def test_rounds_device_buffer_and_kernel_info():
    import torch
    seeds = np.arange(40, 104, dtype=np.uint64)
    sim = make(seeds).create(1000)
    res = sim.run()
    ptr, nbytes = sim.device_buffer(4)
    assert nbytes == 64 * 4

    class Cai:
        __cuda_array_interface__ = {"shape": (64,), "typestr": "<i4", "data": (ptr, False), "version": 2}
    np.testing.assert_array_equal(torch.as_tensor(Cai(), device="cuda:0").cpu().numpy().astype(np.uint32), res.active_rounds)
    assert sim.kernel_info().startswith("lbft_")
    sim.close()


def test_sharded_simulator_single_rank(oracle):
    """ShardedBatchSimulator with world 1 is the plain path; (world > 1: tests/test_distributed_gloo.py on CPU, bench.py
    under torchrun on GPUs)."""
    from librabft_simulator_b200 import RandomDelay, ShardedBatchSimulator
    seeds = np.arange(8000, 8064, dtype=np.uint64)
    res = ShardedBatchSimulator(seeds, 4, RandomDelay.new(10.0, 4.0)).loop_until(1000)
    ref = oracle.run(seeds, 4, 1000)
    np.testing.assert_array_equal(res.commit_counts, ref.commit_counts)
    np.testing.assert_array_equal(res.last_committed_states, ref.last_states)
    np.testing.assert_array_equal(res.active_rounds, ref.counters[:, 6])


def test_run_stream_keeps_one_run_in_flight_and_matches_the_oracle(oracle):
    """BatchSimulator.run_stream / ShardedBatchSimulator.run_stream: one result per batch, in order, each bit-exact — the next
    run is already in flight when a result is handed out, and the counters of the finished run stay readable meanwhile."""
    from librabft_simulator_b200 import RandomDelay, ShardedBatchSimulator
    batches = [np.arange(b, b + 96, dtype=np.uint64) for b in (100, 5000, 70000, 123456)]
    refs = [oracle.run(b, 4, 1000) for b in batches]
    sim = make(batches[0]).create(1000)
    got = 0
    for res, ref in zip(sim.run_stream(batches), refs):
        np.testing.assert_array_equal(res.commit_counts, ref.commit_counts)
        np.testing.assert_array_equal(res.last_committed_states, ref.last_states)
        np.testing.assert_array_equal(res.counters[:, :8], ref.counters[:, :8])   # read while the next batch runs
        got += 1
    assert got == len(batches)
    assert list(sim.run_stream([])) == []
    res = sim.run()                                   # the handle is idle again after a stream
    np.testing.assert_array_equal(res.commit_counts, refs[-1].commit_counts)
    sim.close()
    sharded = ShardedBatchSimulator(batches[0], 4, RandomDelay.new(10.0, 4.0)).create(1000)
    outs = list(sharded.run_stream(batches))
    assert len(outs) == len(batches)
    for res, ref in zip(outs, refs):
        np.testing.assert_array_equal(res.commit_counts, ref.commit_counts)
        np.testing.assert_array_equal(res.last_committed_states, ref.last_states)
        np.testing.assert_array_equal(res.active_rounds, ref.counters[:, 6])
    sharded.close()
