"""A plain C program (tests/cabi/golden_run.c) calling the C ABI reproduces the reference's golden runs — the
boundary works without Python or torch in the process."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_c_caller(tmp_path, name="golden_run"):
    from librabft_simulator_b200 import _build
    _build.build_product()
    exe = str(tmp_path / name)
    libdir = os.path.dirname(_build.LIB_PATH)
    subprocess.run(["gcc", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cabi", name + ".c"), "-I",
                    os.path.join(ROOT, "include"), "-L", libdir, "-llbft_b200", "-Wl,-rpath," + libdir], check=True)
    return exe


@pytest.mark.parametrize("name", ["golden_run", "staged_run", "multi_handle"])
def test_c_caller_compiles_and_links(tmp_path, name):
    # CPU box: the C programs build against include/lbft.h and link the product library
    exe = build_c_caller(tmp_path, name)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_c_caller_reproduces_goldens(tmp_path):
    exe = build_c_caller(tmp_path)
    p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert p.returncode == 0, p.stdout
    assert "golden runs reproduced" in p.stdout


@pytest.mark.gpu
def test_c_caller_staged_run_snapshot_and_round_switches(tmp_path, oracle):
    """lbft_run_until / lbft_snapshot_* / lbft_round_switches from plain C, against the oracle's staged run."""
    exe = build_c_caller(tmp_path, "staged_run")
    p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert p.returncode == 0, p.stdout
    assert "restored handle tracks the original" in p.stdout
    out = {}
    switches = []
    for line in p.stdout.splitlines():
        key, *vals = line.split()
        if key == "switch":
            switches.append(tuple(int(v) for v in vals))
        elif key in ("counts_at_500", "counts", "states", "switches", "snapshot_bytes"):
            out[key] = [int(v) for v in vals]
    mid, end = oracle.run_staged([52], 3, [500]), oracle.run_staged([52], 3, [500, 1000])
    assert out["counts_at_500"] == mid.commit_counts[0].tolist()
    assert out["counts"] == end.commit_counts[0].tolist()
    assert out["states"] == end.last_states[0].tolist()
    assert switches == oracle.round_switches_staged([52], 3, 0, [500, 1000]) and out["switches"] == [len(switches)]
    assert out["snapshot_bytes"][0] > 32 * 4 * 500   # one 32-lane tile of state words


@pytest.mark.gpu
def test_c_caller_drives_eight_handles_from_one_thread(tmp_path):
    """lbft_run_async / lbft_wait: one thread, eight handles (spread over every visible GPU), double-buffered host staging;
    lbft_commit_logs against lbft_commit_log; then a 65 536-instance batch per GPU (at least two handles) on the
    thread-per-instance kernel, whose shared-memory opt-in must hold on every device."""
    import torch
    exe = build_c_caller(tmp_path, "multi_handle")
    env = dict(os.environ, LBFT_TEST_DEVICES=str(torch.cuda.device_count()))
    p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, env=env)
    assert p.returncode == 0, p.stdout
    assert "async handles agree with synchronous runs" in p.stdout
    assert "instances (lbft_event_loop_kernel<16,2," in p.stdout
