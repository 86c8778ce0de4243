#!/usr/bin/env python
"""Times a parameter sweep run as one sweep handle (lbft_create_sweep) against the same grid run as plain handles, and the
price of the sweep kernels on the bench shape.  Kernel times are the library's CUDA-event timings (lbft_timing_info.sim_ms);
wall times end in a device synchronise.  Prints one JSON object (also written to --out if given) with the card's name and
power limit, read in the same call.

  grid     256 points (16 LogNormal delays x 16 NodeConfigs) x 256 seeds, 4 authors, max_clock 1000:
           one sweep handle of 65 536 instances | 256 plain handles run one after the other | the same 256 handles overlapped
           with run_async (every handle has its own stream)
  config3  BASELINE config 3 (65 536 x 4, LogNormal(10, 4), max_clock 1000) as a one-set sweep against the plain handle, whose
           kernel is the compile-time-layout bench kernel; rounds alternate between the two.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from librabft_simulator_b200 import BatchSimulator, NodeConfig, ParamSet, RandomDelay, SweepSimulator  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def grid_256():
    delays = [RandomDelay.new(m, v) for m in (6.0, 8.0, 10.0, 14.0) for v in (0.0, 2.0, 4.0, 8.0)]
    configs = [NodeConfig(delta=d, gamma=g) for d in (20, 30, 40, 60) for g in (1.5, 2.0, 2.5, 3.0)]
    return delays, configs


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", help="also write the JSON object to this file")
    args = ap.parse_args()
    res = {"card": card(), "rounds": args.rounds}

    # ---- the 256 x 256 grid
    delays, configs = grid_256()
    seeds = np.arange(1, 257, dtype=np.uint64)
    sweep = SweepSimulator.grid(seeds, delays, configs, num_nodes=4).create(1000)
    plains = [BatchSimulator(seeds, 4, p.network_delay, p.node_config).create(1000) for p in sweep.param_sets]
    res["grid_kernels"] = {"sweep": sweep.kernel_info(), "plain": plains[0].kernel_info()}
    sweep.run(strict=False)  # warm-up: module load, shared-memory opt-in
    for p in plains:
        p.run(strict=False)

    def run_overlapped():
        for p in plains:
            p.run_async()
        for p in plains:
            p.wait(strict=False)

    run_overlapped()
    rows = []
    for _ in range(args.rounds):
        r = {"sweep_wall_ms": timed(lambda: sweep.run(strict=False)), "sweep_kernel_ms": sweep.timing.sim_ms}
        r["plain_serial_wall_ms"] = timed(lambda: [p.run(strict=False) for p in plains])
        r["plain_serial_kernel_ms_sum"] = sum(p.timing.sim_ms for p in plains)
        r["plain_overlapped_wall_ms"] = timed(run_overlapped)
        rows.append(r)
    res["grid"] = rows
    # the sweep's results equal the plain handles' wherever neither reports a capacity error
    out = sweep.run(strict=False)
    same = clean = 0
    for k, p in enumerate(plains):
        r = p.run(strict=False)
        sl = slice(k * 256, (k + 1) * 256)
        ok = ((r.status & ~np.uint32(64)) == 1) & ((out.status[sl] & ~np.uint32(64)) == 1)
        clean += int(ok.sum())
        same += int((ok & (r.commit_counts == out.commit_counts[sl]).all(1) & (r.last_committed_states == out.last_committed_states[sl]).all(1)).sum())
    res["grid_parity"] = {"clean_instances": clean, "identical_instances": same}
    sweep.close()
    for p in plains:
        p.close()

    # ---- BASELINE config 3 as a one-set sweep against the plain (compile-time-layout) handle
    I = 65536
    seeds3 = np.arange(52, 52 + I, dtype=np.uint64)
    one = SweepSimulator(seeds3, 4, [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig())], np.zeros(I)).create(1000)
    plain = BatchSimulator(seeds3, 4, RandomDelay.new(10.0, 4.0), NodeConfig()).create(1000)
    res["config3_kernels"] = {"sweep": one.kernel_info(), "plain": plain.kernel_info()}
    one.run()
    plain.run()
    rows = []
    for _ in range(args.rounds):
        a = one.run()
        b = plain.run()
        rows.append({"sweep_kernel_ms": one.timing.sim_ms, "plain_kernel_ms": plain.timing.sim_ms})
    res["config3"] = rows
    res["config3_identical"] = bool((a.commit_counts == b.commit_counts).all() and (a.last_committed_states == b.last_committed_states).all()
                                    and (a.status == b.status).all())
    one.close()
    plain.close()

    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
