#!/usr/bin/env python
"""Times fault grids run as one fault sweep (lbft_create_sweep_faults) against the same grids run as one lbft_create_sweep handle
per fault set, one after the other and overlapped with run_async (every handle has its own stream).  Kernel times are the
library's CUDA-event timings (lbft_timing_info.sim_ms); wall times end in a device synchronise.  Every output of every instance
is compared between the two forms.  Prints one JSON object (also written to --out if given) with the card's name and power
limit, read in the same call.

  grid     64 points (4 LogNormal delays x 4 deltas x 4 fault sets: none, node 3 silent, 4 windows x 150 ms, node 0 silent
           with 2 windows x 400 ms) x 1 024 seeds, 4 authors, max_clock 1000: one handle of 65 536 instances | 4 sweep handles
           of 16 384
  config4  BASELINE config 4's shape (8 192 x 64, its voting rights) with 0, 7, 14 and 21 of its silent authors, 2 048 instances
           each: one handle | 4 sweep handles of 2 048
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

from librabft_simulator_b200 import FaultSet, NodeConfig, ParamSet, RandomDelay, SweepSimulator  # noqa: E402

W64 = [1 + (i % 3) for i in range(64)]
SILENT64 = [i for i in range(64) if i % 3 == 0 and i <= 60]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def silent_array(fs, n):
    if not fs.silent:
        return None
    a = np.zeros(n, np.uint8)
    a[list(fs.silent)] = 1
    return a


def compare(name, seeds, nodes, base_sets, faults, max_clock, rounds, **shared):
    """base_sets x faults (faults fastest), each point over `seeds`: one fault sweep against one sweep handle per fault set."""
    k = len(seeds)
    sets = [ParamSet(p.network_delay, p.node_config, f) for p in base_sets for f in faults]
    one = SweepSimulator(np.tile(seeds, len(sets)), nodes, sets, np.repeat(np.arange(len(sets)), k), **shared).create(max_clock)
    per = []
    for f in faults:  # fault set f: the instances of its points, in point order
        per.append(SweepSimulator(np.tile(seeds, len(base_sets)), nodes, base_sets, np.repeat(np.arange(len(base_sets)), k),
                                  silent=silent_array(f, nodes), partition_windows=f.partition_windows,
                                  partition_max_len=f.partition_max_len, **shared).create(max_clock))
    res = {"kernels": {"fault_sweep": one.kernel_info(), "per_fault_set": [p.kernel_info() for p in per]}}
    one.run(strict=False)  # warm-up: module load, shared-memory opt-in
    for p in per:
        p.run(strict=False)

    def overlapped():
        for p in per:
            p.run_async()
        for p in per:
            p.wait(strict=False)

    overlapped()
    rows = []
    for _ in range(rounds):
        r = {"fault_sweep_wall_ms": timed(lambda: one.run(strict=False)), "fault_sweep_kernel_ms": one.timing.sim_ms}
        r["serial_wall_ms"] = timed(lambda: [p.run(strict=False) for p in per])
        r["serial_kernel_ms_sum"] = sum(p.timing.sim_ms for p in per)
        r["overlapped_wall_ms"] = timed(overlapped)
        rows.append(r)
    res["rounds"] = rows
    a = one.run(strict=False)
    same = True
    nf = len(faults)
    for fi, p in enumerate(per):
        b = p.run(strict=False)
        idx = np.concatenate([np.arange((j * nf + fi) * k, (j * nf + fi + 1) * k) for j in range(len(base_sets))])
        for f in ("commit_counts", "last_committed_states", "active_rounds", "status"):
            same &= bool((getattr(a, f)[idx] == getattr(b, f)).all())
        same &= bool((a.counters[idx] == b.counters).all())
    res["identical"] = same
    one.close()
    for p in per:
        p.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", help="also write the JSON object to this file")
    args = ap.parse_args()
    res = {"card": card(), "rounds": args.rounds}
    delays = [RandomDelay.new(m, 4.0) for m in (6.0, 8.0, 10.0, 14.0)]
    base = [ParamSet(d, NodeConfig(delta=x)) for d in delays for x in (20, 30, 40, 60)]
    grid_faults = [FaultSet(), FaultSet((3,)), FaultSet((), 4, 150), FaultSet((0,), 2, 400)]
    res["grid"] = compare("grid", np.arange(1, 1025, dtype=np.uint64), 4, base, grid_faults, 1000, args.rounds)
    c4_faults = [FaultSet(tuple(SILENT64[:n])) for n in (0, 7, 14, 21)]
    res["config4"] = compare("config4", np.arange(52, 52 + 2048, dtype=np.uint64), 64, [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig())],
                             c4_faults, 1000, args.rounds, voting_rights=W64)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
