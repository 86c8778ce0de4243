#!/usr/bin/env python
"""Measures committee sweeps (lbft_create_sweep_committees).  Prints one JSON object (also written to --out if given) with the
card's name and power limit, read in the same call.

  existing  what sweeps without per-set committees cost: tools/measure_rights_sweep.py's two workloads (the 256 x 256 grid sweep
            and BASELINE config 3 as a one-set sweep), kernel time of each run.  With --parent TREE (a checkout of the parent commit
            with its library built) the parent's package and this one run in alternating child processes, and their outputs are
            compared by digest.
  gain      committees of 4, 7, 10 and 16 x 4 delays at 256 and at 4 096 seeds per point: one committee sweep (a layout of 16)
            against one sweep handle per size, run one after the other and overlapped with run_async; kernel and wall times.
            Outputs compared instance by instance on the instances that neither side flags with a capacity error.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from measure_rights_sweep import card, existing, timed  # noqa: E402  (it imports the package of LBFT_MEASURE_TREE)

from librabft_simulator_b200 import NodeConfig, RandomDelay, SweepSimulator  # noqa: E402

SIZES = (4, 7, 10, 16)


def gain(k, rounds):
    delays = [RandomDelay.new(m, 4.0) for m in (6.0, 8.0, 10.0, 14.0)]
    seeds = np.arange(1, k + 1, dtype=np.uint64)
    one = SweepSimulator.grid(seeds, delays, [NodeConfig()], num_nodes=list(SIZES)).create(1000)
    per = [SweepSimulator.grid(seeds, delays, [NodeConfig()], num_nodes=n).create(1000) for n in SIZES]
    res = {"instances": one.num_instances, "kernels": {"committee_sweep": one.kernel_info(),
                                                       "per_size": [p.kernel_info() for p in per]}}
    one.run(strict=False)
    for p in per:
        p.run(strict=False)

    def overlapped():
        for p in per:
            p.run_async()
        for p in per:
            p.wait(strict=False)

    overlapped()
    rs = []
    for _ in range(rounds):
        r = {"committee_sweep_wall_ms": timed(lambda: one.run(strict=False)), "committee_sweep_kernel_ms": one.timing.sim_ms}
        r["serial_wall_ms"] = timed(lambda: [p.run(strict=False) for p in per])
        r["serial_kernel_ms"] = [p.timing.sim_ms for p in per]
        r["overlapped_wall_ms"] = timed(overlapped)
        rs.append(r)
    res["rounds"] = rs
    a = one.run(strict=False)
    same, compared = True, 0
    for n, p in zip(SIZES, per):
        b = p.run(strict=False)
        idx = np.nonzero(one.nodes_of_instance() == n)[0]
        ok = ((a.status[idx] & ~np.uint32(64)) == 1) & ((b.status & ~np.uint32(64)) == 1)
        compared += int(ok.sum())
        same &= bool((a.commit_counts[idx][ok][:, :n] == b.commit_counts[ok]).all())
        same &= bool((a.last_committed_states[idx][ok][:, :n] == b.last_committed_states[ok]).all())
        same &= bool((a.active_rounds[idx][ok] == b.active_rounds[ok]).all() and (a.commit_counts[idx][:, n:] == 0).all())
    res["identical"] = same
    res["compared_instances"] = compared
    one.close()
    for p in per:
        p.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--processes", type=int, default=3, help="child processes per library for 'existing'")
    ap.add_argument("--parent", help="a checkout of the parent commit with its library built, alternated with this tree for 'existing'")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", help="also write the JSON object to this file")
    args = ap.parse_args()
    if args.child:
        print(json.dumps(existing(args.rounds)))
        return
    res = {"card": card(), "rounds": args.rounds}
    trees = {"new": ROOT}
    if args.parent:
        trees["parent"] = os.path.abspath(args.parent)
    runs = {name: [] for name in trees}
    for _ in range(args.processes):
        for name, tree in trees.items():
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--rounds", str(args.rounds)], capture_output=True,
                                 text=True, check=True, cwd=ROOT, env=dict(os.environ, LBFT_MEASURE_TREE=tree)).stdout
            runs[name].append(json.loads(out.strip().splitlines()[-1]))
    res["existing"] = {}
    for name, rs in runs.items():
        res["existing"][name] = {w: {"kernel": rs[0][w]["kernel"], "median_ms": float(np.median([m for r in rs for m in r[w]["kernel_ms"]])),
                                     "process_medians_ms": [float(np.median(r[w]["kernel_ms"])) for r in rs],
                                     "digest": sorted({r[w]["digest"] for r in rs})} for w in rs[0]}
    res["gain"] = {str(k): gain(k, args.rounds) for k in (256, 4096)}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
