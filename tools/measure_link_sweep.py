#!/usr/bin/env python
"""Measures links sweeps (lbft_create_sweep_links).  Prints one JSON object (also written to --out if given) with the card's name,
power limit and SM clock, read in the same call.

  existing  what sweeps without link latencies cost: the 256 x 256 grid sweep and BASELINE config 3 as a one-set sweep
            (tools/measure_rights_sweep.py) and README's committee sweep (4 delays x 4 deltas x committees of 4, 7, 10 and 16 x
            1 024 seeds, commit times on), kernel time of each run.  With --parent TREE (a tree with the parent commit's package
            and library) the parent's package and this one run in alternating child processes, and their outputs are compared by
            digest.
  links     the 256 x 256 grid as a links sweep with an all-zero matrix (outputs compared by digest with the grid without links)
            and with a regional one (nodes 0, 1 near each other, 2 and 3 farther), kernel time.
  gain      4 link matrices (tests/link_support.matrices(7)) x 4 delays x 1 024 seeds of 7 nodes: one links sweep against one
            sweep handle per matrix, run one after the other; kernel and wall times, outputs compared instance by instance.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from measure_rights_sweep import digest, existing as rights_existing, timed  # noqa: E402  (imports the package of LBFT_MEASURE_TREE)

from librabft_simulator_b200 import NodeConfig, RandomDelay, SweepSimulator  # noqa: E402

DELAYS = [RandomDelay.new(m, v) for m in (6.0, 8.0, 10.0, 14.0) for v in (0.0, 2.0, 4.0, 8.0)]
CONFIGS = [NodeConfig(delta=d, gamma=g) for d in (20, 30, 40, 60) for g in (1.5, 2.0, 2.5, 3.0)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def kernel_runs(sim, rounds):
    sim.create(1000)
    r = sim.run(strict=False)
    ms = []
    for _ in range(rounds):
        r = sim.run(strict=False)
        ms.append(sim.timing.sim_ms)
    out = {"kernel": sim.kernel_info(), "kernel_ms": ms, "digest": digest(r)}
    sim.close()
    return out


def existing(rounds):
    """Child process: the two workloads of tools/measure_rights_sweep.py and README's committee sweep."""
    out = rights_existing(rounds)
    delays = [RandomDelay.new(10.0, v) for v in (0.0, 4.0, 16.0, 64.0)]
    configs = [NodeConfig(delta=d) for d in (20, 40, 80, 160)]
    out["committee"] = kernel_runs(SweepSimulator.grid(range(1024), delays, configs, num_nodes=[4, 7, 10, 16], commit_times=True), rounds)
    return out


def links(rounds):
    """Child process: the 256 x 256 grid with an all-zero and with a regional matrix."""
    from librabft_simulator_b200 import regional_latency
    zero = ((0,) * 4,) * 4
    regional = regional_latency([0, 0, 1, 2], [[1, 6, 12], [6, 1, 9], [12, 9, 1]])
    return {"zero": kernel_runs(SweepSimulator.grid(256, DELAYS, CONFIGS, num_nodes=4, link_latency=[zero]), rounds),
            "regional": kernel_runs(SweepSimulator.grid(256, DELAYS, CONFIGS, num_nodes=4, link_latency=[regional], payload_cap=64), rounds)}


def gain(rounds):
    sys.path.insert(0, ROOT)
    from tests.link_support import matrices
    mats = [m for _, m in matrices(7)]
    delays = [RandomDelay.new(m, 4.0) for m in (6.0, 8.0, 10.0, 14.0)]
    seeds = np.arange(1, 1025, dtype=np.uint64)
    one = SweepSimulator.grid(seeds, delays, [NodeConfig()], num_nodes=7, link_latency=mats, payload_cap=128).create(1000)
    per = [SweepSimulator.grid(seeds, delays, [NodeConfig()], num_nodes=7, link_latency=[m], payload_cap=128).create(1000) for m in mats]
    res = {"instances": one.num_instances, "kernels": {"links_sweep": one.kernel_info(), "per_matrix": [p.kernel_info() for p in per]}}
    one.run(strict=False)
    for p in per:
        p.run(strict=False)
    rs = []
    for _ in range(rounds):
        r = {"links_sweep_wall_ms": timed(lambda: one.run(strict=False)), "links_sweep_kernel_ms": one.timing.sim_ms}
        r["serial_wall_ms"] = timed(lambda: [p.run(strict=False) for p in per])
        r["serial_kernel_ms"] = [p.timing.sim_ms for p in per]
        rs.append(r)
    res["rounds"] = rs
    a = one.run(strict=False)
    same, compared = True, 0
    for k, p in enumerate(per):
        b = p.run(strict=False)
        idx = np.nonzero(one.set_of_instance % len(mats) == k)[0]
        ok = ((a.status[idx] & ~np.uint32(64)) == 1) & ((b.status & ~np.uint32(64)) == 1)
        compared += int(ok.sum())
        for field in ("commit_counts", "last_committed_states", "active_rounds"):
            same &= bool((getattr(a, field)[idx][ok] == getattr(b, field)[ok]).all())
    res["identical"] = same
    res["compared_instances"] = compared
    one.close()
    for p in per:
        p.close()
    return res


def summary(rs):
    return {w: {"kernel": rs[0][w]["kernel"], "median_ms": float(np.median([m for r in rs for m in r[w]["kernel_ms"]])),
                "process_medians_ms": [float(np.median(r[w]["kernel_ms"])) for r in rs],
                "digest": sorted({r[w]["digest"] for r in rs})} for w in rs[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--processes", type=int, default=3, help="child processes per library")
    ap.add_argument("--parent", help="a tree with the parent commit's package and library built, alternated with this tree for 'existing'")
    ap.add_argument("--child", choices=("existing", "links"), help=argparse.SUPPRESS)
    ap.add_argument("--out", help="also write the JSON object to this file")
    args = ap.parse_args()
    if args.child:
        print(json.dumps(existing(args.rounds) if args.child == "existing" else links(args.rounds)))
        return
    res = {"card": card(), "rounds": args.rounds}
    trees = {"new": ROOT}
    if args.parent:
        trees["parent"] = os.path.abspath(args.parent)
    runs = {name: [] for name in trees}
    link_runs = []

    def child(kind, tree):
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", kind, "--rounds", str(args.rounds)], capture_output=True,
                             text=True, check=True, cwd=ROOT, env=dict(os.environ, LBFT_MEASURE_TREE=tree)).stdout
        return json.loads(out.strip().splitlines()[-1])

    for _ in range(args.processes):
        for name, tree in trees.items():
            runs[name].append(child("existing", tree))
        link_runs.append(child("links", ROOT))
    res["existing"] = {name: summary(rs) for name, rs in runs.items()}
    res["links"] = summary(link_runs)
    res["links"]["zero_equals_no_links"] = res["links"]["zero"]["digest"] == res["existing"]["new"]["grid256"]["digest"]
    res["gain"] = gain(args.rounds)
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
