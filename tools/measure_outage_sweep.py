#!/usr/bin/env python
"""Measures outage sweeps (lbft_create_sweep_outages).  Prints one JSON object (also written to --out if given) with the card's
name, power limit and SM clock, read in the same call.

  existing  what sweeps without outages cost: the 256 x 256 grid sweep and BASELINE config 3 as a one-set sweep
            (tools/measure_rights_sweep.py) and README's links example (4 link matrices x 4 delays x 1 024 seeds of 7 nodes in
            one links sweep), kernel time of each run.  With --parent TREE (a tree with the parent commit's package and library)
            the parent's package and this one run in alternating child processes, and their outputs are compared by digest.
  outages   the 256 x 256 grid as an outage sweep whose schedules are all empty (outputs compared by digest with the grid
            without outages), kernel time.
  example   README's leader-crash example: 7 nodes, node 0 crash-stop at 500 ms, down over [500, 800), or never down (the faults
            axis), crossed with delta 20 / 40 / 80, 4 096 seeds each, max_clock 2000: kernel time, the mean quorum latency of
            blocks proposed in [200, 500), [500, 800) and [800, 1800) per set, and node 0's mean commit count against the
            others'.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from measure_link_sweep import CONFIGS, DELAYS, card, kernel_runs, summary  # noqa: E402  (imports the package of LBFT_MEASURE_TREE)
from measure_rights_sweep import existing as rights_existing  # noqa: E402

from librabft_simulator_b200 import FaultSet, NodeConfig, RandomDelay, SweepSimulator, _lib  # noqa: E402

EXAMPLE_WINDOWS = ((200, 500), (500, 800), (800, 1800))


def existing(rounds):
    """Child process: the two workloads of tools/measure_rights_sweep.py and README's links example."""
    sys.path.insert(0, ROOT)
    from tests.link_support import matrices
    out = rights_existing(rounds)
    delays = [RandomDelay.new(m, 4.0) for m in (6.0, 8.0, 10.0, 14.0)]
    out["links_example"] = kernel_runs(SweepSimulator.grid(np.arange(1, 1025, dtype=np.uint64), delays, [NodeConfig()], num_nodes=7,
                                                           link_latency=[m for _, m in matrices(7)], payload_cap=128), rounds)
    return out


def outages(rounds):
    """Child process: the 256 x 256 grid as an outage sweep with empty schedules."""
    return {"empty": kernel_runs(SweepSimulator.grid(256, DELAYS, CONFIGS, num_nodes=4, faults=[FaultSet(outages=((0, 5, 5),))]), rounds)}


def example(rounds):
    """README's leader-crash example: kernel time and the read-outs it quotes."""
    scen = [FaultSet(outages=((0, 500, None),)), FaultSet(outages=((0, 500, 800),)), FaultSet()]
    names = ["crash-stop at 500", "down [500, 800)", "never down"]
    deltas = (20, 40, 80)
    sim = SweepSimulator.grid(4096, [RandomDelay.new(10.0, 4.0)], [NodeConfig(delta=d) for d in deltas], num_nodes=7, faults=scen,
                              commit_times=True, round_cap=512)
    sim.create(2000)
    res = sim.run(strict=False)
    ms = []
    for _ in range(rounds):
        res = sim.run(strict=False)
        ms.append(sim.timing.sim_ms)
    out = {"kernel": sim.kernel_info(), "instances": sim.num_instances, "kernel_ms": ms,
           "clean": float(((res.status & np.uint32(_lib.ST_ERROR_MASK)) == 0).mean()), "sets": []}
    lat = {w: res.block_latency_stats("quorum", proposed_from=w[0], proposed_until=w[1]).mean() for w in EXAMPLE_WINDOWS}
    for s, p in enumerate(sim.param_sets):
        idx = sim.set_of_instance == s
        cc = res.commit_counts[idx].astype(np.float64)
        out["sets"].append({"delta": deltas[s // 3], "node0": names[s % 3],
                            "quorum_ms": {"[%d, %d)" % w: None if np.isnan(lat[w][s]) else round(float(lat[w][s]), 2) for w in EXAMPLE_WINDOWS},
                            "node0_commits": round(float(cc[:, 0].mean()), 1), "others_commits": round(float(cc[:, 1:].mean()), 1)})
    sim.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--processes", type=int, default=3, help="child processes per library")
    ap.add_argument("--parent", help="a tree with the parent commit's package and library built, alternated with this tree for 'existing'")
    ap.add_argument("--child", choices=("existing", "outages"), help=argparse.SUPPRESS)
    ap.add_argument("--out", help="also write the JSON object to this file")
    args = ap.parse_args()
    if args.child:
        print(json.dumps(existing(args.rounds) if args.child == "existing" else outages(args.rounds)))
        return
    res = {"card": card(), "rounds": args.rounds}
    trees = {"new": ROOT}
    if args.parent:
        trees["parent"] = os.path.abspath(args.parent)
    runs = {name: [] for name in trees}
    outage_runs = []

    def child(kind, tree):
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", kind, "--rounds", str(args.rounds)], capture_output=True,
                             text=True, check=True, cwd=ROOT, env=dict(os.environ, LBFT_MEASURE_TREE=tree)).stdout
        return json.loads(out.strip().splitlines()[-1])

    for _ in range(args.processes):
        for name, tree in trees.items():
            runs[name].append(child("existing", tree))
        outage_runs.append(child("outages", ROOT))
    res["existing"] = {name: summary(rs) for name, rs in runs.items()}
    res["outages"] = summary(outage_runs)
    res["outages"]["empty_equals_no_outages"] = res["outages"]["empty"]["digest"] == res["existing"]["new"]["grid256"]["digest"]
    res["example"] = example(args.rounds)
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
