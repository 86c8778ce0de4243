#!/usr/bin/env python
"""What a quorum-latency grid costs to read: (a) commit_times() copied to the host and reduced per parameter set with numpy
(each block's quorum-threshold time by sorting its node times; mean, p50, p99), against (b) block_latency_stats("quorum")
reduced on the device, with its mean() and percentile().  Both end in a stream synchronise, so wall time is valid.  One workload
per process (--workload config3: BASELINE config 3 as one commit-times handle; config4: BASELINE config 4, 64 weighted authors,
two nodes per lane; sweep: the 256 x 256 grid of tools/measure_sweep.py as one sweep handle); (a) and (b) alternate, the minimum
and median over --rounds rounds after a warm-up round, and must agree exactly.  Prints one JSON object (also written to --out if given)
with the card's name, power limit and SM clock, read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, make_sim  # noqa: E402
from librabft_simulator_b200 import SweepSimulator, _lib  # noqa: E402
from librabft_simulator_b200.simulator import resolve_threshold  # noqa: E402
from tests.block_latency_support import threshold_times  # noqa: E402
from tools.measure_sweep import grid_256  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def make(workload):
    """(simulator, number of groups); the groups are contiguous blocks of instances of equal size."""
    if workload in ("config3", "config4"):
        c = CONFIGS[int(workload[-1])]
        sim = make_sim(np.arange(c["base_seed"], c["base_seed"] + c["instances"], dtype=np.uint64), c["nodes"], commit_times=True,
                       **c["kw"])
        sim.loop_until(c["max_clock"], strict=False)
        return sim, 1
    delays, configs = grid_256()
    sim = SweepSimulator.grid(256, delays, configs, num_nodes=4, commit_times=True)
    sim.loop_until(1000, strict=False)
    return sim, len(sim.param_sets)


def via_numpy(sim, groups, status):
    """The recipe without the device reduction: the whole commit-time table to the host, then numpy per group."""
    committed, proposed = sim.commit_times()
    weights = np.ones(sim.num_nodes, np.int64) if sim.voting_rights is None else sim.voting_rights.astype(np.int64)
    T, reached = threshold_times(committed, weights, resolve_threshold("quorum", sim.total_voting_rights()))
    on_chain = (committed >= 0).any(axis=1) & ((status & np.uint32(_lib.ST_ERROR_MASK)) == 0)[:, None]
    lat = np.where(on_chain & reached, T - proposed, -1)
    out = np.empty((groups, 3))
    for g, p in enumerate(lat.reshape(groups, -1)):
        x = p[p >= 0]
        out[g] = (x.sum() / len(x), np.percentile(x, 50, method="inverted_cdf"), np.percentile(x, 99, method="inverted_cdf"))
    return out


def via_device(sim):
    s = sim.block_latency_stats("quorum")
    return np.stack([s.mean(), s.percentile(50), s.percentile(99)], axis=1), int(s.hist[:, -1].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("config3", "config4", "sweep"), required=True)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", help="also write the JSON object to this file")
    args = ap.parse_args()
    res = {"card": card(), "workload": args.workload, "rounds": args.rounds}
    sim, groups = make(args.workload)
    status = sim._fetch("lbft_status", np.uint32, (sim.num_instances,))
    res["kernel"], res["sim_ms"], res["groups"] = sim.kernel_info(), float(sim.timing.sim_ms), groups
    res["error_instances"] = int(((status & np.uint32(_lib.ST_ERROR_MASK)) != 0).sum())
    ms = {"a_numpy": [], "b_device": []}
    for r in range(args.rounds + 1):  # (round 0 warms up)
        t0 = time.perf_counter()
        a = via_numpy(sim, groups, status)
        t1 = time.perf_counter()
        b, overflow = via_device(sim)
        t2 = time.perf_counter()
        if r:
            ms["a_numpy"].append((t1 - t0) * 1e3)
            ms["b_device"].append((t2 - t1) * 1e3)
        assert overflow == 0, "latencies in the overflow bin: the percentiles would not be exact"
        assert np.array_equal(a, b), "the two reductions disagree"
    res["agree_exactly"] = True
    res["cap"] = int(sim._fetch("lbft_commit_counts", np.uint32, (sim.num_instances, sim.num_nodes)).max())
    res["mean_latency_ms_first_groups"] = [float(v) for v in b[:4, 0]]
    for k, v in ms.items():
        res["ms_" + k] = {"min": min(v), "median": float(np.median(v)), "all": v}
    res["a_over_b_min"] = res["ms_a_numpy"]["min"] / res["ms_b_device"]["min"]
    sim.close()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
