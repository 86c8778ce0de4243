#!/usr/bin/env python
"""Measures rights sweeps (lbft_create_sweep_rights).  Prints one JSON object (also written to --out if given) with the card's
name and power limit, read in the same call.

  existing  what sweeps that carry no rights cost: the 256 x 256 grid of tools/measure_sweep.py and BASELINE config 3 (65 536 x
            4) as a one-set sweep, kernel time (lbft_timing_info.sim_ms) of each run.  With --parent TREE (a checkout of the parent
            commit with its library built) the parent's package and this one run in alternating child processes (--rounds runs
            each after a warm-up run per process), and their outputs are compared by digest.
  gain      an N = 7 grid of 8 stake rows x 4 delays x 2 048 seeds: one rights sweep against one sweep handle per stake row, run
            one after the other and overlapped with run_async; kernel and wall times.  Outputs compared instance by instance.
  stats     block_latency_stats("quorum") on the rights sweep (per-group thresholds) against the same call on the sweep
            handle of one row (one threshold), wall time of the call.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.environ.get("LBFT_MEASURE_TREE", ROOT))  # (a child process of --parent imports the parent's package)

from librabft_simulator_b200 import NodeConfig, ParamSet, RandomDelay, SweepSimulator  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def digest(res):
    h = hashlib.sha256()
    for a in (res.commit_counts, res.last_committed_states, res.status, res.active_rounds):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def existing(rounds):
    """Child process: kernel ms of the two existing workloads, `rounds` runs each after a warm-up, and their output digests."""
    delays = [RandomDelay.new(m, v) for m in (6.0, 8.0, 10.0, 14.0) for v in (0.0, 2.0, 4.0, 8.0)]
    configs = [NodeConfig(delta=d, gamma=g) for d in (20, 30, 40, 60) for g in (1.5, 2.0, 2.5, 3.0)]
    out = {}
    for name, sim in (("grid256", SweepSimulator.grid(256, delays, configs, num_nodes=4)),
                      ("config3", SweepSimulator(np.arange(1, 65537, dtype=np.uint64), 4, [ParamSet(RandomDelay.new(10.0, 4.0), NodeConfig())],
                                                 np.zeros(65536, np.uint32)))):
        sim.create(1000)
        r = sim.run(strict=False)
        ms = []
        for _ in range(rounds):
            r = sim.run(strict=False)
            ms.append(sim.timing.sim_ms)
        out[name] = {"kernel": sim.kernel_info(), "kernel_ms": ms, "digest": digest(r)}
        sim.close()
    return out


def gain(rounds):
    rows = [(1,) * 7, (3, 1, 1, 1, 1, 1, 1), (5, 2, 2, 2, 2, 2, 2), (6, 2, 2, 2, 2, 2, 2), (0, 1, 1, 1, 1, 1, 1),
            tuple(1000 // (k + 1) for k in range(7)), (1 << 24, 1, 1, 1, 1, 1, 1 << 24), (2, 2, 2, 1, 1, 1, 1)]
    delays = [RandomDelay.new(m, 4.0) for m in (6.0, 8.0, 10.0, 14.0)]
    k = 2048
    seeds = np.arange(1, k + 1, dtype=np.uint64)
    one = SweepSimulator.grid(seeds, delays, [NodeConfig()], num_nodes=7, voting_rights=rows, commit_times=True).create(1000)
    base = [ParamSet(d, NodeConfig()) for d in delays]
    per = [SweepSimulator(np.tile(seeds, len(base)), 7, base, np.repeat(np.arange(len(base)), k), voting_rights=list(r),
                          commit_times=True).create(1000) for r in rows]
    res = {"kernels": {"rights_sweep": one.kernel_info(), "per_row": per[0].kernel_info()}}
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
        r = {"rights_sweep_wall_ms": timed(lambda: one.run(strict=False)), "rights_sweep_kernel_ms": one.timing.sim_ms}
        r["serial_wall_ms"] = timed(lambda: [p.run(strict=False) for p in per])
        r["serial_kernel_ms_sum"] = sum(p.timing.sim_ms for p in per)
        r["overlapped_wall_ms"] = timed(overlapped)
        rs.append(r)
    res["rounds"] = rs
    a = one.run(strict=False)
    same = True
    nr = len(rows)
    for ri, p in enumerate(per):
        b = p.run(strict=False)
        idx = np.concatenate([np.arange((j * nr + ri) * k, (j * nr + ri + 1) * k) for j in range(len(delays))])
        for f in ("commit_counts", "last_committed_states", "active_rounds", "status"):
            same &= bool((getattr(a, f)[idx] == getattr(b, f)).all())
    res["identical"] = same
    # block_latency_stats("quorum"): per-group thresholds on the rights sweep, one threshold on a sweep handle of one row
    a.block_latency_stats("quorum")
    b = per[1].run(strict=False)
    b.block_latency_stats("quorum")
    res["stats"] = {"rights_sweep_ms": [timed(lambda: a.block_latency_stats("quorum")) for _ in range(rounds)],
                    "one_row_sweep_ms": [timed(lambda: b.block_latency_stats("quorum")) for _ in range(rounds)],
                    "instances": [one.num_instances, per[1].num_instances]}
    one.close()
    for p in per:
        p.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--processes", type=int, default=4, help="child processes per library for 'existing'")
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
    res["gain"] = gain(args.rounds)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
