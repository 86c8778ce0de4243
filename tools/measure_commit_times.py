#!/usr/bin/env python
"""The price of commit times (LBFT_FLAG_COMMIT_TIMES): kernel time with the flag off and on, alternated within one run, for
each configuration of bench.py's CONFIGS (its instances, nodes, max_clock, base seed and inputs) and for the 256 x 256 grid of
tools/measure_sweep.py as one sweep handle; plus the time of one lbft_commit_times read-out.  Kernel times are the library's
CUDA-event timings (lbft_timing_info.sim_ms), the minimum and median over the rounds.  Outputs of the two handles are compared
(they must be identical).  Prints one JSON object (also written to --out if given) with the card's name and power limit,
read in the same call.

--build TREE [TREE ...] instead times a full forced build of the product library of each source tree (e.g. a checkout of the
parent commit and this one), alternating over --rounds rounds, into a temporary directory: wall time, and CPU time of the
compiler processes.  No GPU is needed for that."""
import argparse
import importlib.util
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, make_sim  # noqa: E402
from librabft_simulator_b200 import SweepSimulator  # noqa: E402
from tools.measure_sweep import card, grid_256  # noqa: E402


def make_pair(cid):
    c = CONFIGS[cid]
    seeds = np.arange(c["base_seed"], c["base_seed"] + c["instances"], dtype=np.uint64)
    sims = []
    for ct in (False, True):
        sim = make_sim(seeds, c["nodes"], commit_times=ct, **c["kw"])
        sim.create(c["max_clock"])
        sims.append(sim)
    return sims


def sweep_pair():
    delays, configs = grid_256()
    sims = []
    for ct in (False, True):
        sim = SweepSimulator.grid(256, delays, configs, num_nodes=4, commit_times=ct)
        sim.create(1000)
        sims.append(sim)
    return sims


def measure(sims, rounds):
    """Alternating runs of the flag-off and flag-on handles: kernel ms of each, identical outputs, read-out ms."""
    ms = ([], [])
    for _ in range(rounds + 1):  # (the first round warms up)
        for j, sim in enumerate(sims):
            sim.run(strict=False)
            ms[j].append(float(sim.timing.sim_ms))
    off, on = (sim.run(strict=False) for sim in sims)
    same = all(np.array_equal(a, b) for a, b in ((off.commit_counts, on.commit_counts), (off.last_committed_states, on.last_committed_states),
                                               (off.counters, on.counters), (off.status, on.status)))
    t0 = time.perf_counter()
    committed, proposed = on.commit_times()
    readout_ms = (time.perf_counter() - t0) * 1e3
    lat = on.commit_latencies(committed.shape[2])
    out = {"kernel_off": sims[0].kernel_info(), "kernel_on": sims[1].kernel_info(), "identical_outputs": bool(same),
           "readout_ms_incl_copy": readout_ms, "cap": int(committed.shape[2]),
           "mean_latency_ms": float(lat[lat >= 0].mean()) if (lat >= 0).any() else None,
           "device_bytes_off": sims[0].memory_info()[0], "device_bytes_on": sims[1].memory_info()[0]}
    for name, v in (("off", ms[0][1:]), ("on", ms[1][1:])):
        out["ms_" + name] = {"min": min(v), "median": float(np.median(v)), "all": v}
    out["on_over_off_min"] = out["ms_on"]["min"] / out["ms_off"]["min"]
    out["on_over_off_median"] = out["ms_on"]["median"] / out["ms_off"]["median"]
    for sim in sims:
        sim.close()
    return out


def build_times(trees, rounds):
    """Wall and CPU seconds of _build.build_product(force=True) of each tree, alternated over the rounds."""
    out = {t: {"wall_s": [], "cpu_s": []} for t in trees}
    for _ in range(rounds):
        for i, tree in enumerate(trees):
            spec = importlib.util.spec_from_file_location("build_%d" % i, os.path.join(tree, "librabft_simulator_b200", "_build.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            tmp = tempfile.mkdtemp()
            lib = os.path.join(tmp, "liblbft_timed.so")
            r0, t0 = resource.getrusage(resource.RUSAGE_CHILDREN), time.perf_counter()
            mod.build_product(force=True, lib_path=lib)
            wall, r1 = time.perf_counter() - t0, resource.getrusage(resource.RUSAGE_CHILDREN)
            out[tree]["wall_s"].append(wall)
            out[tree]["cpu_s"].append((r1.ru_utime - r0.ru_utime) + (r1.ru_stime - r0.ru_stime))
            shutil.rmtree(os.path.join(mod.CSRC, "build_" + os.path.basename(lib)), ignore_errors=True)  # its object files
            shutil.rmtree(tmp)
    return {"cpus": os.cpu_count(), "trees": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default="1,2,3,4,5")
    ap.add_argument("--out", help="also write the JSON object to this file")
    ap.add_argument("--build", nargs="+", metavar="TREE", help="time full builds of these source trees instead")
    args = ap.parse_args()
    if args.build:
        res = build_times([os.path.abspath(t) for t in args.build], args.rounds)
        print(json.dumps(res, indent=1))
        return
    res = {"card": card(), "rounds": args.rounds}
    for cid in [int(c) for c in args.configs.split(",") if c]:
        res["config%d" % cid] = measure(make_pair(cid), args.rounds)
    res["sweep_256x256"] = measure(sweep_pair(), args.rounds)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
