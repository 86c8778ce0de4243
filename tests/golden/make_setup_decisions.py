#!/usr/bin/env python
"""Generates tests/golden/setup_decisions.json: what the host setup (HostSetup::build / build_sweep, through the host harness
in tests/hostcore) decides for a few hundred configurations placed on the boundaries of its procedure.  Each entry holds
the case and, under "want", tests/test_setup_decisions.py::decisions of it.  Re-run after changing a decision on purpose:
    python tests/golden/make_setup_decisions.py"""
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.support import HostCore  # noqa: E402
from tests.sweep_support import SweepHostCore  # noqa: E402
from tests.test_setup_decisions import decisions  # noqa: E402

NODES = (1, 2, 3, 4, 5, 6, 16, 17, 32, 33, 64)
INSTANCES = (4096, 4097, 12288, 12289, 24576, 24577, 49152, 49153, 65536)
CLOCKS = (1000, 1791, 1792, 3583, 3584, 4095, 4096, 14628, 14629, 16319, 16320, 20000)
FORCE = (None, "thread", "wide")


def pset(kind=0, mean=10.0, variance=4.0, lo=0, hi=0, tci=100000, delta=20, gamma=2.0, lambda_=0.5, reserved=0):
    return dict(delay_kind=kind, reserved=reserved, delay_mean=mean, delay_variance=variance, delay_lo=lo, delay_hi=hi,
                target_commit_interval=tci, delta=delta, gamma=gamma, lambda_=lambda_)


DELAYS = {"ref": {}, "const": dict(delay_variance=0.0), "wide": dict(delay_mean=25.0, delay_variance=200.0),
          "table2k": dict(delay_mean=15.0, delay_variance=30.0), "short": dict(delay_mean=0.5, delay_variance=0.1),
          "uni1": dict(delay_kind=1, delay_lo=1, delay_hi=1), "uni0": dict(delay_kind=1, delay_lo=0, delay_hi=0),
          "uni5_15": dict(delay_kind=1, delay_lo=5, delay_hi=15)}
SET_LISTS = {"ref": [pset()], "mixed": [pset(), pset(mean=5.0, variance=2.0), pset(variance=0.0), pset(kind=1, lo=1, hi=4)],
             "fast_uniform": [pset(), pset(kind=1, lo=1, hi=1)], "wide_table": [pset(mean=25.0, variance=200.0), pset(mean=15.0, variance=30.0)],
             "pacemaker": [pset(delta=15, gamma=1.5, lambda_=1.0), pset(tci=300, delta=100), pset(delta=10, lambda_=2.0)],
             "bad_delta": [pset(), pset(delta=0)], "bad_mean": [pset(), pset(), pset(mean=-1.0)],
             "bad_uniform": [pset(kind=1, lo=5, hi=2)], "bad_kind": [pset(kind=7)], "reserved": [pset(), pset(reserved=1)]}


def case(name, nodes=4, instances=64, max_clock=1000, force=None, sets=None, **kw):
    c = dict(name=name, nodes=nodes, instances=instances, max_clock=max_clock, force=force, kw=kw)
    if sets is not None:
        c["sets"] = SET_LISTS[sets]
    return c


def cases():
    out = [case("grid N=%d I=%d" % (n, i), n, i) for n, i in itertools.product(NODES, INSTANCES)]
    out += [case("forced %s N=%d I=%d" % (f, n, i), n, i, force=f)
            for f, n, i in itertools.product(FORCE[1:], (1, 4, 6, 7, 16, 17, 64), (1024, 4097, 16384, 65536))]
    out += [case("clock %d N=%d I=%d %s" % (mc, n, i, f), n, i, mc, f)
            for mc, n, i, f in itertools.product(CLOCKS, (4, 7, 16), (64, 65536), (None, "wide"))]
    out += [case("long %d N=%d" % (mc, n), n, 64, mc, round_cap=128)
            for mc, n in itertools.product((892857, 892858, 16777151, 16777152), (4, 5))]
    out += [case("queue_cap %d N=%d I=%d" % (q, n, i), n, i, queue_cap=q)
            for q, n, i in itertools.product((0, 64, 65, 512, 513, 1024, 1025, 65520, 65521, 1 << 20, (1 << 20) + 1), (4, 5, 8, 64),
                                             (64, 16384))]
    out += [case("payload_cap %d N=%d I=%d" % (p, n, i), n, i, payload_cap=p)
            for p, n, i in itertools.product((0, 255, 256, 65519, 65520), (4, 8, 16), (64, 65536))]
    out += [case("round_cap %d N=%d" % (r, n), n, 64, 1000, round_cap=r) for r, n in itertools.product((1, 31, 32, 33, 32768, 32769), (4, 16))]
    out += [case("epochs cpe=%d N=%d I=%d mc=%d flags=%d" % (e, n, i, mc, fl), n, i, mc, commands_per_epoch=e, flags=fl)
            for e, n, i, mc, fl in itertools.product((1, 5, 127, 128), (4, 16), (64, 16384), (1000, 20000), (0, 3))]
    out += [case("epochs cpe=5 N=4 queue_cap=%d" % q, 4, 64, 1000, commands_per_epoch=5, queue_cap=q) for q in (64, 100, 512, 1024)]
    out += [case("flags %d N=%d I=%d" % (fl, n, i), n, i, flags=fl)
            for fl, n, i in itertools.product((1, 2, 3, 4, 5, 6, 8), (4, 7, 40), (64, 65536))]
    out += [case("data-sync N=%d payload_cap=%d" % (n, p), n, 64, flags=4, payload_cap=p) for n, p in itertools.product((3, 6, 12), (0, 100))]
    out += [case("delay %s N=%d I=%d" % (d, n, i), n, i, **DELAYS[d])
            for d, n, i in itertools.product(DELAYS, (4, 8, 16), (64, 16384))]
    out += [case("voting rights", 4, voting_rights=[1, 2, 3, 4]), case("silent", 7, silent=[0, 1, 0, 0, 0, 0, 1]),
            case("partitions 4", 7, 16384, partition_windows=4, partition_max_len=150), case("partitions 64", 7, partition_windows=64),
            case("pacemaker", 4, delta=15, gamma=1.5, lambda_=1.0, target_commit_interval=1 << 31)]
    bad = [("num_instances", dict(instances=0)), ("num_nodes 0", dict(nodes=0)), ("num_nodes 65", dict(nodes=65)),
           ("max_clock -1", dict(max_clock=-1)), ("max_clock 2^29", dict(max_clock=1 << 29)), ("flags tds+rec", dict(flags=5)),
           ("commands_per_epoch 0", dict(commands_per_epoch=0)), ("delta -1", dict(delta=-1)), ("tci -1", dict(target_commit_interval=-1)),
           ("delta 0", dict(delta=0)), ("mean 0", dict(delay_mean=0.0)), ("variance -1", dict(delay_variance=-1.0)),
           ("const delay huge", dict(delay_mean=1e12, delay_variance=0.0)), ("uniform hi<lo", dict(delay_kind=1, delay_lo=5, delay_hi=2)),
           ("uniform hi 2^29+1", dict(delay_kind=1, delay_lo=0, delay_hi=(1 << 29) + 1)), ("delay_kind 2", dict(delay_kind=2)),
           ("voting rights 2^24+1", dict(voting_rights=[1 << 24 | 1, 1, 1, 1])), ("voting rights 0", dict(voting_rights=[0, 0, 0, 0])),
           ("partition_windows 65", dict(partition_windows=65)), ("tds epochs", dict(flags=4, commands_per_epoch=5)),
           ("num_nodes 0 and delta 0", dict(nodes=0, delta=0)), ("delta 0 and flags 8", dict(delta=0, flags=8))]
    out += [case("refused " + name, **kw) for name, kw in bad]
    shapes = ((4, 64, 1000), (4, 65536, 1000), (7, 16384, 1000), (8, 1000, 1000), (64, 8192, 1000), (7, 64, 20000))
    out += [case("sweep %s N=%d I=%d mc=%d %s" % (lst, n, i, mc, f), n, i, mc, f, sets=lst)
            for lst, (n, i, mc), f in itertools.product(list(SET_LISTS)[:5], shapes, FORCE)]
    out += [case("sweep refused %s N=%d I=%d" % (lst, n, i), n, i, mc, sets=lst) for lst in list(SET_LISTS)[5:] for n, i, mc in shapes[:2]]
    out += [case("sweep refused " + name, sets="ref", **kw) for name, kw in bad if "instances" not in kw]
    out += [case("sweep refused flags 1", sets="mixed", flags=1), case("sweep refused epochs", sets="mixed", commands_per_epoch=5),
            case("sweep refused too many sets", 4, 2, sets="mixed")]
    return out


def main():
    hostcore, sweep = HostCore(), SweepHostCore()
    out = []
    for c in cases():
        c["want"] = decisions(hostcore, sweep, c)
        out.append(c)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "setup_decisions.json"), "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(c, separators=(",", ":")) for c in out) + "\n]\n")  # one case per line
    print("wrote %d cases, %d refused" % (len(out), sum("error" in c["want"] for c in out)))


if __name__ == "__main__":
    main()
