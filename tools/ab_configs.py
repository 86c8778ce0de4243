#!/usr/bin/env python
"""Isolated A/B of the kernels the BASELINE configurations select: time each configuration of bench.py's CONFIGS (its
instances, nodes, max_clock, base seed and inputs) against each library given on the command line, alternating, through
the plain C ABI (works with older builds of the library too).  Prints the kernel each library selects.
Usage: python tools/ab_configs.py [--rounds R] A.so B.so [C.so ...]"""
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import CONFIGS  # noqa: E402
from librabft_simulator_b200._lib import LbftTiming  # noqa: E402
from tests.support import make_config  # noqa: E402


def time_one(lib, I, N, max_clock, base_seed, kw, reps=3):
    cfg, keep = make_config(np.arange(base_seed, base_seed + I, dtype=np.uint64), N, max_clock, **kw)
    h = ctypes.c_void_p()
    assert lib.lbft_create(ctypes.byref(cfg), ctypes.byref(h)) == 0, lib.lbft_last_error()
    best = 1e30
    for _ in range(reps + 1):
        assert lib.lbft_run(h) == 0, lib.lbft_last_error()
        t = LbftTiming()
        lib.lbft_timing_info(h, ctypes.byref(t))
        best = min(best, t.sim_ms)
    kernel = ctypes.create_string_buffer(256)
    lib.lbft_kernel_info(h, kernel, len(kernel))
    states = np.zeros((I, N), np.uint64)
    lib.lbft_last_states(h, ctypes.c_void_p(states.ctypes.data))
    lib.lbft_destroy(h)
    return best, int(np.bitwise_xor.reduce(states.reshape(-1))), kernel.value.decode()


args = sys.argv[1:]
rounds = 2
if args and args[0] == "--rounds":
    rounds, args = int(args[1]), args[2:]
libs = []
for path in args:
    lib = ctypes.CDLL(os.path.abspath(path))
    lib.lbft_last_error.restype = ctypes.c_char_p
    lib.lbft_create.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]
    for fn in ("lbft_run", "lbft_destroy"):
        getattr(lib, fn).argtypes = [ctypes.c_void_p]
    lib.lbft_timing_info.argtypes = [ctypes.c_void_p, ctypes.POINTER(LbftTiming)]
    lib.lbft_last_states.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.lbft_kernel_info.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t]
    libs.append((os.path.basename(path), lib))
for cid, c in sorted(CONFIGS.items()):
    res = {n: [] for n, _ in libs}
    kernels = {}
    digests = set()
    for _ in range(rounds):
        for n, lib in libs:
            ms, dig, kernels[n] = time_one(lib, c["instances"], c["nodes"], c["max_clock"], c["base_seed"], c["kw"])
            res[n].append(ms)
            digests.add(dig)
    print("config%d %dx%d max_clock=%d   (same results everywhere: %s)" % (cid, c["instances"], c["nodes"], c["max_clock"],
                                                                          len(digests) == 1))
    for n, _ in libs:
        print("    %-28s %s ms   %s" % (n, " / ".join("%.2f" % v for v in res[n]), kernels[n]))
