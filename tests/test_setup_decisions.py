"""The host setup's decisions pinned per configuration (tests/golden/setup_decisions.json, made by
tests/golden/make_setup_decisions.py).  Each case sits on a boundary of HostSetup::build / build_sweep (committee sizes, batch
sizes, horizons, capacities, epochs, flags, delay models, LBFT_FORCE_KERNEL, sweep set lists, refusals) and records the layout
summary, the epoch count, the kernel, and one digest of the Params bytes and every host table, or the error text.  A change
that moves a decision on purpose regenerates the file, and its diff shows which decisions moved."""
import ctypes
import json
import os

import numpy as np
import pytest

from librabft_simulator_b200._lib import LbftParamSet
from tests.support import P, make_config
from tests.sweep_support import SweepHostCore

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "setup_decisions.json")


def decisions(hostcore, sweep, case):
    """What the host setup makes of one case: {"error": text} or the layout summary, epochs, kernel name and digest."""
    I = case["instances"]
    cfg, keep = make_config(np.arange(1, I + 1, dtype=np.uint64), case["nodes"], case["max_clock"], **case["kw"])
    if "sets" in case:
        sets = (LbftParamSet * max(1, len(case["sets"])))(*[LbftParamSet(**s) for s in case["sets"]])
        set_of = np.ascontiguousarray(np.arange(I) % max(1, len(case["sets"])), dtype=np.uint32)
        lib, err = sweep.lib, sweep.lib.hostcore_sweep_last_error
        args = (ctypes.byref(cfg), sets, len(case["sets"]), P(set_of.ctypes.data))
        digest_fn, kernel_fn = lib.hostcore_sweep_setup_digest, lib.hostcore_kernel_info_sweep
    else:
        lib, err = hostcore.lib, hostcore.lib.hostcore_last_error
        args = (ctypes.byref(cfg),)
        digest_fn, kernel_fn = lib.hostcore_setup_digest, lib.hostcore_kernel_info
    if case.get("force"):
        os.environ["LBFT_FORCE_KERNEL"] = case["force"]
    try:
        digest, epochs, info = ctypes.c_uint64(), ctypes.c_uint32(), np.zeros(6, np.uint32)
        if "sets" in case:
            rc = digest_fn(*args, ctypes.byref(digest))
        else:
            rc = digest_fn(*args, ctypes.byref(digest), ctypes.byref(epochs))
        if rc != 0:
            return {"error": err().decode()}
        buf = ctypes.create_string_buffer(128)
        assert kernel_fn(*args, buf, ctypes.sizeof(buf)) == 0
        out = {"kernel": buf.value.decode(), "digest": "%016x" % digest.value}
        if "sets" not in case:
            assert lib.hostcore_setup_info(ctypes.byref(cfg), P(info.ctypes.data)) == 0
            out.update(info=info.tolist(), epochs=epochs.value)
        return out
    finally:
        os.environ.pop("LBFT_FORCE_KERNEL", None)


@pytest.fixture(scope="module")
def sweep():
    return SweepHostCore()


def test_setup_decisions_match_fixture(hostcore, sweep, monkeypatch):
    monkeypatch.delenv("LBFT_FORCE_KERNEL", raising=False)
    cases = json.load(open(FIXTURE))
    assert len(cases) >= 300 and sum("sets" in c for c in cases) >= 20 and sum("error" in c["want"] for c in cases) >= 20
    moved = [(c["name"], c["want"], got) for c in cases for got in [decisions(hostcore, sweep, c)] if got != c["want"]]
    assert not moved, "%d of %d cases moved, first: %r" % (len(moved), len(cases), moved[:3])
