"""The sampler without a GPU: the Xoshiro state solver, the Python restatements of SplitMix64 seeding, Xoshiro256**, rand's
range draws and the ziggurat against the oracle, the product's delay threshold tables against glibc and mpmath, and the
host-compiled twin of the sampler probe (tests/hostcore/sampler_hostcore.cpp: the probe's op dispatcher over the kernels' Core
instantiations) against the oracle on every edge case group the GPU test runs (tests/test_gpu_sampler.py), so that a
regression in the sampler or in the cases fails here before a GPU run.  Also the probe cross-compiling for sm_90a."""
import math
import subprocess

import numpy as np
import pytest

from librabft_simulator_b200 import _build
from tests.rng_support import (CORE_FIXED, CORE_PLAIN, FALLBACK_MODELS, KMAX, MODELS, OP_NEXT_U64, OP_NORMAL, OP_RANGE_U32,
                               OP_RANGE_U64, OP_SEED, TABLE_MODELS, ZMAX, Setup, Sides,
                               StateSolver, case_groups, check_fallback, exact_floor_delay, glibc_delay, largest_deviate,
                               model_of, records, same, sample_single_inclusive, splitmix_seed, standard_normal, xoshiro_next)


@pytest.fixture(scope="module")
def sides():
    return Sides()


@pytest.fixture(scope="module")
def solver():
    return StateSolver()


@pytest.fixture(scope="module")
def groups(sides, solver):
    return case_groups(sides, solver)


def test_state_solver_emits_the_chosen_outputs(solver):
    rng = np.random.default_rng(3)
    outs = rng.integers(0, 1 << 63, (64, 4), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, (64, 4), dtype=np.uint64)
    outs[0] = [1, 0, 0, 0]
    outs[1] = [0, 0, 0, 1]
    outs[2] = [np.uint64((1 << 64) - 1)] * 4
    for o, s in zip(outs, solver.solve(outs)):
        assert s.any()
        s = [int(v) for v in s]
        for k in range(4):
            v, s = xoshiro_next(s)
            assert v == int(o[k])
    with pytest.raises(AssertionError):
        solver.solve([[0, 0, 0, 0]])


def test_restatements_match_the_oracle(sides, solver):
    rng = np.random.default_rng(4)
    setup = Setup(MODELS["baseline"])
    zx, zf, R, _ = sides.tables(setup)
    seeds = np.array([0, 1, 52, (1 << 64) - 1] + list(rng.integers(0, 1 << 63, 60, dtype=np.uint64)), np.uint64)
    got = sides.run_oracle(setup, records(np.ones((len(seeds), 4), np.uint64), OP_SEED, seeds))
    assert [list(map(int, g["s"])) for g in got] == [splitmix_seed(int(s)) for s in seeds]
    states = solver.solve(rng.integers(1, 1 << 63, (2000, 4), dtype=np.uint64))
    for op, fn in ((OP_NEXT_U64, None), (OP_RANGE_U32, 32), (OP_RANGE_U64, 64), (OP_NORMAL, "normal")):
        ns = rng.integers(1, 1 << 31, len(states)) if fn == 32 else rng.integers(1, 1 << 63, len(states), dtype=np.uint64)
        recs = records(states, op, ns if fn in (32, 64) else 0)
        out = sides.run_oracle(setup, recs)
        for r, o in zip(recs, out):
            s = [int(v) for v in r["s"]]
            if fn is None:
                v, s2 = xoshiro_next(s)
                want, d = v, 1
            elif fn == "normal":
                z, s2, d, _ = standard_normal(s, zx, zf, R)
                want = int(np.float64(z).view(np.uint64))
            else:
                want, s2, d = sample_single_inclusive(s, int(r["arg"]), fn)
            assert (int(o["result"]), [int(v) for v in o["s"]], int(o["draws"])) == (want, s2, d)


@pytest.mark.parametrize("name", TABLE_MODELS + FALLBACK_MODELS)
def test_delay_tables_against_glibc_and_mpmath(sides, name):
    """thr[0] = -inf, thr[kmax + 1] = +inf, and thr[k] the smallest double z with (int64) exp(mu + sigma z) >= k under glibc
    for every k; kmax the delay at ZMAX, above the largest deviate the sampler returns.  Where mpmath's exact floor disagrees
    with glibc at a threshold, the table follows glibc by design; the count is reported."""
    _, _, R, per = sides.tables(Setup(MODELS[name]))
    m, thr = per[0]
    assert m.delay_kmax == KMAX[name]
    if not m.delay_kmax:
        assert len(thr) == 0
        return
    assert largest_deviate(R) < ZMAX
    kmax = m.delay_kmax
    assert glibc_delay(m.mu, m.sigma, ZMAX) == kmax and len(thr) == kmax + 2
    assert thr[0] == -math.inf and thr[kmax + 1] == math.inf
    disagree = neg = 0
    for k in range(1, kmax + 1):
        t = float(thr[k])
        if t == -math.inf:
            assert glibc_delay(m.mu, m.sigma, -ZMAX) >= k
            neg += 1
            continue
        below = math.nextafter(t, -math.inf)
        assert glibc_delay(m.mu, m.sigma, t) >= k > glibc_delay(m.mu, m.sigma, below), k
        for z in (t, below):
            disagree += exact_floor_delay(m.mu, m.sigma, z) != glibc_delay(m.mu, m.sigma, z)
    if name == "narrow":
        assert neg == glibc_delay(m.mu, m.sigma, -ZMAX) > 0
    print("%s: kmax %d, %d thresholds at -inf, glibc vs exact floor differs at %d of %d probed z" % (
        name, kmax, neg, disagree, 2 * (kmax - neg)))


def test_host_twin_matches_the_oracle(sides, groups):
    """Every case group through the host twin's plain core (and the fixed core on models with a table): bit-identical to the
    oracle, the twin's libm being glibc; the exp() fallback differs only at the 1e9 cap, where it raises ST_TIME_OVERFLOW."""
    cases, (zx, zf, R) = groups
    for g, (m, recs) in cases.items():
        setup = Setup(model_of(m))
        ref = sides.run_oracle(setup, recs)
        for core in [CORE_PLAIN] + ([CORE_FIXED] if m in TABLE_MODELS else []):
            got = sides.run_host(setup, recs, core)
            if g.startswith("fallback:"):
                flagged, overflowed, differing = check_fallback(recs, got, ref, sides.tables(setup)[3][0][0], zx, zf, R,
                                                                np.zeros(len(recs), bool))
                assert flagged and differing == 0 and (overflowed > 0) == (m == "wide"), g
                continue
            assert same(got, ref).all(), (g, core, np.nonzero(~same(got, ref))[0][:8])
            assert not got["status"].any(), g


def test_case_groups_reach_every_branch(sides, groups):
    """The edge cases reach what they are for: the wedge on both sides at every layer 1..255, the tail's loop both ways, the
    largest deviate, and draws past the first at the range draws' rejection boundary."""
    cases, (zx, zf, R) = groups
    _, recs = cases["normal"]
    out = sides.run_oracle(Setup(MODELS["baseline"]), recs)
    layers_acc, layers_rej, tail_loops, zmax = set(), set(), 0, 0.0
    for r, o in zip(recs, out):
        s = [int(v) for v in r["s"]]
        first, _ = xoshiro_next(s)
        z, _, d, calls = standard_normal(s, zx, zf, R)
        if calls and calls[0][0] == "exp":
            (layers_acc if d == 2 else layers_rej).add(first & 0xFF)
        if calls and calls[0][0] == "log" and len(calls) > 2:
            tail_loops += 1
        zmax = max(zmax, abs(z))
    assert layers_acc == set(range(1, 256)) and layers_rej == set(range(1, 256))
    assert tail_loops > 0 and zmax == largest_deviate(R)
    _, recs = cases["integers"]
    out = sides.run_oracle(Setup(MODELS["baseline"]), recs)
    for op in (OP_RANGE_U32, OP_RANGE_U64):
        assert (out["draws"][recs["op"] == op] > 1).sum() > 64


def test_probe_cross_compiles_for_sm_90a():
    path = _build.build_sampler_probe(force=True)
    elves = subprocess.run(["cuobjdump", "--list-elf", path], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in elves
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    assert sass.count("Function : ") == 2 * (3 + 1 + 3) and "sampler_probe_kernel" in sass
