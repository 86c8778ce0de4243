"""The device sampler against the oracle and exact arithmetic, through the sampler probe (tests/gpuprobe/sampler_probe.cu): every
case group of tests/rng_support.py (seeding and steps, the shuffle's u32 range draws at n = 1..64, the u64 range draws and the
uniform delays at spans 1, 2, 2^k, 2^k + 1, 3 * 2^k and 2^29 + 1 at their rejection boundary, the ziggurat at every layer's
fast-accept boundary, wedge decision and tail loop boundary up to the largest deviate, delay_from_z at every threshold of
tables either side of the shared-memory limit and at the 4096 cap, sample_delay through every delay kind, the exp()
fallback's near-integer band and 1e9 cap) on the generic plain core, the bench kernel's FX_DEFAULT4 core and the sweep core
(every model one set of one sweep, so that thr_off != 0), with 1, 8 and 32 lanes per record and the tables in shared or global
memory; and 2^24 SplitMix64-seeded states through standard_normal and sample_delay at the reference's delay models.

Results are bit-identical to the oracle except where the device's exp / log (CUDA's libm, which the cold paths call) returns
another double than glibc's for an argument the case's ziggurat evaluates: there the wedge decision or the tail deviate may
differ.  Each test prints how many inputs it probed and how many libm differences it met."""
import math

import numpy as np
import pytest

from tests.rng_support import (CORE_FIXED, CORE_PLAIN, CORE_SWEEP, FALLBACK_MODELS, LANES_DISAGREE, MODELS, OP_EXP, OP_LOG,
                               OP_NORMAL, OP_SAMPLE_DELAY, TABLE_MODELS, Setup, Sides,
                               StateSolver, b2f, case_groups, uniform_model, check_fallback, exact_floor_delay, f2b, glibc_delay, model_of,
                               records, same, traced_libm_calls)

pytestmark = pytest.mark.gpu

CONFIGS = ([(CORE_PLAIN, g, m) for g in (1, 8, 32) for m in (True, False)] + [(CORE_FIXED, 1, m) for m in (True, False)]
           + [(CORE_SWEEP, g, m) for g in (1, 8, 32) for m in (True, False)])
CONFIG_IDS = ["%s-G%d-%s" % (("plain", "fixed", "sweep")[c], g, "smem" if m else "global") for c, g, m in CONFIGS]


@pytest.fixture(scope="module")
def sides():
    return Sides(gpu=True)


@pytest.fixture(scope="module")
def cases(sides):
    groups, tabs = case_groups(sides, StateSolver())
    # one sweep over every model: a set's thresholds start at its own thr_off
    keys = sorted({model_key(m) for m, _ in groups.values()})
    sweep_models = [uniform_model(int(k[8:])) if k.startswith("uniform:") else MODELS[k] for k in keys]
    return groups, tabs, keys, Setup(sets=sweep_models)


class LibmDiffs:
    """The device's exp / log against glibc's (math.exp / math.log) at the arguments a case's ziggurat evaluates."""

    def __init__(self, sides):
        self.sides, self.known = sides, {}

    def differs(self, calls_per_record):
        todo = sorted({c for calls in calls_per_record for c in calls} - set(self.known))
        for op, fn in ((OP_EXP, "exp"), (OP_LOG, "log")):
            args = [a for f, a in todo if f == fn]
            if args:
                recs = records(np.ones((len(args), 4), np.uint64), op, np.array([f2b(a) for a in args], np.uint64))
                dev = self.sides.run_device(Setup(MODELS["baseline"]), recs, CORE_PLAIN, 1, False)
                for a, r in zip(args, dev):
                    want = getattr(math, fn)(a)
                    self.known[(fn, a)] = b2f(r["result"]) != want
        return np.array([any(self.known[c] for c in calls) for calls in calls_per_record], bool)

    def count(self):
        return sum(self.known.values()), len(self.known)


@pytest.fixture(scope="module")
def libm(sides):
    return LibmDiffs(sides)


def run_config(sides, cases, config, group):
    """The group's records on the device under `config`, and the oracle's."""
    groups, _, keys, sweep = cases
    core, G, smem = config
    m, recs = groups[group]
    name = model_key(m)
    ref = sides.run_oracle(Setup(model_of(m)), recs)
    if core == CORE_SWEEP:
        r = recs.copy()
        r["set"] = keys.index(name)
        dev = sides.run_device(sweep, r, core, G, smem)
        dev["set"] = 0
    else:
        dev = sides.run_device(Setup(model_of(m)), recs, core, G, smem)
    assert not (dev["status"] & LANES_DISAGREE).any(), (group, config)
    return recs, dev, ref


def model_key(m):
    """A case group's model as a MODELS key or "uniform:<span>"."""
    return m if isinstance(m, str) else "uniform:%d" % (m["delay_hi"] - m["delay_lo"] + 1)


def fixed_ok(core, m):
    return core != CORE_FIXED or m in TABLE_MODELS


@pytest.mark.parametrize("config", CONFIGS, ids=CONFIG_IDS)
def test_integer_ops_are_bit_identical(sides, cases, config):
    recs, dev, ref = run_config(sides, cases, config, "integers")
    assert same(dev, ref).all() and not dev["status"].any()
    n = 0
    for g in cases[0]:
        if g.startswith("uniform:") and config[0] != CORE_FIXED:
            recs, dev, ref = run_config(sides, cases, config, g)
            assert same(dev, ref).all() and not dev["status"].any(), g
            n += len(recs)
    print("integers %s: %d records, %d uniform delays, 0 differences" % (config, len(cases[0]["integers"][1]), n))


@pytest.mark.parametrize("config", CONFIGS, ids=CONFIG_IDS)
def test_ziggurat_edges(sides, cases, libm, config):
    groups, (zx, zf, R), _, _ = cases
    recs, dev, ref = run_config(sides, cases, config, "normal")
    differs = libm.differs(traced_libm_calls(recs, zx, zf, R))
    ok = same(dev, ref)
    assert ok[~differs].all(), np.nonzero(~ok & ~differs)[0][:8]
    assert not dev["status"].any()
    print("ziggurat %s: %d inputs, %d with a device/glibc libm difference (%d decisions or deviates differ there); "
          "libm arguments probed so far %d, differing %d" % (config, len(recs), differs.sum(), (~ok).sum(), libm.count()[1],
                                                            libm.count()[0]))


@pytest.mark.parametrize("config", CONFIGS, ids=CONFIG_IDS)
def test_delays_through_tables_and_constant(sides, cases, libm, config):
    """delay_from_z at every threshold, the double below it, +-ZMAX and the largest deviates equals glibc's (int64) exp(mu +
    sigma z) (and the oracle's); sample_delay on the ziggurat's edge states through every table model and the constant model
    equals the oracle's wherever the case's libm values agree."""
    groups, (zx, zf, R), _, _ = cases
    core = config[0]
    probed = exact_off = 0
    for name in TABLE_MODELS:
        if not fixed_ok(core, name):
            continue
        recs, dev, ref = run_config(sides, cases, config, "delay_from_z:" + name)
        model = sides.tables(Setup(MODELS[name]))[3][0][0]
        zs = recs["arg"].view(np.float64)
        want = np.array([glibc_delay(model.mu, model.sigma, float(z)) for z in zs], np.int64)
        assert (dev["result"].view(np.int64) == want).all() and (ref["result"].view(np.int64) == want).all(), name
        probed += len(recs)
        if config == CONFIGS[0]:
            exact_off += sum(exact_floor_delay(model.mu, model.sigma, float(z)) != w for z, w in zip(zs, want))
    for name in TABLE_MODELS + ["const"]:
        if not fixed_ok(core, name):
            continue
        recs, dev, ref = run_config(sides, cases, config, "sample_delay:" + name)
        differs = libm.differs(traced_libm_calls(recs, zx, zf, R))
        ok = same(dev, ref)
        assert ok[~differs].all() and not dev["status"].any(), name
        probed += len(recs)
    print("delays %s: %d inputs, 0 differences from glibc; glibc vs exact floor differs at %d" % (config, probed, exact_off))


@pytest.mark.parametrize("config", [c for c in CONFIGS if c[0] != CORE_FIXED], ids=[i for c, i in zip(CONFIGS, CONFIG_IDS)
                                                                                    if c[0] != CORE_FIXED])
def test_exp_fallback_flags(sides, cases, libm, config):
    """Past the 4096 cap: a delay that differs from the oracle's carries ST_DELAY_NEAR_INT, the flag fires only within its
    1e-9 band (mpmath), and a delay at or past 1e9 is 1e9 with ST_TIME_OVERFLOW."""
    groups, (zx, zf, R), _, _ = cases
    for name in FALLBACK_MODELS:
        recs, dev, ref = run_config(sides, cases, config, "fallback:" + name)
        differs = libm.differs(traced_libm_calls(recs, zx, zf, R))
        model = sides.tables(Setup(MODELS[name]))[3][0][0]
        flagged, overflowed, differing = check_fallback(recs, dev, ref, model, zx, zf, R, differs)
        assert flagged and (overflowed > 0) == (name == "wide")
        print("fallback %s %s: %d inputs, %d flagged near-integer, %d at the 1e9 cap, %d delays differ from glibc's (all "
              "flagged), %d with a libm difference" % (name, config, len(recs), flagged, overflowed, differing, differs.sum()))


NATURAL = 1 << 24
CHUNK = 1 << 21


def splitmix_states(seeds):
    """seed_from_u64 of every seed, vectorised (uint64 arithmetic wraps)."""
    x = seeds.astype(np.uint64)
    out = np.zeros((len(seeds), 4), np.uint64)
    with np.errstate(over="ignore"):
        for i in range(4):
            x = x + np.uint64(0x9E3779B97F4A7C15)
            z = x
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            out[:, i] = z ^ (z >> np.uint64(31))
    return out


@pytest.mark.parametrize("core", [CORE_PLAIN, CORE_FIXED])
def test_natural_rate_pass(sides, core):
    """2^24 seeded states through standard_normal and sample_delay (LogNormal(10, 4), and uniform [5, 15] on the plain core):
    only tail deviates may differ, by at most an ulp, with the same state and draws, and no delay differs."""
    tail_ulp = tail = 0
    models = ["baseline"] + (["uniform"] if core == CORE_PLAIN else [])
    for start in range(0, NATURAL, CHUNK):
        states = splitmix_states(np.arange(start, start + CHUNK, dtype=np.uint64) * np.uint64(0x2545F4914F6CDD1D) + np.uint64(52))
        recs = records(states, OP_NORMAL)
        setup = Setup(MODELS["baseline"])
        dev, ref = sides.run_device(setup, recs, core, 1, True), sides.run_oracle(setup, recs)
        z = ref["result"].view(np.float64)
        tail += int((np.abs(z) >= 3.6541528853610088).sum())
        off = dev["result"] != ref["result"]
        assert ((dev["s"] == ref["s"]).all(axis=1) & (dev["draws"] == ref["draws"])).all()
        d = np.abs(dev["result"].astype(np.int64) - ref["result"].astype(np.int64))
        assert (d[off] == 1).all() and (np.abs(z[off]) >= 3.6541528853610088).all()
        tail_ulp += int(off.sum())
        for name in models:
            recs["op"] = OP_SAMPLE_DELAY
            setup = Setup(MODELS[name])
            dev, ref = sides.run_device(setup, recs, core, 1, True), sides.run_oracle(setup, recs)
            assert same(dev, ref).all() and not dev["status"].any(), name
    print("natural rate core %d: %d states, %d tail deviates, %d of them an ulp off glibc's, 0 delay differences" % (
        core, NATURAL, tail, tail_ulp))
