"""The compact node / notification encoding of the four-author compile-time layout (sim_core.cuh Core::PACK, FX_DEFAULT4: the
BASELINE config 2/3 kernel, and every handle whose layout is make_layout(4, 128, 64, 32, 0, 2)) at the limits of its
byte-wide fields.

* The field table: where each F_* scalar and author mask lives, as the layout comment of sim_core.cuh documents it, and
  that every field holds its documented bound.
* Round trips of extreme and random values through store_node / put_timeout_hcbr / copy_timeout_hcbr_to_tc and back
  through load_node / node_ld / hcbr_of, with every other word of the warp tile left alone.
* Whole runs that reach the top of the byte fields (round ids up to 127, ~120 commits, timeout certificates, complete
  timeout sets, round and queue overflow), compared field by field with the generic instantiation on the same layout and,
  where no error bit is set, with the oracle.  The compact run must leave the words of the generic layout that it does not
  use at their fill value: that is what keeps a 65 536-instance batch inside an H100's L2."""
from types import SimpleNamespace

import numpy as np
import pytest

from librabft_simulator_b200._lib import ST_ERROR_MASK, ST_QUEUE_OVERFLOW, ST_ROUND_OVERFLOW
from tests.support import assert_same

# sim_params.h NodeField, then the three author masks (packed_field(F_NSCALAR + 0 / 1 / 2))
FIELDS = ["STARTUP", "IGNORE", "CUR", "HQC", "HTC", "HCR", "HCC", "LVR", "LOCKED", "PMR", "PM_START", "PM_DUR", "PM_PERIOD",
          "LQA", "TRK_HCR", "TRK_TIME", "FLAGS", "NEXT_CMD", "LC_ROUND", "COMMITS", "BALLOT", "TOW", "TC_ROUND", "LAST_TIMER",
          "VMASK", "TMASK", "TCMASK"]
F = {name: i for i, name in enumerate(FIELDS)}
NSCALAR = 24
FILL = 0xDEADBEEF

# The layout the comment above Core::packed_field documents: (word, shift, mask).
DOCUMENTED = {
    "STARTUP": (0, 0, 0xFFFFFFFF), "IGNORE": (1, 0, 0xFFFFFFFF), "PM_START": (2, 0, 0xFFFFFFFF), "PM_DUR": (3, 0, 0xFFFFFFFF),
    "PM_PERIOD": (4, 0, 0xFFFFFFFF), "LQA": (5, 0, 0xFFFFFFFF), "TRK_TIME": (6, 0, 0xFFFFFFFF), "LAST_TIMER": (7, 0, 0xFFFFFFFF),
    "BALLOT": (8, 0, 0xFFFFFFFF), "TOW": (9, 0, 0xFFFFFFFF),
    "CUR": (10, 0, 0xFF), "HQC": (10, 8, 0xFF), "HTC": (10, 16, 0xFF), "HCR": (10, 24, 0xFF),
    "HCC": (11, 0, 0xFF), "LVR": (11, 8, 0xFF), "LOCKED": (11, 16, 0xFF), "PMR": (11, 24, 0xFF),
    "TRK_HCR": (12, 0, 0xFF), "LC_ROUND": (12, 8, 0xFF), "TC_ROUND": (12, 16, 0xFF), "COMMITS": (12, 24, 0xFF),
    "FLAGS": (13, 0, 0xFF0F), "TCMASK": (13, 4, 0xF), "VMASK": (13, 16, 0xF), "TMASK": (13, 20, 0xF), "NEXT_CMD": (13, 24, 0xFF),
}
# sim_params.h FL_*: what F_FLAGS holds in a single-epoch run (proposed, election, has-TC, the active leader in bits 8-15)
FL_SINGLE_EPOCH = 0x1 | (3 << 1) | (1 << 3) | (0xFF << 8)

# The largest value each field takes (sim_core.cuh, the bounds under the layout comment): times and vote weights are full
# words; a round id is < 128 and PMR / LVR (an active round, HQC or HTC + 1) are <= 128; a node commits each round and
# proposes in each round at most once, so COMMITS and NEXT_CMD are <= 128; author masks have four bits.
ROUND_FIELDS = ("CUR", "HQC", "HTC", "HCR", "HCC", "LOCKED", "TRK_HCR", "LC_ROUND", "TC_ROUND")
BOUND = {name: 0xFFFFFFFF for name in FIELDS}
BOUND.update({name: 128 for name in ROUND_FIELDS + ("PMR", "LVR", "COMMITS", "NEXT_CMD")})
BOUND.update({"VMASK": 0xF, "TMASK": 0xF, "TCMASK": 0xF, "FLAGS": FL_SINGLE_EPOCH})
HCBR_BOUND = 0xFF  # an hcbr entry is <= HQC < 128; the byte holds 255


def test_field_table_is_the_documented_layout(hostcore):
    info = hostcore.packed_fields()
    assert info["nscalar"] == NSCALAR and len(info["fields"]) == len(FIELDS)
    assert (info["scalar_words"], info["timeout_hcbr"], info["tc_hcbr"], info["packed_words"]) == (14, 14, 15, 16)
    for name, f in F.items():
        assert info["fields"][f] == DOCUMENTED[name], name
    # every field inside words 0-13 and inside 32 bits, no two fields sharing a bit
    used = [0] * info["scalar_words"]
    for name, (word, shift, mask) in zip(FIELDS, info["fields"]):
        assert 0 <= word < info["scalar_words"], name
        assert mask and (mask << shift) < 1 << 32, name
        assert used[word] & (mask << shift) == 0, name
        used[word] |= mask << shift
        # wide enough for the documented bound: every value 0..bound survives the mask (F_FLAGS: every bit it uses)
        assert BOUND[name] & mask == BOUND[name], name
        assert name == "FLAGS" or (mask + 1) & mask == 0, name
    # the compact words sit in front of the generic node block's bitsets; a slot's four words inside the generic slot
    assert info["packed_words"] <= info["n_hasblk"] and info["tc_hcbr"] < info["packed_words"]
    assert info["pay_words"] >= 4 and info["payload_cap"] == 32 and info["round_cap"] == 128


def encode(vals):
    """The 16 compact words of a node holding vals (35 values: scalars, masks, timeout hcbr[4], TC hcbr[4]), by the
    documented layout."""
    w = [0] * 16
    for name, f in F.items():
        word, shift, mask = DOCUMENTED[name]
        w[word] |= (int(vals[f]) & mask) << shift
    w[14] = sum(int(vals[27 + a]) << (8 * a) for a in range(4))
    w[15] = sum(int(vals[31 + a]) << (8 * a) for a in range(4))
    return np.array(w, np.uint32)


def roundtrip(hostcore, info, vals, node, lane, rng):
    tile = rng.integers(0, 1 << 32, info["total_words"] * 32, dtype=np.uint64).astype(np.uint32)
    before = tile.copy()
    by_load, by_ld, t_hcbr, tc_hcbr = hostcore.packed_roundtrip(vals, tile, node, lane)
    v = np.asarray(vals, np.uint32)
    np.testing.assert_array_equal(by_load, v[:27], err_msg="load_node")
    np.testing.assert_array_equal(by_ld, v[:27], err_msg="node_ld")
    np.testing.assert_array_equal(t_hcbr, v[27:31], err_msg="timeout hcbr (put_timeout_hcbr / hcbr_of)")
    np.testing.assert_array_equal(tc_hcbr, v[31:35], err_msg="TC hcbr (copy_timeout_hcbr_to_tc / hcbr_of)")
    nb = info["node_base"] + node * info["node_words"]
    grid, grid0 = tile.reshape(-1, 32), before.reshape(-1, 32)
    np.testing.assert_array_equal(grid[nb:nb + 16, lane], encode(vals), err_msg="compact words")
    grid[nb:nb + 16, lane] = grid0[nb:nb + 16, lane]
    changed = np.argwhere(grid != grid0)
    assert len(changed) == 0, "words outside the node's compact words changed: (word, lane) %s" % changed[:8].tolist()


def test_roundtrip_of_each_field_at_its_bound(hostcore):
    info = hostcore.packed_fields()
    rng = np.random.default_rng(1)
    top = np.array([BOUND[n] for n in FIELDS] + [HCBR_BOUND] * 8, np.uint64)
    for k in range(35):
        one = np.zeros(35, np.uint64)
        one[k] = top[k]
        roundtrip(hostcore, info, one, 2, 7, rng)           # this one at its maximum, the others zero
        rest = top.copy()
        rest[k] = 0
        roundtrip(hostcore, info, rest, 1, 30, rng)         # and the reverse
    roundtrip(hostcore, info, top, 3, 31, rng)
    roundtrip(hostcore, info, np.zeros(35, np.uint64), 0, 1, rng)


def test_roundtrip_of_random_values(hostcore):
    info = hostcore.packed_fields()
    rng = np.random.default_rng(2)
    top = np.array([BOUND[n] for n in FIELDS] + [HCBR_BOUND] * 8, np.uint64)
    for _ in range(200):
        vals = rng.integers(0, top + 1, dtype=np.uint64)
        vals[F["FLAGS"]] &= FL_SINGLE_EPOCH
        roundtrip(hostcore, info, vals, int(rng.integers(4)), int(rng.integers(1, 32)), rng)


# ---- whole runs: N = 4 on the FX_DEFAULT4 layout, 256 seeds each ----
RC = {"round_cap": 128}
CONFIGS = {
    # max round 115-120, commits up to ~107, every instance completes
    "horizon_3000": (3000, RC),
    # every instance needs round 128: ST_ROUND_OVERFLOW throughout
    "round_overflow_4000": (4000, RC),
    # the exact boundary: some instances peak at round 127 and complete, the others need 128 and overflow
    "weighted_boundary": (3000, dict(RC, voting_rights=[1, 2, 5, 1])),
    # short delays: COMMITS and NEXT_CMD near the top of their byte
    "fast_delays": (1500, dict(RC, delay_mean=5.0, delay_variance=1.0)),
    # the commit tracker's query-all path
    "commit_tracker": (3000, dict(RC, target_commit_interval=300, delta=400)),
    # pacemaker settings that make timeouts and timeout certificates common (default capacities)
    "delta_10": (1000, {"delta": 10}),
    "delta_8_lambda_0.9": (1000, {"delta": 8, "lambda_": 0.9}),
    "slow_delays": (1000, {"delay_mean": 20.0, "delay_variance": 10.0}),
    # a queue of 64 entries is too short for this pacemaker: ST_QUEUE_OVERFLOW throughout
    "queue_overflow": (1000, {"delta": 5, "gamma": 1.5, "lambda_": 0.25, "queue_cap": 64}),
}
SEEDS = np.arange(1, 257, dtype=np.uint64)
_RUNS = {}


def runs(oracle, hostcore, name, seeds=SEEDS):
    """(oracle, compact-encoding run, generic run) of a configuration, computed once per session."""
    key = (name, int(seeds[0]), len(seeds))
    if key not in _RUNS:
        max_clock, kw = CONFIGS[name]
        assert hostcore.fixed_shape(4, max_clock, **kw) == 1, "%s no longer selects FX_DEFAULT4" % name
        _RUNS[key] = (oracle.run(seeds, 4, max_clock, **kw), hostcore.final_state(seeds, 4, max_clock, **kw),
                      hostcore.final_state(seeds, 4, max_clock, generic=True, **kw))
    return _RUNS[key]


def check_packed_against_generic(hostcore, p, g, count):
    info = hostcore.packed_fields()
    # the outputs, every instance, errors included
    np.testing.assert_array_equal(p.commit_counts, g.commit_counts)
    np.testing.assert_array_equal(p.last_states, g.last_states)
    np.testing.assert_array_equal(p.lc_round, g.lc_round)
    np.testing.assert_array_equal(p.counters, g.counters)
    np.testing.assert_array_equal(p.status, g.status)
    # every node's final state, field by field
    for f, name in enumerate(FIELDS + ["T_HCBR%d" % a for a in range(4)] + ["TC_HCBR%d" % a for a in range(4)]):
        np.testing.assert_array_equal(p.decoded[:, :, f], g.decoded[:, :, f], err_msg=name)
    # the per-round bitsets of every node, the chain table, the created / QC-made bitsets
    for n in range(4):
        nb = info["node_base"] + n * info["node_words"]
        bits = slice(nb + info["n_hasblk"], nb + info["node_words"])
        np.testing.assert_array_equal(p.raw[:, bits], g.raw[:, bits], err_msg="bitsets of node %d" % n)
        # the words of the generic node block the compact one does not use: never written
        unused = p.raw[:, nb + info["packed_words"]:nb + info["n_hasblk"]]
        assert (unused == FILL).all(), "node %d: unused node words written" % n
    chain = slice(info["chain_base"], info["chain_base"] + 2 * info["round_cap"])
    np.testing.assert_array_equal(p.raw[:, chain], g.raw[:, chain], err_msg="chain table")
    sets = slice(info["created_base"], info["created_base"] + 2 * info["rset_words"])
    np.testing.assert_array_equal(p.raw[:, sets], g.raw[:, sets], err_msg="created / QC-made bitsets")
    # a slot is four words: the rest of each generic slot is never written
    pool = p.raw[:, info["pay_base"]:info["pay_base"] + info["payload_cap"] * info["pay_words"]]
    assert (pool[:, 4 * info["payload_cap"]:] == FILL).all(), "slot words past the compact pitch written"
    # the lanes of the last tile that hold no instance: nothing at all
    for r in (p, g):
        assert (r.raw_tiles[-1, :, count % 32 or 32:] == FILL).all(), "words of an empty lane written"


def subset(r, idx):
    return SimpleNamespace(commit_counts=r.commit_counts[idx], last_states=r.last_states[idx], counters=r.counters[idx])


def check_against_oracle(o, p, max_round_limit=True):
    """The instances without an error bit equal the oracle's; returns which ones those are."""
    ok = (p.status & ST_ERROR_MASK) == 0
    assert_same(subset(o, ok), subset(p, ok), "instances without an error bit")
    assert ((p.status[ok] & ~np.uint32(64)) == 1).all()
    if max_round_limit:
        # Round ids end at 127: an instance overflows exactly when the reference's pacemaker reaches round 128, or when a
        # node certifies round 127 (a QC, HQC = 127, or a TC, HTC = 127) and its record store would move to round 128 —
        # which the reference may do in the last event before the horizon, with its active round still 127.
        overflow = (p.status & ST_ROUND_OVERFLOW) != 0
        cert_127 = ((p.decoded[:, :, F["HQC"]] == 127) | (p.decoded[:, :, F["HTC"]] == 127)).any(axis=1)
        np.testing.assert_array_equal(overflow, (o.counters[:, 6] >= 128) | cert_127)
    return ok


@pytest.mark.parametrize("name", list(CONFIGS))
def test_packed_run_matches_generic_and_oracle(oracle, hostcore, name):
    o, p, g = runs(oracle, hostcore, name)
    check_packed_against_generic(hostcore, p, g, len(SEEDS))
    ok = check_against_oracle(o, p, max_round_limit=name != "queue_overflow")
    if name == "round_overflow_4000":
        assert not ok.any() and (p.status & ST_ROUND_OVERFLOW).all()
    elif name == "queue_overflow":
        assert (p.status & ST_QUEUE_OVERFLOW).all()
    elif name == "weighted_boundary":
        # both sides of the boundary occur, and the completed side reaches round 127
        assert 0 < ok.sum() < len(ok) and o.counters[ok, 6].max() == 127
    else:
        assert ok.all()


def test_boundary_split_over_more_seeds(oracle, hostcore):
    # seeds 7279 and 7603 overflow with the reference's active round still 127: a QC for round 127 in the last event
    seeds = np.arange(7001, 8025, dtype=np.uint64)
    o, p, g = runs(oracle, hostcore, "weighted_boundary", seeds)
    check_packed_against_generic(hostcore, p, g, len(seeds))
    ok = check_against_oracle(o, p)
    overflow = (p.status & ST_ROUND_OVERFLOW) != 0
    assert ok.any() and (overflow & (o.counters[:, 6] >= 128)).any() and (overflow & (o.counters[:, 6] == 127)).any()


@pytest.mark.parametrize("count", [1, 31, 33])
def test_ragged_batches(oracle, hostcore, count):
    seeds = np.arange(101, 101 + count, dtype=np.uint64)
    for name in ("weighted_boundary", "queue_overflow"):
        o, p, g = runs(oracle, hostcore, name, seeds)
        check_packed_against_generic(hostcore, p, g, count)
        check_against_oracle(o, p, max_round_limit=name != "queue_overflow")


def test_runs_reach_the_edges_of_the_encoding(oracle, hostcore):
    """The configurations above drive the compact fields to their limits: without this, the comparisons would pass just
    as well on runs that never leave the low half of each byte."""
    d = np.concatenate([runs(oracle, hostcore, name)[1].decoded.reshape(-1, 35) for name in CONFIGS])
    assert (d[:, F["CUR"]] == 127).any()
    assert d[:, F["CUR"]].max() <= 127 and d[:, [F[n] for n in ROUND_FIELDS]].max() <= 127   # round ids stay below rspan
    assert (d[:, F["COMMITS"]] >= 120).any()
    assert ((d[:, F["HTC"]] > 0) & (d[:, F["TCMASK"]] != 0)).any()
    # A complete timeout set: four authors hold every voting right, so the insert that completes the set also forms the TC,
    # and update_current_round clears tmask in the same step — the set is stored as the TC's authors (the weighted
    # configuration: authors 0, 1, 3 carry 4 of the 7 a quorum needs).  The current set keeps up to three, author 3 included.
    assert (d[:, F["TCMASK"]] == 0xF).any()
    tmask = d[:, F["TMASK"]]
    assert ((np.bitwise_count(tmask) == 3) & (tmask & 8 != 0)).any()
    for name in ("PMR", "LVR", "COMMITS", "NEXT_CMD"):
        assert d[:, F[name]].max() <= 128, name
