"""The lane-block form of the compact encoding (sim_core.cuh TileMem LB), which the bench kernel and its commit-times twin run:
inside the rows a warp tile already gives a node's 16 compact words and a notification slot's 4 words, each lane's words are
contiguous, so that a thread moves them with 128-bit accesses.  The lane-interleaved form that tests/test_packed_encoding.py
pins stays the definition; this file shows that the lane-block form is an exact permutation of it.

* TileMem::block_word, the one definition of the mapping, permutes the words of each node's compact rows and of each slot's
  rows among themselves, with every lane's block contiguous and 16-byte aligned.
* Round trips of extreme and random values through the lane-block core's writers and readers, with every other word of the
  tile left alone.
* Whole runs of test_packed_encoding's configurations (round and queue overflow included): the same outputs, counters,
  status and decoded node fields as the lane-interleaved core, and the same final state word for word once mapped back
  through block_word; the words neither form uses, and every word of an empty lane, keep their fill value."""
import ctypes

import numpy as np
import pytest

from librabft_simulator_b200 import _build
from tests import test_packed_encoding as pe
from tests.support import P, Result, make_config

FILL = pe.FILL
WORDS = 35  # roundtrip values: 24 scalars, 3 masks, 4 timeout hcbr, 4 TC hcbr


class LaneBlockCore:
    """ctypes wrapper of tests/hostcore/lane_block_hostcore.cpp."""

    def __init__(self):
        self.lib = ctypes.CDLL(_build.build_lane_block_hostcore())
        self.lib.lane_block_last_error.restype = ctypes.c_char_p
        self.lib.lane_block_word.restype = ctypes.c_uint64
        self.lib.lane_block_word.argtypes = [ctypes.c_uint32] * 4
        self.lib.lane_block_roundtrip.argtypes = [P, ctypes.c_uint32, ctypes.c_uint32, P, P]
        self.lib.lane_block_final_state.argtypes = [ctypes.c_void_p, P, P, P, P, P, P, P]

    def error(self):
        return RuntimeError(self.lib.lane_block_last_error().decode())

    def block_word(self, base, K, k, lane):
        return int(self.lib.lane_block_word(base, K, k, lane))

    def roundtrip(self, vals, tile, node, lane):
        v = np.ascontiguousarray(vals, dtype=np.uint32)
        out = np.zeros(62, np.uint32)
        if self.lib.lane_block_roundtrip(P(v.ctypes.data), node, lane, P(tile.ctypes.data), P(out.ctypes.data)) != 0:
            raise self.error()
        return out[:27], out[27:54], out[54:58], out[58:62]

    def final_state(self, seeds, num_nodes, max_clock, words, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        res.decoded = np.zeros((I, num_nodes, 35), np.uint32)
        res.raw_tiles = np.zeros(((I + 31) // 32, words, 32), np.uint32)
        rc = self.lib.lane_block_final_state(ctypes.addressof(cfg), P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data),
                                             P(res.lc_round.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data),
                                             P(res.decoded.ctypes.data), P(res.raw_tiles.ctypes.data))
        if rc != 0:
            raise self.error()
        return res


@pytest.fixture(scope="module")
def lane():
    return LaneBlockCore()


def regions(info):
    """(base word, K) of every region of compact blocks: the 16 compact rows of each node, the 4 rows of each slot."""
    nodes = [(info["node_base"] + n * info["node_words"], info["packed_words"]) for n in range(4)]
    return nodes + [(info["pay_base"] + 4 * s, 4) for s in range(info["payload_cap"])]


_PERM = {}


def permutation(lane, info):
    """lb[i] for every tile offset i of the lane-interleaved form: where block_word puts that word (identity outside the
    regions of compact blocks); and `owner`, the lane each lane-block offset belongs to."""
    if "perm" not in _PERM:
        n = info["total_words"] * 32
        perm, owner = np.arange(n), np.arange(n) % 32
        for base, K in regions(info):
            for k in range(K):
                for ln in range(32):
                    off = lane.block_word(base, K, k, ln)
                    perm[(base + k) * 32 + ln] = off
                    owner[off] = ln
        _PERM["perm"], _PERM["owner"] = perm, owner
    return _PERM["perm"], _PERM["owner"]


def test_block_word_permutes_each_region(hostcore, lane):
    info = hostcore.packed_fields()
    for base, K in regions(info):
        offs = np.array([[lane.block_word(base, K, k, ln) for k in range(K)] for ln in range(32)])
        # the region's K x 32 words, each exactly once
        np.testing.assert_array_equal(np.sort(offs.ravel()), np.arange(base * 32, (base + K) * 32))
        # a lane's words contiguous, in order, starting on a 16-byte boundary (the tile starts on a 128-byte one)
        np.testing.assert_array_equal(offs - offs[:, :1], np.broadcast_to(np.arange(K), offs.shape))
        assert (offs[:, 0] % 4 == 0).all()


def lane_roundtrip(hostcore, lane, info, vals, node, lane_id, rng):
    tile = rng.integers(0, 1 << 32, info["total_words"] * 32, dtype=np.uint64).astype(np.uint32)
    before = tile.copy()
    by_load, by_ld, t_hcbr, tc_hcbr = lane.roundtrip(vals, tile, node, lane_id)
    v = np.asarray(vals, np.uint32)
    np.testing.assert_array_equal(by_load, v[:27], err_msg="load_node")
    np.testing.assert_array_equal(by_ld, v[:27], err_msg="node_ld")
    np.testing.assert_array_equal(t_hcbr, v[27:31], err_msg="timeout hcbr")
    np.testing.assert_array_equal(tc_hcbr, v[31:35], err_msg="TC hcbr")
    nb = info["node_base"] + node * info["node_words"]
    first = lane.block_word(nb, 16, 0, lane_id)
    np.testing.assert_array_equal(tile[first:first + 16], pe.encode(vals), err_msg="compact words")
    tile[first:first + 16] = before[first:first + 16]
    changed = np.flatnonzero(tile != before)
    assert len(changed) == 0, "words outside the lane's block changed: %s" % changed[:8].tolist()


def test_roundtrip_of_each_field_at_its_bound(hostcore, lane):
    info = hostcore.packed_fields()
    rng = np.random.default_rng(11)
    top = np.array([pe.BOUND[n] for n in pe.FIELDS] + [pe.HCBR_BOUND] * 8, np.uint64)
    for k in range(WORDS):
        one = np.zeros(WORDS, np.uint64)
        one[k] = top[k]
        lane_roundtrip(hostcore, lane, info, one, 2, 7, rng)
        rest = top.copy()
        rest[k] = 0
        lane_roundtrip(hostcore, lane, info, rest, 1, 30, rng)
    lane_roundtrip(hostcore, lane, info, top, 3, 31, rng)
    lane_roundtrip(hostcore, lane, info, np.zeros(WORDS, np.uint64), 0, 0, rng)


def test_roundtrip_of_random_values(hostcore, lane):
    info = hostcore.packed_fields()
    rng = np.random.default_rng(12)
    top = np.array([pe.BOUND[n] for n in pe.FIELDS] + [pe.HCBR_BOUND] * 8, np.uint64)
    for _ in range(200):
        vals = rng.integers(0, top + 1, dtype=np.uint64)
        vals[pe.F["FLAGS"]] &= pe.FL_SINGLE_EPOCH
        lane_roundtrip(hostcore, lane, info, vals, int(rng.integers(4)), int(rng.integers(32)), rng)


def check_against_interleaved(hostcore, lane, name, seeds):
    info = hostcore.packed_fields()
    max_clock, kw = pe.CONFIGS[name]
    ref = hostcore.final_state(seeds, 4, max_clock, **kw)
    lb = lane.final_state(seeds, 4, max_clock, info["total_words"], **kw)
    for field in ("commit_counts", "last_states", "lc_round", "counters", "status", "decoded"):
        np.testing.assert_array_equal(getattr(lb, field), getattr(ref, field), err_msg=field)
    perm, owner = permutation(lane, info)
    tiles = lb.raw_tiles.reshape(len(lb.raw_tiles), -1)
    # the whole state, word for word, once every compact word is read from where block_word put it
    np.testing.assert_array_equal(tiles[:, perm], ref.raw_tiles.reshape(len(tiles), -1), err_msg="state mapped back")
    # words neither form uses: a node's generic words behind its compact ones, slot words behind the compact pitch
    rows = lb.raw_tiles
    for n in range(4):
        nb = info["node_base"] + n * info["node_words"]
        assert (rows[:, nb + info["packed_words"]:nb + info["n_hasblk"], :] == FILL).all(), "node %d: unused words written" % n
    pool = info["pay_base"] + 4 * info["payload_cap"]
    assert (rows[:, pool:info["pay_base"] + info["payload_cap"] * info["pay_words"], :] == FILL).all(), "slot words past the pitch"
    # the lanes of the last tile that hold no instance: nothing at all, wherever their blocks are
    empty = owner >= (len(seeds) % 32 or 32)
    assert (tiles[-1, empty] == FILL).all(), "words of an empty lane written"
    return ref


@pytest.mark.parametrize("name", list(pe.CONFIGS))
def test_runs_match_the_interleaved_form(hostcore, lane, name):
    ref = check_against_interleaved(hostcore, lane, name, pe.SEEDS)
    if name in ("round_overflow_4000", "queue_overflow"):  # the runs reach the overflow paths
        assert (ref.status & (pe.ST_ROUND_OVERFLOW | pe.ST_QUEUE_OVERFLOW)).all()


@pytest.mark.parametrize("count", [1, 31, 33])
def test_ragged_batches(hostcore, lane, count):
    for name in ("weighted_boundary", "queue_overflow"):
        check_against_interleaved(hostcore, lane, name, np.arange(101, 101 + count, dtype=np.uint64))
