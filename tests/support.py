"""Test support: ctypes wrappers of the ORACLE (oracle/liblbft_oracle.so) and of the host-compiled
device core (tests/hostcore/libhostcore.so).  Both are test infrastructure; nothing here is imported
by the product package."""
import ctypes
import os

import numpy as np

from librabft_simulator_b200 import _build
from librabft_simulator_b200._lib import LbftCommit, LbftConfig

P = ctypes.c_void_p

# Reference defaults: librabft-v2/tests/simulated_run.rs:29-42 == main.rs:72-172
REF = dict(delay_mean=10.0, delay_variance=4.0, target_commit_interval=100000, delta=20, gamma=2.0,
           lambda_=0.5, commands_per_epoch=30000)


def make_config(seeds, num_nodes, max_clock=1000, **kw):
    """Build an lbft_config; returns (config, keepalive) — keepalive owns the arrays it points to."""
    seeds = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).reshape(-1))
    c = LbftConfig()
    c.struct_size = ctypes.sizeof(LbftConfig)
    c.num_instances, c.num_nodes, c.delay_kind = len(seeds), num_nodes, 0
    c.seeds = seeds.ctypes.data
    c.max_clock = max_clock
    keep = [seeds]
    vals = dict(REF)
    vals.update(kw)
    for k, v in vals.items():
        if k in ("voting_rights", "silent"):
            if v is None:
                continue
            arr = np.ascontiguousarray(v, dtype=np.uint64 if k == "voting_rights" else np.uint8)
            keep.append(arr)
            setattr(c, k, arr.ctypes.data)
        else:
            setattr(c, k, v)
    return c, keep


class Result:
    def __init__(self, I, N):
        self.commit_counts = np.zeros((I, N), np.uint32)
        self.last_states = np.zeros((I, N), np.uint64)
        self.counters = np.zeros((I, 12), np.uint32)
        self.status = np.zeros(I, np.uint32)
        self.seconds = 0.0


class LbftRoundSwitch(ctypes.Structure):
    """include/lbft.h lbft_round_switch"""
    _fields_ = [("node", ctypes.c_uint32), ("round", ctypes.c_uint32), ("time", ctypes.c_int64)]


FLAG_ROUND_SWITCHES = 1
FLAG_RESUMABLE = 2
FLAG_TRUE_DATA_SYNC = 4


def _round_switches(fn, err, seeds, num_nodes, instance, max_clock, **kw):
    """Calls an (cfg, instance, out, cap, n) entry point twice (size, then data); returns [(node, round, time)]."""
    kw.setdefault("flags", FLAG_ROUND_SWITCHES)
    cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
    n = ctypes.c_size_t()
    if fn(ctypes.byref(cfg), instance, None, 0, ctypes.byref(n)) != 0:
        raise RuntimeError(err().decode())
    buf = (LbftRoundSwitch * max(n.value, 1))()
    if fn(ctypes.byref(cfg), instance, buf, n.value, ctypes.byref(n)) != 0:
        raise RuntimeError(err().decode())
    return [(buf[i].node, buf[i].round, buf[i].time) for i in range(n.value)]


class Oracle:
    def __init__(self, native=False):
        """native=True: the -O3 -march=native build made on this machine (the CPU-baseline leg of bench.py)."""
        if native:
            path, self.build_flags = _build.build_oracle_native()
        else:
            path, self.build_flags = _build.build_oracle(), "-O2"
        self.lib = ctypes.CDLL(path)
        L = self.lib
        L.lbfo_last_error.restype = ctypes.c_char_p
        L.lbfo_siphash13.restype = ctypes.c_uint64
        L.lbfo_siphash13.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
        L.lbfo_state_key.restype = ctypes.c_uint64
        L.lbfo_state_key.argtypes = [ctypes.POINTER(LbftCommit), ctypes.c_size_t]
        L.lbfo_run_batch.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, P, P, P, P,
                                     ctypes.POINTER(ctypes.c_double)]
        L.lbfo_commit_log.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(LbftCommit),
                                      ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.lbfo_xoshiro_seq.argtypes = [ctypes.c_uint64, P, ctypes.c_size_t]
        L.lbfo_pick_author.argtypes = [P, ctypes.c_uint32, ctypes.c_uint64]
        L.lbfo_pick_author.restype = ctypes.c_uint32
        L.lbfo_leader.argtypes = [P, ctypes.c_uint32, ctypes.c_uint64]
        L.lbfo_leader.restype = ctypes.c_uint32
        L.lbfo_quorum_threshold.argtypes = [P, ctypes.c_uint32]
        L.lbfo_quorum_threshold.restype = ctypes.c_uint64
        L.lbfo_ziggurat_tables.argtypes = [P, P]
        L.lbfo_delay_samples.argtypes = [ctypes.c_uint64, ctypes.c_double, ctypes.c_double, P, ctypes.c_size_t]
        L.lbfo_normal_samples.argtypes = [ctypes.c_uint64, P, ctypes.c_size_t]
        L.lbfo_shuffle.argtypes = [ctypes.c_uint64, P, ctypes.c_size_t]
        L.lbfo_round_durations.argtypes = [ctypes.c_int64, ctypes.c_double, ctypes.c_double, P, P, ctypes.c_size_t]
        L.lbfo_selftest.argtypes = [ctypes.c_char_p, ctypes.c_size_t]

    def run(self, seeds, num_nodes, max_clock=1000, threads=0, first=0, count=None, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        I = cfg.num_instances
        count = I - first if count is None else count
        res = Result(I, num_nodes)
        sec = ctypes.c_double()
        threads = threads or (os.cpu_count() or 1)
        rc = self.lib.lbfo_run_batch(ctypes.byref(cfg), first, count, threads, P(res.commit_counts.ctypes.data),
                                     P(res.last_states.ctypes.data), P(res.counters.ctypes.data),
                                     P(res.status.ctypes.data), ctypes.byref(sec))
        if rc != 0:
            raise RuntimeError(self.lib.lbfo_last_error().decode())
        res.seconds = sec.value
        return res

    def round_switches(self, seeds, num_nodes, instance, max_clock=1000, **kw):
        """DataWriter::nodes_round_switch of one instance (data_writer.rs:34-50), node-major."""
        fn = self.lib.lbfo_round_switches
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.POINTER(LbftRoundSwitch), ctypes.c_size_t,
                       ctypes.POINTER(ctypes.c_size_t)]
        return _round_switches(fn, self.lib.lbfo_last_error, seeds, num_nodes, instance, max_clock, **kw)

    def run_staged(self, seeds, num_nodes, stops, max_clock=1000, threads=0, **kw):
        """loop_until called once per stop on the same simulators (simulator.rs:380); max_clock is only the horizon
        the device side is configured with (the oracle itself needs none)."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        res = Result(cfg.num_instances, num_nodes)
        st = np.asarray(stops, dtype=np.int64)
        fn = self.lib.lbfo_run_batch_staged
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, P, ctypes.c_size_t, P, P, P, P]
        rc = fn(ctypes.byref(cfg), 0, cfg.num_instances, threads or (os.cpu_count() or 1), P(st.ctypes.data), len(st),
                P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data))
        if rc != 0:
            raise RuntimeError(self.lib.lbfo_last_error().decode())
        return res

    def round_switches_staged(self, seeds, num_nodes, instance, stops, max_clock=1000, **kw):
        st = np.asarray(stops, dtype=np.int64)
        fn = self.lib.lbfo_round_switches_staged
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, P, ctypes.c_size_t, ctypes.POINTER(LbftRoundSwitch), ctypes.c_size_t,
                       ctypes.POINTER(ctypes.c_size_t)]
        return _round_switches(lambda c, i, out, cap, n: fn(c, i, P(st.ctypes.data), len(st), out, cap, n), self.lib.lbfo_last_error,
                               seeds, num_nodes, instance, max_clock, **kw)

    def commit_log(self, seeds, num_nodes, instance, node, max_clock=1000, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        n = ctypes.c_size_t()
        buf = (LbftCommit * 65536)()
        rc = self.lib.lbfo_commit_log(ctypes.byref(cfg), instance, node, buf, 65536, ctypes.byref(n))
        if rc != 0:
            raise RuntimeError(self.lib.lbfo_last_error().decode())
        return [(int(buf[i].proposer), int(buf[i].index), int(buf[i].time)) for i in range(n.value)]

    def commit_log_staged(self, seeds, num_nodes, instance, node, stops, max_clock=1000, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        st = np.asarray(stops, dtype=np.int64)
        n = ctypes.c_size_t()
        buf = (LbftCommit * 65536)()
        fn = self.lib.lbfo_commit_log_staged
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.c_uint32, P, ctypes.c_size_t, ctypes.POINTER(LbftCommit),
                       ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        if fn(ctypes.byref(cfg), instance, node, P(st.ctypes.data), len(st), buf, 65536, ctypes.byref(n)) != 0:
            raise RuntimeError(self.lib.lbfo_last_error().decode())
        return [(int(buf[i].proposer), int(buf[i].index), int(buf[i].time)) for i in range(n.value)]

    def state_key(self, log):
        buf = (LbftCommit * max(1, len(log)))()
        for i, (p, idx, t) in enumerate(log):
            buf[i].proposer, buf[i].index, buf[i].time = p, idx, t
        return int(self.lib.lbfo_state_key(buf, len(log)))

    def selftest(self):
        buf = ctypes.create_string_buffer(8192)
        return self.lib.lbfo_selftest(buf, 8192), buf.value.decode()


class HostCore:
    """The device state machine compiled for the host (CPU-side check of the kernel's logic)."""

    def __init__(self):
        path = _build.build_hostcore()
        self.lib = ctypes.CDLL(path)
        self.lib.hostcore_last_error.restype = ctypes.c_char_p
        self.lib.hostcore_run.argtypes = [ctypes.POINTER(LbftConfig), P, P, P, P, P, ctypes.POINTER(ctypes.c_uint32)]

    def setup_info(self, num_nodes, max_clock=1000, **kw):
        cfg, keep = make_config([1], num_nodes, max_clock, **kw)
        out = np.zeros(6, np.uint32)
        rc = self.lib.hostcore_setup_info(ctypes.byref(cfg), P(out.ctypes.data))
        if rc != 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        return dict(zip(("delay_kmax", "queue_scan", "round_cap", "queue_cap", "payload_cap", "words"), out.tolist()))

    def fixed_shape(self, num_nodes, max_clock=1000, **kw):
        """sim_params.h FX_* of the instantiation `run` takes for this configuration (0: the generic one)."""
        cfg, keep = make_config([1], num_nodes, max_clock, **kw)
        return self.lib.hostcore_fixed_shape(ctypes.byref(cfg))

    def kernel_info(self, seeds, num_nodes, max_clock=1000, **kw):
        """The product's lbft_kernel_info for this configuration (the kernel the host selects; honours LBFT_FORCE_KERNEL)."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        buf = ctypes.create_string_buffer(128)
        if self.lib.hostcore_kernel_info(ctypes.byref(cfg), buf, ctypes.sizeof(buf)) != 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        return buf.value.decode()

    def run(self, seeds, num_nodes, max_clock=1000, **kw):
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        I = cfg.num_instances
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        w = ctypes.c_uint32()
        rc = self.lib.hostcore_run(ctypes.byref(cfg), P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data),
                                   P(res.lc_round.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data),
                                   ctypes.byref(w))
        if rc != 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        res.words_per_instance = w.value
        return res

    def round_switches(self, seeds, num_nodes, instance, max_clock=1000, **kw):
        fn = self.lib.hostcore_round_switches
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, ctypes.POINTER(LbftRoundSwitch), ctypes.c_size_t,
                       ctypes.POINTER(ctypes.c_size_t)]
        return _round_switches(fn, self.lib.hostcore_last_error, seeds, num_nodes, instance, max_clock, **kw)

    def run_staged(self, seeds, num_nodes, stops, max_clock=1000, **kw):
        """One launch per stop over the same state (what lbft_run_until does); needs flags with FLAG_RESUMABLE."""
        kw.setdefault("flags", FLAG_RESUMABLE)
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        res = Result(cfg.num_instances, num_nodes)
        res.lc_round = np.zeros((cfg.num_instances, num_nodes), np.uint32)
        st = np.asarray(stops, dtype=np.int64)
        fn = self.lib.hostcore_run_staged
        fn.argtypes = [ctypes.POINTER(LbftConfig), P, ctypes.c_size_t, P, P, P, P, P]
        rc = fn(ctypes.byref(cfg), P(st.ctypes.data), len(st), P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data),
                P(res.lc_round.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data))
        if rc != 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        return res

    def round_switches_staged(self, seeds, num_nodes, instance, stops, max_clock=1000, **kw):
        kw.setdefault("flags", FLAG_RESUMABLE | FLAG_ROUND_SWITCHES)
        st = np.asarray(stops, dtype=np.int64)
        fn = self.lib.hostcore_round_switches_staged
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_uint32, P, ctypes.c_size_t, ctypes.POINTER(LbftRoundSwitch), ctypes.c_size_t,
                       ctypes.POINTER(ctypes.c_size_t)]
        return _round_switches(lambda c, i, out, cap, n: fn(c, i, P(st.ctypes.data), len(st), out, cap, n), self.lib.hostcore_last_error,
                               seeds, num_nodes, instance, max_clock, **kw)

    # ---- the compact encoding of the four-author compile-time layout (sim_core.cuh Core::PACK, FX_DEFAULT4) ----
    LAYOUT_KEYS = ("node_base", "node_words", "n_hasblk", "rset_words", "created_base", "qcmade_base", "chain_base", "round_cap",
                   "pay_base", "pay_words", "payload_cap", "total_words")
    DECODED_WORDS = 24 + 3 + 4 + 4  # per node: F_* scalars, vmask / tmask / tcmask, timeout hcbr[4], TC hcbr[4]

    def packed_fields(self):
        """The core's packed_field() table and constants, and the offsets of fixed_layout(FX_DEFAULT4): a dict with
        'nscalar', 'scalar_words', 'packed_words', 'timeout_hcbr', 'tc_hcbr', 'fields' ([(word, shift, mask)] for F_* 0 ..
        F_NSCALAR + 2, the last three the vote / timeout / TC author masks) and the layout keys of LAYOUT_KEYS."""
        out = np.zeros(256, np.uint32)
        fn = self.lib.hostcore_packed_fields
        fn.argtypes = [P, ctypes.c_size_t]
        k = fn(P(out.ctypes.data), len(out))
        if k < 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        v = [int(x) for x in out[:k]]
        info = dict(zip(("nscalar", "scalar_words", "packed_words", "timeout_hcbr", "tc_hcbr"), v[:5]))
        nf = info["nscalar"] + 3
        info["fields"] = [tuple(v[5 + 3 * f: 8 + 3 * f]) for f in range(nf)]
        info.update(zip(self.LAYOUT_KEYS, v[5 + 3 * nf:]))
        return info

    def packed_roundtrip(self, vals, tile, node, lane):
        """vals (24 scalars, 3 masks, 4 timeout hcbr, 4 TC hcbr) through store_node / put_timeout_hcbr /
        copy_timeout_hcbr_to_tc into node `node` of lane `lane` of `tile` (uint32 [total_words * 32], updated in place), and
        back: returns (load_node's 27 values, node_ld's 27 values, hcbr_of of the timeout vector, hcbr_of of the TC vector)."""
        v = np.ascontiguousarray(vals, dtype=np.uint32)
        assert v.shape == (35,) and tile.dtype == np.uint32 and tile.flags["C_CONTIGUOUS"]
        out = np.zeros(62, np.uint32)
        fn = self.lib.hostcore_packed_roundtrip
        fn.argtypes = [P, ctypes.c_uint32, ctypes.c_uint32, P, P]
        if fn(P(v.ctypes.data), node, lane, P(tile.ctypes.data), P(out.ctypes.data)) != 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        return out[:27], out[27:54], out[54:58], out[58:62]

    def final_state(self, seeds, num_nodes, max_clock=1000, generic=False, **kw):
        """One FX_DEFAULT4 configuration through the compact-encoding instantiation (or, generic=True, the generic one on
        the same layout) in a state buffer filled with 0xdeadbeef.  Returns a Result with lc_round, plus `decoded`
        [instance, node, DECODED_WORDS] (hcbr entries of authors outside tmask / tcmask read 0) and `raw` [instance,
        total_words], the instance's words out of its warp tile; `raw_tiles` is the whole buffer [tile, word, lane]."""
        cfg, keep = make_config(seeds, num_nodes, max_clock, **kw)
        I = cfg.num_instances
        words = self.setup_info(num_nodes, max_clock, **kw)["words"]
        tiles = (I + 31) // 32
        res = Result(I, num_nodes)
        res.lc_round = np.zeros((I, num_nodes), np.uint32)
        res.decoded = np.zeros((I, num_nodes, self.DECODED_WORDS), np.uint32)
        res.raw_tiles = np.zeros((tiles, words, 32), np.uint32)
        fn = self.lib.hostcore_final_state
        fn.argtypes = [ctypes.POINTER(LbftConfig), ctypes.c_int, P, P, P, P, P, P, P]
        rc = fn(ctypes.byref(cfg), 1 if generic else 0, P(res.commit_counts.ctypes.data), P(res.last_states.ctypes.data),
                P(res.lc_round.ctypes.data), P(res.counters.ctypes.data), P(res.status.ctypes.data), P(res.decoded.ctypes.data),
                P(res.raw_tiles.ctypes.data))
        if rc != 0:
            raise RuntimeError(self.lib.hostcore_last_error().decode())
        res.raw = res.raw_tiles.transpose(0, 2, 1).reshape(tiles * 32, words)[:I]
        return res


def assert_same(a, b, what=""):
    """Bit-exact comparison of two Result objects on everything the reference exposes."""
    np.testing.assert_array_equal(a.commit_counts, b.commit_counts, err_msg="commit counts differ " + what)
    np.testing.assert_array_equal(a.last_states, b.last_states, err_msg="last committed states differ " + what)
    # processed-by-kind, cancelled timers, creation stamps, max active round, RNG draws
    np.testing.assert_array_equal(a.counters[:, :8], b.counters[:, :8], err_msg="event counters differ " + what)
    np.testing.assert_array_equal(a.counters[:, 9], b.counters[:, 9], err_msg="scheduled notifications differ " + what)
