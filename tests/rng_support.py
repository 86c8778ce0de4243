"""Test support for the sampler: plain-Python restatements of rand_xoshiro 0.6.0 (SplitMix64 seeding, Xoshiro256**), rand 0.8.3's
``sample_single_inclusive`` and rand_distr 0.4.0's ziggurat; a solver for the Xoshiro state that emits chosen outputs; ctypes
wrappers of the three sides that run sampler records (the device probe tests/gpuprobe/sampler_probe.cu, its host-compiled twin
tests/hostcore/sampler_hostcore.cpp and the oracle's lbfo_sampler); and the edge cases themselves, with the libm calls each
one makes, so that a device/glibc difference in exp or log can be told from a sampler bug.

libm values come from ``math.exp`` / ``math.log`` (the host's glibc, what the oracle and the host tables call) or from the
oracle, never from numpy's vectorised exp / log, which is a different implementation.  Exact values come from mpmath."""
import ctypes
import math
import struct

import mpmath
import numpy as np

from librabft_simulator_b200 import _build
from librabft_simulator_b200._lib import LbftConfig, LbftParamSet
from tests.support import make_config

M64 = (1 << 64) - 1
REC = np.dtype([("s", "<u8", (4,)), ("arg", "<u8"), ("result", "<u8"), ("op", "<u4"), ("set", "<u4"), ("draws", "<u4"),
                ("status", "<u4")])  # sampler_ops.cuh Rec
assert REC.itemsize == 64
OP_SEED, OP_NEXT_U64, OP_RANGE_U32, OP_RANGE_U64, OP_NORMAL, OP_DELAY_FROM_Z, OP_SAMPLE_DELAY, OP_EXP, OP_LOG = range(9)
CORE_PLAIN, CORE_FIXED, CORE_SWEEP = range(3)
ST_DELAY_NEAR_INT, ST_TIME_OVERFLOW, LANES_DISAGREE = 1 << 6, 1 << 7, 1 << 31
ZMAX = 14.0  # HostSetup::build_delay_table: the tables cover |z| <= ZMAX

# Delay models at the table's edges (lbft_config delay fields).  The kmax each must get is asserted by the CPU suite.
MODELS = {
    "baseline": dict(delay_mean=10.0, delay_variance=4.0),  # the reference's LogNormal(10, 4)
    "kmax254": dict(delay_mean=10.0, delay_variance=5.58),  # the largest table held in shared memory (kmax + 2 <= 256)
    "kmax255": dict(delay_mean=10.0, delay_variance=5.593),  # the smallest one read from global memory
    "kmax4096": dict(delay_mean=10.0, delay_variance=20.986),  # the widest table
    "kmax4097": dict(delay_mean=10.0, delay_variance=20.987),  # the first model past it: the exp() fallback
    "narrow": dict(delay_mean=100.0, delay_variance=1.0),  # thr[1..D(-ZMAX)] = -inf
    "below1": dict(delay_mean=0.5, delay_variance=0.01),  # mean below 1: most delays 0
    "wide": dict(delay_mean=1000.0, delay_variance=1e8),  # exp() fallback whose tail reaches the 1e9 cap
    "uniform": dict(delay_kind=1, delay_lo=5, delay_hi=15),  # BASELINE configs[1]
}
TABLE_MODELS = ["baseline", "kmax254", "kmax255", "kmax4096", "narrow", "below1"]
KMAX = {"baseline": 156, "kmax254": 254, "kmax255": 255, "kmax4096": 4096, "kmax4097": 0, "narrow": 115, "below1": 7, "wide": 0}


def f2b(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def b2f(b):
    return struct.unpack("<d", struct.pack("<Q", int(b) & M64))[0]


def b2f_array(a):
    return np.asarray(a, np.uint64).view(np.float64)


# ---- restatements -------------------------------------------------------------------------------------------------------
def splitmix_seed(seed):
    """rand_xoshiro 0.6.0 Xoshiro256StarStar::seed_from_u64: four SplitMix64 outputs."""
    x, out = seed & M64, []
    for _ in range(4):
        x = (x + 0x9E3779B97F4A7C15) & M64
        z = x
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        out.append(z ^ (z >> 31))
    return out


def rotl(x, k):
    return ((x << k) | (x >> (64 - k))) & M64


def xoshiro_next(s):
    """One Xoshiro256** step: (output, next state)."""
    s0, s1, s2, s3 = s
    out = (rotl((s1 * 5) & M64, 7) * 9) & M64
    t = (s1 << 17) & M64
    s2 ^= s0
    s3 ^= s1
    s1 ^= s2
    s0 ^= s3
    s2 ^= t
    s3 = rotl(s3, 45)
    return out, [s0, s1, s2, s3]


def sample_single_inclusive(s, n, bits):
    """rand 0.8.3 UniformInt<u32 / u64>::sample_single_inclusive(0, n - 1) (bits = 32 / 64): (value, state, draws)."""
    mask = (1 << bits) - 1
    zone = ((n << (bits - n.bit_length())) & mask) - 1
    draws = 0
    while True:
        v, s = xoshiro_next(s)
        draws += 1
        if bits == 32:
            v >>= 32
        m = v * n
        if m & mask <= zone:
            return m >> bits, s, draws


def standard_normal(s, zx, zf, R):
    """rand_distr 0.4.0 StandardNormal (256-layer ziggurat) over host floats: (z, state, draws, libm calls), the calls as
    ("exp" | "log", argument) in the order the sampler makes them."""
    draws, calls = 0, []

    def nxt():
        nonlocal s, draws
        v, s = xoshiro_next(s)
        draws += 1
        return v

    while True:
        bits = nxt()
        i = bits & 0xFF
        u = b2f((1024 << 52) | (bits >> 12)) - 3.0
        x = u * zx[i]
        if abs(x) < zx[i + 1]:
            return x, s, draws, calls
        if i == 0:
            xx, yy = 1.0, 0.0
            while -2.0 * yy < xx * xx:
                a = open01(nxt())
                b = open01(nxt())
                calls += [("log", a), ("log", b)]
                xx = math.log(a) / R
                yy = math.log(b)
            return (xx - R if u < 0.0 else R - xx), s, draws, calls
        g = (nxt() >> 11) * (1.0 / 9007199254740992.0)
        arg = -x * x / 2.0
        calls.append(("exp", arg))
        if zf[i + 1] + (zf[i] - zf[i + 1]) * g < math.exp(arg):
            return x, s, draws, calls


def open01(v):
    """rand 0.8 Open01 for f64 of one output."""
    return b2f((1023 << 52) | (v >> 12)) - (1.0 - 2.220446049250313e-16 / 2.0)


# ---- state construction -------------------------------------------------------------------------------------------------
_INV9, _INV5 = pow(9, -1, 1 << 64), pow(5, -1, 1 << 64)


def s1_of_output(o):
    """The s1 that makes the output o: output = rotl(s1 * 5, 7) * 9 is a bijection of s1."""
    y = (o * _INV9) & M64
    return (((y >> 7) | (y << 57)) & M64) * _INV5 & M64


class StateSolver:
    """The Xoshiro256** state whose next four outputs are chosen.  The step is linear over GF(2), so s1 at steps 0..3 is a
    linear map of the 256 state bits; it has full rank, so any four outputs are reachable and fix the state.  The all-zero
    state (a fixed point: every output 0) is the image of four zero outputs only, and is refused."""

    def __init__(self):
        cols = []
        for j in range(256):
            s = [0, 0, 0, 0]
            s[j // 64] = 1 << (j % 64)
            col = 0
            for k in range(4):
                col |= s[1] << (64 * k)
                _, s = xoshiro_next(s)
            cols.append(col)
        M = np.array([[(cols[j] >> i) & 1 for j in range(256)] for i in range(256)], np.uint8)
        self.inv = _gf2_inverse(M).astype(np.float32)
        self.rank = 256

    def solve(self, outputs):
        """outputs: (n, 4) uint64-like; returns (n, 4) uint64 states."""
        outputs = np.asarray(outputs, dtype=np.uint64).reshape(-1, 4)
        assert (outputs != 0).any(axis=1).all(), "four zero outputs: the all-zero state"
        n = len(outputs)
        t = np.zeros((n, 256), np.float32)
        for k in range(4):
            s1 = np.array([s1_of_output(int(o)) for o in outputs[:, k]], dtype=np.uint64)
            t[:, 64 * k:64 * (k + 1)] = ((s1[:, None] >> np.arange(64, dtype=np.uint64)) & np.uint64(1)).astype(np.float32)
        x = (t @ self.inv.T).astype(np.int64) & 1  # exact: sums of at most 256 ones
        w = (x.reshape(n, 4, 64).astype(np.uint64) << np.arange(64, dtype=np.uint64)).sum(axis=2, dtype=np.uint64)
        return w


def _gf2_inverse(M):
    n = len(M)
    A = np.concatenate([M.copy(), np.eye(n, dtype=np.uint8)], axis=1)
    for c in range(n):
        piv = c + int(np.nonzero(A[c:, c])[0][0])
        if piv != c:
            A[[c, piv]] = A[[piv, c]]
        rows = np.nonzero(A[:, c])[0]
        rows = rows[rows != c]
        A[rows] ^= A[c]
    assert (A[:, :n] == np.eye(n, dtype=np.uint8)).all()
    return A[:, n:]


# ---- the three sides ----------------------------------------------------------------------------------------------------
class SweepSetC(ctypes.Structure):
    """sim_params.h SweepSet: one set's delay model."""
    _fields_ = [("delay_kind", ctypes.c_uint32), ("delay_const", ctypes.c_uint32), ("delay_const_value", ctypes.c_int64),
                ("mu", ctypes.c_double), ("sigma", ctypes.c_double), ("uni_lo", ctypes.c_uint64), ("uni_span", ctypes.c_uint64),
                ("tci", ctypes.c_int32), ("delay_kmax", ctypes.c_uint32), ("thr_off", ctypes.c_uint32), ("rt_off", ctypes.c_uint32)]


P = ctypes.c_void_p
_ARGS = [ctypes.POINTER(LbftConfig), ctypes.POINTER(LbftParamSet), ctypes.c_uint32]


def param_set(model):
    p = LbftParamSet()
    p.delay_kind = model.get("delay_kind", 0)
    p.delay_mean = model.get("delay_mean", 10.0)
    p.delay_variance = model.get("delay_variance", 4.0)
    p.delay_lo = model.get("delay_lo", 0)
    p.delay_hi = model.get("delay_hi", 0)
    p.target_commit_interval, p.delta, p.gamma, p.lambda_ = 100000, 20, 2.0, 0.5
    return p


class Setup:
    """A delay model, or a sweep over several (set s = models[s]), in the C form the three sides take."""

    def __init__(self, model=None, sets=None):
        self.models = sets
        self.cfg, self.keep = make_config([1], 4, 1000, **(model or {}))
        self.sets = (LbftParamSet * len(sets))(*[param_set(m) for m in sets]) if sets else None
        self.num_sets = len(sets) if sets else 0

    def args(self):
        return ctypes.byref(self.cfg), self.sets, self.num_sets


class Sides:
    """The oracle, the host twin and (gpu=True) the device probe, each running a copy of the records."""

    def __init__(self, gpu=False):
        self.oracle = ctypes.CDLL(_build.build_oracle())
        self.oracle.lbfo_sampler.argtypes = _ARGS + [P, ctypes.c_size_t]
        self.oracle.lbfo_last_error.restype = ctypes.c_char_p
        self.host = ctypes.CDLL(_build.build_sampler_hostcore())
        self.host.sampler_host.argtypes = _ARGS + [ctypes.c_uint32, P, ctypes.c_uint64]
        self.host.sampler_host_last_error.restype = ctypes.c_char_p
        self.host.sampler_tables.argtypes = _ARGS + [P, P, P, P, P, ctypes.c_uint64, P]
        self.probe = None
        if gpu:
            self.probe = ctypes.CDLL(_build.build_sampler_probe())
            self.probe.sampler_probe.argtypes = _ARGS + [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, P, ctypes.c_uint64]
            self.probe.sampler_probe_last_error.restype = ctypes.c_char_p

    def run_oracle(self, setup, recs):
        out = np.ascontiguousarray(recs.copy())
        if self.oracle.lbfo_sampler(*setup.args(), out.ctypes.data, len(out)) != 0:
            raise RuntimeError(self.oracle.lbfo_last_error().decode())
        return out

    def run_host(self, setup, recs, core):
        out = np.ascontiguousarray(recs.copy())
        if self.host.sampler_host(*setup.args(), core, out.ctypes.data, len(out)) != 0:
            raise RuntimeError(self.host.sampler_host_last_error().decode())
        return out

    def run_device(self, setup, recs, core, G, smem):
        out = np.ascontiguousarray(recs.copy())
        if self.probe.sampler_probe(*setup.args(), core, G, int(smem), out.ctypes.data, len(out)) != 0:
            raise RuntimeError(self.probe.sampler_probe_last_error().decode())
        return out

    def tables(self, setup):
        """(zig_x, zig_f, R, [per set: (SweepSetC, thresholds)]) from the product's HostSetup."""
        zx, zf = np.zeros(257), np.zeros(257)
        R = ctypes.c_double()
        n = max(1, setup.num_sets)
        models = (SweepSetC * n)()
        cap = 1 << 20
        thr = np.zeros(cap)
        length = ctypes.c_uint64()
        if self.host.sampler_tables(*setup.args(), zx.ctypes.data, zf.ctypes.data, ctypes.byref(R), ctypes.addressof(models),
                                    thr.ctypes.data, cap, ctypes.byref(length)) != 0:
            raise RuntimeError(self.host.sampler_host_last_error().decode())
        per = []
        for m in models:
            t = thr[m.thr_off:m.thr_off + m.delay_kmax + 2] if m.delay_kmax else np.zeros(0)
            per.append((m, t.copy()))
        return [float(v) for v in zx], [float(v) for v in zf], R.value, per


def records(states, op, arg=0, set_=0):
    r = np.zeros(len(states), REC)
    r["s"] = np.asarray(states, np.uint64).reshape(-1, 4)
    r["op"] = op
    r["arg"] = arg
    r["set"] = set_
    return r


def concat(*rs):
    return np.concatenate([r for r in rs if len(r)])


# ---- edge cases ---------------------------------------------------------------------------------------------------------
def u_of(m):
    """The ziggurat's u for the 52-bit mantissa m: u = -1 + m * 2^-51, exactly."""
    return (m - (1 << 51)) * 2.0 ** -51


def _bisect(lo, hi, pred):
    """The smallest integer in [lo, hi] with pred true, for pred monotone (false ... true); hi + 1 if none."""
    if not pred(hi):
        return hi + 1
    while lo < hi:
        mid = (lo + hi) // 2
        if pred(mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def fast_accept_ms(i, zx):
    """Mantissas at layer i's fast-accept boundary: the largest |u| with |u x_i| < x_{i+1} on each side and the next
    mantissa past it, and u = -1, u = 1 - 2^-51."""
    acc = lambda m: abs(u_of(m) * zx[i]) < zx[i + 1]  # noqa: E731
    ms = {0, (1 << 52) - 1}
    top = _bisect(1 << 51, (1 << 52) - 1, lambda m: not acc(m))  # first rejected u >= 0
    ms |= {top - 1, top} if top > 1 << 51 else {top}
    bot = _bisect(0, 1 << 51, lambda m: acc(m))  # first accepted u <= 0
    ms |= {bot - 1, bot} if bot <= 1 << 51 else {1 << 51}
    return sorted(m for m in ms if 0 <= m < (1 << 52))


def wedge_ks(i, m, zx, zf):
    """53-bit g's that put the wedge's lhs on each side of exp(-x^2 / 2) at layer i, u = u_of(m)."""
    x = u_of(m) * zx[i]
    rhs = math.exp(-x * x / 2.0)
    lhs = lambda k: zf[i + 1] + (zf[i] - zf[i + 1]) * (k * (1.0 / 9007199254740992.0))  # noqa: E731
    k = _bisect(0, (1 << 53) - 1, lambda k: lhs(k) < rhs)  # lhs falls with k
    return sorted({min(max(k + d, 0), (1 << 53) - 1) for d in (-1, 0)} | {0, (1 << 53) - 1})


def tail_a_ms(R, count=48):
    """Open01 mantissas for the tail's first uniform a: from the smallest a that can still end the loop (the largest deviate)
    up to a = 1 - 2^-53, spread log-uniformly."""
    m_min = largest_deviate_m(R)
    ms = {m_min, m_min + 1, (1 << 52) - 1}
    for e in np.linspace(math.log2(m_min + 1), 52, count):
        ms.add(min(int(2 ** e), (1 << 52) - 1))
    return sorted(ms)


def loop_exits(a, b, R):
    xx = math.log(a) / R
    return not (-2.0 * math.log(b) < xx * xx)


def largest_deviate_m(R):
    """The smallest Open01 mantissa of a with which the tail loop can end (b = 2^-53, its smallest): the largest deviate."""
    b = open01(0)
    return _bisect(0, (1 << 52) - 1, lambda m: loop_exits(open01(m << 12), b, R))


def largest_deviate(R):
    """R - ln(a) / R at that a: the largest |z| the ziggurat returns."""
    return R - math.log(open01(largest_deviate_m(R) << 12)) / R


def tail_b_ms(a, R):
    """Open01 mantissas of b either side of the loop boundary -2 ln b = (ln a / R)^2 for this a (empty if none exits)."""
    k = _bisect(0, (1 << 52) - 1, lambda m: not loop_exits(a, open01(m << 12), R))  # first b that continues
    if k == 0:
        return []
    return sorted(m for m in {k - 1, k, 0} if m < (1 << 52))


class Cases:
    """Records of one case group with what each is for: recs (REC), label per record."""

    def __init__(self):
        self.parts, self.labels = [], []

    def add(self, recs, label):
        self.parts.append(recs)
        self.labels += [label] * len(recs)

    def build(self):
        return concat(*self.parts), np.array(self.labels)


def normal_cases(solver, zx, zf, R, rng):
    """standard_normal at the edges of every layer: the fast-accept boundary, u = -1 and 1 - 2^-51, the wedge decision either
    side of exp(-x^2/2) (layers 1..255), the tail loop either side of its boundary and at the largest deviate (layer 0)."""
    outs, labels = [], []
    junk = lambda: int(rng.integers(0, 1 << 63)) | 1  # noqa: E731
    a_ms = tail_a_ms(R)
    for i in range(256):
        for m in fast_accept_ms(i, zx):
            o0 = (m << 12) | (int(rng.integers(0, 16)) << 8) | i
            x = u_of(m) * zx[i]
            if abs(x) < zx[i + 1]:
                outs.append([o0, junk(), junk(), junk()])
                labels.append("fast")
            elif i > 0:
                for k in wedge_ks(i, m, zx, zf):
                    outs.append([o0, (k << 11) | int(rng.integers(0, 1 << 11)), junk(), junk()])
                    labels.append("wedge")
            else:
                for ma in a_ms[::4] + [a_ms[0]]:
                    a = open01(ma << 12)
                    for mb in tail_b_ms(a, R):
                        outs.append([o0, (ma << 12) | int(rng.integers(0, 1 << 12)), (mb << 12) | int(rng.integers(0, 1 << 12)), junk()])
                        labels.append("tail")
    return solver.solve(np.array(outs, dtype=np.uint64)), np.array(labels)


def delay_z_values(thr, R):
    """z = thr[k] and the double below it for every finite threshold, +-ZMAX, +-the largest deviate and 0."""
    zs = {ZMAX, -ZMAX, 0.0, largest_deviate(R), -largest_deviate(R)}
    for t in thr[1:-1]:
        if math.isfinite(t):
            zs |= {float(t), math.nextafter(float(t), -math.inf)}
    return sorted(z for z in zs if -ZMAX <= z <= ZMAX)


def glibc_delay(mu, sigma, z):
    """(int64) exp(mu + sigma z) with the host libm, as the oracle and the tables compute it."""
    v = math.exp(mu + sigma * z)
    return int(v) if v < 9.0e18 else None


def exact_floor_delay(mu, sigma, z):
    """floor(exp(t)) exactly, t the double mu + sigma z."""
    t = mu + sigma * z
    with mpmath.workprec(256):
        return int(mpmath.floor(mpmath.exp(mpmath.mpf(t))))


def near_int_states(solver, mu, sigma, zx, rng, targets=(1, 2, 3, 7, 10, 57, 100, 999, 1000, 12345, 99999, 150000)):
    """States whose standard_normal is a layer-0 fast accept z near (ln(n (1 + d)) - mu) / sigma: delays within, at and just
    outside the 1e-9 band of the exp() fallback's near-integer advisory."""
    outs = []
    R = zx[1]
    with mpmath.workprec(200):
        for n in targets:
            for d in (0.0, 0.5e-9, -0.5e-9, 0.99e-9, -0.99e-9, 1.01e-9, -1.01e-9, 2e-9, -2e-9):
                z = (mpmath.log(mpmath.mpf(n) * (1 + mpmath.mpf(d))) - mpmath.mpf(mu)) / mpmath.mpf(sigma)
                if not abs(z) < R:
                    continue
                m0 = int(mpmath.nint((z / mpmath.mpf(zx[0]) + 1) * mpmath.mpf(2) ** 51))
                for m in range(m0 - 2, m0 + 3):
                    outs.append([(m << 12) | (int(rng.integers(0, 16)) << 8) | 0, int(rng.integers(1, 1 << 63)), 1, 1])
    return solver.solve(np.array(outs, dtype=np.uint64))


def near_int_band(mu, sigma, z):
    """(in_band, distance): whether exp(t) (t = mu + sigma z, exact exp) is within 1e-9 max(r, 1) of the nearest integer r."""
    t = mu + sigma * z
    with mpmath.workprec(256):
        v = mpmath.exp(mpmath.mpf(t))
        r = mpmath.nint(v)
        dist = abs(v - r)
        return dist < mpmath.mpf(1e-9) * max(r, 1), float(dist / max(r, 1))


def range_first_outputs(n, bits):
    """First outputs at the rejection boundary of sample_single_inclusive(0, n - 1): the largest accepted low product
    (v n mod 2^bits <= zone) and the smallest rejected one, each solved for v (the low 32 bits of a u32 draw's output are
    free)."""
    mask = (1 << bits) - 1
    zone = ((n << (bits - n.bit_length())) & mask) - 1
    tz = (n & -n).bit_length() - 1
    odd = n >> tz
    span = 1 << (bits - tz)
    inv = pow(odd, -1, span) if span > 1 else 0
    res = []
    for lo in ((zone >> tz) << tz, ((zone >> tz) + 1) << tz):
        if lo > mask:
            continue
        v = ((lo >> tz) * inv) % span
        assert (v * n) & mask == lo
        res.append((v << 32) | 0x9E3779B9 if bits == 32 else v)
    return res


UNIFORM_SPANS = sorted({1, 2, 3, (1 << 29) + 1} | {1 << k for k in range(1, 30)} | {(1 << k) + 1 for k in range(1, 29)}
                       | {3 << k for k in range(0, 28)})


MODELS["const"] = dict(delay_mean=10.0, delay_variance=0.0)  # sigma = 0: the host's exp(mu), the deviate still drawn
FALLBACK_MODELS = ["kmax4097", "wide"]


def uniform_model(span):
    lo = 5 if 5 + span - 1 <= 1 << 29 else 0
    return dict(delay_kind=1, delay_lo=lo, delay_hi=lo + span - 1)


def case_groups(sides, solver, seed=7):
    """Every case group: name -> (model name or uniform model dict, records).  Models are MODELS keys except the uniform
    spans ("uniform:<span>")."""
    rng = np.random.default_rng(seed)
    rand_states = lambda n: solver.solve(rng.integers(1, 1 << 63, (n, 4), dtype=np.uint64))  # noqa: E731
    zx, zf, R, _ = sides.tables(Setup(MODELS["baseline"]))
    groups = {}
    # integers: seeding, steps, the shuffle's u32 draws at n = 1..64, the u64 draws at the spans and beyond
    seeds = np.array([0, 1, 2, 52, M64, 1 << 63, 0x9E3779B97F4A7C15] + list(rng.integers(0, 1 << 63, 57, dtype=np.uint64)), np.uint64)
    parts = [records(np.ones((len(seeds), 4), np.uint64), OP_SEED, seeds), records(rand_states(256), OP_NEXT_U64)]
    for n in range(1, 65):
        firsts = range_first_outputs(n, 32)
        st = solver.solve([[f, int(rng.integers(1, 1 << 63)), int(rng.integers(1, 1 << 63)), 1] for f in firsts])
        parts += [records(st, OP_RANGE_U32, n), records(rand_states(8), OP_RANGE_U32, n)]
    for n in UNIFORM_SPANS + [(1 << 63) + 1, M64, 3 << 62, (1 << 64) - (1 << 32), 1 << 63]:
        firsts = range_first_outputs(n, 64)
        st = solver.solve([[f, int(rng.integers(1, 1 << 63)), int(rng.integers(1, 1 << 63)), 1] for f in firsts])
        parts += [records(st, OP_RANGE_U64, n), records(rand_states(4), OP_RANGE_U64, n)]
    groups["integers"] = ("baseline", concat(*parts))
    # the ziggurat's edges, and the same states through every delay model
    normal_states, labels = normal_cases(solver, zx, zf, R, rng)
    groups["normal"] = ("baseline", records(normal_states, OP_NORMAL))
    tail = normal_states[labels == "tail"]
    for name in TABLE_MODELS + ["const"]:
        groups["sample_delay:" + name] = (name, records(normal_states, OP_SAMPLE_DELAY))
    for name in TABLE_MODELS:
        _, _, _, per = sides.tables(Setup(MODELS[name]))
        zs = np.array([f2b(z) for z in delay_z_values(per[0][1], R)], np.uint64)
        groups["delay_from_z:" + name] = (name, records(np.ones((len(zs), 4), np.uint64), OP_DELAY_FROM_Z, zs))
    for name in FALLBACK_MODELS:
        _, _, _, per = sides.tables(Setup(MODELS[name]))
        m = per[0][0]
        near = near_int_states(solver, m.mu, m.sigma, zx, rng)
        groups["fallback:" + name] = (name, records(concat(near, tail, normal_states[:512]), OP_SAMPLE_DELAY))
    for span in UNIFORM_SPANS:
        st = solver.solve([[f, int(rng.integers(1, 1 << 63)), int(rng.integers(1, 1 << 63)), 1] for f in range_first_outputs(span, 64)])
        groups["uniform:%d" % span] = (uniform_model(span), records(concat(st, rand_states(4)), OP_SAMPLE_DELAY))
    return groups, (zx, zf, R)


def model_of(name_or_model):
    return MODELS[name_or_model] if isinstance(name_or_model, str) else name_or_model


def traced_libm_calls(recs, zx, zf, R):
    """Per OP_NORMAL record, the libm calls its standard_normal makes (glibc's path)."""
    return [standard_normal([int(v) for v in r["s"]], zx, zf, R)[3] for r in recs]


def same(a, b):
    """Per record: result, state and draws identical."""
    return (a["result"] == b["result"]) & (a["s"] == b["s"]).all(axis=1) & (a["draws"] == b["draws"])


def check_fallback(inp, dev, ref, model, zx, zf, R, libm_differs):
    """The exp() fallback's contract on records run through sample_delay: a delay at or past 1e9 is 1e9 with
    ST_TIME_OVERFLOW; a delay that differs from the oracle's carries ST_DELAY_NEAR_INT (soundness); the flag fires only when
    exp(mu + sigma z) is within 1e-9 max(r, 1) of an integer r (precision, exactly with mpmath).  Returns (flagged, overflowed,
    differing) counts."""
    mu, sigma = model.mu, model.sigma
    flagged = overflowed = differing = 0
    for k in range(len(dev)):
        d, r = dev[k], ref[k]
        if libm_differs[k]:
            continue
        assert (d["s"] == r["s"]).all() and d["draws"] == r["draws"], k
        st, z = int(d["status"]), zs_of(inp[k], zx, zf, R)
        v = math.exp(mu + sigma * z)
        if st & ST_TIME_OVERFLOW:
            assert v >= 1e9 and int(d["result"]) == 1000000000, k
            overflowed += 1
            continue
        assert v < 1e9, k
        if st & ST_DELAY_NEAR_INT:
            flagged += 1
            in_band, dist = near_int_band(mu, sigma, z)
            assert in_band or dist < 1e-9 + 1e-15, (k, dist)
        if d["result"] != r["result"]:
            differing += 1
            assert st & ST_DELAY_NEAR_INT, k
    return flagged, overflowed, differing


_Z_CACHE = {}


def zs_of(rec, zx, zf, R):
    """The deviate standard_normal draws from the record's state (an input record; glibc's path)."""
    key = tuple(int(v) for v in rec["s"])
    if key not in _Z_CACHE:
        _Z_CACHE[key] = standard_normal(list(key), zx, zf, R)[0]
    return _Z_CACHE[key]
