"""Build recipes for the native pieces (run by ``__graft_entry__.build()``).

* ``csrc/liblbft_b200.so`` — the product: sm_90a (H100) CUDA kernels + the C ABI of ``include/lbft.h``.
* ``oracle/liblbft_oracle.so``, ``tests/hostcore/libhostcore.so``, ``tests/hostcore/libhostcore_sweep.so``,
  ``tests/hostcore/libhostcore_ct.so``, ``tests/hostcore/libhostcore_latency.so``, ``tests/hostcore/libhostcore_fault.so``, ``tests/hostcore/libhostcore_rights.so``,
  ``tests/hostcore/libhostcore_committee.so``, ``tests/hostcore/libhostcore_link.so``, ``tests/hostcore/libhostcore_outage.so``,
  ``tests/hostcore/libhostcore_block_latency.so``, ``tests/hostcore/libhostcore_lane_block.so`` and ``tests/hostcore/libhostcore_sampler.so`` — test
  infrastructure only; so are ``tests/gpuprobe/libblock_threshold_probe.so`` and ``tests/gpuprobe/libsampler_probe.so``, CUDA probes of device
  functions.
All artefacts are built in-tree and git-ignored.
"""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "librabft_simulator_b200", "csrc")
LIB_PATH = os.environ.get("LBFT_LIB_PATH") or os.path.join(CSRC, "liblbft_b200.so")
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_PATH = os.path.join(ORACLE_DIR, "liblbft_oracle.so")
HOSTCORE_DIR = os.path.join(ROOT, "tests", "hostcore")
HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore.so")
SWEEP_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_sweep.so")
CT_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_ct.so")
LATENCY_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_latency.so")
FAULT_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_fault.so")
RIGHTS_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_rights.so")
COMMITTEE_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_committee.so")
LINK_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_link.so")
OUTAGE_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_outage.so")
BLOCK_LATENCY_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_block_latency.so")
LANE_BLOCK_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_lane_block.so")
SAMPLER_HOSTCORE_PATH = os.path.join(HOSTCORE_DIR, "libhostcore_sampler.so")
GPUPROBE_DIR = os.path.join(ROOT, "tests", "gpuprobe")
BLOCK_THRESHOLD_PROBE_PATH = os.path.join(GPUPROBE_DIR, "libblock_threshold_probe.so")
SAMPLER_PROBE_PATH = os.path.join(GPUPROBE_DIR, "libsampler_probe.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]
# Translation units of the product library: the host runtime (C ABI) and the kernel instantiations, one group per file so
# that they compile in parallel and the bench kernel (k_fixed.cu) can be rebuilt alone; the sweep twins (lbft_create_sweep)
# and the commit-times twins (LBFT_FLAG_COMMIT_TIMES) in units of their own.
PRODUCT_UNITS = ["lbft_api.cu", "k_fixed.cu", "k_scan.cu", "k_calendar.cu", "k_heap.cu", "k_wide.cu", "k_sweep_thread.cu",
                 "k_sweep_wide.cu", "k_ct_thread.cu", "k_ct_wide.cu", "k_ct_sweep_thread.cu", "k_ct_sweep_wide.cu"]
PRODUCT_HEADERS = ["kernels.cuh", "sim_core.cuh", "sim_params.h", "host_setup.hpp"]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _run(cmd, cwd):
    proc = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), proc.stdout))
    return proc.stdout


def nvcc_path():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build_product(force=False, verbose_ptxas=False, lib_path=None):
    """nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo on every unit (objects in csrc/build/, in parallel), then one
    shared library.  Only units older than their sources are recompiled."""
    from concurrent.futures import ThreadPoolExecutor
    lib_path = lib_path or LIB_PATH
    headers = [os.path.join(CSRC, f) for f in PRODUCT_HEADERS] + [os.path.join(ROOT, "include", "lbft.h")]
    sources = headers + [os.path.join(CSRC, u) for u in PRODUCT_UNITS]
    if not (force or verbose_ptxas) and _newer(lib_path, sources):
        return lib_path  # (the objects need not exist: on the GPU box only the library travels)
    objdir = os.path.join(CSRC, "build" if lib_path == LIB_PATH else "build_" + os.path.basename(lib_path))
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for unit in PRODUCT_UNITS:
        obj = os.path.join(objdir, unit.replace(".cu", ".o"))
        if force or verbose_ptxas or not _newer(obj, headers + [os.path.join(CSRC, unit)]):
            jobs.append((unit, obj))
    flags = NVCC_FLAGS + (["-Xptxas", "-v"] if verbose_ptxas else [])
    with ThreadPoolExecutor(max_workers=min(len(PRODUCT_UNITS), os.cpu_count() or 2)) as pool:
        outs = list(pool.map(lambda j: _run([nvcc_path()] + flags + ["-c", "-o", j[1], j[0]], CSRC), jobs))
    if verbose_ptxas:
        print("\n".join(outs))
    objs = [os.path.join(objdir, u.replace(".cu", ".o")) for u in PRODUCT_UNITS]
    if jobs or not _newer(lib_path, objs):
        _run([nvcc_path()] + GENCODE + ["-shared", "-o", lib_path] + objs, CSRC)
    return lib_path


def build_oracle(force=False):
    srcs = [os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "oracle_selftest.cpp", "lbft_oracle.hpp")]
    srcs.append(os.path.join(ROOT, "include", "lbft.h"))
    if not force and _newer(ORACLE_PATH, srcs):
        return ORACLE_PATH
    _run(["make", "-B", "liblbft_oracle.so"], ORACLE_DIR)
    return ORACLE_PATH


def build_oracle_native():
    """The CPU-baseline build of the oracle (-O3 -march=native), compiled on the machine that times it under the temporary
    directory (the source tree may be read-only there).  The file name carries a hash of the CPU and of the oracle's
    sources and build recipe, so that neither a copy built for another CPU nor one built from another checkout's sources
    is ever loaded.  Falls back to the portable build if no compiler is available.  Returns (path, flags description)."""
    import hashlib
    import platform
    import tempfile
    try:
        cpu = [ln for ln in open("/proc/cpuinfo") if ln.startswith(("model name", "flags"))][:2]
    except OSError:
        cpu = [platform.processor()]
    h = hashlib.sha1("".join(cpu).encode())
    for src in [os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "oracle_selftest.cpp", "lbft_oracle.hpp", "Makefile")] + [
            os.path.join(ROOT, "include", "lbft.h")]:
        with open(src, "rb") as f:
            h.update(f.read())
    outdir = os.path.join(tempfile.gettempdir(), "lbft-oracle-native-%d" % os.getuid())
    path = os.path.join(outdir, "liblbft_oracle_native_%s.so" % h.hexdigest()[:16])
    if os.path.exists(path):
        return path, "-O3 -march=native"
    try:
        os.makedirs(outdir, exist_ok=True)
        tmp = "%s.%d.tmp" % (path, os.getpid())
        _run(["make", "-B", "liblbft_oracle_native.so", "NATIVE_OUT=" + tmp], ORACLE_DIR)
        os.replace(tmp, path)
        return path, "-O3 -march=native"
    except Exception:
        return build_oracle(), "-O2 (portable build: native build failed)"


def build_hostcore(force=False):
    srcs = [os.path.join(HOSTCORE_DIR, "hostcore.cpp")] + [
        os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")]
    if not force and _newer(HOSTCORE_PATH, srcs):
        return HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", HOSTCORE_PATH, "hostcore.cpp"], HOSTCORE_DIR)
    return HOSTCORE_PATH


def build_sweep_hostcore(force=False):
    """The host-compiled core of sweep handles (tests/hostcore/sweep_hostcore.cpp): test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, "sweep_hostcore.cpp"), os.path.join(ROOT, "include", "lbft.h")] + [
        os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")]
    if not force and _newer(SWEEP_HOSTCORE_PATH, srcs):
        return SWEEP_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", SWEEP_HOSTCORE_PATH, "sweep_hostcore.cpp"], HOSTCORE_DIR)
    return SWEEP_HOSTCORE_PATH


def build_ct_hostcore(force=False):
    """The host-compiled core of commit-times handles and the oracle observed per event (tests/hostcore/ct_hostcore.cpp):
    test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, "ct_hostcore.cpp"), os.path.join(ROOT, "include", "lbft.h")] + [
        os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(CT_HOSTCORE_PATH, srcs):
        return CT_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", CT_HOSTCORE_PATH, "ct_hostcore.cpp"], HOSTCORE_DIR)
    return CT_HOSTCORE_PATH


def build_latency_hostcore(force=False):
    """The CT core with the product's commit-latency statistics on the host (tests/hostcore/latency_hostcore.cpp, which compiles
    ct_hostcore.cpp into itself): test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("latency_hostcore.cpp", "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(LATENCY_HOSTCORE_PATH, srcs):
        return LATENCY_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", LATENCY_HOSTCORE_PATH, "latency_hostcore.cpp"], HOSTCORE_DIR)
    return LATENCY_HOSTCORE_PATH


def build_fault_hostcore(force=False):
    """The SW and SW + CT cores of fault sweeps over the product's host setup (tests/hostcore/fault_hostcore.cpp, which compiles
    ct_hostcore.cpp into itself): test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("fault_hostcore.cpp", "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(FAULT_HOSTCORE_PATH, srcs):
        return FAULT_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", FAULT_HOSTCORE_PATH, "fault_hostcore.cpp"], HOSTCORE_DIR)
    return FAULT_HOSTCORE_PATH


def build_block_latency_hostcore(force=False):
    """The CT cores of plain handles, sweeps and fault sweeps with the product's block-latency statistics on the host
    (tests/hostcore/block_latency_hostcore.cpp, which compiles fault_hostcore.cpp and ct_hostcore.cpp into itself): test
    infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("block_latency_hostcore.cpp", "fault_hostcore.cpp", "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(BLOCK_LATENCY_HOSTCORE_PATH, srcs):
        return BLOCK_LATENCY_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", BLOCK_LATENCY_HOSTCORE_PATH, "block_latency_hostcore.cpp"], HOSTCORE_DIR)
    return BLOCK_LATENCY_HOSTCORE_PATH


def build_lane_block_hostcore(force=False):
    """The bench kernel's core with its compact node words and slots in lane blocks (tests/hostcore/lane_block_hostcore.cpp):
    test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, "lane_block_hostcore.cpp")] + [
        os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")]
    if not force and _newer(LANE_BLOCK_HOSTCORE_PATH, srcs):
        return LANE_BLOCK_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", LANE_BLOCK_HOSTCORE_PATH, "lane_block_hostcore.cpp"], HOSTCORE_DIR)
    return LANE_BLOCK_HOSTCORE_PATH


def build_block_threshold_probe(force=False):
    """The lane form of the block threshold time (sim_core.cuh block_threshold_time_lanes) over synthetic tables on the device
    (tests/gpuprobe/block_threshold_probe.cu), with the product's nvcc flags: test infrastructure, never linked into the
    product library."""
    srcs = [os.path.join(GPUPROBE_DIR, "block_threshold_probe.cu")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h")]
    if not force and _newer(BLOCK_THRESHOLD_PROBE_PATH, srcs):
        return BLOCK_THRESHOLD_PROBE_PATH
    _run([nvcc_path()] + NVCC_FLAGS + ["-shared", "-o", BLOCK_THRESHOLD_PROBE_PATH, "block_threshold_probe.cu"], GPUPROBE_DIR)
    return BLOCK_THRESHOLD_PROBE_PATH


def _sampler_sources(main):
    return [main, os.path.join(GPUPROBE_DIR, "sampler_ops.cuh"), os.path.join(ROOT, "include", "lbft.h")] + [
        os.path.join(CSRC, f) for f in PRODUCT_HEADERS]


def build_sampler_probe(force=False):
    """The device sampler (sim_core.cuh Core's RNG, range draws, ziggurat and delay lookup) on records with explicit states
    (tests/gpuprobe/sampler_probe.cu), with the product's nvcc flags: test infrastructure, never linked into the product
    library."""
    srcs = _sampler_sources(os.path.join(GPUPROBE_DIR, "sampler_probe.cu"))
    if not force and _newer(SAMPLER_PROBE_PATH, srcs):
        return SAMPLER_PROBE_PATH
    _run([nvcc_path()] + NVCC_FLAGS + ["-shared", "-o", SAMPLER_PROBE_PATH, "sampler_probe.cu"], GPUPROBE_DIR)
    return SAMPLER_PROBE_PATH


def build_sampler_hostcore(force=False):
    """The host-compiled twin of the sampler probe (tests/hostcore/sampler_hostcore.cpp): test infrastructure."""
    srcs = _sampler_sources(os.path.join(HOSTCORE_DIR, "sampler_hostcore.cpp"))
    if not force and _newer(SAMPLER_HOSTCORE_PATH, srcs):
        return SAMPLER_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", SAMPLER_HOSTCORE_PATH, "sampler_hostcore.cpp"], HOSTCORE_DIR)
    return SAMPLER_HOSTCORE_PATH


def build_rights_hostcore(force=False):
    """The SW and SW + CT cores of rights sweeps over the product's host setup and set table (tests/hostcore/rights_hostcore.cpp,
    which compiles fault_hostcore.cpp and ct_hostcore.cpp into itself): test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("rights_hostcore.cpp", "fault_hostcore.cpp", "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(RIGHTS_HOSTCORE_PATH, srcs):
        return RIGHTS_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", RIGHTS_HOSTCORE_PATH, "rights_hostcore.cpp"], HOSTCORE_DIR)
    return RIGHTS_HOSTCORE_PATH


def build_committee_hostcore(force=False):
    """The SW and SW + CT cores of committee sweeps over the product's host setup and set table
    (tests/hostcore/committee_hostcore.cpp, which compiles rights_hostcore.cpp, fault_hostcore.cpp and ct_hostcore.cpp into
    itself): test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("committee_hostcore.cpp", "rights_hostcore.cpp", "fault_hostcore.cpp", "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(COMMITTEE_HOSTCORE_PATH, srcs):
        return COMMITTEE_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", COMMITTEE_HOSTCORE_PATH, "committee_hostcore.cpp"], HOSTCORE_DIR)
    return COMMITTEE_HOSTCORE_PATH


def build_link_hostcore(force=False):
    """The SW and SW + CT cores of links sweeps over the product's host setup and set table, and the oracle with link latencies
    (tests/hostcore/link_hostcore.cpp with tests/hostcore/link_oracle.hpp, which compiles committee_hostcore.cpp,
    rights_hostcore.cpp, fault_hostcore.cpp and ct_hostcore.cpp into itself): test infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("link_hostcore.cpp", "link_oracle.hpp", "committee_hostcore.cpp", "rights_hostcore.cpp",
                                                   "fault_hostcore.cpp", "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(LINK_HOSTCORE_PATH, srcs):
        return LINK_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", LINK_HOSTCORE_PATH, "link_hostcore.cpp"], HOSTCORE_DIR)
    return LINK_HOSTCORE_PATH


def build_outage_hostcore(force=False):
    """The SW and SW + CT cores of outage sweeps over the product's host setup and set table, and the oracle with link latencies
    and outage windows (tests/hostcore/outage_hostcore.cpp with tests/hostcore/outage_oracle.hpp, which compiles
    link_hostcore.cpp, committee_hostcore.cpp, rights_hostcore.cpp, fault_hostcore.cpp and ct_hostcore.cpp into itself): test
    infrastructure."""
    srcs = [os.path.join(HOSTCORE_DIR, f) for f in ("outage_hostcore.cpp", "outage_oracle.hpp", "link_hostcore.cpp", "link_oracle.hpp",
                                                   "committee_hostcore.cpp", "rights_hostcore.cpp", "fault_hostcore.cpp",
                                                   "ct_hostcore.cpp")] + [
        os.path.join(ROOT, "include", "lbft.h")] + [os.path.join(CSRC, f) for f in ("sim_core.cuh", "sim_params.h", "host_setup.hpp")] + [
        os.path.join(ORACLE_DIR, f) for f in ("oracle_capi.cpp", "lbft_oracle.hpp")]
    if not force and _newer(OUTAGE_HOSTCORE_PATH, srcs):
        return OUTAGE_HOSTCORE_PATH
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-DLBFT_CHECK_C1",
          "-o", OUTAGE_HOSTCORE_PATH, "outage_hostcore.cpp"], HOSTCORE_DIR)
    return OUTAGE_HOSTCORE_PATH


def build_all(force=False):
    return (build_product(force), build_oracle(force), build_hostcore(force), build_sweep_hostcore(force), build_ct_hostcore(force),
            build_latency_hostcore(force), build_fault_hostcore(force), build_block_latency_hostcore(force),
            build_lane_block_hostcore(force), build_block_threshold_probe(force), build_rights_hostcore(force),
            build_committee_hostcore(force), build_link_hostcore(force), build_outage_hostcore(force),
            build_sampler_probe(force), build_sampler_hostcore(force))
