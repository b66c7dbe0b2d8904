"""Builds libsdbg.so (the sm_90a kernels + C ABI) in-tree with nvcc. No JIT cache: the .so lives
under serenedb_b200/_lib/, next to the package that loads it."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "_lib")
LIB_PATH = os.path.join(LIB_DIR, "libsdbg.so")
SOURCES = [os.path.join(CSRC, "sdbg_abi.cu"), os.path.join(CSRC, "posting_format.cpp")]
DEPS = SOURCES + [os.path.join(CSRC, f) for f in ("bm25_kernels.cuh", "bm25_stream.cuh", "bm25_merge.cuh", "bm25_count.cuh", "bm25_emit.cuh", "bm25_agg.cuh", "bm25_facet.cuh", "bm25_sort.cuh", "bm25_phrase.cuh", "column_kernels.cuh", "device_common.cuh",
                                                   "posting_format.hpp")] + [
    os.path.join(os.path.dirname(HERE), "include", "sdbg.h")]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-cudart", "static"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def is_stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a. Returns the library path."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = nvcc_path()
    if nvcc is None:
        if os.path.exists(LIB_PATH):
            return LIB_PATH  # no compiler here and no source changed since the last build: use that build
        raise RuntimeError("nvcc not found and no prebuilt libsdbg.so")
    os.makedirs(LIB_DIR, exist_ok=True)
    tmp = LIB_PATH + ".tmp"
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + SOURCES + ["-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB_PATH)
    if verbose:
        print(res.stderr)
    return LIB_PATH


HOST_DIR = os.path.join(HERE, "host")
SELFTEST = os.path.join(LIB_DIR, "adapter_selftest")


def build_adapters(force=False):
    """Compile the C++ adapters (GpuTopKIterator : irs::DocIterator, GpuAggScan) against the mock
    reference headers and link them with libsdbg.so into a self-test binary."""
    srcs = [os.path.join(HOST_DIR, f) for f in ("adapter_selftest.cpp", "gpu_adapters.cpp")]
    deps = srcs + [os.path.join(HOST_DIR, f) for f in ("gpu_adapters.hpp", "irs_mock.hpp")] + [LIB_PATH]
    if not force and os.path.exists(SELFTEST) and all(os.path.getmtime(d) <= os.path.getmtime(SELFTEST) for d in deps):
        return SELFTEST
    gxx = shutil.which("g++")
    if gxx is None:
        if os.path.exists(SELFTEST):
            return SELFTEST
        raise RuntimeError("g++ not found")
    cmd = [gxx, "-std=c++20", "-O2", "-Wall", "-Wextra", "-o", SELFTEST] + srcs + ["-L" + LIB_DIR, "-lsdbg", "-Wl,-rpath,$ORIGIN"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed:\n" + res.stdout + res.stderr)
    return SELFTEST


if __name__ == "__main__":
    print(build(force=True, verbose=True))
