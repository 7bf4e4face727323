"""Build libovb200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

Per-feature geometry (k_triangulate.cu, k_feature.cu) is compiled with -fmad=false so its rounding sequence follows the
reference's non-FMA Eigen arithmetic (SURVEY.md App. A.11); the dense algebra (TSQR, EKF) keeps FMA contraction.
Usage: python -m open_vins_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libovb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]

UNITS = [
    # (source, extra flags)
    ("k_triangulate.cu", ["-fmad=false"]),
    ("k_feature.cu", ["-fmad=false"]),
    ("k_tsqr.cu", []),
    ("k_gram.cu", []),
    ("k_cholqr.cu", []),
    ("k_ekf.cu", []),
    ("ovb_api.cu", []),
    ("anchor_change.cu", ["-fmad=false"]),  # UpdaterSLAM::perform_anchor_change, one source for the host and the device
    ("k_init_batch.cu", ["-fmad=false"]),  # the mean update between delayed-init landmarks, include/ovb200_math.hpp's source
]
HEADERS = ["ovb_internal.cuh", "geom.cuh", "chol.cuh", "chol_tiles.cuh", "chi2_table.inc", os.path.join("..", "..", "include", "ovb200.h"),
           os.path.join("..", "..", "include", "ovb200_math.hpp")]


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs = []
    for src, extra in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(CSRC, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            cmd = [NVCC] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), flush=True)
            subprocess.check_call(cmd)
    if force or _stale(OUT, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", OUT] + objs + ["-lcudart"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return OUT


def build_host_test(force: bool = False) -> str:
    """Compile tests/cpp/host_shim_test.cpp (the C++ host mirror of include/ovb200_host.hpp driving one update) against
    the in-tree library; returns the executable's path."""
    root = os.path.dirname(HERE)
    src = os.path.join(root, "tests", "cpp", "host_shim_test.cpp")
    exe = os.path.join(root, "tests", "cpp", "host_shim_test")
    deps = [src, os.path.join(root, "include", "ovb200_host.hpp"), os.path.join(root, "include", "ovb200.h"), OUT]
    if force or _stale(exe, deps):
        cmd = [os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-Wall", "-I", os.path.join(root, "include"), src, "-L", HERE, "-lovb200",
               "-Wl,-rpath,$ORIGIN/../../open_vins_b200", "-o", exe]
        subprocess.check_call(cmd)
    return exe


def build_sim_tools(force: bool = False) -> str:
    """rpng_sim runner (tools/run_simulation.cpp over include/ovb200_vio.hpp) with the CUDA engine as backend:
    open_vins_b200/ovb_run_simulation. (The checker twin with the CPU backend is built by the test infrastructure.)"""
    root = os.path.dirname(HERE)
    src = os.path.join(root, "tools", "run_simulation.cpp")
    inc = os.path.join(root, "include")
    hdrs = [os.path.join(inc, h) for h in ("ovb200.h", "ovb200_host.hpp", "ovb200_math.hpp", "ovb200_sim.hpp", "ovb200_vio.hpp")]
    cxx = os.environ.get("CXX", "g++")
    exe = os.path.join(HERE, "ovb_run_simulation")
    if force or _stale(exe, [src, OUT] + hdrs):
        subprocess.check_call([cxx, "-std=c++17", "-O2", "-Wall", "-pthread", "-DOVB_SIM_ENGINE", "-I", inc, src, "-L", HERE, "-lovb200", "-Wl,-rpath,$ORIGIN",
                               "-o", exe])
    return exe


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
