"""Shared by the ovb_cov_propagate_imu tests: builds tests/cpp/prop_probe.cpp and the host-propagation twin of the rpng_sim
runner, reads the probe's dump, and restates the host accumulation of Propagator::propagate_and_clone in numpy.

The numpy restatement uses only elementwise multiplies and adds in the host loop's order (each entry one dot product over
ascending k, starting from 0.0), so its results are the host's bits, not merely close to them."""
from __future__ import annotations

import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "open_vins_b200")
INC = os.path.join(ROOT, "include")
CALIB_N = {0: 15, 1: 30, 2: 39}  # no IMU intrinsics / intrinsics without g-sensitivity / with


def build_probe(out_dir) -> str:
    exe = os.path.join(str(out_dir), "prop_probe")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-Wall", "-I", INC, os.path.join(ROOT, "tests", "cpp", "prop_probe.cpp"),
                           "-L", LIBDIR, "-lovb200", "-Wl,-rpath," + LIBDIR, "-o", exe])
    return exe


def build_host_propagation_runner(out_dir) -> str:
    """tools/run_simulation.cpp on the engine, with the IMU accumulation left on the host (tests/cpp/host_propagation_backend.hpp),
    compiled like the product runner (open_vins_b200.build.build_sim_tools)."""
    exe = os.path.join(str(out_dir), "run_simulation_host_propagation")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-Wall", "-pthread", "-DOVB_SIM_HOST_PROPAGATION", "-I",
                           os.path.join(ROOT, "tests", "cpp"), "-I", INC, os.path.join(ROOT, "tools", "run_simulation.cpp"), "-L", LIBDIR, "-lovb200",
                           "-Wl,-rpath," + LIBDIR, "-o", exe])
    return exe


def probe(exe, method, calib, steps, seed, path):
    """Runs the probe; returns a dict with the per-step inputs, the offsets and the host path's Phi / Q."""
    subprocess.run([exe, method, str(calib), str(steps), str(seed), str(path)], check=True)
    with open(path, "rb") as f:
        hdr = f.readline().decode()
        assert hdr.startswith("PROPIMU1"), hdr
        kv = {k: int(v) for k, v in re.findall(r"(\w+)=(-?\d+)", hdr)}
        n, S, nold, cs = kv["n"], kv["steps"], kv["nold"], kv["clone_size"]

        def rd(dt, count):
            return np.frombuffer(f.read(np.dtype(dt).itemsize * count), dtype=dt).copy()
        d = dict(kv)
        d["old_off"], d["old_sz"] = rd("<i4", nold), rd("<i4", nold)
        d["F"] = rd("<f8", S * n * n).reshape(S, n, n)
        d["G"] = rd("<f8", S * n * 12).reshape(S, n, 12)
        d["qc"] = rd("<f8", S * 4).reshape(S, 4)
        d["dnc"] = rd("<f8", cs)
        d["Phi"] = rd("<f8", n * n).reshape(n, n)
        d["Q"] = rd("<f8", n * n).reshape(n, n)
    return d


def _dot(A, B):
    """A @ B as the host computes it: acc = 0; acc += A[i, k] * B[k, j] for ascending k."""
    acc = np.zeros((A.shape[0], B.shape[1]))
    for k in range(A.shape[1]):
        acc = acc + A[:, k, None] * B[None, k, :]
    return acc


def accumulate(F, G, qc):
    """Phi, Q of Propagator::propagate_and_clone (state/Propagator.cpp:83-99, Qd :453-464) in the host's arithmetic."""
    steps, n = F.shape[0], F.shape[1]
    Phi, Q = np.eye(n), np.zeros((n, n))
    for s in range(steps):
        Qt = np.zeros((n, n))
        for k in range(12):
            Qt = Qt + (G[s][:, k, None] * qc[s, k // 3]) * G[s][None, :, k]
        Qd = 0.5 * (Qt + Qt.T)
        Phi = _dot(F[s], Phi)
        T = _dot(_dot(F[s], Q), F[s].T) + Qd
        Q = 0.5 * (T + T.T)
    return Phi, Q


def seeded_prior(N, seed, scale=1e-3):
    """A symmetric positive definite N x N covariance."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((N, N))
    P = scale * (A @ A.T / N + np.eye(N))
    return 0.5 * (P + P.T)
