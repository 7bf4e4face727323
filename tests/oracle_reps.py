"""TEST INFRASTRUCTURE: ctypes loader for tests/cpp/ovo_slam_reps.cpp, the CPU oracle's SLAM update with one representation
per landmark and the SINGLE branch of delayed_init, built on the oracle's own routines (oracle/ovo_core.hpp).

The library is compiled with oracle/Makefile's flags into the temporary directory (keyed by the sources' content), so the
repository tree is never written."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from open_vins_b200 import capi
from open_vins_b200.capi import FeatOut, _ptr, c_double_p, c_int_p, ovb_stats
from oracle import ovo_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "ovo_slam_reps.cpp")
DEPS = [SRC] + [os.path.join(ROOT, "oracle", f) for f in ("ovo_core.hpp", "ovo_math.hpp")] + [os.path.join(ROOT, "include", "ovb200.h")]
# oracle/Makefile's CXXFLAGS: the rounding sequence of the oracle itself
CXXFLAGS = ["-std=c++17", "-O3", "-fno-math-errno", "-funroll-loops", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in DEPS:
            h.update(open(p, "rb").read())
        h.update(" ".join(CXXFLAGS).encode())
        so = os.path.join(tempfile.gettempdir(), f"ovo_slam_reps_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            fd, tmp = tempfile.mkstemp(suffix=".so")
            os.close(fd)
            subprocess.check_call([os.environ.get("CXX", "g++")] + CXXFLAGS + ["-shared", "-o", tmp, SRC])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def slam_update(frame, feats, landmarks, opts, P, feat_rep=None):
    """ovo_py.slam_update with feat_rep: one ovb_feat_rep per landmark, or None for opts.feat_rep.
    Returns dict(status, P, out, dx, stats, order_off, order_sz, H_big, res_big, Rdiag_big)."""
    P = np.array(P, dtype=np.float64, order="C", copy=True)
    N = P.shape[0]
    out = FeatOut(feats.n_feats)
    dx = np.zeros(N)
    stats = ovb_stats()
    tab = ovo_py.chi2_table()
    order_off = np.zeros(capi.OVB_MAX_VARS, dtype=np.int32)  # the dump keeps the first OVB_MAX_VARS variables (as ovo_py's)
    order_sz = np.zeros(capi.OVB_MAX_VARS, dtype=np.int32)
    n_order = C.c_int32(0)
    cap = int(2 * feats.n_meas) + 1
    H_big, res_big, Rd_big = np.zeros((cap, N)), np.zeros(cap), np.zeros(cap)
    reps = None if feat_rep is None else np.ascontiguousarray(feat_rep, dtype=np.int32)
    fs, bs, ls, os_ = frame.struct(), feats.struct(), landmarks.struct(), out.struct()
    st = lib().ovo_slam_update_reps(C.byref(fs), C.byref(bs), C.byref(ls), C.byref(opts), _ptr(tab, c_double_p), _ptr(P, c_double_p), C.c_int(N),
                                    C.byref(os_), _ptr(dx, c_double_p), C.byref(stats), _ptr(order_off, c_int_p), _ptr(order_sz, c_int_p),
                                    C.byref(n_order), _ptr(H_big, c_double_p), _ptr(res_big, c_double_p), _ptr(Rd_big, c_double_p), C.c_int(cap),
                                    _ptr(reps, c_int_p))
    no = min(n_order.value, capi.OVB_MAX_VARS)
    cols, rows = stats.cols_stacked, stats.rows_stacked
    return dict(status=st, P=P, out=out, dx=dx, stats=stats, order_off=order_off[:no].copy(), order_sz=order_sz[:no].copy(),
                H_big=H_big.reshape(-1)[:rows * cols].reshape(rows, cols).copy(), res_big=res_big[:rows].copy(),
                Rdiag_big=Rd_big[:rows].copy())


def slam_single_init_system(Hf, Hx, res):
    """The ANCHORED_INVERSE_DEPTH_SINGLE branch of UpdaterSLAM::delayed_init: [Hx | Hf[:,2] | res] with the bearing columns
    Hf[:,0:2] nullspace-projected out (Givens). Returns (H_R (rows-2 x n), h_L (rows-2 x 1), res (rows-2))."""
    Hf = np.ascontiguousarray(Hf, dtype=np.float64)
    Hx = np.ascontiguousarray(Hx, dtype=np.float64)
    res = np.ascontiguousarray(res, dtype=np.float64)
    rows, n = Hx.shape
    if rows < 3:
        raise ValueError(f"ovo_slam_single_init_system: {rows} rows")
    H_R, h_L, r = np.zeros((rows - 2, n)), np.zeros((rows - 2, 1)), np.zeros(rows - 2)
    lib().ovo_slam_single_init_system(_ptr(Hf, c_double_p), _ptr(Hx, c_double_p), _ptr(res, c_double_p), C.c_int(rows), C.c_int(n),
                                      _ptr(H_R, c_double_p), _ptr(h_L, c_double_p), _ptr(r, c_double_p))
    return H_R, h_L, r
