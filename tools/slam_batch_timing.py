#!/usr/bin/env python
"""Device time of ovb_slam_update per call (stats.ms_total: CUDA events from the first upload to the last download) for the
two max_slam_in_update settings of SURVEY.md config 4 and for the full 8-camera, 48-clone window. Every call starts from
ovb_cov_set of the same prior; median over --calls calls after --warmup. Prints the GPU and its power limit first.
Four calls of 25 and one call of 100 are different filters in the reference (the mean moves between batches): they are
the two settings of max_slam_in_update, not two ways of computing one update."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from open_vins_b200 import capi, sim  # noqa: E402
import make_fullsize as mf  # noqa: E402


def _subset(case, a, b):
    return mf.slam_subset(case, a, b)


def _time(eng, case, batches, opts, calls, warmup, reps=None):
    per = []
    for it in range(warmup + calls):
        eng.cov_set(case.P)
        tot = 0.0
        for feats, lms in batches:
            st, out, dx, stats = eng.slam_update(case.frame, feats, lms, opts, feat_rep=reps)
            assert st == 0, st
            tot += stats.ms_total
        if it >= warmup:
            per.append(tot)
    return float(np.median(per)), stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown")
    calib = dict(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, col_order=capi.COLS_CANONICAL)
    c4 = sim.make_slam_case(**mf.SLAM4)
    w25 = sim.make_slam_case(n_landmarks=25, n_clones=48, n_cams=8, seed=30, rep=capi.REP_GLOBAL_3D)
    w100 = sim.make_slam_case(n_landmarks=100, n_clones=48, n_cams=8, seed=7, rep=capi.REP_GLOBAL_3D)
    # every other landmark in the 1-wide ANCHORED_INVERSE_DEPTH_SINGLE, the others in config 4's representation
    mixed = [capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE if i % 2 else mf.SLAM4["rep"] for i in range(mf.SLAM4["n_landmarks"])]
    c4m = sim.make_slam_case(**{**mf.SLAM4, "rep": mixed})
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D, **calib)
    cases = [
        ("config 4, 100 landmarks as 4 calls of 25 (ms per 4 calls)", c4, [_subset(c4, a, b) for a, b in mf.slam_batches(c4)]),
        ("config 4, 100 landmarks in 1 call", c4, [(c4.feats, c4.landmarks)]),
        ("8 cams x 48 clones, calibrated, 25 landmarks in 1 call", w25, [(w25.feats, w25.landmarks)]),
        ("8 cams x 48 clones, calibrated, 100 landmarks in 1 call", w100, [(w100.feats, w100.landmarks)]),
        ("config 4, 100 landmarks in 1 call, half SINGLE", c4m, [(c4m.feats, c4m.landmarks)], mixed),
    ]
    eng = capi.Engine(max_state=1024, max_feats=256, max_meas=16384)
    eng.set_slam_unbounded()
    for name, case, batches, *reps in cases:
        ms, stats = _time(eng, case, batches, opts, a.calls, a.warmup, reps[0] if reps else None)
        print(f"{name:58s} N={case.P.shape[0]:4d} rows={stats.rows_stacked:5d} cols={stats.cols_stacked:4d}  median {1e3 * ms:8.1f} us")
    eng.close()


if __name__ == "__main__":
    main()
