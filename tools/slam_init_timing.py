#!/usr/bin/env python
"""Wall-clock time of the delayed initialisation (UpdaterSLAM::delayed_init in one call) per call and per processed landmark,
through ovb_slam_delayed_init (a host callback moves the frame after every accepted landmark: one stream synchronisation
and one frame upload per landmark) and through ovb_slam_delayed_init_batch (the engine moves its frame itself: two
synchronisations per call).

Three cases: config-4 sizes (4 cameras, 31 clone poses, full calibration) with 25 and with 100 new tracks of up to 124
measurements, and 8 cameras x 48 clone poses with 25 tracks. Every call starts from ovb_cov_set of the same prior and a
fresh copy of the frame; the callback applies dx to the frame as a caller's Type::update would. The two paths alternate call
by call in one process (--paths callback,batch; an earlier commit's copy of this file runs the callback path alone). Each
call ends in a stream synchronisation, so the host clock around it is the call's time. Prints the card's name and power
limit, then one JSON line per case and path.

  python tools/slam_init_timing.py [--calls 20] [--warmup 3] [--tag new] [--paths callback,batch]

It imports the package next to it, so an A/B against an earlier commit runs a copy of this file from a built checkout of
that commit, alternating with this one in the same session. Needs a GPU; there is no CPU path."""
import argparse
import copy
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from open_vins_b200 import capi, sim  # noqa: E402

CASES = {
    "c4_25": dict(n_feats=25, n_clones=31, n_cams=4),
    "c4_100": dict(n_feats=100, n_clones=31, n_cams=4),
    "8x48_25": dict(n_feats=25, n_clones=48, n_cams=8),
}


def _apply_dx(fr, dx):
    for c, o in enumerate(fr.clone_off):
        fr.clone_R[c] = (sim.exp_so3(-dx[o:o + 3]) @ fr.clone_R[c].reshape(3, 3)).reshape(fr.clone_R[c].shape)
        fr.clone_p[c] += dx[o + 3:o + 6]
    for k in range(fr.n_cams):
        o = fr.cam_ext_off[k]
        if o >= 0:
            fr.cam_R[k] = (sim.exp_so3(-dx[o:o + 3]) @ fr.cam_R[k].reshape(3, 3)).reshape(fr.cam_R[k].shape)
            fr.cam_p[k] += dx[o + 3:o + 6]
        o = fr.cam_intr_off[k]
        if o >= 0:
            fr.cam_intr[k] += dx[o:o + 8]


def _quat(R):
    """JPL quaternion of a rotation (quat_ops.h rot_2_quat's trace branch; the window's rotations are far from 180 degrees)."""
    R = np.asarray(R).reshape(9)
    w = math.sqrt(1.0 + R[0] + R[4] + R[8]) / 2
    q = np.array([(R[5] - R[7]) / (4 * w), (R[6] - R[2]) / (4 * w), (R[1] - R[3]) / (4 * w), w])
    return q / np.linalg.norm(q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tag", default="new")
    ap.add_argument("--paths", default="callback,batch")
    a = ap.parse_args()
    paths = a.paths.split(",")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True, capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    for name, kw in CASES.items():
        case = sim.make_update_case(seed=4, full_track_frac=0.5, calib_ext=True, calib_intr=True, outlier_frac=0.05,
                                    degenerate_frac=0.05, **kw)
        opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
        N0 = case.P.shape[0]
        eng = capi.Engine(max_state=N0 + 3 * kw["n_feats"] + 8, max_feats=128, max_meas=128 * 400)
        cq = np.array([_quat(R) for R in case.frame.clone_R])
        kq = np.array([_quat(R) for R in case.frame.cam_R])
        times = {p: [] for p in paths}
        n_init, counters = {}, {}
        for it in range(a.warmup + a.calls):
            for p in (paths if it % 2 == 0 else paths[::-1]):
                fr = copy.deepcopy(case.frame)
                eng.cov_set(case.P)
                cnt = [0]

                def on_init(f, lm_off, dx_new, dx):
                    cnt[0] += 1
                    _apply_dx(fr, dx)
                t0 = time.perf_counter()
                if p == "callback":
                    out, lm_off = eng.slam_delayed_init(fr, case.feats, opts, on_init)
                else:
                    out, lm_off, _, _ = eng.slam_delayed_init_batch(fr, cq, kq, case.feats, opts)
                t1 = time.perf_counter()
                if it >= a.warmup:
                    times[p].append(t1 - t0)
                    n_init[p] = int((lm_off >= 0).sum())
                    counters[p] = eng.last_init_counters()
        processed = int((out.status == capi.FEAT_OK).sum() + (out.status == capi.FEAT_CHI2).sum())
        for p in paths:
            t = np.array(times[p]) * 1e3
            rec = dict(tool="slam_init_timing", tag=a.tag, path=p, case=name, N0=N0, tracks=kw["n_feats"],
                       max_meas=int(np.diff(case.feats.meas_off).max()), initialised=n_init[p], processed=processed,
                       ms_median=float(np.median(t)), ms_min=float(t.min()), ms_max=float(t.max()),
                       ms_per_landmark=float(np.median(t)) / max(processed, 1), counters=counters[p])
            print(json.dumps(rec), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
