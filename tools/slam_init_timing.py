#!/usr/bin/env python
"""Wall-clock time of ovb_slam_delayed_init (UpdaterSLAM::delayed_init in one call) per call and per processed landmark.

Three cases: config-4 sizes (4 cameras, 31 clone poses, full calibration) with 25 and with 100 new tracks of up to 124
measurements, and 8 cameras x 48 clone poses with 25 tracks. Every call starts from ovb_cov_set of the same prior and a
fresh copy of the frame; the callback applies dx to the frame as a caller's Type::update would. The call ends in a stream
synchronisation, so the host clock around it is the call's time. Prints one JSON line per case.

  python tools/slam_init_timing.py [--calls 20] [--warmup 3] [--tag new]

It imports the package next to it, so an A/B against an earlier commit runs a copy of this file from a built checkout of
that commit, alternating with this one in the same session. Needs a GPU; there is no CPU path."""
import argparse
import copy
import json
import os
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tag", default="new")
    a = ap.parse_args()
    for name, kw in CASES.items():
        case = sim.make_update_case(seed=4, full_track_frac=0.5, calib_ext=True, calib_intr=True, outlier_frac=0.05,
                                    degenerate_frac=0.05, **kw)
        opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
        N0 = case.P.shape[0]
        eng = capi.Engine(max_state=N0 + 3 * kw["n_feats"] + 8, max_feats=128, max_meas=128 * 400)
        times, n_init = [], 0
        for it in range(a.warmup + a.calls):
            fr = copy.deepcopy(case.frame)
            eng.cov_set(case.P)
            cnt = [0]

            def on_init(f, lm_off, dx_new, dx):
                cnt[0] += 1
                _apply_dx(fr, dx)
            t0 = time.perf_counter()
            out, _ = eng.slam_delayed_init(fr, case.feats, opts, on_init)
            t1 = time.perf_counter()
            if it >= a.warmup:
                times.append(t1 - t0)
                n_init = cnt[0]
        processed = int((out.status == capi.FEAT_OK).sum() + (out.status == capi.FEAT_CHI2).sum())
        t = np.array(times) * 1e3
        rec = dict(tool="slam_init_timing", tag=a.tag, case=name, N0=N0, tracks=kw["n_feats"],
                   max_meas=int(np.diff(case.feats.meas_off).max()), initialised=n_init, processed=processed,
                   ms_median=float(np.median(t)), ms_min=float(t.min()), ms_max=float(t.max()),
                   ms_per_landmark=float(np.median(t)) / max(processed, 1))
        if hasattr(eng.lib, "ovb_last_init_counters"):
            rec["counters"] = eng.last_init_counters()
        print(json.dumps(rec), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
