#!/usr/bin/env python
"""The end-of-frame window shift as one ovb_marginalize_window against the call sequence it replaces, on one GPU.

  python tools/window_timing.py [--calls 200] [--warmup 20] [--out FILE]

Host clock around (a) the existing sequence: ovb_slam_anchor_change + ovb_cov_propagate (Q = 0) per re-anchored landmark, then
ovb_cov_marginalize per lost landmark and the oldest clone, highest offset first; (b) one ovb_marginalize_window. Both end in
their stream synchronisation; the two alternate call by call in one process, each on its own context re-loaded with the same
P before every call (the upload is outside the timed window). Shapes: config 4 (4 cameras, 31 clones, 100 landmarks,
N = 582) with k_anchor in {4, 25} and k_lost in {3, 10}, and the 8-camera, 48-clone window (N = 665: a quarter of the
landmarks are 1 wide) with 25 and 10.
One JSON line per shape (median, min, max, and the 10th / 90th percentiles in microseconds), the card's name, power limit
and max SM clock first. Needs a GPU; there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from open_vins_b200 import build as b  # noqa: E402
from open_vins_b200 import capi  # noqa: E402
from tests.test_gpu_window import _setup  # noqa: E402
from tests.test_window_cpu import sequence  # noqa: E402

SHAPES = [("config4", 31, 4, 75, ka, kl) for ka in (4, 25) for kl in (3, 10)] + [("cams8_clones48", 48, 8, 0, 25, 10)]


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def stats(ts):
    ts = np.asarray(ts)
    return {"median_us": float(np.median(ts)), "p10_us": float(np.percentile(ts, 10)), "p90_us": float(np.percentile(ts, 90)), "min_us": float(ts.min()),
            "max_us": float(ts.max()), "calls": int(ts.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    b.build()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    emit({"gpu": q.stdout.strip().splitlines()[0]}, args.out)
    for name, n_clones, n_cams, pad, ka, kl in SHAPES:
        case, anchors, marg = _setup(n_clones, n_cams, 100, 4 if n_cams == 4 else 8, pad, ka, kl)
        opts = capi.default_opts(do_calib_camera_pose=1)
        mo, ms = [o for o, _ in marg], [s for _, s in marg]
        seq, win = capi.Engine(max_state=800, max_feats=16, max_meas=256), capi.Engine(max_state=800, max_feats=16, max_meas=256)

        def propagate(o, Phi, Q, off, sz):
            assert seq.cov_propagate(o, Phi, Q, off, sz) == capi.OVB_OK

        t_seq, t_win = [], []
        for i in range(args.warmup + args.calls):
            seq.cov_set(case.P)
            win.cov_set(case.P)
            t0 = time.perf_counter()
            sequence(case, anchors, marg, 1, 1, capi.slam_anchor_change, propagate, seq.cov_marginalize)
            t1 = time.perf_counter()
            assert win.marginalize_window(case.frame, opts, mo, ms, anchors) == capi.OVB_OK
            t2 = time.perf_counter()
            if i >= args.warmup:
                t_seq.append(1e6 * (t1 - t0))
                t_win.append(1e6 * (t2 - t1))
        same = seq.cov_dim() == win.cov_dim()
        seq.close()
        win.close()
        emit({"shape": name, "N": int(case.P.shape[0]), "k_anchor": ka, "k_lost": kl, "same_N": same, "sequence": stats(t_seq),
              "marginalize_window": stats(t_win)}, args.out)


if __name__ == "__main__":
    main()
