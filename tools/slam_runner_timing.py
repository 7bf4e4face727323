#!/usr/bin/env python
"""Per-frame stage times of the rpng_sim runner with SLAM landmarks on the CUDA engine, on one GPU.

  python tools/slam_runner_timing.py [--frames 300] [--out FILE]

Runs open_vins_b200/ovb_run_simulation at config 1 (mono, 11 clones, 50 MSCKF features, 200 points, calibration on, 300
frames) and at a stereo window (2 cameras, 20 clones, 120 MSCKF features, 300 points, 80 frames), each with --slam 0, 25 and
50 (GLOBAL_3D, max_slam_in_update 25), and reads the timing CSV the runner writes (the columns of VioManager's timing file).
Prints one JSON line per run: the mean host wall time per frame of propagation, the MSCKF update (with the feature selection
and marginalize_slam before it), the SLAM updates, the delayed initialisation, the end-of-frame marginalization and the
total, each over the frames after the first 20 (milliseconds), plus the run's ATE and live landmarks; the card's name, power
limit and max SM clock first. Every stage ends in its device synchronisation. Needs a GPU; there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from open_vins_b200 import build as b  # noqa: E402
from open_vins_b200 import simrun  # noqa: E402

SHAPES = {"config1": dict(cams=1, clones=11, msckf=50, pts=200, calib=1), "stereo20": dict(cams=2, clones=20, msckf=120, pts=300, calib=1, frames=80)}
WARM = 20  # frames left out of the means: first launches, the window filling up


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300, help="frames of the config-1 runs")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], check=True, capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    emit({"card": card}, a.out)
    exe = b.build_sim_tools()
    with tempfile.TemporaryDirectory() as d:
        for shape, kw in SHAPES.items():
            kw = dict(kw)
            kw.setdefault("frames", a.frames)
            for m in (0, 25, 50):
                csv = os.path.join(d, f"{shape}_{m}.csv")
                s = simrun.run(exe=exe, timing=csv, slam=m, **kw)
                t = np.loadtxt(csv, delimiter=",", ndmin=2)[WARM:]
                cols = ["propagation", "msckf_update"] + (["slam_update", "slam_delayed"] if m else []) + ["marginalization", "total"]
                ms = {c: float(1e3 * t[:, 2 + i].mean()) for i, c in enumerate(cols)}
                if not m:
                    ms["slam_update"] = ms["slam_delayed"] = 0.0
                emit({"shape": shape, "slam": m, "frames_timed": int(len(t)), "ms_per_frame": ms, "ate_pos_m": s["ate_pos_m"],
                      "state_dim_end": s["state_dim"], "mean_slam_live": s.get("mean_slam_live", 0.0)}, a.out)


if __name__ == "__main__":
    main()
