#!/usr/bin/env python
"""Estimator options in the rpng_sim closed loop on the engine (INTEGRATION.md §8, "Estimator options"), config 1 (mono,
11 clones, 50 features, calibration on), 300 frames.

FEJ study: one --runs K --consistency batch (measurement seeds 0 .. K-1) with --use-fej 1 and one with --use-fej 0. Per arm:
the runner's mean and population standard deviation over the runs of the per-run mean orientation / position NEES, the ATE,
and from the consistency files the average NEES per frame (simrun.average_nees): its mean over the frames and the fraction
of frames inside the two-sided 95 % band of a consistent filter.

Representations: per --feat-rep-msckf, --reps single runs (seed 0) with --timing, the order of the six rotating from round
to round: the ATE and the mean per-frame "msckf update" time of the timing CSV (the host clock around the update call,
which ends in a device synchronisation).

  python tools/sim_options_study.py [--runs 16] [--reps 3] [--out FILE]

Prints one JSON line per measurement, the card's name, power limit and max SM clock first and last. Needs a GPU; there is
no CPU path."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from monte_carlo_timing import gpu_info  # noqa: E402
from open_vins_b200 import build as b  # noqa: E402
from open_vins_b200 import simrun  # noqa: E402

CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1, frames=300)
REPS = ("GLOBAL_3D", "GLOBAL_FULL_INVERSE_DEPTH", "ANCHORED_3D", "ANCHORED_FULL_INVERSE_DEPTH", "ANCHORED_MSCKF_INVERSE_DEPTH",
        "ANCHORED_INVERSE_DEPTH_SINGLE")


def fej_arm(exe, use_fej, runs, tmp):
    d = os.path.join(tmp, f"fej{use_fej}")
    r = simrun.run(exe=exe, runs=runs, jobs=runs, out_dir=d, consistency=True, use_fej=use_fej, **CONFIG1)
    a = simrun.average_nees([os.path.join(d, f"consistency_{e['seed']}.txt") for e in r["per_run"]])
    return dict(tool="sim_options_study", study="fej", use_fej=use_fej, runs=runs, nees_ori_mean=r["nees_ori_mean"], nees_ori_std=r["nees_ori_std"],
                nees_pos_mean=r["nees_pos_mean"], nees_pos_std=r["nees_pos_std"], anees_ori_mean=float(np.mean(a["anees_ori"])),
                anees_pos_mean=float(np.mean(a["anees_pos"])), band=a["band"], inside_ori=a["inside_ori"], inside_pos=a["inside_pos"],
                ate_pos_m_mean=r["ate_pos_m_mean"], ate_pos_m_std=r["ate_pos_m_std"], ate_ori_deg_mean=r["ate_ori_deg_mean"])


def rep_run(exe, rep, rnd, tmp):
    csv = os.path.join(tmp, f"timing_{rep}_{rnd}.csv")
    r = simrun.run(exe=exe, timing=csv, feat_rep_msckf=rep, **CONFIG1)
    with open(csv) as f:
        cols = f.readline().lstrip("# ").strip().split(",")
    t = np.loadtxt(csv, delimiter=",", comments="#", ndmin=2)
    ms = 1e3 * t[:, cols.index("msckf update")]
    return dict(tool="sim_options_study", study="feat_rep_msckf", feat_rep_msckf=rep, round=rnd, ate_pos_m=r["ate_pos_m"], ate_ori_deg=r["ate_ori_deg"],
                status_hist=r["status_hist"], mean_rows=r["mean_rows"], mean_ms_msckf_update=float(ms.mean()), median_ms_msckf_update=float(np.median(ms)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    exe = b.build_sim_tools()
    recs = [dict(tool="sim_options_study", gpu=gpu_info())]
    print(json.dumps(recs[-1]), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        simrun.run(exe=exe, **dict(CONFIG1, frames=20))  # warm-up: driver, page cache
        for use_fej in (1, 0):
            recs.append(fej_arm(exe, use_fej, a.runs, tmp))
            print(json.dumps(recs[-1]), flush=True)
        for rnd in range(a.reps):
            for k in range(len(REPS)):
                recs.append(rep_run(exe, REPS[(k + rnd) % len(REPS)], rnd, tmp))
                print(json.dumps(recs[-1]), flush=True)
    recs.append(dict(tool="sim_options_study", gpu_after=gpu_info()))
    print(json.dumps(recs[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in recs))


if __name__ == "__main__":
    main()
