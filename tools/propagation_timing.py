#!/usr/bin/env python
"""Propagation on the device (ovb_cov_propagate_imu) against the host accumulation of the parent build, on one GPU.

  python tools/propagation_timing.py --parent DIR [--reps 5] [--parts runner,call,batch,bench] [--out FILE]

DIR is a checkout of the commit before ovb_cov_propagate_imu, built with its __graft_entry__.build() (its
open_vins_b200/ovb_run_simulation accumulates Phi and Qd on the host). This tree is built here. Measurements, one JSON line
each, the card's name, power limit and max SM clock first:
  runner    BASELINE config-1 and config-2 shapes (calib on, rk4): the parent and this runner alternate, --reps times each;
            mean_ms_propagation and mean_ms_total as the runner reports them, and the process wall time, with min / max /
            standard deviation over the reps. The estimate files of both must be identical.
  call      host clock around ovb_cov_propagate_imu (n = 39, one clone; 0, 41 and 400 IMU steps) at the shapes' state sizes;
            each call ends in its stream synchronisation; median after a warm-up.
  batch     Monte-Carlo batches (--runs K --jobs K, config-1 shape) at K = 1 and 16, parent and this runner alternating:
            process wall time, as tools/monte_carlo_timing.py measures it.
  bench     bench.py --dump-outputs for configs 1-5 from both trees: the .npy files must be byte-identical.
Needs a GPU; there is no CPU path."""
import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from open_vins_b200 import build as b  # noqa: E402
from open_vins_b200 import capi, simrun  # noqa: E402

SHAPES = {
    "config1": dict(cams=1, clones=11, msckf=50, pts=200, frames=300),
    "config2": dict(cams=2, clones=20, msckf=400, pts=6000, frames=100),
}


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def spread(xs):
    return {"mean": statistics.fmean(xs), "std": statistics.pstdev(xs), "min": min(xs), "max": max(xs), "n": len(xs)}


def run_timed(exe, **kw):
    t0 = time.perf_counter()
    r = simrun.run(exe=exe, traj=simrun.TRAJ_FIXTURE, calib=1, integration="rk4", **kw)
    return r, time.perf_counter() - t0


def state_dim(shape):
    s = SHAPES[shape]
    return 15 + 24 + 1 + 14 * s["cams"] + 6 * s["clones"]


def time_call(N, steps, reps=200, warmup=20):
    rng = np.random.default_rng(0)
    n = 39
    F = np.eye(n) + 1e-3 * rng.standard_normal((steps, n, n))
    G = 1e-3 * rng.standard_normal((steps, n, 12))
    qc = np.abs(rng.standard_normal((steps, 4))) * 1e-3
    A = rng.standard_normal((N, N))
    P0 = 1e-3 * (A @ A.T / N + np.eye(N))
    eng = capi.Engine(max_state=640, max_feats=16, max_meas=256)
    ts = []
    for i in range(warmup + reps):
        eng.cov_set(P0)
        t0 = time.perf_counter()
        st, _, _ = eng.cov_propagate_imu(F, G, qc, 0, [0, 15, 21, 27, 36], [15, 6, 6, 9, 3], 0, 6, np.ones(6), 39)
        t1 = time.perf_counter()
        assert st == capi.OVB_OK
        if i >= warmup:
            ts.append(1e6 * (t1 - t0))
    eng.close()
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="built checkout of the parent commit")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parts", default="runner,call,batch,bench")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    parts = set(args.parts.split(","))
    parent = os.path.abspath(args.parent)
    exes = {"parent": os.path.join(parent, "open_vins_b200", "ovb_run_simulation"), "new": os.path.join(ROOT, "open_vins_b200", "ovb_run_simulation")}
    b.build()
    b.build_sim_tools()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    emit({"gpu": q.stdout.strip().splitlines()[0]}, args.out)
    tmp = tempfile.mkdtemp(prefix="prop_timing_")
    for shape, kw in SHAPES.items() if "runner" in parts else ():
        rows = {k: {"prop": [], "total": [], "wall": []} for k in exes}
        same = True
        for rep in range(args.reps):
            order = list(exes) if rep % 2 == 0 else list(exes)[::-1]
            for which in order:
                est = os.path.join(tmp, f"{shape}_{which}_{rep}.txt")
                r, wall = run_timed(exes[which], est=est, **kw)
                rows[which]["prop"].append(r["mean_ms_propagation"])
                rows[which]["total"].append(r["mean_ms_total"])
                rows[which]["wall"].append(wall)
            same &= filecmp.cmp(os.path.join(tmp, f"{shape}_parent_{rep}.txt"), os.path.join(tmp, f"{shape}_new_{rep}.txt"), shallow=False)
        for which, v in rows.items():
            emit({"runner": which, "shape": shape, **kw, "mean_ms_propagation": spread(v["prop"]), "mean_ms_total": spread(v["total"]),
                  "process_wall_s": spread(v["wall"])}, args.out)
        emit({"shape": shape, "est_files_identical": same}, args.out)
    # steps = 0: the call without the accumulation (staging, EKFPropagation, clone, synchronisation)
    for shape, steps in (("config1", 0), ("config1", 41), ("config2", 41), ("config1", 400)) if "call" in parts else ():
        ts = time_call(state_dim(shape), steps)
        emit({"call": "ovb_cov_propagate_imu", "n": 39, "steps": steps, "N": state_dim(shape), "median_us": statistics.median(ts), "min_us": min(ts),
              "max_us": max(ts), "calls": len(ts)}, args.out)
    for K in (1, 16) if "batch" in parts else ():
        walls = {k: [] for k in exes}
        for rep in range(2):
            for which in (list(exes) if rep % 2 == 0 else list(exes)[::-1]):
                t0 = time.perf_counter()
                simrun.run(exe=exes[which], traj=simrun.TRAJ_FIXTURE, calib=1, integration="rk4", runs=K, jobs=K,
                           out_dir=os.path.join(tmp, f"mc_{which}_{K}_{rep}"), **SHAPES["config1"])
                walls[which].append(time.perf_counter() - t0)
        for which, w in walls.items():
            emit({"batch": which, "K": K, "shape": "config1", "process_wall_s": spread(w), "runs_per_s": K / statistics.fmean(w)}, args.out)
    for cfg in (1, 2, 3, 4, 5) if "bench" in parts else ():
        dirs = {}
        for which, tree in (("parent", parent), ("new", ROOT)):
            d = os.path.join(tmp, f"bench_{which}_{cfg}")
            subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--config", str(cfg), "--steps", "3", "--warmup", "1", "--no-cpu-baseline",
                            "--dump-outputs", d], cwd=tree, check=True, capture_output=True, text=True)
            dirs[which] = d
        names = sorted(os.listdir(dirs["parent"]))
        same = names == sorted(os.listdir(dirs["new"])) and all(
            filecmp.cmp(os.path.join(dirs["parent"], f), os.path.join(dirs["new"], f), shallow=False) for f in names)
        emit({"bench_config": cfg, "outputs": names, "byte_identical": same}, args.out)


if __name__ == "__main__":
    main()
