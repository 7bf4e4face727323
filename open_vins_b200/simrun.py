"""Python side of the rpng_sim runner (tools/run_simulation.cpp over include/ovb200_vio.hpp): launch the product executable
open_vins_b200/ovb_run_simulation (CUDA engine) and read what it writes — the JSON summary, the estimate/ground-truth
trajectory file, the timing CSV (columns of ov_msckf/src/core/VioManager.cpp:117-121), the consistency file (INTEGRATION.md
§8) and captured update cases."""
from __future__ import annotations

import ctypes as C
import json
import os
import re
import subprocess

import numpy as np

from . import capi

HERE = os.path.dirname(os.path.abspath(__file__))
ENGINE_EXE = os.path.join(HERE, "ovb_run_simulation")
TRAJ_FIXTURE = os.path.join(os.path.dirname(HERE), "tests", "golden", "traj_tum_corridor1_head.bin")
# update cases captured from rpng_sim runs (tests/golden/make_rpng_sim_cases.py): BASELINE.json configs 1 and 2
CASE_CONFIG1 = os.path.join(os.path.dirname(HERE), "tests", "golden", "rpng_sim_mono11_f50.case.gz")
CASE_CONFIG2 = os.path.join(os.path.dirname(HERE), "tests", "golden", "rpng_sim_stereo20_f400.case.gz")


def run(exe=None, traj=None, cams=2, clones=11, msckf=10, pts=250, frames=0, calib=1, est=None, timing=None, capture=None, integration="rk4",
        compress="cholqr2", seed_init=0, seed_perturb=0, seed_meas=0, runs=None, jobs=None, out_dir=None, consistency=None, cam_model=None,
        slam=None, slam_in_update=None, slam_delay=None, feat_rep_slam=None, slam_log=None, perturb=False, feat_rep_msckf=None, use_fej=None,
        fi_triangulate_1d=None, fi_refine_features=None, up_msckf_sigma_px=None, up_msckf_chi2_multipler=None, up_slam_sigma_px=None,
        up_slam_chi2_multipler=None, calib_cam_extrinsics=None, calib_cam_intrinsics=None, calib_cam_timeoffset=None, calib_imu_intrinsics=None,
        calib_imu_g_sensitivity=None, timeout=1800):
    """Runs the simulation; returns the parsed JSON summary. capture = (frame_index, path_prefix) dumps that update's inputs.
    seed_init / seed_perturb / seed_meas: the simulator's random seeds (rpng_sim's sim_seed_state_init, sim_seed_preturb,
    sim_seed_measurements). runs = K: a Monte-Carlo batch in one process, run r with measurement seed seed_meas + r, on
    `jobs` host threads (default min(K, hardware threads)); out_dir receives est_<seed>.txt per run and, when `timing` is
    truthy, timing_<seed>.csv. The batch summary lists every run under "per_run" with the mean and population standard
    deviation of both ATEs. consistency = PATH (single run) or True (batch; out_dir receives consistency_<seed>.txt): record
    the per-frame errors, σ and NEES (load_consistency); the summary gains the mean nees_ori / nees_pos, per run in a batch
    with their mean and population standard deviation over the runs. cam_model = "radtan" or "equi" for every camera, or a
    sequence with one model per camera (a mixed rig): equidistant cameras take the TUM-VI cam0 intrinsics on a 512 x 512
    image (INTEGRATION.md §8), and the summary gains "cam_model". None runs the rpng_sim radtan cameras. slam = M: at most M SLAM
    landmarks (--slam), with slam_in_update / slam_delay / feat_rep_slam (a representation name, e.g. "ANCHORED_3D") passed as
    --slam-in-update / --slam-delay / --feat-rep-slam when given; for M > 0 the summary gains the SLAM fields (INTEGRATION.md
    §8). slam_log = PATH writes the per-frame landmark log (--slam-log, single runs). perturb = True starts the filter from a
    calibration perturbed with seed_perturb (seed_perturb + r for run r of a batch; --perturb, needs calib=1); the summary
    gains "perturb" and the RMS of err/σ per calibration block at the first and last frame ("calib_nerr_first",
    "calib_nerr_last"), with their mean and population standard deviation over a batch. The estimator options (INTEGRATION.md
    §8, "Estimator options") are passed as the runner flag of the same name when given (feat_rep_msckf = a representation
    name; use_fej and the fi_* and calib_* options 0 or 1; the up_* options positive numbers); the summary then lists those
    that differ from the defaults under "estimator"."""
    cmd = [exe or ENGINE_EXE, "--traj", traj or TRAJ_FIXTURE, "--cams", str(cams), "--clones", str(clones), "--msckf", str(msckf), "--pts", str(pts),
           "--frames", str(frames), "--calib", str(int(calib)), "--integration", integration, "--compress", compress,
           "--seed-init", str(seed_init), "--seed-perturb", str(seed_perturb), "--seed-meas", str(seed_meas)]
    if est:
        cmd += ["--est", est]
    if timing:
        cmd += ["--timing"] if runs else ["--timing", timing]
    if consistency:
        cmd += ["--consistency"] if runs or consistency is True else ["--consistency", str(consistency)]
    if cam_model is not None:
        cmd += ["--cam-model", cam_model if isinstance(cam_model, str) else ",".join(cam_model)]
    for flag, v in (("--slam", slam), ("--slam-in-update", slam_in_update), ("--slam-delay", slam_delay), ("--feat-rep-slam", feat_rep_slam),
                    ("--slam-log", slam_log)):
        if v is not None:
            cmd += [flag, str(v)]
    if perturb:
        cmd += ["--perturb"]
    estimator = dict(feat_rep_msckf=feat_rep_msckf, use_fej=use_fej, fi_triangulate_1d=fi_triangulate_1d, fi_refine_features=fi_refine_features,
                     up_msckf_sigma_px=up_msckf_sigma_px, up_msckf_chi2_multipler=up_msckf_chi2_multipler, up_slam_sigma_px=up_slam_sigma_px,
                     up_slam_chi2_multipler=up_slam_chi2_multipler, calib_cam_extrinsics=calib_cam_extrinsics, calib_cam_intrinsics=calib_cam_intrinsics,
                     calib_cam_timeoffset=calib_cam_timeoffset, calib_imu_intrinsics=calib_imu_intrinsics, calib_imu_g_sensitivity=calib_imu_g_sensitivity)
    for name, v in estimator.items():
        if v is not None:
            cmd += ["--" + name.replace("_", "-"), str(int(v)) if isinstance(v, bool) else str(v)]
    if capture:
        cmd += ["--capture", str(capture[0]), capture[1]]
    if runs:
        cmd += ["--runs", str(runs)]
        if jobs:
            cmd += ["--jobs", str(jobs)]
        if out_dir:
            cmd += ["--out-dir", str(out_dir)]
    out = subprocess.run(cmd, check=True, capture_output=True, text=True, timeout=timeout)
    return json.loads(out.stdout.strip().splitlines()[-1])


def load_estimate(path):
    """rows: t, est p(3) q(4), gt p(3) q(4)"""
    a = np.loadtxt(path, comments="#")
    return a[:, 0], a[:, 1:4], a[:, 4:8], a[:, 8:11], a[:, 11:15]


def ate_rmse(p_est, p_gt):
    """ov_eval/src/calc/ResultTrajectory.cpp:82-109 (position part, alignment 'none'): sqrt(mean |p_gt - p_est|^2)"""
    return float(np.sqrt(np.mean(np.sum((p_gt - p_est) ** 2, axis=1))))


def load_consistency(path):
    """The runner's consistency file: returns a dict with the columns t, nees_ori, nees_pos (F), cov6 (F x 6 x 6, the [theta p]
    block of the IMU, symmetric), err and sigma (F x n), and "ids": the variable ids of the header (imu, dw, ..., cam0_ext,
    ..., n = the base state's size)."""
    with open(path) as f:
        hdr = f.readline()
    assert hdr.startswith("#"), hdr
    ids = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", hdr.split("ids:", 1)[1])}
    n = ids["n"]
    a = np.loadtxt(path, comments="#", ndmin=2)
    assert a.shape[1] == 3 + 21 + 2 * n, (a.shape, n)
    cov6 = np.zeros((len(a), 6, 6))
    iu = np.triu_indices(6)
    cov6[:, iu[0], iu[1]] = a[:, 3:24]
    cov6[:, iu[1], iu[0]] = a[:, 3:24]
    return dict(t=a[:, 0], nees_ori=a[:, 1], nees_pos=a[:, 2], cov6=cov6, err=a[:, 24:24 + n], sigma=a[:, 24 + n:], ids=ids)


def average_nees(paths):
    """Average NEES over K runs of the same trajectory (one consistency file each, same frames): per frame, the mean over
    the runs of the orientation and of the position NEES (3 DOF each). For a consistent filter K * ANEES is chi-square with
    3K degrees of freedom, so the two-sided 95 % band is chi2.ppf([0.025, 0.975], 3K) / K; "inside_ori" / "inside_pos" are
    the fractions of frames whose ANEES lies in it."""
    from scipy.stats import chi2
    runs = [load_consistency(p) for p in paths]
    K = len(runs)
    assert K > 0 and all(np.array_equal(r["t"], runs[0]["t"]) for r in runs), "the runs must cover the same frames"
    ori = np.mean([r["nees_ori"] for r in runs], axis=0)
    pos = np.mean([r["nees_pos"] for r in runs], axis=0)
    lo, hi = chi2.ppf([0.025, 0.975], 3 * K) / K
    inside = lambda x: float(np.mean((x >= lo) & (x <= hi)))  # noqa: E731
    return dict(t=runs[0]["t"], anees_ori=ori, anees_pos=pos, band=(float(lo), float(hi)), inside_ori=inside(ori), inside_pos=inside(pos), runs=K)


def load_case(path):
    """One captured MSCKF update (written by the runner's --capture): returns (FrameArrays, FeatArrays, ovb_opts, P)."""
    import gzip
    with (gzip.open(path, "rb") if str(path).endswith(".gz") else open(path, "rb")) as f:
        hdr = f.readline().decode()
        assert hdr.startswith("OVBCASE1"), hdr
        kv = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)", hdr)}
        C_, K, F, M, NK, N = kv["n_clones"], kv["n_cams"], kv["n_feats"], kv["n_meas"], kv["n_keys"], kv["N"]

        def rd(dt, n):
            return np.frombuffer(f.read(np.dtype(dt).itemsize * n), dtype=dt).copy()
        clone_R, clone_p, clone_Rf, clone_pf = rd("<f8", 9 * C_), rd("<f8", 3 * C_), rd("<f8", 9 * C_), rd("<f8", 3 * C_)
        clone_off = rd("<i4", C_)
        cam_R, cam_p, cam_intr = rd("<f8", 9 * K), rd("<f8", 3 * K), rd("<f8", 8 * K)
        cam_model, cam_ext, cam_intr_off = rd("<i4", K), rd("<i4", K), rd("<i4", K)
        meas_off, cam, clone = rd("<i4", F + 1), rd("u1", M), rd("<u2", M)
        uv, uvn = rd("<f4", 2 * M), rd("<f4", 2 * M)
        keys_off, keys = rd("<i4", F + 1), rd("u1", NK)
        opts = capi.ovb_opts.from_buffer_copy(f.read(kv["opts"]))
        P = rd("<f8", N * N).reshape(N, N)
    frame = capi.FrameArrays(clone_R.reshape(C_, 9), clone_p.reshape(C_, 3), clone_Rf.reshape(C_, 9), clone_pf.reshape(C_, 3), clone_off,
                             cam_R.reshape(K, 9), cam_p.reshape(K, 3), cam_intr.reshape(K, 8), cam_model, cam_ext, cam_intr_off)
    feats = capi.FeatArrays(meas_off, cam, clone, uv.reshape(M, 2), uvn.reshape(M, 2), keys_off, keys)
    return frame, feats, opts, P
