"""SLAM landmarks in the rpng_sim closed loop, on the CPU: the oracle-backed runner (tests/cpp/run_simulation_oracle) with
--slam, and the runner's restatement of ov_type::Landmark (tests/cpp/landmark_probe).

- Without --slam, or with --slam 0, the runner writes what it always wrote.
- Malformed SLAM flags exit with status 2.
- SlamLandmark: get_xyz(set_from_xyz(p)) = p for all six representations, update() moves the point the way the update's H_f
  columns say (finite differences through the oracle's UpdaterSLAM::update), and re-anchoring keeps ovb_slam_anchor_change's
  new_value.
- Per-frame invariants of SLAM runs, read from --slam-log, and the filter's consistency over 8 seeds."""
import os
import subprocess

import numpy as np
import pytest

from open_vins_b200 import capi, sim, simrun

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1)  # BASELINE config 1: mono, 11 clones, 50 features
STEREO = dict(cams=2, clones=20, msckf=120, pts=300, frames=80, calib=1)
REPS = list(range(6))
NAMES = ["GLOBAL_3D", "GLOBAL_FULL_INVERSE_DEPTH", "ANCHORED_3D", "ANCHORED_FULL_INVERSE_DEPTH", "ANCHORED_MSCKF_INVERSE_DEPTH",
         "ANCHORED_INVERSE_DEPTH_SINGLE"]
SINGLE = capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE


def oracle_runner():
    """tests/cpp/run_simulation_oracle, rebuilt when tests/cpp/oracle_slam_backend.hpp (which oracle/ovo_py.py's staleness
    check does not list) is newer than it."""
    from oracle import ovo_py
    exe = os.path.join(ROOT, "tests", "cpp", "run_simulation_oracle")
    hdr = os.path.join(ROOT, "tests", "cpp", "oracle_slam_backend.hpp")
    return ovo_py.build_sim_runner(force=os.path.exists(exe) and os.path.getmtime(hdr) > os.path.getmtime(exe))


@pytest.fixture(scope="module")
def runner():
    return oracle_runner()


@pytest.fixture(scope="module")
def probe():
    capi_lib = os.path.join(ROOT, "open_vins_b200")
    exe = os.path.join(ROOT, "tests", "cpp", "landmark_probe")
    src = os.path.join(ROOT, "tests", "cpp", "landmark_probe.cpp")
    hdr = os.path.join(ROOT, "include", "ovb200_vio.hpp")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-L", capi_lib,
                               "-lovb200", "-Wl,-rpath,$ORIGIN/../../open_vins_b200", "-o", exe])
    return exe


def _probe(exe, lines):
    out = subprocess.run([exe], input="\n".join(lines) + "\n", check=True, capture_output=True, text=True).stdout
    return [np.array([float(x) for x in ln.split()]) for ln in out.strip().splitlines()]


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _drop_times(summary):
    return {k: v for k, v in summary.items() if "ms" not in k and k not in ("wall_s", "runs_per_s", "frames_per_s")}


# ---------------------------------------------------------------------------------------------------------------- output identity
def test_slam_zero_writes_what_no_flag_writes(runner, tmp_path):
    """--slam 0 (with the other SLAM flags) and no flag: the same JSON line but for wall-clock fields, and byte-identical
    estimate, consistency and capture files; the timing CSV keeps the MSCKF-only columns."""
    outs = []
    for tag, extra in (("none", {}), ("zero", dict(slam=0, slam_in_update=7, feat_rep_slam="ANCHORED_3D"))):
        d = tmp_path / tag
        d.mkdir()
        s = simrun.run(exe=runner, **CONFIG1, frames=60, est=str(d / "est.txt"), timing=str(d / "t.csv"), consistency=str(d / "c.txt"),
                       capture=(30, str(d / "cap")), **extra)
        outs.append((s, d))
    (a, da), (b, db) = outs
    assert _drop_times(a) == _drop_times(b) and "max_slam" not in b
    for f in ("est.txt", "c.txt", "cap.case"):
        assert _read(da / f) == _read(db / f), f
    ta, tb = [np.loadtxt(d / "t.csv", delimiter=",") for d in (da, db)]
    assert ta.shape == tb.shape and ta.shape[1] == 6 and np.array_equal(ta[:, 0], tb[:, 0])
    assert open(db / "t.csv").readline() == "# timestamp (sec),tracking,propagation,msckf update,marginalization,total\n"


@pytest.mark.parametrize("bad", [["--slam", "x"], ["--slam", "-1"], ["--slam", "2.5"], ["--slam"], ["--slam-in-update", "0"],
                                 ["--slam-in-update", "ten"], ["--slam-delay", "-1"], ["--slam-delay", "nan"], ["--feat-rep-slam", "GLOBAL"],
                                 ["--feat-rep-slam", "anchored_3d"], ["--slam", "5", "--runs", "2", "--slam-log", "x.txt"]])
def test_malformed_slam_flags_exit_2(runner, bad):
    r = subprocess.run([runner, "--traj", simrun.TRAJ_FIXTURE, "--frames", "2"] + bad, capture_output=True, text=True)
    assert r.returncode == 2, (bad, r.stdout, r.stderr)
    assert r.stdout == ""


def test_slam_timing_columns_and_json(runner, tmp_path):
    s = simrun.run(exe=runner, **CONFIG1, frames=40, slam=10, slam_delay=0.5, feat_rep_slam="ANCHORED_3D", timing=str(tmp_path / "t.csv"))
    assert open(tmp_path / "t.csv").readline() == "# timestamp (sec),tracking,propagation,msckf update,slam update,slam delayed,marginalization,total\n"
    assert np.loadtxt(tmp_path / "t.csv", delimiter=",").shape == (s["frames"], 8)
    assert s["max_slam"] == 10 and s["feat_rep_slam"] == "ANCHORED_3D" and s["dt_slam_delay"] == 0.5
    assert len(s["slam_status_hist"]) == len(s["init_status_hist"]) == 9
    assert 0 < s["max_slam_live"] <= 10 and s["slam_initialized"] > 0
    assert s["slam_initialized"] - s["slam_marginalized"] >= 0


# ---------------------------------------------------------------------------------------------------------------- Landmark
def _points(rng, n):
    return np.column_stack([rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), rng.uniform(0.5, 9, n)])


@pytest.mark.parametrize("rep", REPS, ids=NAMES)
def test_landmark_set_get_round_trip(probe, rep):
    """get_xyz(set_from_xyz(p)) = p to 1e-13 for the value and for the FEJ value. The FEJ value of the two MSCKF-style
    inverse-depth representations is not read back: Landmark::get_xyz returns their value's point whatever getfej says."""
    rng = np.random.default_rng(100 + rep)
    P, Q = _points(rng, 200), _points(rng, 200)
    res = _probe(probe, [f"rt {rep} " + " ".join(repr(float(x)) for x in np.r_[p, q]) for p, q in zip(P, Q)])
    fej_read = rep not in (capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, SINGLE)
    for p, q, r in zip(P, Q, res):
        assert np.abs(r[:3] - p).max() <= 1e-13 * np.linalg.norm(p)
        assert np.abs(r[3:6] - (q if fej_read else p)).max() <= 1e-13 * np.linalg.norm(p)
    same = _probe(probe, [f"rt {rep} " + " ".join(repr(float(x)) for x in np.r_[p, p]) for p in P])
    for p, r in zip(P, same):
        assert np.abs(r[3:6] - p).max() <= 1e-13 * np.linalg.norm(p)


@pytest.mark.parametrize("rep", REPS, ids=NAMES)
def test_landmark_update_follows_the_update_jacobian(probe, oracle, rep):
    """Landmark::update(δ) moves the point the way the SLAM update's landmark columns are defined: feeding the oracle's
    UpdaterSLAM::update the point after update(±h e_k) differences the residuals into -H_f's column k (FEJ off)."""
    case = sim.make_slam_case(n_landmarks=4, n_clones=6, n_cams=2, seed=71 + rep, rep=rep, two_classes=False)
    lm = case.landmarks
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, feat_rep=rep, do_fej=0, chi2_multipler=1e12)
    mk = lambda v: capi.LandmarkArrays(lm.lm_off, v, v, lm.anchor_cam, lm.anchor_clone)  # noqa: E731
    r0 = oracle.slam_update(case.frame, case.feats, mk(lm.value), opts, case.P)
    assert (r0["out"].status == 0).all()
    cols = np.concatenate([np.arange(o, o + s) for o, s in zip(r0["order_off"], r0["order_sz"])])
    w = 1 if rep == SINGLE else 3
    h = 1e-4 if rep in (capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_FULL_INVERSE_DEPTH) else 1e-2
    if rep in (capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, SINGLE):
        h = 1e-3
    row = 0
    for f in range(4):
        m = 2 * int(case.feats.meas_off[f + 1] - case.feats.meas_off[f]) - (2 if rep == SINGLE else 0)
        for k in range(w):
            d = np.zeros(3)
            d[k] = h
            lines = [f"upd {rep} " + " ".join(repr(float(x)) for x in np.r_[lm.value[f], s * d]) for s in (1, -1)]
            (xp, xm) = [r[:3] for r in _probe(probe, lines)]
            vp, vm = lm.value.copy(), lm.value.copy()
            vp[f], vm[f] = xp, xm
            rp = oracle.slam_update(case.frame, case.feats, mk(vp), opts, case.P)["res_big"][row:row + m]
            rm = oracle.slam_update(case.frame, case.feats, mk(vm), opts, case.P)["res_big"][row:row + m]
            fd = -(rp - rm) / (2 * h)
            j = int(np.flatnonzero(cols == case.lm_off[f] + k)[0])
            an = r0["H_big"][row:row + m, j]
            assert np.abs(fd - an).max() <= 5e-3 * max(np.abs(an).max(), 1.0), (f, k, np.abs(fd - an).max(), np.abs(an).max())
        row += m


@pytest.mark.parametrize("rep", [2, 3, 4, 5], ids=NAMES[2:])
def test_reanchored_landmark_keeps_the_anchor_change_value(probe, rep):
    """The runner re-anchors a landmark with set_from_xyz(new_value) / set_from_xyz(new_value_fej); its get_xyz then returns
    ovb_slam_anchor_change's new_value (and, where get_xyz reads it, new_value_fej) to 1e-13."""
    case = sim.make_slam_case(n_landmarks=6, n_clones=7, n_cams=2, seed=90 + rep, rep=rep)
    fr, lm = case.frame, case.landmarks
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=0, feat_rep=rep, do_fej=1)
    lines, want = [], []
    for f in range(6):
        nv, nvf = capi.slam_anchor_change(fr, opts, lm.lm_off[f], lm.value[f], lm.value_fej[f], int(lm.anchor_cam[f]), int(lm.anchor_clone[f]),
                                          f % 2, 6)[:2]
        lines.append(f"rt {rep} " + " ".join(repr(float(x)) for x in np.r_[nv, nvf]))
        want.append((nv, nvf if rep in (2, 3) else nv))
    for (nv, nvf), r in zip(want, _probe(probe, lines)):
        assert np.abs(r[:3] - nv).max() <= 1e-13 * np.linalg.norm(nv)
        assert np.abs(r[3:6] - nvf).max() <= 1e-13 * np.linalg.norm(nvf)


# ---------------------------------------------------------------------------------------------------------------- per-frame invariants
def _load_log(path):
    frames = []
    for ln in open(path):
        tag, *rest = ln.split()
        if tag == "F":
            frames.append(dict(t=float(rest[0]), since=float(rest[1]), N=int(rest[2]), clones=int(rest[3]), n=int(rest[4]), L=[]))
        elif tag == "L":
            frames[-1]["L"].append(tuple(int(x) for x in rest))
        elif tag == "X":
            frames[-1]["X"] = {int(a): int(b) for a, b in (x.split(":") for x in rest)}
        else:
            frames[-1][tag] = [int(x) for x in rest]
    return frames


@pytest.mark.parametrize("case,opts", [
    ("mono_global3d", dict(CONFIG1, frames=300, slam=25)),
    ("stereo_msckf_inverse_depth", dict(STEREO, slam=50, feat_rep_slam="ANCHORED_MSCKF_INVERSE_DEPTH")),
    ("mono_full_inverse_depth", dict(CONFIG1, frames=200, slam=25, feat_rep_slam="ANCHORED_FULL_INVERSE_DEPTH")),
    ("mono_single", dict(CONFIG1, frames=200, slam=25, feat_rep_slam="ANCHORED_INVERSE_DEPTH_SINGLE")),
    ("mono_unbounded", dict(CONFIG1, frames=200, slam=100, slam_in_update=100)),
])
def test_slam_frame_invariants(runner, tmp_path, case, opts):
    log = tmp_path / "slam.txt"
    s = simrun.run(exe=runner, slam_log=str(log), **opts)
    frames = _load_log(log)
    assert len(frames) == s["frames"] > 0
    M = opts["slam"]
    base = 15 + 25 + 14 * opts["cams"]
    delay = 1.0  # dt_slam_delay
    reinit = 0
    for fr in frames:
        widths = sum(w for _, _, w, _ in fr["L"])
        assert fr["N"] == base + 6 * fr["clones"] + widths, fr["t"]
        # the ids tile [0, N): the base state, 6-wide clones, and the landmarks' blocks do not overlap
        blocks = sorted((i, w) for _, i, w, _ in fr["L"])
        assert all(a[0] + a[1] <= b[0] for a, b in zip(blocks, blocks[1:])) and all(base <= i and i + w <= fr["N"] for i, w in blocks)
        assert fr["n"] == len(fr["L"]) <= M
        assert all(a != 0 for _, _, _, a in fr["L"]), "an anchored landmark's anchor clone left the window"
        # MSCKF and SLAM batches are disjoint. A single-depth landmark's track of one measurement is skipped by UpdaterSLAM::update
        # without being deleted (UpdaterSLAM.cpp:278-290), so it can reach the MSCKF lists of a later frame while the landmark
        # still takes it: the reference does the same
        assert not set(fr["M"]) & set(fr["D"]), "MSCKF and delayed-init batches overlap"
        if opts.get("feat_rep_slam") != "ANCHORED_INVERSE_DEPTH_SINGLE":
            assert not set(fr["M"]) & set(fr["U"]), "MSCKF and SLAM update batches overlap"
        if fr["since"] < delay:
            assert not fr["P"], "promotion before dt_slam_delay"
        # a marginalised landmark is not updated as an old one in the frame that removed it
        for fid, fails in fr["X"].items():
            assert fid not in fr["U"]
            reinit += fails > 1 and fid in fr["D"]
    assert min(fr["since"] for fr in frames) < delay and any(fr["P"] for fr in frames) and sum(len(fr["I"]) for fr in frames) == s["slam_initialized"]
    assert sum(len(fr["X"]) for fr in frames) == s["slam_marginalized"]
    print(f"\n{case}: ATE {s['ate_pos_m']:.6f} m, live landmarks mean {s['mean_slam_live']:.1f} max {s['max_slam_live']}, "
          f"initialised {s['slam_initialized']}, marginalised {s['slam_marginalized']}, anchor changes {s['anchor_changes']}, "
          f"handed to delayed_init after two failures {reinit}")


def test_failed_landmark_goes_to_delayed_init_in_the_same_frame(runner, tmp_path):
    """A landmark that failed its update twice leaves the state before the updates (marginalize_slam, where the reference
    calls it) and, when its track goes on in that frame, delayed_init takes the track as a new feature: it is in the frame's
    delayed list, never in its update list. (Its track holds only the measurements since its last update, usually fewer than
    delayed_init's two, so few come back.)"""
    log = tmp_path / "slam.txt"
    s = simrun.run(exe=runner, slam_log=str(log), **CONFIG1, frames=300, slam=100, slam_in_update=100)
    seen = 0
    for fr in _load_log(log):
        for fid, fails in fr["X"].items():
            if fails > 1 and fid in fr["D"]:
                seen += 1
                assert fid not in fr["U"] and fid not in fr["M"]
    assert seen > 0 and s["slam_status_hist"][8] > 0


# ---------------------------------------------------------------------------------------------------------------- consistency
# Oracle runner, config 1, 8 measurement seeds, 300 frames: mean over the runs of each run's mean NEES (3 DOF each).
# Measured: SLAM (--slam 25) ori 1.020, pos 0.198; MSCKF only ori 0.905, pos 0.415 (both conservative, below 3).
ANEES_BAND = {"ori": (0.6, 1.6), "pos": (0.1, 0.35)}


def test_slam_consistency_eight_seeds(runner, tmp_path):
    slam = simrun.run(exe=runner, **CONFIG1, frames=300, slam=25, runs=8, consistency=True, out_dir=str(tmp_path / "slam"))
    msckf = simrun.run(exe=runner, **CONFIG1, frames=300, runs=8, consistency=True, out_dir=str(tmp_path / "msckf"))
    print(f"\nATE over 8 seeds: SLAM {slam['ate_pos_m_mean']:.5f} ± {slam['ate_pos_m_std']:.5f} m, MSCKF only "
          f"{msckf['ate_pos_m_mean']:.5f} ± {msckf['ate_pos_m_std']:.5f} m; ANEES ori {slam['nees_ori_mean']:.3f} "
          f"(MSCKF {msckf['nees_ori_mean']:.3f}), pos {slam['nees_pos_mean']:.3f} (MSCKF {msckf['nees_pos_mean']:.3f})")
    for k in ("ori", "pos"):
        lo, hi = ANEES_BAND[k]
        assert lo <= slam[f"nees_{k}_mean"] <= hi, (k, slam[f"nees_{k}_mean"])
    assert all(r["max_slam_live"] <= 25 and r["slam_initialized"] > 0 for r in slam["per_run"])
    # every per_run entry of a batch is the single run of its seed
    one = simrun.run(exe=runner, **CONFIG1, frames=300, slam=25, seed_meas=3)
    r3 = slam["per_run"][3]
    assert r3["seed"] == 3 and r3["ate_pos_m"] == pytest.approx(one["ate_pos_m"], rel=1e-11)
    assert r3["slam_status_hist"] == one["slam_status_hist"] and r3["init_status_hist"] == one["init_status_hist"]
