"""CPU tests of filter-consistency recording in the rpng_sim runner (tools/run_simulation.cpp --consistency, consistency_sample
in include/ovb200_vio.hpp, simrun.load_consistency / average_nees) on the oracle-backed runner (tests/cpp/run_simulation_oracle):
the error convention of P's error state, a numpy restatement of every recorded quantity, unchanged output without the
flag, the Monte-Carlo batch, and the measured NEES of the filter."""
import json
import os
import subprocess

import numpy as np
import pytest

from open_vins_b200 import simrun

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MONO = dict(traj=simrun.TRAJ_FIXTURE, cams=1, clones=11, msckf=50, pts=200, frames=60)  # BASELINE config-1 shape, 60 frames


@pytest.fixture(scope="module")
def runner():
    from oracle import ovo_py
    ovo_py.build()
    return ovo_py.build_sim_runner()


@pytest.fixture(scope="module")
def probe(runner):
    exe = os.path.join(ROOT, "tests", "cpp", "consistency_probe")
    src = os.path.join(ROOT, "tests", "cpp", "consistency_probe.cpp")
    deps = [src] + [os.path.join(ROOT, "include", h) for h in ("ovb200_vio.hpp", "ovb200_math.hpp", "ovb200_sim.hpp", "ovb200_host.hpp")]
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), src, "-L", os.path.join(ROOT, "open_vins_b200"),
                               "-lovb200", "-Wl,-rpath,$ORIGIN/../../open_vins_b200", "-o", exe])
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    return {line.split()[0]: np.array([float(x) for x in line.split()[1:]]) for line in out.strip().splitlines()}


def _read(path):
    with open(path, "rb") as f:
        return f.read()


# numpy restatement of the JPL helpers (ov_core/src/utils/quat_ops.h quat_2_Rot, log_so3)
def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def _quat_2_rot(q):
    v, w = np.asarray(q[:3], float), float(q[3])
    return (2 * w * w - 1) * np.eye(3) - 2 * w * _skew(v) + 2 * np.outer(v, v)


def _log_so3(R):
    tr = np.trace(R)
    mag = 0.5 - (tr - 3.0) / 12.0 if tr - 3.0 >= -1e-7 else np.arccos((tr - 1.0) / 2.0) / (2.0 * np.sin(np.arccos((tr - 1.0) / 2.0)))
    return mag * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])


def _nees(e, S):
    return float(e @ np.linalg.solve(S, e))


def _same(got, want):
    return np.allclose(got, want, rtol=1e-12, atol=0)


def test_error_convention_and_nees(probe):
    """q_true = dq(dtheta) ⊗ q_est (the left JPL update of apply_dx) with q_est far from identity: the recorded error is
    dtheta and the NEES is dtheta' P_thth^-1 dtheta, both to 1e-12 relative; the same for a camera's q_ItoC and for
    q_GYROtoIMU. The error taken in the other frame, -log(R_est' R_true), is not dtheta here and fails the same check."""
    imu = probe["imu"]
    dth, err, other, dp, err_p = imu[0:3], imu[3:6], imu[6:9], imu[9:12], imu[12:15]
    nees_ori, nees_pos = imu[15], imu[16]
    P_th, P_p = imu[17:26].reshape(3, 3), imu[26:35].reshape(3, 3)
    assert not np.allclose(P_th, np.diag(np.diag(P_th)))  # a non-diagonal block
    assert _same(err, dth) and _same(err_p, dp)
    assert nees_ori == pytest.approx(_nees(dth, P_th), rel=1e-12) and nees_pos == pytest.approx(_nees(dp, P_p), rel=1e-12)
    assert not _same(other, dth) and not _same(-other, dth)
    assert np.linalg.norm(other - dth) > 1e-3 * np.linalg.norm(dth)  # not a rounding-level miss
    cam = probe["cam"]
    assert _same(cam[3:6], cam[0:3])
    assert not _same(cam[6:9], cam[0:3]) and not _same(-cam[6:9], cam[0:3])
    gyro = probe["gyro"]
    assert _same(gyro[3:6], gyro[0:3])
    dsig, n = probe["sigma"]
    assert n == 54 and dsig == 0.0


@pytest.fixture(scope="module")
def mono_run(runner, tmp_path_factory):
    d = tmp_path_factory.mktemp("mono")
    est0, est1, cons = str(d / "e0.txt"), str(d / "e1.txt"), str(d / "c.txt")
    r0 = simrun.run(exe=runner, est=est0, **MONO)
    r1 = simrun.run(exe=runner, est=est1, consistency=cons, **MONO)
    return dict(r0=r0, r1=r1, est0=est0, est1=est1, cons=cons)


def test_restatement_in_numpy(mono_run):
    """On a 60-frame config-1 run, every column the test can restate from the estimate file and the recorded 6x6 block agrees
    to 1e-10: the orientation and position errors, their σ, both NEES per frame and the JSON's means."""
    c = simrun.load_consistency(mono_run["cons"])
    t, p_est, q_est, p_gt, q_gt = simrun.load_estimate(mono_run["est1"])
    ids = c["ids"]
    assert ids["n"] == 54 and ids["imu"] == 0 and ids["dw"] == 15 and ids["da"] == 21 and ids["tg"] == 27 and ids["gyro"] == 36
    assert ids["dt"] == 39 and ids["cam0_ext"] == 40 and ids["cam0_intr"] == 46
    assert len(c["t"]) == MONO["frames"] and np.array_equal(c["t"], t)
    e_th = np.array([-_log_so3(_quat_2_rot(qg) @ _quat_2_rot(qe).T) for qe, qg in zip(q_est, q_gt)])
    e_p = p_gt - p_est
    np.testing.assert_allclose(c["err"][:, 0:3], e_th, rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(c["err"][:, 3:6], e_p, rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(c["sigma"][:, 0:6], np.sqrt(np.diagonal(c["cov6"], axis1=1, axis2=2)), rtol=1e-10, atol=0)
    nees_ori = np.array([_nees(e, S[:3, :3]) for e, S in zip(e_th, c["cov6"])])
    nees_pos = np.array([_nees(e, S[3:, 3:]) for e, S in zip(e_p, c["cov6"])])
    np.testing.assert_allclose(c["nees_ori"], nees_ori, rtol=1e-10)
    np.testing.assert_allclose(c["nees_pos"], nees_pos, rtol=1e-10)
    assert mono_run["r1"]["nees_ori"] == pytest.approx(np.mean(nees_ori), rel=1e-10)
    assert mono_run["r1"]["nees_pos"] == pytest.approx(np.mean(nees_pos), rel=1e-10)
    assert np.all(c["sigma"] > 0) and np.all(np.isfinite(c["err"]))


def test_flag_changes_nothing_else(mono_run):
    """With --consistency the estimate file is byte-identical and the JSON is the flag-less JSON plus nees_ori and nees_pos."""
    assert _read(mono_run["est0"]) == _read(mono_run["est1"])
    r0, r1 = mono_run["r0"], mono_run["r1"]
    assert list(r1) == list(r0) + ["nees_ori", "nees_pos"]
    for k in r0:
        if not k.startswith("mean_ms_"):
            assert r1[k] == r0[k], k


def test_batch_files_equal_single_runs(runner, tmp_path):
    """A 3-run batch writes consistency_<seed>.txt byte-identical to the single run of that seed; its NEES statistics are
    numpy's over per_run, and without the flag the batch JSON lacks exactly the new keys."""
    S, kw = 21, dict(MONO, frames=30)
    out = tmp_path / "mc"
    batch = simrun.run(exe=runner, runs=3, jobs=3, out_dir=str(out), consistency=True, seed_meas=S, **kw)
    plain = simrun.run(exe=runner, runs=3, jobs=3, seed_meas=S, **kw)
    assert sorted(os.listdir(out)) == sorted([f"est_{s}.txt" for s in range(S, S + 3)] + [f"consistency_{s}.txt" for s in range(S, S + 3)])
    for entry, pe in zip(batch["per_run"], plain["per_run"]):
        seed = entry["seed"]
        single = str(tmp_path / f"c_{seed}.txt")
        r = simrun.run(exe=runner, consistency=single, seed_meas=seed, **kw)
        assert _read(single) == _read(out / f"consistency_{seed}.txt"), seed
        assert entry["nees_ori"] == pytest.approx(r["nees_ori"], rel=1e-11) and entry["nees_pos"] == pytest.approx(r["nees_pos"], rel=1e-11)
        assert list(entry) == list(pe) + ["nees_ori", "nees_pos"] and all(entry[k] == pe[k] for k in pe)
    no = np.array([r["nees_ori"] for r in batch["per_run"]])
    npos = np.array([r["nees_pos"] for r in batch["per_run"]])
    assert batch["nees_ori_mean"] == pytest.approx(np.mean(no), rel=1e-14) and batch["nees_ori_std"] == pytest.approx(np.std(no), rel=1e-12)
    assert batch["nees_pos_mean"] == pytest.approx(np.mean(npos), rel=1e-14) and batch["nees_pos_std"] == pytest.approx(np.std(npos), rel=1e-12)
    new = ["nees_ori_mean", "nees_ori_std", "nees_pos_mean", "nees_pos_std"]
    assert list(batch) == list(plain) + new
    for k in plain:
        if k not in ("per_run", "wall_s", "runs_per_s", "frames_per_s"):
            assert batch[k] == plain[k], k


def test_measured_nees_of_the_filter(runner, tmp_path):
    """8 seeds x 300 frames at config 1. Measured on the oracle (DESIGN.md §5): mean ANEES 0.905 for orientation and 0.415 for
    position. Both are below 3 because the runs start from the truth: yaw and global position are unobservable, so they
    keep their initial σ (1°, 5 cm) while their error starts at zero. The calibration coordinates, which the updates do
    observe, have RMS errors of 0.38 to 1.28 σ (0.87 over all of them). The bounds are a factor of about 1.5 around these
    values. With θ and p swapped the mean NEES would be 0.005 and 544, so the bounds catch it. A σ column belonging to
    another variable is off by orders of magnitude. An error taken in the other frame changes the orientation mean by only
    17 %, so test_error_convention_and_nees is what catches that."""
    out = tmp_path / "mc"
    batch = simrun.run(exe=runner, runs=8, jobs=8, out_dir=str(out), consistency=True, seed_meas=0, **dict(MONO, frames=300))
    paths = [str(out / f"consistency_{s}.txt") for s in range(8)]
    a = simrun.average_nees(paths)
    assert len(a["t"]) == 300 and a["runs"] == 8
    assert 0.6 <= np.mean(a["anees_ori"]) <= 1.4, np.mean(a["anees_ori"])
    assert 0.25 <= np.mean(a["anees_pos"]) <= 0.7, np.mean(a["anees_pos"])
    assert batch["nees_ori_mean"] == pytest.approx(np.mean(a["anees_ori"]), rel=1e-12)
    assert batch["nees_pos_mean"] == pytest.approx(np.mean(a["anees_pos"]), rel=1e-12)
    cs = [simrun.load_consistency(p) for p in paths]
    z = np.stack([c["err"] for c in cs]) / np.stack([c["sigma"] for c in cs])
    rms = np.sqrt(np.mean(z ** 2, axis=(0, 1)))[15:]  # every calibration coordinate: dw da tg gyro dt cam0_ext cam0_intr
    assert np.all((rms >= 0.25) & (rms <= 2.0)), rms
    assert 0.6 <= np.sqrt(np.mean(rms ** 2)) <= 1.3


@pytest.mark.parametrize("extra", [["--consistency"], ["--consistency", "--est", "x.txt"]])
def test_consistency_without_path_is_refused(runner, tmp_path, extra):
    r = subprocess.run([runner, "--traj", MONO["traj"], "--frames", "5"] + extra, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 2 and "--consistency" in r.stderr and r.stdout == ""
    assert os.listdir(tmp_path) == []


def _write_hand_made(path, nees_ori, nees_pos, n=15):
    F = len(nees_ori)
    rows = np.zeros((F, 3 + 21 + 2 * n))
    rows[:, 0] = np.arange(F) * 0.1
    rows[:, 1], rows[:, 2] = nees_ori, nees_pos
    rows[:, 24 + n:] = 1.0
    with open(path, "w") as f:
        f.write(f"# t nees_ori nees_pos cov6[21] err[n] sigma[n] | ids: imu=0 n={n}\n")
        np.savetxt(f, rows, fmt="%.17g")


def test_average_nees_band_and_fraction(tmp_path):
    """K = 2 runs: 3K = 6 degrees of freedom, chi2.ppf(0.025, 6) = 1.237344, chi2.ppf(0.975, 6) = 14.449375, so the band on
    the average is [0.618672, 7.224688]. Per-frame averages 0.5, 1, 3, 7, 8 (ori: 3 of 5 inside) and 2, 2, 2, 2, 0.1 (pos:
    4 of 5 inside)."""
    a, b = str(tmp_path / "a.txt"), str(tmp_path / "b.txt")
    _write_hand_made(a, [0.4, 1.5, 2.0, 6.0, 9.0], [1.0, 3.0, 2.5, 0.0, 0.1])
    _write_hand_made(b, [0.6, 0.5, 4.0, 8.0, 7.0], [3.0, 1.0, 1.5, 4.0, 0.1])
    r = simrun.average_nees([a, b])
    assert r["runs"] == 2
    np.testing.assert_allclose(r["anees_ori"], [0.5, 1.0, 3.0, 7.0, 8.0], rtol=1e-15)
    np.testing.assert_allclose(r["anees_pos"], [2.0, 2.0, 2.0, 2.0, 0.1], rtol=1e-15)
    # chi-square with 6 degrees of freedom in closed form: P(X <= x) = 1 - exp(-x/2) (1 + x/2 + (x/2)^2 / 2)
    cdf6 = lambda x: 1 - np.exp(-x / 2) * (1 + x / 2 + (x / 2) ** 2 / 2)  # noqa: E731
    lo, hi = r["band"]
    assert cdf6(2 * lo) == pytest.approx(0.025, abs=1e-12) and cdf6(2 * hi) == pytest.approx(0.975, abs=1e-12)
    assert lo == pytest.approx(0.618672, abs=1e-6) and hi == pytest.approx(7.224688, abs=1e-6)
    assert r["inside_ori"] == pytest.approx(3 / 5) and r["inside_pos"] == pytest.approx(4 / 5)
    c = simrun.load_consistency(a)
    assert c["ids"] == {"imu": 0, "n": 15} and c["err"].shape == (5, 15) and np.all(c["sigma"] == 1.0)
