"""CPU tests of the rpng_sim runner's Monte-Carlo mode (tools/run_simulation.cpp: --seed-init / --seed-perturb / --seed-meas,
--runs K --jobs J --out-dir DIR) on the oracle-backed runner (tests/cpp/run_simulation_oracle): seeds reach the simulator,
a run is the same bits alone or inside a concurrent batch, and without --runs the runner prints and writes what it did
before the batch mode existed."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from open_vins_b200 import simrun

MONO = dict(traj=simrun.TRAJ_FIXTURE, cams=1, clones=11, msckf=50, pts=200, frames=60)  # BASELINE config-1 shape, 60 frames


@pytest.fixture(scope="module")
def runner():
    from oracle import ovo_py
    ovo_py.build()
    return ovo_py.build_sim_runner()


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def test_same_seed_is_bit_identical(runner, tmp_path):
    a, b = str(tmp_path / "a.txt"), str(tmp_path / "b.txt")
    ra = simrun.run(exe=runner, est=a, seed_meas=3, seed_init=1, seed_perturb=2, **MONO)
    rb = simrun.run(exe=runner, est=b, seed_meas=3, seed_init=1, seed_perturb=2, **MONO)
    assert _read(a) == _read(b)
    assert ra["status_hist"] == rb["status_hist"] and ra["ate_pos_m"] == rb["ate_pos_m"]


def test_measurement_seed_changes_measurements_and_estimate(runner, tmp_path):
    """Simulator::get_next_cam draws the pixel noise from gen_meas_cams (seeded by sim_seed_measurements): another seed gives
    other pixels for the same map points and another estimate."""
    cases, ests, sums = [], [], []
    for seed in (3, 4):
        est, cap = str(tmp_path / f"e{seed}.txt"), str(tmp_path / f"c{seed}")
        sums.append(simrun.run(exe=runner, est=est, capture=(20, cap), seed_meas=seed, **MONO))
        cases.append(simrun.load_case(cap + ".case"))
        ests.append(_read(est))
    assert sums[0]["map_points"] == sums[1]["map_points"]  # the map comes from sim_seed_state_init only
    uv0, uv1 = cases[0][1].uv, cases[1][1].uv
    n = min(len(uv0), len(uv1))
    assert n > 10 and not np.array_equal(uv0[:n], uv1[:n])
    assert ests[0] != ests[1]
    assert sums[0]["ate_pos_m"] != sums[1]["ate_pos_m"]


def test_runs_equal_separate_single_runs(runner, tmp_path):
    """--runs 3 --jobs 3 with measurement seed S runs seeds S, S+1, S+2 concurrently; each estimate file is byte-identical to
    the single run of that seed, and the summary's statistics are numpy's over the per-run ATEs."""
    S = 11
    out = tmp_path / "mc"
    batch = simrun.run(exe=runner, runs=3, jobs=3, out_dir=str(out), timing=True, seed_meas=S, **MONO)
    assert batch["runs"] == 3 and batch["jobs"] == 3 and batch["seed_meas"] == S
    assert [r["seed"] for r in batch["per_run"]] == [S, S + 1, S + 2]
    assert sorted(os.listdir(out)) == sorted([f"est_{s}.txt" for s in (S, S + 1, S + 2)] + [f"timing_{s}.csv" for s in (S, S + 1, S + 2)])
    for entry in batch["per_run"]:
        seed = entry["seed"]
        single = str(tmp_path / f"single_{seed}.txt")
        r = simrun.run(exe=runner, est=single, seed_meas=seed, **MONO)
        assert _read(single) == _read(out / f"est_{seed}.txt"), seed
        assert entry["frames"] == r["frames"] == MONO["frames"]
        assert entry["status_hist"] == r["status_hist"]
        assert entry["ate_pos_m"] == pytest.approx(r["ate_pos_m"], rel=1e-11)  # the single run prints 12 digits
        assert entry["ate_ori_deg"] == pytest.approx(r["ate_ori_deg"], rel=1e-11)
        rows = open(out / f"timing_{seed}.csv").read().strip().splitlines()
        assert rows[0].startswith("# timestamp (sec),tracking,propagation") and len(rows) == MONO["frames"] + 1
    p = np.array([r["ate_pos_m"] for r in batch["per_run"]])
    o = np.array([r["ate_ori_deg"] for r in batch["per_run"]])
    assert batch["ate_pos_m_mean"] == pytest.approx(np.mean(p), rel=1e-14) and batch["ate_pos_m_std"] == pytest.approx(np.std(p), rel=1e-12)
    assert batch["ate_ori_deg_mean"] == pytest.approx(np.mean(o), rel=1e-14) and batch["ate_ori_deg_std"] == pytest.approx(np.std(o), rel=1e-12)
    assert batch["frames_total"] == 3 * MONO["frames"] and batch["wall_s"] > 0
    assert batch["runs_per_s"] == pytest.approx(3 / batch["wall_s"], rel=1e-4)


def test_more_runs_than_jobs(runner, tmp_path):
    """Two threads share five runs through the counter; every seed is run once and the files equal a one-thread batch."""
    a, b = tmp_path / "a", tmp_path / "b"
    kw = dict(MONO, frames=20)
    ra = simrun.run(exe=runner, runs=5, jobs=2, out_dir=str(a), seed_meas=100, **kw)
    rb = simrun.run(exe=runner, runs=5, jobs=1, out_dir=str(b), seed_meas=100, **kw)
    assert [r["seed"] for r in ra["per_run"]] == list(range(100, 105)) and ra["jobs"] == 2
    for s in range(100, 105):
        assert _read(a / f"est_{s}.txt") == _read(b / f"est_{s}.txt")
    assert ra["per_run"] == rb["per_run"]


# What the runner printed and wrote before it had seeds and a batch mode, for
#   run_simulation_oracle --traj tests/golden/traj_tum_corridor1_head.bin --cams 1 --clones 11 --msckf 50 --pts 200 --frames 60 --est E
# (the mean_ms_* host times are left out: they are wall-clock measurements).
PREVIOUS_STDOUT = ('{"backend": "oracle", "frames": 60, "cams": 1, "max_clones": 11, "max_msckf_in_update": 50, "num_pts": 200, "calib": 1, '
                   '"state_dim": 120, "ate_pos_m": 0.0342014810462, "ate_ori_deg": 0.357636958111, "mean_feats_in": 24.13, "mean_feats_used": 17.97, '
                   '"mean_rows": 289.1, "mean_ms_propagation": 0, "mean_ms_msckf_update": 0, "mean_ms_total": 0, "map_points": 2026, '
                   '"status_hist": [1078, 0, 215, 0, 0, 0, 5, 0, 51]}')
PREVIOUS_EST_SHA256 = "d25f549fe225383ffa565cd7acaa356c9df651833a752b2a9c60f3c6f3d6bcc9"


def test_without_runs_output_is_unchanged(runner, tmp_path):
    est = str(tmp_path / "e.txt")
    cmd = [runner, "--traj", MONO["traj"], "--cams", "1", "--clones", "11", "--msckf", "50", "--pts", "200", "--frames", "60", "--est", est]
    out = subprocess.run(cmd, check=True, capture_output=True, text=True).stdout
    assert out.endswith("}\n") and out.count("\n") == 1
    got, want = json.loads(out), json.loads(PREVIOUS_STDOUT)
    assert list(got) == list(want)
    for k in want:
        if not k.startswith("mean_ms_"):
            assert got[k] == want[k], k
    assert hashlib.sha256(_read(est)).hexdigest() == PREVIOUS_EST_SHA256
    # the seed flags at their defaults change nothing
    est0 = str(tmp_path / "e0.txt")
    subprocess.run(cmd[:-1] + [est0, "--seed-init", "0", "--seed-perturb", "0", "--seed-meas", "0"], check=True, capture_output=True)
    assert _read(est0) == _read(est)


@pytest.mark.parametrize("extra", [["--runs", "2", "--est", "x.txt"], ["--runs", "2", "--capture", "3", "x"], ["--jobs", "2"], ["--out-dir", "d"],
                                   ["--runs", "-1"]])
def test_inconsistent_batch_options_are_refused(runner, tmp_path, extra):
    r = subprocess.run([runner, "--traj", MONO["traj"], "--frames", "5"] + extra, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 2 and "--runs" in r.stderr and r.stdout == ""
    assert os.listdir(tmp_path) == []
