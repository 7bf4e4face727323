"""CPU tests of the perturbed calibration start in rpng_sim runs (Simulator::perturb_parameters in include/ovb200_sim.hpp, the
runner's --perturb): the draws, the untouched measurement streams, the error the filter starts from, the refusals, the
unchanged flag-less output, and online calibration's measured convergence, with the CPU oracle as backend
(tests/cpp/run_simulation_oracle). Reference: ov_msckf/src/sim/Simulator.cpp:209-265."""
import os
import subprocess

import numpy as np
import pytest

from open_vins_b200 import simrun

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAJ = simrun.TRAJ_FIXTURE
MONO = dict(traj=TRAJ, cams=1, clones=11, msckf=50, pts=200)  # BASELINE config-1 shape
BLOCKS = ("dt", "ext_ori", "ext_pos", "intr_fc", "intr_dist", "dw", "da", "tg", "gyro")
# made by tests/golden/make_rpng_sim_perturbed_case.py: seeds 0, update of frame 27
CASE_PERTURBED = os.path.join(ROOT, "tests", "golden", "rpng_sim_perturbed_mono11_f50.case.gz")
K_CAM0 = np.array([458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05])  # rpng_sim cam0


@pytest.fixture(scope="module")
def runner():
    from oracle import ovo_py
    ovo_py.build()
    return ovo_py.build_sim_runner()


@pytest.fixture(scope="module")
def probe(runner):
    exe = os.path.join(ROOT, "tests", "cpp", "perturb_probe")
    src = os.path.join(ROOT, "tests", "cpp", "perturb_probe.cpp")
    deps = [src] + [os.path.join(ROOT, "include", h) for h in ("ovb200_vio.hpp", "ovb200_math.hpp", "ovb200_sim.hpp", "ovb200_host.hpp")]
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), src, "-L", os.path.join(ROOT, "open_vins_b200"),
                               "-lovb200", "-Wl,-rpath,$ORIGIN/../../open_vins_b200", "-o", exe])
    return exe


def _probe(probe, cams, seed, frames=300):
    out = dict(line.split(None, 1) for line in subprocess.run([probe, TRAJ, str(cams), str(seed), str(frames)], check=True, capture_output=True,
                                                              text=True).stdout.splitlines())
    draws, err = (np.array(out[k].split()[1:], dtype=float) for k in ("draws", "init_err"))
    return draws, err, out


def _prior_sigma(cams):
    """σ of each draw, in draw order: the prior σ of its block in P0 (include/ovb200_vio.hpp, VioManager)."""
    cam = [1.0] * 4 + [0.005] * 4 + [0.005] * 3 + [0.015] * 3
    return np.array([0.01] + cam * cams + [0.005, 0.008] * 6 + [0.005] * 3 + [0.005] * 9)


def _draw_ids(ids, cams):
    """The consistency file's column of each draw, in draw order."""
    out = [ids["dt"]]
    for c in range(cams):
        out += list(range(ids[f"cam{c}_intr"], ids[f"cam{c}_intr"] + 8)) + list(range(ids[f"cam{c}_ext"], ids[f"cam{c}_ext"] + 6))
    for j in range(6):
        out += [ids["dw"] + j, ids["da"] + j]
    return out + list(range(ids["gyro"], ids["gyro"] + 3)) + list(range(ids["tg"], ids["tg"] + 9))


def _rotation_mask(cams):
    """True at the draws that are rotation vectors (extrinsic rotation per camera, R_GYROtoIMU)."""
    m = [False] + ([False] * 8 + [True] * 3 + [False] * 3) * cams + [False] * 12 + [True] * 3 + [False] * 9
    return np.array(m)


@pytest.mark.parametrize("cams", [1, 2])
def test_draws_are_deterministic_per_seed_and_differ_across_seeds(probe, cams):
    """39 draws per camera-one rig (1 + 14 per camera + 24), the same for the same seed, others for another seed, of the
    size their prior σ says; the estimator's initial error is the negated draw for additive coordinates and the draw
    itself for rotations (R_est = exp(w) R_true gives -log(R_true R_est') = w)."""
    d0, e0, _ = _probe(probe, cams, 7, frames=1)
    d1, e1, _ = _probe(probe, cams, 7, frames=1)
    d2, _, _ = _probe(probe, cams, 8, frames=1)
    assert len(d0) == 1 + 14 * cams + 24 and np.array_equal(d0, d1) and np.array_equal(e0, e1)
    assert np.all(d0 != d2)
    z = np.concatenate([_probe(probe, cams, s, frames=1)[0] / _prior_sigma(cams) for s in range(20)])
    assert 0.85 <= np.sqrt(np.mean(z ** 2)) <= 1.15 and abs(np.mean(z)) < 0.15
    rot = _rotation_mask(cams)
    assert np.allclose(e0[rot], d0[rot], rtol=0, atol=1e-15)
    assert np.allclose(e0[~rot], -d0[~rot], rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("cams", [1, 2])
def test_measurements_and_map_do_not_depend_on_the_perturbation(probe, cams):
    """The perturbation draws only from its own generator: the map, the IMU readings and every pixel of 300 frames are the
    same with and without it, and the simulator keeps the true parameters while the estimator gets the perturbed copy."""
    _, _, out = _probe(probe, cams, 3)
    assert out["true_params"] == "1"
    n_map, map_same = out["map"].split()
    assert int(n_map) > 1000 and map_same == "1"
    n_imu, n_cam, n_pix, same = (int(x) for x in out["streams"].split())
    assert n_cam == 300 and n_imu > 11000 and n_pix > 50000 * cams and same == 1


@pytest.mark.parametrize("cams", [1, 2])
def test_first_consistency_row_is_the_initial_error(runner, probe, tmp_path, cams):
    """The first consistency row (after frame 0's update) carries the initial calibration error, truth - estimate: over 8
    seeds its RMS distance from the probe's initial error is 0.28 prior σ on the mono rig and 0.42 on the stereo rig
    (one update's correction), while a sign error in either convention would put it near 2."""
    dz, flipped = [], []
    for seed in range(8):
        _, e, _ = _probe(probe, cams, seed, frames=1)
        path = str(tmp_path / f"c{seed}.txt")
        r = simrun.run(exe=runner, frames=1, perturb=True, seed_perturb=seed, consistency=path, **dict(MONO, cams=cams))
        assert r["perturb"] is True and set(r["calib_nerr_first"]) == set(BLOCKS)
        c = simrun.load_consistency(path)
        row = c["err"][0, _draw_ids(c["ids"], cams)]
        dz.append((row - e) / _prior_sigma(cams))
        flipped.append((row + e) / _prior_sigma(cams))
    assert np.sqrt(np.mean(np.square(dz))) <= 0.6
    assert np.sqrt(np.mean(np.square(flipped))) >= 1.5


def test_calib_0_is_refused(runner, tmp_path):
    """--perturb without online calibration would leave the filter an error it cannot estimate: status 2, before anything
    runs, nothing printed or written; --runs batches too."""
    for extra in ([], ["--runs", "2", "--out-dir", "d"]):
        r = subprocess.run([runner, "--traj", TRAJ, "--frames", "5", "--calib", "0", "--perturb"] + extra, capture_output=True, text=True, cwd=tmp_path)
        assert r.returncode == 2 and "--perturb" in r.stderr and r.stdout == ""
        assert os.listdir(tmp_path) == []


def test_without_perturb_the_perturbation_seed_changes_nothing(runner, tmp_path):
    """Without --perturb nothing draws from the perturbation generator: estimate, consistency, timing columns and JSON are
    those of --seed-perturb 0 for any other seed, single runs and batches alike, and carry no "perturb" field."""
    kw = dict(MONO, frames=20)
    outs = []
    for s in (0, 11):
        d = tmp_path / str(s)
        d.mkdir()
        r = simrun.run(exe=runner, seed_perturb=s, est=str(d / "e.txt"), consistency=str(d / "c.txt"), **kw)
        b = simrun.run(exe=runner, seed_perturb=s, runs=2, out_dir=str(d / "mc"), consistency=True, **kw)
        strip = lambda j: {k: v for k, v in j.items() if not k.startswith("mean_ms_") and k not in ("seed_perturb", "wall_s", "runs_per_s", "frames_per_s")}  # noqa: E731
        files = [(d / n).read_bytes() for n in ("e.txt", "c.txt", "mc/est_0.txt", "mc/est_1.txt", "mc/consistency_0.txt", "mc/consistency_1.txt")]
        outs.append((strip(r), strip(b), files))
        assert "perturb" not in r and "perturb" not in b and all("perturb" not in e for e in b["per_run"])
    assert outs[0] == outs[1]


def test_batch_runs_take_consecutive_perturbation_seeds(runner, tmp_path):
    """Run r of a --perturb batch uses seed_perturb + r and seed_meas + r, and writes what the same seeds write alone."""
    kw = dict(MONO, frames=40, perturb=True)
    b = simrun.run(exe=runner, runs=3, out_dir=str(tmp_path / "mc"), seed_perturb=5, seed_meas=2, **kw)
    assert b["perturb"] is True and [e["seed_perturb"] for e in b["per_run"]] == [5, 6, 7] and [e["seed"] for e in b["per_run"]] == [2, 3, 4]
    for r, e in enumerate(b["per_run"]):
        single = str(tmp_path / f"s{r}.txt")
        s = simrun.run(exe=runner, est=single, seed_perturb=5 + r, seed_meas=2 + r, **kw)
        assert open(single, "rb").read() == (tmp_path / "mc" / f"est_{2 + r}.txt").read_bytes()
        for k in ("calib_nerr_first", "calib_nerr_last"):
            assert e[k] == pytest.approx(s[k], rel=1e-10)
    for k in ("calib_nerr_first", "calib_nerr_last"):
        v = np.array([[e[k][blk] for blk in BLOCKS] for e in b["per_run"]])
        assert np.allclose([b[k + "_mean"][blk] for blk in BLOCKS], v.mean(axis=0), rtol=1e-12)
        assert np.allclose([b[k + "_std"][blk] for blk in BLOCKS], v.std(axis=0), rtol=1e-9, atol=1e-15)


def test_captured_perturbed_case_is_away_from_truth_and_start(runner, probe):
    """The golden perturbed update (tests/golden/make_rpng_sim_perturbed_case.py): its camera intrinsics are the estimate of
    the run after frame 26, and fx there is at least 1 σ (its 1 px prior) from both the truth and the perturbed start."""
    frame, feats, _, _ = simrun.load_case(CASE_PERTURBED)
    intr = frame.cam_intr[0]
    _, e, _ = _probe(probe, 1, 0, frames=1)
    start = K_CAM0 - e[1:9]
    moved = np.minimum(np.abs(intr - K_CAM0), np.abs(intr - start))[:4]
    assert moved.max() >= 1.0, moved
    assert len(feats.meas_off) - 1 >= 40


def test_online_calibration_converges(runner, tmp_path):
    """8 perturbation seeds (and measurement seeds) x 300 frames at config 1 on the oracle (DESIGN.md §5). Measured, per block
    over the 8 runs, from the first frame to the last: σ shrinks to 0.005 (dt) to 0.28 (fx fy cx cy) of its value, the RMS
    absolute error to 0.006 to 0.30 of its value, and the final RMS of err/σ is 0.87 to 1.20. Every block converges in
    300 frames. The bars: σ ratio <= 0.5, error ratio <= 0.6, final RMS(err/σ) <= 2."""
    out = tmp_path / "mc"
    batch = simrun.run(exe=runner, runs=8, jobs=8, out_dir=str(out), consistency=True, perturb=True, **dict(MONO, frames=300))
    cs = [simrun.load_consistency(out / f"consistency_{e['seed']}.txt") for e in batch["per_run"]]
    ids = cs[0]["ids"]
    e, i = ids["cam0_ext"], ids["cam0_intr"]
    cols = dict(dt=[ids["dt"]], ext_ori=range(e, e + 3), ext_pos=range(e + 3, e + 6), intr_fc=range(i, i + 4), intr_dist=range(i + 4, i + 8),
                dw=range(ids["dw"], ids["dw"] + 6), da=range(ids["da"], ids["da"] + 6), tg=range(ids["tg"], ids["tg"] + 9),
                gyro=range(ids["gyro"], ids["gyro"] + 3))
    rms = lambda x: float(np.sqrt(np.mean(np.square(x))))  # noqa: E731
    for blk, cc in cols.items():
        cc = list(cc)
        e0, e1 = np.array([c["err"][0, cc] for c in cs]), np.array([c["err"][-1, cc] for c in cs])
        s0, s1 = np.array([c["sigma"][0, cc] for c in cs]), np.array([c["sigma"][-1, cc] for c in cs])
        print(f"\n{blk}: sigma ratio {np.mean(s1 / s0):.3f}, error ratio {rms(e1) / rms(e0):.3f}, final RMS(err/sigma) {rms(e1 / s1):.3f}", end="")
        assert np.mean(s1 / s0) <= 0.5 and np.all(s1 < s0), blk
        assert rms(e1) <= 0.6 * rms(e0), blk
        assert rms(e1 / s1) <= 2.0, blk
        # the JSON's per-run figures are these RMS values, per run
        for c, entry in zip(cs, batch["per_run"]):
            assert entry["calib_nerr_last"][blk] == pytest.approx(rms(c["err"][-1, cc] / c["sigma"][-1, cc]), rel=1e-9)
            assert entry["calib_nerr_first"][blk] == pytest.approx(rms(c["err"][0, cc] / c["sigma"][0, cc]), rel=1e-9)
