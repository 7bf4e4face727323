"""CPU tests of the rpng_sim runner's estimator options (tools/run_simulation.cpp; INTEGRATION.md §8, "Estimator options"):
the refusals, a closed loop with every option on the oracle-backed runner (tests/cpp/run_simulation_oracle) and the state
layout it implies, the "estimator" JSON object, captures that keep their options, and outputs without the flags that are
byte for byte those of the runner before the flags existed."""
import hashlib
import math
import os
import re
import subprocess

import numpy as np
import pytest

from open_vins_b200 import capi, simrun

TRAJ = simrun.TRAJ_FIXTURE
CONFIG1 = dict(traj=TRAJ, cams=1, clones=11, msckf=50, pts=200, calib=1)  # BASELINE config 1: mono, 11 clones, 50 features
REPS = ("GLOBAL_3D", "GLOBAL_FULL_INVERSE_DEPTH", "ANCHORED_3D", "ANCHORED_FULL_INVERSE_DEPTH", "ANCHORED_MSCKF_INVERSE_DEPTH",
        "ANCHORED_INVERSE_DEPTH_SINGLE")
CALIB_BLOCKS = ("calib_cam_extrinsics", "calib_cam_intrinsics", "calib_cam_timeoffset", "calib_imu_intrinsics", "calib_imu_g_sensitivity")

# one closed-loop case per option: simrun.run keyword arguments, and the "estimator" object the run must report
OPTIONS = {f"feat_rep_msckf_{r}": (dict(feat_rep_msckf=r), {} if r == "GLOBAL_3D" else {"feat_rep_msckf": r}) for r in REPS}
OPTIONS.update({
    "use_fej_0": (dict(use_fej=0), {"use_fej": 0}),
    "fi_triangulate_1d_1": (dict(fi_triangulate_1d=1), {"fi_triangulate_1d": 1}),
    "fi_refine_features_0": (dict(fi_refine_features=0), {"fi_refine_features": 0}),
    "up_msckf_sigma_chi2": (dict(up_msckf_sigma_px=1.5, up_msckf_chi2_multipler=2), {"up_msckf_sigma_px": 1.5, "up_msckf_chi2_multipler": 2}),
})
OPTIONS.update({f"{b}_0": (dict(**{b: 0}), {b: 0, **({"calib_imu_g_sensitivity": 0} if b == "calib_imu_intrinsics" else {})}) for b in CALIB_BLOCKS})


@pytest.fixture(scope="module")
def runner():
    from oracle import ovo_py
    ovo_py.build()
    return ovo_py.build_sim_runner()


def layout(cams, calib=1, **flags):
    """The consistency header's ids for the calibration blocks the flags leave on (State.cpp:28-131: IMU 15 | dw 6 | da 6 |
    tg 9 | R_GYROtoIMU 3 | dt 1 | per camera: extrinsics 6, intrinsics 8)."""
    on = {b: bool(flags.get(b, calib)) for b in CALIB_BLOCKS}
    ids, i = {"imu": 0}, 15
    if on["calib_imu_intrinsics"]:
        ids["dw"], ids["da"], i = i, i + 6, i + 12
        if on["calib_imu_g_sensitivity"]:
            ids["tg"], i = i, i + 9
        ids["gyro"], i = i, i + 3
    if on["calib_cam_timeoffset"]:
        ids["dt"], i = i, i + 1
    for c in range(cams):
        if on["calib_cam_extrinsics"]:
            ids[f"cam{c}_ext"], i = i, i + 6
        if on["calib_cam_intrinsics"]:
            ids[f"cam{c}_intr"], i = i, i + 8
    ids["n"] = i
    return ids


def _run(runner, args, cwd):
    return subprocess.run([runner, "--traj", TRAJ, "--frames", "5"] + args, capture_output=True, text=True, cwd=cwd)


REFUSED = [
    ["--feat-rep-msckf", "GLOBAL"], ["--feat-rep-msckf", "global_3d"], ["--feat-rep-msckf"], ["--use-fej", "2"], ["--use-fej", "yes"], ["--use-fej"],
    ["--fi-triangulate-1d", "-1"], ["--fi-refine-features", "1.0"], ["--up-msckf-sigma-px", "0"], ["--up-msckf-sigma-px", "-1"],
    ["--up-msckf-chi2-multipler", "nan"], ["--up-slam-sigma-px", "inf"], ["--up-slam-chi2-multipler", "0"], ["--up-slam-chi2-multipler", "2x"],
    ["--calib-cam-extrinsics", "2"], ["--calib-cam-intrinsics", ""], ["--calib-cam-timeoffset", "on"], ["--calib-imu-intrinsics", "-0.5"],
    ["--calib-imu-g-sensitivity", "1", "--calib-imu-intrinsics", "0"], ["--calib-imu-intrinsics", "0", "--calib-imu-g-sensitivity", "1"],
    ["--calib", "0", "--calib-imu-g-sensitivity", "1"],
    ["--perturb", "--calib-cam-timeoffset", "0"], ["--perturb", "--calib-imu-g-sensitivity", "0"], ["--calib", "0", "--perturb", "--calib-cam-extrinsics", "1"],
]


@pytest.mark.parametrize("args", REFUSED, ids=[" ".join(a) or "empty" for a in REFUSED])
def test_malformed_or_refused_exits_2_before_running(runner, tmp_path, args):
    """Status 2 with a message, nothing printed on stdout and nothing written, single runs and --runs batches alike."""
    for extra in (["--est", "e.txt", "--consistency", "c.txt"], ["--runs", "2", "--out-dir", "d", "--consistency"]):
        r = _run(runner, extra + args, tmp_path)
        assert r.returncode == 2 and r.stdout == "" and r.stderr, (args, r.stderr)
        assert os.listdir(tmp_path) == []


def test_perturb_is_accepted_with_every_block_on(runner, tmp_path):
    """The --perturb refusal is about the blocks: every block switched on explicitly under --calib 0 runs."""
    on = [x for b in CALIB_BLOCKS for x in ("--" + b.replace("_", "-"), "1")]
    r = _run(runner, ["--calib", "0", "--perturb", "--cams", "1", "--frames", "3"] + on, tmp_path)
    assert r.returncode == 0, r.stderr
    assert '"perturb": true' in r.stdout and '"estimator": {"calib_cam_extrinsics": 1' in r.stdout


@pytest.mark.parametrize("case", list(OPTIONS))
def test_oracle_closed_loop_with_each_option(runner, tmp_path, case):
    """30 frames of config 1 with one option changed: a finite ATE, the "estimator" object, and a consistency header whose ids
    are the state layout the calibration flags imply."""
    kw, reported = OPTIONS[case]
    c = str(tmp_path / "c.txt")
    r = simrun.run(exe=runner, frames=30, consistency=c, **CONFIG1, **kw)
    assert r["frames"] == 30 and math.isfinite(r["ate_pos_m"]) and r["ate_pos_m"] < 0.3
    assert r.get("estimator", {}) == reported
    ids = simrun.load_consistency(c)["ids"]
    assert ids == layout(1, **kw)
    assert r["state_dim"] == ids["n"] + 6 * 11


def test_calib_block_flags_override_calib_wherever_they_stand(runner, tmp_path):
    """A --calib-* flag sets its block whether it comes before or after --calib; the others follow --calib."""
    hdr = []
    for args in (["--calib", "0", "--calib-cam-intrinsics", "1"], ["--calib-cam-intrinsics", "1", "--calib", "0"]):
        c = tmp_path / f"c{len(hdr)}.txt"
        r = _run(runner, ["--cams", "2", "--clones", "5", "--pts", "100", "--consistency", str(c)] + args, tmp_path)
        assert r.returncode == 0, r.stderr
        assert '"estimator": {"calib_cam_intrinsics": 1}' in r.stdout
        hdr.append(simrun.load_consistency(c)["ids"])
    assert hdr[0] == hdr[1] == layout(2, calib=0, calib_cam_intrinsics=1)


def test_capture_keeps_the_options(runner, tmp_path):
    """A captured update carries the ovb_opts the run used: representation, FEJ, triangulation, noise, gate and the
    calibration columns."""
    kw = dict(feat_rep_msckf="ANCHORED_INVERSE_DEPTH_SINGLE", use_fej=0, fi_triangulate_1d=1, fi_refine_features=0, up_msckf_sigma_px=1.5,
              up_msckf_chi2_multipler=3, calib_cam_extrinsics=0)
    prefix = str(tmp_path / "cap")
    simrun.run(exe=runner, frames=12, capture=(10, prefix), **CONFIG1, **kw)
    frame, _, opts, P = simrun.load_case(prefix + ".case")
    assert opts.feat_rep == REPS.index("ANCHORED_INVERSE_DEPTH_SINGLE") and opts.do_fej == 0
    assert opts.triangulate_1d == 1 and opts.refine_features == 0 and opts.sigma_pix == 1.5 and opts.chi2_multipler == 3
    assert opts.do_calib_camera_pose == 0 and opts.do_calib_camera_intrinsics == 1
    assert np.all(frame.cam_ext_off == -1) and np.all(frame.cam_intr_off >= 0)
    d = capi.default_opts()
    simrun.run(exe=runner, frames=12, capture=(10, prefix), **CONFIG1)
    _, _, opts0, _ = simrun.load_case(prefix + ".case")
    assert (opts0.feat_rep, opts0.do_fej, opts0.triangulate_1d, opts0.refine_features, opts0.sigma_pix) == (d.feat_rep, 1, 0, 1, 1.0)


def test_batch_runs_with_an_option_equal_single_runs(runner, tmp_path):
    """--runs with a non-default option: every per_run entry reports it, and each run writes what the same seed writes alone."""
    kw = dict(CONFIG1, frames=25, use_fej=0, feat_rep_msckf="ANCHORED_3D")
    b = simrun.run(exe=runner, runs=3, jobs=3, out_dir=str(tmp_path / "mc"), consistency=True, seed_meas=4, **kw)
    want = {"feat_rep_msckf": "ANCHORED_3D", "use_fej": 0}
    assert b["estimator"] == want and all(e["estimator"] == want for e in b["per_run"])
    for e in b["per_run"]:
        single = tmp_path / f"s{e['seed']}.txt"
        s = simrun.run(exe=runner, est=str(single), seed_meas=e["seed"], **kw)
        assert single.read_bytes() == (tmp_path / "mc" / f"est_{e['seed']}.txt").read_bytes()
        assert s["status_hist"] == e["status_hist"]


# ---------------------------------------------------------------------------------------------------------------------
# Without the new flags (or with each at its default value), every output is byte for byte what the runner wrote before
# the flags existed: the SHA-256 digests below were taken with the oracle-backed runner built from the parent commit. Host
# time fields (stdout's mean_ms_*, wall_s, runs_per_s, frames_per_s; the timing CSV's stage columns) are masked.
_TIME_FIELDS = re.compile(r'("(?:mean_ms_\w+|wall_s|runs_per_s|frames_per_s)": )[-+0-9.eE]+')
DEFAULT_COMMANDS = {
    "single": ["--cams", "1", "--clones", "11", "--msckf", "50", "--pts", "200", "--frames", "30", "--est", "est.txt", "--consistency", "cons.txt",
               "--timing", "timing.csv", "--capture", "20", "cap"],
    "slam": ["--cams", "1", "--clones", "11", "--msckf", "50", "--pts", "200", "--frames", "40", "--slam", "25", "--feat-rep-slam", "ANCHORED_3D",
             "--slam-log", "slam.txt", "--est", "est.txt"],
    "batch": ["--cams", "2", "--clones", "8", "--msckf", "40", "--pts", "150", "--frames", "20", "--runs", "2", "--jobs", "2", "--out-dir", "mc",
              "--consistency", "--timing"],
    "calib0": ["--cams", "1", "--clones", "11", "--msckf", "50", "--pts", "200", "--frames", "20", "--calib", "0", "--est", "est.txt",
               "--consistency", "cons.txt"],
}
DEFAULT_DIGESTS = {
    "single": {
        "cap.case": "fc59b9c7dab3263825870fc2723336ec22ea557a767aa4692011792d73edfbe8",
        "cons.txt": "5a63347868925a705841c7cd274ab0452aa4b3a8eb7d5445f21d30407472572e",
        "est.txt": "190fc9b4a81f4044fdcf199e56009733910b21493eed03b8c22942033e8eedb0",
        "stdout": "d966368651273ba3b53ead57ce326b7e2e2b1dff3a7020045a906c9034af2aac",
        "timing.csv": "5b2939c61d64202a78706bcca5de19635c9cf2b09fd43a68b7a3b806f33d4d40",
    },
    "slam": {
        "est.txt": "71b33cd2779d0694842ce77218d10d7cc80b380a48a2efac02ff18a784c2e30b",
        "slam.txt": "57870f9a769927b0346b5ba335f2791b248729e9e73e92b4ebcdda22a7f91ba0",
        "stdout": "307920371f7062123acc2420b844f20d6f9d041d29f3efc0691131a035e48c61",
    },
    "batch": {
        "mc/consistency_0.txt": "67bd58fcf477321dd7394e261153eb3251762931b3e151d84729091e0814cfb6",
        "mc/consistency_1.txt": "91402d2774113a2101c1a2616ede6eda3788ff40237aecd079f1e3ccabb90559",
        "mc/est_0.txt": "1eec864e69c0a73eb8c519a603ecde2ae1b8121ec9be03ac5b336a66be10875f",
        "mc/est_1.txt": "8c7bd5872625a1e8351ce5d5112f780d3128d60e6c2c6927b8a9d31a78e34e35",
        "mc/timing_0.csv": "a333140fd88aa801124779018b7e69cdbe0ee48d26f9863d0f8d1b31802775d3",
        "mc/timing_1.csv": "4278b357ea107faa3dc0d3226644cba9c27885f2ec5468c195b0b49dfcda2e3c",
        "stdout": "d8fbdbf356ff91b3e3cd4653e78191cb1d331a014316041d3efac3c4e8425cc4",
    },
    "calib0": {
        "cons.txt": "16da4c2e6f8003a925c291f65d216d3af32ec3cc985e21cc61629882b39e7e23",
        "est.txt": "0aa1e44f170c67029cf1291935796b67c6f3e8ae76f96a90000fcb6a4df7d0f1",
        "stdout": "d8900066ae144a43528e04666502be14072c655a870273920b17bb022d7543b4",
    },
}
DEFAULT_VALUED_FLAGS = ["--feat-rep-msckf", "GLOBAL_3D", "--use-fej", "1", "--fi-triangulate-1d", "0", "--fi-refine-features", "1",
                        "--up-msckf-sigma-px", "1", "--up-msckf-chi2-multipler", "1", "--up-slam-sigma-px", "1.0", "--up-slam-chi2-multipler", "1"]


def default_output_digests(exe, args, cwd):
    """SHA-256 of stdout and of every file the command writes (time fields masked)."""
    r = subprocess.run([exe, "--traj", TRAJ] + args, capture_output=True, text=True, cwd=cwd, check=True)
    out = {"stdout": hashlib.sha256(_TIME_FIELDS.sub(r"\1X", r.stdout).encode()).hexdigest()}
    for root, _, files in os.walk(cwd):
        for name in files:
            path = os.path.join(root, name)
            data = open(path, "rb").read()
            if name.endswith(".csv"):  # the timing CSV: header and timestamps
                data = b"\n".join(line.split(b",")[0] for line in data.splitlines())
            out[os.path.relpath(path, cwd)] = hashlib.sha256(data).hexdigest()
    return out


@pytest.mark.parametrize("name", list(DEFAULT_COMMANDS))
@pytest.mark.parametrize("flags", ["none", "defaults"])
def test_outputs_without_the_flags_are_unchanged(runner, tmp_path, name, flags):
    args = DEFAULT_COMMANDS[name]
    calib = ["--calib-" + b[6:].replace("_", "-") for b in CALIB_BLOCKS]
    if flags == "defaults":  # every new flag at its default value (the calibration blocks at --calib's)
        on = "0" if "--calib" in args and args[args.index("--calib") + 1] == "0" else "1"
        args = args + DEFAULT_VALUED_FLAGS + [x for f in calib for x in (f, on)]
    assert default_output_digests(runner, args, tmp_path) == DEFAULT_DIGESTS[name]
