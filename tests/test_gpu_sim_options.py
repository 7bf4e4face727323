"""GPU tests of the rpng_sim runner's estimator options (INTEGRATION.md §8, "Estimator options") on the CUDA engine: the
closed loop against the oracle-backed runner on the same seeds, 300 frames at config 1 and at the stereo shape of
tests/test_gpu_sim.py, for each MSCKF representation, FEJ off, 1-D triangulation, refinement off, a non-unit σ and χ²
multiplier, each calibration block off alone, and SLAM runs with FEJ off or the SLAM σ and multiplier changed; a concurrent
--runs batch with options against the same seeds run alone; and the engine runner's outputs without the flags, byte for byte
those of the runner before the flags existed.

Bars: the convention of tests/test_gpu_sim_equi.py — three times the noise floor between two builds of the CPU oracle, with
and without FMA contraction (tools/ate_noise_floor.sh with the case's options), rounded up to one significant digit. A case
whose floor lies below its shape's default run (GLOBAL_3D, every option at its default) takes the default run's: any two
builds that are not bit-identical settle that far apart (tests/test_gpu_sim.py). Both oracle builds take the same gate,
triangulation, SLAM and delayed-init decisions in every case. Floors and measured engine values: DESIGN.md §5."""
import math

import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import simrun
from tests.test_sim_options_cpu import CALIB_BLOCKS, DEFAULT_COMMANDS, DEFAULT_VALUED_FLAGS, REPS, default_output_digests, layout

pytestmark = pytest.mark.gpu

SHAPES = {
    "mono": dict(cams=1, clones=11, msckf=50, pts=200, calib=1, frames=300),  # BASELINE config 1: mono, 11 clones, 50 features
    "stereo": dict(cams=2, clones=20, msckf=120, pts=300, calib=1, frames=80),  # the stereo run of tests/test_gpu_sim.py
}
OPTIONS = {r: dict(feat_rep_msckf=r) for r in REPS}
OPTIONS.update({
    "no_fej": dict(use_fej=0),
    "triangulate_1d": dict(fi_triangulate_1d=1),
    "no_refine": dict(fi_refine_features=0),
    "msckf_sigma_chi2": dict(up_msckf_sigma_px=1.5, up_msckf_chi2_multipler=2),
})
OPTIONS.update({f"no_{blk[6:]}": {blk: 0} for blk in CALIB_BLOCKS})
SLAM = {
    "slam_no_fej_anchored_3d": dict(SHAPES["mono"], slam=25, use_fej=0, feat_rep_slam="ANCHORED_3D"),
    "slam_sigma_chi2_msckf_inverse_depth": dict(SHAPES["mono"], slam=25, feat_rep_slam="ANCHORED_MSCKF_INVERSE_DEPTH", up_slam_sigma_px=1.5,
                                                up_slam_chi2_multipler=2),
}

# Floors (pointwise position [m], |ΔATE| [m], max relative σ, max |ΔNEES| of orientation and position) per case
FLOORS = {
    "mono": {"GLOBAL_3D": (5.86e-6, 1.04e-6, 2.72e-5, 2.91e-4), "GLOBAL_FULL_INVERSE_DEPTH": (5.86e-6, 2.09e-6, 1.10e-5, 3.99e-4),
             "ANCHORED_3D": (6.06e-6, 1.10e-6, 2.10e-5, 3.58e-4), "ANCHORED_FULL_INVERSE_DEPTH": (5.86e-6, 4.35e-7, 1.93e-5, 3.94e-4),
             "ANCHORED_MSCKF_INVERSE_DEPTH": (5.86e-6, 6.72e-7, 1.10e-5, 3.98e-4), "ANCHORED_INVERSE_DEPTH_SINGLE": (5.86e-6, 6.72e-7, 1.10e-5, 3.98e-4),
             "no_fej": (6.55e-6, 4.73e-7, 3.32e-5, 1.01e-3), "triangulate_1d": (7.68e-6, 2.16e-7, 2.17e-5, 3.81e-4),
             "no_refine": (1.61e-6, 4.54e-7, 1.70e-6, 5.14e-4), "msckf_sigma_chi2": (3.66e-6, 5.50e-7, 1.06e-5, 3.49e-4),
             "no_cam_extrinsics": (7.33e-6, 5.12e-7, 1.57e-5, 6.43e-4), "no_cam_intrinsics": (4.25e-6, 1.16e-7, 1.64e-5, 3.84e-4),
             "no_cam_timeoffset": (1.01e-5, 1.37e-6, 2.17e-5, 3.31e-4), "no_imu_intrinsics": (3.27e-6, 6.84e-8, 1.21e-5, 1.88e-4),
             "no_imu_g_sensitivity": (9.57e-6, 9.11e-7, 1.28e-5, 1.14e-3)},
    "stereo": {"GLOBAL_3D": (5.86e-6, 5.12e-7, 2.19e-5, 1.97e-4), "GLOBAL_FULL_INVERSE_DEPTH": (5.85e-6, 6.43e-7, 2.19e-5, 1.97e-4),
               "ANCHORED_3D": (5.85e-6, 6.09e-7, 2.19e-5, 1.74e-4), "ANCHORED_FULL_INVERSE_DEPTH": (5.85e-6, 4.97e-7, 2.19e-5, 2.05e-4),
               "ANCHORED_MSCKF_INVERSE_DEPTH": (5.86e-6, 5.82e-7, 2.19e-5, 1.40e-4), "ANCHORED_INVERSE_DEPTH_SINGLE": (5.86e-6, 5.82e-7, 2.19e-5, 1.40e-4),
               "no_fej": (9.78e-6, 1.58e-6, 2.67e-5, 5.14e-4), "triangulate_1d": (2.36e-6, 1.08e-7, 1.89e-5, 2.14e-4),
               "no_refine": (5.70e-7, 1.64e-8, 1.98e-6, 1.98e-4), "msckf_sigma_chi2": (2.58e-6, 3.16e-7, 1.65e-5, 2.48e-4),
               "no_cam_extrinsics": (4.40e-6, 1.94e-7, 1.98e-5, 1.48e-4), "no_cam_intrinsics": (3.07e-6, 4.70e-7, 1.31e-5, 2.29e-4),
               "no_cam_timeoffset": (4.33e-6, 4.75e-7, 1.75e-5, 1.51e-4), "no_imu_intrinsics": (4.19e-6, 4.64e-7, 1.72e-5, 5.37e-4),
               "no_imu_g_sensitivity": (3.69e-6, 4.87e-7, 1.64e-5, 1.35e-4)},
    "slam": {"slam_no_fej_anchored_3d": (1.36e-5, 4.96e-6, 1.50e-5, 3.17e-4), "slam_sigma_chi2_msckf_inverse_depth": (5.87e-6, 9.80e-7, 1.18e-5, 2.91e-4)},
}
COUNTS = ("status_hist", "slam_status_hist", "init_status_hist", "slam_initialized", "slam_marginalized", "anchor_changes", "max_slam_live",
          "state_dim")


def bars(floor, default):
    """Three times the larger of the case's floor and its shape's default floor, rounded up to one significant digit."""
    out = []
    for f, d in zip(floor, default):
        x = 3 * max(f, d)
        e = 10.0 ** math.floor(math.log10(x))
        out.append(math.ceil(x / e - 1e-9) * e)
    return out


@pytest.fixture(scope="module")
def exes():
    from oracle import ovo_py
    ovo_py.build()
    return b.build_sim_tools(), ovo_py.build_sim_runner()


def _closed_loop(exes, tmp_path, name, cfg, floor, default):
    eng, orc = exes
    bar_p, bar_ate, bar_sigma, bar_nees = bars(floor, default)
    eg, eo, cg, co = (str(tmp_path / n) for n in ("eg.txt", "eo.txt", "cg.txt", "co.txt"))
    rg = simrun.run(exe=eng, est=eg, consistency=cg, **cfg)
    ro = simrun.run(exe=orc, est=eo, consistency=co, **cfg)
    assert rg["frames"] == ro["frames"] == cfg["frames"]
    assert rg.get("estimator") == ro.get("estimator")
    for k in COUNTS:
        assert rg.get(k) == ro.get(k), f"{k}: engine {rg.get(k)} oracle {ro.get(k)}"
    _, pg, _, _, _ = simrun.load_estimate(eg)
    _, po, _, _, _ = simrun.load_estimate(eo)
    g, o = simrun.load_consistency(cg), simrun.load_consistency(co)
    dp, date = np.abs(pg - po).max(), abs(rg["ate_pos_m"] - ro["ate_pos_m"])
    rel = np.abs(g["sigma"] - o["sigma"]) / o["sigma"]
    dn = max(np.abs(g["nees_ori"] - o["nees_ori"]).max(), np.abs(g["nees_pos"] - o["nees_pos"]).max())
    print(f"\n{name}: ATE engine {rg['ate_pos_m']:.6f} m oracle {ro['ate_pos_m']:.6f} m; max |dp| {dp:.3e} m (bar {bar_p:.0e}), |dATE| {date:.3e} m "
          f"(bar {bar_ate:.0e}), |dATE ori| {abs(rg['ate_ori_deg'] - ro['ate_ori_deg']):.3e} deg, max rel dsigma {rel.max():.3e} (bar {bar_sigma:.0e}), "
          f"max |dNEES| {dn:.3e} (bar {bar_nees:.0e}); engine ms/frame: msckf update {rg['mean_ms_msckf_update']:.3f}")
    assert dp <= bar_p and date <= bar_ate
    assert abs(rg["ate_ori_deg"] - ro["ate_ori_deg"]) <= 1e-4
    assert rg["ate_pos_m"] < 0.3
    assert g["ids"] == o["ids"] and np.array_equal(g["t"], o["t"])
    assert rel.max() <= bar_sigma and dn <= bar_nees
    return rg, g


@pytest.mark.parametrize("option", list(OPTIONS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_closed_loop_engine_vs_oracle(exes, tmp_path, shape, option):
    cfg = dict(SHAPES[shape], **OPTIONS[option])
    _, g = _closed_loop(exes, tmp_path, f"{shape} {option}", cfg, FLOORS[shape][option], FLOORS[shape]["GLOBAL_3D"])
    assert g["ids"] == layout(cfg["cams"], **OPTIONS[option])


@pytest.mark.parametrize("case", list(SLAM))
def test_slam_closed_loop_engine_vs_oracle(exes, tmp_path, case):
    rg, _ = _closed_loop(exes, tmp_path, case, SLAM[case], FLOORS["slam"][case], FLOORS["mono"]["GLOBAL_3D"])
    assert rg["slam_initialized"] > 0 and rg["anchor_changes"] > 0


def test_concurrent_batch_with_options_equals_single_runs(exes, tmp_path):
    """--runs 4 --jobs 4 with FEJ off, an anchored MSCKF representation and the time offset out of the state: each run's
    estimate and consistency file are bit for bit those of the same seed run alone."""
    eng, _ = exes
    S, K = 7, 4
    kw = dict(SHAPES["mono"], frames=100, use_fej=0, feat_rep_msckf="ANCHORED_FULL_INVERSE_DEPTH", calib_cam_timeoffset=0)
    out = tmp_path / "mc"
    batch = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(out), consistency=True, seed_meas=S, **kw)
    want = {"feat_rep_msckf": "ANCHORED_FULL_INVERSE_DEPTH", "use_fej": 0, "calib_cam_timeoffset": 0}
    assert batch["backend"] == "engine" and batch["estimator"] == want and [r["seed"] for r in batch["per_run"]] == list(range(S, S + K))
    for entry in batch["per_run"]:
        seed = entry["seed"]
        est, cons = tmp_path / f"e{seed}.txt", tmp_path / f"c{seed}.txt"
        r = simrun.run(exe=eng, est=str(est), consistency=str(cons), seed_meas=seed, **kw)
        assert est.read_bytes() == (out / f"est_{seed}.txt").read_bytes(), f"seed {seed}: the concurrent run differs from the run alone"
        assert cons.read_bytes() == (out / f"consistency_{seed}.txt").read_bytes()
        assert entry["estimator"] == r["estimator"] == want and entry["status_hist"] == r["status_hist"]


# SHA-256 of tests/test_sim_options_cpu.py's commands (time fields masked) on the engine runner built from the commit before
# the estimator flags existed, on an H100 80GB HBM3
ENGINE_DEFAULT_DIGESTS = {
    "single": {
        "cap.case": "cfaa050928d1c326bfdf61787e5968e41d2f697fa07453d9d0bb4beef43edaf2",
        "cons.txt": "5f46998e44dcecd8f6e76e87f0ab919459e2caee65e766272f4598fceebc896b",
        "est.txt": "b878e545baec238d7382d96774c9333e47cdc270e82821b80b88129ffdcd18de",
        "stdout": "85855696089ee88c3bc92d27f96e4689330136f31b25e444f55f25a043cdcdb9",
        "timing.csv": "5b2939c61d64202a78706bcca5de19635c9cf2b09fd43a68b7a3b806f33d4d40",
    },
    "slam": {
        "est.txt": "a4bbf105fde645ca8e1f78caa8055dd9958b4071da0fe5f84162cca66c6fca75",
        "slam.txt": "57870f9a769927b0346b5ba335f2791b248729e9e73e92b4ebcdda22a7f91ba0",
        "stdout": "f5dbe53045afe80cd2055c0e5c60c092722d2e70ce171e59c9d4e95766338352",
    },
    "batch": {
        "mc/consistency_0.txt": "4ec8046c2e3cbf39a6fd0506d9af8de0a6b6a9ca7b596f784b4a7175115e6e85",
        "mc/consistency_1.txt": "9f27546039a0f95eb1f388d9dee756b823134e97d5b1e12420f114f8d5c4c58b",
        "mc/est_0.txt": "39c579b718a9f4f4600076d7e1fe1a5e5dcc91cf9d5fd37f7a6f4d478972eeb4",
        "mc/est_1.txt": "2c41b5ea24d3ac9eabd072913f17f459f55f7e356cb81deff204a702bd8716dd",
        "mc/timing_0.csv": "a333140fd88aa801124779018b7e69cdbe0ee48d26f9863d0f8d1b31802775d3",
        "mc/timing_1.csv": "bc3d8b2b1c5f76774a38db5a48a8d3e46d0607d6a6a54029add17d040ca5bf3b",
        "stdout": "efb87800518ac17fa57d853561618782ffa798e58aff36f3529ef9726c544d2a",
    },
    "calib0": {
        "cons.txt": "51cab45ae735a0f00be9244accc9702c05dab898cef6e880891d7f0c452ff39f",
        "est.txt": "64d8cc7492a8ce4640c09c54da8e6fdc8f6ea3ae9a3fbee6de86514c7eaa5683",
        "stdout": "3dfecb2946c12a44ed8e9e73c3638b1b3028551a0c36af0a7070beb8113e14f4",
    },
}


@pytest.mark.parametrize("name", list(DEFAULT_COMMANDS))
@pytest.mark.parametrize("flags", ["none", "defaults"])
def test_engine_outputs_without_the_flags_are_unchanged(exes, tmp_path, name, flags):
    args = DEFAULT_COMMANDS[name]
    if flags == "defaults":
        on = "0" if "--calib" in args and args[args.index("--calib") + 1] == "0" else "1"
        args = args + DEFAULT_VALUED_FLAGS + [x for blk in CALIB_BLOCKS for x in ("--" + blk.replace("_", "-"), on)]
    assert default_output_digests(exes[0], args, tmp_path) == ENGINE_DEFAULT_DIGESTS[name]
