"""GPU tests of SLAM landmarks in the rpng_sim closed loop: the engine runner (ovb_run_simulation --slam) against the
oracle-backed runner on the same inputs, and a concurrent --runs batch against the same seeds run alone.

Bars: the noise floor between two builds of the CPU oracle, with and without FMA contraction (tools/ate_noise_floor.sh with the
SLAM options), times three and rounded up to one significant digit, the convention of tests/test_gpu_sim.py and
tests/test_gpu_sim_equi.py. Both oracle builds take the same MSCKF, SLAM and delayed-init decisions over every horizon used
here. Floors and measured engine values: DESIGN.md §5."""
import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import simrun
from tests.test_sim_slam_cpu import oracle_runner

pytestmark = pytest.mark.gpu

CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1, frames=300)  # BASELINE config 1: mono, 11 clones, 50 features
STEREO = dict(cams=2, clones=20, msckf=120, pts=300, frames=80, calib=1)  # the stereo run of tests/test_gpu_sim.py

# (runner options, pointwise position bar [m], |ΔATE| bar [m], max relative σ bar, max |ΔNEES| bar). Floors (pointwise, ATE,
# σ, NEES ori / pos): global3d 6.3e-6, 5.0e-7, 1.1e-5, 3.7e-4 / 1.7e-4; stereo 7.0e-6, 4.8e-7, 2.2e-5, 1.9e-4 / 9.4e-5;
# full inverse depth 1.1e-5, 1.7e-7, 1.4e-5, 7.8e-4 / 2.4e-4; single 6.3e-6, 2.2e-6, 1.9e-5, 9.9e-4 / 2.9e-4; unbounded
# 6.3e-6, 5.2e-7, 1.2e-5, 2.9e-4 / 1.7e-4. On the full-inverse-depth run the two oracle builds' ATE errors happened to cancel
# to 1.7e-7 m while they differ by 1.1e-5 m pointwise; its |ΔATE| bar is the global-3D run's (same horizon and shape), 2e-6.
CLOSED_LOOP = {
    "mono_global3d": (dict(CONFIG1, slam=25), 2e-5, 2e-6, 4e-5, 2e-3),
    "stereo_msckf_inverse_depth": (dict(STEREO, slam=50, feat_rep_slam="ANCHORED_MSCKF_INVERSE_DEPTH"), 3e-5, 2e-6, 7e-5, 6e-4),
    "mono_full_inverse_depth": (dict(CONFIG1, slam=25, feat_rep_slam="ANCHORED_FULL_INVERSE_DEPTH"), 4e-5, 2e-6, 5e-5, 3e-3),
    "mono_single": (dict(CONFIG1, slam=25, feat_rep_slam="ANCHORED_INVERSE_DEPTH_SINGLE"), 2e-5, 7e-6, 6e-5, 3e-3),
    "mono_unbounded": (dict(CONFIG1, slam=100, slam_in_update=100), 2e-5, 2e-6, 4e-5, 9e-4),
}
COUNTS = ("status_hist", "slam_status_hist", "init_status_hist", "slam_initialized", "slam_marginalized", "anchor_changes", "max_slam_live")


@pytest.fixture(scope="module")
def exes():
    from oracle import ovo_py
    ovo_py.build()
    return b.build_sim_tools(), oracle_runner()


def _read(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.parametrize("case", list(CLOSED_LOOP))
def test_slam_closed_loop_engine_vs_oracle(exes, tmp_path, case):
    cfg, bar_p, bar_ate, bar_sigma, bar_nees = CLOSED_LOOP[case]
    eng, orc = exes
    eg, eo, cg, co = (str(tmp_path / n) for n in ("eg.txt", "eo.txt", "cg.txt", "co.txt"))
    rg = simrun.run(exe=eng, est=eg, consistency=cg, **cfg)
    ro = simrun.run(exe=orc, est=eo, consistency=co, **cfg)
    assert rg["frames"] == ro["frames"] == cfg["frames"]
    for k in COUNTS:
        assert rg[k] == ro[k], f"{k}: engine {rg[k]} oracle {ro[k]}"
    assert rg["state_dim"] == ro["state_dim"] and rg["slam_initialized"] > 0 and rg["max_slam_live"] <= cfg["slam"]
    if cfg.get("feat_rep_slam", "GLOBAL_3D").startswith("ANCHORED"):
        assert rg["anchor_changes"] > 0
    _, pg, _, _, _ = simrun.load_estimate(eg)
    _, po, _, _, _ = simrun.load_estimate(eo)
    g, o = simrun.load_consistency(cg), simrun.load_consistency(co)
    dp, date = np.abs(pg - po).max(), abs(rg["ate_pos_m"] - ro["ate_pos_m"])
    rel = np.abs(g["sigma"] - o["sigma"]) / o["sigma"]
    dn = max(np.abs(g["nees_ori"] - o["nees_ori"]).max(), np.abs(g["nees_pos"] - o["nees_pos"]).max())
    print(f"\n{case}: ATE engine {rg['ate_pos_m']:.6f} m oracle {ro['ate_pos_m']:.6f} m; max |dp| {dp:.3e} m, |dATE| {date:.3e} m, "
          f"|dATE ori| {abs(rg['ate_ori_deg'] - ro['ate_ori_deg']):.3e} deg, max rel dsigma {rel.max():.3e}, max |dNEES| {dn:.3e}; "
          f"live landmarks mean {rg['mean_slam_live']:.1f}, initialised {rg['slam_initialized']}, anchor changes {rg['anchor_changes']}; "
          f"engine ms/frame: SLAM update {rg['mean_ms_slam_update']:.3f}, delayed init {rg['mean_ms_slam_delayed']:.3f}")
    assert dp <= bar_p and date <= bar_ate
    assert abs(rg["ate_ori_deg"] - ro["ate_ori_deg"]) <= 1e-4
    assert rg["ate_pos_m"] < 0.3
    assert g["ids"] == o["ids"] and np.array_equal(g["t"], o["t"])
    assert rel.max() <= bar_sigma and dn <= bar_nees


def test_concurrent_slam_batch_equals_single_runs(exes, tmp_path):
    """--runs with --slam: each of 8 concurrent runs writes the same estimate, bit for bit, and the same SLAM counts as the
    same seed run alone."""
    eng, _ = exes
    S, K, kw = 20, 8, dict(CONFIG1, frames=120, slam=25, feat_rep_slam="ANCHORED_MSCKF_INVERSE_DEPTH")
    out = tmp_path / "mc"
    batch = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(out), seed_meas=S, **kw)
    assert batch["backend"] == "engine" and [r["seed"] for r in batch["per_run"]] == list(range(S, S + K))
    for entry in batch["per_run"]:
        seed = entry["seed"]
        single = str(tmp_path / f"single_{seed}.txt")
        r = simrun.run(exe=eng, est=single, seed_meas=seed, **kw)
        assert _read(single) == _read(out / f"est_{seed}.txt"), f"seed {seed}: the concurrent run differs from the run alone"
        for k in COUNTS:
            assert entry[k] == r[k], (seed, k)
        assert entry["frames"] == r["frames"] == 120
    p = np.array([r["ate_pos_m"] for r in batch["per_run"]])
    assert len(set(p.tolist())) == K and np.all(p < 0.3)
