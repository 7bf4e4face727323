"""GPU tests of equidistant (fisheye) cameras on the CUDA engine: one captured fisheye update against the oracle
(tests/golden/rpng_sim_equi_mono11_f50.case.gz), the closed loop against the oracle-backed runner on a mono, a stereo and a
mixed radtan + equidistant rig, and a concurrent --runs batch against the same seeds run alone.

The closed-loop bars follow the radtan ones of tests/test_gpu_sim.py and tests/test_gpu_consistency.py: the noise floor
between two builds of the CPU oracle, with and without FMA contraction (tools/ate_noise_floor.sh with --cam-model), times
three and rounded up to one significant digit. Floors and measured engine values: DESIGN.md §5."""
import os

import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import capi, simrun

pytestmark = pytest.mark.gpu

# made by tests/golden/make_rpng_sim_equi_case.py
CASE_EQUI = os.path.join(os.path.dirname(simrun.CASE_CONFIG1), "rpng_sim_equi_mono11_f50.case.gz")
CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1)  # BASELINE config 1: mono, 11 clones, 50 features
STEREO = dict(cams=2, clones=20, msckf=120, pts=300, frames=80, calib=1)  # the stereo run of tests/test_gpu_sim.py

# (runner options, pointwise position bar [m], |ΔATE| bar [m], max relative σ bar, max |ΔNEES| bar). Floors (pointwise,
# ATE, σ, NEES): mono 6.4e-6, 7.2e-7, 6.2e-5, 4.5e-4; stereo 3.1e-5, 1.05e-5, 5.1e-5, 9.5e-3; mixed 5.5e-5, 9.4e-6, 1.9e-4,
# 5.9e-3.
CLOSED_LOOP = {
    "mono_equi": (dict(CONFIG1, frames=300, cam_model="equi"), 2e-5, 3e-6, 2e-4, 2e-3),
    "stereo_equi": (dict(STEREO, cam_model="equi"), 1e-4, 4e-5, 2e-4, 3e-2),
    "mixed_radtan_equi": (dict(STEREO, cam_model="radtan,equi"), 2e-4, 3e-5, 6e-4, 2e-2),
}


@pytest.fixture(scope="module")
def exes():
    from oracle import ovo_py
    ovo_py.build()
    return b.build_sim_tools(), ovo_py.build_sim_runner()


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def test_captured_fisheye_update_engine_vs_oracle(oracle):
    """One MSCKF update captured from a fisheye config-1 run (mono, 11 clones, at most 50 features, calibration on; 43
    features in, 28 triangulated): the parity bars
    of tests/test_gpu_parity.py. Stage-0 residuals go through the device's double atan and products where the oracle calls
    glibc's atan and std::pow; the count of bit-identical residuals is printed (DESIGN.md §5) and bounded by one float32 ulp
    of a pixel in [256, 512)."""
    frame, feats, opts, P = simrun.load_case(CASE_EQUI)
    assert np.all(frame.cam_model == capi.CAM_EQUI)
    F = feats.n_feats
    eng = capi.Engine(max_state=256, max_feats=1024, max_meas=1024 * 48)
    try:
        # triangulation: bit-identical on >= 99 % of the features, within 1e-12 on all
        ref, _ = oracle.triangulate(frame, feats, opts)
        got = eng.triangulate(frame, feats, opts)
        assert np.array_equal(got.status, ref.status)
        ok = ref.status == capi.FEAT_OK
        assert ok.sum() >= 0.5 * F
        rel = np.linalg.norm(got.p_FinG[ok] - ref.p_FinG[ok], axis=1) / np.linalg.norm(ref.p_FinG[ok], axis=1)
        assert rel.max() <= 1e-12, rel.max()
        exact = np.all(got.p_FinG[ok] == ref.p_FinG[ok], axis=1).mean()
        assert exact >= 0.99, exact
        # stage 0: residuals of the pre-nullspace rows
        eng.cov_set(P)
        Hf, Hx, res, row_off, cols = eng.feature_jacobians(frame, feats, opts, ref.copy(), 0)
        Hf_r, Hx_r, res_r, row_off_r = oracle.feature_jacobians(frame, feats, opts, ref.copy(), 0, cols)
        assert np.array_equal(row_off, row_off_r)
        same = int(np.sum(res.view(np.uint64) == res_r.view(np.uint64)))
        print(f"\nstage-0 residuals bit-identical to the oracle: {same} of {res.size}")
        assert same >= 0.99 * res.size and np.abs(res - res_r).max() <= 2.0**-14
        assert np.abs(Hx - Hx_r).max() <= 1e-12 * max(np.abs(Hx_r).max(), 1.0)
        assert np.abs(Hf - Hf_r).max() <= 1e-12 * max(np.abs(Hf_r).max(), 1.0)
        # stage 1: gate decisions
        out_g, out_r = ref.copy(), ref.copy()
        eng.feature_jacobians(frame, feats, opts, out_g, 1)
        oracle.feature_jacobians(frame, feats, opts, out_r, 1, cols, P=P)
        assert np.array_equal(out_g.status, out_r.status), "chi² gate decisions differ"
        # the whole update: P+ and dx within 1e-9 relative Frobenius
        eng.cov_set(P)
        st, out, dx, stats = eng.msckf_update(frame, feats, opts)
        ur = oracle.msckf_update(frame, feats, opts, P, dumps=False)
        assert st == ur["status"] == 0 and np.array_equal(out.status, ur["out"].status) and stats.n_feats_used > 5
        assert np.linalg.norm(eng.cov_get() - ur["P"]) <= 1e-9 * np.linalg.norm(ur["P"])
        assert np.linalg.norm(dx - ur["dx"]) <= 1e-9 * np.linalg.norm(ur["dx"])
    finally:
        eng.close()


@pytest.mark.parametrize("case", list(CLOSED_LOOP))
def test_closed_loop_engine_vs_oracle(exes, tmp_path, case):
    cfg, bar_p, bar_ate, bar_sigma, bar_nees = CLOSED_LOOP[case]
    eng, orc = exes
    eg, eo, cg, co = (str(tmp_path / n) for n in ("eg.txt", "eo.txt", "cg.txt", "co.txt"))
    rg = simrun.run(exe=eng, est=eg, consistency=cg, **cfg)
    ro = simrun.run(exe=orc, est=eo, consistency=co, **cfg)
    assert rg["frames"] == ro["frames"] == cfg["frames"]
    assert rg["cam_model"] == ro["cam_model"] == (cfg["cam_model"].split(",") * cfg["cams"])[:cfg["cams"]]
    assert rg["status_hist"] == ro["status_hist"], "gate / triangulation decisions differ between the engine and the oracle"
    _, pg, _, _, _ = simrun.load_estimate(eg)
    _, po, _, _, _ = simrun.load_estimate(eo)
    g, o = simrun.load_consistency(cg), simrun.load_consistency(co)
    dp, date = np.abs(pg - po).max(), abs(rg["ate_pos_m"] - ro["ate_pos_m"])
    rel = np.abs(g["sigma"] - o["sigma"]) / o["sigma"]
    dn = max(np.abs(g["nees_ori"] - o["nees_ori"]).max(), np.abs(g["nees_pos"] - o["nees_pos"]).max())
    print(f"\n{case}: ATE engine {rg['ate_pos_m']:.6f} m oracle {ro['ate_pos_m']:.6f} m; max |dp| {dp:.3e} m, |dATE| {date:.3e} m, "
          f"|dATE ori| {abs(rg['ate_ori_deg'] - ro['ate_ori_deg']):.3e} deg, max rel dsigma {rel.max():.3e}, max |dNEES| {dn:.3e}")
    assert dp <= bar_p and date <= bar_ate
    assert abs(rg["ate_ori_deg"] - ro["ate_ori_deg"]) <= 1e-4
    assert rg["ate_pos_m"] < 0.3
    assert g["ids"] == o["ids"] and np.array_equal(g["t"], o["t"])
    assert rel.max() <= bar_sigma and dn <= bar_nees


def test_concurrent_fisheye_batch_equals_single_runs(exes, tmp_path):
    """--runs with --cam-model equi: each of 8 concurrent runs writes the same estimate, bit for bit, as the same seed run
    alone (tests/test_gpu_monte_carlo.py's radtan check)."""
    eng, _ = exes
    S, K, kw = 40, 8, dict(CONFIG1, frames=100, cam_model="equi")
    out = tmp_path / "mc"
    batch = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(out), seed_meas=S, **kw)
    assert batch["backend"] == "engine" and batch["cam_model"] == ["equi"] and [r["seed"] for r in batch["per_run"]] == list(range(S, S + K))
    for entry in batch["per_run"]:
        seed = entry["seed"]
        single = str(tmp_path / f"single_{seed}.txt")
        r = simrun.run(exe=eng, est=single, seed_meas=seed, **kw)
        assert _read(single) == _read(out / f"est_{seed}.txt"), f"seed {seed}: the concurrent run differs from the run alone"
        assert entry["status_hist"] == r["status_hist"] and entry["frames"] == r["frames"] == 100
    p = np.array([r["ate_pos_m"] for r in batch["per_run"]])
    assert len(set(p.tolist())) == K and np.all(p < 0.3)
