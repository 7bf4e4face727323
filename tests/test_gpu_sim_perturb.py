"""GPU tests of the perturbed calibration start (--perturb) on the CUDA engine: the closed loop against the oracle-backed
runner on config 1, a stereo run and config 1 with SLAM landmarks, one captured update from a perturbed run
(tests/golden/rpng_sim_perturbed_mono11_f50.case.gz) against the oracle, and a concurrent --runs batch against the same
seeds run alone. With --perturb every update evaluates the device's camera-intrinsic, extrinsic and time-offset columns
away from the true calibration, where a wrong column no longer multiplies a zero error.

The closed-loop bars follow tests/test_gpu_sim_equi.py: the noise floor between two builds of the CPU oracle, with and without
FMA contraction (tools/ate_noise_floor.sh with --perturb and the run's options), times three and rounded up to one
significant digit. Floors and measured engine values: DESIGN.md §5."""
import os

import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import capi, simrun
from tests.test_sim_slam_cpu import oracle_runner

pytestmark = pytest.mark.gpu

# made by tests/golden/make_rpng_sim_perturbed_case.py
CASE_PERTURBED = os.path.join(os.path.dirname(simrun.CASE_CONFIG1), "rpng_sim_perturbed_mono11_f50.case.gz")
CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1, frames=300, perturb=True)  # BASELINE config 1
STEREO = dict(cams=2, clones=20, msckf=120, pts=300, calib=1, frames=80, perturb=True)  # the stereo run of tests/test_gpu_sim.py

# (runner options, pointwise position bar [m], |ΔATE| bar [m], max relative σ bar, max |ΔNEES| bar, max |Δ calib_nerr| bar).
# Floors (pointwise, ATE, σ, NEES, calib_nerr): config 1 4.4e-6, 5.1e-7, 1.7e-5, 9.0e-4, 1.05e-4; stereo 4.4e-6, 1.03e-6,
# 2.1e-5, 2.4e-3, 1.6e-4; SLAM 3.7e-6, 9.6e-7, 1.7e-5, 6.9e-4, 2.0e-4.
CLOSED_LOOP = {
    "mono": (CONFIG1, 2e-5, 2e-6, 6e-5, 3e-3, 4e-4),
    "stereo": (STEREO, 2e-5, 4e-6, 7e-5, 8e-3, 5e-4),
    "mono_slam": (dict(CONFIG1, slam=25), 2e-5, 3e-6, 6e-5, 3e-3, 6e-4),
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
def test_perturbed_closed_loop_engine_vs_oracle(exes, tmp_path, case):
    cfg, bar_p, bar_ate, bar_sigma, bar_nees, bar_calib = CLOSED_LOOP[case]
    eng, orc = exes
    eg, eo, cg, co = (str(tmp_path / n) for n in ("eg.txt", "eo.txt", "cg.txt", "co.txt"))
    rg = simrun.run(exe=eng, est=eg, consistency=cg, **cfg)
    ro = simrun.run(exe=orc, est=eo, consistency=co, **cfg)
    assert rg["frames"] == ro["frames"] == cfg["frames"] and rg["perturb"] is ro["perturb"] is True
    for k in COUNTS:
        assert rg.get(k) == ro.get(k), f"{k}: engine {rg.get(k)} oracle {ro.get(k)}"
    _, pg, _, _, _ = simrun.load_estimate(eg)
    _, po, _, _, _ = simrun.load_estimate(eo)
    g, o = simrun.load_consistency(cg), simrun.load_consistency(co)
    dp, date = np.abs(pg - po).max(), abs(rg["ate_pos_m"] - ro["ate_pos_m"])
    rel = np.abs(g["sigma"] - o["sigma"]) / o["sigma"]
    dn = max(np.abs(g["nees_ori"] - o["nees_ori"]).max(), np.abs(g["nees_pos"] - o["nees_pos"]).max())
    dc = max(abs(rg[k][blk] - ro[k][blk]) for k in ("calib_nerr_first", "calib_nerr_last") for blk in ro[k])
    print(f"\n{case}: ATE engine {rg['ate_pos_m']:.6f} m oracle {ro['ate_pos_m']:.6f} m; max |dp| {dp:.3e} m, |dATE| {date:.3e} m, "
          f"|dATE ori| {abs(rg['ate_ori_deg'] - ro['ate_ori_deg']):.3e} deg, max rel dsigma {rel.max():.3e}, max |dNEES| {dn:.3e}, "
          f"max |d calib_nerr| {dc:.3e}; engine calib_nerr_last {rg['calib_nerr_last']}")
    assert dp <= bar_p and date <= bar_ate
    assert abs(rg["ate_ori_deg"] - ro["ate_ori_deg"]) <= 1e-4
    assert rg["ate_pos_m"] < 0.3
    assert g["ids"] == o["ids"] and np.array_equal(g["t"], o["t"])
    assert rel.max() <= bar_sigma and dn <= bar_nees
    assert dc <= bar_calib


def test_captured_perturbed_update_engine_vs_oracle(oracle):
    """One MSCKF update captured from a perturbed config-1 run (frame 27, where fx is 1.5 σ from the truth and 1.2 σ from the
    perturbed start; tests/test_sim_perturb_cpu.py checks that): the parity bars of tests/test_gpu_parity.py —
    triangulated points within 1e-12, the same gate decisions, P and dx within 1e-9 relative Frobenius."""
    frame, feats, opts, P = simrun.load_case(CASE_PERTURBED)
    eng = capi.Engine(max_state=256, max_feats=1024, max_meas=1024 * 48)
    try:
        ref, _ = oracle.triangulate(frame, feats, opts)
        got = eng.triangulate(frame, feats, opts)
        assert np.array_equal(got.status, ref.status)
        ok = ref.status == capi.FEAT_OK
        assert ok.sum() >= 0.5 * feats.n_feats
        rel = np.linalg.norm(got.p_FinG[ok] - ref.p_FinG[ok], axis=1) / np.linalg.norm(ref.p_FinG[ok], axis=1)
        assert rel.max() <= 1e-12, rel.max()
        eng.cov_set(P)
        _, _, _, _, cols = eng.feature_jacobians(frame, feats, opts, ref.copy(), 0)
        out_g, out_r = ref.copy(), ref.copy()
        eng.feature_jacobians(frame, feats, opts, out_g, 1)
        oracle.feature_jacobians(frame, feats, opts, out_r, 1, cols, P=P)
        assert np.array_equal(out_g.status, out_r.status), "chi² gate decisions differ"
        eng.cov_set(P)
        st, out, dx, stats = eng.msckf_update(frame, feats, opts)
        ur = oracle.msckf_update(frame, feats, opts, P, dumps=False)
        assert st == ur["status"] == 0 and np.array_equal(out.status, ur["out"].status) and stats.n_feats_used > 5
        eP = np.linalg.norm(eng.cov_get() - ur["P"]) / np.linalg.norm(ur["P"])
        edx = np.linalg.norm(dx - ur["dx"]) / np.linalg.norm(ur["dx"])
        print(f"\nperturbed case: {stats.n_feats_used}/{stats.n_feats_in} features used, relerr P {eP:.2e} dx {edx:.2e}")
        assert eP <= 1e-9 and edx <= 1e-9
    finally:
        eng.close()


def test_concurrent_perturbed_batch_equals_single_runs(exes, tmp_path):
    """--runs 4 --perturb: run r (perturbation seed S + r, measurement seed S + r) writes the same estimate, bit for bit, as
    those seeds run alone, and reports the same per-block calibration errors."""
    eng, _ = exes
    S, K, kw = 30, 4, dict(CONFIG1, frames=100)
    out = tmp_path / "mc"
    batch = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(out), seed_meas=S, seed_perturb=S, **kw)
    assert batch["backend"] == "engine" and batch["perturb"] is True
    assert [r["seed"] for r in batch["per_run"]] == [r["seed_perturb"] for r in batch["per_run"]] == list(range(S, S + K))
    for entry in batch["per_run"]:
        seed = entry["seed"]
        single = str(tmp_path / f"single_{seed}.txt")
        r = simrun.run(exe=eng, est=single, seed_meas=seed, seed_perturb=seed, **kw)
        assert _read(single) == _read(out / f"est_{seed}.txt"), f"seed {seed}: the concurrent run differs from the run alone"
        assert entry["status_hist"] == r["status_hist"] and entry["frames"] == r["frames"] == 100
        for k in ("calib_nerr_first", "calib_nerr_last"):  # the single run prints 12 significant digits
            assert entry[k] == pytest.approx(r[k], rel=1e-11)
    p = np.array([r["ate_pos_m"] for r in batch["per_run"]])
    assert len(set(p.tolist())) == K and np.all(p < 0.3)
