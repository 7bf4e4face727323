"""ovb_slam_update on batches of more than 64 state variables and wider than 512 columns, each in ONE call, against the
oracle's single dense EKFUpdate over the same batch (UpdaterSLAM::update, update/UpdaterSLAM.cpp:253-479). Batches wider than
512 columns are split into column groups and applied as sequential EKF updates at one linearization point. Batches of more
than 64 variables need ovb_set_slam_unbounded(ctx, 1); a default context refuses them with OVB_ERR_CAPACITY."""
import os
import sys

import numpy as np
import pytest

from open_vins_b200 import capi, sim

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_fullsize as mf  # noqa: E402

pytestmark = pytest.mark.gpu

REPS = [capi.REP_GLOBAL_3D, capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH,
        capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE]
CALIB = dict(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)


def _frame_cols(case):
    fr = case.frame
    return 6 * fr.n_clones + sum(6 for o in fr.cam_ext_off if o >= 0) + sum(8 for o in fr.cam_intr_off if o >= 0)


def _check(eng, oracle, case, opts, P=None):
    P = case.P if P is None else P
    ref = oracle.slam_update(case.frame, case.feats, case.landmarks, opts, P)
    st, out, dx, stats = eng.slam_update(case.frame, case.feats, case.landmarks, opts)
    assert st == ref["status"] == 0
    assert np.array_equal(out.status, ref["out"].status)
    ok = ref["out"].status == 0
    np.testing.assert_allclose(out.chi2[ok], ref["out"].chi2[ok], rtol=1e-8)
    assert stats.n_feats_used == ref["stats"].n_feats_used
    assert stats.rows_stacked == ref["stats"].rows_stacked and stats.cols_stacked == ref["stats"].cols_stacked
    Pg = eng.cov_get()
    assert np.linalg.norm(Pg - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * max(np.linalg.norm(ref["dx"]), 1e-300)
    assert np.array_equal(Pg, Pg.T)
    return ref, out, stats


@pytest.mark.parametrize("order", [capi.COLS_REFERENCE_FIRST_SEEN, capi.COLS_CANONICAL])
def test_config4_100_landmarks_one_call(oracle, order):
    """SURVEY.md config 4 with max_slam_in_update = 100: 31 clones + 8 calibration blocks + 100 landmarks = 139 variables,
    242 + 300 = 542 columns (two column groups)."""
    case = sim.make_slam_case(**mf.SLAM4)
    assert _frame_cols(case) + 300 == 542
    opts = capi.default_opts(feat_rep=mf.SLAM4["rep"], **CALIB, col_order=order)
    eng = capi.Engine(max_state=640, max_feats=256, max_meas=16384)
    eng.set_slam_unbounded()
    eng.cov_set(case.P)
    ref, out, stats = _check(eng, oracle, case, opts)
    assert stats.n_feats_used >= 80
    eng.close()


@pytest.mark.parametrize("rep", REPS)
def test_window_8x48_25_landmarks(oracle, rep):
    """The full 8-camera, 48-clone window with calibration (64 frame variables, 400 columns) and 25 landmarks: 89 variables
    in one column group (475 columns, 425 for the 1-wide SINGLE landmarks)."""
    case = sim.make_slam_case(n_landmarks=25, n_clones=48, n_cams=8, seed=30 + rep, rep=rep)
    assert _frame_cols(case) == 400
    opts = capi.default_opts(feat_rep=rep, **CALIB)
    eng = capi.Engine(max_state=640, max_feats=64, max_meas=8192)
    eng.set_slam_unbounded()
    eng.cov_set(case.P)
    _check(eng, oracle, case, opts)
    eng.close()


@pytest.mark.parametrize("rep", [capi.REP_GLOBAL_3D, capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE])
def test_long_window_many_landmarks(oracle, rep):
    """48 clone poses, 2 calibrated cameras (316 frame columns) and 150 landmarks: three column groups for the 3-wide
    representations (766 columns), one for SINGLE (466 columns)."""
    case = sim.make_slam_case(n_landmarks=150, n_clones=48, n_cams=2, seed=40 + rep, rep=rep)
    assert _frame_cols(case) == 316
    opts = capi.default_opts(feat_rep=rep, **CALIB)
    eng = capi.Engine(max_state=1024, max_feats=256, max_meas=8192)
    eng.set_slam_unbounded()
    eng.cov_set(case.P)
    _check(eng, oracle, case, opts)
    eng.close()


def test_gate_across_groups(oracle):
    """Gross errors on landmarks of different column groups are rejected exactly as the oracle rejects them: every gate
    sees the prior P, not one already updated by an earlier group."""
    case = sim.make_slam_case(**mf.SLAM4)
    lm = case.landmarks
    val = lm.value.copy()
    bad = [3, 41, 95]  # groups of 90 landmarks: 0, 0, 1
    val[bad] += np.array([0.8, -0.6, 0.9])
    case.landmarks = capi.LandmarkArrays(lm.lm_off, val, lm.value_fej, lm.anchor_cam, lm.anchor_clone, lm.sigma_pix, lm.chi2_multipler)
    opts = capi.default_opts(feat_rep=mf.SLAM4["rep"], **CALIB, col_order=capi.COLS_CANONICAL)
    eng = capi.Engine(max_state=640, max_feats=256, max_meas=16384)
    eng.set_slam_unbounded()
    eng.cov_set(case.P)
    ref, out, stats = _check(eng, oracle, case, opts)
    assert (out.status[bad] == capi.FEAT_CHI2).all()
    eng.close()


def test_msckf_then_100_landmarks_on_the_resident_covariance(oracle):
    """VioManager order (core/VioManager.cpp:525-547): an MSCKF update, then one SLAM update of 100 landmarks (two column
    groups) on the covariance the MSCKF update left on the device."""
    rep = capi.REP_GLOBAL_3D
    sl = sim.make_slam_case(n_landmarks=100, n_clones=31, n_cams=4, seed=4, rep=rep)
    ms = sim.make_update_case(n_feats=200, n_clones=31, n_cams=4, seed=4, calib_ext=True, calib_intr=True)
    assert np.array_equal(ms.frame.clone_R, sl.frame.clone_R)
    opts = capi.default_opts(feat_rep=rep, **CALIB, col_order=capi.COLS_CANONICAL)
    eng = capi.Engine(max_state=640, max_feats=256, max_meas=32768)
    eng.set_slam_unbounded()
    eng.cov_set(sl.P)
    st, out, dx, stats = eng.msckf_update(ms.frame, ms.feats, opts)
    r1 = oracle.msckf_update(ms.frame, ms.feats, opts, sl.P, dumps=False)
    assert st == 0 and np.array_equal(out.status, r1["out"].status)
    _check(eng, oracle, sl, opts, P=r1["P"])
    eng.close()


def test_config4_window_65_variables_in_one_call(oracle):
    """Config 4's window (4 cameras, 31 clone poses, tracks of up to 124 measurements: the per-feature innovation is
    245 x 245 and lives in the kernel's global-memory scratch instead of shared memory) with online calibration, then a
    SLAM update of 25 landmarks (31 + 8 + 25 = 64 state variables), then one of 26 (65 variables: refused by a default
    context, one update with ovb_set_slam_unbounded). Oracle parity at a feature count the CPU restatement finishes in about a second."""
    ms = sim.make_update_case(n_feats=40, n_clones=31, n_cams=4, seed=4, calib_ext=True, calib_intr=True)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, col_order=capi.COLS_CANONICAL)
    assert int((ms.feats.meas_off[1:] - ms.feats.meas_off[:-1]).max()) == 124
    eng = capi.Engine(max_state=384, max_feats=256, max_meas=8192)
    eng.set_slam_unbounded()
    eng.cov_set(ms.P)
    st, out, dx, stats = eng.msckf_update(ms.frame, ms.feats, opts)
    ref = oracle.msckf_update(ms.frame, ms.feats, opts, ms.P, dumps=False)
    assert st == ref["status"] == 0 and np.array_equal(out.status, ref["out"].status) and stats.n_feats_used > 30
    ok = ref["out"].status == 0
    np.testing.assert_allclose(out.chi2[ok], ref["out"].chi2[ok], rtol=1e-8)
    assert np.linalg.norm(eng.cov_get() - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * np.linalg.norm(ref["dx"])
    sl = sim.make_slam_case(n_landmarks=25, n_clones=31, n_cams=4, seed=4, rep=capi.REP_GLOBAL_3D)
    eng.cov_set(sl.P)
    st, out, dx, stats = eng.slam_update(sl.frame, sl.feats, sl.landmarks, opts)
    ref = oracle.slam_update(sl.frame, sl.feats, sl.landmarks, opts, sl.P)
    assert st == ref["status"] == 0 and np.array_equal(out.status, ref["out"].status) and stats.n_feats_used > 15
    assert stats.cols_stacked == ref["stats"].cols_stacked
    assert np.linalg.norm(eng.cov_get() - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * np.linalg.norm(ref["dx"])
    # one landmark more: 65 variables in one call, the same single update as the oracle's
    sl2 = sim.make_slam_case(n_landmarks=26, n_clones=31, n_cams=4, seed=4, rep=capi.REP_GLOBAL_3D)
    eng2 = capi.Engine(max_state=384, max_feats=256, max_meas=8192)
    eng2.set_slam_unbounded()
    eng2.cov_set(sl2.P)
    _check(eng2, oracle, sl2, opts)
    eng.close()
    eng2.close()


def test_default_context_keeps_the_64_variable_limit():
    """without ovb_set_slam_unbounded a batch of more than 64 variables is refused, as before; the same context takes it
    once the switch is on"""
    case = sim.make_slam_case(**mf.SLAM4)
    opts = capi.default_opts(feat_rep=mf.SLAM4["rep"], **CALIB, col_order=capi.COLS_CANONICAL)
    eng = capi.Engine(max_state=640, max_feats=256, max_meas=16384)
    eng.cov_set(case.P)
    with pytest.raises(capi.OvbError) as ei:
        eng.slam_update(case.frame, case.feats, case.landmarks, opts)
    assert ei.value.code == capi.OVB_ERR_CAPACITY
    assert np.array_equal(eng.cov_get(), case.P)
    eng.set_slam_unbounded()
    st, out, dx, stats = eng.slam_update(case.frame, case.feats, case.landmarks, opts)
    assert st == 0 and stats.n_feats_used >= 80
    eng.set_slam_unbounded(False)
    eng.cov_set(case.P)
    with pytest.raises(capi.OvbError):
        eng.slam_update(case.frame, case.feats, case.landmarks, opts)
    eng.close()
