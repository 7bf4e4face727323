"""CPU tests for feature tracks longer than 128 measurements: the 8-camera generator and the oracle on a full
8-camera x 48-clone track (384 measurements) against the numpy twin."""
import numpy as np
import pytest

from open_vins_b200 import capi, sim
from tests import np_twin


@pytest.mark.parametrize("n_cams", [5, 6, 7, 8])
def test_generator_up_to_eight_cameras(n_cams):
    n_clones = 48
    case = sim.make_update_case(n_feats=8, n_clones=n_clones, n_cams=n_cams, seed=3, full_track_frac=1.0, outlier_frac=0.0,
                                degenerate_frac=0.0)
    fr = case.frame
    R = fr.cam_R.reshape(n_cams, 3, 3)
    for k in range(n_cams):
        assert np.allclose(R[k] @ R[k].T, np.eye(3), atol=1e-12) and abs(np.linalg.det(R[k]) - 1.0) < 1e-12
    for a in range(n_cams):
        for b in range(a):
            assert np.abs(R[a] - R[b]).max() > 1e-3 or np.abs(fr.cam_p[a] - fr.cam_p[b]).max() > 1e-3
    M = np.diff(case.feats.meas_off)
    assert M.max() == n_cams * n_clones
    assert (M == n_cams * n_clones).mean() >= 0.5
    # measurements grouped by camera, descending visit order, every (camera, clone) pair once
    f = int(np.argmax(M))
    m0, m1 = case.feats.meas_off[f], case.feats.meas_off[f + 1]
    cams, clones = case.feats.cam[m0:m1], case.feats.clone[m0:m1]
    assert list(dict.fromkeys(cams.tolist())) == list(range(n_cams))[::-1]
    assert len(set(zip(cams.tolist(), clones.tolist()))) == m1 - m0
    sl = sim.make_slam_case(n_landmarks=6, n_clones=40, n_cams=n_cams, seed=4, track_len=(36, 40))
    Ms = np.diff(sl.feats.meas_off)
    assert Ms.max() > 128 and Ms.max() <= n_cams * 40
    assert sl.frame.cam_R.reshape(-1, 9).shape[0] == n_cams


def test_generator_rejects_nine_cameras():
    with pytest.raises(ValueError):
        sim.make_update_case(n_feats=2, n_clones=4, n_cams=9)


def test_oracle_on_384_measurement_tracks_against_twin(oracle):
    case = sim.make_update_case(n_feats=6, n_clones=48, n_cams=8, seed=11, full_track_frac=1.0, outlier_frac=0.0, degenerate_frac=0.0)
    M = np.diff(case.feats.meas_off)
    assert M.max() == 384
    opts = capi.default_opts(refine_features=0)
    out, _ = oracle.triangulate(case.frame, case.feats, opts)
    ok = np.flatnonzero(out.status == capi.FEAT_OK)
    assert len(ok) >= 4 and M[ok].max() == 384
    for f in ok:
        pA, pG, cond = np_twin.triangulate_linear(case.frame, case.feats, f, out.anchor_cam[f], out.anchor_clone[f])
        assert np.linalg.norm(out.p_FinA[f] - pA) <= 1e-11 * cond * np.linalg.norm(pA)
        assert np.linalg.norm(out.p_FinG[f] - pG) <= 1e-11 * cond * np.linalg.norm(pG)
    # pre-nullspace residuals of every measurement = measured pixel - projection of the triangulated point
    cols = np.arange(case.layout.N)
    _, _, res, row_off = oracle.feature_jacobians(case.frame, case.feats, opts, out.copy(), 0, cols)
    for f in ok:
        m0, m1 = case.feats.meas_off[f], case.feats.meas_off[f + 1]
        pred = np.concatenate([np_twin.project(case.frame, int(case.feats.cam[i]), int(case.feats.clone[i]), out.p_FinG[f]) for i in range(m0, m1)])
        meas = case.feats.uv[m0:m1].astype(np.float64).reshape(-1)
        got = res[row_off[f]:row_off[f + 1]]
        assert got.shape == (2 * (m1 - m0),)
        assert np.abs(got - (meas - pred)).max() <= 1e-4  # the projection rounds the normalised point to float32 (reference)
