"""Per-landmark representations in one SLAM batch (UpdaterSLAM::update reads landmark->_feat_representation per landmark):
the oracle's mixed batches, the SINGLE branch of delayed_init, and make_slam_case with one representation per landmark."""
import numpy as np
import pytest
import scipy.linalg

from open_vins_b200 import capi, sim
from tests import oracle_reps

REPS = [capi.REP_GLOBAL_3D, capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH,
        capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE]
CALIB = dict(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, col_order=capi.COLS_CANONICAL)


def _feature_blocks(r, feats, N):
    """{feature: its rows of the stacked system as dense rows over the covariance (and their residuals)}, accepted features
    in batch order; a SINGLE landmark has 2M-2 rows, the others 2M."""
    cols = np.concatenate([np.arange(o, o + s) for o, s in zip(r["order_off"], r["order_sz"])])
    H = np.zeros((r["H_big"].shape[0], N))
    H[:, cols] = r["H_big"]
    return H, r["res_big"]


def _split(H, res, feats, status, widths):
    out, row = {}, 0
    for f in range(feats.n_feats):
        if status[f] != 0:
            continue
        m = 2 * (feats.meas_off[f + 1] - feats.meas_off[f]) - (2 if widths[f] == 1 else 0)
        out[f] = (H[row:row + m], res[row:row + m])
        row += m
    assert row == H.shape[0]
    return out


def test_mixed_batch_rows_equal_uniform_batches(oracle):
    """Every landmark of a batch cycling through the six representations gets, block for block, the rows (and chi²) it gets in
    a uniform batch of its own representation over the same landmarks."""
    n = 18
    reps = [REPS[i % 6] for i in range(n)]
    case = sim.make_slam_case(n_landmarks=n, n_clones=8, n_cams=2, seed=71, rep=reps)
    N = case.P.shape[0]
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D, **CALIB)
    mixed = oracle_reps.slam_update(case.frame, case.feats, case.landmarks, opts, case.P, feat_rep=reps)
    assert mixed["status"] == 0 and (mixed["out"].status == 0).sum() >= 12
    widths = [1 if r == capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE else 3 for r in reps]
    H, res = _feature_blocks(mixed, case.feats, N)
    blocks = _split(H, res, case.feats, mixed["out"].status, widths)
    lm = case.landmarks
    for k in REPS:
        idx = [f for f in range(n) if reps[f] == k]
        sub = capi.LandmarkArrays(lm.lm_off[idx], lm.value[idx], lm.value_fej[idx], lm.anchor_cam[idx], lm.anchor_clone[idx],
                                  lm.sigma_pix[idx], lm.chi2_multipler[idx])
        feats = case.feats.subset(idx)
        uni = oracle.slam_update(case.frame, feats, sub, capi.default_opts(feat_rep=k, **CALIB), case.P)
        assert np.array_equal(uni["out"].status, mixed["out"].status[idx])
        assert np.array_equal(uni["out"].chi2, mixed["out"].chi2[idx], equal_nan=True)
        Hu, ru = _feature_blocks(uni, feats, N)
        ub = _split(Hu, ru, feats, uni["out"].status, [widths[f] for f in idx])
        for j, f in enumerate(idx):
            if f in blocks:
                assert np.array_equal(ub[j][0], blocks[f][0]) and np.array_equal(ub[j][1], blocks[f][1])


def test_single_init_system_projection(oracle):
    """ovo_slam_single_init_system (the SINGLE branch of UpdaterSLAM::delayed_init): the two bearing columns are annihilated,
    and the projected normal equations equal those of an orthonormal basis of their left nullspace."""
    rng = np.random.default_rng(5)
    rows, n = 14, 20
    Hf, Hx, res = rng.standard_normal((rows, 3)), rng.standard_normal((rows, n)), rng.standard_normal(rows)
    H_R, h_L, r = oracle_reps.slam_single_init_system(Hf, Hx, res)
    assert H_R.shape == (rows - 2, n) and h_L.shape == (rows - 2, 1) and r.shape == (rows - 2,)
    # the bearing columns, carried along as two more state columns, come out as zero
    H_R2, _, _ = oracle_reps.slam_single_init_system(Hf, np.hstack([Hx, Hf[:, :2]]), res)
    assert np.abs(H_R2[:, n:]).max() <= 1e-12 * np.abs(Hf).max()
    Q2 = scipy.linalg.null_space(Hf[:, :2].T)
    A = Q2.T @ np.column_stack([Hx, Hf[:, 2], res])
    B = np.column_stack([H_R, h_L, r])
    assert np.linalg.norm(B.T @ B - A.T @ A) <= 1e-12 * np.linalg.norm(A.T @ A)


def test_single_init_system_too_few_rows(oracle):
    with pytest.raises(ValueError):
        oracle_reps.slam_single_init_system(np.ones((2, 3)), np.ones((2, 4)), np.ones(2))


@pytest.mark.parametrize("rep", REPS)
def test_make_slam_case_rep_sequence(rep):
    """One representation per landmark, all equal, is the int form byte for byte (same RNG draws)."""
    a = sim.make_slam_case(n_landmarks=9, n_clones=6, n_cams=2, seed=3, rep=rep)
    b = sim.make_slam_case(n_landmarks=9, n_clones=6, n_cams=2, seed=3, rep=[rep] * 9)
    assert a.P.tobytes() == b.P.tobytes() and a.lm_off.tobytes() == b.lm_off.tobytes() and a.lm_off.dtype == b.lm_off.dtype
    for k in ("meas_off", "cam", "clone", "uv", "uvn"):
        assert getattr(a.feats, k).tobytes() == getattr(b.feats, k).tobytes()
    for k in ("lm_off", "value", "value_fej", "anchor_cam", "anchor_clone", "sigma_pix", "chi2_multipler"):
        assert getattr(a.landmarks, k).tobytes() == getattr(b.landmarks, k).tobytes()


def test_make_slam_case_mixed_layout():
    reps = [capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE, capi.REP_GLOBAL_3D, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE]
    c = sim.make_slam_case(n_landmarks=4, n_clones=6, n_cams=2, seed=2, rep=reps)
    N0 = c.meta["N0"]
    assert list(c.lm_off) == [N0, N0 + 1, N0 + 4, N0 + 7] and c.P.shape[0] == N0 + 8
    assert list(c.landmarks.anchor_cam >= 0) == [True, False, True, True]
    M = c.feats.meas_off[1:] - c.feats.meas_off[:-1]
    assert M[0] >= 2 and M[3] >= 2
