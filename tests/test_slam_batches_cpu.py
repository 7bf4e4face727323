"""The algebra behind ovb_slam_update's column groups: a SLAM batch wider than the engine's 512-column systems is cut into
contiguous feature ranges, each range's whitened rows [H_g | r_g] are compressed by QR to [R_g | z_g], and the groups are
applied as sequential EKF updates with the innovation corrected by the state change so far, z_g - R_g dx_acc. For one
linearization point this equals the joint update over all rows (information form: the per-group terms add up)."""
import numpy as np


def _ekf(P, H, r):
    S = H @ P @ H.T + np.eye(H.shape[0])
    K = P @ H.T @ np.linalg.inv(S)
    return P - K @ H @ P, K @ r


def _block_arrow(rng, n_frame=40, n_lm=30, lmw=3, rows_per=(2, 8)):
    """frame columns (shared by every feature) followed by one lmw-wide landmark block per feature; whitened rows"""
    N = n_frame + n_lm * lmw + 7  # 7 state columns no feature touches
    A = rng.standard_normal((N, N))
    P = A @ A.T / N + 0.1 * np.eye(N)
    Hs, rs, feats = [], [], []
    for f in range(n_lm):
        m = int(rng.integers(rows_per[0], rows_per[1] + 1))
        H = np.zeros((m, N))
        used = rng.choice(n_frame, size=12, replace=False)
        H[:, used] = rng.standard_normal((m, 12))
        o = n_frame + lmw * f
        H[:, o:o + lmw] = rng.standard_normal((m, lmw))
        Hs.append(H)
        rs.append(rng.standard_normal(m))
        feats.append(o)
    return P, Hs, rs, feats, n_frame, lmw


def _grouped(P, Hs, rs, feats, n_frame, lmw, per):
    N = P.shape[0]
    dx_acc = np.zeros(N)
    for g0 in range(0, len(Hs), per):
        idx = range(g0, min(g0 + per, len(Hs)))
        cols = list(range(n_frame)) + [feats[f] + k for f in idx for k in range(lmw)]
        H = np.vstack([Hs[f][:, cols] for f in idx])
        r = np.concatenate([rs[f] for f in idx])
        R = np.linalg.qr(np.hstack([H, r[:, None]]), mode="r")  # compress: [R_g | z_g]
        n = len(cols)
        k = min(R.shape[0], n)
        Rg, zg = R[:k, :n], R[:k, n]
        zg = zg - Rg @ dx_acc[cols]  # innovation at the mean already moved by the earlier groups
        Hg = np.zeros((k, N))
        Hg[:, cols] = Rg
        P, dx = _ekf(P, Hg, zg)
        dx_acc = dx_acc + dx
    return P, dx_acc


def test_sequential_groups_equal_the_joint_update():
    rng = np.random.default_rng(11)
    P0, Hs, rs, feats, n_frame, lmw = _block_arrow(rng)
    Pj, dxj = _ekf(P0, np.vstack(Hs), np.concatenate(rs))
    for per in (30, 11, 7, 1):
        Pg, dxg = _grouped(P0, Hs, rs, feats, n_frame, lmw, per)
        assert np.linalg.norm(Pg - Pj) <= 1e-12 * np.linalg.norm(Pj)
        assert np.linalg.norm(dxg - dxj) <= 1e-12 * np.linalg.norm(dxj)


def test_without_the_correction_the_groups_differ():
    """the innovation correction is what makes the groups exact: leaving it out moves dx by far more than rounding"""
    rng = np.random.default_rng(12)
    P0, Hs, rs, feats, n_frame, lmw = _block_arrow(rng, lmw=1)
    Pj, dxj = _ekf(P0, np.vstack(Hs), np.concatenate(rs))
    Pg, dxg = _grouped(P0, Hs, rs, feats, n_frame, lmw, 9)
    assert np.linalg.norm(dxg - dxj) <= 1e-12 * np.linalg.norm(dxj)
    N = P0.shape[0]
    P, dx_naive = P0, np.zeros(N)
    for g0 in range(0, len(Hs), 9):
        idx = range(g0, min(g0 + 9, len(Hs)))
        P, dx = _ekf(P, np.vstack([Hs[f] for f in idx]), np.concatenate([rs[f] for f in idx]))
        dx_naive += dx
    assert np.linalg.norm(dx_naive - dxj) > 1e-3 * np.linalg.norm(dxj)
