"""rpng_sim-like synthetic update cases (inputs only).

The reference's Simulator (ov_msckf/src/sim/Simulator.cpp) + BsplineSE3 are "next" rows of SURVEY.md §8f and are not
restated yet; this generator produces update cases with the rpng_sim calibration and noise defaults
(config/rpng_sim/kalibr_imucam_chain.yaml, estimator_config.yaml: 10 Hz camera, feature depth U[5,7] m, sigma_px 1,
radtan 752x480 cameras, descending camera visit order of a GCC-built reference, SURVEY.md App. A.4) on a smooth
analytic trajectory, so that the oracle and the CUDA path consume byte-identical inputs. It is the `data: synthetic`
of bench.py.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from .capi import FeatArrays, FrameArrays

# config/rpng_sim/kalibr_imucam_chain.yaml (T_imu_cam = [R_CtoI, p_CinI]); cams 0..3 (4..7: _cam_extrinsic)
_T_IMU_CAM = [
    [[0.0148655429818, -0.999880929698, 0.00414029679422, -0.0216401454975],
     [0.999557249008, 0.0149672133247, 0.025715529948, -0.064676986768],
     [-0.0257744366974, 0.00375618835797, 0.999660727178, 0.00981073058949]],
    [[0.0125552670891, -0.999755099723, 0.0182237714554, -0.0198435579556],
     [0.999598781151, 0.0130119051815, 0.0251588363115, 0.0453689425024],
     [-0.0253898008918, 0.0179005838253, 0.999517347078, 0.00786212447038]],
    [[0.0148655429818, -0.999880929698, 0.00414029679422, -0.0216401454975],
     [0.999557249008, 0.0149672133247, 0.025715529948, 0.124676986768],
     [-0.0257744366974, 0.00375618835797, 0.999660727178, 0.00981073058949]],
    [[0.0125552670891, -0.999755099723, 0.0182237714554, -0.0198435579556],
     [0.999598781151, 0.0130119051815, 0.0251588363115, 0.2253689425024],
     [-0.0253898008918, 0.0179005838253, 0.999517347078, 0.00786212447038]],
]
_INTR = [
    [458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05],
    [457.587, 456.134, 379.999, 255.238, -0.28368365, 0.07451284, -0.00010473, -3.55590700e-05],
    [458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05],
    [457.587, 456.134, 379.999, 255.238, -0.28368365, 0.07451284, -0.00010473, -3.55590700e-05],
]
def _cam_extrinsic(k):
    """T_imu_cam of camera k: cameras 0..3 are the rpng_sim chain; cameras 4..7 repeat cameras 0..3 on a second rig
    level, 0.3 m below and yawed by 5 degrees about the IMU z axis (deterministic, no random draws: the generated cases
    of n_cams <= 4 stay bit-identical)."""
    T = np.array(_T_IMU_CAM[k % 4])
    if k < 4:
        return T
    Rz = exp_so3(np.array([0.0, 0.0, np.deg2rad(5.0)]))
    return np.hstack([Rz @ T[:, :3], (Rz @ T[:, 3] + np.array([0.0, 0.0, -0.3]))[:, None]])


# a mild equidistant set for the fisheye model tests
_INTR_EQUI = [190.978, 190.973, 254.93, 256.897, 0.0034, 0.0007, -0.0020, 0.0002]


def skew(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0.0]])


def exp_so3(w):
    th = np.linalg.norm(w)
    K = skew(w)
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * K @ K


def _orthonormalize(R):
    U, _, Vt = np.linalg.svd(R)
    return U @ Vt


def distort(model, intr, xn, yn):
    """double-precision camera model (no float casts): generator side only."""
    fx, fy, cx, cy, k1, k2, k3, k4 = intr
    if model == 0:
        r2 = xn * xn + yn * yn
        r4 = r2 * r2
        x1 = xn * (1 + k1 * r2 + k2 * r4) + 2 * k3 * xn * yn + k4 * (r2 + 2 * xn * xn)
        y1 = yn * (1 + k1 * r2 + k2 * r4) + k3 * (r2 + 2 * yn * yn) + 2 * k4 * xn * yn
    else:
        r = np.sqrt(xn * xn + yn * yn)
        th = np.arctan(r)
        thd = th + k1 * th**3 + k2 * th**5 + k3 * th**7 + k4 * th**9
        c = thd / r if r > 1e-8 else 1.0
        x1, y1 = xn * c, yn * c
    return fx * x1 + cx, fy * y1 + cy


def undistort(model, intr, u, v, iters=30):
    """Newton inverse of `distort` to ~1e-13 (stands in for cv::undistortPoints in TrackSIM, track/TrackSIM.cpp:62)."""
    fx, fy, cx, cy = intr[:4]
    x, y = (u - cx) / fx, (v - cy) / fy
    for _ in range(iters):
        u0, v0 = distort(model, intr, x, y)
        e = np.array([u - u0, v - v0])
        if np.abs(e).max() < 1e-11:
            break
        h = 1e-7
        ux, vx = distort(model, intr, x + h, y)
        uy, vy = distort(model, intr, x, y + h)
        J = np.array([[(ux - u0) / h, (uy - u0) / h], [(vx - v0) / h, (vy - v0) / h]])
        d = np.linalg.solve(J, e)
        x, y = x + d[0], y + d[1]
    return x, y


@dataclass
class StateLayout:
    """Covariance layout following ov_msckf/src/state/State.cpp:34-131: [IMU 15][dw 6, da 6, tg 9, R 3][dt 1]
    [per cam: extrinsics 6, intrinsics 8][clones 6 each, oldest first]."""
    n_cams: int
    n_clones: int
    calib_ext: bool = False
    calib_intr: bool = False
    calib_imu: bool = False
    calib_dt: bool = False
    imu_off: int = 0
    dt_off: int = -1
    cam_ext_off: list = field(default_factory=list)
    cam_intr_off: list = field(default_factory=list)
    clone_off: list = field(default_factory=list)
    N: int = 0

    def __post_init__(self):
        cur = 15
        if self.calib_imu:
            cur += 6 + 6 + 9 + 3
        if self.calib_dt:
            self.dt_off = cur
            cur += 1
        self.cam_ext_off, self.cam_intr_off = [], []
        for _ in range(self.n_cams):
            if self.calib_ext:
                self.cam_ext_off.append(cur)
                cur += 6
            else:
                self.cam_ext_off.append(-1)
            if self.calib_intr:
                self.cam_intr_off.append(cur)
                cur += 8
            else:
                self.cam_intr_off.append(-1)
        self.clone_off = []
        for _ in range(self.n_clones):
            self.clone_off.append(cur)
            cur += 6
        self.N = cur

    def sigmas(self):
        s = np.full(self.N, 1e-3)
        s[0:3] = 2e-3   # q
        s[3:6] = 2e-2   # p
        s[6:9] = 2e-2   # v
        s[9:12] = 1e-3  # bg
        s[12:15] = 5e-3 # ba
        if self.dt_off >= 0:
            s[self.dt_off] = 1e-3
        for k in range(self.n_cams):
            if self.cam_ext_off[k] >= 0:
                s[self.cam_ext_off[k]:self.cam_ext_off[k] + 3] = 1e-3
                s[self.cam_ext_off[k] + 3:self.cam_ext_off[k] + 6] = 2e-3
            if self.cam_intr_off[k] >= 0:
                s[self.cam_intr_off[k]:self.cam_intr_off[k] + 4] = 0.3
                s[self.cam_intr_off[k] + 4:self.cam_intr_off[k] + 8] = 5e-4
        for o in self.clone_off:
            s[o:o + 3] = 2e-3
            s[o + 3:o + 6] = 2e-2
        return s


@dataclass
class UpdateCase:
    layout: StateLayout
    frame: FrameArrays
    feats: FeatArrays
    P: np.ndarray
    p_true: np.ndarray  # [F][3] true feature positions (for sanity checks only)
    meta: dict


def _trajectory(t):
    """smooth IMU pose at time t: ~1 m/s through a corridor-like Lissajous, gentle rotation."""
    p = np.array([3.0 * np.sin(0.35 * t), 2.0 * np.sin(0.23 * t + 0.4), 0.4 * np.sin(0.51 * t) + 1.2])
    yaw = 0.5 * np.sin(0.21 * t) + 0.15 * t
    pitch = 0.10 * np.sin(0.33 * t + 1.0)
    roll = 0.08 * np.sin(0.27 * t + 0.3)
    R_ItoG = exp_so3(np.array([0, 0, yaw])) @ exp_so3(np.array([0, pitch, 0])) @ exp_so3(np.array([roll, 0, 0]))
    return R_ItoG.T, p  # R_GtoI, p_IinG


def make_update_case(n_feats=50, n_clones=12, n_cams=1, seed=0, calib_ext=False, calib_intr=False, calib_imu=False,
                     calib_dt=False, full_track_frac=0.5, min_track=5, outlier_frac=0.04, degenerate_frac=0.02,
                     sigma_px=1.0, cam_model=0, cam_order="descending", t0=3.0, dt_cam=0.1, depth=(5.0, 7.0),
                     mono_frac=0.0) -> UpdateCase:
    """One MSCKF update's worth of inputs: window of `n_clones` clone poses (the reference holds max_clones+1 during
    the update, SURVEY.md §3.2), `n_feats` feature tracks, prior covariance P and a state estimate drawn from it."""
    rng = np.random.default_rng(seed)
    lay = StateLayout(n_cams, n_clones, calib_ext, calib_intr, calib_imu, calib_dt)
    N = lay.N
    # ---- truth
    R_true, p_true = [], []
    for c in range(n_clones):
        R, p = _trajectory(t0 + dt_cam * c)
        R_true.append(R)
        p_true.append(p)
    R_true, p_true = np.array(R_true), np.array(p_true)
    if not 1 <= n_cams <= 8:
        raise ValueError(f"n_cams={n_cams}: the generator has 8 cameras")
    camR_true = np.array([_cam_extrinsic(k)[:, :3].T for k in range(n_cams)])  # R_ItoC = R_CtoI'
    camp_true = np.array([-camR_true[k] @ _cam_extrinsic(k)[:, 3] for k in range(n_cams)])  # p_IinC
    intr_true = np.array([_INTR[k % 4] if cam_model == 0 else _INTR_EQUI for k in range(n_cams)], dtype=np.float64)
    # ---- prior covariance: D (0.6 I + 0.4 U U'/k) D, SPD with cross-correlations
    sig = lay.sigmas()
    k = 12
    U = rng.standard_normal((N, k))
    Cn = 0.6 * np.eye(N) + 0.4 * (U @ U.T) / k
    P = (sig[:, None] * Cn) * sig[None, :]
    P = 0.5 * (P + P.T)
    # ---- estimate = truth (+) error ~ N(0,P)
    Lc = np.linalg.cholesky(P)
    err = Lc @ rng.standard_normal(N)
    R_est, p_est = [], []
    for c in range(n_clones):
        o = lay.clone_off[c]
        R_est.append(exp_so3(err[o:o + 3]) @ R_true[c])  # JPL: R_true = (I - [dth x]) R_est
        p_est.append(p_true[c] - err[o + 3:o + 6])
    R_est, p_est = np.array(R_est), np.array(p_est)
    # FEJ = estimate with a small extra perturbation (first estimates differ from current ones after updates)
    R_fej = np.array([exp_so3(-2e-4 * rng.standard_normal(3)) @ R_est[c] for c in range(n_clones)])
    p_fej = p_est + 2e-3 * rng.standard_normal(p_est.shape)
    # the newest clone was just appended: its FEJ equals its value (StateHelper::clone copies the fej)
    R_fej[-1], p_fej[-1] = R_est[-1], p_est[-1]
    camR_est, camp_est, intr_est = camR_true.copy(), camp_true.copy(), intr_true.copy()
    for kk in range(n_cams):
        if calib_ext:
            o = lay.cam_ext_off[kk]
            camR_est[kk] = exp_so3(err[o:o + 3]) @ camR_true[kk]
            camp_est[kk] = camp_true[kk] - err[o + 3:o + 6]
        if calib_intr:
            o = lay.cam_intr_off[kk]
            intr_est[kk] = intr_true[kk] - err[o:o + 8]
    R_est = np.array([_orthonormalize(R) for R in R_est])
    R_fej = np.array([_orthonormalize(R) for R in R_fej])
    camR_est = np.array([_orthonormalize(R) for R in camR_est])
    # ---- features
    meas_off = [0]
    cam_l, clone_l, uv_l, uvn_l, ptrue = [], [], [], [], []
    cams_visit = list(range(n_cams))[::-1] if cam_order == "descending" else list(range(n_cams))
    n_out = 0
    for f in range(n_feats):
        if rng.random() < full_track_frac:
            s, e = 0, n_clones - 1
        else:
            L = int(rng.integers(min_track, n_clones + 1))
            e = int(rng.integers(L - 1, n_clones))
            s = e - L + 1
        degenerate = rng.random() < degenerate_frac
        if degenerate:  # two-view track: tiny baseline, exercises the triangulation / baseline rejections
            e = min(s + 1, n_clones - 1)
            s = e - 1
        # point in front of camera 0 at the middle clone of the track
        cm = (s + e) // 2
        z = rng.uniform(*depth)
        un, vn = rng.uniform(-0.45, 0.45), rng.uniform(-0.30, 0.30)
        p_c = np.array([un * z, vn * z, z])
        R_GtoC = camR_true[0] @ R_true[cm]
        p_CinG = p_true[cm] - R_GtoC.T @ camp_true[0]
        pf = R_GtoC.T @ p_c + p_CinG
        ptrue.append(pf)
        outlier = rng.random() < outlier_frac
        mono = rng.random() < mono_frac
        cnt = 0
        for cam in cams_visit:
            if mono and cam != 0:
                continue
            for c in range(s, e + 1):
                pc = camR_true[cam] @ (R_true[c] @ (pf - p_true[c])) + camp_true[cam]
                if pc[2] < 0.2:
                    continue
                u, v = distort(cam_model, intr_true[cam], pc[0] / pc[2], pc[1] / pc[2])
                u += sigma_px * rng.standard_normal()
                v += sigma_px * rng.standard_normal()
                if outlier and c == s + (e - s) // 3:
                    u += 25.0
                    v -= 18.0
                uf, vf = np.float32(u), np.float32(v)
                xn, yn = undistort(cam_model, intr_est[cam], float(uf), float(vf))
                cam_l.append(cam)
                clone_l.append(c)
                uv_l.append((uf, vf))
                uvn_l.append((np.float32(xn), np.float32(yn)))
                cnt += 1
        n_out += int(outlier)
        meas_off.append(meas_off[-1] + cnt)
    frame = FrameArrays(R_est, p_est, R_fej, p_fej, lay.clone_off, camR_est, camp_est, intr_est,
                        [cam_model] * n_cams, lay.cam_ext_off, lay.cam_intr_off)
    feats = FeatArrays(meas_off, cam_l, clone_l, np.array(uv_l, dtype=np.float32).reshape(-1, 2),
                       np.array(uvn_l, dtype=np.float32).reshape(-1, 2))
    meta = dict(n_feats=n_feats, n_clones=n_clones, n_cams=n_cams, seed=seed, N=N, n_meas=int(meas_off[-1]),
                outliers=n_out, calib_ext=calib_ext, calib_intr=calib_intr)
    return UpdateCase(lay, frame, feats, P, np.array(ptrue), meta)


@dataclass
class SlamCase:
    frame: FrameArrays
    feats: FeatArrays
    landmarks: "LandmarkArrays"
    P: np.ndarray
    lm_off: np.ndarray
    meta: dict


def make_slam_case(n_landmarks=12, n_clones=8, n_cams=2, seed=0, rep=0, calib_ext=True, calib_intr=True, track_len=(1, 4),
                   two_classes=True) -> SlamCase:
    """One UpdaterSLAM::update batch: `n_landmarks` landmarks already in the state (3-wide variables appended after the
    clone window, as State::_variables does), each observed in the newest 1..4 clones; prior P over the augmented state.
    rep: ovb_feat_rep of all landmarks (global or anchored; the anchor is camera 0 at the track's oldest clone), or a sequence of
    one representation per landmark (widths, offsets, prior sigmas and anchors then follow each landmark)."""
    from .capi import LandmarkArrays
    rng = np.random.default_rng(seed)
    base = make_update_case(n_feats=n_landmarks, n_clones=n_clones, n_cams=n_cams, seed=seed, calib_ext=calib_ext, calib_intr=calib_intr,
                            full_track_frac=1.0, outlier_frac=0.0, degenerate_frac=0.0)
    lay, fr = base.layout, base.frame
    N0 = lay.N
    reps = [int(rep)] * n_landmarks if np.ndim(rep) == 0 else [int(r) for r in rep]
    assert len(reps) == n_landmarks
    lm_size = np.array([1 if r == 5 else 3 for r in reps])  # ANCHORED_INVERSE_DEPTH_SINGLE keeps only the inverse depth in the state
    N = N0 + int(lm_size.sum())
    lm_off = N0 + np.concatenate([[0], np.cumsum(lm_size)[:-1]]).astype(np.int64)
    sig = np.concatenate([lay.sigmas()] + [(0.01 if r == 5 else 0.05) * np.ones(w) for r, w in zip(reps, lm_size)])
    U = rng.standard_normal((N, 12))
    Cn = 0.6 * np.eye(N) + 0.4 * (U @ U.T) / 12
    P = (sig[:, None] * Cn) * sig[None, :]
    P = 0.5 * (P + P.T)
    # keep only the newest `track_len` clones of every track (SLAM features are updated as they are re-observed)
    fa = base.feats
    keep, meas_off = [], [0]
    first_clone = []
    for f in range(n_landmarks):
        L = int(rng.integers(max(track_len[0], 2 if reps[f] == 5 else 1), track_len[1] + 1))
        idx = [i for i in range(fa.meas_off[f], fa.meas_off[f + 1]) if fa.clone[i] >= n_clones - L]
        keep += idx
        meas_off.append(meas_off[-1] + len(idx))
        first_clone.append(n_clones - L)
    keep = np.array(keep, dtype=np.int64)
    feats = FeatArrays(meas_off, fa.cam[keep], fa.clone[keep], fa.uv[keep], fa.uvn[keep])
    # landmark estimates: truth minus an error of the prior's size; FEJ value = estimate + a small offset
    p_est = base.p_true - 0.03 * rng.standard_normal(base.p_true.shape)
    p_fej = p_est + 2e-3 * rng.standard_normal(p_est.shape)
    anchor_cam = np.full(n_landmarks, -1, dtype=np.int32)
    anchor_clone = np.full(n_landmarks, -1, dtype=np.int32)
    value, value_fej = p_est.copy(), p_fej.copy()
    for f in range(n_landmarks):
        if reps[f] in (2, 3, 4, 5):  # anchored
            c = first_clone[f]
            anchor_cam[f], anchor_clone[f] = 0, c
            to_anchor = lambda pG: fr.cam_R[0] @ (fr.clone_R[c] @ (pG - fr.clone_p[c])) + fr.cam_p[0]
            value[f], value_fej[f] = to_anchor(p_est[f]), to_anchor(p_fej[f])
    sigma_pix = chi2_mult = None
    if two_classes:  # the first third plays the "aruco" class with its own noise / gate (UpdaterSLAM.cpp:391-393, :407-408)
        sigma_pix = np.where(np.arange(n_landmarks) < n_landmarks // 3, 1.5, 1.0)
        chi2_mult = np.where(np.arange(n_landmarks) < n_landmarks // 3, 2.0, 1.0)
    lms = LandmarkArrays(lm_off, value, value_fej, anchor_cam, anchor_clone, sigma_pix, chi2_mult)
    return SlamCase(fr, feats, lms, P, lm_off, dict(N=N, N0=N0, rep=rep, n_landmarks=n_landmarks))


def make_compress_case(m=8000, n=500, seed=0, structured=False):
    """config 5 (SURVEY.md §8d): H m x n, res, SPD P = A A'/n + 1e-4 I."""
    rng = np.random.default_rng(seed)
    if not structured:
        H = rng.standard_normal((m, n))
    else:
        H = np.zeros((m, n))
        ngroups = n // 6
        r = 0
        while r < m:
            rows = min(81, m - r)
            g = rng.choice(ngroups, size=min(21, ngroups), replace=False)
            for gi in g:
                H[r:r + rows, 6 * gi:6 * gi + 6] = rng.standard_normal((rows, 6))
            r += rows
    res = rng.standard_normal(m)
    A = rng.standard_normal((n, n))
    P = A @ A.T / n + 1e-4 * np.eye(n)
    return H, res, 0.5 * (P + P.T)
