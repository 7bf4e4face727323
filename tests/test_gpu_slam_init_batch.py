"""ovb_slam_delayed_init_batch: the delayed initialisation with the frame moved on the device between the landmarks, against
ovb_slam_delayed_init_reps with a callback that applies the same mean update (VioManager::apply_dx: JPLQuat::update of the
clone and extrinsic quaternions, R = quat_2_Rot(q), additive positions and intrinsics) and hands the frame back. The two
must agree bit for bit: P, N, statuses, chi2, landmark offsets, dx_new and every dx row. The host side of the mean update
below restates include/ovb200_math.hpp operation for operation (Python floats round every product and sum on their own,
as the library's unit does)."""
import ctypes as C
import math

import numpy as np
import pytest

from open_vins_b200 import capi, sim

pytestmark = pytest.mark.gpu

SINGLE = capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE
REPS = [capi.REP_GLOBAL_3D, capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH,
        capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, SINGLE]


# ---- include/ovb200_math.hpp, operation for operation
def _skew(w):
    return [0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0]


def _normalize(t):
    if t[3] < 0:
        t = [-v for v in t]
    n = math.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2] + t[3] * t[3])
    return [v / n for v in t]


def quat_2_Rot(q):
    v = q[:3]
    a, b = 2 * q[3] * q[3] - 1, 2 * q[3]
    S = _skew(v)
    E = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    return [(a * E[3 * i + j] - b * S[3 * i + j]) + 2.0 * (v[i] * v[j]) for i in range(3) for j in range(3)]


def quat_multiply(q, p):
    S = _skew(q[:3])
    t = [(q[3] * float(i == 0) - S[3 * i]) * p[0] + (q[3] * float(i == 1) - S[3 * i + 1]) * p[1] + (q[3] * float(i == 2) - S[3 * i + 2]) * p[2]
         + q[i] * p[3] for i in range(3)]
    t.append(-q[0] * p[0] - q[1] * p[1] - q[2] * p[2] + q[3] * p[3])
    return _normalize(t)


def jpl_update(q, d):
    return quat_multiply(_normalize([.5 * d[0], .5 * d[1], .5 * d[2], 1.0]), q)


def rot_2_quat(R):
    """A unit JPL quaternion of R (quat_ops.h:88-133); the frame's R is then recomputed from it with quat_2_Rot."""
    T = R[0] + R[4] + R[8]
    if R[0] >= T and R[0] >= R[4] and R[0] >= R[8]:
        x = math.sqrt((1 + 2 * R[0] - T) / 4)
        q = [x, (R[1] + R[3]) / (4 * x), (R[2] + R[6]) / (4 * x), (R[5] - R[7]) / (4 * x)]
    elif R[4] >= T and R[4] >= R[0] and R[4] >= R[8]:
        y = math.sqrt((1 + 2 * R[4] - T) / 4)
        q = [(R[1] + R[3]) / (4 * y), y, (R[5] + R[7]) / (4 * y), (R[6] - R[2]) / (4 * y)]
    elif R[8] >= T and R[8] >= R[0] and R[8] >= R[4]:
        z = math.sqrt((1 + 2 * R[8] - T) / 4)
        q = [(R[2] + R[6]) / (4 * z), (R[5] + R[7]) / (4 * z), z, (R[1] - R[3]) / (4 * z)]
    else:
        w = math.sqrt((1 + T) / 4)
        q = [(R[5] - R[7]) / (4 * w), (R[6] - R[2]) / (4 * w), (R[1] - R[3]) / (4 * w), w]
    return _normalize(q)


class MovingFrame:
    """A case's frame with the quaternions behind its rotations; move(dx) is VioManager::apply_dx on the frame's variables."""

    def __init__(self, case, opts):
        self.fr, self.opts = case.frame, opts
        cR, kR = self.fr.clone_R.reshape(-1, 9), self.fr.cam_R.reshape(-1, 9)
        self.cq = [rot_2_quat(list(cR[c])) for c in range(self.fr.n_clones)]
        self.kq = [rot_2_quat(list(kR[k])) for k in range(self.fr.n_cams)]
        for c, q in enumerate(self.cq):
            cR[c] = quat_2_Rot(q)
        for k, q in enumerate(self.kq):
            kR[k] = quat_2_Rot(q)

    def quats(self):
        return np.array(self.cq), np.array(self.kq)

    def move(self, dx):
        cR, cp = self.fr.clone_R.reshape(-1, 9), self.fr.clone_p.reshape(-1, 3)
        for c, o in enumerate(int(x) for x in self.fr.clone_off):
            self.cq[c] = jpl_update(self.cq[c], dx[o:o + 3])
            cR[c] = quat_2_Rot(self.cq[c])
            cp[c] = [float(cp[c][j]) + float(dx[o + 3 + j]) for j in range(3)]
        kR, kp, ki = self.fr.cam_R.reshape(-1, 9), self.fr.cam_p.reshape(-1, 3), self.fr.cam_intr.reshape(-1, 8)
        for k in range(self.fr.n_cams):
            if self.opts.do_calib_camera_pose:
                o = int(self.fr.cam_ext_off[k])
                self.kq[k] = jpl_update(self.kq[k], dx[o:o + 3])
                kR[k] = quat_2_Rot(self.kq[k])
                kp[k] = [float(kp[k][j]) + float(dx[o + 3 + j]) for j in range(3)]
            if self.opts.do_calib_camera_intrinsics:
                o = int(self.fr.cam_intr_off[k])
                ki[k] = [float(ki[k][j]) + float(dx[o + j]) for j in range(8)]


def _compare(kw, opts, reps=None, sp=None, cm=None, max_state=256, min_init=1):
    """The callback path and the batch path from the same prior; returns the batch's results."""
    F = sim.make_update_case(**kw).feats.n_feats
    reps = reps if reps is not None else [opts.feat_rep] * F
    eng = capi.Engine(max_state=max_state, max_feats=max(F, 64), max_meas=max(F, 64) * 400)
    # callback path
    case_a = sim.make_update_case(**kw)
    mf_a = MovingFrame(case_a, opts)
    eng.cov_set(case_a.P)
    log = {}

    def on_init(f, lm_off, dx_new, dx):
        log[f] = (lm_off, dx_new, dx)
        mf_a.move(dx)
    out_a, lm_a = eng.slam_delayed_init(case_a.frame, case_a.feats, opts, on_init, sigma_pix=sp, chi2_multipler=cm, feat_rep=reps)
    P_a, N_a = eng.cov_get(), eng.cov_dim()
    # batch path
    case_b = sim.make_update_case(**kw)
    mf_b = MovingFrame(case_b, opts)
    eng.cov_set(case_b.P)
    cq, kq = mf_b.quats()
    out_b, lm_b, dxn_b, dx_b = eng.slam_delayed_init_batch(case_b.frame, cq, kq, case_b.feats, opts, sigma_pix=sp, chi2_multipler=cm, feat_rep=reps)
    P_b, N_b = eng.cov_get(), eng.cov_dim()
    counters = eng.last_init_counters()
    eng.close()
    assert np.array_equal(out_a.status, out_b.status) and np.array_equal(lm_a, lm_b)
    assert out_a.chi2.tobytes() == out_b.chi2.tobytes()
    for k in ("p_FinA", "p_FinG", "anchor_cam", "anchor_clone"):
        assert getattr(out_a, k).tobytes() == getattr(out_b, k).tobytes(), k
    assert sorted(log) == [int(f) for f in np.flatnonzero(lm_b >= 0)] and len(log) >= min_init
    for f, (lm_off, dx_new, dx) in log.items():
        w = 1 if reps[f] == SINGLE else 3
        assert lm_off == lm_b[f] and len(dx_new) == w and len(dx) == lm_off + w
        assert dx_new.tobytes() == dxn_b[f, :w].tobytes() and dx.tobytes() == dx_b[f, :lm_off + w].tobytes()
    assert np.isnan(dx_b[lm_b < 0]).all() and np.isnan(dxn_b[lm_b < 0]).all()
    assert N_a == N_b and P_a.tobytes() == P_b.tobytes()
    assert counters["syncs"] <= 2
    return out_b, lm_b, counters


@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("calib", [True, False], ids=["calib", "nocalib"])
def test_every_representation(rep, calib):
    """Uniform representation per call; FEJ and the camera count vary with the case."""
    kw = dict(n_feats=10, n_clones=8, n_cams=[1, 2, 4][rep % 3], seed=31 + rep, calib_ext=calib, calib_intr=calib, outlier_frac=0.0,
              degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=int(calib), do_calib_camera_intrinsics=int(calib), do_fej=(rep + int(calib)) % 2, feat_rep=rep)
    _compare(kw, opts, min_init=3)


@pytest.mark.parametrize("fej", [0, 1])
@pytest.mark.parametrize("cam_model", [0, 1], ids=["radtan", "equi"])
def test_fej_and_camera_models(fej, cam_model):
    kw = dict(n_feats=10, n_clones=10, n_cams=4, seed=41 + cam_model, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0,
              cam_model=cam_model)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, do_fej=fej, feat_rep=capi.REP_ANCHORED_3D)
    _compare(kw, opts, min_init=3)


@pytest.mark.parametrize("rep,seed", [(capi.REP_GLOBAL_3D, 53), (capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, 56), (SINGLE, 57)])
def test_gate_rejections_and_triangulation_failures(rep, seed):
    """Outliers and degenerate tracks fail the triangulation; a tight multiplier on every third feature and a second noise
    class send some of the rest through the gate's rejection, between accepted landmarks."""
    kw = dict(n_feats=16, n_clones=8, n_cams=2, seed=seed, calib_ext=True, calib_intr=True, outlier_frac=0.2, degenerate_frac=0.2)
    F = sim.make_update_case(**kw).feats.n_feats
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, feat_rep=rep)
    sp = np.array([1.5 if f % 2 else 1.0 for f in range(F)])
    cm = np.array([0.02 if f % 3 == 0 else 1.0 for f in range(F)])
    out, lm_off, _ = _compare(kw, opts, sp=sp, cm=cm)
    assert (out.status == capi.FEAT_CHI2).any() and ((out.status != capi.FEAT_OK) & (out.status != capi.FEAT_CHI2)).any()
    assert (out.status == capi.FEAT_OK).any()


def test_class_mix_of_3wide_representations():
    kw = dict(n_feats=10, n_clones=8, n_cams=2, seed=24, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
    reps = [capi.REP_GLOBAL_3D if f < 3 else capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH for f in range(10)]
    _compare(kw, opts, reps=reps, sp=np.array([1.5] * 3 + [1.0] * 7), cm=np.array([2.0] * 3 + [1.0] * 7), min_init=3)


@pytest.mark.parametrize("rep", [capi.REP_ANCHORED_3D, SINGLE])
def test_nothing_accepted_leaves_P_bitwise(rep):
    case = sim.make_update_case(n_feats=10, n_clones=8, n_cams=2, seed=71, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, feat_rep=rep)
    mf = MovingFrame(case, opts)
    eng = capi.Engine(max_state=256, max_feats=64, max_meas=2048)
    eng.cov_set(case.P)
    out, lm_off, dx_new, dx = eng.slam_delayed_init_batch(case.frame, *mf.quats(), case.feats, opts,
                                                          chi2_multipler=np.full(case.feats.n_feats, 1e-12))
    assert (lm_off == -1).all() and (out.status == capi.FEAT_CHI2).sum() >= 5 and np.isnan(dx).all()
    assert eng.cov_dim() == case.P.shape[0] and eng.cov_get().tobytes() == np.ascontiguousarray(case.P).tobytes()
    assert eng.last_init_counters()["syncs"] == 2
    eng.close()


@pytest.mark.parametrize("rep", [capi.REP_GLOBAL_3D, SINGLE])
def test_long_tracks_8x48(rep):
    """Full tracks of 8 cameras x 48 clone poses: 384 measurements, the long-track layout."""
    kw = dict(n_feats=3, n_clones=48, n_cams=8, seed=62, full_track_frac=1.0, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    assert int(np.diff(sim.make_update_case(**kw).feats.meas_off).max()) == 384
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, feat_rep=rep)
    _compare(kw, opts, max_state=640, min_init=1)


@pytest.mark.parametrize("n_feats", [1, 25, 100])
def test_two_synchronisations(n_feats):
    """The triangulation's read-back and the final one, whatever the number of landmarks."""
    kw = dict(n_feats=n_feats, n_clones=11, n_cams=2, seed=90 + n_feats, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
    _, lm_off, c = _compare(kw, opts, max_state=640)
    assert c["syncs"] == 2 and c["features"] >= (lm_off >= 0).sum() >= min(n_feats, 10) // 2


def test_refusals_leave_P():
    """The refusals of ovb_slam_delayed_init_reps, a NULL quaternion array, a short ld_dx and a covariance without room for
    every triangulated landmark: P and N stay."""
    case = sim.make_update_case(n_feats=6, n_clones=8, n_cams=2, seed=25, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
    mf = MovingFrame(case, opts)
    N = case.P.shape[0]
    P0 = np.ascontiguousarray(case.P).tobytes()

    def unchanged(eng):
        return eng.cov_dim() == N and eng.cov_get().tobytes() == P0
    eng = capi.Engine(max_state=256, max_feats=64, max_meas=2048)
    eng.cov_set(case.P)
    for reps in ([SINGLE, 0, SINGLE, SINGLE, SINGLE, SINGLE], [0, 0, 6, 0, 0, 0]):
        with pytest.raises(capi.OvbError) as ei:
            eng.slam_delayed_init_batch(case.frame, *mf.quats(), case.feats, opts, feat_rep=reps)
        assert ei.value.code == capi.OVB_ERR_ARG and unchanged(eng)
    # raw calls: NULL quat, then an ld_dx one short of N + 3 x (triangulated features)
    lib, F = eng.lib, case.feats.n_feats
    tri = eng.triangulate(case.frame, case.feats, opts)
    need = N + 3 * int((tri.status == 0).sum())
    cq, kq = (np.ascontiguousarray(a) for a in mf.quats())
    quat = capi.ovb_frame_quat(cq.ctypes.data_as(capi.c_double_p), kq.ctypes.data_as(capi.c_double_p))
    out, lm = capi.FeatOut(F), np.full(F, -1, dtype=np.int32)
    dxn, dx = np.zeros((F, 3)), np.zeros((F, need))
    args = lambda q, ld: (eng.h, C.byref(case.frame.struct()), q, C.byref(case.feats.struct()), C.byref(opts), None, None, None, C.byref(out.struct()),
                          lm.ctypes.data_as(capi.c_int_p), dxn.ctypes.data_as(capi.c_double_p), dx.ctypes.data_as(capi.c_double_p), ld)
    assert lib.ovb_slam_delayed_init_batch(*args(None, need)) == capi.OVB_ERR_ARG and unchanged(eng)
    assert lib.ovb_slam_delayed_init_batch(*args(C.byref(quat), need - 1)) == capi.OVB_ERR_ARG and unchanged(eng)
    assert lib.ovb_slam_delayed_init_batch(*args(C.byref(quat), need)) == capi.OVB_OK and eng.cov_dim() > N
    eng.close()
    # room for fewer landmarks than were triangulated
    eng = capi.Engine(max_state=N + 5, max_feats=64, max_meas=2048)
    eng.cov_set(case.P)
    with pytest.raises(capi.OvbError) as ei:
        eng.slam_delayed_init_batch(case.frame, *mf.quats(), case.feats, opts)
    assert ei.value.code == capi.OVB_ERR_CAPACITY and unchanged(eng)
    eng.close()
