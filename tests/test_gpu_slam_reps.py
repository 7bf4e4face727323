"""ovb_slam_update_reps / ovb_slam_delayed_init_reps: every SLAM landmark in its own representation (UpdaterSLAM::update reads
landmark->_feat_representation per landmark; delayed_init picks feat_rep_aruco or feat_rep_slam per feature), against the
oracle with the bars of test_gpu_slam.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

from open_vins_b200 import build, capi, sim
from tests import oracle_reps

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_fullsize as mf  # noqa: E402

pytestmark = pytest.mark.gpu

REPS = [capi.REP_GLOBAL_3D, capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH,
        capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE]
SINGLE = capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE
CALIB = dict(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)


def _check(eng, oracle, case, opts, reps):
    ref = oracle_reps.slam_update(case.frame, case.feats, case.landmarks, opts, case.P, feat_rep=reps)
    eng.cov_set(case.P)
    st, out, dx, stats = eng.slam_update(case.frame, case.feats, case.landmarks, opts, feat_rep=reps)
    assert st == ref["status"] == 0
    assert np.array_equal(out.status, ref["out"].status)
    ok = ref["out"].status == 0
    np.testing.assert_allclose(out.chi2[ok], ref["out"].chi2[ok], rtol=1e-8)
    assert stats.n_feats_used == ref["stats"].n_feats_used and stats.rows_stacked == ref["stats"].rows_stacked
    assert stats.cols_stacked == ref["stats"].cols_stacked
    Pg = eng.cov_get()
    assert np.linalg.norm(Pg - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * max(np.linalg.norm(ref["dx"]), 1e-300)
    assert np.array_equal(Pg, Pg.T)
    return ref, out, stats


@pytest.mark.parametrize("n", [14, 24])
@pytest.mark.parametrize("order", [capi.COLS_REFERENCE_FIRST_SEEN, capi.COLS_CANONICAL])
def test_mixed_batch(oracle, n, order):
    """All six representations cycled over the landmarks of one batch, 2 calibrated cameras."""
    reps = [REPS[(i + n) % 6] for i in range(n)]
    case = sim.make_slam_case(n_landmarks=n, n_clones=8, n_cams=2, seed=80 + n, rep=reps)
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D, col_order=order, **CALIB)
    eng = capi.Engine(max_state=256, max_feats=256, max_meas=4096)
    ref, out, stats = _check(eng, oracle, case, opts, reps)
    assert stats.n_feats_used >= n // 2
    eng.close()


def test_aruco_single_and_slam_classes(oracle):
    """ArUco landmarks (the first third: own sigma_pix 1.5 and gate multiplier 2) in ANCHORED_INVERSE_DEPTH_SINGLE next to SLAM
    landmarks in ANCHORED_MSCKF_INVERSE_DEPTH."""
    n = 18
    reps = [SINGLE if i < n // 3 else capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH for i in range(n)]
    case = sim.make_slam_case(n_landmarks=n, n_clones=8, n_cams=2, seed=91, rep=reps, two_classes=True)
    opts = capi.default_opts(feat_rep=capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, col_order=capi.COLS_REFERENCE_FIRST_SEEN, **CALIB)
    eng = capi.Engine(max_state=256, max_feats=256, max_meas=4096)
    ref, out, stats = _check(eng, oracle, case, opts, reps)
    assert (out.status[:n // 3] == 0).sum() >= 3 and stats.n_feats_used >= n // 2
    eng.close()


def test_config4_100_mixed_widths_two_groups(oracle):
    """Config 4 with 100 landmarks, every tenth in the 1-wide SINGLE: 242 frame + 280 landmark columns, two column groups."""
    n = mf.SLAM4["n_landmarks"]
    reps = [SINGLE if i % 10 == 3 else REPS[i % 5] for i in range(n)]
    case = sim.make_slam_case(**{**mf.SLAM4, "rep": reps})
    assert 242 + sum(1 if r == SINGLE else 3 for r in reps) > 512
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D, col_order=capi.COLS_CANONICAL, **CALIB)
    eng = capi.Engine(max_state=640, max_feats=256, max_meas=16384)
    eng.set_slam_unbounded()
    ref, out, stats = _check(eng, oracle, case, opts, reps)
    assert stats.n_feats_used >= 80
    eng.close()


def test_long_tracks_8x48_mixed(oracle):
    """8 cameras x 48 clone poses, tracks of up to 8 x 22 measurements (the long-track path of the per-feature kernel), SINGLE
    next to 3-wide landmarks."""
    reps = [SINGLE, capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_GLOBAL_3D, SINGLE]
    case = sim.make_slam_case(n_landmarks=len(reps), n_clones=48, n_cams=8, seed=12, rep=reps, track_len=(18, 22))
    assert (case.feats.meas_off[1:] - case.feats.meas_off[:-1]).max() > 128
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D, **CALIB)
    eng = capi.Engine(max_state=640, max_feats=64, max_meas=64 * 400)
    eng.set_slam_unbounded()
    ref, out, stats = _check(eng, oracle, case, opts, reps)
    assert stats.n_feats_used >= 2
    eng.close()


@pytest.mark.parametrize("rep", REPS)
def test_uniform_reps_equal_opts_rep(rep):
    """feat_rep = [rep] * F computes byte for byte what feat_rep = NULL (ovb_opts.feat_rep = rep) computes."""
    case = sim.make_slam_case(n_landmarks=14, n_clones=8, n_cams=2, seed=60 + rep, rep=rep)
    opts = capi.default_opts(feat_rep=rep, **CALIB)
    eng = capi.Engine(max_state=256, max_feats=256, max_meas=4096)
    res = []
    for reps in (None, [rep] * case.feats.n_feats):
        eng.cov_set(case.P)
        st, out, dx, stats = eng.slam_update(case.frame, case.feats, case.landmarks, opts, feat_rep=reps)
        res.append((st, out.status.copy(), out.chi2.copy(), dx.copy(), eng.cov_get()))
    (s0, st0, c0, d0, P0), (s1, st1, c1, d1, P1) = res
    assert s0 == s1 == 0 and np.array_equal(st0, st1)
    assert c0.tobytes() == c1.tobytes() and d0.tobytes() == d1.tobytes() and P0.tobytes() == P1.tobytes()
    eng.close()


def test_argument_errors_leave_P():
    """An entry outside 0..5, an anchored landmark without an anchor, and landmark blocks that overlap with their own widths are
    argument errors; P keeps its prior."""
    eng = capi.Engine(max_state=256, max_feats=64, max_meas=1024)
    glob = sim.make_slam_case(n_landmarks=5, n_clones=5, n_cams=1, seed=1, rep=capi.REP_GLOBAL_3D, calib_ext=False, calib_intr=False)
    single = sim.make_slam_case(n_landmarks=5, n_clones=5, n_cams=1, seed=1, rep=SINGLE, calib_ext=False, calib_intr=False)
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D)
    bad = [(glob, [0, 7, 0, 0, 0]), (glob, [0, -1, 0, 0, 0]), (glob, [0, 0, capi.REP_ANCHORED_3D, 0, 0]),
           (single, [SINGLE, capi.REP_GLOBAL_3D, SINGLE, SINGLE, SINGLE])]
    for case, reps in bad:
        eng.cov_set(case.P)
        with pytest.raises(capi.OvbError) as ei:
            eng.slam_update(case.frame, case.feats, case.landmarks, opts, feat_rep=reps)
        assert ei.value.code == capi.OVB_ERR_ARG
        assert eng.cov_get().tobytes() == np.ascontiguousarray(case.P).tobytes()
    eng.close()


def _apply_dx_to_frame(fr, dx):
    """Host side of StateHelper::EKFUpdate's mean update for the frame's variables (as in test_gpu_slam.py)."""
    for c, o in enumerate(fr.clone_off):
        fr.clone_R[c] = (sim.exp_so3(-dx[o:o + 3]) @ fr.clone_R[c].reshape(3, 3)).reshape(fr.clone_R[c].shape)
        fr.clone_p[c] += dx[o + 3:o + 6]
    for k in range(fr.n_cams):
        o = fr.cam_ext_off[k]
        if o >= 0:
            fr.cam_R[k] = (sim.exp_so3(-dx[o:o + 3]) @ fr.cam_R[k].reshape(3, 3)).reshape(fr.cam_R[k].shape)
            fr.cam_p[k] += dx[o + 3:o + 6]
        o = fr.cam_intr_off[k]
        if o >= 0:
            fr.cam_intr[k] += dx[o:o + 8]


def _delayed_init_vs_oracle(oracle, reps_of, sigma_of, mult_of, seed):
    kw = dict(n_feats=10, n_clones=8, n_cams=2, seed=seed, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    case_g, case_o = sim.make_update_case(**kw), sim.make_update_case(**kw)
    F = case_g.feats.n_feats
    reps = [reps_of(f) for f in range(F)]
    sp, cm = np.array([sigma_of(f) for f in range(F)]), np.array([mult_of(f) for f in range(F)])
    opts = capi.default_opts(**CALIB)
    N0 = case_g.P.shape[0]
    eng = capi.Engine(max_state=256, max_feats=64, max_meas=2048)
    eng.cov_set(case_g.P)
    log_g = []

    def on_init(f, lm_off, dx_new, dx):
        log_g.append((f, lm_off, dx_new, dx))
        _apply_dx_to_frame(case_g.frame, dx)
    out_g, lm_off = eng.slam_delayed_init(case_g.frame, case_g.feats, opts, on_init, sigma_pix=sp, chi2_multipler=cm, feat_rep=reps)
    # ---- oracle composition: triangulate -> stage-0 Jacobians in the feature's representation -> (SINGLE: bearing
    # projection) -> StateHelper::initialize with the feature's width
    fr = case_o.frame
    tri, _ = oracle.triangulate(fr, case_o.feats, opts)
    P = case_o.P.copy()
    log_o, status_o = [], tri.status.copy()
    for f in np.flatnonzero(tri.status == 0):
        one = case_o.feats.subset([f])
        o = capi.FeatOut(1)
        o.status[:] = 0
        o.p_FinA[0], o.p_FinG[0] = tri.p_FinA[f], tri.p_FinG[f]
        o.anchor_cam[0], o.anchor_clone[0] = tri.anchor_cam[f], tri.anchor_clone[f]
        cols = []
        for off, sz in sorted([(int(x), 6) for x in fr.clone_off] + [(int(x), 6) for x in fr.cam_ext_off if x >= 0] + [(int(x), 8) for x in fr.cam_intr_off if x >= 0]):
            cols += list(range(off, off + sz))
        cols = np.array(cols)
        opts_f = capi.default_opts(feat_rep=reps[f], **CALIB)
        Hf, Hx, res, _ = oracle.feature_jacobians(fr, one, opts_f, o, 0, cols)
        used = np.flatnonzero(np.abs(Hx).sum(axis=0) > 0)
        cc = cols[used]
        starts = [0] + [i for i in range(1, len(cc)) if cc[i] != cc[i - 1] + 1] + [len(cc)]
        off = [int(cc[a]) for a in starts[:-1]]
        sz = [int(b - a) for a, b in zip(starts[:-1], starts[1:])]
        H_R, H_L = Hx[:, used], Hf
        if reps[f] == SINGLE:
            H_R, H_L, res = oracle_reps.slam_single_init_system(Hf, Hx[:, used], res)
        st, acc, P, dxn, dx = oracle.cov_initialize(P, off, sz, H_R, H_L, res, sigma2=sp[f] ** 2, chi2_mult=float(cm[f]))
        assert st == 0
        if acc:
            log_o.append((int(f), P.shape[0] - H_L.shape[1], dxn, dx))
            _apply_dx_to_frame(fr, dx)
        else:
            status_o[f] = capi.FEAT_CHI2
    assert np.array_equal(out_g.status, status_o)
    assert len(log_g) == len(log_o) >= 4
    n_dx = N0
    for (fg, og, dng, dg), (fo, oo, dno, do) in zip(log_g, log_o):
        w = 1 if reps[fg] == SINGLE else 3
        n_dx += w
        assert fg == fo and og == oo == lm_off[fg] and len(dng) == w and len(dg) == n_dx
        assert np.linalg.norm(dng - dno) <= 1e-8 * max(np.linalg.norm(dno), 1e-12)
        assert np.linalg.norm(dg - do) <= 1e-8 * max(np.linalg.norm(do), 1e-300)
    assert (lm_off[out_g.status != 0] == -1).all()
    Pg = eng.cov_get()
    assert Pg.shape == P.shape and eng.cov_dim() == n_dx
    assert np.linalg.norm(Pg - P) <= 1e-9 * np.linalg.norm(P)
    eng.close()


def test_delayed_init_single_one_call(oracle):
    """ANCHORED_INVERSE_DEPTH_SINGLE in the one-call delayed init: each accepted landmark adds 1 to the covariance."""
    _delayed_init_vs_oracle(oracle, lambda f: SINGLE, lambda f: 1.0, lambda f: 1.0, seed=23)


def test_delayed_init_class_mix(oracle):
    """Two classes with their own representation, pixel noise and gate multiplier (ArUco: the first three features)."""
    _delayed_init_vs_oracle(oracle, lambda f: capi.REP_GLOBAL_3D if f < 3 else capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH,
                            lambda f: 1.5 if f < 3 else 1.0, lambda f: 2.0 if f < 3 else 1.0, seed=24)


def test_delayed_init_refuses_single_with_3wide():
    """SINGLE mixed with a 3-wide representation in one delayed init, and an entry outside 0..5, are argument errors; P and its
    size stay."""
    case = sim.make_update_case(n_feats=6, n_clones=8, n_cams=2, seed=25, calib_ext=True, calib_intr=True, outlier_frac=0.0,
                                degenerate_frac=0.0)
    opts = capi.default_opts(**CALIB)
    eng = capi.Engine(max_state=256, max_feats=64, max_meas=2048)
    eng.cov_set(case.P)
    for reps in ([SINGLE, 0, SINGLE, SINGLE, SINGLE, SINGLE], [0, 0, 6, 0, 0, 0]):
        with pytest.raises(capi.OvbError) as ei:
            eng.slam_delayed_init(case.frame, case.feats, opts, feat_rep=reps)
        assert ei.value.code == capi.OVB_ERR_ARG
        assert eng.cov_dim() == case.P.shape[0] and eng.cov_get().tobytes() == np.ascontiguousarray(case.P).tobytes()
    eng.close()


def test_host_mirror_two_classes(tmp_path):
    """ovb200::UpdaterSLAM::update (include/ovb200_host.hpp) with ArUco landmarks in SINGLE and SLAM landmarks in
    ANCHORED_MSCKF_INVERSE_DEPTH gives bit for bit the dx and P of the ctypes call with the same per-landmark inputs."""
    n, n_aruco = 12, 4
    reps = [SINGLE if i < n_aruco else capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH for i in range(n)]
    case = sim.make_slam_case(n_landmarks=n, n_clones=6, n_cams=1, seed=44, rep=reps, two_classes=False)
    fr, fb, lm = case.frame, case.feats, case.landmarks
    cls = dict(slam=(1.0, 1.0), aruco=(1.5, 2.0))
    sp = np.array([cls["aruco" if i < n_aruco else "slam"][0] for i in range(n)])
    cm = np.array([cls["aruco" if i < n_aruco else "slam"][1] for i in range(n)])
    lms = capi.LandmarkArrays(lm.lm_off, lm.value, lm.value_fej, lm.anchor_cam, lm.anchor_clone, sp, cm)
    opts = capi.default_opts(do_fej=1, col_order=capi.COLS_CANONICAL, **CALIB)
    eng = capi.Engine(max_state=512, max_feats=256, max_meas=8192)
    eng.cov_set(case.P)
    st, out, dx, stats = eng.slam_update(fr, fb, lms, opts, feat_rep=reps)
    assert st == 0 and stats.n_feats_used >= n // 2
    P_c = eng.cov_get()
    eng.close()
    # ---- the same update through the C++ host mirror
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "slam_reps_host_test")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-Wall", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "slam_reps_host_test.cpp"), "-L", os.path.dirname(build.OUT), "-lovb200",
                           "-Wl,-rpath," + os.path.dirname(build.OUT), "-o", exe])
    C, K, N, F, M = fr.n_clones, fr.n_cams, case.P.shape[0], fb.n_feats, fb.n_meas
    times = 10.0 + 0.5 * np.arange(C)
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32).tobytes()
    f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64).tobytes()
    blob = b"".join([i32([C, K, N, F, M, 1, 1, n_aruco]), f64([cls["slam"][0], cls["slam"][1], cls["aruco"][0], cls["aruco"][1]]), f64(times),
                     f64(fr.clone_R), f64(fr.clone_p), f64(fr.clone_R_fej), f64(fr.clone_p_fej), i32(fr.clone_off), f64(fr.cam_R),
                     f64(fr.cam_p), f64(fr.cam_intr), i32(fr.cam_model), i32(fr.cam_ext_off), i32(fr.cam_intr_off), f64(case.P),
                     i32(fb.meas_off), np.ascontiguousarray(fb.cam, dtype=np.uint8).tobytes(),
                     np.ascontiguousarray(fb.clone, dtype=np.uint16).tobytes(), np.ascontiguousarray(fb.uv, dtype=np.float32).tobytes(),
                     np.ascontiguousarray(fb.uvn, dtype=np.float32).tobytes(), i32(lm.lm_off), i32(reps), i32(lm.anchor_cam),
                     i32(lm.anchor_clone), f64(lm.value), f64(lm.value_fej)])
    (tmp_path / "case.bin").write_bytes(blob)
    subprocess.check_call([exe, str(tmp_path / "case.bin"), str(tmp_path / "out.bin")])
    raw = (tmp_path / "out.bin").read_bytes()
    dx_h = np.frombuffer(raw[:8 * N], dtype=np.float64)
    P_h = np.frombuffer(raw[8 * N:8 * (N + N * N)], dtype=np.float64).reshape(N, N)
    st_h = np.frombuffer(raw[8 * (N + N * N):], dtype=np.int32)
    assert np.array_equal(st_h, out.status)
    assert dx_h.tobytes() == dx.tobytes() and P_h.tobytes() == P_c.tobytes()
