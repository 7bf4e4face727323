"""ovb_slam_delayed_init on the device (UpdaterSLAM::delayed_init, update/UpdaterSLAM.cpp:61-251) against the oracle
composition of test_gpu_slam.py::test_delayed_init_one_call: triangulation, stage-0 Jacobians in each feature's
representation, (SINGLE: bearing projection), StateHelper::initialize with its gate, the caller's mean update between the
features. Every representation, calibration and FEJ on and off, 1 / 2 / 4 cameras, gate rejections and triangulation
failures, and tracks on the BIG (124 measurements) and long-track (384) layouts."""
import numpy as np
import pytest

from open_vins_b200 import capi, sim
from tests import oracle_reps
from tests.test_gpu_slam import _apply_dx_to_frame

pytestmark = pytest.mark.gpu

SINGLE = capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE
REPS = [capi.REP_GLOBAL_3D, capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH,
        capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, SINGLE]


def _oracle_composition(oracle, case, opts, reps, sp, cm):
    fr = case.frame
    tri, _ = oracle.triangulate(fr, case.feats, opts)
    P = case.P.copy()
    log, status = [], tri.status.copy()
    cols = []
    for off, sz in sorted([(int(x), 6) for x in fr.clone_off] + [(int(x), 6) for x in fr.cam_ext_off if x >= 0] +
                          [(int(x), 8) for x in fr.cam_intr_off if x >= 0]):
        cols += list(range(off, off + sz))
    cols = np.array(cols)
    for f in np.flatnonzero(tri.status == 0):
        one = case.feats.subset([f])
        o = capi.FeatOut(1)
        o.status[:] = 0
        o.p_FinA[0], o.p_FinG[0] = tri.p_FinA[f], tri.p_FinG[f]
        o.anchor_cam[0], o.anchor_clone[0] = tri.anchor_cam[f], tri.anchor_clone[f]
        opts_f = capi.default_opts(feat_rep=reps[f], do_calib_camera_pose=opts.do_calib_camera_pose,
                                   do_calib_camera_intrinsics=opts.do_calib_camera_intrinsics, do_fej=opts.do_fej)
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
            log.append((int(f), P.shape[0] - H_L.shape[1], dxn, dx))
            _apply_dx_to_frame(fr, dx)
        else:
            status[f] = capi.FEAT_CHI2
    return status, log, P


def _run(oracle, kw, calib=True, fej=1, rep=capi.REP_GLOBAL_3D, sigma_of=lambda f: 1.0, mult_of=lambda f: 1.0, min_init=1,
         max_state=256):
    case_g, case_o = sim.make_update_case(**kw), sim.make_update_case(**kw)
    F = case_g.feats.n_feats
    reps = [rep] * F
    sp, cm = np.array([sigma_of(f) for f in range(F)]), np.array([mult_of(f) for f in range(F)])
    opts = capi.default_opts(do_calib_camera_pose=int(calib), do_calib_camera_intrinsics=int(calib), do_fej=fej, feat_rep=rep)
    N0 = case_g.P.shape[0]
    eng = capi.Engine(max_state=max_state, max_feats=64, max_meas=64 * 400)
    eng.cov_set(case_g.P)
    log_g = []

    def on_init(f, lm_off, dx_new, dx):
        log_g.append((f, lm_off, dx_new, dx))
        _apply_dx_to_frame(case_g.frame, dx)
    out_g, lm_off = eng.slam_delayed_init(case_g.frame, case_g.feats, opts, on_init, sigma_pix=sp, chi2_multipler=cm, feat_rep=reps)
    status_o, log_o, P = _oracle_composition(oracle, case_o, opts, reps, sp, cm)
    assert np.array_equal(out_g.status, status_o)
    assert np.array_equal(out_g.status == capi.FEAT_OK, lm_off >= 0)
    assert len(log_g) == len(log_o) >= min_init
    w = 1 if rep == SINGLE else 3
    n_dx = N0
    for (fg, og, dng, dg), (fo, oo, dno, do) in zip(log_g, log_o):
        n_dx += w
        assert fg == fo and og == oo == lm_off[fg] and len(dng) == w and len(dg) == n_dx
        assert np.linalg.norm(dng - dno) <= 1e-8 * max(np.linalg.norm(dno), 1e-12)
        assert np.linalg.norm(dg - do) <= 1e-8 * max(np.linalg.norm(do), 1e-300)
    Pg = eng.cov_get()
    assert Pg.shape == P.shape and eng.cov_dim() == n_dx
    assert np.linalg.norm(Pg - P) <= 1e-9 * np.linalg.norm(P)
    assert np.array_equal(Pg, Pg.T)
    c = eng.last_init_counters()
    assert c["features"] >= len(log_g) and c["syncs"] <= c["features"] + 1
    eng.close()
    return out_g, status_o


@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("calib", [True, False], ids=["calib", "nocalib"])
def test_every_representation(oracle, rep, calib):
    """Uniform representation per call; the FEJ flag and the camera count vary with the case."""
    n_cams = [1, 2, 4][rep % 3]
    kw = dict(n_feats=10, n_clones=8, n_cams=n_cams, seed=31 + rep, calib_ext=calib, calib_intr=calib, outlier_frac=0.0,
              degenerate_frac=0.0)
    _run(oracle, kw, calib=calib, fej=(rep + int(calib)) % 2, rep=rep, min_init=3)


@pytest.mark.parametrize("fej", [0, 1])
@pytest.mark.parametrize("rep", [capi.REP_ANCHORED_3D, SINGLE])
def test_fej_four_cameras(oracle, fej, rep):
    kw = dict(n_feats=10, n_clones=10, n_cams=4, seed=41, calib_ext=True, calib_intr=True, outlier_frac=0.0, degenerate_frac=0.0)
    _run(oracle, kw, fej=fej, rep=rep, min_init=3)


@pytest.mark.parametrize("rep,seed", [(capi.REP_GLOBAL_3D, 53), (capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, 56), (SINGLE, 57)])
def test_gate_rejections_and_triangulation_failures(oracle, rep, seed):
    """Outliers and degenerate tracks fail the triangulation; a tight per-feature multiplier on every third feature and a
    second noise class push some of the rest through the gate's rejection branch."""
    kw = dict(n_feats=16, n_clones=8, n_cams=2, seed=seed, calib_ext=True, calib_intr=True, outlier_frac=0.2, degenerate_frac=0.2)
    out, status = _run(oracle, kw, rep=rep, sigma_of=lambda f: 1.5 if f % 2 else 1.0, mult_of=lambda f: 0.02 if f % 3 == 0 else 1.0)
    assert (status == capi.FEAT_CHI2).any()
    assert ((status != capi.FEAT_OK) & (status != capi.FEAT_CHI2)).any()


@pytest.mark.parametrize("rep", [capi.REP_ANCHORED_FULL_INVERSE_DEPTH, SINGLE])
def test_big_tracks_config4(oracle, rep):
    """Full tracks of 4 cameras x 31 clone poses: 124 measurements, the BIG layout."""
    kw = dict(n_feats=5, n_clones=31, n_cams=4, seed=61, full_track_frac=1.0, calib_ext=True, calib_intr=True, outlier_frac=0.0,
              degenerate_frac=0.0)
    _run(oracle, kw, rep=rep, max_state=640)


@pytest.mark.parametrize("rep", [capi.REP_GLOBAL_3D, SINGLE])
def test_long_tracks_8x48(oracle, rep):
    """Full tracks of 8 cameras x 48 clone poses: 384 measurements, the long-track layout."""
    kw = dict(n_feats=3, n_clones=48, n_cams=8, seed=62, full_track_frac=1.0, calib_ext=True, calib_intr=True, outlier_frac=0.0,
              degenerate_frac=0.0)
    case = sim.make_update_case(**kw)
    assert int(np.diff(case.feats.meas_off).max()) > 256
    _run(oracle, kw, rep=rep, max_state=640)


@pytest.mark.parametrize("rep", [capi.REP_ANCHORED_3D, SINGLE])
def test_all_gated_leaves_P_bitwise(rep):
    """A call whose features all fail the gate changes nothing: P bitwise, its size, no callback, no landmark offsets."""
    case = sim.make_update_case(n_feats=10, n_clones=8, n_cams=2, seed=71, calib_ext=True, calib_intr=True, outlier_frac=0.0,
                                degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, feat_rep=rep)
    eng = capi.Engine(max_state=256, max_feats=64, max_meas=2048)
    eng.cov_set(case.P)
    calls = []
    out, lm_off = eng.slam_delayed_init(case.frame, case.feats, opts, lambda *a: calls.append(a),
                                        chi2_multipler=np.full(case.feats.n_feats, 1e-12))
    assert not calls and (lm_off == -1).all()
    assert (out.status == capi.FEAT_CHI2).sum() >= 5 and not (out.status == capi.FEAT_OK).any()
    assert eng.cov_dim() == case.P.shape[0]
    assert eng.cov_get().tobytes() == np.ascontiguousarray(case.P).tobytes()
    eng.close()


def test_counters_one_sync_per_feature_and_no_dump():
    """One stream synchronisation per processed feature beyond the triangulation's, and a read-back per feature of at most
    the correction (N0 + k doubles) plus a small head: no Jacobian dump crosses the bus."""
    case = sim.make_update_case(n_feats=12, n_clones=31, n_cams=4, seed=81, full_track_frac=1.0, calib_ext=True, calib_intr=True,
                                outlier_frac=0.0, degenerate_frac=0.0)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
    eng = capi.Engine(max_state=640, max_feats=64, max_meas=64 * 400)
    eng.cov_set(case.P)
    sizes = []

    def on_init(f, lm_off, dx_new, dx):
        sizes.append(len(dx))
        _apply_dx_to_frame(case.frame, dx)
    out, _ = eng.slam_delayed_init(case.frame, case.feats, opts, on_init)
    c = eng.last_init_counters()
    F = case.feats.n_feats
    assert c["features"] >= len(sizes) >= 3
    assert c["syncs"] <= c["features"] + 1
    tri_bytes = 256 * F  # the triangulation's per-feature records
    N = eng.cov_dim()
    assert c["d2h_bytes"] <= tri_bytes + c["features"] * (8 * N + 256)
    rows = 2 * int(np.diff(case.feats.meas_off).min())
    assert c["d2h_bytes"] < rows * 516 * 8
    eng.close()
