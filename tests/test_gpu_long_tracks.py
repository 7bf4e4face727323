"""Feature tracks longer than 128 measurements (up to OVB_MAX_MEAS_PER_FEAT = 8 cameras x 48 clone poses = 384) on the GPU
against the CPU oracle. Every case asserts that its longest track exceeds 128 measurements.

Bars: gate decisions identical, triangulated points <= 1e-12 relative (bit-identical on >= 99 %), chi2 1e-8, P and dx
<= 1e-9 relative Frobenius, P exactly symmetric.
"""
import numpy as np
import pytest

from open_vins_b200 import capi, sim

pytestmark = pytest.mark.gpu

REPS = [capi.REP_GLOBAL_3D, capi.REP_GLOBAL_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH,
        capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE]
FOUR_CAMS = dict(n_feats=40, n_clones=48, n_cams=4, seed=7, calib_ext=True, calib_intr=True, calib_imu=True, calib_dt=True)
EIGHT_CAMS = dict(n_feats=6, n_clones=48, n_cams=8, seed=11, full_track_frac=1.0, calib_ext=True, calib_intr=True)


@pytest.fixture(scope="module")
def eng():
    e = capi.Engine(max_state=640, max_feats=1024, max_meas=1024 * 64)
    yield e
    e.close()


def _opts(case, **kw):
    return capi.default_opts(do_calib_camera_pose=int(case.meta["calib_ext"]), do_calib_camera_intrinsics=int(case.meta["calib_intr"]), **kw)


def _longest(feats):
    return int(np.diff(feats.meas_off).max())


def _check_update(eng, oracle, case, opts):
    ref = oracle.msckf_update(case.frame, case.feats, opts, case.P, dumps=False)
    eng.cov_set(case.P)
    st, out, dx, stats = eng.msckf_update(case.frame, case.feats, opts)
    P = eng.cov_get()
    assert st == ref["status"] == capi.OVB_OK
    assert np.array_equal(out.status, ref["out"].status)
    ok = ref["out"].status == 0
    assert ok.any()
    rel = np.linalg.norm(out.p_FinG[ok] - ref["out"].p_FinG[ok], axis=1) / np.linalg.norm(ref["out"].p_FinG[ok], axis=1)
    assert rel.max() <= 1e-12
    assert np.all(out.p_FinG[ok] == ref["out"].p_FinG[ok], axis=1).mean() >= 0.99
    seen = np.isfinite(ref["out"].chi2)
    assert np.allclose(out.chi2[seen], ref["out"].chi2[seen], rtol=1e-8, atol=0)
    assert stats.n_feats_used == ref["stats"].n_feats_used and stats.rows_stacked == ref["stats"].rows_stacked
    assert np.linalg.norm(P - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * np.linalg.norm(ref["dx"])
    assert np.array_equal(P, P.T)
    return out, ref


@pytest.mark.parametrize("compress", [capi.COMPRESS_CHOLQR2, capi.COMPRESS_HOUSEHOLDER_TSQR])
@pytest.mark.parametrize("order", [capi.COLS_REFERENCE_FIRST_SEEN, capi.COLS_CANONICAL])
def test_four_cameras_48_clones(eng, oracle, compress, order):
    """4 cameras x 48 clone poses, full calibration: tracks of up to 192 measurements next to short ones."""
    case = sim.make_update_case(**FOUR_CAMS)
    assert _longest(case.feats) > 128
    out, ref = _check_update(eng, oracle, case, _opts(case, compress=compress, col_order=order))
    M = np.diff(case.feats.meas_off)
    assert (ref["out"].status[M > 128] == 0).any()  # long tracks pass the gate and reach the update


@pytest.mark.parametrize("rep", REPS)
def test_eight_cameras_384_measurements(eng, oracle, rep):
    """8 cameras x 48 clone poses, extrinsics + intrinsics calibrated, 6 full tracks of 384 measurements each. The CPU
    oracle takes about 2.5 s for this update (6 features, N = 415)."""
    case = sim.make_update_case(**EIGHT_CAMS)
    assert _longest(case.feats) == 384
    _check_update(eng, oracle, case, _opts(case, feat_rep=rep))


def _mixed_case():
    """A few 384-measurement tracks among a few hundred short ones (mostly single-camera, at most 48 measurements)."""
    case = sim.make_update_case(n_feats=300, n_clones=48, n_cams=8, seed=6, full_track_frac=0.05, mono_frac=0.9, calib_ext=True)
    M = np.diff(case.feats.meas_off)
    assert (M == 384).sum() >= 2 and (M <= 48).sum() >= 250
    return case, M


def test_mixed_batch_routes_each_track(eng, oracle):
    case, M = _mixed_case()
    opts = _opts(case)
    out, _ = _check_update(eng, oracle, case, opts)
    # the short tracks alone give the same per-feature results bit for bit: they run on their own path either way
    short = np.flatnonzero(M <= 128)
    eng.cov_set(case.P)
    st, out_s, _, _ = eng.msckf_update(case.frame, case.feats.subset(short), opts)
    assert st == 0
    assert np.array_equal(out_s.status, out.status[short])
    assert np.array_equal(out_s.p_FinG, out.p_FinG[short], equal_nan=True)
    assert np.array_equal(out_s.chi2, out.chi2[short], equal_nan=True)


def test_feature_jacobians_long_tracks(eng, oracle):
    case = sim.make_update_case(**EIGHT_CAMS)
    assert _longest(case.feats) == 384
    opts = _opts(case)
    eng.cov_set(case.P)
    tri, _ = oracle.triangulate(case.frame, case.feats, opts)
    # stage 0: pre-nullspace rows
    Hf, Hx, res, row_off, cols = eng.feature_jacobians(case.frame, case.feats, opts, tri.copy(), 0)
    Hf_r, Hx_r, res_r, row_off_r = oracle.feature_jacobians(case.frame, case.feats, opts, tri.copy(), 0, cols)
    assert np.array_equal(row_off, row_off_r) and np.array_equal(res, res_r)
    assert np.abs(Hx - Hx_r).max() <= 1e-12 * max(np.abs(Hx_r).max(), 1.0)
    assert np.abs(Hf - Hf_r).max() <= 1e-12 * max(np.abs(Hf_r).max(), 1.0)
    # stage 1: nullspace projection + gate; the projected rows agree on their invariants
    out_g, out_r = tri.copy(), tri.copy()
    _, Hx, res, row_off, cols = eng.feature_jacobians(case.frame, case.feats, opts, out_g, 1)
    _, Hx_r, res_r, row_off_r = oracle.feature_jacobians(case.frame, case.feats, opts, out_r, 1, cols, P=case.P)
    assert np.array_equal(row_off, row_off_r) and np.array_equal(out_g.status, out_r.status)
    seen = np.isfinite(out_r.chi2)
    assert np.allclose(out_g.chi2[seen], out_r.chi2[seen], rtol=1e-8, atol=0)
    for f in range(case.feats.n_feats):
        a, b = row_off[f], row_off[f + 1]
        if out_r.status[f] != 0:
            assert not Hx[a:b].any() and not res[a:b].any()
            continue
        G, Gr = Hx[a:b].T @ Hx[a:b], Hx_r[a:b].T @ Hx_r[a:b]
        assert np.linalg.norm(G - Gr) <= 1e-12 * np.linalg.norm(Gr)
        assert abs(res[a:b] @ res[a:b] - res_r[a:b] @ res_r[a:b]) <= 1e-12 * (res_r[a:b] @ res_r[a:b])


@pytest.mark.parametrize("rep", [capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE])
def test_slam_update_long_tracks(oracle, rep):
    """8 landmarks seen over the newest 36-40 clone poses by 4 cameras (tracks of 144-160 measurements; 40 clones + 8
    calibration blocks + 8 landmarks = 56 state variables, within the per-call limit of 64). SINGLE projects out two
    columns of H_f (two reflectors on up to 320 rows), MSCKF_INVERSE_DEPTH none. The CPU oracle's dense SLAM update
    dominates the run time of this test."""
    case = sim.make_slam_case(n_landmarks=8, n_clones=40, n_cams=4, seed=3, rep=rep, track_len=(36, 40))
    assert _longest(case.feats) > 128
    opts = capi.default_opts(feat_rep=rep, do_calib_camera_pose=1, do_calib_camera_intrinsics=1)
    ref = oracle.slam_update(case.frame, case.feats, case.landmarks, opts, case.P)
    eng = capi.Engine(max_state=640, max_feats=64, max_meas=64 * 400)
    eng.cov_set(case.P)
    st, out, dx, stats = eng.slam_update(case.frame, case.feats, case.landmarks, opts)
    assert st == ref["status"] == 0
    assert np.array_equal(out.status, ref["out"].status)
    ok = ref["out"].status == 0
    assert ok.any()
    np.testing.assert_allclose(out.chi2[ok], ref["out"].chi2[ok], rtol=1e-8)
    Pg = eng.cov_get()
    assert np.linalg.norm(Pg - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * max(np.linalg.norm(ref["dx"]), 1e-300)
    assert np.array_equal(Pg, Pg.T)
    eng.close()


def _apply_dx_to_frame(fr, dx):
    """The caller's mean update between delayed-init features (state/StateHelper.cpp:185-188) for the frame's variables:
    JPL left error on rotations, additive elsewhere; FEJ values stay."""
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


def test_slam_delayed_init_long_tracks(oracle):
    """One ovb_slam_delayed_init call on full tracks of 4 cameras x 40 clone poses (160 measurements) against the same
    sequence composed from the oracle: triangulation, long-track Jacobians, StateHelper::initialize with its gate, and the
    identical mean update between the features. Gate decisions, each appended landmark's correction and the final
    covariance (appended blocks included) must agree."""
    kw = dict(n_feats=6, n_clones=40, n_cams=4, seed=23, full_track_frac=1.0, calib_ext=True, calib_intr=True, outlier_frac=0.0,
              degenerate_frac=0.0)
    case_g, case_o = sim.make_update_case(**kw), sim.make_update_case(**kw)
    assert _longest(case_g.feats) > 128
    opts = _opts(case_g)
    eng = capi.Engine(max_state=640, max_feats=64, max_meas=64 * 400)
    eng.cov_set(case_g.P)
    log_g = []

    def on_init(f, lm_off, dx_new, dx):
        log_g.append((f, lm_off, dx_new, dx))
        _apply_dx_to_frame(case_g.frame, dx)
    out_g, lm_off = eng.slam_delayed_init(case_g.frame, case_g.feats, opts, on_init)
    fr = case_o.frame
    tri, _ = oracle.triangulate(fr, case_o.feats, opts)
    P = case_o.P.copy()
    log_o, status_o = [], tri.status.copy()
    cols = []
    for off, sz in sorted([(int(x), 6) for x in fr.clone_off] + [(int(x), 6) for x in fr.cam_ext_off if x >= 0] +
                          [(int(x), 8) for x in fr.cam_intr_off if x >= 0]):
        cols += list(range(off, off + sz))
    cols = np.array(cols)
    for f in np.flatnonzero(tri.status == 0):
        one = case_o.feats.subset([f])
        o = capi.FeatOut(1)
        o.status[:] = 0
        o.p_FinA[0], o.p_FinG[0] = tri.p_FinA[f], tri.p_FinG[f]
        o.anchor_cam[0], o.anchor_clone[0] = tri.anchor_cam[f], tri.anchor_clone[f]
        Hf, Hx, res, _ = oracle.feature_jacobians(fr, one, opts, o, 0, cols)
        used = np.flatnonzero(np.abs(Hx).sum(axis=0) > 0)
        cc = cols[used]
        starts = [0] + [i for i in range(1, len(cc)) if cc[i] != cc[i - 1] + 1] + [len(cc)]
        off = [int(cc[a]) for a in starts[:-1]]
        sz = [int(b - a) for a, b in zip(starts[:-1], starts[1:])]
        st, acc, P, dxn, dx = oracle.cov_initialize(P, off, sz, Hx[:, used], Hf, res, sigma2=1.0, chi2_mult=float(opts.chi2_multipler))
        assert st == 0
        if acc:
            log_o.append((int(f), P.shape[0] - 3, dxn, dx))
            _apply_dx_to_frame(fr, dx)
        else:
            status_o[f] = capi.FEAT_CHI2
    assert np.array_equal(out_g.status, status_o)
    assert np.array_equal(out_g.status == capi.FEAT_OK, lm_off >= 0)
    assert len(log_g) == len(log_o) >= 1
    for (fg, og, dng, dg), (fo, oo, dno, do) in zip(log_g, log_o):
        assert fg == fo and og == oo == lm_off[fg]
        assert np.linalg.norm(dng - dno) <= 1e-8 * max(np.linalg.norm(dno), 1e-12)
        assert np.linalg.norm(dg - do) <= 1e-8 * max(np.linalg.norm(do), 1e-300)
    Pg = eng.cov_get()
    assert Pg.shape == P.shape and np.linalg.norm(Pg - P) <= 1e-9 * np.linalg.norm(P)
    N0 = case_g.P.shape[0]
    assert np.linalg.norm(Pg[N0:] - P[N0:]) <= 1e-9 * np.linalg.norm(P[N0:])  # the appended landmark rows on their own
    eng.close()


def test_sharded_long_tracks_match_single(oracle):
    """shard_compress_range + shard_finish on one GPU (two contexts stand in for two ranks) = the single-call update = the
    oracle. shard_finish compresses the stacked blocks in place, so every rank gets its own copy of the all-gather."""
    import torch
    from open_vins_b200 import multigpu
    case = sim.make_update_case(**FOUR_CAMS)
    assert _longest(case.feats) > 128
    opts = _opts(case, col_order=capi.COLS_CANONICAL)
    ref = oracle.msckf_update(case.frame, case.feats, opts, case.P, dumps=False)
    world = 2
    dev = torch.device("cuda", 0)
    engs = [capi.Engine(max_state=640, max_feats=512, max_meas=512 * 200) for _ in range(world)]
    parts = multigpu.partition_features(case.feats.meas_off, world)
    cap = 640 * 648
    blocks = []
    for r, e in enumerate(engs):
        e.cov_set(case.P)
        buf = torch.zeros(cap, dtype=torch.float64, device=dev)
        n, ld = e.shard_compress_range(case.frame, case.feats, parts[r][0], parts[r][1], opts, buf.data_ptr(), cap)
        torch.cuda.synchronize()
        blocks.append(buf[: n * ld].clone())
    status = []
    for r, e in enumerate(engs):
        stacked = torch.cat(blocks).contiguous()
        st, out, dx, _ = e.shard_finish(stacked.data_ptr(), world, parts[r][1] - parts[r][0])
        assert st == 0
        status.append(out.status)
        P = e.cov_get()
        assert np.linalg.norm(P - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
        assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * np.linalg.norm(ref["dx"])
        assert np.array_equal(P, P.T)
        if r == 0:
            P0, dx0 = P, dx
        else:
            assert np.array_equal(P, P0) and np.array_equal(dx, dx0)  # replicas stay bitwise identical
    assert np.array_equal(np.concatenate(status), ref["out"].status)
    for e in engs:
        e.close()


def test_track_over_the_limit_is_refused(eng):
    case = sim.make_update_case(n_feats=2, n_clones=48, n_cams=8, seed=11, full_track_frac=1.0, outlier_frac=0.0, degenerate_frac=0.0)
    f = case.feats
    M = np.diff(f.meas_off)
    assert M[0] == 384
    # repeat the last measurement of feature 0 (same camera, so the camera grouping stays valid): 385 measurements
    ins = int(f.meas_off[1])
    idx = np.concatenate([np.arange(ins), [ins - 1], np.arange(ins, f.meas_off[-1])])
    meas_off = np.array(f.meas_off, dtype=np.int64)
    meas_off[1:] += 1
    big = capi.FeatArrays(meas_off, f.cam[idx], f.clone[idx], f.uv[idx], f.uvn[idx])
    opts = _opts(case)
    with pytest.raises(capi.OvbError) as e:
        eng.triangulate(case.frame, big, opts)
    assert e.value.code == capi.OVB_ERR_CAPACITY
    eng.cov_set(case.P)
    with pytest.raises(capi.OvbError) as e:
        eng.msckf_update(case.frame, big, opts)
    assert e.value.code == capi.OVB_ERR_CAPACITY
    # exactly at the limit is accepted
    assert eng.triangulate(case.frame, f, opts).status.shape == (2,)
