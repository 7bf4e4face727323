"""Launch counts and per-call profiles on the GPU: every kernel goes through ovb_launch, which counts it and, while
profiling is on, times it. So the profile of a call lists exactly the kernels ovb_last_counters reports for it, and a
second identical call reports the same list (the profile starts afresh with every call, however long the call)."""
import numpy as np
import pytest

from open_vins_b200 import capi, sim, simrun
from tests.test_window_cpu import window_case

pytestmark = pytest.mark.gpu

CALIB = dict(do_calib_camera_pose=1, do_calib_camera_intrinsics=1)


def _twice(eng, call):
    """the profiled kernel names of two consecutive calls, each checked against the call's launch counter"""
    eng.set_profile(True)
    runs = []
    for _ in range(2):
        call()
        names = [nm for nm, _ in eng.profile_read()]
        cnt = eng.last_counters()
        assert len(names) == cnt["launches"], (len(names), cnt)
        assert sum("k_tsqr_level" in nm for nm in names) == cnt["tsqr_level_launches"]
        runs.append(names)
    eng.set_profile(False)
    assert runs[0] == runs[1]
    return runs[1]


def _msckf(eng, frame, feats, opts, P):
    def call():
        eng.cov_set(P)
        st, _, _, _ = eng.msckf_update(frame, feats, opts)
        assert st == capi.OVB_OK
    return _twice(eng, call)


@pytest.mark.parametrize("config", [1, 2])
def test_msckf_update_configs_1_2(config):
    frame, feats, opts, P = simrun.load_case(simrun.CASE_CONFIG1 if config == 1 else simrun.CASE_CONFIG2)
    opts.col_order = capi.COLS_CANONICAL
    eng = capi.Engine(max_state=256, max_feats=1024, max_meas=65536)
    names = _msckf(eng, frame, feats, opts, P)
    for k in ("k_cam_poses", "k_triangulate", "k_feature_system", "k_column_map", "k_cq_gram", "k_ekf_prep"):
        assert any(k in nm for nm in names), (k, names)
    eng.close()


def test_msckf_update_config4_wide():
    c = sim.make_update_case(n_feats=800, n_clones=31, n_cams=4, seed=0, calib_ext=True, calib_intr=True, calib_imu=True, calib_dt=True)
    opts = capi.default_opts(**CALIB, col_order=capi.COLS_CANONICAL)
    eng = capi.Engine(max_state=640, max_feats=1024, max_meas=max(65536, int(c.feats.n_meas) + 1024))
    names = _msckf(eng, c.frame, c.feats, opts, c.P)
    # the blocked factorisation of the wide route: more than one trsm and gemm per pass
    assert sum("k_cq_gemm_nt" in nm for nm in names) > 2 and any("k_cq_trmm_wide" in nm for nm in names), names
    eng.close()


def test_msckf_update_first_seen_order():
    frame, feats, opts, P = simrun.load_case(simrun.CASE_CONFIG1)
    opts.col_order = capi.COLS_REFERENCE_FIRST_SEEN
    eng = capi.Engine(max_state=256, max_feats=1024, max_meas=65536)
    names = _msckf(eng, frame, feats, opts, P)
    assert any("k_gather_cols" in nm for nm in names) and any("k_tsqr_level" in nm for nm in names), names
    eng.close()


def test_slam_update_two_groups():
    case = sim.make_slam_case(n_landmarks=100, n_clones=31, n_cams=4, seed=4, rep=capi.REP_GLOBAL_3D)  # 542 columns: two groups
    opts = capi.default_opts(feat_rep=capi.REP_GLOBAL_3D, **CALIB)
    eng = capi.Engine(max_state=640, max_feats=256, max_meas=16384)
    eng.set_slam_unbounded()

    def call():
        eng.cov_set(case.P)
        st, _, _, _ = eng.slam_update(case.frame, case.feats, case.landmarks, opts)
        assert st == capi.OVB_OK
    names = _twice(eng, call)
    assert sum("k_group_take_z" in nm for nm in names) == 2 and any("k_group_finish" in nm for nm in names), names
    eng.close()


def test_ekf_update_8000x500():
    H, res, P = sim.make_compress_case(m=8000, n=500, seed=0, structured=False)
    eng = capi.Engine(max_state=512, max_feats=64, max_meas=4096, max_rows=8192)

    def call():
        eng.cov_set(P)
        eng.ekf_update([0], [500], H, res, sigma2=1.0)
    names = _twice(eng, call)
    assert any("k_cq_trmm_wide" in nm for nm in names), names  # the blocked compression of 501 columns
    eng.close()


def test_cov_propagate_imu():
    n, steps, N = 15, 12, 15 + 6 * 4
    rng = np.random.default_rng(3)
    A = rng.standard_normal((N, N))
    P = A @ A.T / N + np.eye(N)
    F = np.eye(n) + 0.01 * rng.standard_normal((steps, n, n))
    G = 0.01 * rng.standard_normal((steps, n, 12))
    qc = np.abs(rng.standard_normal((steps, 4)))
    dnc = rng.standard_normal(6)
    eng = capi.Engine(max_state=256, max_feats=16, max_meas=256)

    def call():
        eng.cov_set(P)
        st, _, _ = eng.cov_propagate_imu(F, G, qc, 0, [0], [n], 0, 6, dnc, 14)
        assert st == capi.OVB_OK
    names = _twice(eng, call)
    for k in ("k_prop_accumulate", "k_prop_C", "k_prop_PCP", "k_prop_write", "k_cov_clone", "k_cov_dt_cols", "k_cov_dt_rows"):
        assert any(k in nm for nm in names), (k, names)
    eng.close()


def test_marginalize_window():
    case, anchors, marg = window_case([5, 2, 5, 5, 4, 3, 5, 2, 4, 5, 3, 2], n_clones=9, n_cams=3, seed=12, k_anchor=9, k_lost=2)
    opts = capi.default_opts(do_calib_camera_pose=1)
    eng = capi.Engine(max_state=800, max_feats=16, max_meas=256)

    def call():
        eng.cov_set(case.P)
        assert eng.marginalize_window(case.frame, opts, [o for o, _ in marg], [s for _, s in marg], anchors) == capi.OVB_OK
    names = _twice(eng, call)
    for k in ("k_anchor_phi", "k_win_rows", "k_win_blocks", "k_win_compact"):
        assert any(k in nm for nm in names), (k, names)
    eng.close()
