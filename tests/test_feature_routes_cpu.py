"""Invariants of the per-feature kernel's routing mirror (tests/feature_routes.py) and of the GPU case list built on it."""
import numpy as np
import pytest

from open_vins_b200 import sim
from tests import feature_routes as fr
from tests.test_gpu_feature_routes import ROUTE_CASES, TIGHT_CASES, WINDOWS

ROUTES = (fr.TILE, fr.BIG, fr.LONG)


@pytest.mark.parametrize("inst", fr.INSTANCES, ids=lambda i: i.name)
@pytest.mark.parametrize("window", WINDOWS, ids=lambda w: f"{w[0]}x{w[1]}")
def test_path_monotone_and_all_routes(inst, window):
    n_all, n_slots = fr.window_dims(*window)
    paths = [fr.path_of(inst, M, n_all, n_slots) for M in range(1, fr.OVB_MAX_MEAS_PER_FEAT + 1)]
    assert paths == sorted(paths), "tile, then BIG, then long-track as the track grows"
    for r in ROUTES:
        first, last = fr.find_M(inst, r, n_all, n_slots), fr.find_M(inst, r, n_all, n_slots, last=True)
        assert first is not None and last is not None, fr.ROUTE_NAMES[r]
        assert fr.path_of(inst, first, n_all, n_slots) == fr.path_of(inst, last, n_all, n_slots) == r
        if first > 2:
            assert fr.path_of(inst, first - 1, n_all, n_slots) == r - 1
        if last < fr.OVB_MAX_MEAS_PER_FEAT:
            assert fr.path_of(inst, last + 1, n_all, n_slots) == r + 1
    # BIG ends where d_scratch's slices end; the long-track layout takes the rest
    assert fr.find_M(inst, fr.BIG, n_all, n_slots, last=True) == fr.OVB_BIG_MAX_MEAS
    assert fr.find_M(inst, fr.LONG, n_all, n_slots, last=True) == fr.OVB_MAX_MEAS_PER_FEAT
    # the last tile length fits the limit, the next one does not
    MT = fr.find_M(inst, fr.TILE, n_all, n_slots, last=True)
    dm = fr.feature_dims(n_all, n_slots, inst)
    assert fr.feature_smem_bytes(MT, dm, inst.nblk, fr.TILE) <= fr.FT_SMEM_LIMIT < fr.feature_smem_bytes(MT + 1, dm, inst.nblk, fr.TILE)


def test_boundaries_of_the_calibrated_windows():
    """The last tile length of every instance in the two windows the GPU cases use"""
    want = {(4, 31): dict(msckf_global=78, msckf_anchored=74, slam_3wide=70, slam_single=70, init_3wide=74, init_single=74),
            (8, 48): dict(msckf_global=70, msckf_anchored=66, slam_3wide=62, slam_single=62, init_3wide=66, init_single=66)}
    for w, d in want.items():
        n_all, n_slots = fr.window_dims(*w)
        assert {i.name: fr.find_M(i, fr.TILE, n_all, n_slots, last=True) for i in fr.INSTANCES} == d


@pytest.mark.parametrize("inst", fr.INSTANCES, ids=lambda i: i.name)
def test_tight_window_headroom(inst):
    """Each instance has a GPU case on both sides of the tile / BIG boundary in a window where the last tile length leaves
    less than 1 KB of shared memory below the limit, so that a limit or byte count off by 1 KB moves the boundary"""
    window = fr.tight_window(inst)
    n_all, n_slots = fr.window_dims(*window)
    MT = fr.find_M(inst, fr.TILE, n_all, n_slots, last=True)
    assert 0 <= fr.tile_headroom(inst, n_all, n_slots) < 1024 and window[0] * window[1] > MT
    dm = fr.feature_dims(n_all, n_slots, inst)
    assert fr.feature_path(MT, dm, inst.nblk, fr.FT_SMEM_LIMIT - 1024) == fr.BIG
    assert {M for n, w, M in TIGHT_CASES if n == inst.name and w == window} == {MT, MT + 1}
    assert fr.path_of(inst, MT, n_all, n_slots) == fr.TILE and fr.path_of(inst, MT + 1, n_all, n_slots) == fr.BIG


def test_frame_dims_from_frame_arrays():
    for n_cams, n_clones, calib in [(4, 31, True), (8, 48, True), (2, 6, False)]:
        case = sim.make_update_case(n_feats=1, n_clones=n_clones, n_cams=n_cams, calib_ext=calib, calib_intr=calib)
        assert fr.frame_dims(case.frame, calib, calib) == fr.window_dims(n_cams, n_clones, calib)
    # calibration blocks in the state but not estimated are not columns of the system
    case = sim.make_update_case(n_feats=1, n_clones=5, n_cams=2, calib_ext=True, calib_intr=True)
    assert fr.frame_dims(case.frame, True, False) == (30 + 12, 7)
    # estimated calibration without a block in the state is refused, as the host refuses the frame
    case = sim.make_update_case(n_feats=1, n_clones=5, n_cams=2)
    with pytest.raises(AssertionError):
        fr.frame_dims(case.frame, True, False)


def test_route_cases_cover_every_cell():
    """Every (instance, layout, boundary side) cell that exists in a window appears in the GPU case list, at the length
    the mirror gives for it."""
    for window in WINDOWS:
        n_all, n_slots = fr.window_dims(*window)
        cap = window[0] * window[1]
        for inst in fr.INSTANCES:
            MT = fr.find_M(inst, fr.TILE, n_all, n_slots, last=True)
            cells = {(fr.TILE, "first"): 2, (fr.TILE, "last"): MT, (fr.BIG, "first"): MT + 1, (fr.BIG, "last"): 128,
                     (fr.LONG, "first"): 129, (fr.LONG, "last"): 384}
            got = {M for (i, w, M, _) in ROUTE_CASES if i == inst.name and w == window}
            for (r, side), M in cells.items():
                assert fr.path_of(inst, M, n_all, n_slots) == r
                if M <= cap:
                    assert M in got, (inst.name, window, fr.ROUTE_NAMES[r], side, M)
            assert got <= set(range(2, cap + 1))


def test_launch_plan_size_classes_and_clamps():
    inst = fr.INSTANCE["msckf_global"]
    n_all, n_slots = fr.window_dims(8, 48)
    sm = 132
    # tile tracks only, more than one per SM: three size classes on the main and first side stream ... and the second
    lens = [40] * 50 + [20] * 50 + [10] * 50
    plan = fr.launch_plan(lens, inst, n_all, n_slots, sm)
    assert [(l.path, l.lo, l.hi, l.stream) for l in plan] == [(fr.TILE, 0, 50, 0), (fr.TILE, 50, 100, 1), (fr.TILE, 100, 150, 2)]
    # with BIG and long tracks in front, the tile classes move to the side streams
    plan = fr.launch_plan([130] * 3 + [100] * 300 + lens, inst, n_all, n_slots, sm)
    assert [(l.path, l.stream, l.grid) for l in plan] == [(fr.LONG, 0, 3), (fr.BIG, 0, 2 * sm), (fr.TILE, 1, 50), (fr.TILE, 2, 50),
                                                         (fr.TILE, 2, 50)]
    # no more tile tracks than SMs: one tile launch; SLAM never splits
    assert len(fr.launch_plan([10] * sm, inst, n_all, n_slots, sm)) == 1
    assert len(fr.launch_plan(lens, fr.INSTANCE["slam_single"], n_all, n_slots, sm)) == 1
    # long tracks: one CTA per SM at most
    plan = fr.launch_plan([129] * (sm + 5), inst, n_all, n_slots, sm)
    assert [(l.path, l.grid) for l in plan] == [(fr.LONG, sm)]


def test_cut_tracks_keeps_camera_groups():
    case = sim.make_update_case(n_feats=3, n_clones=10, n_cams=4, seed=5, full_track_frac=1.0, outlier_frac=0.0, degenerate_frac=0.0)
    for prefix in (False, True):
        cut = fr.cut_tracks(case.feats, [2, 17, 40], prefix=prefix)
        assert list(np.diff(cut.meas_off)) == [2, 17, 40]
        for f in range(3):
            cams = cut.cam[cut.meas_off[f]:cut.meas_off[f + 1]]
            runs = [c for i, c in enumerate(cams) if i == 0 or c != cams[i - 1]]
            assert len(runs) == len(set(runs)), "every camera's measurements are contiguous"
    spread = fr.cut_tracks(case.feats, [40, 40, 40])
    assert len(set(spread.cam[:40])) == 4 and len(set(spread.clone[:40])) == 10


def test_reference_against_dense_inverse():
    """gate_chi2_ref equals r'(Q2' S Q2)^-1 r formed explicitly, for every projection width"""
    rng = np.random.default_rng(3)
    m, n = 20, 12
    H = rng.standard_normal((m, n))
    A = rng.standard_normal((n, n))
    P = A @ A.T / n + 0.1 * np.eye(n)
    r = rng.standard_normal(m)
    S = H @ P @ H.T + 0.7 * np.eye(m)
    for k in (0, 2, 3):
        B = rng.standard_normal((m, k)) if k else None
        chi2, kappa = fr.gate_chi2_ref(H, B, r, P, 0.7)
        if k:
            Q2 = np.linalg.qr(B, mode="complete")[0][:, k:]
            want = (Q2.T @ r) @ np.linalg.solve(Q2.T @ S @ Q2, Q2.T @ r)
        else:
            want = r @ np.linalg.solve(S, r)
        assert abs(chi2 - want) <= 1e-12 * want and kappa >= 1
    Hf = rng.standard_normal((m, 3))
    G, g, rr = fr.projected_invariants_ref(H, Hf, r)
    Q2 = np.linalg.qr(Hf, mode="complete")[0][:, 3:]
    Ho, ro = Q2.T @ H, Q2.T @ r
    assert np.abs(np.asarray(G, dtype=float) - Ho.T @ Ho).max() <= 1e-12 * np.abs(Ho.T @ Ho).max()
    assert np.abs(np.asarray(g, dtype=float) - Ho.T @ ro).max() <= 1e-12 * np.abs(Ho.T @ ro).max()
    assert abs(float(rr) - ro @ ro) <= 1e-12 * (ro @ ro)
