"""The per-feature kernel's Mahalanobis gate (k_feature_system, csrc/k_feature.cu) on every layout (tile, BIG, long-track)
of every instantiation (MSCKF, SLAM, INIT), at the track lengths on both sides of each layout boundary, against an
extended-precision reference computed from the engine's own stage-0 Jacobians, so that only the projection and the gate
are tested.

Reference (tests/feature_routes.py, long double = 64-bit mantissa): chi2 = r_o'(Q2' S Q2)^-1 r_o with S = H P H' + s^2 I,
evaluated as a'a - (C'a)'(C'C)^-1(C'a), a = L^-1 r, C = L^-1 B. MSCKF and INIT: H = H_x, B = H_f. SLAM 3-wide: H = [H_x H_f]
with the landmark's block of P, no projection. SLAM SINGLE: H = [H_x H_f[:, 2]], B = H_f[:, :2].
Bar: |chi2 - ref| <= max(1e-12, 1e-14 kappa_2(S_o)) ref, S_o = Q2' S Q2.
Threshold pins: the gate multiplier at ref / q95(dof) (1 -+ m) must reject / accept, with dof as the oracle counts it and
the margin m = max(1e-7, 4 bar) wider than the chi2 bar, narrower than the gap to the other instantiations' dof.
Route proof: the profiled kernel names (every launch of ovb_msckf_update, ovb_slam_update and ovb_slam_delayed_init) hold
the instantiation of each layout the mirror gives the call's tracks, and no other layout of it. Track lengths come from
the mirror (tests/feature_routes.py), among them the tile / BIG boundary of a window where the last tile length leaves
less than 1 KB of shared memory below the limit.
The per-feature noise of SLAM landmarks and delayed-init features differs from the call-wide sigma_pix.
Run with -s to see the largest error per instance and layout and the smallest pin margin left.
"""
import os
from concurrent.futures import ProcessPoolExecutor
import multiprocessing

import numpy as np
import pytest

from open_vins_b200 import capi, sim
from tests import feature_routes as fr

pytestmark = pytest.mark.gpu

WINDOWS = ((4, 31), (8, 48))  # cameras x clone poses, extrinsics and intrinsics calibrated: tracks of up to 124 / 384


def _lengths(inst, window):
    n_all, n_slots = fr.window_dims(*window)
    MT = fr.find_M(inst, fr.TILE, n_all, n_slots, last=True)
    return sorted({M for M in (2, 3, MT - 1, MT, MT + 1, 127, 128, 129, 384) if M <= window[0] * window[1]})


# (instance, window, M, layout)
ROUTE_CASES = tuple((inst.name, w, M, fr.path_of(inst, M, *fr.window_dims(*w))) for inst in fr.INSTANCES for w in WINDOWS
                    for M in _lengths(inst, w))
# tight windows: (instance, window, M) at the last tile length and the first BIG one
TIGHT_CASES = tuple((inst.name, fr.tight_window(inst), M) for inst in fr.INSTANCES
                    for M in (lambda MT: (MT, MT + 1))(fr.find_M(inst, fr.TILE, *fr.window_dims(*fr.tight_window(inst)), last=True)))
REPORT = {}  # (instance, layout) -> [largest error / bar, largest relative error, cases]
PIN_ROOM = [np.inf, None]  # smallest (margin - |chi2 - ref| / ref) over the pins, and where
FEATURE_SIGMA = 1.3  # per-feature sigma_pix over the call-wide one (SLAM landmarks, delayed-init features)


@pytest.fixture(scope="module", autouse=True)
def _longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("the reference needs an extended-precision long double (64-bit mantissa)")
    yield
    print("\n(instance, layout): largest |chi2 - ref| / bar, largest |chi2 - ref| / ref, features")
    for k in sorted(REPORT):
        print(k, REPORT[k])
    print("smallest pin margin left (relative):", PIN_ROOM)


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    e = capi.Engine(max_state=1024, max_feats=1024, max_meas=1024 * 64)
    yield e
    e.close()


@pytest.fixture(scope="module")
def pool():
    """Worker processes for the long-double references of the large batches (pure numpy, no device)"""
    with ProcessPoolExecutor(max_workers=max(1, min(16, (os.cpu_count() or 1) - 1)), mp_context=multiprocessing.get_context("spawn")) as p:
        yield p


def _refs(jobs, pool=None):
    if pool is None or len(jobs) < 8:
        return [fr.gate_chi2_ref(*j) for j in jobs]
    return list(pool.map(fr.gate_chi2_ref, *zip(*jobs), chunksize=4))


def _check_chi2(inst, M, chi2, ref, n_all, n_slots, what):
    val, kappa = ref
    bar = max(1e-12, 1e-14 * kappa)
    err = abs(chi2 - val) / val
    route = fr.ROUTE_NAMES[fr.path_of(inst, M, n_all, n_slots)]
    r = REPORT.setdefault((inst.name, route), [0.0, 0.0, 0])
    r[0], r[1], r[2] = max(r[0], err / bar), max(r[1], err), r[2] + 1
    assert err <= bar, f"{inst.name} M={M} {what}: chi2 {chi2!r} reference {val!r} (rel {err:.3g}, kappa {kappa:.3g})"


def _assert_routes(names, inst, routes, what):
    """the profiled kernel names hold the instantiation of every layout in `routes` and of no other layout of `inst`"""
    feat = [nm for nm in names if "k_feature_system" in nm]
    for r in (fr.TILE, fr.BIG, fr.LONG):
        seen = any(inst.mangled[r] in nm for nm in feat)
        assert seen == (r in routes), (what, fr.ROUTE_NAMES[r], "expected" if r in routes else "unexpected", feat)


def _pin_margin(inst, M, ref, chi2):
    """the relative margin of the threshold pins: wider than the chi2 bar, narrower than the relative gap between q95 of
    this instantiation's dof and of the others' (2M - 3, 2M - 2, 2M); records the room the kernel's chi2 leaves"""
    val, kappa = ref
    margin = max(1e-7, 4 * max(1e-12, 1e-14 * kappa))
    dof = inst.dof(M)
    q = fr.gate_threshold(dof)
    gap = min(abs(fr.gate_threshold(d) / q - 1) for d in (2 * M - 3, 2 * M - 2, 2 * M) if d != dof and d >= 1)
    assert margin < gap / 2, (inst.name, M, margin, gap)
    room = margin - abs(chi2 - val) / val
    if room < PIN_ROOM[0]:
        PIN_ROOM[:] = [room, (inst.name, M, margin)]
    return margin


def _opts(inst, sigma=1.0, mult=1.0, rep=None):
    return capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, feat_rep=inst.rep if rep is None else rep,
                             sigma_pix=sigma, chi2_multipler=mult)


def _jac_rep(inst):
    """the representation whose Jacobians the kernel evaluates (SINGLE: ANCHORED_MSCKF_INVERSE_DEPTH's)"""
    return fr.REP_ANCHORED_MSCKF_INVERSE_DEPTH if inst.rep == fr.REP_SINGLE else inst.rep


def _stage0(eng, frame, feats, opts, tri):
    Hf, Hx, res, row_off, cols = eng.feature_jacobians(frame, feats, opts, tri.copy(), 0)
    out = []
    for f in range(feats.n_feats):
        a, b = row_off[f], row_off[f + 1]
        used = np.flatnonzero(np.abs(Hx[a:b]).sum(axis=0) > 0)
        out.append((Hx[a:b][:, used], Hf[a:b], res[a:b], cols[used], used))
    return out, cols


# ---------------------------------------------------------------------------------------------------------------- MSCKF
def _update_case(window, K, M, seed, prefix=False):
    case = sim.make_update_case(n_feats=K, n_clones=window[1], n_cams=window[0], seed=seed, full_track_frac=1.0, outlier_frac=0.0,
                                degenerate_frac=0.0, calib_ext=True, calib_intr=True)
    lens = M if np.ndim(M) else [M] * K
    return case, fr.cut_tracks(case.feats, lens, prefix=prefix)


def run_msckf(eng, inst, window, case, feats, pscale=1.0, sigma=1.0, pool=None, pins=True):
    n_all, n_slots = fr.window_dims(*window)
    P = case.P * pscale
    opts = _opts(inst, sigma, 1e6)
    eng.cov_set(P)
    tri = eng.triangulate(case.frame, feats, opts)
    ok = np.flatnonzero(tri.status == capi.FEAT_OK)
    assert len(ok) >= 1, "no track reaches the gate"
    sys0, cols = _stage0(eng, case.frame, feats, opts, tri)
    refs = dict(zip(ok, _refs([(Hx, Hf, r, P[np.ix_(c, c)], sigma ** 2) for f, (Hx, Hf, r, c, _) in enumerate(sys0) if f in set(ok)], pool)))
    M = np.diff(feats.meas_off)
    # stage 1: chi2 and the projected rows' invariants
    eng.cov_set(P)
    out1 = tri.copy()
    _, Hx1, res1, row1, cols1 = eng.feature_jacobians(case.frame, feats, opts, out1, 1)
    assert np.array_equal(cols1, cols)
    assert (out1.status[ok] == capi.FEAT_OK).all()  # rows of a rejected feature are zero: the multiplier lets all pass
    for f in ok:
        _check_chi2(inst, M[f], out1.chi2[f], refs[f], n_all, n_slots, "feature_jacobians")
        Hx, Hf, r, _, used = sys0[f]
        G, g, rr = fr.projected_invariants_ref(Hx, Hf, r)
        a, b = row1[f], row1[f + 1]
        Ho, ro = Hx1[a:b][:, used], res1[a:b]
        assert not np.delete(Hx1[a:b], used, axis=1).any()
        Gf = np.asarray(G, dtype=np.float64)
        assert np.linalg.norm(Ho.T @ Ho - Gf) <= 1e-12 * np.linalg.norm(Gf)
        assert np.linalg.norm(Ho.T @ ro - np.asarray(g, dtype=np.float64)) <= 1e-12 * np.sqrt(np.linalg.norm(Gf) * float(rr))
        assert abs(ro @ ro - float(rr)) <= 1e-12 * float(rr)
    # the update: chi2 and the route from the profiled kernel name
    eng.cov_set(P)
    eng.set_profile(True)
    st, out, _, _ = eng.msckf_update(case.frame, feats, opts)
    names = [nm for nm, _ in eng.profile_read()]
    eng.set_profile(False)
    assert st == capi.OVB_OK
    assert np.array_equal(out.p_FinG, tri.p_FinG, equal_nan=True)
    for f in ok:
        _check_chi2(inst, M[f], out.chi2[f], refs[f], n_all, n_slots, "msckf_update")
    _assert_routes(names, inst, {fr.path_of(inst, m, n_all, n_slots) for m in M}, "msckf_update")
    if pins:  # the multiplier is global: one feature per call
        for f in ok:
            thr = fr.gate_threshold(inst.dof(int(M[f])))
            mg = _pin_margin(inst, int(M[f]), refs[f], out.chi2[f])
            for side, want in ((-1, capi.FEAT_CHI2), (1, capi.FEAT_OK)):
                eng.cov_set(P)
                _, o, _, _ = eng.msckf_update(case.frame, feats.subset([f]), _opts(inst, sigma, refs[f][0] / thr * (1 + side * mg)))
                assert o.status[0] == want, (inst.name, int(M[f]), side)
    return out, refs, names


# ---------------------------------------------------------------------------------------------------------------- SLAM
def _slam_case(inst, window, K, M, seed, prefix=False):
    case = sim.make_slam_case(n_landmarks=K, n_clones=window[1], n_cams=window[0], seed=seed, rep=inst.rep,
                              track_len=(window[1], window[1]), two_classes=False)
    lens = M if np.ndim(M) else [M] * K
    return case, fr.cut_tracks(case.feats, lens, prefix=prefix)


def _landmarks(case, sigma, mult, idx=None):
    lm = case.landmarks
    idx = np.arange(len(lm.lm_off)) if idx is None else np.asarray(idx)
    n = len(idx)
    return capi.LandmarkArrays(lm.lm_off[idx], lm.value[idx], lm.value_fej[idx], lm.anchor_cam[idx], lm.anchor_clone[idx],
                               np.full(n, sigma), np.broadcast_to(np.asarray(mult, dtype=np.float64), (len(lm.lm_off),))[idx].copy())


def _slam_refs(eng, inst, case, feats, P, sigma, pool):
    """stage-0 Jacobians at the landmarks' values (ANCHORED_MSCKF_INVERSE_DEPTH's for both widths) and the references"""
    fa, lm = case.frame, case.landmarks
    K = feats.n_feats
    tri = capi.FeatOut(K)
    tri.status[:] = 0
    for f in range(K):
        c, k = int(lm.anchor_clone[f]), int(lm.anchor_cam[f])
        tri.p_FinA[f] = lm.value[f]
        tri.p_FinG[f] = fa.clone_R[c].T @ (fa.cam_R[k].T @ (lm.value[f] - fa.cam_p[k])) + fa.clone_p[c]
        tri.anchor_cam[f], tri.anchor_clone[f] = k, c
    sys0, _ = _stage0(eng, fa, feats, _opts(inst, sigma, rep=_jac_rep(inst)), tri)
    jobs = []
    for f, (Hx, Hf, r, c, _) in enumerate(sys0):
        o = int(lm.lm_off[f])
        if inst.single:
            H, B, idx = np.concatenate([Hx, Hf[:, 2:3]], axis=1), Hf[:, :2], np.concatenate([c, [o]])
        else:
            H, B, idx = np.concatenate([Hx, Hf], axis=1), None, np.concatenate([c, [o, o + 1, o + 2]])
        jobs.append((H, B, r, P[np.ix_(idx, idx)], sigma ** 2))
    return _refs(jobs, pool)


def run_slam(eng, inst, window, case, feats, pscale=1.0, sigma=1.0, pool=None, pins=True):
    n_all, n_slots = fr.window_dims(*window)
    P = case.P * pscale
    K = feats.n_feats
    eng.cov_set(P)
    refs = _slam_refs(eng, inst, case, feats, P, sigma, pool)
    M = np.diff(feats.meas_off)
    eng.set_slam_unbounded(True)
    eng.set_profile(True)
    st, out, _, _ = eng.slam_update(case.frame, feats, _landmarks(case, sigma, 1e6), _opts(inst, sigma / FEATURE_SIGMA))
    names = [nm for nm, _ in eng.profile_read()]
    eng.set_profile(False)
    assert st == capi.OVB_OK and (out.status == capi.FEAT_OK).all()
    for f in range(K):
        _check_chi2(inst, M[f], out.chi2[f], refs[f], n_all, n_slots, "slam_update")
    _assert_routes(names, inst, {fr.path_of(inst, m, n_all, n_slots) for m in M}, "slam_update")
    if pins:  # per-landmark multipliers: the whole batch in one call per side
        thr = np.array([fr.gate_threshold(inst.dof(int(m))) for m in M])
        val = np.array([r[0] for r in refs])
        mg = np.array([_pin_margin(inst, int(M[f]), refs[f], out.chi2[f]) for f in range(K)])
        for side, want in ((-1, capi.FEAT_CHI2), (1, capi.FEAT_OK)):
            eng.cov_set(P)
            _, o, _, _ = eng.slam_update(case.frame, feats, _landmarks(case, sigma, val / thr * (1 + side * mg)), _opts(inst, sigma / FEATURE_SIGMA))
            assert (o.status == want).all(), (inst.name, side, o.status)
    return out, refs, names


# ---------------------------------------------------------------------------------------------------------------- INIT
def run_init(eng, inst, window, case, feats, pscale=1.0, sigma=1.0, pool=None):
    """one feature per ovb_slam_delayed_init call (the initialisation is sequential), the gate pinned from both sides"""
    n_all, n_slots = fr.window_dims(*window)
    P = case.P * pscale
    opts = _opts(inst, sigma / FEATURE_SIGMA)  # the gate must use the feature's own sigma, not the call's
    eng.cov_set(P)
    tri = eng.triangulate(case.frame, feats, opts)
    ok = np.flatnonzero(tri.status == capi.FEAT_OK)
    assert len(ok) >= 1, "no track reaches the gate"
    sys0, _ = _stage0(eng, case.frame, feats, _opts(inst, sigma, rep=_jac_rep(inst)), tri)
    refs = dict(zip(ok, _refs([(sys0[f][0], sys0[f][1], sys0[f][2], P[np.ix_(sys0[f][3], sys0[f][3])], sigma ** 2) for f in ok], pool)))
    M = np.diff(feats.meas_off)
    for f in ok:
        thr = fr.gate_threshold(inst.dof(int(M[f])))
        mg = None
        for side, want in ((-1, capi.FEAT_CHI2), (1, capi.FEAT_OK)):
            eng.cov_set(P)
            eng.set_profile(True)
            if mg is None:  # the first call at the reference itself gives the kernel's chi2 the margin is checked against
                o, _ = eng.slam_delayed_init(case.frame, feats.subset([f]), opts, None, sigma_pix=[sigma], chi2_multipler=[1e6])
                _check_chi2(inst, M[f], o.chi2[0], refs[f], n_all, n_slots, "slam_delayed_init")
                mg = _pin_margin(inst, int(M[f]), refs[f], o.chi2[0])
                eng.cov_set(P)
            o, lm_off = eng.slam_delayed_init(case.frame, feats.subset([f]), opts, None, sigma_pix=[sigma],
                                              chi2_multipler=[refs[f][0] / thr * (1 + side * mg)])
            names = [nm for nm, _ in eng.profile_read()]
            eng.set_profile(False)
            _assert_routes(names, inst, {fr.path_of(inst, int(M[f]), n_all, n_slots)}, "slam_delayed_init")
            assert o.status[0] == want, (inst.name, int(M[f]), side)
            assert (lm_off[0] >= 0) == (want == capi.FEAT_OK)
            assert np.array_equal(o.p_FinG[0], tri.p_FinG[f])
            _check_chi2(inst, M[f], o.chi2[0], refs[f], n_all, n_slots, "slam_delayed_init")
    return refs


def run(eng, inst, window, M, K, seed, pscale=1.0, sigma=1.0, prefix=False, pool=None):
    if inst.kind == "slam":
        case, feats = _slam_case(inst, window, K, M, seed, prefix)
        return run_slam(eng, inst, window, case, feats, pscale, sigma, pool)
    case, feats = _update_case(window, K, M, seed, prefix)
    if inst.kind == "msckf":
        return run_msckf(eng, inst, window, case, feats, pscale, sigma, pool)
    return run_init(eng, inst, window, case, feats, pscale, sigma, pool)


@pytest.mark.parametrize("name,window,M,route", ROUTE_CASES, ids=[f"{n}-{w[0]}x{w[1]}-M{M}" for n, w, M, _ in ROUTE_CASES])
def test_gate_at_route_boundary(eng, name, window, M, route):
    inst = fr.INSTANCE[name]
    run(eng, inst, window, M, K=1 if M > 256 else 2, seed=1000 * M + 7 * window[0] + len(name))


@pytest.mark.parametrize("name,window,M", TIGHT_CASES, ids=[f"{n}-{w[0]}x{w[1]}-M{M}" for n, w, M in TIGHT_CASES])
def test_gate_at_tight_tile_limit(eng, name, window, M):
    """The tile / BIG boundary in a window where the last tile length leaves less than 1 KB of shared memory: a limit or a
    byte count off by that much in the host routing moves the boundary, and the profiled instantiation shows it."""
    inst = fr.INSTANCE[name]
    assert fr.tile_headroom(inst, *fr.window_dims(*window)) < 1024
    run(eng, inst, window, M, K=2, seed=3000 + M + 11 * window[0] + len(name))


# ---------------------------------------------------------------------------------------------------------------- conditioning
def _variant_cases():
    out = []
    for inst in fr.INSTANCES:
        n_all, n_slots = fr.window_dims(8, 48)
        MT = fr.find_M(inst, fr.TILE, n_all, n_slots, last=True)
        out += [(inst.name, M) for M in (MT, MT + 1, 129)]
    return out


@pytest.mark.parametrize("name,M", _variant_cases())
def test_gate_large_prior_fine_noise(eng, name, M):
    """P x 1e4 and sigma = 0.1 px: S is dominated by H P H', its condition number grows and the bar with it"""
    run(eng, fr.INSTANCE[name], (8, 48), M, K=2, seed=77 + M, pscale=1e4, sigma=0.1)


@pytest.mark.parametrize("name,M", [(n, M) for n in ("msckf_global", "msckf_anchored", "slam_3wide", "slam_single", "init_3wide", "init_single")
                                    for M in (8, 10)])
def test_gate_short_baseline(eng, name, M):
    """The first M measurements of a track: one camera in adjacent clone poses, so that H_f is close to rank deficient"""
    inst = fr.INSTANCE[name]
    case_seed = 90 + M
    if inst.kind == "slam":
        case, feats = _slam_case(inst, (4, 31), 3, M, case_seed, prefix=True)
    else:
        case, feats = _update_case((4, 31), 3, M, case_seed, prefix=True)
    assert len(set(feats.cam[:M])) == 1 and int(feats.clone[M - 1]) - int(feats.clone[0]) == M - 1
    if inst.kind == "slam":
        run_slam(eng, inst, (4, 31), case, feats)
    elif inst.kind == "msckf":
        run_msckf(eng, inst, (4, 31), case, feats)
    else:
        run_init(eng, inst, (4, 31), case, feats)


# ---------------------------------------------------------------------------------------------------------------- batches
def _alone(eng, case, feats, P, opts, out):
    """every feature run on its own gives the batch's status, chi2 and triangulated point bit for bit"""
    for f in range(feats.n_feats):
        eng.cov_set(P)
        _, o, _, _ = eng.msckf_update(case.frame, feats.subset([f]), opts)
        assert o.status[0] == out.status[f], f
        assert np.array_equal(o.chi2[:1], out.chi2[f:f + 1], equal_nan=True), f
        assert np.array_equal(o.p_FinG[0], out.p_FinG[f], equal_nan=True), f


def _msckf_batch(eng, sm_count, pool, lens, seed, want):
    inst = fr.INSTANCE["msckf_global"]
    window = (8, 48)
    n_all, n_slots = fr.window_dims(*window)
    plan = fr.launch_plan(lens, inst, n_all, n_slots, sm_count)
    assert [(l.path, l.stream, l.grid) for l in plan] == want(plan), plan
    case, feats = _update_case(window, len(lens), lens, seed)
    out, refs, names = run_msckf(eng, inst, window, case, feats, pool=pool, pins=False)
    assert len(refs) >= 0.9 * len(lens)
    _alone(eng, case, feats, case.P, _opts(inst, 1.0, 1e6), out)
    return plan, names


def test_msckf_batch_big_scratch_reuse(eng, sm_count, pool):
    """More than 2 x SM BIG tracks, half of them 128 long (the 257 x 257 scratch slice full): the grid is clamped to
    2 x SM CTAs that loop over the features and reuse their slices"""
    inst = fr.INSTANCE["msckf_global"]
    MT = fr.find_M(inst, fr.TILE, *fr.window_dims(8, 48), last=True)
    K = 2 * sm_count + 6
    lens = [128 if i % 2 == 0 else MT + 1 + (7 * i) % (128 - MT) for i in range(K)]
    _, names = _msckf_batch(eng, sm_count, pool, lens, 501, lambda p: [(fr.BIG, 0, 2 * sm_count)])
    _assert_routes(names, inst, {fr.BIG}, "BIG batch")


def test_msckf_batch_long_more_than_sms(eng, sm_count, pool):
    """More long tracks (129-130 measurements) than SMs: one CTA per SM, each looping over features in its scratch slice"""
    inst = fr.INSTANCE["msckf_global"]
    lens = [129 + i % 2 for i in range(sm_count + 5)]
    _, names = _msckf_batch(eng, sm_count, pool, lens, 502, lambda p: [(fr.LONG, 0, sm_count)])
    _assert_routes(names, inst, {fr.LONG}, "long batch")


@pytest.mark.parametrize("mixed", [False, True], ids=["tile_only", "with_big_and_long"])
def test_msckf_batch_tile_size_classes(eng, sm_count, pool, mixed):
    """More tile tracks than SMs over the three size classes (> 32, 17-32, <= 16 measurements): three launches on the main
    and side streams, or all three on the side streams behind BIG and long tracks"""
    MT = fr.find_M(fr.INSTANCE["msckf_global"], fr.TILE, *fr.window_dims(8, 48), last=True)
    tile = [(2, 3, 9, 16, 17, 24, 32, 33, 50, MT)[i % 10] for i in range(sm_count + 20)]
    lens = ([129, 200, 128, 100, MT + 1] if mixed else []) + tile

    def want(plan):
        n = len(tile)
        c = [sum(1 for m in tile if m > 32), sum(1 for m in tile if 16 < m <= 32), sum(1 for m in tile if m <= 16)]
        if mixed:
            return [(fr.LONG, 0, 2), (fr.BIG, 0, 3), (fr.TILE, 1, c[0]), (fr.TILE, 2, c[1]), (fr.TILE, 2, c[2])]
        assert sum(c) == n
        return [(fr.TILE, 0, c[0]), (fr.TILE, 1, c[1]), (fr.TILE, 2, c[2])]
    _msckf_batch(eng, sm_count, pool, lens, 503 + int(mixed), want)


def test_slam_batch_big_scratch_reuse(eng, sm_count, pool):
    """More than 2 x SM BIG landmark tracks in one ovb_slam_update call (SINGLE: 1-wide landmarks, the two bearing columns
    projected out on the BIG layout), half of them 128 long"""
    inst = fr.INSTANCE["slam_single"]
    window = (8, 48)
    n_all, n_slots = fr.window_dims(*window)
    MT = fr.find_M(inst, fr.TILE, n_all, n_slots, last=True)
    K = 2 * sm_count + 6
    lens = [128 if i % 2 == 0 else MT + 1 + (5 * i) % (128 - MT) for i in range(K)]
    plan = fr.launch_plan(lens, inst, n_all, n_slots, sm_count)
    assert [(l.path, l.grid) for l in plan] == [(fr.BIG, 2 * sm_count)]
    case, feats = _slam_case(inst, window, K, lens, 601)
    out, _, names = run_slam(eng, inst, window, case, feats, pool=pool, pins=False)
    _assert_routes(names, inst, {fr.BIG}, "SLAM BIG batch")
    for f in range(K):
        eng.cov_set(case.P)
        _, o, _, _ = eng.slam_update(case.frame, feats.subset([f]), _landmarks(case, 1.0, 1e6, [f]), _opts(inst, 1.0 / FEATURE_SIGMA))
        assert o.status[0] == out.status[f] and np.array_equal(o.chi2[:1], out.chi2[f:f + 1], equal_nan=True), f
