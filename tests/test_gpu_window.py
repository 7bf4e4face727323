"""ovb_marginalize_window on the GPU: one call against the existing call sequence it replaces (ovb_slam_anchor_change +
ovb_cov_propagate per re-anchored landmark, then ovb_cov_marginalize per range, highest first) on two contexts holding the
same P, bit for bit; against the oracle's sequence; and its error returns, which leave P and N untouched."""
import functools

import numpy as np
import pytest

from open_vins_b200 import capi, sim
from tests.test_window_cpu import sequence, window_case

pytestmark = pytest.mark.gpu

CYCLE = [capi.REP_ANCHORED_3D, capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE, capi.REP_ANCHORED_FULL_INVERSE_DEPTH]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


@functools.lru_cache(maxsize=None)
def _window(n_clones, n_cams, n_lm, seed, pad):
    """make_slam_case's state with `pad` more variables at the end (config 4: 4 cameras, 31 clones, 100 landmarks, pad = 75 gives N = 582)."""
    reps = tuple(CYCLE[i % 4] for i in range(n_lm))
    case = sim.make_slam_case(n_landmarks=n_lm, n_clones=n_clones, n_cams=n_cams, seed=seed, rep=list(reps))
    if pad:
        rng = np.random.default_rng(seed)
        N0 = case.P.shape[0]
        A = rng.standard_normal((N0 + pad, 8)) * 0.01
        P = A @ A.T
        P[:N0, :N0] += case.P
        P[N0:, N0:] += 1e-2 * np.eye(pad)
        case.P = 0.5 * (P + P.T)
    return case, reps


def _setup(n_clones, n_cams, n_lm, seed, pad, k_anchor, k_lost, ext=True):
    case, reps = _window(n_clones, n_cams, n_lm, seed, pad)
    lm, fr = case.landmarks, case.frame
    width = np.array([1 if r == capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE else 3 for r in reps])
    # re-anchor every third landmark from the front (all four representations), lose landmarks from the back; the oldest
    # clone goes too
    moved = np.arange(0, 3 * k_anchor, 3)
    lost = np.arange(n_lm - 1, n_lm - 1 - k_lost, -1)
    old_cam = lm.anchor_cam[moved]
    anchors = capi.AnchorChanges(lm.lm_off[moved], np.asarray(reps)[moved], lm.value[moved], lm.value_fej[moved], old_cam, np.zeros(len(moved)),
                                 (old_cam + 1 + np.arange(len(moved))) % n_cams, np.full(len(moved), n_clones - 1))
    marg = [(int(lm.lm_off[f]), int(width[f])) for f in lost] + [(int(fr.clone_off[0]), 6)]
    return case, anchors, marg


def _compare(case, anchors, marg, fej=1, ext=1):
    opts = capi.default_opts(do_fej=fej, do_calib_camera_pose=ext)
    a = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    b = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    a.cov_set(case.P)
    b.cov_set(case.P)

    def propagate(o, Phi, Q, off, sz):
        assert a.cov_propagate(o, Phi, Q, off, sz) == capi.OVB_OK

    nv, nvf, _ = sequence(case, anchors, marg, fej, ext, capi.slam_anchor_change, propagate, a.cov_marginalize)
    assert b.marginalize_window(case.frame, opts, [o for o, _ in marg], [s for _, s in marg], anchors) == capi.OVB_OK
    assert a.cov_dim() == b.cov_dim() == case.P.shape[0] - sum(s for _, s in marg)
    Pa, Pb = a.cov_get(), b.cov_get()
    a.close()
    b.close()
    assert np.array_equal(_bits(anchors.new_value), _bits(nv)) and np.array_equal(_bits(anchors.new_value_fej), _bits(nvf))
    assert np.array_equal(_bits(Pa), _bits(Pb))
    return Pb


@pytest.mark.parametrize("k_anchor", [0, 1, 4, 25])
@pytest.mark.parametrize("k_lost", [0, 3, 10])
def test_config4_window_is_the_call_sequence(k_anchor, k_lost):
    case, anchors, marg = _setup(31, 4, 100, 4, 75, k_anchor, k_lost)
    assert case.P.shape[0] == 582
    _compare(case, anchors, marg)


@pytest.mark.parametrize("fej,ext", [(0, 1), (1, 0), (0, 0)])
def test_fej_and_extrinsics_off(fej, ext):
    case, anchors, marg = _setup(31, 4, 100, 4, 75, 8, 3)
    _compare(case, anchors, marg, fej=fej, ext=ext)


def test_eight_camera_48_clone_window():
    case, anchors, marg = _setup(48, 8, 100, 8, 0, 25, 10)
    _compare(case, anchors, marg)


def test_mixed_widths_adjacent_and_new_camera():
    """1-wide SINGLE landmarks next to 3-wide ones of the other representations, every re-anchoring to another camera."""
    reps = [5, 2, 5, 5, 4, 3, 5, 2, 4, 5, 3, 2]
    case, anchors, marg = window_case(reps, n_clones=9, n_cams=3, seed=12, k_anchor=9, k_lost=2)
    anchors.new_cam[:] = (anchors.old_cam + 1) % 3
    _compare(case, anchors, marg)


def test_empty_anchor_list_and_no_anchors():
    case, anchors, marg = _setup(31, 4, 100, 4, 75, 0, 10)
    _compare(case, anchors, marg)
    a = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    a.cov_set(case.P)
    assert a.marginalize_window(None, None, [o for o, _ in marg], [s for _, s in marg], None) == capi.OVB_OK
    b = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    b.cov_set(case.P)
    for o, s in sorted(marg, reverse=True):
        b.cov_marginalize(o, s)
    assert np.array_equal(_bits(a.cov_get()), _bits(b.cov_get()))


def test_oldest_clone_only_is_cov_marginalize():
    case, _, _ = _setup(31, 4, 100, 4, 75, 0, 0)
    off = int(case.frame.clone_off[0])
    a = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    b = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    a.cov_set(case.P)
    b.cov_set(case.P)
    a.cov_marginalize(off, 6)
    assert b.marginalize_window(None, None, [off], [6], None) == capi.OVB_OK
    assert np.array_equal(_bits(a.cov_get()), _bits(b.cov_get()))


def test_against_the_oracle_sequence(oracle):
    case, anchors, marg = _setup(31, 4, 100, 4, 75, 25, 10)
    Pg = _compare(case, anchors, marg)
    box = {"P": case.P.copy()}

    def propagate(o, Phi, Q, off, sz):
        st, box["P"] = oracle.cov_propagate(box["P"], o, Phi, Q, off, sz)
        assert st == 0

    def marginalize(o, s):
        box["P"] = oracle.cov_marginalize(box["P"], o, s)

    nv, nvf, _ = sequence(case, anchors, marg, 1, 1, oracle.anchor_change, propagate, marginalize)
    assert np.linalg.norm(Pg - box["P"]) <= 1e-12 * np.linalg.norm(box["P"])
    np.testing.assert_allclose(anchors.new_value, nv, rtol=1e-13, atol=1e-15)


def _untouched(eng, P, fn):
    N = eng.cov_dim()
    with pytest.raises(capi.OvbError) as ei:
        fn()
    assert ei.value.code == capi.OVB_ERR_ARG
    assert eng.cov_dim() == N and np.array_equal(_bits(eng.cov_get()), _bits(P))


def test_argument_errors_leave_p_untouched():
    case, anchors, marg = _setup(31, 4, 100, 4, 75, 4, 3)
    fr, lm = case.frame, case.landmarks
    opts = capi.default_opts(do_calib_camera_pose=1)
    eng = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    eng.cov_set(case.P)
    N = case.P.shape[0]
    mo, ms = [o for o, _ in marg], [s for _, s in marg]

    def with_anchors(**kw):
        d = dict(lm_off=anchors.lm_off, feat_rep=anchors.feat_rep, value=anchors.value, value_fej=anchors.value_fej, old_cam=anchors.old_cam,
                 old_clone=anchors.old_clone, new_cam=anchors.new_cam, new_clone=anchors.new_clone)
        d.update(kw)
        an = capi.AnchorChanges(**d)
        return lambda: eng.marginalize_window(fr, opts, mo, ms, an), an

    cases = [
        lambda: eng.marginalize_window(fr, opts, mo + [mo[0] + 1], ms + [1], anchors),      # overlapping ranges
        lambda: eng.marginalize_window(fr, opts, mo + [N - 2], ms + [3], anchors),          # outside N
        lambda: eng.marginalize_window(fr, opts, mo + [int(anchors.lm_off[1])], ms + [3], anchors),  # re-anchored and lost
    ]
    bad = []
    rep = anchors.feat_rep.copy()
    rep[2] = capi.REP_GLOBAL_3D
    bad.append(with_anchors(feat_rep=rep))
    for key, val in [("old_clone", fr.n_clones), ("new_clone", -1), ("old_cam", fr.n_cams), ("new_cam", -1)]:
        arr = getattr(anchors, key).copy()
        arr[1] = val
        bad.append(with_anchors(**{key: arr}))
    arr = anchors.new_clone.copy()
    arr[0] = 3
    cases.append(lambda: eng.marginalize_window(fr, opts, mo + [int(fr.clone_off[3])], ms + [6], with_anchors(new_clone=arr)[1]))  # new clone lost
    lo = anchors.lm_off.copy()
    lo[3] = lo[2]
    bad.append(with_anchors(lm_off=lo))                                                     # listed twice
    for fn in cases + [f for f, _ in bad]:
        _untouched(eng, case.P, fn)
    for _, an in bad:
        assert np.isnan(an.new_value).all() and np.isnan(an.new_value_fej).all()
    eng.close()


def test_negative_diagonal_returns_status_with_p_untouched():
    """A symmetric P that is not positive semi-definite in a re-anchored landmark's prior block: the propagated diagonal goes
    negative. ovb_cov_propagate reports it after writing; ovb_marginalize_window reports it with P and N as they were."""
    case, anchors, marg = _setup(31, 4, 100, 4, 75, 4, 3)
    P = case.P.copy()
    o = int(anchors.lm_off[1])
    w = 1 if anchors.feat_rep[1] == capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE else 3
    P[o:o + w, o:o + w] = -1e3 * np.eye(w)
    ref = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    ref.cov_set(P)
    opts = capi.default_opts(do_calib_camera_pose=1, feat_rep=int(anchors.feat_rep[1]))
    _, _, off, sz, Phi = capi.slam_anchor_change(case.frame, opts, o, anchors.value[1], anchors.value_fej[1], anchors.old_cam[1], anchors.old_clone[1],
                                                 anchors.new_cam[1], anchors.new_clone[1])
    assert ref.cov_propagate(o, Phi, np.zeros((w, w)), off, sz) == capi.OVB_ERR_NEG_DIAG
    ref.close()
    eng = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    eng.cov_set(P)
    st = eng.marginalize_window(case.frame, capi.default_opts(do_calib_camera_pose=1), [o2 for o2, _ in marg], [s for _, s in marg], anchors)
    assert st == capi.OVB_ERR_NEG_DIAG
    assert eng.cov_dim() == P.shape[0] and np.array_equal(_bits(eng.cov_get()), _bits(P))
    assert np.isnan(anchors.new_value).all()
    eng.close()


def test_host_mirror_against_its_three_step_tail(tmp_path):
    """include/ovb200_host.hpp: ovb200::marginalize_window against StateHelper::marginalize_slam, UpdaterSLAM::change_anchors
    and StateHelper::marginalize_old_clone on the same state (tests/cpp/window_shim_test.cpp), bit for bit."""
    import os
    import subprocess
    from open_vins_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(build.build())
    exe = str(tmp_path / "window_shim_test")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "window_shim_test.cpp"),
                    "-L", libdir, "-lovb200", "-Wl,-rpath," + libdir, "-o", exe], check=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and "window_shim_test: ok" in res.stdout, res.stdout + res.stderr


@pytest.mark.parametrize("rep", [capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH, capi.REP_ANCHORED_FULL_INVERSE_DEPTH])
def test_singular_new_anchor_jacobian_leaves_p_untouched(rep):
    """A NaN landmark value makes H_f in the new anchor singular: ovb_slam_anchor_change refuses it, and so does the window
    call, with P's bytes, N and the new values unchanged. MSCKF inverse depth finds it on the device (the kernels that would
    read the landmark's Phi do nothing), full inverse depth on the host before anything is enqueued."""
    case, anchors, marg = _setup(31, 4, 100, 4, 75, 8, 3)
    l = int(np.flatnonzero(anchors.feat_rep == rep)[0])
    anchors.value[l] = np.nan
    opts = capi.default_opts(do_calib_camera_pose=1, feat_rep=rep)
    with pytest.raises(capi.OvbError) as ei:
        capi.slam_anchor_change(case.frame, opts, anchors.lm_off[l], anchors.value[l], anchors.value_fej[l], anchors.old_cam[l], anchors.old_clone[l],
                                anchors.new_cam[l], anchors.new_clone[l])
    assert ei.value.code == capi.OVB_ERR_ARG
    eng = capi.Engine(max_state=800, max_feats=16, max_meas=256)
    eng.cov_set(case.P)
    _untouched(eng, case.P, lambda: eng.marginalize_window(case.frame, capi.default_opts(do_calib_camera_pose=1), [o for o, _ in marg],
                                                           [s for _, s in marg], anchors))
    assert np.isnan(anchors.new_value).all() and np.isnan(anchors.new_value_fej).all()
    # the context still works: the same call without the NaN goes through
    anchors.value[l] = case.landmarks.value[3 * l]
    assert eng.marginalize_window(case.frame, capi.default_opts(do_calib_camera_pose=1), [o for o, _ in marg], [s for _, s in marg],
                                  anchors) == capi.OVB_OK
    eng.close()
