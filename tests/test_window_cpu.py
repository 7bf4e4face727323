"""ovb_marginalize_window without a GPU: the ovb_anchor_changes layout against the header, and the batched formulation its
kernels compute (phase-1 rows, phase-2 blocks, one compaction) restated in numpy against the oracle's sequence
perform_anchor_change + EKFPropagation per landmark, then marginalize per range (UpdaterSLAM::change_anchors,
StateHelper::marginalize_slam / marginalize_old_clone)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from open_vins_b200 import capi, sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANCHORED = [capi.REP_ANCHORED_3D, capi.REP_ANCHORED_FULL_INVERSE_DEPTH, capi.REP_ANCHORED_MSCKF_INVERSE_DEPTH,
            capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE]


def test_anchor_changes_layout_matches_header(tmp_path):
    fields = [f for f, _ in capi.ovb_anchor_changes._fields_]
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ovb200.h"\nint main(void) {\n  printf("%zu\\n", sizeof(ovb_anchor_changes));\n'
                   + "".join(f'  printf("%zu\\n", offsetof(ovb_anchor_changes, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "probe"
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == C.sizeof(capi.ovb_anchor_changes)
    assert got[1:] == [getattr(capi.ovb_anchor_changes, f).offset for f in fields]


def window_np(P, moved, ranges):
    """The kernels' formulation. moved: [(lm_off, idx (q,), Phi (p, q))] in call order, idx = covariance index of each of Phi's
    columns; ranges: [(off, size)] to marginalize. Returns P after the anchor changes and the marginalization."""
    N = P.shape[0]
    rows = [(l, j) for l, (_, _, Phi) in enumerate(moved) for j in range(Phi.shape[0])]
    K = len(rows)
    g = np.array([moved[l][0] + j for l, j in rows], dtype=np.int64)
    # phase 1: R[u][a] = C_l[a][j] = sum_k P[a][idx_l[k]] Phi_l[j][k] on the prior, for every a
    R = np.zeros((K, N))
    for u, (l, j) in enumerate(rows):
        R[u] = P[:, moved[l][1]] @ moved[l][2][j]
    # phase 2: the K x K blocks. Own block: Phi_l C_l[idx_l] (Q = 0); landmarks E < L: L's step reads E's moved row
    B = np.zeros((K, K))
    for u, (lu, i) in enumerate(rows):
        for v, (lv, j) in enumerate(rows):
            if lu == lv:
                B[u, v] = moved[lu][2][i] @ R[v][moved[lu][1]]
            else:
                L, e, jL = (lu, v, i) if lu > lv else (lv, u, j)
                B[u, v] = R[e][moved[L][1]] @ moved[L][2][jL]
    Pp = P.copy()
    for u in range(K):
        Pp[g[u], :] = R[u]
        Pp[:, g[u]] = R[u]
    if K:
        Pp[np.ix_(g, g)] = B
    # one compaction; a lower-triangle entry with a removed range between its row and column is read mirrored
    gone = np.concatenate([np.arange(o, o + s) for o, s in ranges]) if ranges else np.zeros(0, dtype=np.int64)
    keep = np.setdiff1d(np.arange(N), gone)
    I, J = np.meshgrid(np.arange(len(keep)), np.arange(len(keep)), indexing="ij")
    tr = (I > J) & (keep[I] - keep[J] != I - J)
    out = Pp[np.ix_(keep, keep)]
    out[tr] = Pp[keep[J][tr], keep[I][tr]]
    return out


def window_case(reps, n_clones=6, n_cams=2, seed=0, ext=True, k_anchor=3, k_lost=2):
    """A SLAM state with one landmark per entry of reps. The first k_anchor landmarks are re-anchored from the oldest clone to
    the newest (camera old + 1 + l), the next k_lost are lost; the oldest clone is marginalized with them."""
    case = sim.make_slam_case(n_landmarks=len(reps), n_clones=n_clones, n_cams=n_cams, seed=seed, rep=list(reps), calib_ext=ext)
    lm, fr = case.landmarks, case.frame
    width = np.array([1 if r == capi.REP_ANCHORED_INVERSE_DEPTH_SINGLE else 3 for r in reps])
    moved = np.arange(k_anchor)
    lost = np.arange(k_anchor, k_anchor + k_lost)
    old_cam = lm.anchor_cam[moved]
    anchors = capi.AnchorChanges(lm.lm_off[moved], np.asarray(reps)[moved], lm.value[moved], lm.value_fej[moved], old_cam,
                                 np.zeros(k_anchor), (old_cam + 1 + moved) % n_cams, np.full(k_anchor, n_clones - 1))
    marg = [(int(lm.lm_off[f]), int(width[f])) for f in lost] + [(int(fr.clone_off[0]), 6)]
    return case, anchors, marg


def sequence(case, anchors, marg, fej, ext, anchor_change, propagate, marginalize):
    """The existing calls in the reference's order: each anchor change then its EKFPropagation (Q = 0), then the ranges,
    highest offset first. Returns the new values and Phi / column order of every landmark."""
    fr = case.frame
    nv, nvf, phis = [], [], []
    for l in range(len(anchors.lm_off)):
        opts = capi.default_opts(do_fej=fej, do_calib_camera_pose=ext, feat_rep=int(anchors.feat_rep[l]))
        v, vf, off, sz, Phi = anchor_change(fr, opts, anchors.lm_off[l], anchors.value[l], anchors.value_fej[l], anchors.old_cam[l],
                                            anchors.old_clone[l], anchors.new_cam[l], anchors.new_clone[l])
        propagate(int(anchors.lm_off[l]), Phi, np.zeros((Phi.shape[0], Phi.shape[0])), off, sz)
        nv.append(v)
        nvf.append(vf)
        phis.append((int(anchors.lm_off[l]), np.concatenate([np.arange(o, o + s) for o, s in zip(off, sz)]), Phi))
    for o, s in sorted(marg, reverse=True):
        marginalize(o, s)
    return np.array(nv).reshape(-1, 3), np.array(nvf).reshape(-1, 3), phis


@pytest.mark.parametrize("rep", ANCHORED + ["mixed"])
@pytest.mark.parametrize("ext,fej", [(1, 1), (0, 1), (1, 0), (0, 0)])
def test_batched_formulation_matches_the_oracle_sequence(oracle, rep, ext, fej):
    reps = [2, 5, 3, 5, 4, 2, 5, 3, 4, 5] if rep == "mixed" else [rep] * 10
    case, anchors, marg = window_case(reps, n_clones=7, n_cams=2, seed=40 + len(str(rep)) + 3 * ext + fej, ext=bool(ext), k_anchor=5, k_lost=3)
    box = {"P": case.P.copy()}

    def propagate(lm_off, Phi, Q, off, sz):
        st, box["P"] = oracle.cov_propagate(box["P"], lm_off, Phi, Q, off, sz)
        assert st == 0

    def marginalize(o, s):
        box["P"] = oracle.cov_marginalize(box["P"], o, s)

    _, _, phis = sequence(case, anchors, marg, fej, ext, oracle.anchor_change, propagate, marginalize)
    got = window_np(case.P, phis, marg)
    ref = box["P"]
    assert got.shape == ref.shape == (case.P.shape[0] - sum(s for _, s in marg),) * 2
    assert np.linalg.norm(got - ref) <= 1e-13 * np.linalg.norm(ref)


def test_compaction_alone_is_the_sequence_of_marginalizations(oracle):
    """No anchor changes, an asymmetric P: the mirrored reads of the one-pass compaction are those of k_cov_marg applied
    range by range, highest first (exactly, not to rounding)."""
    rng = np.random.default_rng(4)
    P = rng.standard_normal((50, 50))
    marg = [(3, 2), (10, 6), (30, 1), (44, 3)]
    ref = P.copy()
    for o, s in sorted(marg, reverse=True):
        ref = oracle.cov_marginalize(ref, o, s)
    assert np.array_equal(window_np(P, [], marg), ref)
