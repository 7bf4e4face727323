"""The algebra the device's delayed initialisation relies on: StateHelper::initialize (state/StateHelper.cpp:393-577) built
from a three-column Householder QR of H_f (the per-feature kernel's split) equals the oracle's Givens split. For
ANCHORED_INVERSE_DEPTH_SINGLE the QR covers all three columns (two bearing, one depth): rows 0-1 are dropped, row 2 is the
1-wide init row and rows 3.. are the projected rows, where the reference projects the bearing columns out first and then
splits the depth column. No GPU."""
import numpy as np
import pytest
import scipy.stats

from tests import oracle_reps
from tests.test_slam_cpu import _init_case


def _householder_initialize(P, off, sz, H_x, H_f, res, s2, single, compress):
    """Augmented covariance, dx_new and the EKF update of the projected rows from Q'[H_x | H_f | r], Q = Householder QR of
    the three columns of H_f. compress: the projected rows are first reduced to their R factor (rows > columns)."""
    N = P.shape[0]
    c = np.concatenate([np.arange(o, o + s) for o, s in zip(off, sz)])
    Q, _ = np.linalg.qr(H_f, mode="complete")
    X, L, z = Q.T @ H_x, Q.T @ H_f, Q.T @ res
    i0 = 2 if single else 0
    HR, HL, r0 = X[i0:3], L[i0:3, i0:3], z[i0:3]
    Hup, rup = X[3:], z[3:]
    k = 3 - i0
    # gate: chi2 of the projected rows against S = Hup P Hup' + s2 I
    S = Hup @ P[np.ix_(c, c)] @ Hup.T + s2 * np.eye(len(rup))
    chi2 = rup @ np.linalg.solve(S, rup)
    # initialize_invertible
    Hinv = np.linalg.inv(HL)
    Pa = np.zeros((N + k, N + k))
    Pa[:N, :N] = P
    m = P[:, c] @ HR.T
    Pa[:N, N:] = -m @ Hinv.T
    Pa[N:, :N] = Pa[:N, N:].T
    Pa[N:, N:] = Hinv @ (HR @ m[c] + s2 * np.eye(k)) @ Hinv.T
    dxn = Hinv @ r0
    # EKFUpdate with the projected rows on the augmented covariance
    if compress:
        R = np.linalg.qr(np.hstack([Hup, rup[:, None]]), mode="r")
        Hup, rup = R[:len(c), :len(c)], R[:len(c), len(c)]
    Sa = Hup @ Pa[np.ix_(c, c)] @ Hup.T + s2 * np.eye(len(rup))
    K = Pa[:, c] @ Hup.T @ np.linalg.inv(Sa)
    Pn = Pa - K @ Hup @ Pa[c, :]
    return chi2, Pn, dxn, K @ rup


@pytest.mark.parametrize("single", [False, True], ids=["3wide", "single"])
@pytest.mark.parametrize("seed,r", [(1, 12), (2, 20), (3, 60), (4, 90)])
def test_householder_split_equals_givens_split(oracle, seed, r, single):
    P, off, sz, H_x, H_f, res = _init_case(seed, r=r)
    n = sum(sz)
    s2 = 1.0  # pixel units, as the delayed initialisation runs: S stays well conditioned enough for a 1e-12 bar
    if single:
        H_R, H_L, res_o = oracle_reps.slam_single_init_system(H_f, H_x, res)
    else:
        H_R, H_L, res_o = H_x, H_f, res
    st, acc, P_o, dxn_o, dx_o = oracle.cov_initialize(P, off, sz, H_R, H_L, res_o, sigma2=s2, chi2_mult=1e9)
    assert st == 0 and acc
    rup = r - 3
    for compress in ([False, True] if rup > n else [False]):
        chi2, P_h, dxn_h, dx_h = _householder_initialize(P, off, sz, H_x, H_f, res, s2, single, compress)
        assert P_h.shape == P_o.shape
        assert np.linalg.norm(P_h - P_o) <= 1e-12 * np.linalg.norm(P_o)
        assert np.linalg.norm(dxn_h - dxn_o) <= 1e-12 * np.linalg.norm(dxn_o)
        assert np.linalg.norm(dx_h - dx_o) <= 1e-12 * np.linalg.norm(dx_o)
        assert np.isfinite(chi2) and chi2 > 0


@pytest.mark.parametrize("single", [False, True], ids=["3wide", "single"])
def test_gate_statistic_is_the_same(oracle, single):
    """The gate decision of the Householder split is the oracle's: a consistent system passes and a shifted one fails at the
    threshold of the initialize system's row count."""
    P, off, sz, H_x, H_f, res = _init_case(7, r=30)
    s2 = 0.05 ** 2
    for shift, want in ((0.0, True), (3.0, False)):
        rr = res + shift
        if single:
            H_R, H_L, res_o = oracle_reps.slam_single_init_system(H_f, H_x, rr)
        else:
            H_R, H_L, res_o = H_x, H_f, rr
        st, acc, _, _, _ = oracle.cov_initialize(P, off, sz, H_R, H_L, res_o, sigma2=s2, chi2_mult=1.0)
        chi2, _, _, _ = _householder_initialize(P, off, sz, H_x, H_f, rr, s2, single, False)
        assert st == 0 and bool(acc) == want
        assert (chi2 <= scipy.stats.chi2.ppf(0.95, len(res_o))) == want
