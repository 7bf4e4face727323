"""References for the covariance structure operations on the resident P (csrc/k_ekf.cu, ovb_api.cu): EKFPropagation
(ovb_cov_propagate), clone and its time-offset term (ovb_cov_clone), marginalize (ovb_cov_marginalize), the marginal read
(ovb_cov_get_marginal) and initialize_invertible (the augmentation of ovb_cov_initialize).

Index semantics are the reference's (oracle/ovo_core.hpp), and they are what a symmetric P cannot check:
  clone            new row N+j copies row old_off+j, new column N+j copies column old_off+j
  marginalize      the kept block below the removed range and left of it is read transposed (StateHelper.cpp:303-306)
  propagation      C = P[:, old] Phi', S = Q_u + Phi C[old, :], Q_u = Q's upper triangle mirrored (StateHelper.cpp:80-100)
  time offset      P[:, new] += P[:, dt] dnc', then P[new, :] += dnc P[dt, :] on the updated P (StateHelper.cpp:611-614)
  initialize       P_xL = -P[:, cols] H_R' H_L^-T,  P_LL = H_L^-1 M_u H_L^-T,  M = H_R P[cols, cols] H_R' + s2 I,  M_u its
                   upper triangle mirrored (StateHelper.cpp:484-577)
Copies are mirrored bit for bit. Products are computed in long double (64-bit mantissa) with a componentwise bar

    |got - ref| <= C_BAR * (K + 2) * u * (|A| |B|)_ij,     u = 2^-53,

K the inner dimension of the whole chain (2q for S = Q_u + Phi P Phi', say) and |A| |B| the same chain on absolute values,
formed in long double. An index or orientation error changes an entry by O(1) of its size, i.e. by ~1e13 bars.
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
U = 2.0 ** -53
C_BAR = 4  # covers the double-precision chain (FMA-contracted or not) and H_L^-1's Gauss-Jordan rounding at kappa < 10


def have_longdouble() -> bool:
    return np.finfo(LD).nmant >= 63


def asymmetric_prior(N: int, seed: int) -> np.ndarray:
    """SPD (eigenvalues of the symmetric part >= 1 before scaling) plus a small antisymmetric part, scaled by a diagonal
    spread over 1.5 decades: P[i][j] != P[j][i] and every entry has its own magnitude, so a transposed or shifted read
    changes bits."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((N, N))
    S = A @ A.T / N + np.eye(N)
    K = rng.standard_normal((N, N))
    K = 0.1 * (K - K.T) / np.sqrt(N)
    d = 10.0 ** rng.uniform(-1.5, 0.0, N)
    return (d[:, None] * (0.5 * (S + S.T) + K)) * d[None, :]


def indices(off, sz) -> np.ndarray:
    """Covariance index of each column of a variable list, in list order (the kernels' old_idx / col_state)."""
    return np.concatenate([np.arange(o, o + s) for o, s in zip(off, sz)]).astype(np.int64)


# ---- bit-exact mirrors
def clone(P: np.ndarray, old_off: int, size: int) -> np.ndarray:
    """StateHelper::clone without the time-offset term (ovo_core.hpp cov_clone)."""
    N = P.shape[0]
    out = np.zeros((N + size, N + size))
    out[:N, :N] = P
    out[N:, N:] = P[old_off:old_off + size, old_off:old_off + size]
    out[:N, N:] = P[:, old_off:old_off + size]
    out[N:, :N] = P[old_off:old_off + size, :]
    return out


def marginalize(P: np.ndarray, off: int, size: int) -> np.ndarray:
    """StateHelper::marginalize (ovo_core.hpp cov_marginalize): output (i, j) from (src i, src j), read transposed for
    i >= off > j."""
    N = P.shape[0]
    src = np.r_[0:off, off + size:N]
    out = P[np.ix_(src, src)].copy()
    out[off:, :off] = P[np.ix_(src[:off], src[off:])].T
    return out


def get_marginal(P: np.ndarray, off, sz) -> np.ndarray:
    idx = indices(off, sz)
    return P[np.ix_(idx, idx)].copy()


# ---- long-double references: (value, absolute-value chain), both long double
def _ld(a):
    return np.asarray(a, dtype=LD)


def upper_mirrored(Q) -> np.ndarray:
    Q = np.asarray(Q)
    return np.triu(Q) + np.triu(Q, 1).T


def propagate(P, new_off: int, Phi, Q, idx):
    """EKFPropagation. Returns the full propagated P (long double) and its bar matrix. Entries outside the rows and
    columns new_off..new_off+p have bar 0 (they must keep their bits)."""
    P, Phi, Qu = _ld(P), _ld(Phi), _ld(upper_mirrored(Q))
    p, q = Phi.shape
    Pc, aPc, aPhi = P[:, idx], np.abs(P[:, idx]), np.abs(Phi)
    C, aC = Pc @ Phi.T, aPc @ aPhi.T
    S, aS = Qu + Phi @ C[idx, :], np.abs(Qu) + aPhi @ aC[idx, :]
    out, bar = P.copy(), np.zeros(P.shape, dtype=LD)
    nb = slice(new_off, new_off + p)
    out[:, nb], out[nb, :] = C, C.T
    out[nb, nb] = S
    bar[:, nb], bar[nb, :] = C_BAR * (q + 2) * U * aC, C_BAR * (q + 2) * U * aC.T
    bar[nb, nb] = C_BAR * (2 * q + 2) * U * aS
    return out, bar


def clone_dt(P, old_off: int, size: int, dnc, dt_off: int):
    """StateHelper::clone followed by augment_clone's time-offset term: columns first, then the rows, which read row
    dt_off after the column step. Returns (value, bar), (N+size)^2 long double; the prior block has bar 0."""
    N = P.shape[0]
    X = _ld(clone(np.asarray(P), old_off, size))
    A = np.abs(X)
    d = _ld(dnc)
    for M, dd in ((X, d), (A, np.abs(d))):
        M[:, N:] += M[:, dt_off, None] * dd[None, :]
        M[N:, :] += dd[:, None] * M[None, dt_off, :]
    bar = C_BAR * (2 + 2) * U * A
    bar[:N, :N] = 0
    return X, bar


def givens_split(H_R, H_L):
    """The Givens split of ovb_cov_initialize (ovb_api.cu make_givens and its rotation loop, StateHelper.cpp:429-440) in
    double, operation for operation. With r = k it rotates H_L to upper-triangular form and H_R along with it; the
    residual is not needed here."""
    HR, HL = np.array(H_R, dtype=np.float64), np.array(H_L, dtype=np.float64)
    r, k = HL.shape

    def make_givens(p, q):
        if q == 0.0:
            return (-1.0 if p < 0.0 else 1.0), 0.0
        if p == 0.0:
            return 0.0, (1.0 if q < 0.0 else -1.0)
        if abs(p) > abs(q):
            t = q / p
            u = np.sqrt(1.0 + t * t)
            u = -u if p < 0.0 else u
            c = 1.0 / u
            return c, -t * c
        t = p / q
        u = np.sqrt(1.0 + t * t)
        u = -u if q < 0.0 else u
        s = -1.0 / u
        return -t * s, s

    for c0 in range(k):
        for m in range(r - 1, c0, -1):
            c, s = make_givens(HL[m - 1, c0], HL[m, c0])
            for M, j0 in ((HL, c0), (HR, 0)):
                x0, y0 = M[m - 1, j0:].copy(), M[m, j0:].copy()
                M[m - 1, j0:] = c * x0 - s * y0
                M[m, j0:] = s * x0 + c * y0
    return HR, HL


def inverse_ld(A) -> np.ndarray:
    """A^-1 in long double (Gauss-Jordan, partial pivoting; k <= 3)."""
    A = _ld(A).copy()
    k = A.shape[0]
    X = np.eye(k, dtype=LD)
    for c in range(k):
        piv = c + int(np.argmax(np.abs(A[c:, c])))
        A[[c, piv]], X[[c, piv]] = A[[piv, c]], X[[piv, c]]
        X[c] /= A[c, c]
        A[c] /= A[c, c]
        for i in range(k):
            if i != c:
                X[i] -= A[i, c] * X[c]
                A[i] -= A[i, c] * A[c]
    return X


def initialize_invertible(P, cols, H_R, H_L, sigma2: float):
    """initialize_invertible on the split system (H_R k x n, H_L k x k). Returns the (N+k)^2 augmented P and its bar
    (0 on the prior block)."""
    N, k = P.shape[0], H_L.shape[0]
    n = len(cols)
    P, HR, Hinv = _ld(P), _ld(H_R), inverse_ld(H_L)
    aHR, aHinv = np.abs(HR), np.abs(Hinv)
    Pc, aPc = P[:, cols], np.abs(P[:, cols])
    m, am = Pc @ HR.T, aPc @ aHR.T
    M, aM = HR @ m[cols, :] + LD(sigma2) * np.eye(k, dtype=LD), aHR @ am[cols, :] + LD(sigma2) * np.eye(k, dtype=LD)
    M, aM = _ld(upper_mirrored(M)), _ld(upper_mirrored(aM))
    out, bar = np.zeros((N + k, N + k), dtype=LD), np.zeros((N + k, N + k), dtype=LD)
    out[:N, :N] = P
    out[:N, N:] = -(m @ Hinv.T)
    out[N:, :N] = out[:N, N:].T
    out[N:, N:] = Hinv @ M @ Hinv.T
    b_xl = C_BAR * (n + 2 * k + 2) * U * (am @ aHinv.T)
    bar[:N, N:], bar[N:, :N] = b_xl, b_xl.T
    bar[N:, N:] = C_BAR * (2 * n + 3 * k + 2) * U * (aHinv @ aM @ aHinv.T)
    return out, bar


def worst(got, ref, bar):
    """max |got - ref| / bar over the entries (an entry with bar 0 must be equal: inf otherwise) and where it is."""
    err = np.abs(_ld(got) - _ld(ref))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bar > 0, err / np.where(bar > 0, bar, 1), np.where(err > 0, np.inf, 0))
    i = np.unravel_index(int(np.argmax(r)), r.shape)
    return float(r[i]), tuple(int(x) for x in i)
