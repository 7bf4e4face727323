"""Pure-Python mirror of the host-side routing of the EKF update (launch_ekf_update, csrc/k_ekf.cu), so that tests can
choose (n, r, max_state) that reach each kernel chain, and an extended-precision reference of the update and its gate.

Mirrored, line for line:
  launch_ekf_update        one-shot products, factor and solve choice, byte
                           formulas of k_ekf_chol / k_ekf_trsm                 k_ekf.cu:428-475
  launch_chol_ekf_dmma     r + 1 <= CQ_MAXRB * 8, r <= CQ_MAXN, even ld       k_cholqr.cu:1106-1121
  launch_trsm_rows         the DMMA factor's row solve                         k_cholqr.cu:1123-1135
  cq_launch_trsm           k_cq_trsm instance from ceil(nt / 8)                k_cholqr.cu:674-685
  launch_chol_solve_wide   r <= CQ_WMAX - 8, even ld, r < ld                  k_cholqr.cu:1209-1224
  cq_chol_blocked          128-column blocks, the residual row below them     k_cholqr.cu:1169-1183
  cq_trsm_blocked          the blocked solve                                   k_cholqr.cu:1185-1192
  ovb_ekf_update           r > n is compressed (CholeskyQR2) to r = n          ovb_api.cu:1993-1997
  ovb_cov_initialize       the gate on rows k.., Householder TSQR when r - k > n ovb_api.cu:2106-2129
A change to any of them has to be repeated here; tests/test_ekf_routes_cpu.py checks the mirror's invariants.

Kernel names are Itanium length-prefixed ("10k_ekf_gemm", "11k_ekf_gemm1"), as they appear in the mangled names the
profile reports, so that a name never matches a longer one it prefixes.
"""
from __future__ import annotations

from functools import lru_cache
from typing import NamedTuple

import numpy as np

from tests.cholqr_geometry import CQ_MAXN, CQ_WB, CQ_WMAX, instance_of

EK1_KMAX = 160
CQ_MAXRB = 22
TR_ROWS = 8
EKF_SMEM_LIMIT = 200 * 1024  # dynamic shared memory granted to k_ekf_chol / k_ekf_trsm (k_ekf.cu:422-423)
ONE_SHOT_SMEM_LIMIT = 100 * 1024  # ... and to k_ekf_gemm1 / k_ekf_downdate1 (k_ekf.cu:424-425)
OVB_MAX_COLS = 512

CHAINS = ("E1", "E2", "E3", "E4", "O1", "O2", "O3", "O4", "O5", "O6")
GATE_ROUTES = ("A", "B", "C", "D")  # DMMA, blocked, k_ekf_chol in shared memory, k_ekf_chol in global memory


def mangled(name: str) -> str:
    return f"{len(name)}{name}"


def cq_trsm(nt: int) -> str:
    a, b = instance_of(nt)
    return f"9k_cq_trsmILi{a}ELi{b}EE"


# every kernel a chain may launch from the products to the downdate (k_ekf_prep excluded): the route proof checks that
# the launched subset of these is exactly the chain's
ALL_KERNELS = frozenset([mangled(k) for k in ("k_ekf_gemm", "k_ekf_gemm1", "k_ekf_downdate", "k_ekf_downdate1", "k_ekf_chol", "k_ekf_trsm",
                                              "k_cq_chol_ekf", "k_cq_gemm_nt", "k_cq_copy_row", "k_cq_inv_diag")]
                        + [cq_trsm(nt) for nt in (8, 80, 120, 160)])


# ---- shared-memory footprints (bytes), k_ekf.cu
def ekf_chol_smem_bytes(r: int) -> int:
    """k_ekf_chol's working copy of S and the residual row: (r + 1) rows of pitch r | 1 (k_ekf.cu:440)"""
    return 8 * (r + 1) * (r | 1)


def ekf_trsm_smem_bytes(r: int) -> int:
    """k_ekf_trsm with L in shared memory: TR_ROWS solution rows, r reciprocal pivots, L at pitch r | 1 (k_ekf.cu:463-465)"""
    return 8 * (TR_ROWS * r + r) + 8 * r * (r | 1)


def gemm1_smem_bytes(n: int) -> int:
    return 8 * (n * 33 + 32 * (n | 1))  # k_ekf.cu:433


def downdate1_smem_bytes(r: int) -> int:
    return 8 * (64 * (r | 1) + r)  # k_ekf.cu:471


def chol_in_smem(r: int) -> bool:
    return ekf_chol_smem_bytes(r) <= EKF_SMEM_LIMIT


def trsm_L_in_smem(r: int) -> bool:
    return ekf_trsm_smem_bytes(r) <= EKF_SMEM_LIMIT


# ---- the blocked (wide) path
def wide_blocks(r: int) -> tuple[int, ...]:
    """widths of cq_chol_blocked's column blocks: CQ_WB each, the last one r mod CQ_WB when that is not zero"""
    return tuple(min(CQ_WB, r - J) for J in range(0, r, CQ_WB))


def _blocked_kernels(r: int, solve: bool) -> set[str]:
    ks = {mangled("k_cq_copy_row"), mangled("k_cq_inv_diag")}
    J = 0
    for nb in wide_blocks(r):
        ks.add(mangled("k_cq_chol_ekf"))
        ks.add(cq_trsm(nb))  # the panel below the block, the residual row at least
        if r - (J + nb) > 0:
            ks.add(mangled("k_cq_gemm_nt"))  # trailing update; the last block issues none
        if solve:
            if J > 0:
                ks.add(mangled("k_cq_gemm_nt"))
            ks.add(cq_trsm(nb))
        J += nb
    return ks


class Chain(NamedTuple):
    name: str
    one_shot: bool
    factor: str  # "dmma", "blocked", "chol_smem", "chol_global"
    solve: str   # "cq_trsm", "blocked", "trsm_smem", "trsm_global"
    kernels: frozenset


def _route(n: int, r: int, ld: int, gate_only: bool) -> Chain:
    assert 1 <= r <= n <= ld and n <= OVB_MAX_COLS
    even = ld % 2 == 0
    one_shot = n <= EK1_KMAX and r <= EK1_KMAX
    ks = {mangled("k_ekf_gemm1" if one_shot else "k_ekf_gemm")}
    dmma = r + 1 <= CQ_MAXRB * 8 and r <= CQ_MAXN and even
    wide = not dmma and r <= CQ_WMAX - 8 and even and r < ld
    if dmma:
        factor, solve = "dmma", "cq_trsm"
        ks.add(mangled("k_cq_chol_ekf"))
        if not gate_only:
            ks.add(cq_trsm(r))
    elif wide:
        factor, solve = "blocked", "blocked"
        ks |= _blocked_kernels(r, not gate_only)
    else:
        factor = "chol_smem" if chol_in_smem(r) else "chol_global"
        solve = "trsm_smem" if trsm_L_in_smem(r) else "trsm_global"
        ks.add(mangled("k_ekf_chol"))
        if not gate_only:
            ks.add(mangled("k_ekf_trsm"))
    if not gate_only:
        ks.add(mangled("k_ekf_downdate1" if one_shot else "k_ekf_downdate"))  # the wide path is never one-shot
    if even:
        name = "E1" if one_shot else "E2" if dmma else "E3" if wide else "E4"
    else:
        name = ("O1" if r <= 155 else "O2" if r <= 159 else "O3") if one_shot else ("O4" if r <= 155 else "O5" if r <= 159 else "O6")
    return Chain(name, one_shot, factor, solve, frozenset(ks))


@lru_cache(maxsize=None)
def chain(n: int, r: int, ld: int) -> Chain:
    """The kernel chain ovb_ekf_update runs for r rows (after compression) over n columns with max_state ld."""
    c = _route(n, r, ld, False)
    if c.name in ("O1", "O4"):
        assert c.factor == "chol_smem" and c.solve == "trsm_smem"
    if c.name in ("O2", "O5"):
        assert c.factor == "chol_smem" and c.solve == "trsm_global"
    return c


def update_rows(n: int, rows: int) -> int:
    """rows handed to launch_ekf_update by ovb_ekf_update: more rows than columns are compressed to n"""
    return n if rows > n else rows


class GateRoute(NamedTuple):
    route: str        # A, B, C or D
    compressed: bool  # the gate's rows were compressed by the Householder TSQR (r_up > n)
    r: int            # rows of the factored system
    kernels: frozenset


@lru_cache(maxsize=None)
def gate_route(n: int, r_up: int, ld: int) -> GateRoute:
    """The gate of ovb_cov_initialize on r_up = r - k projected rows (launch_ekf_update with gate_only)."""
    compressed = r_up > n
    r = n if compressed else r_up
    c = _route(n, r, ld, True)
    letter = {"dmma": "A", "blocked": "B", "chol_smem": "C", "chol_global": "D"}[c.factor]
    return GateRoute(letter, compressed, r, c.kernels)


# ---------------------------------------------------------------------------------------------------------------- GPU cases
class Case(NamedTuple):
    chain: str
    ld: int     # max_state
    N: int
    n: int
    rows: int   # rows given to ovb_ekf_update (> n: compressed to n)
    level: int  # sigma^2 = SIGMA_LEVELS[level] * mean diag(H P H')
    seed: int

    @property
    def r(self) -> int:
        return update_rows(self.n, self.rows)

    @property
    def compressed(self) -> bool:
        return self.rows > self.n


SIGMA_LEVELS = (1.0, 1e-4, 1e-8)
R_EDGES = (1, 7, 8, 9, 31, 32, 33, 40, 41, 80, 81, 120, 121, 155, 156, 159, 160)
R_EDGES_WIDE = (161, 255, 256, 257, 383, 384, 385, 511, 512)
E4_SIZES = (162, 256, 512)
N_RESIDUES = (0, 1, 31)
BLOCK = 4  # states of the uncorrelated block at the end of the state (N - BLOCK .. N - 1)


def _n_for(chain_name: str, r: int, i: int) -> int:
    """n of the i-th case of a chain at r: r itself on every other case where the chain allows r = n"""
    narrow = chain_name in ("E1", "O1", "O2", "O3")
    if narrow:
        return r if i % 2 == 0 or r >= EK1_KMAX else min(EK1_KMAX, r + 3 + (i % 5))
    if r > EK1_KMAX and i % 2 == 0:
        return r  # E3 / O6: r = n
    return min(OVB_MAX_COLS, max(r + 3 + (i % 7), 161 + (i % 13) * 17))


def _N_for(n: int, i: int, ld: int) -> int:
    want = N_RESIDUES[i % 3]
    N = n + BLOCK
    while N % 32 != want:
        N += 1
    return min(N, ld)


def _build_cases() -> tuple[Case, ...]:
    out = []
    edges = {c: R_EDGES for c in CHAINS}
    edges["E3"] = R_EDGES_WIDE
    edges["O6"] = (160, 161, 257, 512)
    seed = 1
    for name in CHAINS:
        if name == "E4":
            for i, s in enumerate(E4_SIZES):
                out.append(Case(name, s, s, s, s if i != 1 else 2 * s, 2 if i == 2 else i, seed))
                seed += 1
            continue
        ld = 640 if name[0] == "E" else 641
        rs = [r for r in edges[name] if any(chain(n, r, ld).name == name for n in (r, 161, 200, max(r, 161)) if r <= n <= OVB_MAX_COLS)]
        for i, r in enumerate(rs):
            n = _n_for(name, r, i)
            N = _N_for(n, i, ld)
            level = 2 if r == rs[-1] else i % 3
            # a compressed input (rows > n) on the chain's largest-r case of E1, E3, O1 (n = r: compressed to r = n)
            rows = 2 * n + 1 if (name in ("E1", "E3", "O1") and i == len(rs) - 2) else r
            if rows > r:
                n = r
                N = _N_for(n, i, ld)
            out.append(Case(name, ld, N, n, rows, level, seed))
            seed += 1
    return tuple(out)


CASES = _build_cases()


# gate cases: (route, compressed, ld, N, n, r_up, k)
GATE_CASES = (
    ("A", False, 640, 120, 60, 45, 3), ("A", True, 640, 120, 60, 97, 3),
    ("B", False, 640, 400, 300, 257, 3), ("B", True, 640, 300, 200, 260, 1),
    ("C", False, 641, 120, 60, 45, 3), ("C", True, 641, 120, 60, 97, 2),
    ("D", False, 641, 300, 200, 170, 3), ("D", True, 641, 300, 200, 260, 3),
)


# ---------------------------------------------------------------------------------------------------------------- inputs
def widths_for(n: int, rng) -> list[int]:
    """variable widths from {1, 3, 6, 8} summing to n"""
    w = []
    left = n
    while left > 0:
        c = [x for x in (1, 3, 6, 8) if x <= left]
        w.append(int(rng.choice(c)))
        left -= w[-1]
    return w


def place_variables(n: int, N_free: int, rng, exclude=()) -> tuple[list[int], list[int]]:
    """(off, sz) of variables of widths 1, 3, 6, 8 totalling n columns, scattered over states [0, N_free) apart from
    `exclude`, listed in a shuffled (non-ascending) order"""
    excl = set(exclude)
    free = [i for i in range(N_free) if i not in excl]
    assert len(free) >= n
    w = widths_for(n, rng)
    gaps = rng.multinomial(len(free) - n, np.ones(len(w) + 1) / (len(w) + 1))
    # lay the variables over the free states in order, with random gaps, then split any that straddle an excluded state
    off, sz, p = [], [], 0
    for wi, g in zip(w, gaps):
        p += int(g)
        idx = free[p:p + wi]
        p += wi
        start = idx[0]
        for a, b in zip(idx, idx[1:] + [None]):
            if b != a + 1:
                off.append(start)
                sz.append(a - start + 1)
                start = b
    order = rng.permutation(len(off))
    if len(off) > 1 and np.all(np.diff(order) > 0):
        order = order[::-1]
    return [off[i] for i in order], [sz[i] for i in order]


def columns(off, sz) -> np.ndarray:
    return np.concatenate([np.arange(o, o + s) for o, s in zip(off, sz)])


@lru_cache(maxsize=None)
def make_P(N: int, seed: int, block: int = BLOCK) -> np.ndarray:
    """P = D C D: C a random correlation with eigenvalues from 1e-8 to 1 before normalisation, standard deviations D from
    1e-5 to 10; the last `block` states are uncorrelated with all others. Exactly symmetric."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
    A = (Q * np.logspace(-8, 0, N)[rng.permutation(N)]) @ Q.T
    if block:
        A[N - block:, :N - block] = 0.0
        A[:N - block, N - block:] = 0.0
    d = np.sqrt(np.diag(A))
    C = A / np.outer(d, d)
    D = np.logspace(-5, 1, N)[rng.permutation(N)]
    P = C * np.outer(D, D)
    P = np.triu(P) + np.triu(P, 1).T
    P.setflags(write=False)
    return P


def int_system(rows: int, n: int, rng) -> tuple[np.ndarray, np.ndarray]:
    """H [rows x n], res with integer entries in [-4, 4] and power-of-two column scales 2^-3..2^3: [H r]'[H r] is exact in
    float64 (all terms are multiples of the smallest scale below 2^53 of them)."""
    A = rng.integers(-4, 5, size=(rows, n + 1)).astype(np.float64)
    A *= 2.0 ** rng.integers(-3, 4, size=n + 1)
    return A[:, :n].copy(), A[:, n].copy()


class Inputs(NamedTuple):
    P: np.ndarray
    off: list
    sz: list
    cols: np.ndarray
    H: np.ndarray
    res: np.ndarray
    sigma2: float
    Rdiag: np.ndarray
    block: tuple  # states uncorrelated with every other one and unobserved (empty when the update observes them)


@lru_cache(maxsize=None)
def case_inputs(case: Case) -> Inputs:
    rng = np.random.default_rng(case.seed)
    blk = BLOCK if case.N - case.n >= BLOCK else 0
    P = make_P(case.N, case.seed, blk)
    off, sz = place_variables(case.n, case.N - blk, rng)
    cols = columns(off, sz)
    if case.compressed:
        H, res = int_system(case.rows, case.n, rng)
    else:
        H = rng.standard_normal((case.rows, case.n))
    hph = np.einsum("ij,jk,ik->i", H, P[np.ix_(cols, cols)], H).mean()
    if not case.compressed:
        res = rng.standard_normal(case.rows) * np.sqrt(hph)
    sigma2 = SIGMA_LEVELS[case.level] * hph
    Rdiag = sigma2 * rng.uniform(0.5, 2.0, size=case.rows)
    for a in (H, res, Rdiag):
        a.setflags(write=False)
    return Inputs(P, off, sz, cols, H, res, float(sigma2), Rdiag, tuple(range(case.N - blk, case.N)))


@lru_cache(maxsize=None)
def case_reference(case: Case, noise: str):
    """the long-double reference of a case, noise "sigma2" or "rdiag"; the compressed cases go through the long-double
    Cholesky factor of [H r]'[H r]"""
    x = case_inputs(case)
    nz = x.sigma2 if noise == "sigma2" else x.Rdiag
    if case.compressed:
        R, z, s2 = compressed_ld(x.H, x.res, nz)
        return reference_update(x.P, x.cols, R, z, s2)
    return reference_update(x.P, x.cols, x.H, x.res, nz)


# ---------------------------------------------------------------------------------------------------------------- reference
def have_longdouble() -> bool:
    return np.finfo(np.longdouble).nmant >= 63


def chol_ld(S) -> np.ndarray:
    """lower Cholesky factor in long double (left-looking, one matrix-vector product per column)"""
    S = np.asarray(S, dtype=np.longdouble)
    r = S.shape[0]
    L = np.zeros_like(S)
    for j in range(r):
        v = S[j:, j] - L[j:, :j] @ L[j, :j]
        if not v[0] > 0:
            raise np.linalg.LinAlgError(f"reference S not positive definite at pivot {j}")
        L[j, j] = np.sqrt(v[0])
        L[j + 1:, j] = v[1:] / L[j, j]
    return L


def forward_ld(L, B) -> np.ndarray:
    """X = L^-1 B (B: r x m), long double"""
    B = np.asarray(B, dtype=np.longdouble)
    X = np.zeros_like(B)
    for j in range(L.shape[0]):
        X[j] = (B[j] - L[j, :j] @ X[:j]) / L[j, j]
    return X


def compressed_ld(H, res, noise):
    """(R, z, s2) of the whitened system in long double: R'R = Hw'Hw, R'z = Hw'rw from the Cholesky factor of [Hw rw]'[Hw rw];
    s2 the noise variance left (sigma^2, or 1 after whitening by a diagonal R)"""
    Hl, rl = np.asarray(H, dtype=np.longdouble), np.asarray(res, dtype=np.longdouble)
    if np.ndim(noise):
        s = np.sqrt(np.asarray(noise, dtype=np.longdouble))
        Hl, rl, s2 = Hl / s[:, None], rl / s, 1.0
    else:
        s2 = noise
    A = np.column_stack([Hl, rl])
    Lg = chol_ld(A.T @ A)
    n = H.shape[1]
    return Lg[:n, :n].T, Lg[n, :n], s2


def scaled_kappa(S) -> float:
    S = np.asarray(S, dtype=np.float64)
    d = np.sqrt(np.diag(S))
    return float(np.linalg.cond(S / np.outer(d, d)))


def reference_update(P, cols, H, res, noise):
    """EKF update in long double: M = P[:, c] H', S = H P[c, c] H' + R, S = L L', Y = M L^-T, w = L^-1 res, P+ = P - Y Y',
    dx = Y w. noise: sigma^2 (scalar) or the diagonal of R. Returns dict(P, dx, wnorm, kappa, chi2)."""
    Pl = np.asarray(P, dtype=np.longdouble)
    Hl, rl = np.asarray(H, dtype=np.longdouble), np.asarray(res, dtype=np.longdouble)
    M = Pl[:, cols] @ Hl.T
    S = Hl @ M[cols, :]
    S = 0.5 * (S + S.T)
    S[np.diag_indices_from(S)] += np.asarray(noise, dtype=np.longdouble)
    L = chol_ld(S)
    Y = forward_ld(L, M.T).T
    w = forward_ld(L, rl[:, None])[:, 0]
    return dict(P=Pl - Y @ Y.T, dx=Y @ w, wnorm=float(np.sqrt(w @ w)), kappa=scaled_kappa(S), chi2=float(w @ w))


def bar_of(kappa: float) -> float:
    return max(1e-12, 1e-14 * kappa)


def errors(P0, Pg, dxg, ref, skip=()):
    """(P+ error, dx error), each scaled per entry: |dP_ij| / sqrt(|P_ii P_jj|), |ddx_i| / (sqrt|P_ii| |w|); rows and columns
    in `skip` are left out"""
    d = np.sqrt(np.abs(np.diag(np.asarray(P0, dtype=np.longdouble))))
    keep = np.ones(len(d), dtype=bool)
    keep[list(skip)] = False
    EP = np.abs(np.asarray(Pg, dtype=np.longdouble) - ref["P"]) / np.outer(d, d)
    Edx = np.abs(np.asarray(dxg, dtype=np.longdouble) - ref["dx"]) / (d * max(ref["wnorm"], 1e-300))
    return float(EP[np.ix_(keep, keep)].max()), float(Edx[keep].max())
