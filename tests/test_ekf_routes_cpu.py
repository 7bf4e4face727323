"""The routing mirror of the EKF update (tests/ekf_routes.py): every chain and gate route is reachable, the shared-memory
boundaries sit where the byte formulas put them, tests/test_gpu_ekf_routes.py's case list covers every cell, and the
long-double reference agrees with the numpy twin and with 50-digit arithmetic."""
import numpy as np
import pytest

from tests import ekf_routes as er
from tests import np_twin


def test_every_chain_reachable():
    seen = {}
    for ld in (640, 641):
        for n in range(1, er.OVB_MAX_COLS + 1):
            for r in range(1, n + 1):
                seen.setdefault(er.chain(n, r, ld).name, (n, r, ld))
    for s in er.E4_SIZES:
        seen.setdefault(er.chain(s, s, s).name, (s, s, s))
    assert set(seen) == set(er.CHAINS), seen


def test_chain_table():
    """the factor / solve / products of each chain, as the issue table of the routing lists them"""
    want = {"E1": (True, "dmma", "cq_trsm"), "E2": (False, "dmma", "cq_trsm"), "E3": (False, "blocked", "blocked"),
            "E4": (False, "chol_global", "trsm_global"), "O1": (True, "chol_smem", "trsm_smem"), "O2": (True, "chol_smem", "trsm_global"),
            "O3": (True, "chol_global", "trsm_global"), "O4": (False, "chol_smem", "trsm_smem"), "O5": (False, "chol_smem", "trsm_global"),
            "O6": (False, "chol_global", "trsm_global")}
    for c in er.CASES:
        ch = er.chain(c.n, c.r, c.ld)
        assert ch.name == c.chain and (ch.one_shot, ch.factor, ch.solve) == want[c.chain], c
        assert ch.kernels <= er.ALL_KERNELS
        assert (er.mangled("k_ekf_gemm1") in ch.kernels) == ch.one_shot
        assert (er.mangled("k_ekf_downdate1") in ch.kernels) == ch.one_shot


def test_every_gate_route_reachable():
    seen = set()
    for ld in (640, 641):
        for k in (1, 3):
            for n in range(1, er.OVB_MAX_COLS + 1, 7):
                N = ld - k
                if n > N:
                    continue
                for r_up in range(1, n + 200, 5):
                    g = er.gate_route(n, r_up, ld)
                    assert g.r <= n
                    seen.add((g.route, g.compressed))
    assert seen == {(a, b) for a in er.GATE_ROUTES for b in (False, True)}
    for route, compressed, ld, N, n, r_up, k in er.GATE_CASES:
        assert N + k <= ld and n <= N
        g = er.gate_route(n, r_up, ld)
        assert (g.route, g.compressed) == (route, compressed)
        assert not g.kernels & {er.mangled("k_ekf_trsm"), er.mangled("k_ekf_downdate"), er.mangled("k_ekf_downdate1")}
    assert {(c[0], c[1]) for c in er.GATE_CASES} == seen


def test_byte_formula_boundaries():
    assert er.chol_in_smem(159) and not er.chol_in_smem(160)
    assert er.trsm_L_in_smem(155) and not er.trsm_L_in_smem(156)
    assert all(er.chol_in_smem(r) == (r <= 159) for r in range(1, 513))
    assert all(er.trsm_L_in_smem(r) == (r <= 155) for r in range(1, 513))
    # the one-shot kernels' footprints fit the shared memory they are granted at every size they take
    assert er.gemm1_smem_bytes(er.EK1_KMAX) <= er.ONE_SHOT_SMEM_LIMIT
    assert er.downdate1_smem_bytes(er.EK1_KMAX) <= er.ONE_SHOT_SMEM_LIMIT
    # 160 | 161: the DMMA factor and the one-shot products stop at CQ_MAXN = EK1_KMAX
    assert er.chain(160, 160, 640).name == "E1" and er.chain(161, 161, 640).name == "E3"
    assert er.chain(161, 160, 640).name == "E2"
    assert er.chain(160, 160, 641).name == "O3" and er.chain(161, 161, 641).name == "O6"
    listed = {(c.chain, c.r) for c in er.CASES}
    for pair in (("O1", 155), ("O2", 156), ("O4", 155), ("O5", 156), ("O2", 159), ("O3", 160), ("O5", 159), ("O6", 160),
                 ("E1", 160), ("E3", 161), ("E2", 160), ("O6", 161)):
        assert pair in listed, pair


def test_wide_blocks():
    assert er.wide_blocks(161) == (128, 33)
    assert er.wide_blocks(256) == (128, 128)
    assert er.wide_blocks(257) == (128, 128, 1)
    assert er.wide_blocks(385) == (128, 128, 128, 1)
    assert er.wide_blocks(512) == (128,) * 4
    for r in range(161, 513):
        b = er.wide_blocks(r)
        assert sum(b) == r and len(b) == -(-r // 128) and b[-1] == (r % 128 or 128)


def test_cases_cover_every_cell():
    by = {}
    for c in er.CASES:
        assert c.r <= c.n <= c.N <= c.ld and c.n <= er.OVB_MAX_COLS
        assert er.chain(c.n, c.r, c.ld).name == c.chain
        by.setdefault(c.chain, []).append(c)
    assert set(by) == set(er.CHAINS)
    for name, cs in by.items():
        rs = {c.r for c in cs}
        ld = 640 if name[0] == "E" else 641
        edges = er.R_EDGES_WIDE if name == "E3" else er.E4_SIZES if name == "E4" else er.R_EDGES + er.R_EDGES_WIDE
        for r in edges:
            if name == "E4":
                assert r in rs
                continue
            reach = any(er.chain(n, r, ld).name == name for n in range(r, er.OVB_MAX_COLS + 1))
            if reach and name != "O6":
                assert r in rs, (name, r)
        if name == "O6":
            assert {160, 161, 257, 512} <= rs
        # both r = n and r < n wherever the chain allows them
        if any(er.chain(n, n, ld).name == name for n in range(1, 513)) or name == "E4":
            assert any(c.r == c.n for c in cs), name
        if any(er.chain(n, r, ld).name == name for n in range(1, 513) for r in range(1, n)):
            assert any(c.r < c.n for c in cs), name
        if len(cs) >= 3 and name != "E4":
            assert {c.N % 32 for c in cs} >= {0, 1, 31}, name
            assert any(c.N % 8 for c in cs), name
    assert {c.chain for c in er.CASES if c.compressed} >= {"E1", "E3", "E4"}
    assert any(c.compressed for c in er.CASES if c.chain[0] == "O")
    assert any(c.n == 160 and c.chain in ("E1", "O3") for c in er.CASES)


def _kappa(c):
    x = er.case_inputs(c)
    Pc = x.P[np.ix_(x.cols, x.cols)]
    if c.compressed:
        R = np.linalg.qr(x.H, mode="r")
        return er.scaled_kappa(R @ Pc @ R.T + x.sigma2 * np.eye(c.n))
    return er.scaled_kappa(x.H @ Pc @ x.H.T + x.sigma2 * np.eye(c.r))


def test_cases_reach_ill_conditioning():
    """every chain has a case with kappa >= 1e6 of the diagonally scaled S, and the compressed inputs keep kappa_2(H) <= 1e3"""
    worst = {}
    for c in er.CASES:
        worst[c.chain] = max(worst.get(c.chain, 0.0), _kappa(c))
        if c.compressed:
            assert np.linalg.cond(er.case_inputs(c).H) <= 1e3
    assert all(k >= 1e6 for k in worst.values()), worst


def test_inputs_structure():
    for c in er.CASES[::7]:
        x = er.case_inputs(c)
        assert np.array_equal(x.P, x.P.T)
        assert int(np.sum(x.sz)) == c.n and len(set(x.cols)) == c.n and x.cols.max() < c.N
        assert not set(x.cols) & set(x.block)
        assert set(x.sz) <= {1, 2, 3, 4, 5, 6, 7, 8}
        assert len(x.off) == 1 or not np.all(np.diff(x.off) > 0), "variables listed in ascending order"
        if x.block:
            b = list(x.block)
            rest = [i for i in range(c.N) if i not in b]
            assert not x.P[np.ix_(b, rest)].any()
            assert c.N - 1 in b


pytestmark_ld = pytest.mark.skipif(not er.have_longdouble(), reason="the reference needs an extended-precision long double")


@pytestmark_ld
@pytest.mark.parametrize("seed,N,n,r,compressed", [(0, 40, 20, 20, False), (1, 50, 24, 9, False), (2, 64, 30, 61, True), (3, 33, 17, 17, False)])
def test_reference_matches_numpy_twin(seed, N, n, r, compressed):
    """well conditioned small cases: the long-double reference and np_twin.ekf_update (float64) agree to the double bar"""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((N, N))
    P = A @ A.T / N + 0.1 * np.eye(N)
    off, sz = er.place_variables(n, N, rng)
    cols = er.columns(off, sz)
    H, res = er.int_system(r, n, rng) if compressed else (rng.standard_normal((r, n)), rng.standard_normal(r))
    Rd = rng.uniform(0.5, 2.0, size=r)
    if compressed:
        R, z, s2 = er.compressed_ld(H, res, Rd)
        ref = er.reference_update(P, cols, R, z, s2)
    else:
        ref = er.reference_update(P, cols, H, res, Rd)
    Pt, dxt = np_twin.ekf_update(P, cols, H, res, Rd)
    eP, edx = er.errors(P, Pt, dxt, ref)
    bar = er.bar_of(ref["kappa"])
    assert eP <= bar and edx <= bar, (eP, edx, bar)


@pytestmark_ld
@pytest.mark.parametrize("seed,N,n,r", [(5, 10, 6, 6), (6, 12, 7, 4)])
def test_reference_matches_50_digits(seed, N, n, r):
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 50
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((N, N))
    P = A @ A.T / N + 1e-3 * np.eye(N)
    P = np.triu(P) + np.triu(P, 1).T
    off, sz = er.place_variables(n, N, rng)
    cols = er.columns(off, sz)
    H, res = rng.standard_normal((r, n)), rng.standard_normal(r)
    s2 = 0.01
    ref = er.reference_update(P, cols, H, res, s2)
    Pm = mp.matrix(P.tolist())
    Hm = mp.zeros(r, N)
    for i in range(r):
        for j, c in enumerate(cols):
            Hm[i, int(c)] = mp.mpf(float(H[i, j]))
    S = Hm * Pm * Hm.T + mp.mpf(s2) * mp.eye(r)
    K = Pm * Hm.T * mp.inverse(S)
    Pn = Pm - K * Hm * Pm
    dxn = K * mp.matrix(res.tolist())
    d = np.sqrt(np.diag(P))
    for i in range(N):
        assert abs(float(ref["dx"][i]) - float(dxn[i])) <= 1e-17 * d[i] * ref["wnorm"]
        for j in range(N):
            assert abs(float(ref["P"][i, j]) - float(Pn[i, j])) <= 1e-17 * d[i] * d[j]
