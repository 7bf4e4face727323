"""ovb_ekf_update on every kernel chain launch_ekf_update routes to (csrc/k_ekf.cu; the chains E1-E4 at an even max_state,
O1-O6 at an odd one, tests/ekf_routes.py), and the Mahalanobis gate of ovb_cov_initialize on every factor route, against
an extended-precision reference.

Bars (tests/ekf_routes.py): with S~ = D^-1/2 S D^-1/2 (D = diag S), kappa = kappa_2(S~) and bar = max(1e-12, 1e-14 kappa):
  max |P+ - P+_ref|_ij / sqrt(P_ii P_jj) <= bar       (Y Y' <= P, so |(Y Y')_ij| <= sqrt(P_ii P_jj))
  max |dx - dx_ref|_i / (sqrt(P_ii) |w_ref|) <= bar   (|dx_i| <= sqrt(P_ii) |w|)
  |chi2 - chi2_ref| <= bar chi2_ref, plus 1e-14 |res_up|^2 / sigma^2 when the gate compresses (|res|^2 - |z|^2 cancels)
Per entry, so that an error in a small-variance state is not hidden under the largest ones.

Route proof: the profile (set_profile, then the call) must list every kernel of the chain and no other kernel of any
chain's products, factor, solve or downdate. Whether k_ekf_chol and k_ekf_trsm work in shared or global memory is not
visible in the profile (the same kernels run either way); that choice is covered by the mirror's byte formulas
(tests/test_ekf_routes_cpu.py) and by cases on both sides of each boundary (r = 155 | 156, 159 | 160).
"""
import numpy as np
import pytest

from open_vins_b200 import capi
from tests import ekf_routes as er

pytestmark = pytest.mark.gpu

WORST = {}  # chain or gate route -> worst error / bar ratios and kappa, printed at the end of the module


def _note(key, **kv):
    w = WORST.setdefault(key, {})
    for k, v in kv.items():
        w[k] = max(w.get(k, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def _longdouble():
    if not er.have_longdouble():
        pytest.skip("the reference needs an extended-precision long double (64-bit mantissa)")
    yield
    for k in sorted(WORST):
        print(f"\n{k}: " + " ".join(f"{a}={b:.3g}" for a, b in sorted(WORST[k].items())), end="")


def _engine(ld):
    return capi.Engine(max_state=ld, max_feats=16, max_meas=1024, max_rows=2048)


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(ld):
        if ld not in made:
            made[ld] = _engine(ld)
        return made[ld]
    yield get
    for e in made.values():
        e.close()


def _after_prep(names):
    """the launches of the last launch_ekf_update (each begins with k_ekf_prep); compression kernels come before it"""
    idx = [i for i, nm in enumerate(names) if er.mangled("k_ekf_prep") in nm]
    assert idx, names
    return names[idx[-1] + 1:]


def _kernels(names):
    """the kernels of er.ALL_KERNELS among the launched names"""
    return {k for k in er.ALL_KERNELS for nm in names if nm.startswith("_Z" + k)}


def _route_proof(names, want):
    got = _kernels(_after_prep(names))
    assert got == set(want), (sorted(got), sorted(want))


def _update(eng, x, P, noise, allow=()):
    eng.cov_set(P)
    kw = dict(sigma2=x.sigma2) if noise == "sigma2" else dict(Rdiag=x.Rdiag)
    eng.set_profile(True)
    st, dx = eng.ekf_update(x.off, x.sz, x.H, x.res, allow=allow, **kw)
    names = [nm for nm, _ in eng.profile_read()]
    eng.set_profile(False)
    return st, dx, eng.cov_get(), names


@pytest.mark.parametrize("case", er.CASES, ids=lambda c: f"{c.chain}-ld{c.ld}-N{c.N}-n{c.n}-rows{c.rows}")
@pytest.mark.parametrize("noise", ["sigma2", "rdiag"])
def test_ekf_chain(engines, case, noise):
    x = er.case_inputs(case)
    ch = er.chain(case.n, case.r, case.ld)
    eng = engines(case.ld)
    st, dx, Pg, names = _update(eng, x, x.P, noise)
    # at sigma^2 = 1e-8 mean diag(H P H') a well-observed state's posterior variance can be below the update's rounding
    # (the bar allows it): the status must then report the negative diagonal it left, and only then
    assert st in (capi.OVB_OK, capi.OVB_ERR_NEG_DIAG)
    assert (st == capi.OVB_ERR_NEG_DIAG) == bool((np.diag(Pg) < 0).any())
    _route_proof(names, ch.kernels)
    # exact structure
    assert np.array_equal(Pg, Pg.T), "P+ not exactly symmetric"
    if x.block:
        b = list(x.block)
        assert Pg[b].tobytes() == x.P[b].tobytes() and Pg[:, b].tobytes() == x.P[:, b].tobytes(), "uncorrelated block changed"
        assert np.all(dx[b] == 0.0)
    st2, dx2, Pg2, _ = _update(eng, x, x.P, noise)
    assert st2 == st and Pg2.tobytes() == Pg.tobytes() and dx2.tobytes() == dx.tobytes(), "second call in the same context differs"
    fresh = _engine(case.ld)
    try:
        st3, dx3, Pg3, _ = _update(fresh, x, x.P, noise)
    finally:
        fresh.close()
    assert st3 == st and Pg3.tobytes() == Pg.tobytes() and dx3.tobytes() == dx.tobytes(), "call in a fresh context differs"
    # values
    ref = er.case_reference(case, noise)
    bar = er.bar_of(ref["kappa"])
    eP, edx = er.errors(x.P, Pg, dx, ref)
    _note(case.chain, P=eP / bar, dx=edx / bar, kappa=ref["kappa"])
    assert eP <= bar, (eP, bar, ref["kappa"])
    assert edx <= bar, (edx, bar, ref["kappa"])


# ---------------------------------------------------------------------------------------------------------------- the gate
def _gate_system(ld, N, n, r_up, k, seed, level):
    """P (N x N), variables, H_R [k + r_up x n], H_L [k + r_up x k] upper triangular with a positive diagonal in its first k
    rows and zero below (the host's Givens split is then the identity: the gate sees H_R[k:] and res[k:] bit for bit),
    res, sigma^2"""
    rng = np.random.default_rng(seed)
    P = er.make_P(N, seed, 0)
    off, sz = er.place_variables(n, N, rng)
    cols = er.columns(off, sz)
    r = k + r_up
    HR = rng.standard_normal((r, n))
    HL = np.zeros((r, k))
    HL[:k] = np.triu(rng.uniform(-1, 1, size=(k, k)), 1) + np.diag(rng.uniform(0.5, 2.0, size=k))
    hph = np.einsum("ij,jk,ik->i", HR[k:], P[np.ix_(cols, cols)], HR[k:]).mean()
    sigma2 = er.SIGMA_LEVELS[level] * hph
    # a residual the model explains: chi2 of the order of r_up, so the compressed gate's |res|^2 / sigma^2 stays moderate
    lam, V = np.linalg.eigh(P[np.ix_(cols, cols)])
    dxs = V @ (np.sqrt(np.clip(lam, 0.0, None)) * rng.standard_normal(n))
    res = np.concatenate([rng.standard_normal(k), HR[k:] @ dxs + np.sqrt(sigma2) * rng.standard_normal(r_up)])
    return P, off, sz, cols, HR, HL, res, sigma2


def _chi2_ref(P, cols, H, res, s2):
    Pl = np.asarray(P, dtype=np.longdouble)
    Hl = np.asarray(H, dtype=np.longdouble)
    S = Hl @ Pl[np.ix_(cols, cols)] @ Hl.T
    S = 0.5 * (S + S.T)
    S[np.diag_indices_from(S)] += s2
    L = er.chol_ld(S)
    w = er.forward_ld(L, np.asarray(res, dtype=np.longdouble)[:, None])[:, 0]
    return float(w @ w)


@pytest.mark.parametrize("route,compressed,ld,N,n,r_up,k", er.GATE_CASES)
def test_gate_route(engines, route, compressed, ld, N, n, r_up, k):
    g = er.gate_route(n, r_up, ld)
    assert (g.route, g.compressed) == (route, compressed)
    level = 1 if compressed else 2
    P, off, sz, cols, HR, HL, res, s2 = _gate_system(ld, N, n, r_up, k, seed=ld + N + n + r_up, level=level)
    Hup = HR[k:]
    ref = _chi2_ref(P, cols, Hup, res[k:], s2)
    if compressed:
        Rq = np.linalg.qr(Hup, mode="r")
        kappa = er.scaled_kappa(Rq @ P[np.ix_(cols, cols)] @ Rq.T + s2 * np.eye(n))
    else:
        kappa = er.scaled_kappa(Hup @ P[np.ix_(cols, cols)] @ Hup.T + s2 * np.eye(r_up))
    bar = er.bar_of(kappa) + (1e-14 * float(res[k:] @ res[k:]) / s2 / ref if compressed else 0.0)
    m = max(1e-7, 4 * bar)
    q = float(capi.load_library().ovb_chi2_quantile95(k + r_up))
    eng = engines(ld)
    # just below the reference chi2: rejected, nothing changes
    eng.cov_set(P)
    eng.set_profile(True)
    st, acc, _, _ = eng.cov_initialize(off, sz, HR, HL, res, sigma2=s2, chi2_mult=ref / q * (1 - m))
    names = [nm for nm, _ in eng.profile_read()]
    eng.set_profile(False)
    assert st == capi.OVB_OK and not acc, "gate accepted below the reference chi2"
    assert eng.cov_dim() == N and eng.cov_get().tobytes() == P.tobytes()
    _route_proof(names, g.kernels)
    # just above: accepted, the covariance grows by k
    eng.cov_set(P)
    st, acc, _, _ = eng.cov_initialize(off, sz, HR, HL, res, sigma2=s2, chi2_mult=ref / q * (1 + m))
    assert st == capi.OVB_OK and acc, "gate rejected above the reference chi2"
    assert eng.cov_dim() == N + k
    _note(f"gate-{route}{'-compressed' if compressed else ''}", kappa=kappa, pin_margin_over_bar=m / bar)
    WORST.setdefault("pin", {})["smallest_m"] = min(WORST.get("pin", {}).get("smallest_m", 1.0), m)


# ---------------------------------------------------------------------------------------------------------------- failure exits
# (route, ld, N, n = r, position of the failing pivot in S)
NOT_SPD = (("A", 640, 100, 40, 3), ("B", 640, 400, 300, 5), ("B", 640, 400, 300, 290), ("C", 641, 100, 40, 3), ("D", 641, 300, 200, 5))


def _not_spd_system(N, n, pos, seed):
    """P whose observed state cols[pos] has a negative variance and no correlation: with H = I over the variables S is
    indefinite and its first failing pivot is `pos`"""
    rng = np.random.default_rng(seed)
    P = er.make_P(N, seed, 0).copy()
    off, sz = er.place_variables(n, N, rng)
    cols = er.columns(off, sz)
    j = cols[pos]
    P[j, :] = 0.0
    P[:, j] = 0.0
    P[j, j] = -1.0
    return P, off, sz, cols


@pytest.mark.parametrize("route,ld,N,n,pos", NOT_SPD)
def test_not_spd_update(engines, route, ld, N, n, pos):
    P, off, sz, cols = _not_spd_system(N, n, pos, seed=N + pos)
    ch = er.chain(n, n, ld)
    assert {"dmma": "A", "blocked": "B", "chol_smem": "C", "chol_global": "D"}[ch.factor] == route
    if route == "B":
        assert (pos < 128) == (pos == 5) and (pos >= 256) == (pos == 290)  # first block / last 128-column block
    eng = engines(ld)
    eng.cov_set(P)
    eng.set_profile(True)
    st, dx = eng.ekf_update(off, sz, np.eye(n), np.ones(n), sigma2=1e-3, allow=(capi.OVB_ERR_NOT_SPD,))
    names = [nm for nm, _ in eng.profile_read()]
    eng.set_profile(False)
    assert st == capi.OVB_ERR_NOT_SPD
    assert eng.cov_get().tobytes() == P.tobytes(), "a failed factor changed P"
    assert not dx.any()
    _route_proof(names, ch.kernels)


@pytest.mark.parametrize("route,ld,N,n,pos", NOT_SPD)
def test_not_spd_gate(engines, route, ld, N, n, pos):
    P, off, sz, cols = _not_spd_system(N - 3, n, pos, seed=N + pos + 1)
    assert er.gate_route(n, n, ld).route == route
    k = 3
    HR = np.vstack([np.ones((k, n)), np.eye(n)])
    HL = np.vstack([np.eye(k), np.zeros((n, k))])
    eng = engines(ld)
    eng.cov_set(P)
    st, acc, _, _ = eng.cov_initialize(off, sz, HR, HL, np.ones(n + k), sigma2=1e-3, chi2_mult=1e300)
    assert st == capi.OVB_OK and not acc, "the gate accepted an indefinite S"
    assert eng.cov_dim() == N - 3 and eng.cov_get().tobytes() == P.tobytes()


# (route, ld, N, n = r): two unobserved negative variances in different 32-row tiles, neither in tile 0
NEG_DIAG = (("A", 640, 200, 40), ("B", 640, 400, 300), ("C", 641, 200, 40), ("D", 641, 300, 200))
NEG_AT = (37, 101)


@pytest.mark.parametrize("route,ld,N,n", NEG_DIAG)
def test_negative_diagonal(engines, route, ld, N, n):
    seed = 7 * N + n
    rng = np.random.default_rng(seed)
    P = er.make_P(N, seed, 0).copy()
    for i in NEG_AT:
        P[i, :] = 0.0
        P[:, i] = 0.0
        P[i, i] = -0.25
    off, sz = er.place_variables(n, N, rng, exclude=NEG_AT)
    cols = er.columns(off, sz)
    assert not set(cols) & set(NEG_AT)
    H = rng.standard_normal((n, n))
    res = rng.standard_normal(n)
    s2 = float(np.einsum("ij,jk,ik->i", H, P[np.ix_(cols, cols)], H).mean())
    ch = er.chain(n, n, ld)
    assert {"dmma": "A", "blocked": "B", "chol_smem": "C", "chol_global": "D"}[ch.factor] == route
    eng = engines(ld)
    eng.cov_set(P)
    eng.set_profile(True)
    st, dx = eng.ekf_update(off, sz, H, res, sigma2=s2)
    names = [nm for nm, _ in eng.profile_read()]
    eng.set_profile(False)
    assert st == capi.OVB_ERR_NEG_DIAG
    assert f"diagonal at {min(NEG_AT)} is negative" in (eng.lib.ovb_last_error(eng.h) or b"").decode()
    _route_proof(names, ch.kernels)
    Pg = eng.cov_get()
    b = list(NEG_AT)
    assert Pg[b].tobytes() == P[b].tobytes() and Pg[:, b].tobytes() == P[:, b].tobytes()
    assert np.all(dx[b] == 0.0)
    ref = er.reference_update(P, cols, H, res, s2)
    bar = er.bar_of(ref["kappa"])
    eP, edx = er.errors(P, Pg, dx, ref, skip=NEG_AT)
    assert eP <= bar and edx <= bar, (eP, edx, bar)
