"""ovb_compress_cholqr2 (csrc/k_cholqr.cu) at every slab / round route of the narrow path's k_cq_solve_gram and at the block
edges of the wide path, against an extended-precision reference.

Inputs have integer entries in [-4, 4] with each column scaled by 2^k, k in [-10, 10]: every product and every partial
sum of G = [H r]'[H r] is a multiple of 2^(ki + kj) below 2^53 of those units, so G is EXACT in float64 whatever the
summation order. R'R and R'z are checked against that exact G; the factor against the long-double (64-bit mantissa
on x86) Cholesky of G with the compression's two shifts applied (see SHIFT1, SHIFT2). Shapes
are chosen at run time with the geometry mirror (tests/cholqr_geometry.py) for the SM count of the device, so each case
reaches its route on any card.
"""
from functools import lru_cache

import numpy as np
import pytest

from open_vins_b200 import capi, sim
from tests import cholqr_geometry as geo

pytestmark = pytest.mark.gpu

# every (template instance, BW) class of k_cq_solve_gram at its edges: nt = n + 1 = 8, 32 | 33, 40 | 64 | 65, 80 | 81, 96 |
# 97, 120 | 121, 128 | 129, 160
EDGE_N = (7, 31, 32, 39, 63, 64, 79, 80, 95, 96, 119, 120, 127, 128, 159)
# (n, route): each edge n at every route its instance has (the split routes need a buffer shorter than a round)
NARROW_CASES = tuple((n, r) for n in EDGE_N for r in geo.ROUTES if r not in geo.SPLIT_ROUTES or geo.instance_of(n + 1)[1] > 0)
WIDE_N = (160, 255, 256, 257, 383, 384, 385, 511, 512)


def route_m(n, route, sm_count):
    """The m a NARROW_CASES entry runs at: at least 2n rows (so that the factor can be compared with the reference's) except
    for the routes that need fewer; one slab is taken near its 32-row limit, m <= n at m = n."""
    m_min = {"one_slab": 29, "m_le_n": n}.get(route, 2 * n)
    return geo.find_m(n, route, sm_count, m_min=m_min)


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    e = capi.Engine(max_state=256, max_feats=64, max_meas=1024, max_rows=65536)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng_wide():
    e = capi.Engine(max_state=640, max_feats=64, max_meas=1024, max_rows=16384)
    yield e
    e.close()


@pytest.fixture(scope="module", autouse=True)
def _longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("the reference needs an extended-precision long double (64-bit mantissa)")


def _chol_ld(G):
    """Upper Cholesky factor (diag >= 0) of an SPD matrix in long double."""
    A = np.array(G, dtype=np.longdouble)
    n = A.shape[0]
    R = np.zeros_like(A)
    for k in range(n):
        d = A[k, k]
        assert d > 0, "reference Gram matrix not positive definite"
        R[k, k] = np.sqrt(d)
        R[k, k + 1:] = A[k, k + 1:] / R[k, k]
        A[k + 1:, k + 1:] -= np.outer(R[k, k + 1:], R[k, k + 1:])
    return R


# The compression's shifts (k_cholqr.cu): pass 1 factors G + s1 I with s1 = 1e-11 max diag G, pass 2 factors
# Q1'Q1 + s2 I with s2 = 1e-13 max diag Q1'Q1 = 1e-13 (1 - O(1e-11)). In exact arithmetic the result is therefore the
# Cholesky factor of G + s2 (G + s1 I), not of G. Columns 2^20 apart in scale put s2 s1 at ~2e-12 of the smallest
# G_jj, as large as the bar on the factor itself; so the factor is compared with the Cholesky of that shifted G (known
# exactly in long double), while the invariants below compare R'R and R'z with the exact G.
SHIFT1, SHIFT2 = 1e-11, 1e-13


@lru_cache(maxsize=None)
def _system(m, n, seed, dependent=0):
    """[H r] with exact Gram matrix G (float64); `dependent` pairs of columns c_j = c_i + e, e one +-1 entry. Returns
    (A, G, Rfull, kappa): Rfull the long-double Cholesky factor of the shifted G and kappa the condition number of its
    column-scaled form, when the system has full column rank and m >= 2n (else None, None)."""
    rng = np.random.default_rng(seed)
    A = rng.integers(-4, 5, size=(m, n + 1)).astype(np.float64)
    for _ in range(dependent):
        i, j = rng.choice(n, size=2, replace=False)
        A[:, j] = A[:, i]
        A[rng.integers(m), j] += rng.choice([-1.0, 1.0])
    A *= 2.0 ** rng.integers(-10, 11, size=n + 1)
    A.setflags(write=False)
    G = A.T @ A
    G.setflags(write=False)
    Rfull = kappa = None
    if m >= 2 * n and np.linalg.matrix_rank(A) == n + 1:
        Gl = G.astype(np.longdouble)
        s1 = SHIFT1 * Gl.diagonal().max()
        Rfull = _chol_ld(Gl + SHIFT2 * (Gl + s1 * np.eye(n + 1, dtype=np.longdouble)))
        kappa = float(np.linalg.cond((Rfull / np.sqrt(Gl.diagonal())[None, :]).astype(np.float64)))
    return A, G, Rfull, kappa


def _errors(A, G, Rfull, R, z):
    """The bars' quantities for one result; asserts the structural ones."""
    n = R.shape[0]
    assert np.isfinite(R).all() and np.isfinite(z).all()
    assert np.array_equal(np.tril(R, -1), np.zeros_like(R)), "R not exactly upper triangular"
    assert (np.diag(R) >= 0).all()
    GH, Ghr = G[:n, :n].astype(np.longdouble), G[:n, n].astype(np.longdouble)
    Rl, zl = R.astype(np.longdouble), z.astype(np.longdouble)
    dG = Rl.T @ Rl - GH
    dz = Rl.T @ zl - Ghr
    d = np.sqrt(np.diag(G).astype(np.longdouble))
    d = np.where(d > 0, d, 1)
    e = dict(gram=float(np.linalg.norm(dG.astype(np.float64)) / np.linalg.norm(G[:n, :n])),
             rhs=float(np.linalg.norm(dz.astype(np.float64)) / (np.linalg.norm(A[:, :n]) * np.linalg.norm(A[:, n]))),
             scaled=float(max(np.abs(dG / np.outer(d[:n], d[:n])).max(), np.abs(dz / (d[:n] * d[n])).max())))
    if Rfull is not None:
        e["factor"] = float(max(np.abs((Rl - Rfull[:n, :n]) / d[None, :n]).max(), np.abs((zl - Rfull[:n, n]) / d[n]).max()))
    return e


def _check(errs):
    """R'R and R'z against the exact G: 1e-12 relative in norm and 1e-11 per column-scaled entry; the column-scaled
    factor against the reference's to 1e-12, for full column rank and m >= 2n."""
    assert errs["gram"] <= 1e-12, errs
    assert errs["rhs"] <= 1e-12, errs
    assert errs["scaled"] <= 1e-11, errs
    if "factor" in errs:
        assert errs["factor"] <= 1e-12, errs


def run_case(eng, m, n, seed, dependent=0, max_rows=65536):
    """Compress the (m, n) system twice in `eng` and once in a fresh context; returns the bars' quantities after checking
    that all three results are byte-identical (the compression is deterministic: replicas stay bitwise equal)."""
    A, G, Rfull, _ = _system(m, n, seed, dependent)
    H, r = A[:, :n], A[:, n]
    R, z = eng.compress(H, r, mode=capi.COMPRESS_CHOLQR2)
    R2, z2 = eng.compress(H, r, mode=capi.COMPRESS_CHOLQR2)
    fresh = capi.Engine(max_state=max(n, 256), max_feats=64, max_meas=1024, max_rows=max(m, max_rows))
    try:
        R3, z3 = fresh.compress(H, r, mode=capi.COMPRESS_CHOLQR2)
    finally:
        fresh.close()
    assert R.tobytes() == R2.tobytes() and z.tobytes() == z2.tobytes(), "second call in the same context differs"
    assert R.tobytes() == R3.tobytes() and z.tobytes() == z3.tobytes(), "call in a fresh context differs"
    return _errors(A, G, Rfull, R, z)


@pytest.mark.parametrize("n,route", NARROW_CASES)
def test_cholqr2_narrow_route(eng, sm_count, n, route):
    m = route_m(n, route, sm_count)
    if m is None:
        pytest.skip(f"no m reaches route {route} at n={n} with {sm_count} SMs")
    g = geo.narrow_geometry(m, n, sm_count)
    assert route in geo.routes(g)
    _check(run_case(eng, m, n, seed=1000 * m + n, max_rows=4096))


# Nearly dependent integer columns on the split routes; G stays exact. Two or three column pairs c_j = c_i + e give the
# column-scaled system a condition number of 600-900, and every bar stays as it is: the compression has no condition-number
# factor in R'R (DESIGN.md section 4), and against the shifted reference the factor's error is of rounding size.
@pytest.mark.parametrize("n,route,pairs", [(100, "split", 3), (119, "multi_split", 2), (127, "tail_max", 3), (154, "split", 2),
                                           (159, "multi_split", 3)])
def test_cholqr2_narrow_ill_conditioned(eng, sm_count, n, route, pairs):
    m = route_m(n, route, sm_count)
    if m is None:
        pytest.skip(f"no m reaches route {route} at n={n} with {sm_count} SMs")
    assert _system(m, n, 7 * m + n, pairs)[3] > 100
    _check(run_case(eng, m, n, seed=7 * m + n, dependent=pairs, max_rows=4096))


def test_cholqr2_context_reuse(sm_count):
    """One context whose Gpart / Qtail scratch grows and shrinks: small slabs, the longest scratch tail, small again,
    another instance's longest tail, a narrow system; every result equals the one from a context of its own."""
    seq = [(300, 100), (route_m(154, "tail_max", sm_count), 154), (301, 100), (route_m(100, "multi_split", sm_count), 100),
           (route_m(127, "tail_max", sm_count), 127), (64, 7), (300, 100)]
    e = capi.Engine(max_state=256, max_feats=64, max_meas=1024, max_rows=65536)
    try:
        for m, n in seq:
            _check(run_case(e, m, n, seed=m + n, max_rows=4096))
    finally:
        e.close()


def _wide_m(n, sm_count):
    """the smallest m >= 2n with several slabs and a last slab at least 8 rows shorter than the others (at most about
    3 (nslab - 1) rows shorter when m >= 2n: slab_rows is ceil(m / nslab) rounded up to 4)"""
    return geo.find_m_wide(n, sm_count, 2 * n, lambda g: g.nslab >= 3 and g.last_rows <= g.slab_rows - 8)


@pytest.mark.parametrize("n", WIDE_N)
def test_cholqr2_wide_edges(eng_wide, sm_count, n):
    m = _wide_m(n, sm_count)
    g = geo.wide_geometry(m, n, sm_count)
    assert g.nslab >= 3 and g.last_rows <= g.slab_rows - 8
    _check(run_case(eng_wide, m, n, seed=m + 3 * n, max_rows=16384))


def test_cholqr2_wide_capacity(eng_wide):
    """n = 513: nt = 514 is past the wide path's 513 columns, within max_state"""
    rng = np.random.default_rng(5)
    with pytest.raises(capi.OvbError) as ei:
        eng_wide.compress(rng.integers(-4, 5, size=(1200, 513)).astype(np.float64), np.ones(1200), mode=capi.COMPRESS_CHOLQR2)
    assert ei.value.code == capi.OVB_ERR_CAPACITY


@pytest.mark.parametrize("n,route", [(100, "split"), (154, "multi_split")])
def test_cholqr2_gram_cluster(monkeypatch, sm_count, n, route):
    """OVB_GRAM_CLUSTER=1 (read at ovb_create): pass 1 pre-reduces clusters of 4 slabs in distributed shared memory. Its
    reduction order differs from the default's, so only the invariants are checked, not bit identity."""
    m = route_m(n, route, sm_count)
    assert geo.narrow_geometry(m, n, sm_count).nslab >= 8
    monkeypatch.setenv("OVB_GRAM_CLUSTER", "1")
    e = capi.Engine(max_state=256, max_feats=64, max_meas=1024, max_rows=65536)
    try:
        A, G, Rfull, _ = _system(m, n, 11 * m + n)
        R, z = e.compress(A[:, :n], A[:, n], mode=capi.COMPRESS_CHOLQR2)
    finally:
        e.close()
    _check(_errors(A, G, Rfull, R, z))


# ---------------------------------------------------------------------------------------------------------------- in the update
# One camera with extrinsic and intrinsic calibration: the update's stacked system has n = 6 n_clones + 14 columns
# (14 clones: nt = 99, instance <10,5>, BW 4; 18 clones: nt = 123, instance <10,10>, BW 4). The number of features is chosen
# at run time so that the staged rows, sum of 2 M_f - 3 over all input features, make the first slab a split round.
MSCKF_CASES = [(14, (10, 5), "ILi10ELi5EE"), (18, (10, 10), "ILi10ELi10EE")]


@lru_cache(maxsize=None)
def _msckf_case(n_clones, sm_count):
    kw = dict(n_clones=n_clones, n_cams=1, seed=n_clones, calib_ext=True, calib_intr=True)
    big = sim.make_update_case(n_feats=1000, **kw)  # features are drawn in order: a case of k features is this one's prefix
    M = np.diff(big.feats.meas_off)
    rows = np.cumsum(np.where(M >= 2, 2 * M - 3, 0))
    n = 6 * n_clones + 14
    for k in range(1, len(rows) + 1):
        g = geo.narrow_geometry(int(rows[k - 1]), n, sm_count)
        if g.nslab > 1 and g.first[-1][1] > 0 and len(g.first) == 1:
            case = sim.make_update_case(n_feats=k, **kw)
            assert np.array_equal(case.feats.meas_off, big.feats.meas_off[:k + 1])
            return case, int(rows[k - 1]), n
    raise AssertionError("no feature count puts the first slab on a split round")


@pytest.mark.parametrize("order", [capi.COLS_CANONICAL, capi.COLS_REFERENCE_FIRST_SEEN])
@pytest.mark.parametrize("n_clones,instance,mangled", MSCKF_CASES)
def test_update_split_route(oracle, sm_count, n_clones, instance, mangled, order):
    case, m, n = _msckf_case(n_clones, sm_count)
    g = geo.narrow_geometry(m, n, sm_count)
    assert g.instance == instance and g.BW == 4 and "split" in geo.routes(g)
    opts = capi.default_opts(do_calib_camera_pose=1, do_calib_camera_intrinsics=1, compress=capi.COMPRESS_CHOLQR2, col_order=order)
    e = capi.Engine(max_state=256, max_feats=1024, max_meas=1024 * 24)
    try:
        e.cov_set(case.P)
        e.set_profile(True)
        st, out, dx, stats = e.msckf_update(case.frame, case.feats, opts)
        names = [nm for nm, _ in e.profile_read()]
        P = e.cov_get()
    finally:
        e.close()
    assert stats.cols_stacked == n, "every frame variable is in the stacked system"
    assert any("k_cq_solve_gram" in nm and mangled in nm for nm in names), names
    ref = oracle.msckf_update(case.frame, case.feats, opts, case.P, dumps=False)
    assert st == ref["status"] == 0
    assert np.array_equal(out.status, ref["out"].status)
    assert np.linalg.norm(P - ref["P"]) <= 1e-9 * np.linalg.norm(ref["P"])
    assert np.linalg.norm(dx - ref["dx"]) <= 1e-9 * np.linalg.norm(ref["dx"])
