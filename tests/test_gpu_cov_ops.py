"""The covariance structure operations on the resident P (ovb_cov_propagate, ovb_cov_clone, ovb_cov_marginalize,
ovb_cov_get_marginal and the augmentation of ovb_cov_initialize) on the H100, against tests/cov_ops.py on asymmetric
priors, at their shape and capacity edges. Every case checks that the entries outside the written rows and columns keep
their bits and that N is what the reference says. Two contexts: max_state 600 (even ldP) and 301 (odd ldP)."""
import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import capi
from tests import cov_ops as co

pytestmark = pytest.mark.gpu
needs_ld = pytest.mark.skipif(not co.have_longdouble(), reason="the reference needs an extended-precision long double")

OVB_MAX_COLS = 512  # csrc/ovb_internal.cuh
MAX_MEAS = 300
CONTEXTS = {"even": 600, "odd": 301}
WORST = {}  # operation -> largest error / bar over the module


def hs_cap(max_state, max_meas, max_rows=0):
    """ctx->Hs_cap, the device staging matrix in doubles, as ovb_create sizes it (ovb_api.cu:70-75, 151-155)."""
    ms, mm = max(max_state, 32), max(max_meas, 2)
    rows = max(max_rows if max_rows > 0 else 2 * mm, 2 * mm)
    return rows * (min(OVB_MAX_COLS, ms) + 8)


def propagate_fits(p, q, cap):
    """ovb_cov_propagate stages Phi (p x q) and Q (p x p) doubles, then the q int32 old indices, in d_Hs (ovb_api.cu:494-521)."""
    return p * q + p * p + (q + 1) // 2 <= cap


@pytest.fixture(scope="module", autouse=True)
def report():
    b.build()
    yield
    for op, r in sorted(WORST.items()):
        print(f"\n{op}: largest |got - ref| / bar = {r:.3g}")


@pytest.fixture(scope="module", params=sorted(CONTEXTS))
def ctx(request):
    ms = CONTEXTS[request.param]
    eng = capi.Engine(max_state=ms, max_feats=1, max_meas=MAX_MEAS)
    yield eng, ms
    eng.close()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _status(call, *args):
    """the call's status; the Engine methods that return nothing raise on every status but OVB_OK"""
    try:
        st = call(*args)
    except capi.OvbError as e:
        return e.code
    return capi.OVB_OK if st is None else st


def _note(op, r):
    WORST[op] = max(WORST.get(op, 0.0), r)


def _sizes(top):
    """a small N, one past the 256 threads of a CTA, and top"""
    return sorted({97, 300, top})


def _chunks(base, n):
    """[base, base + n) as variables of sizes 4, 3, 6, 2, ... listed from the last to the first (unsorted)."""
    off, sz, pat = [], [], (4, 3, 6, 2, 5)
    x, i = base, 0
    while x < base + n:
        s = min(pat[i % len(pat)], base + n - x)
        off.append(x)
        sz.append(s)
        x, i = x + s, i + 1
    return off[::-1], sz[::-1]


# ------------------------------------------------------------------------------------------------------ propagate
def _prop_cases(N):
    """(name, new_off, p, old_off, old_sz): the old variables are non-contiguous or listed out of order."""
    cases = [("p=1", N // 2, 1, [N // 3, 5], [2, 1]),
             ("anchor p=3 q=15", N - 3, 3, [N - 3, 12, 0], [3, 6, 6]),
             ("anchor p=3 q=27", 40, 3, [40, N - 12, 7, N - 6, 20], [3, 6, 6, 6, 6]),
             ("p!=q, new outside old", N - 6, 6, [10, N // 2, 2], [3, 6, 1]),
             ("whole state", 0, N, *_chunks(0, N))]
    for p in (15, 30, 39):
        cases.append((f"imu p=q={p}", 0, p, *_chunks(0, p)))
    cases.append(("imu p=q=15 at N-p", N - 15, 15, *_chunks(N - 15, 15)))
    return cases


def _check_propagate(eng, ms, N, new_off, p, off, sz, seed):
    rng = np.random.default_rng(seed)
    idx = co.indices(off, sz)
    q = idx.size
    P0 = co.asymmetric_prior(N, seed)
    Phi = rng.standard_normal((p, q)) / np.sqrt(q)
    Q = 1e-4 * rng.standard_normal((p, p))  # the lower triangle is garbage: only the upper one may be read
    np.fill_diagonal(Q, np.abs(np.diag(Q)))
    eng.cov_set(P0)
    st = _status(eng.cov_propagate, new_off, Phi, Q, off, sz)
    P = eng.cov_get()
    assert eng.cov_dim() == N
    if not propagate_fits(p, q, hs_cap(ms, MAX_MEAS)):
        assert st == capi.OVB_ERR_CAPACITY and np.array_equal(_bits(P), _bits(P0))
        return None
    assert st == capi.OVB_OK
    nb = slice(new_off, new_off + p)
    kept = np.ones((N, N), dtype=bool)
    kept[nb, :] = kept[:, nb] = False
    assert np.array_equal(_bits(P)[kept], _bits(P0)[kept])
    rest = np.r_[0:new_off, new_off + p:N]
    assert np.array_equal(_bits(P[rest][:, nb]), _bits(P[nb][:, rest].T))  # P[a][new+j] == P[new+j][a], bitwise
    r, at = co.worst(P, *co.propagate(P0, new_off, Phi, Q, idx))
    _note("ovb_cov_propagate", r)
    assert r <= 1.0, (r, at)
    return r


@needs_ld
def test_propagate(ctx):
    eng, ms = ctx
    for N in _sizes(ms):
        for name, new_off, p, off, sz in _prop_cases(N):
            _check_propagate(eng, ms, N, new_off, p, off, sz, N + p)


@needs_ld
def test_propagate_staging_capacity_edge():
    """max_state 600, max_meas 300: Hs_cap = 600 x 520 doubles. At p = 520 the largest q whose Phi, Q and old indices fit
    is accepted and computed; one more column is refused with P and N unchanged, although Phi and Q alone would still fit."""
    ms, p = 600, 520
    cap = hs_cap(ms, MAX_MEAS)
    q = max(q for q in range(1, ms - p + 1) if propagate_fits(p, q, cap))
    assert p * (q + 1) + p * p <= cap  # the edge lies where only the index array overflows
    eng = capi.Engine(max_state=ms, max_feats=1, max_meas=MAX_MEAS)
    try:
        assert _check_propagate(eng, ms, ms, 0, p, *_chunks(p, q), 1) is not None
        assert _check_propagate(eng, ms, ms, 0, p, *_chunks(p, q + 1), 2) is None
        assert b"ovb_cov_propagate" in eng.lib.ovb_last_error(eng.h)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------ clone
@needs_ld
def test_clone(ctx):
    eng, ms = ctx
    for N in _sizes(ms - 6):
        P0 = co.asymmetric_prior(N, N)
        dnc = np.random.default_rng(N).standard_normal(64)
        for old_off, size, dt_off in [(0, 6, None), (N - 6, 6, None), (N - 1, 1, None), (0, 6, N - 1), (N - 6, 6, N - 4), (3, 64, N - 1),
                                      (N - 64, 64, 0)]:
            if N + size > ms:
                continue
            eng.cov_set(P0)
            d = None if dt_off is None else dnc[:size]
            eng.cov_clone(old_off, size, d, -1 if dt_off is None else dt_off)
            P = eng.cov_get()
            assert P.shape == (N + size,) * 2
            assert np.array_equal(_bits(P[:N, :N]), _bits(P0))
            if d is None:
                assert np.array_equal(_bits(P), _bits(co.clone(P0, old_off, size))), (N, old_off, size)
            else:
                r, at = co.worst(P, *co.clone_dt(P0, old_off, size, d, dt_off))
                _note("ovb_cov_clone (time offset)", r)
                assert r <= 1.0, (N, old_off, size, dt_off, r, at)


def test_clone_refusals(ctx):
    eng, ms = ctx
    N = 97
    P0 = co.asymmetric_prior(N, 4)
    eng.cov_set(P0)
    assert _status(eng.cov_clone, 0, 65, np.ones(65), N - 1) == capi.OVB_ERR_ARG  # the time offset takes at most 64
    assert eng.cov_dim() == N and np.array_equal(_bits(eng.cov_get()), _bits(P0))
    for N in (ms - 6, ms - 5):
        P0 = co.asymmetric_prior(N, N)
        eng.cov_set(P0)
        st = _status(eng.cov_clone, N - 6, 6)
        if N + 6 <= ms:
            assert st == capi.OVB_OK and eng.cov_dim() == ms
            assert np.array_equal(_bits(eng.cov_get()), _bits(co.clone(P0, N - 6, 6)))
        else:
            assert st == capi.OVB_ERR_CAPACITY and eng.cov_dim() == N
            assert np.array_equal(_bits(eng.cov_get()), _bits(P0))


# ------------------------------------------------------------------------------------------------------ marginalize
def test_marginalize(ctx):
    eng, ms = ctx
    for N in _sizes(ms):
        P0 = co.asymmetric_prior(N, N + 1)
        for off, size in [(0, 6), (N - 6, 6), (N // 2, 3), (1, N - 1), (0, N - 1)]:
            eng.cov_set(P0)
            eng.cov_marginalize(off, size)
            assert eng.cov_dim() == N - size
            assert np.array_equal(_bits(eng.cov_get()), _bits(co.marginalize(P0, off, size))), (N, off, size)


# ------------------------------------------------------------------------------------------------------ get_marginal
def test_get_marginal(ctx):
    eng, ms = ctx
    for N in _sizes(ms):
        P0 = co.asymmetric_prior(N, N + 2)
        eng.cov_set(P0)
        for off, sz in [([N // 2, 0, N - 1], [6, 3, 1]), ([N - 6, 7, 4], [6, 1, 1]), ([0], [N]), ([N - 1, 0], [1, 1])]:
            got = eng.cov_get_marginal(off, sz)
            assert np.array_equal(_bits(got), _bits(co.get_marginal(P0, off, sz))), (N, off, sz)
        assert eng.cov_dim() == N and np.array_equal(_bits(eng.cov_get()), _bits(P0))


# ------------------------------------------------------------------------------------------------------ initialize
def _init_system(k, n, seed, leading_zero):
    """H_R (k x n), H_L (k x k, kappa < 10). With leading_zero H_L[0][0] = 0: make_givens' p == 0 branch then swaps the
    rows (r = k, so the split leaves H_L upper triangular and the Gauss-Jordan pivots stay on the diagonal)."""
    rng = np.random.default_rng(seed)
    H_R = rng.standard_normal((k, n))
    H_L = np.eye(k) * 2.0 + 0.3 * rng.standard_normal((k, k))
    if leading_zero:
        H_L[[0, k - 1]] = H_L[[k - 1, 0]]
        H_L[0, 0] = 0.0
    return H_R, H_L, rng.standard_normal(k)


@needs_ld
def test_initialize_augmentation(ctx):
    """ovb_cov_initialize with r = k: no gate, no update, only k_cov_init_augment (N > 256 strides its row loops)."""
    eng, ms = ctx
    for k in (1, 2, 3):
        for N in sorted({40, 290, ms - k}):
            for leading_zero in ((False, True) if k > 1 else (False,)):
                off, sz = [N - 4, 2, N // 2, 11], [3, 6, 2, 1]
                cols = co.indices(off, sz)
                P0 = co.asymmetric_prior(N, N + k)
                H_R, H_L, res = _init_system(k, cols.size, N + k, leading_zero)
                eng.cov_set(P0)
                st, accepted, _, _ = eng.cov_initialize(off, sz, H_R, H_L, res, sigma2=0.7)
                assert st == capi.OVB_OK and accepted and eng.cov_dim() == N + k
                P = eng.cov_get()
                assert np.array_equal(_bits(P[:N, :N]), _bits(P0))
                assert np.array_equal(_bits(P[N:, :N]), _bits(P[:N, N:].T))
                assert np.array_equal(_bits(P[N:, N:]), _bits(P[N:, N:].T))  # P_LL exactly symmetric
                HR, HL = co.givens_split(H_R, H_L)
                r, at = co.worst(P, *co.initialize_invertible(P0, cols, HR, HL, 0.7))
                _note("ovb_cov_initialize (augmentation)", r)
                assert r <= 1.0, (k, N, leading_zero, r, at)
    # one past max_state
    k, N = 3, ms - 2
    P0 = co.asymmetric_prior(N, 5)
    H_R, H_L, res = _init_system(k, 4, 5, False)
    eng.cov_set(P0)
    assert _status(eng.cov_initialize, [0, 10], [3, 1], H_R, H_L, res) == capi.OVB_ERR_CAPACITY
    assert eng.cov_dim() == N and np.array_equal(_bits(eng.cov_get()), _bits(P0))
