"""tests/cov_ops.py against the CPU oracle on asymmetric covariances: the bit-exact mirrors agree with it bit for bit, the
long-double references agree with its double arithmetic within their bars, and an index or orientation error planted in a
reference breaks the bar by orders of magnitude."""
import numpy as np
import pytest

from oracle import ovo_py
from tests import cov_ops as co

needs_ld = pytest.mark.skipif(not co.have_longdouble(), reason="the reference needs an extended-precision long double")
BROKEN = 1e6  # a planted error must exceed the bar at least this much (an O(1) change is ~1e13 bars)


@pytest.fixture(scope="module", autouse=True)
def oracle_built():
    ovo_py.build()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def test_prior_is_asymmetric_and_well_conditioned():
    P = co.asymmetric_prior(40, 0)
    off = ~np.eye(40, dtype=bool)
    assert np.all(P[off] != P.T[off])
    assert np.unique(np.abs(P)).size == P.size  # every entry's magnitude is its own
    assert np.linalg.eigvalsh(0.5 * (P + P.T)).min() > 0 and np.linalg.cond(P) < 1e4


@pytest.mark.parametrize("N,old_off,size", [(37, 0, 6), (37, 31, 6), (37, 12, 1), (64, 3, 64 - 3)])
def test_clone_mirror_matches_oracle(N, old_off, size):
    P = co.asymmetric_prior(N, N + old_off)
    assert np.array_equal(_bits(co.clone(P, old_off, size)), _bits(ovo_py.cov_clone(P, old_off, size)))


@pytest.mark.parametrize("N,off,size", [(37, 0, 6), (37, 31, 6), (37, 10, 3), (37, 1, 36), (37, 0, 36)])
def test_marginalize_mirror_matches_oracle(N, off, size):
    P = co.asymmetric_prior(N, N + off)
    assert np.array_equal(_bits(co.marginalize(P, off, size)), _bits(ovo_py.cov_marginalize(P, off, size)))


@pytest.mark.parametrize("off,sz", [([20, 0, 36], [6, 3, 1]), ([0], [37]), ([36, 5], [1, 1])])
def test_get_marginal_mirror_matches_oracle(off, sz):
    P = co.asymmetric_prior(37, 3)
    assert np.array_equal(_bits(co.get_marginal(P, off, sz)), _bits(ovo_py.cov_get_marginal(P, off, sz)))


def _prop_case(N, new_off, p, off, sz, seed):
    rng = np.random.default_rng(seed)
    q = int(np.sum(sz))
    P = co.asymmetric_prior(N, seed)
    Phi = rng.standard_normal((p, q)) / np.sqrt(q)
    Q = 1e-4 * rng.standard_normal((p, p))  # garbage below the diagonal: only the upper triangle is read
    return P, Phi, Q, co.indices(off, sz)


PROP = [(40, 0, 15, [4, 0, 10], [6, 4, 5]), (40, 25, 3, [25, 7, 1], [3, 6, 6]), (40, 39, 1, [3], [2]), (40, 0, 40, [20, 0], [20, 20]),
        (40, 34, 6, [10, 2], [3, 1])]


@needs_ld
@pytest.mark.parametrize("N,new_off,p,off,sz", PROP)
def test_propagate_reference_bounds_the_oracle(N, new_off, p, off, sz):
    P, Phi, Q, idx = _prop_case(N, new_off, p, off, sz, 5)
    st, got = ovo_py.cov_propagate(P, new_off, Phi, Q, off, sz)
    ref, bar = co.propagate(P, new_off, Phi, Q, idx)
    r, at = co.worst(got, ref, bar)
    assert r <= 1.0, (r, at)
    # planted: P read transposed, Q's lower triangle, the old rows one off
    assert co.worst(got, *co.propagate(P.T, new_off, Phi, Q, idx))[0] > BROKEN
    if p > 1:
        assert co.worst(got, *co.propagate(P, new_off, Phi, Q.T, idx))[0] > BROKEN
    assert co.worst(got, *co.propagate(P, new_off, Phi, Q, (idx + 1) % N))[0] > BROKEN


@needs_ld
@pytest.mark.parametrize("N,old_off,size,dt_off", [(37, 0, 6, 36), (37, 31, 6, 33), (37, 12, 3, 0), (70, 2, 64, 69)])
def test_clone_dt_reference_bounds_the_oracle(N, old_off, size, dt_off):
    P = co.asymmetric_prior(N, 7)
    dnc = np.random.default_rng(8).standard_normal(size)
    got = ovo_py.cov_clone(P, old_off, size, dnc, dt_off)
    r, at = co.worst(got, *co.clone_dt(P, old_off, size, dnc, dt_off))
    assert r <= 1.0, (r, at)
    # planted: the dt row / column one off, and the prior transposed
    assert co.worst(got, *co.clone_dt(P, old_off, size, dnc, dt_off - 1))[0] > BROKEN
    assert co.worst(got, *co.clone_dt(P.T, old_off, size, dnc, dt_off))[0] > BROKEN


def init_system(k, n, seed, leading_zero=False):
    """H_R (k x n), H_L (k x k, kappa < 10) and res for a k-row initialize; with leading_zero, H_L[0][0] = 0."""
    rng = np.random.default_rng(seed)
    H_R = rng.standard_normal((k, n))
    H_L = np.eye(k) * 2.0 + 0.3 * rng.standard_normal((k, k))
    if leading_zero:
        H_L[[0, k - 1]] = H_L[[k - 1, 0]]
        H_L[0, 0] = 0.0
    return H_R, H_L, rng.standard_normal(k)


@needs_ld
@pytest.mark.parametrize("k,leading_zero", [(1, False), (2, False), (2, True), (3, False), (3, True)])
def test_initialize_reference_bounds_the_oracle(k, leading_zero):
    N = 40
    off, sz = [30, 2, 17], [3, 6, 1]
    cols = co.indices(off, sz)
    P = co.asymmetric_prior(N, k)
    H_R, H_L, res = init_system(k, len(cols), k, leading_zero)
    assert np.linalg.cond(H_L) < 10
    st, acc, got, _, _ = ovo_py.cov_initialize(P, off, sz, H_R, H_L, res, sigma2=0.7)
    assert st == 0 and acc
    HR, HL = co.givens_split(H_R, H_L)
    r, at = co.worst(got, *co.initialize_invertible(P, cols, HR, HL, 0.7))
    assert r <= 1.0, (r, at)
    # planted: P[cols, :] instead of P[:, cols], and the columns one off
    assert co.worst(got, *co.initialize_invertible(P.T, cols, HR, HL, 0.7))[0] > BROKEN
    assert co.worst(got, *co.initialize_invertible(P, (cols + 1) % N, HR, HL, 0.7))[0] > BROKEN


def test_planted_mirror_errors_change_bits():
    """The transposed read is what separates marginalize from a plain block copy, and the clone's column copy from its row
    copy: on an asymmetric P each changes bits."""
    P = co.asymmetric_prior(37, 1)
    plain = P[np.ix_(np.r_[0:10, 13:37], np.r_[0:10, 13:37])]
    assert not np.array_equal(co.marginalize(P, 10, 3), plain)
    c = co.clone(P, 5, 6)
    assert not np.array_equal(c[37:, :37], c[:37, 37:].T)
