"""Factor streaming of csrc/k_cholqr.cu: pass 1's k_cq_chol_gram and the EKF's k_cq_chol_ekf publish their factor block
column by block column, and k_cq_solve_gram / k_cq_trsm, made resident early by PDL, consume it while the pivot chain
runs. Profile mode launches without PDL, so each consumer starts after its producer has finished: the serialised run.
The overlapped run must give the same bytes, on every route that streams.
"""
import numpy as np
import pytest

from open_vins_b200 import capi, sim
from tests import ekf_routes as er
from tests.test_gpu_cholqr_geometry import NARROW_CASES, _system, route_m

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    e = capi.Engine(max_state=256, max_feats=64, max_meas=1024, max_rows=65536)
    yield e
    e.close()


def _both(e, call):
    """(overlapped, serialised) results of call(e)"""
    e.set_profile(False)
    a = call(e)
    e.set_profile(True)
    try:
        b = call(e)
    finally:
        e.set_profile(False)
    return a, b


@pytest.mark.parametrize("n,route", NARROW_CASES)
def test_compress_overlapped_equals_serialised(eng, sm_count, n, route):
    m = route_m(n, route, sm_count)
    if m is None:
        pytest.skip(f"route {route} is not reachable at n={n} on {sm_count} SMs")
    A = _system(m, n, seed=1000 + n)[0]
    (R1, z1), (R2, z2) = _both(eng, lambda e: e.compress(A[:, :n], A[:, n], mode=capi.COMPRESS_CHOLQR2))
    assert R1.tobytes() == R2.tobytes() and z1.tobytes() == z2.tobytes()


NARROW_EKF = [c for c in er.CASES if er.chain(c.n, c.r, c.ld).factor == "dmma"]


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(ld):
        if ld not in made:
            made[ld] = capi.Engine(max_state=ld, max_feats=16, max_meas=1024, max_rows=2048)
        return made[ld]
    yield get
    for e in made.values():
        e.close()


@pytest.mark.parametrize("case", NARROW_EKF, ids=lambda c: f"{c.chain}-ld{c.ld}-N{c.N}-n{c.n}-rows{c.rows}")
def test_ekf_overlapped_equals_serialised(engines, case):
    x = er.case_inputs(case)

    def run(e):
        e.cov_set(x.P)
        st, dx = e.ekf_update(x.off, x.sz, x.H, x.res, Rdiag=x.Rdiag)
        return st, dx, e.cov_get()
    (s1, dx1, P1), (s2, dx2, P2) = _both(engines(case.ld), run)
    assert s1 == s2 and dx1.tobytes() == dx2.tobytes() and P1.tobytes() == P2.tobytes()


@pytest.mark.parametrize("ld,N,n,pos", [(640, 100, 40, 3), (640, 200, 150, 140), (641, 100, 40, 3)])
@pytest.mark.parametrize("kind", ["negative", "nan"])
def test_failed_factor_overlapped(engines, ld, N, n, pos, kind):
    """a non-SPD or NaN pivot with the consumer overlapped: the call returns, P is untouched, the flags are the serialised run's"""
    rng = np.random.default_rng(N + pos)
    P = er.make_P(N, N + pos, 0).copy()
    off, sz = er.place_variables(n, N, rng)
    j = er.columns(off, sz)[pos]
    P[j, :] = 0.0
    P[:, j] = 0.0
    P[j, j] = -1.0 if kind == "negative" else np.nan
    allow = (capi.OVB_ERR_NOT_SPD, capi.OVB_ERR_NONFINITE)

    def run(e):
        e.cov_set(P)
        st, dx = e.ekf_update(off, sz, np.eye(n), np.ones(n), sigma2=1e-3, allow=allow)
        return st, dx, e.cov_get()
    (s1, dx1, P1), (s2, dx2, P2) = _both(engines(ld), run)
    assert s1 == s2 and s1 != capi.OVB_OK
    assert P1.tobytes() == P.tobytes() and P2.tobytes() == P.tobytes()
    assert dx1.tobytes() == dx2.tobytes()


CAPTURED = {  # the shapes of bench.py's configs 1 and 2
    "config1": dict(n_feats=50, n_clones=12, n_cams=1, seed=1),
    "config2": dict(n_feats=400, n_clones=21, n_cams=2, seed=2),
}


@pytest.mark.parametrize("name", sorted(CAPTURED))
def test_update_overlapped_serialised_and_replayed(name):
    """one whole MSCKF update overlapped and serialised, and 50 back-to-back replays of it, end in the same bytes"""
    case = sim.make_update_case(**CAPTURED[name])
    opts = capi.default_opts(col_order=capi.COLS_CANONICAL)
    e = capi.Engine(max_state=256, max_feats=512, max_meas=512 * 2 * 21)
    try:
        e.set_replay(True)

        def run(eng):
            eng.cov_set(case.P)
            st, out, dx, stats = eng.msckf_update(case.frame, case.feats, opts)
            return st, dx.copy(), eng.cov_get()
        (s1, dx1, P1), (s2, dx2, P2) = _both(e, run)
        assert s1 == s2 == capi.OVB_OK
        assert dx1.tobytes() == dx2.tobytes() and P1.tobytes() == P2.tobytes()
        run(e)
        e.msckf_replay(50)
        assert e.cov_get().tobytes() == P1.tobytes()
    finally:
        e.close()
