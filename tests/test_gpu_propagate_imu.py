"""ovb_cov_propagate_imu on the H100: the IMU accumulation of Propagator::propagate_and_clone, EKFPropagation and
augment_clone in one device call, bit-identical to the host loop followed by ovb_cov_propagate and ovb_cov_clone."""
import ctypes as C

import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import capi, simrun
from tests import prop_imu

pytestmark = pytest.mark.gpu
N_CLONES = 5  # clones already in the prior


@pytest.fixture(scope="module")
def exes(tmp_path_factory):
    b.build()
    b.build_sim_tools()
    d = tmp_path_factory.mktemp("prop_imu")
    return {"probe": prop_imu.build_probe(d), "host_prop": prop_imu.build_host_propagation_runner(d)}


@pytest.fixture(scope="module")
def dumps(exes, tmp_path_factory):
    cache, d = {}, tmp_path_factory.mktemp("dumps")

    def get(method, calib, steps):
        key = (method, calib, steps)
        if key not in cache:
            cache[key] = prop_imu.probe(exes["probe"], method, calib, steps, 1000 * calib + steps, d / f"{method}_{calib}_{steps}.bin")
        return cache[key]
    return get


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _engine():
    return capi.Engine(max_state=256, max_feats=16, max_meas=256)


def _prior(d, seed):
    return prop_imu.seeded_prior(d["N"] + 6 * N_CLONES, seed)


def _call(eng, d, with_dt=True, F=None, G=None, qc=None):
    return eng.cov_propagate_imu(d["F"] if F is None else F, d["G"] if G is None else G, d["qc"] if qc is None else qc, d["new_off"], d["old_off"],
                                 d["old_sz"], d["clone_off"], d["clone_size"], d["dnc"] if with_dt else None, d["dt_off"] if with_dt else -1)


def _two_calls(P0, d, Phi, Q, with_dt=True):
    """The host path's device side: ovb_cov_propagate with the host's Phi / Q, then ovb_cov_clone."""
    eng = _engine()
    eng.cov_set(P0)
    st = eng.cov_propagate(d["new_off"], Phi, Q, d["old_off"], d["old_sz"])
    if st == capi.OVB_OK:
        eng.cov_clone(d["clone_off"], d["clone_size"], d["dnc"] if with_dt else None, d["dt_off"] if with_dt else -1)
    P = eng.cov_get()
    eng.close()
    return st, P


GRID = [(m, c, s) for m in ("discrete", "rk4", "analytical") for c in (0, 1, 2) for s in (0, 1, 41, 400)]


@pytest.mark.parametrize("method,calib,steps", GRID)
def test_phi_q_match_host_loop(dumps, method, calib, steps):
    d = dumps(method, calib, steps)
    assert d["n"] == prop_imu.CALIB_N[calib]
    eng = _engine()
    eng.cov_set(_prior(d, 7))
    st, Phi, Q = _call(eng, d)
    assert st == capi.OVB_OK
    assert np.array_equal(_bits(Phi), _bits(d["Phi"])), np.abs(Phi - d["Phi"]).max()
    assert np.array_equal(_bits(Q), _bits(d["Q"])), np.abs(Q - d["Q"]).max()
    eng.close()


@pytest.mark.parametrize("with_dt", [True, False])
@pytest.mark.parametrize("method,calib,steps", GRID)
def test_p_matches_propagate_then_clone(dumps, method, calib, steps, with_dt):
    d = dumps(method, calib, steps)
    P0 = _prior(d, 11 + steps)
    eng = _engine()
    eng.cov_set(P0)
    st, _, _ = _call(eng, d, with_dt)
    P = eng.cov_get()
    eng.close()
    st_ref, P_ref = _two_calls(P0, d, d["Phi"], d["Q"], with_dt)
    assert st == st_ref == capi.OVB_OK
    assert P.shape == P_ref.shape == (P0.shape[0] + 6,) * 2
    assert np.array_equal(_bits(P), _bits(P_ref))


def test_staging_grows_beyond_the_reservation(dumps):
    """2000 steps (five seconds of 400 Hz IMU) outgrow the staging reserved at ovb_create; that call and an ordinary one
    after it on the same context both match the host path."""
    eng = _engine()
    for steps in (2000, 41):
        d = dumps("rk4", 2, steps)
        P0 = _prior(d, 3)
        eng.cov_set(P0)
        st, Phi, Q = _call(eng, d)
        assert st == capi.OVB_OK
        assert np.array_equal(_bits(Phi), _bits(d["Phi"])) and np.array_equal(_bits(Q), _bits(d["Q"]))
        st_ref, P_ref = _two_calls(P0, d, d["Phi"], d["Q"])
        assert st_ref == capi.OVB_OK and np.array_equal(_bits(eng.cov_get()), _bits(P_ref))
    eng.close()


def test_refusals_leave_p_untouched(dumps):
    d = dumps("rk4", 2, 41)
    P0 = _prior(d, 5)
    N, n, S = P0.shape[0], d["n"], d["steps"]
    eng = _engine()
    eng.cov_set(P0)
    lib, h = eng.lib, eng.h
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    F, G, qc, dnc = (np.ascontiguousarray(d[k]) for k in ("F", "G", "qc", "dnc"))
    off, sz = np.ascontiguousarray(d["old_off"]), np.ascontiguousarray(d["old_sz"])

    def p(a, t):
        return None if a is None else a.ctypes.data_as(t)

    def call(n=n, steps=S, F=F, G=G, qc=qc, new_off=0, off=off, sz=sz, nold=len(off), clone_off=0, clone_size=6, dnc=dnc, dt_off=d["dt_off"]):
        return lib.ovb_cov_propagate_imu(h, n, steps, p(F, dp), p(G, dp), p(qc, dp), new_off, p(off, ip), p(sz, ip), nold, clone_off, clone_size,
                                         p(dnc, dp), dt_off, None, None)
    bad_off = off.copy()
    bad_off[-1] = N - 1
    refused = {
        "F NULL": (call(F=None), capi.OVB_ERR_ARG),
        "G NULL": (call(G=None), capi.OVB_ERR_ARG),
        "qc NULL": (call(qc=None), capi.OVB_ERR_ARG),
        "old_off NULL": (call(off=None), capi.OVB_ERR_ARG),
        "old_sz NULL": (call(sz=None), capi.OVB_ERR_ARG),
        "nold = 0": (call(nold=0), capi.OVB_ERR_ARG),
        "steps < 0": (call(steps=-1), capi.OVB_ERR_ARG),
        "new block past N": (call(new_off=N - n + 1), capi.OVB_ERR_ARG),
        "old variable past N": (call(off=bad_off), capi.OVB_ERR_ARG),
        "old sizes != n": (call(nold=len(off) - 1), capi.OVB_ERR_ARG),
        "clone past N": (call(clone_off=N - 5), capi.OVB_ERR_ARG),
        "dt_off past N": (call(dt_off=N), capi.OVB_ERR_ARG),
        "n = 65": (call(n=65), capi.OVB_ERR_CAPACITY),
    }
    for what, (st, want) in refused.items():
        assert st == want, (what, st)
        assert eng.cov_dim() == N, what
        assert np.array_equal(_bits(eng.cov_get()), _bits(P0)), what
    assert b"65" in lib.ovb_last_error(h)
    # a prior the clone would push past max_state
    big = _engine()
    P_big = prop_imu.seeded_prior(253, 1)
    big.cov_set(P_big)
    st = big.lib.ovb_cov_propagate_imu(big.h, n, S, p(F, dp), p(G, dp), p(qc, dp), 0, p(off, ip), p(sz, ip), len(off), 0, 6, None, -1, None, None)
    assert st == capi.OVB_ERR_CAPACITY and big.cov_dim() == 253 and np.array_equal(_bits(big.cov_get()), _bits(P_big))
    big.close()
    eng.close()


def test_negative_diagonal_status_and_no_clone(dumps):
    """Noise densities that drive the propagated diagonal negative: the same status as ovb_cov_propagate on the host's Phi / Q,
    P holds the propagated values, and N does not grow."""
    d = dumps("rk4", 2, 1)
    qc = -1e6 * np.abs(d["qc"])
    Phi, Q = prop_imu.accumulate(d["F"], d["G"], qc)
    P0 = _prior(d, 9)
    eng = _engine()
    eng.cov_set(P0)
    st, Phi_dev, Q_dev = _call(eng, d, qc=qc)
    ref = _engine()
    ref.cov_set(P0)
    st_ref = ref.cov_propagate(d["new_off"], Phi, Q, d["old_off"], d["old_sz"])
    assert st == st_ref == capi.OVB_ERR_NEG_DIAG
    assert np.array_equal(_bits(Phi_dev), _bits(Phi)) and np.array_equal(_bits(Q_dev), _bits(Q))
    assert eng.cov_dim() == P0.shape[0]
    assert np.array_equal(_bits(eng.cov_get()), _bits(ref.cov_get()))
    eng.close()
    ref.close()


@pytest.mark.parametrize("cams,clones,msckf,frames,method", [(1, 11, 50, 300, "discrete"), (1, 11, 50, 300, "rk4"), (1, 11, 50, 300, "analytical"),
                                                             (2, 20, 80, 80, "rk4")])
def test_closed_loop_matches_host_accumulation(exes, tmp_path, cams, clones, msckf, frames, method):
    """The product runner (one ovb_cov_propagate_imu per frame) against the same runner whose engine backend keeps the host
    accumulation: identical estimate files and ATEs."""
    kw = dict(traj=simrun.TRAJ_FIXTURE, cams=cams, clones=clones, msckf=msckf, pts=200, frames=frames, calib=1, integration=method)
    r_dev = simrun.run(est=str(tmp_path / "dev.txt"), **kw)
    r_host = simrun.run(exe=exes["host_prop"], est=str(tmp_path / "host.txt"), **kw)
    assert r_dev["frames"] == r_host["frames"] == frames
    assert (tmp_path / "dev.txt").read_bytes() == (tmp_path / "host.txt").read_bytes()
    assert r_dev["ate_pos_m"] == r_host["ate_pos_m"] and r_dev["ate_ori_deg"] == r_host["ate_ori_deg"]
