"""CPU tests around ovb_cov_propagate_imu: the binding's argument checks, and the host path it must reproduce — the IMU
accumulation of Propagator::propagate_and_clone (include/ovb200_vio.hpp, state/Propagator.cpp:83-99) behind CovBackend."""
import ctypes as C

import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import capi, simrun
from tests import prop_imu


@pytest.fixture(scope="module")
def lib():
    b.build()
    return capi.load_library()


@pytest.fixture(scope="module")
def probe_exe(lib, tmp_path_factory):
    return prop_imu.build_probe(tmp_path_factory.mktemp("prop_probe"))


def _unbound_engine(lib):
    eng = capi.Engine.__new__(capi.Engine)  # no context: the checks below must refuse before the C call
    eng.lib, eng.h = lib, None
    return eng


def test_binding_checks_shapes(lib):
    eng = _unbound_engine(lib)
    F, G, qc = np.zeros((2, 15, 15)), np.zeros((2, 15, 12)), np.zeros((2, 4))
    args = dict(new_off=0, old_off=[0], old_sz=[15], clone_off=0, clone_size=6)
    with pytest.raises(ValueError):
        eng.cov_propagate_imu(F[:, :, :14], G, qc, **args)
    with pytest.raises(ValueError):
        eng.cov_propagate_imu(F, G[:, :, :11], qc, **args)
    with pytest.raises(ValueError):
        eng.cov_propagate_imu(F, G, qc[:1], **args)
    with pytest.raises(ValueError):
        eng.cov_propagate_imu(F, G, qc, new_off=0, old_off=[0, 3], old_sz=[15], clone_off=0, clone_size=6)
    with pytest.raises(ValueError):
        eng.cov_propagate_imu(F, G, qc, dnc_dt=np.zeros(5), dt_off=15, **args)


def test_null_context_is_refused(lib):
    st = lib.ovb_cov_propagate_imu(None, 15, 0, None, None, None, 0, (C.c_int * 1)(0), (C.c_int * 1)(15), 1, 0, 6, None, -1, None, None)
    assert st == capi.OVB_ERR_ARG


@pytest.mark.parametrize("steps", [0, 1, 41, 400])
@pytest.mark.parametrize("calib", [0, 1, 2])
@pytest.mark.parametrize("method", ["discrete", "rk4", "analytical"])
def test_host_path_matches_the_loop(probe_exe, tmp_path, method, calib, steps):
    """The per-step F, G, qc that propagate_and_clone hands to CovBackend::propagate_imu, accumulated by the base (host)
    implementation, give the Phi / Q of the reference loop bit for bit (numpy restatement in the loop's order)."""
    d = prop_imu.probe(probe_exe, method, calib, steps, 1000 * calib + steps, tmp_path / "dump.bin")
    assert d["n"] == prop_imu.CALIB_N[calib] and d["steps"] == steps
    assert int(d["old_sz"].sum()) == d["n"] and d["clone_size"] == 6
    Phi, Q = prop_imu.accumulate(d["F"], d["G"], d["qc"])
    assert np.array_equal(Phi.view(np.uint64), d["Phi"].view(np.uint64))
    assert np.array_equal(Q.view(np.uint64), d["Q"].view(np.uint64))
    if steps == 0:
        assert np.array_equal(Phi, np.eye(d["n"])) and not Q.any()
    else:
        assert np.all(np.diag(Q)[:15] > 0) and np.array_equal(Q, Q.T)  # the IMU intrinsics carry no process noise


@pytest.mark.parametrize("method", ["discrete", "rk4", "analytical"])
def test_oracle_runner_is_repeatable(oracle, tmp_path, method):
    """Two oracle-backed closed-loop runs through the host propagation path write identical estimates, for each integrator."""
    exe = oracle.build_sim_runner()
    kw = dict(exe=exe, traj=simrun.TRAJ_FIXTURE, cams=1, clones=11, msckf=50, pts=200, frames=60, integration=method)
    r1 = simrun.run(est=str(tmp_path / "a.txt"), **kw)
    r2 = simrun.run(est=str(tmp_path / "b.txt"), **kw)
    assert (tmp_path / "a.txt").read_bytes() == (tmp_path / "b.txt").read_bytes()
    assert r1["frames"] == 60 and r1["ate_pos_m"] == r2["ate_pos_m"] and r1["ate_pos_m"] < 0.2
