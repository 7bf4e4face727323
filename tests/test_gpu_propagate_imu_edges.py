"""ovb_cov_propagate_imu at every width edge of its accumulation kernel (k_prop_accumulate, csrc/k_ekf.cu): synthetic F
(near identity), G and positive qc for n = 1 .. 64. From n = 45 the n(n+1)/2 symmetrised pairs outnumber the kernel's 1024
threads, and n = 64 takes its whole shared-memory budget. Phi / Q are the host loop's bits (tests/prop_imu.accumulate) and
P is the bits of ovb_cov_propagate + ovb_cov_clone on them; n = 65 is refused with P unchanged."""
import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import capi
from tests import prop_imu

pytestmark = pytest.mark.gpu
N_CLONES = 5  # clones already in the prior


@pytest.fixture(scope="module")
def eng():
    b.build()
    e = capi.Engine(max_state=256, max_feats=16, max_meas=256)
    yield e
    e.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


@pytest.mark.parametrize("steps", [0, 1, 2, 3, 41])
@pytest.mark.parametrize("n", [1, 2, 16, 31, 32, 33, 44, 45, 46, 63, 64, 65])
def test_accumulation_width_edges(eng, n, steps):
    rng = np.random.default_rng(100 * n + steps)
    F = np.eye(n) + 0.01 * rng.standard_normal((steps, n, n))
    G = 0.1 * rng.standard_normal((steps, n, 12))
    qc = rng.uniform(0.5, 2.0, (steps, 4))
    h = (n + 1) // 2
    old_off, old_sz = ([h, 0], [n - h, h]) if n > 1 else ([0], [1])  # the IMU block's variables, listed out of order
    N = n + 6 * N_CLONES
    clone_off, dnc, dt_off = n, rng.standard_normal(6), N - 1
    P0 = prop_imu.seeded_prior(N, n)
    eng.cov_set(P0)
    if n > 64:
        with pytest.raises(capi.OvbError) as e:
            eng.cov_propagate_imu(F, G, qc, 0, old_off, old_sz, clone_off, 6, dnc, dt_off)
        assert e.value.code == capi.OVB_ERR_CAPACITY
        assert eng.cov_dim() == N and np.array_equal(_bits(eng.cov_get()), _bits(P0))
        return
    st, Phi, Q = eng.cov_propagate_imu(F, G, qc, 0, old_off, old_sz, clone_off, 6, dnc, dt_off)
    P = eng.cov_get()
    Phi_ref, Q_ref = prop_imu.accumulate(F, G, qc)
    assert st == capi.OVB_OK
    assert np.array_equal(_bits(Phi), _bits(Phi_ref)), np.abs(Phi - Phi_ref).max()
    assert np.array_equal(_bits(Q), _bits(Q_ref)), np.abs(Q - Q_ref).max()
    # the two-call path on the same context: ovb_cov_propagate with the host's Phi / Q, then ovb_cov_clone
    eng.cov_set(P0)
    assert eng.cov_propagate(0, Phi_ref, Q_ref, old_off, old_sz) == capi.OVB_OK
    eng.cov_clone(clone_off, 6, dnc, dt_off)
    P_ref = eng.cov_get()
    assert P.shape == P_ref.shape == (N + 6,) * 2
    assert np.array_equal(_bits(P), _bits(P_ref))
