"""GPU tests of the rpng_sim runner's Monte-Carlo mode on the CUDA engine (open_vins_b200/ovb_run_simulation --runs K
--jobs J): every run owns its ovb_ctx on the same device, and the engine is deterministic (no floating-point atomics, fixed
reduction orders, DESIGN.md §4), so a run gives the same bits alone or beside seven others. A non-zero seed is also
checked against the oracle-backed runner."""
import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import simrun

pytestmark = pytest.mark.gpu

CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1)  # BASELINE config 1: mono, 11 clones, 50 features


@pytest.fixture(scope="module")
def exes():
    from oracle import ovo_py
    ovo_py.build()
    return b.build_sim_tools(), ovo_py.build_sim_runner()


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def test_concurrent_runs_equal_single_runs(exes, tmp_path):
    eng, _ = exes
    S, K = 40, 8
    out = tmp_path / "mc"
    batch = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(out), seed_meas=S, frames=100, **CONFIG1)
    assert batch["backend"] == "engine" and batch["runs"] == K and batch["jobs"] == K
    assert [r["seed"] for r in batch["per_run"]] == list(range(S, S + K))
    for entry in batch["per_run"]:
        seed = entry["seed"]
        single = str(tmp_path / f"single_{seed}.txt")
        r = simrun.run(exe=eng, est=single, seed_meas=seed, frames=100, **CONFIG1)
        assert _read(single) == _read(out / f"est_{seed}.txt"), f"seed {seed}: the concurrent run differs from the run alone"
        assert entry["status_hist"] == r["status_hist"] and entry["frames"] == r["frames"] == 100
    # the batch's statistics are numpy's (population standard deviation, ddof = 0) over the per-run ATEs
    p = np.array([r["ate_pos_m"] for r in batch["per_run"]])
    o = np.array([r["ate_ori_deg"] for r in batch["per_run"]])
    assert batch["ate_pos_m_mean"] == pytest.approx(np.mean(p), rel=1e-14) and batch["ate_pos_m_std"] == pytest.approx(np.std(p), rel=1e-12)
    assert batch["ate_ori_deg_mean"] == pytest.approx(np.mean(o), rel=1e-14) and batch["ate_ori_deg_std"] == pytest.approx(np.std(o), rel=1e-12)
    assert len(set(p.tolist())) == K  # eight seeds, eight different noise draws
    assert np.all(p < 0.3)


def test_nonzero_seed_engine_vs_oracle(exes, tmp_path):
    """Same decision equality and trajectory bars as tests/test_gpu_sim.py, at another point of the seed space. The bars
    are the float32-cast noise floor between any two builds that are not bit-identical (DESIGN.md §5): 2e-5 m pointwise
    and 3e-6 m in position ATE."""
    eng, orc = exes
    kw = dict(seed_init=3, seed_perturb=5, seed_meas=7, frames=300, **CONFIG1)
    eg, eo = str(tmp_path / "g.txt"), str(tmp_path / "o.txt")
    rg = simrun.run(exe=eng, est=eg, **kw)
    ro = simrun.run(exe=orc, est=eo, **kw)
    assert rg["frames"] == ro["frames"] == kw["frames"]
    assert rg["status_hist"] == ro["status_hist"], "gate / triangulation decisions differ between the engine and the oracle"
    _, pg, _, _, _ = simrun.load_estimate(eg)
    _, po, _, _, _ = simrun.load_estimate(eo)
    assert np.abs(pg - po).max() <= 2e-5
    assert abs(rg["ate_pos_m"] - ro["ate_pos_m"]) <= 3e-6
    assert abs(rg["ate_ori_deg"] - ro["ate_ori_deg"]) <= 1e-4
    assert rg["ate_pos_m"] < 0.3
