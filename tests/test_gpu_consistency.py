"""GPU tests of consistency recording (--consistency) on the CUDA engine: the engine's per-frame NEES and σ of every
base-state coordinate, calibration included, against the oracle-backed runner on the configurations of
tests/test_gpu_sim.py and the non-zero-seed case of tests/test_gpu_monte_carlo.py; and a concurrent batch whose
consistency files equal the same seeds run alone, with estimate files unchanged by the recording."""
import numpy as np
import pytest

from open_vins_b200 import build as b
from open_vins_b200 import simrun

pytestmark = pytest.mark.gpu

CONFIG1 = dict(cams=1, clones=11, msckf=50, pts=200, calib=1)  # BASELINE config 1: mono, 11 clones, 50 features

# (runner options, max relative σ difference, max |ΔNEES|). The bars are the float32-cast noise floor between two builds of
# the same CPU arithmetic, with and without FMA contraction (tools/ate_noise_floor.sh, DESIGN.md §5), times three as for
# the ATE bars of tests/test_gpu_sim.py (3e-6 m over a 1.04e-6 m floor). Floors (σ, NEES): config1 2.7e-5, 2.9e-4;
# stereo 2.2e-5, 2.0e-4; nocalib 1.7e-5, 1.8e-4; seed357 3.0e-5, 9.0e-4.
CASES = {
    "config1": (dict(CONFIG1, frames=300), 8e-5, 9e-4),
    "stereo": (dict(cams=2, clones=20, msckf=120, pts=300, frames=80, calib=1), 7e-5, 6e-4),
    "nocalib": (dict(cams=1, clones=11, msckf=50, pts=200, frames=150, calib=0), 5e-5, 6e-4),
    "seed357": (dict(CONFIG1, seed_init=3, seed_perturb=5, seed_meas=7, frames=300), 9e-5, 2.7e-3),
}


@pytest.fixture(scope="module")
def exes():
    from oracle import ovo_py
    ovo_py.build()
    return b.build_sim_tools(), ovo_py.build_sim_runner()


def _read(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.parametrize("case", list(CASES))
def test_consistency_engine_vs_oracle(exes, tmp_path, case):
    cfg, bar_sigma, bar_nees = CASES[case]
    eng, orc = exes
    cg, co = str(tmp_path / "g.txt"), str(tmp_path / "o.txt")
    rg = simrun.run(exe=eng, consistency=cg, **cfg)
    ro = simrun.run(exe=orc, consistency=co, **cfg)
    assert rg["frames"] == ro["frames"] == cfg["frames"]
    assert rg["status_hist"] == ro["status_hist"], "gate / triangulation decisions differ between the engine and the oracle"
    g, o = simrun.load_consistency(cg), simrun.load_consistency(co)
    assert g["ids"] == o["ids"] and np.array_equal(g["t"], o["t"]) and len(g["t"]) == cfg["frames"]
    assert g["sigma"].shape[1] == g["ids"]["n"]
    rel = np.abs(g["sigma"] - o["sigma"]) / o["sigma"]
    worst = np.unravel_index(np.argmax(rel), rel.shape)
    assert rel.max() <= bar_sigma, f"σ of coordinate {worst[1]} at frame {worst[0]}: relative difference {rel.max():.3e}"
    d_ori, d_pos = np.abs(g["nees_ori"] - o["nees_ori"]).max(), np.abs(g["nees_pos"] - o["nees_pos"]).max()
    assert d_ori <= bar_nees and d_pos <= bar_nees, (d_ori, d_pos)
    assert rg["nees_ori"] == pytest.approx(ro["nees_ori"], abs=bar_nees) and rg["nees_pos"] == pytest.approx(ro["nees_pos"], abs=bar_nees)


def test_concurrent_batch_consistency_equals_single_runs(exes, tmp_path):
    eng, _ = exes
    S, K, kw = 40, 8, dict(CONFIG1, frames=100)
    on, off = tmp_path / "on", tmp_path / "off"
    batch = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(on), consistency=True, seed_meas=S, **kw)
    plain = simrun.run(exe=eng, runs=K, jobs=K, out_dir=str(off), seed_meas=S, **kw)
    assert batch["backend"] == "engine" and [r["seed"] for r in batch["per_run"]] == list(range(S, S + K))
    for entry, pe in zip(batch["per_run"], plain["per_run"]):
        seed = entry["seed"]
        assert _read(on / f"est_{seed}.txt") == _read(off / f"est_{seed}.txt"), f"seed {seed}: the recording changed the estimate"
        assert entry["status_hist"] == pe["status_hist"] and entry["ate_pos_m"] == pe["ate_pos_m"]
        single = str(tmp_path / f"c_{seed}.txt")
        r = simrun.run(exe=eng, consistency=single, seed_meas=seed, **kw)
        assert _read(single) == _read(on / f"consistency_{seed}.txt"), f"seed {seed}: the concurrent run differs from the run alone"
        assert entry["nees_ori"] == pytest.approx(r["nees_ori"], rel=1e-11) and entry["nees_pos"] == pytest.approx(r["nees_pos"], rel=1e-11)
    no = np.array([r["nees_ori"] for r in batch["per_run"]])
    assert batch["nees_ori_mean"] == pytest.approx(np.mean(no), rel=1e-14) and batch["nees_ori_std"] == pytest.approx(np.std(no), rel=1e-12)
