"""CPU tests of equidistant (fisheye) cameras in the host-side rpng_sim pipeline (SimCamera in include/ovb200_sim.hpp, the
runner's --cam-model): the restated cv::fisheye::undistortPoints and CamEqui::distort_f, the simulator's fisheye pixels, the
flag, and the measured consistency of the filter on a fisheye rig, with the CPU oracle as backend
(tests/cpp/run_simulation_oracle). Reference: ov_core/src/cam/CamEqui.h, ov_msckf/src/sim/Simulator.cpp."""
import os
import subprocess

import numpy as np
import pytest

from open_vins_b200 import simrun

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAJ = simrun.TRAJ_FIXTURE
K_EQUI = np.array([[190.978, 0, 254.93], [0, 190.973, 256.897], [0, 0, 1.0]])  # TUM-VI cam0, 512 x 512 (open_vins_b200/sim.py)
D_EQUI = np.array([0.0034, 0.0007, -0.0020, 0.0002])
MONO = dict(traj=TRAJ, cams=1, clones=11, msckf=50, pts=200)  # BASELINE config-1 shape


@pytest.fixture(scope="module")
def runner():
    from oracle import ovo_py
    ovo_py.build()
    return ovo_py.build_sim_runner()


@pytest.fixture(scope="module")
def probe(runner):
    exe = os.path.join(ROOT, "tests", "cpp", "equi_probe")
    src = os.path.join(ROOT, "tests", "cpp", "equi_probe.cpp")
    deps = [src, os.path.join(ROOT, "oracle", "ovo_core.hpp")] + [os.path.join(ROOT, "include", h) for h in
                                                                    ("ovb200_vio.hpp", "ovb200_math.hpp", "ovb200_sim.hpp", "ovb200_host.hpp")]
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), src, "-L", os.path.join(ROOT, "open_vins_b200"),
                               "-lovb200", "-Wl,-rpath,$ORIGIN/../../open_vins_b200", "-o", exe])
    return exe


def _undistort(probe, uv, D=None):
    inp = "".join(f"{float(u)!r} {float(v)!r}\n" for u, v in uv)
    out = subprocess.run([probe, "undistort"] + ([repr(float(k)) for k in D] if D is not None else []), input=inp, check=True, capture_output=True, text=True).stdout.split()
    return np.array([float(x) for x in out], dtype=np.float64).astype(np.float32).reshape(-1, 2)


def test_undistort_matches_opencv_fisheye(probe):
    """SimCamera::undistort_f of an equidistant camera = cv::fisheye::undistortPoints (cam/CamEqui.h:104-124), bit for bit in
    float32: a 65 x 65 pixel grid over the whole 512 x 512 image, corners included (theta_d there is past pi/2 and clamped),
    the principal point (theta_d below the solver's epsilon), rings of points at theta_d = pi/2 (1 + e) for small e, and
    pixels far outside the image."""
    cv2 = pytest.importorskip("cv2")
    g = np.linspace(0, 512, 65)
    pts = [(u, v) for u in g for v in g]
    cx, cy, fx, fy = K_EQUI[0, 2], K_EQUI[1, 2], K_EQUI[0, 0], K_EQUI[1, 1]
    pts.append((cx, cy))
    for e in (-1e-3, -1e-6, -1e-9, 0.0, 1e-9, 1e-6, 1e-3, 0.5, 3.0):
        for a in np.linspace(0, 2 * np.pi, 13):
            th = np.pi / 2 * (1 + e)
            pts.append((cx + fx * th * np.cos(a), cy + fy * th * np.sin(a)))
    pts += [(-5000.0, 10.0), (1e5, -1e5), (cx + 1e-6, cy)]
    uv = np.array(pts, dtype=np.float32)
    ref = cv2.fisheye.undistortPoints(uv.reshape(-1, 1, 2), K_EQUI, D_EQUI).reshape(-1, 2)
    assert ref.dtype == np.float32
    got = _undistort(probe, uv)
    bad = np.flatnonzero(np.any(got.view(np.uint32) != ref.view(np.uint32), axis=1))
    assert bad.size == 0, f"{bad.size} of {len(uv)} points differ, first {uv[bad[:3]]}: {got[bad[:3]]} vs {ref[bad[:3]]}"
    # with these intrinsics every point converges, the clamped corners included
    assert np.all(got[:, 0] != -1e6)


@pytest.mark.parametrize("D", [[-1.0, 0.5, 0.0, 0.0], [2.0, -3.0, 1.0, 0.0]])
def test_undistort_failure_exit_matches_opencv_fisheye(probe, D):
    """OpenCV's other exit: with distortion strong enough that the Newton solve on theta fails to converge in 10 steps or
    flips theta's sign, undistortPoints returns (-1e6, -1e6). Same grid test, bit for bit, on a 111 x 111 grid that reaches
    1.6 image widths out."""
    cv2 = pytest.importorskip("cv2")
    g = np.linspace(-300, 800, 111)
    uv = np.array([(u, v) for u in g for v in g], dtype=np.float32)
    ref = cv2.fisheye.undistortPoints(uv.reshape(-1, 1, 2), K_EQUI, np.array(D)).reshape(-1, 2)
    got = _undistort(probe, uv, D)
    bad = np.flatnonzero(np.any(got.view(np.uint32) != ref.view(np.uint32), axis=1))
    assert bad.size == 0, f"{bad.size} of {len(uv)} points differ, first {uv[bad[:3]]}: {got[bad[:3]]} vs {ref[bad[:3]]}"
    failed = np.all(got == -1e6, axis=1)
    assert 300 < failed.sum() < 0.1 * len(uv)


def test_distort_matches_oracle(probe):
    """SimCamera::distort_f of an equidistant camera (CamEqui::distort_f, cam/CamEqui.h:136-158) and the oracle's equidistant
    distort_d (oracle/ovo_core.hpp), which the update residual restates: the same float pixel, bit for bit, on 1.45 million
    normalized points out to theta = 1.34 rad and around the small-radius switch at r = 1e-8."""
    n, diff = (int(x) for x in subprocess.run([probe, "oracle"], check=True, capture_output=True, text=True).stdout.split())
    assert n == 1201 * 1201 + 81 * 4 and diff == 0


@pytest.mark.parametrize("models", ["equi", "radtan,equi"])
def test_simulated_pixels_against_opencv_projection(probe, models):
    """Third-party pin of the simulator's fisheye measurements (Simulator::project_pointcloud through CamEqui::distort_f):
    the map points under the true pose go through cv2.fisheye.projectPoints (cv2.projectPoints for a radtan camera of the
    mixed rig) with the conventions of tests/test_sim_cpu.py's radtan twin. The simulator's noise-free float32 pixels agree
    to float32 rounding (the same 5e-4 px bar as the radtan test)."""
    cv2 = pytest.importorskip("cv2")
    from scipy.spatial.transform import Rotation
    out = subprocess.run([probe, "simproj", TRAJ, models], check=True, capture_output=True, text=True).stdout.strip().splitlines()
    i, seen, worst = 0, set(), 0.0
    while i < len(out):
        head = out[i].split()
        assert head[0] == "FRAME"
        n = int(head[2])
        v = np.array([float(x) for x in head[3:]])
        q_GtoI, p_IinG, q_ItoC, p_IinC = v[0:4], v[4:7], v[7:11], v[11:14]
        model, w, h, intr = int(v[14]), int(v[15]), int(v[16]), v[17:25]
        pts = np.array([[float(x) for x in line.split()] for line in out[i + 1:i + 1 + n]])
        i += 1 + n
        if n == 0:
            continue
        R_GtoI = Rotation.from_quat(q_GtoI).as_matrix().T
        R_ItoC = Rotation.from_quat(q_ItoC).as_matrix().T
        R_GtoC = R_ItoC @ R_GtoI
        t = R_ItoC @ (-R_GtoI @ p_IinG) + p_IinC
        K = np.array([[intr[0], 0, intr[2]], [0, intr[1], intr[3]], [0, 0, 1.0]])
        rvec = cv2.Rodrigues(R_GtoC)[0]
        P = np.ascontiguousarray(pts[:, :3]).reshape(-1, 1, 3)  # cv2.fisheye misreads a strided view
        if model == 1:
            assert (w, h) == (512, 512) and np.array_equal(K, K_EQUI) and np.array_equal(intr[4:], D_EQUI)
            img, _ = cv2.fisheye.projectPoints(P, rvec, t, K, np.ascontiguousarray(intr[4:8]))
        else:
            assert (w, h) == (752, 480)
            img, _ = cv2.projectPoints(P, rvec, t, K, np.ascontiguousarray(intr[4:8]))
        worst = max(worst, float(np.abs(img.reshape(-1, 2) - pts[:, 3:5]).max()))
        seen.add(model)
        pc = (R_GtoC @ pts[:, :3].T).T + t
        assert np.all(pc[:, 2] > 0.1) and np.all((pts[:, 3] >= 0) & (pts[:, 3] <= w) & (pts[:, 4] >= 0) & (pts[:, 4] <= h))
    assert seen == ({0, 1} if "," in models else {1})
    assert worst <= 5e-4, worst


@pytest.mark.parametrize("arg,cams", [("fisheye", 1), ("", 1), ("equi,", 1), ("Equi", 2), ("radtan,equi", 1), ("equi,equi,equi", 2),
                                      ("radtan,equi", 3)])
def test_bad_cam_model_is_refused(runner, tmp_path, arg, cams):
    """An unknown model, an empty entry, or a per-camera list whose length is not the camera count: status 2, nothing
    printed or written."""
    est = str(tmp_path / "e.txt")
    r = subprocess.run([runner, "--traj", TRAJ, "--cams", str(cams), "--frames", "5", "--est", est, "--cam-model", arg], capture_output=True,
                       text=True, cwd=tmp_path)
    assert r.returncode == 2 and "--cam-model" in r.stderr and r.stdout == ""
    assert os.listdir(tmp_path) == []


def test_flag_reaches_the_run_and_radtan_is_unchanged(runner, tmp_path):
    """--cam-model radtan is the flag-less run, byte for byte, plus the JSON's "cam_model"; one value stands for every
    camera; equi changes the measurements, and a mixed rig is its own run."""
    kw = dict(MONO, cams=2, frames=30)
    e0, e1 = str(tmp_path / "e0.txt"), str(tmp_path / "e1.txt")
    r0 = simrun.run(exe=runner, est=e0, **kw)
    r1 = simrun.run(exe=runner, est=e1, cam_model="radtan", **kw)
    assert open(e0, "rb").read() == open(e1, "rb").read()
    assert "cam_model" not in r0 and r1["cam_model"] == ["radtan", "radtan"]
    assert {k: v for k, v in r1.items() if k != "cam_model" and not k.startswith("mean_ms_")} == {k: v for k, v in r0.items() if not k.startswith("mean_ms_")}
    re_ = simrun.run(exe=runner, cam_model="equi", **kw)
    rm = simrun.run(exe=runner, cam_model=["radtan", "equi"], **kw)
    assert re_["cam_model"] == ["equi", "equi"] and rm["cam_model"] == ["radtan", "equi"]
    assert len({r0["ate_pos_m"], re_["ate_pos_m"], rm["ate_pos_m"]}) == 3
    assert re_["frames"] == rm["frames"] == 30 and re_["ate_pos_m"] < 0.2 and rm["ate_pos_m"] < 0.2


def test_measured_nees_of_the_filter_on_fisheye(runner, tmp_path):
    """8 seeds x 300 frames at config 1 on an equidistant camera, on the oracle (DESIGN.md §5). Measured: mean ANEES 1.32 for
    orientation and 1.19 for position (radtan: 0.905 and 0.415), and RMS errors of 0.49 to 2.89 σ per calibration
    coordinate, 1.16 σ over all of them; the largest are the camera's fx, fy, cx, cy (2.9, 2.6, 2.5, 2.0 σ). The bounds are
    a factor of about 1.5 around these values, as in the radtan twin of tests/test_consistency_cpu.py."""
    out = tmp_path / "mc"
    batch = simrun.run(exe=runner, runs=8, jobs=8, out_dir=str(out), consistency=True, seed_meas=0, cam_model="equi", **dict(MONO, frames=300))
    assert batch["cam_model"] == ["equi"]
    paths = [str(out / f"consistency_{s}.txt") for s in range(8)]
    a = simrun.average_nees(paths)
    assert len(a["t"]) == 300 and a["runs"] == 8
    assert 0.9 <= np.mean(a["anees_ori"]) <= 2.0, np.mean(a["anees_ori"])
    assert 0.8 <= np.mean(a["anees_pos"]) <= 1.8, np.mean(a["anees_pos"])
    assert batch["nees_ori_mean"] == pytest.approx(np.mean(a["anees_ori"]), rel=1e-12)
    assert batch["nees_pos_mean"] == pytest.approx(np.mean(a["anees_pos"]), rel=1e-12)
    cs = [simrun.load_consistency(p) for p in paths]
    z = np.stack([c["err"] for c in cs]) / np.stack([c["sigma"] for c in cs])
    rms = np.sqrt(np.mean(z ** 2, axis=(0, 1)))[15:]  # every calibration coordinate: dw da tg gyro dt cam0_ext cam0_intr
    assert np.all((rms >= 0.3) & (rms <= 4.5)), rms
    assert 0.8 <= np.sqrt(np.mean(rms ** 2)) <= 1.7
