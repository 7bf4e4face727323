#!/usr/bin/env python
"""Regenerates tests/golden/rpng_sim_equi_mono11_f50.case.gz, the captured update of an rpng_sim run on an equidistant
(fisheye) camera, in the format and from the same runner as tests/golden/make_rpng_sim_cases.py (the oracle-backed twin,
trajectory head, seeds 0, full online calibration).
  config 1 on a fisheye camera: mono, max_clones 11, max_msckf_in_update 50, --cam-model equi (TUM-VI cam0 intrinsics,
  512 x 512), num_pts 200 (the closed-loop runs' value; with 400 the wide field of view leaves most tracks too short to
  triangulate), update of frame 25: 43 features in, 28 triangulated
"""
import gzip
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ovo_py  # noqa: E402
exe = ovo_py.build_sim_runner()
traj = os.path.join(ROOT, "tests", "golden", "traj_tum_corridor1_head.bin")
name, frame = "rpng_sim_equi_mono11_f50", 25
args = ["--cams", "1", "--clones", "11", "--msckf", "50", "--pts", "200", "--frames", "30", "--cam-model", "equi"]
prefix = os.path.join("/tmp", name)
subprocess.check_call([exe, "--traj", traj, "--capture", str(frame), prefix] + args)
with open(prefix + ".case", "rb") as f, gzip.GzipFile(os.path.join(ROOT, "tests", "golden", name + ".case.gz"), "wb", mtime=0) as g:
    g.write(f.read())
print("wrote", name)
