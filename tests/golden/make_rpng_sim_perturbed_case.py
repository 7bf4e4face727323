#!/usr/bin/env python
"""Regenerates tests/golden/rpng_sim_perturbed_mono11_f50.case.gz, the captured update of an rpng_sim run whose filter
starts from a perturbed calibration (--perturb), in the format and from the same runner as
tests/golden/make_rpng_sim_cases.py (the oracle-backed twin, trajectory head, full online calibration).
  config 1 with --perturb: mono, max_clones 11, max_msckf_in_update 50, num_pts 200, seeds 0, update of frame 27. There
  the camera's fx estimate is 1.5 σ from the truth and 1.2 σ from the perturbed start (σ = its 1 px prior), so the
  update's intrinsic columns are evaluated away from both (tests/test_sim_perturb_cpu.py checks it).
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
name, frame = "rpng_sim_perturbed_mono11_f50", 27
args = ["--cams", "1", "--clones", "11", "--msckf", "50", "--pts", "200", "--frames", "30", "--perturb", "--seed-perturb", "0"]
prefix = os.path.join("/tmp", name)
subprocess.check_call([exe, "--traj", traj, "--capture", str(frame), prefix] + args)
with open(prefix + ".case", "rb") as f, gzip.GzipFile(os.path.join(ROOT, "tests", "golden", name + ".case.gz"), "wb", mtime=0) as g:
    g.write(f.read())
print("wrote", name)
