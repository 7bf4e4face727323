#!/bin/bash
# How far apart are two builds of the SAME CPU arithmetic on an rpng_sim run? Builds the oracle twice — as shipped
# (-ffp-contract=off) and with FMA contraction (-ffp-contract=fast -mfma, what an -O3 build of the reference's Eigen code is
# free to do) — runs the 300-frame config-1 simulation with each and prints the pointwise and ATE differences, and from the
# two runs' consistency files (--consistency) the max relative σ difference over every base-state coordinate and the max
# |ΔNEES| of orientation and position. With --perturb, also the max |Δ| of the JSON's per-block calibration errors
# (calib_nerr_first / calib_nerr_last, RMS of err/σ).
#   tools/ate_noise_floor.sh [FRAMES] [extra runner options, e.g. --cams 2 --clones 20 --msckf 120 --pts 300]
# Measured here: max |dp| = 5.9e-6 m, |dATE| = 1.04e-6 m  => the floor under BASELINE.json's "ATE within 1e-6 m".
# σ and NEES floors per configuration: DESIGN.md §5.
set -e
cd "$(dirname "$0")/.."
D=/tmp/ovb_ate_floor; mkdir -p $D
g++ -std=c++17 -O3 -fno-math-errno -funroll-loops -ffp-contract=fast -mfma -mavx2 -fPIC -shared -o $D/libovoracle.so oracle/ovo_capi.cpp
g++ -std=c++17 -O2 -DOVB_SIM_ORACLE -I tests/cpp -I include tools/run_simulation.cpp -L open_vins_b200 -lovb200 -L $D -lovoracle \
    -Wl,-rpath,$PWD/open_vins_b200 -Wl,-rpath,$D -o $D/run_fma
A="--traj tests/golden/traj_tum_corridor1_head.bin --cams 1 --clones 11 --msckf 50 --pts 200 --frames ${1:-300} ${*:2}"
$D/run_fma $A --est $D/est_fma.txt --consistency $D/cons_fma.txt > $D/json_fma.txt
python -c "from oracle import ovo_py; print(ovo_py.build_sim_runner())" > /dev/null
tests/cpp/run_simulation_oracle $A --est $D/est_ref.txt --consistency $D/cons_ref.txt > $D/json_ref.txt
python - <<PY
import numpy as np
from open_vins_b200 import simrun
a=np.loadtxt('$D/est_fma.txt',comments='#'); b=np.loadtxt('$D/est_ref.txt',comments='#')
g=b[:,8:11]; ate=lambda p:np.sqrt(np.mean(np.sum((p-g)**2,axis=1)))
print('max |dp| = %.3e m   |dATE| = %.3e m   (ATE %.6f m)' % (np.abs(a[:,1:4]-b[:,1:4]).max(), abs(ate(a[:,1:4])-ate(b[:,1:4])), ate(b[:,1:4])))
ca=simrun.load_consistency('$D/cons_fma.txt'); cb=simrun.load_consistency('$D/cons_ref.txt')
print('max rel dsigma = %.3e   max |dNEES| ori = %.3e  pos = %.3e   (max NEES ori %.3f pos %.3f)' % (
    np.max(np.abs(ca['sigma']-cb['sigma'])/cb['sigma']), np.max(np.abs(ca['nees_ori']-cb['nees_ori'])),
    np.max(np.abs(ca['nees_pos']-cb['nees_pos'])), cb['nees_ori'].max(), cb['nees_pos'].max()))
import json
ja=json.load(open('$D/json_fma.txt')); jb=json.load(open('$D/json_ref.txt'))
if 'calib_nerr_last' in jb:
    print('max |d calib_nerr| = %.3e' % max(abs(ja[k][b]-jb[k][b]) for k in ('calib_nerr_first','calib_nerr_last') for b in jb[k]))
PY
