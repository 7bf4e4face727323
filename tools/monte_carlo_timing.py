#!/usr/bin/env python
"""Monte-Carlo batches of the rpng_sim runner on one GPU: how far K concurrent closed-loop runs overlap.

For each shape and K in --ks, one process of open_vins_b200/ovb_run_simulation --runs K --jobs K (K host threads, one
ovb_ctx each on device 0, measurement seeds 0 .. K-1). The host clock goes around the whole process: start-up, CUDA
initialisation, K context creations, K closed loops and teardown. runs/s = K / that time; frames/s = the frames of all
runs / that time. The runner's own wall clock (threads only) is reported beside it.

Then, per shape, one single run under tools/alloc_probe.c (LD_PRELOAD, built in a temporary directory): the device
memory one ovb_create takes (cudaMemGetInfo before and after) and every cudaMalloc the engine makes outside ovb_create,
i.e. each time a buffer that grows on demand is (re)allocated, with the update it happened in and the library function
that made it. A reallocation frees first, and cudaFree waits for the whole device, so growth after the first updates
would stall the other runs of a batch.

  python tools/monte_carlo_timing.py [--ks 1,2,4,8,16] [--out FILE]
  python tools/monte_carlo_timing.py --consistency ab --ks 1,16 [--reps 3]

--consistency on runs every batch with --consistency (per frame, one read of the covariance's base block and its
synchronisation, the errors and NEES, and DIR/consistency_<seed>.txt). --consistency ab measures its cost: for each shape
and K, --reps rounds of both arms back to back, the order alternating from round to round; both arms write their estimate
files to a temporary --out-dir, so the difference is the consistency recording alone. The growth probe is skipped.

Prints one JSON line per measurement, the card's name, power limit and max SM clock among them. Needs a GPU; there is no
CPU path."""
import argparse
import bisect
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from open_vins_b200 import build as b  # noqa: E402
from open_vins_b200 import simrun  # noqa: E402

SHAPES = {
    # BASELINE config 1: mono, 11 clones, 50 features per update
    "config1": dict(cams=1, clones=11, msckf=50, pts=200, frames=300),
    # BASELINE config 2: stereo, 20 clones, 400 features per update (the map size tests/golden/make_rpng_sim_cases.py uses)
    "config2": dict(cams=2, clones=20, msckf=400, pts=6000, frames=100),
}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,memory.total"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], check=True, capture_output=True, text=True).stdout
    name, power, clock, mem = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock, memory_total=mem, host_cpus=os.cpu_count())


def runner_cmd(exe, shape):
    s = SHAPES[shape]
    return [exe, "--traj", simrun.TRAJ_FIXTURE, "--cams", str(s["cams"]), "--clones", str(s["clones"]), "--msckf", str(s["msckf"]), "--pts",
            str(s["pts"]), "--frames", str(s["frames"])]


def time_batch(exe, shape, k, consistency=False, out_dir=None):
    extra = (["--consistency"] if consistency else []) + (["--out-dir", out_dir] if out_dir else [])
    t0 = time.perf_counter()
    out = subprocess.run(runner_cmd(exe, shape) + ["--runs", str(k), "--jobs", str(k)] + extra, check=True, capture_output=True, text=True).stdout
    wall = time.perf_counter() - t0
    r = json.loads(out.strip().splitlines()[-1])
    rec = dict(tool="monte_carlo_timing", shape=shape, runs=k, jobs=r["jobs"], frames_total=r["frames_total"], process_s=wall,
               runs_per_s=k / wall, frames_per_s=r["frames_total"] / wall, runner_wall_s=r["wall_s"], runner_runs_per_s=r["runs_per_s"],
               ate_pos_m_mean=r["ate_pos_m_mean"], ate_pos_m_std=r["ate_pos_m_std"])
    if consistency:
        rec.update(consistency=True, runner_frames_per_s=r["frames_per_s"], nees_ori_mean=r["nees_ori_mean"], nees_pos_mean=r["nees_pos_mean"])
    elif out_dir:
        rec.update(consistency=False, runner_frames_per_s=r["frames_per_s"])
    return rec


def text_symbols(lib):
    """(address, demangled name) of the library's functions, sorted, from its symbol table."""
    out = subprocess.run(["nm", "-C", "--defined-only", lib], check=True, capture_output=True, text=True).stdout
    syms = []
    for line in out.splitlines():
        parts = line.split(" ", 2)
        if len(parts) == 3 and parts[1] in "tTW":
            syms.append((int(parts[0], 16), parts[2]))
    syms.sort()
    return syms


def probe_growth(exe, shape, tmp):
    src = os.path.join(ROOT, "tools", "alloc_probe.c")
    so = os.path.join(tmp, "alloc_probe.so")
    if not os.path.exists(so):
        subprocess.check_call([os.environ.get("CC", "cc"), "-shared", "-fPIC", "-O2", "-o", so, src, "-ldl", "-lpthread"])
    log = os.path.join(tmp, f"alloc_{shape}.log")
    env = dict(os.environ, LD_PRELOAD=so, OVB_ALLOC_LOG=log)
    subprocess.run(runner_cmd(exe, shape), check=True, capture_output=True, text=True, env=env)
    syms = text_symbols(b.OUT)
    addrs = [a for a, _ in syms]
    create_bytes, sites = [], {}
    for line in open(log):
        f = line.split()
        if f[0] == "create":
            create_bytes.append(int(f[1]))
            continue
        update, nbytes, off, obj = int(f[1]), int(f[2]), int(f[3]), f[4]
        i = bisect.bisect_right(addrs, off) - 1
        fn = syms[i][1] if os.path.basename(obj) == os.path.basename(b.OUT) and i >= 0 else os.path.basename(obj)
        site = sites.setdefault(fn.split("(")[0], dict(count=0, updates=[], bytes=[]))
        site["count"] += 1
        site["updates"].append(update)
        site["bytes"].append(nbytes)
    return dict(tool="monte_carlo_timing", shape=shape, probe="growth", ovb_create_device_bytes=create_bytes, growth_sites=sites)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--consistency", choices=["off", "on", "ab"], default="off", help="record consistency in every batch, or A/B it")
    ap.add_argument("--reps", type=int, default=3, help="rounds of both arms per shape and K with --consistency ab")
    a = ap.parse_args()
    exe = b.build_sim_tools()
    recs = [dict(tool="monte_carlo_timing", gpu=gpu_info())]
    print(json.dumps(recs[-1]), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        for shape in a.shapes.split(","):
            subprocess.run(runner_cmd(exe, shape)[:-2] + ["--frames", "20"], check=True, capture_output=True)  # warm-up: driver, page cache
            for k in [int(x) for x in a.ks.split(",")]:
                if a.consistency != "ab":
                    recs.append(time_batch(exe, shape, k, consistency=a.consistency == "on"))
                    print(json.dumps(recs[-1]), flush=True)
                    continue
                for rep in range(a.reps):
                    for arm in ((False, True) if rep % 2 == 0 else (True, False)):
                        d = tempfile.mkdtemp(dir=tmp)
                        recs.append(dict(time_batch(exe, shape, k, consistency=arm, out_dir=d), rep=rep))
                        print(json.dumps(recs[-1]), flush=True)
            if a.consistency != "ab":
                recs.append(probe_growth(exe, shape, tmp))
                print(json.dumps(recs[-1]), flush=True)
    recs.append(dict(tool="monte_carlo_timing", gpu_after=gpu_info()))
    print(json.dumps(recs[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in recs))


if __name__ == "__main__":
    main()
