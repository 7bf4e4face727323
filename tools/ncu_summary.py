"""Summarise an `ncu --set full` report (.ncu-rep) into a JSON file: per kernel (short name, averaged over
its captured launches; for k_feature_system the SUM of its three size-class launches = one step's worth) the DRAM bytes,
duration and the DMMA / FP64 / issue utilisation.

Usage: python tools/ncu_summary.py <report>.ncu-rep <out>.json ["how the capture was made"]
Needs `ncu` on PATH (reading a report needs no GPU)."""
import csv
import io
import json
import re
import subprocess
import sys

METRICS = {
    "gpu__time_duration.sum": ("duration_us", 1.0),
    "dram__bytes_read.sum": ("dram_bytes_read", None),
    "dram__bytes_write.sum": ("dram_bytes_write", None),
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": ("sm_throughput_pct", 1.0),
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": ("dram_throughput_pct", 1.0),
    "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active": ("fp64_pipe_active_pct", 1.0),
    "sm__inst_executed_pipe_tensor_subpipe_dmma.avg.pct_of_peak_sustained_active": ("dmma_inst_pct_of_peak", 1.0),
    "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed": ("tensor_pipe_active_pct", 1.0),
    "smsp__issue_active.avg.pct_of_peak_sustained_active": ("issue_active_pct", 1.0),
    "sm__warps_active.avg.pct_of_peak_sustained_active": ("warps_active_pct", 1.0),
    "launch__registers_per_thread": ("registers_per_thread", 1.0),
    "launch__grid_size": ("grid_size", 1.0),
    "launch__block_size": ("block_size", 1.0),
    "smsp__inst_executed.sum": ("warp_instructions", 1.0),
}
UNIT_SCALE = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "us": 1.0, "ns": 1e-3, "ms": 1e3, "msecond": 1e3, "usecond": 1.0, "nsecond": 1e-3}


def short(name: str) -> str:
    m = re.match(r"(?:void )?([A-Za-z0-9_]+)", name)
    return m.group(1) if m else name


def main():
    rep, out = sys.argv[1], sys.argv[2]
    how = sys.argv[3] if len(sys.argv) > 3 else "ncu --set full --clock-control none, cold cache (ncu flushes L2 before every replayed launch)"
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], check=True, capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(hdr)}
    launches = {}
    for r in rows[2:]:
        k = short(r[col["Kernel Name"]])
        rec = {}
        for m, (key, _) in METRICS.items():
            if m not in col or r[col[m]] == "":
                continue
            try:
                v = float(r[col[m]].replace(",", ""))
            except ValueError:
                continue
            rec[key] = v * UNIT_SCALE.get(units[col[m]], 1.0)
        launches.setdefault(k, []).append(rec)
    kernels = {}
    for k, recs in launches.items():
        keys = sorted({q for r in recs for q in r})
        if k == "k_feature_system" and len(recs) % 3 == 0:
            # three size-class launches per step: per-step sums for bytes / time / instructions, the long-track class for the rest
            steps = len(recs) // 3
            agg = {}
            for q in keys:
                vals = [r.get(q, 0.0) for r in recs]
                if q in ("dram_bytes_read", "dram_bytes_write", "duration_us", "warp_instructions", "grid_size"):
                    agg[q] = sum(vals) / steps
                else:
                    agg[q] = sum(vals[0::3]) / steps
            agg["note"] = "sum over the three size-class launches of one step (serialised by ncu; they run side by side in the stream); utilisation figures are the long-track class's"
            kernels[k] = agg
        else:
            kernels[k] = {q: sum(r.get(q, 0.0) for r in recs) / len(recs) for q in keys}
        kernels[k]["launches_captured"] = len(recs)
    json.dump({"how": how, "report": rep, "kernels": kernels}, open(out, "w"), indent=1, sort_keys=True)
    for k, v in kernels.items():
        print(f"{k:24s} {v.get('duration_us', 0):8.1f} us  dram rd {v.get('dram_bytes_read', 0) / 1e6:8.2f} MB  wr {v.get('dram_bytes_write', 0) / 1e6:8.2f} MB  "
              f"fp64 {v.get('fp64_pipe_active_pct', 0):5.1f}%  dmma {v.get('dmma_inst_pct_of_peak', 0):5.1f}%  tensor {v.get('tensor_pipe_active_pct', 0):5.1f}%  issue {v.get('issue_active_pct', 0):5.1f}%")


if __name__ == "__main__":
    main()
