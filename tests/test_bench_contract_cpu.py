"""bench.py's reference arm runs on the host alone: check that it prints exactly ONE JSON line with the contract's keys.
(The GPU arm needs an H100; its line is produced by the same code path for the shared keys.)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_contract_line():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference"
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["metric"] == "msckf_updates_per_sec" and d["unit"] == "updates/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and abs(d["value"] * d["ms_per_step"] - 1e3) < 1e-6 * 1e3
    assert "workload" in d["config"] and "400 MSCKF features" in d["config"]["workload"]
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] == 1 and cb["value"] == d["value"] and cb["sample"]
    e = d["e2e"]
    assert e["value"] == d["value"] and e["unit"] == d["unit"] and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0
    assert d["vs_baseline"] is None and d["dtype"] == "f64" and d["data"] == "rpng_sim"
