"""bench.py's CPU arm prints exactly one JSON line with the contract's keys (no GPU needed)."""
import json
import os
import subprocess
import sys

from conftest import ROOT


def test_reference_arm_prints_one_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--points", "20000", "--cpu-cols", "100"], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "cpd_em_iterations_per_sec" and d["unit"] == "it/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["ms_per_step"] > 0
    assert d["cpu_baseline"]["kind"] == "port"
    assert d["cpu_baseline"]["cores"] >= 1 and "sample" in d["cpu_baseline"]
    assert d["config"]["workload"].startswith("rigid CPD, synthetic 3-D N=M=20000")
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    assert "workload" in d["config"]


def test_reference_arm_says_unavailable_for_the_config_without_a_cpu_counterpart():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--config", "5", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([l for l in r.stdout.splitlines() if l.strip()][0])
    assert d["impl"] == "reference" and "unavailable" in d


def test_workload_strings_are_shared_by_both_arms():
    sys.path.insert(0, ROOT)
    import importlib
    src = open(os.path.join(ROOT, "bench.py")).read()
    assert src.count("workload_string(args.config") >= 3          # reference arm, rigid/affine arm, non-rigid arm
