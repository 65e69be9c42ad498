"""CPU: bench.py's reference arm runs without a GPU and prints exactly ONE JSON line on stdout with the contract keys."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "0"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, p.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "TFLOP/s" and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["value"] > 0 and d["config"]["workload"].startswith("cfg5")
    for k in ("metric", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "vs_baseline", "dtype", "data"):
        assert k in d


def test_ours_arm_refuses_to_run_without_gpu():
    import torch
    if torch.cuda.is_available():
        return
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300)
    assert p.returncode != 0 and "no CPU fallback" in (p.stderr + p.stdout)


def test_metric_is_baseline_json_verbatim_and_recorded_line_has_the_contract_keys():
    """The metric string is BASELINE.json's, and the line recorded on an H100 (profiles/) carries every contract key."""
    sys.path.insert(0, ROOT)
    import bench
    assert bench.METRIC == json.load(open(os.path.join(ROOT, "BASELINE.json")))["metric"]
    d = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_n1.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"):
        assert k in d, k
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(d["roofline"])
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"])
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"])
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["gpu_launches"] > 0 and d["config"]["workload"].startswith("cfg5")
