"""bench.py's output contract, checked without a GPU: (1) the `--impl reference` arm (CPU oracle port, the one arm that runs here)
prints ONE JSON line with the keys the driver parses; (2) the device arm refuses to run without CUDA (there is no CPU fallback to time
by accident); (3) the committed line of a single-H100 run carries every key of the contract."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
             "data", "config", "e2e", "cpu_baseline")


def _run(args, env=None, timeout=600):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, env=e, timeout=timeout, cwd=ROOT)


def test_reference_arm_prints_one_contract_line():
    r = _run(["--impl", "reference", "--steps", "1", "--warmup", "0"], env={"THB_BENCH_CPU_ITEMS": "2"})
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and all(k in d for k in BASE_KEYS)
    assert d["value"] > 0 and d["higher_is_better"] is True and d["scaling"] == "strong" and d["dtype"] == "f64"
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] == 2 and "2 of 2048" in d["cpu_baseline"]["sample"]
    assert "workload" in d["config"] and "model" not in d["config"]


def test_device_arm_does_not_run_without_cuda():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a CUDA device is present")
    r = _run(["--steps", "1", "--warmup", "1", "--no-cpu-baseline", "--no-c2"], timeout=300)
    assert r.returncode != 0
    assert not [ln for ln in r.stdout.splitlines() if ln.startswith("{")]      # no number is printed
    assert "NVIDIA" in r.stderr or "CUDA" in r.stderr or "cuda" in r.stderr


def test_committed_final_line_has_every_contract_key():
    d = json.loads(open(os.path.join(ROOT, "profiles", "h100_bench_n1_line.json")).read())
    for k in BASE_KEYS + ("clocks", "gpu_launches", "roofline"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["gpu_launches"] > 0 and d["vs_baseline"] is None
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"]) and d["e2e"]["h2d_bytes_per_step"] > 0
    assert d["e2e"]["value"] < d["value"]                                         # copies inside the timed region cost something
    rf = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(rf) and abs(rf["frac"] - rf["achieved"] / rf["peak"]) < 1e-9
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"])
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"]) and not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert d["parity"]["ok"] is True
