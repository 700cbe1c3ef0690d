"""bench.py contract: the reference arm runs on CPU and prints one JSON line with the required
keys; the CUDA arm (gpu) prints the full line including roofline / e2e / clocks / gpu_launches."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, timeout=600):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, timeout=timeout,
                       cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout[-2000:]
    return json.loads(lines[0])


def test_reference_arm_json_line():
    d = _run(["--impl", "reference", "--config", "tiny", "--ref-batch", "2", "--steps", "2", "--warmup", "1"])
    assert d["impl"] == "reference" and d["unit"] == "images/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["steps"] == 2 and d["warmup"] == 1
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["gpu_launches"] == 0 and d["vs_baseline"] is None


def test_reference_arm_nonzero_rank_is_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--config", "tiny"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""


@pytest.mark.gpu
def test_b200_arm_json_line():
    d = _run(["--config", "tiny", "--batch", "8", "--steps", "2", "--warmup", "3", "--ref-batch", "2", "--extras", "vq,cpu"])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["scaling"] == "weak" and d["data"] == "synthetic" and d["dtype"].startswith("fp16")
    assert d["config"]["precision"] == "fp16"
    v = d["vq"]["depth1"]                              # BASELINE metric part 2 in the same line
    assert d["vq"]["tokens"] == 131072 and v["ms"] > 0 and v["gb_s"] > 0 and 0 < v["frac_of_fp32_fma_peak"] < 1.2
    assert d["gpu_launches"] > 50                     # libb200vq kernels really ran inside the timed region
    assert d["e2e"]["h2d_bytes_per_step"] == 8 * 3 * 64 * 64 * 4 and d["e2e"]["d2h_bytes_per_step"] == 4
    assert d["e2e"]["value"] > 0 and d["e2e"]["value"] != d["value"]
    r = d["roofline"]
    assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and "workload" in d["config"]
