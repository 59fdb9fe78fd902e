"""bench.py contract pieces that can run without a GPU: the reference arm
(CPU port of the reference path) prints one JSON line with the agreed keys,
and the GPU arm refuses to run (no CPU fallback) on a GPU-less box."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference",
                          "--steps", "1", "--warmup", "3"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "transpose_GiB_per_s" and d["unit"] == "GiB/s"
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["value"] > 0
    assert d["config"]["round_trip_bit_exact"] is True
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "GiB/s", "h2d_bytes_per_step": 0,
                        "d2h_bytes_per_step": 0}


def test_b200_arm_has_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode != 0
    assert "no CPU fallback" in (out.stderr + out.stdout)
