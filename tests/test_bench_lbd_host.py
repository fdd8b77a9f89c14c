"""tools/bench_lbd.py runs its host side without a GPU (the CPU arm) and prints one JSON line; the GPU run prints the device
stages, the KITTI-config figure and the HBM byte count."""
import json
import os
import subprocess
import sys

import pytest

from conftest import ROOT
from oracle import lbd

SCRIPT = os.path.join(ROOT, "tools", "bench_lbd.py")


def _run(*extra):
    out = subprocess.run([sys.executable, SCRIPT, *extra], capture_output=True, text=True, check=True, timeout=600).stdout
    lines = [l for l in out.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    return json.loads(lines[0])


def test_bench_lbd_cpu_arm():
    line = _run("--impl", "reference", "--images", "4")
    assert line["unit"] == "images/s"
    if lbd.available():
        assert line["value"] > 0 and line["cpu_baseline"]["cores"] >= 1
    else:
        assert line["value"] is None and line["cpu_baseline"] is None


@pytest.mark.gpu
def test_bench_lbd_gpu_line():
    line = _run("--gpus", "1", "--steps", "2", "--warmup", "1", "--images", "4", "--no-cpu")
    assert line["value"] > 0 and line["kitti_config"]["value"] > 0
    assert all(v > 0 for v in line["kernel_ms_per_step"].values())
    assert line["hbm"]["algorithmic_bytes_per_step"] > 0
