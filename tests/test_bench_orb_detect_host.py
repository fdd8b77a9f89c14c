"""tools/bench_orb_detect.py runs its host side without a GPU (the CPU arm) and prints one JSON line; the GPU run prints the
device stages and the key points per image."""
import json
import os
import subprocess
import sys

import pytest

from conftest import ROOT

SCRIPT = os.path.join(ROOT, "tools", "bench_orb_detect.py")


def _run(*extra):
    out = subprocess.run([sys.executable, SCRIPT, *extra], capture_output=True, text=True, check=True, timeout=600).stdout
    lines = [l for l in out.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    return json.loads(lines[0])


@pytest.mark.parametrize("config", ["default", "kitti"])
def test_bench_orb_detect_cpu_arm(config):
    line = _run("--impl", "reference", "--pairs", "2", "--config", config)
    assert line["unit"] == "images/s" and line["value"] > 0
    assert line["cpu_baseline"]["cores"] >= 1 and line["config"]["orb"] == config


@pytest.mark.gpu
def test_bench_orb_detect_gpu_line():
    line = _run("--gpus", "1", "--steps", "2", "--warmup", "1", "--pairs", "4", "--no-cpu")
    assert line["value"] > 0 and line["config"]["keypoints_per_image"] >= 1000
    assert all(v > 0 for v in line["kernel_ms_per_step"].values())
