"""Host side of dcreg_icp_run_odometry: the step / lane numbering, the local-map windows and the per-step point limit of
odom_plan.hpp, compiled as plain host C++."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_odom_plan(tmp_path):
    """odom_plan::make_push onto the empty history (a one-shot call): frames numbered step by step with the lanes in
    sequence order, every window frame of every lane's map in ascending order with its points contiguous, map offsets,
    previous-frame indices, and the point limit."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = tmp_path / "test_odom_plan"
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tools", "test_odom_plan.cpp")], check=True,
                   capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_PLAN_OK" in res.stdout
