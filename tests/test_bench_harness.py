"""The benchmark tools on a machine without a GPU: every tool answers --help, no tool imports another one (what they
share lives in tools/bench_harness.py), and the harness's pose_errors on a known offset."""
import ast
import glob
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
BENCHMARKS = sorted(p for p in glob.glob(os.path.join(TOOLS, "bench_*.py")) + [os.path.join(TOOLS, "sweep_odometry_voxel.py")]
                    if os.path.basename(p) != "bench_harness.py")


def test_fourteen_benchmarks():
    assert len(BENCHMARKS) == 14


@pytest.mark.parametrize("path", BENCHMARKS, ids=os.path.basename)
def test_help(path):
    r = subprocess.run([sys.executable, path, "--help"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "--runs" in r.stdout and "--dump-outputs" in r.stdout


def test_no_tool_imports_a_benchmark():
    names = {os.path.splitext(os.path.basename(p))[0] for p in BENCHMARKS}
    for path in glob.glob(os.path.join(TOOLS, "*.py")):
        tree = ast.parse(open(path).read(), path)
        imported = set()
        for node in ast.walk(tree):
            if isinstance(node, ast.Import):
                imported.update(a.name.split(".")[0] for a in node.names)
            elif isinstance(node, ast.ImportFrom) and node.module:
                imported.add(node.module.split(".")[0])
        assert not imported & names, (os.path.basename(path), sorted(imported & names))


def test_pose_errors():
    sys.path.insert(0, TOOLS)
    try:
        import bench_harness as h
    finally:
        sys.path.remove(TOOLS)
    from dcreg_b200.scenes import pose6d_to_matrix
    angle = math.radians(2.5)
    T_true = [pose6d_to_matrix(1.0, -2.0, 0.5, 0.1, -0.2, 0.3), pose6d_to_matrix(4.0, 1.0, 0.0, 0.0, 0.0, 1.0)]
    axis = np.array([1.0, 2.0, -2.0]) / 3.0
    K = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    E = np.eye(4)
    E[:3, :3] = np.eye(3) + math.sin(angle) * K + (1.0 - math.cos(angle)) * K @ K
    E[:3, 3] = [0.03, -0.04, 0.12]                             # |t| = 0.13 m
    T = [T_true[0] @ E, T_true[1]]                             # only the first pose is off
    dt, dr = h.pose_errors(T_true, T)
    assert dt == pytest.approx(0.13, rel=1e-12)
    assert dr == pytest.approx(2.5, rel=1e-9)
    assert h.pose_errors(T_true, T_true) == pytest.approx((0.0, 0.0), abs=1e-12)
