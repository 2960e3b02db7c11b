"""Host side of the voxel map (dcreg_icp_run_odometry_map, dcreg_odometry_open_map): odom_plan::map_step's layout of
every step's map update, for random recordings run as one call and pushed in random chunks, compiled as plain host
C++."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_odom_map_plan(tmp_path):
    """Sequences of 1 - 30 frames, one call and pushes of up to 1, 3 or 12 frames per sequence with empty entries: every
    lane's map holds exactly its sequence's earlier frames in order, is pruned at the previous frame, comes first in its
    update, and a session's maps after every push hold every frame pushed so far, packed by sequence."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = tmp_path / "test_odom_map_plan"
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tools", "test_odom_map_plan.cpp")],
                   check=True, capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_MAP_PLAN_OK" in res.stdout
