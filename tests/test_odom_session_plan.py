"""Host side of the odometry session (dcreg_odometry_push): odom_plan::make_push against one push of the whole
recording onto the empty history, for random recordings pushed in random chunks, compiled as plain host C++."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_odom_session_plan(tmp_path):
    """Sequences of 1 - 40 frames, map_frames 1, 3 and 100, pushes of up to 1, 3 or 12 frames per sequence with empty
    entries: every registered frame's step, previous frames and window pieces name the frames of the one-call plan and
    read their points, the retained window after every push is the last min(map_frames, frames so far) frames, and the
    per-step point limit holds."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = tmp_path / "test_odom_session_plan"
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tools", "test_odom_session_plan.cpp")],
                   check=True, capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_SESSION_PLAN_OK" in res.stdout
