"""Host side of the odometry session (dcreg_odometry_push): odom_plan::make_push against one push of the whole
recording onto the empty history, for random recordings pushed in random chunks, compiled as plain host C++."""
import subprocess

from harness import tool_program


def test_odom_session_plan(tmp_path):
    """Sequences of 1 - 40 frames, map_frames 1, 3 and 100, pushes of up to 1, 3 or 12 frames per sequence with empty
    entries: every registered frame's step, previous frames and window pieces name the frames of the one-call plan and
    read their points, the retained window after every push is the last min(map_frames, frames so far) frames, and the
    per-step point limit holds."""
    exe = tool_program(tmp_path, "test_odom_session_plan.cpp")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_SESSION_PLAN_OK" in res.stdout
