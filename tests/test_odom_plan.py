"""Host side of dcreg_icp_run_odometry: the step / lane numbering, the local-map windows and the per-step point limit of
odom_plan.hpp, compiled as plain host C++."""
import subprocess

from harness import tool_program


def test_odom_plan(tmp_path):
    """odom_plan::make_push onto the empty history (a one-shot call): frames numbered step by step with the lanes in
    sequence order, every window frame of every lane's map in ascending order with its points contiguous, map offsets,
    previous-frame indices, and the point limit."""
    exe = tool_program(tmp_path, "test_odom_plan.cpp")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_PLAN_OK" in res.stdout
