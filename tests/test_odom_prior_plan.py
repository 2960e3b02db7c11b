"""Host side of the prior map (dcreg_set_prior_map): odom_plan.hpp's plan without anchors or maps, compiled as plain
host C++."""
import os
import subprocess
import sys

from harness import tool_program


def test_odom_prior_plan(tmp_path):
    """odom_plan::make_push with prior = true: step j holds frame j of every sequence, first frames start from T_init
    (prev -1), the history keeps two poses and no points, and any chunking gives one push's references; the window plan
    keeps its anchors."""
    exe = tool_program(tmp_path, "test_odom_prior_plan.cpp")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_PRIOR_PLAN_OK" in res.stdout


def test_measurement_tool_answers_help():
    """tools/measure_odometry_prior_map.py, which builds on tools/bench_harness.py, parses its options without a GPU"""
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools",
                        "measure_odometry_prior_map.py")
    r = subprocess.run([sys.executable, tool, "--help"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "--runs" in r.stdout and "--dump-outputs" in r.stdout and "--workloads" in r.stdout
