"""Host side of dcreg_set_map_input_voxel: odom_plan.hpp's two point ranges per frame (the points a frame registers
with, and the points it gives the maps), compiled as plain host C++; the setting's C and Python bindings; and the
measurement tool's options."""
import ctypes
import math
import os
import subprocess
import sys

import pytest

from harness import tool_program


def test_map_input_plan(tmp_path):
    """odom_plan::make_push with a frame's map-input offsets: the loop's ranges stay the source's, the window pieces, the
    voxel-map updates, the retained window and the point limit follow the map input; without it (or with the source's
    own offsets) the plan is unchanged, in one call, ragged pushes and one frame per push."""
    exe = tool_program(tmp_path, "test_odom_map_input_plan.cpp")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ODOM_MAP_INPUT_PLAN_OK" in res.stdout


@pytest.fixture(scope="module")
def lib():
    from dcreg_b200 import build, api
    build.build()
    return api.load_library()


def test_setting_is_bound(lib):
    from dcreg_b200 import api
    assert "dcreg_set_map_input_voxel" in api.EXPORTS
    f = lib.dcreg_set_map_input_voxel
    assert f.argtypes == [ctypes.c_void_p, ctypes.c_double]
    assert callable(getattr(api.Context, "set_map_input_voxel"))


@pytest.mark.parametrize("voxel", [0.0, 0.1, math.nan, -1.0, math.inf])
def test_null_context_is_refused(lib, voxel):
    from dcreg_b200 import api
    assert lib.dcreg_set_map_input_voxel(None, voxel) == api.BAD_ARG


def test_measurement_tool_answers_help():
    """tools/measure_odometry_map_input.py, which builds on tools/bench_harness.py, parses its options without a GPU"""
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools",
                        "measure_odometry_map_input.py")
    r = subprocess.run([sys.executable, tool, "--help"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "--runs" in r.stdout and "--dump-outputs" in r.stdout and "--small" in r.stdout
