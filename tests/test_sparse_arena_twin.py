"""The sparse arena of odometry's local maps and icp_run_pairs' targets (dcreg_set_sparse_maps) on the CPU: its host
twin, built from the same headers as the device build (sparse_index::layout, arena_plan::plan_or_sparse), against a
literal per-cloud build of sparse_index.hpp (tools/test_sparse_arena.cpp)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sparse_arena_twin(tmp_path):
    """Random sets of clouds, single points, +-2^19-edge coordinates, clouds whose cells add no extra entries, rows
    whose occupied cells are 8-10 and 17-19 apart: the two-pass order is every cloud's own order shifted, the counts,
    capacities and offsets are the per-cloud builds' back to back, every table slice is the cloud's own table with cs
    shifted; plan_or_sparse goes sparse for cell counts only, and map_failure reports nothing for a sparse step."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = tmp_path / "test_sparse_arena"
    subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-o", str(exe),
                    os.path.join(ROOT, "tools", "test_sparse_arena.cpp")], check=True, capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "SPARSE_ARENA_OK" in res.stdout
