"""The sparse arena of odometry's local maps and icp_run_pairs' targets (dcreg_set_sparse_maps) on the CPU: its host
twin, built from the same headers as the device build (sparse_index::layout, arena_plan::plan_or_sparse), against a
literal per-cloud build of sparse_index.hpp (tools/test_sparse_arena.cpp)."""
import subprocess

from harness import tool_program


def test_sparse_arena_twin(tmp_path):
    """Random sets of clouds, single points, +-2^19-edge coordinates, clouds whose cells add no extra entries, rows
    whose occupied cells are 8-10 and 17-19 apart: the two-pass order is every cloud's own order shifted, the counts,
    capacities and offsets are the per-cloud builds' back to back, every table slice is the cloud's own table with cs
    shifted; plan_or_sparse goes sparse for cell counts only, and map_failure reports nothing for a sparse step."""
    exe = tool_program(tmp_path, "test_sparse_arena.cpp", "-Wall", "-Wextra", "-Werror")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "SPARSE_ARENA_OK" in res.stdout
