"""The sparse row index of dcreg_set_target_sparse (sparse_index.hpp) on the CPU: its host twin, built from the same
header as the device build, against a literal reading of cs, of the table's contents and of the range rule the searches
apply (tools/test_sparse_index.cpp)."""
import subprocess

from harness import tool_program


def test_sparse_index_twin(tmp_path):
    """Random clouds with repeated cells, negative and +-2^19-edge coordinates, rows whose occupied cells are 8, 9, 10
    (and 17, 18, 19) apart: every table entry holds the literal cs, the table is exactly the dilation union, the points
    are in the dense order, and every window of width 1..9 around an occupied cell gives exactly its cells' points."""
    exe = tool_program(tmp_path, "test_sparse_index.cpp", "-Wall", "-Wextra", "-Werror")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "SPARSE_INDEX_OK" in res.stdout
