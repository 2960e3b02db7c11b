"""Host side of dcreg_icp_run_scans (a batch of different scans against one map): the ragged tile rule of loop_plan.hpp
compiled as plain host C++, and the seeded C3-shaped frame generator the benchmark and the GPU tests use."""
import subprocess

import numpy as np

from harness import tool_program


def test_scan_tile_plan(tmp_path):
    """loop_plan::plan_scan_tiles: one grid for scans of ragged sizes, sized by the largest; every slot of every scan taken
    by exactly one block, the blocks past a smaller scan's end take none, full tiles, at most 64 blocks per scan."""
    exe = tool_program(tmp_path, "test_scan_plan.cpp")
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "SCAN_PLAN_OK" in res.stdout


def test_parking_frames_seeded_ragged_inside_the_map():
    from dcreg_b200.scenes import make_parking, make_parking_frames
    frames, T_true, T_init, tgt = make_parking_frames(12, n_map=120_000, n_scan=1_500)
    again = make_parking_frames(12, n_map=120_000, n_scan=1_500)
    assert all(np.array_equal(a, b) for a, b in zip(frames, again[0]))                   # seeded
    assert np.array_equal(T_init, again[2]) and np.array_equal(tgt, again[3])
    other = make_parking_frames(12, seed=48, n_map=120_000, n_scan=1_500)
    assert not np.array_equal(frames[0], other[0][0])
    assert np.array_equal(tgt, make_parking(n_map=120_000, seed=43)[1])                 # the make_parking map
    sizes = np.array([len(f) for f in frames])
    assert len(set(sizes.tolist())) > 6 and 1_000 < sizes.min() and sizes.max() < 2_200   # ragged, about n_scan
    lo, hi = tgt.min(axis=0), tgt.max(axis=0)
    for f, T, Ti in zip(frames, T_true, T_init):
        assert f.dtype == np.float32 and f.shape[1] == 3
        pm = f.astype(np.float64) @ T[:3, :3].T + T[:3, 3]                               # back in map coordinates
        assert np.all(pm >= lo - 0.05) and np.all(pm <= hi + 0.05)
        assert np.abs(np.hypot(pm[:, 0] - T[0, 3], pm[:, 1] - T[1, 3])).max() < 30.05     # range-limited
        D = np.linalg.inv(T) @ Ti                                                         # the icp_pk01.yaml offset
        assert abs(np.linalg.norm(D[:3, 3]) - np.linalg.norm([0.15, 0.12, 0.13])) < 1e-9
        ang = np.degrees(np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1)))
        assert 2.0 < ang < 3.0
    steps = np.linalg.norm(np.diff(T_true[:, :3, 3], axis=0), axis=1)
    assert np.all(steps > 0.5)                                                            # frames along a path
