"""Host side of dcreg_icp_run_pairs (many scan/target pairs, each against its own target): the grid-arena planning of
arena_plan.hpp compiled as plain host C++, and the seeded scan-to-submap pair generator the benchmark and the GPU tests
use."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_arena_plan(tmp_path):
    """arena_plan: per-cloud dims and cell offsets, the +-2^19 cell range, the dense-cell limits per cloud and per call,
    the offset tables, and the arena's grouping of every cloud equal to the cloud grouped alone."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = tmp_path / "test_arena_plan"
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tools", "test_arena_plan.cpp")],
                   check=True, capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "ARENA_PLAN_OK" in res.stdout


@pytest.fixture(scope="module")
def pairs():
    from dcreg_b200.scenes import make_parking_pairs
    return make_parking_pairs(6, n_map=200_000, n_scan=2_000)


def test_parking_pairs_seeded_ragged_dense(pairs):
    from dcreg_b200.scenes import make_parking_pairs
    src, tgt, T_true, T_init = pairs
    again = make_parking_pairs(6, n_map=200_000, n_scan=2_000)
    assert all(np.array_equal(a, b) for a, b in zip(src, again[0]))                      # seeded
    assert all(np.array_equal(a, b) for a, b in zip(tgt, again[1]))
    assert np.array_equal(T_true, again[2]) and np.array_equal(T_init, again[3])
    other = make_parking_pairs(6, seed=54, n_map=200_000, n_scan=2_000)
    assert not np.array_equal(tgt[0], other[1][0])
    assert len(src) == len(tgt) == len(T_true) == len(T_init) == 6
    ns, nt = [len(s) for s in src], [len(t) for t in tgt]
    assert len(set(ns)) > 3 and len(set(nt)) > 3                                          # ragged
    assert all(t.dtype == np.float32 and t.shape[1] == 3 for t in src + tgt)
    assert all(10 * a < b for a, b in zip(ns, nt))                                        # a frame against a submap
    for t in tgt:                                                                          # dense grid at 0.5
        lo, hi = np.floor(t.min(axis=0) / 0.5), np.floor(t.max(axis=0) / 0.5)
        assert np.prod(hi - lo + 1) <= 2 ** 27
        assert np.hypot(t[:, 0], t[:, 1]).max() < 30.05                                   # range-limited, sensor frame
    D = np.linalg.inv(T_true) @ T_init                                                     # the icp_pk01.yaml offsets
    for d in D:
        assert abs(np.linalg.norm(d[:3, 3]) - np.linalg.norm([0.15, 0.12, 0.13])) < 1e-9


def test_parking_pairs_true_pose_aligns(pairs):
    """T_true maps each source onto its own target: the median nearest-neighbour distance is a few mm (a source point
    and its target point are the same map point with independent 5 mm noise: about 11 mm median apart)."""
    from scipy.spatial import cKDTree
    src, tgt, T_true, T_init = pairs
    rng = np.random.default_rng(0)
    for s, t, T, Ti in zip(src, tgt, T_true, T_init):
        p = s[rng.choice(len(s), 300, replace=False)].astype(np.float64)
        tree = cKDTree(t.astype(np.float64))
        d_true = tree.query(p @ T[:3, :3].T + T[:3, 3])[0]
        d_init = tree.query(p @ Ti[:3, :3].T + Ti[:3, 3])[0]
        assert np.median(d_true) < 0.02
        assert np.median(d_init) > 3 * np.median(d_true)
