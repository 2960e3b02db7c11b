"""dcreg_b200.api.voxel_downsample with max_points, the NumPy twin of dcreg_voxel_downsample_n: against a literal reading
of KISS-ICP's VoxelHashMap::AddPoints (points inserted one at a time in order, a voxel taking a point while it holds
fewer than max_points), on the CPU."""
import math

import numpy as np
import pytest

from dcreg_b200.api import VOXEL_LIMIT, voxel_downsample
from harness import direct, holes, voxel_lattice


def insertion_loop(P, voxel, max_points):
    """The rule read literally: walk the points in order; the voxel of a finite point is floor(float64(c) * (1 / voxel))
    per axis, and a voxel holding fewer than max_points points takes it."""
    inv = 1.0 / voxel
    voxels = {}
    kept = []
    for i, p in enumerate(np.asarray(P, dtype=np.float32)):
        c = [float(np.float64(v)) for v in p[:3]]
        if not all(math.isfinite(v) for v in c):
            continue
        key = tuple(math.floor(v * inv) for v in c)
        assert all(-VOXEL_LIMIT <= k < VOXEL_LIMIT for k in key)
        held = voxels.setdefault(key, [])
        if len(held) < max_points:
            held.append(i)
            kept.append(i)
    return np.array(kept, dtype=np.int64)


def check(P, voxel, max_points):
    P = np.asarray(P, dtype=np.float32)
    pts, idx = voxel_downsample(P, voxel, max_points)
    ref = insertion_loop(P, voxel, max_points)
    assert idx.dtype == np.int64 and pts.dtype == np.float32 and pts.shape == (len(idx), 3)
    assert np.array_equal(idx, ref)
    assert pts.tobytes() == np.ascontiguousarray(P[ref, :3]).tobytes()       # kept rows bit for bit
    return pts, idx


CAPS = [1, 2, 3, 4, 20]


@pytest.mark.parametrize("max_points", CAPS)
@pytest.mark.parametrize("voxel", [0.05, 0.3, 1.0, 7.5])
def test_random_clouds(voxel, max_points):
    rng = np.random.default_rng(int(voxel * 100) + max_points)
    P = (rng.standard_normal((3000, 3)) * [10.0, 5.0, 1.0]).astype(np.float32)
    check(P, voxel, max_points)


@pytest.mark.parametrize("max_points", CAPS)
@pytest.mark.parametrize("voxel", [0.25, 0.1])
def test_lattice_on_voxel_boundaries(voxel, max_points):
    pts, idx = check(voxel_lattice(voxel), voxel, max_points)
    keys = np.floor(pts.astype(np.float64) * (1.0 / voxel))
    _, counts = np.unique(keys, axis=0, return_counts=True)
    assert counts.max() <= max_points and (keys < 0).any()


@pytest.mark.parametrize("max_points", CAPS)
def test_duplicates_and_non_finite_rows(max_points):
    rng = np.random.default_rng(3)
    base = rng.uniform(-4, 4, (200, 3)).astype(np.float32)
    check(np.concatenate([base, base, base[::-1], base]), 0.5, max_points)
    pts, idx = check(holes(rng), 0.4, max_points)
    assert np.isfinite(pts).all() and not np.isin(idx, np.arange(0, 600, 7)).any()


@pytest.mark.parametrize("max_points", [1, 2, 7, 20, 4999, 5000, 5001])
def test_one_voxel_holding_thousands(max_points):
    """5000 points in one voxel among a sparse background: the voxel keeps exactly its first max_points of them"""
    rng = np.random.default_rng(9)
    crowd = rng.uniform(0.01, 0.49, (5000, 3)).astype(np.float32)
    background = rng.uniform(-20, 20, (800, 3)).astype(np.float32)
    P = np.concatenate([rng.permutation(np.concatenate([crowd, background])), crowd])    # crowd interleaved, then again
    pts, idx = check(P, 0.5, max_points)
    in_crowd = (np.floor(pts.astype(np.float64) * 2.0) == 0).all(axis=1)
    assert in_crowd.sum() == min(max_points, (np.floor(P.astype(np.float64) * 2.0) == 0).all(axis=1).sum())


@pytest.mark.parametrize("voxel", [0.05, 0.25, 1.0])
def test_one_point_per_voxel_is_the_first_point_filter(voxel):
    rng = np.random.default_rng(21)
    for P in (rng.standard_normal((2000, 3)).astype(np.float32) * 4, voxel_lattice(voxel), holes(rng)):
        pts, idx = voxel_downsample(P, voxel, 1)
        pts0, idx0 = voxel_downsample(P, voxel)
        assert np.array_equal(idx, direct(P, voxel)) and np.array_equal(idx, idx0)
        assert pts.tobytes() == pts0.tobytes()


def test_kept_sets_nest():
    rng = np.random.default_rng(22)
    P = np.concatenate([(rng.standard_normal((4000, 3)) * 2).astype(np.float32), voxel_lattice(0.25)])
    prev = voxel_downsample(P, 0.25, 1)[1]
    for n in range(2, 12):
        idx = voxel_downsample(P, 0.25, n)[1]
        assert np.isin(prev, idx).all() and len(idx) >= len(prev)
        prev = idx


def test_a_cap_above_every_occupancy_keeps_every_finite_point():
    rng = np.random.default_rng(23)
    P = holes(rng, 3000)
    finite = np.nonzero(np.isfinite(P[:, :3]).all(axis=1))[0]
    keys = np.floor(P[finite, :3].astype(np.float64) * (1.0 / 0.5))
    top = np.unique(keys, axis=0, return_counts=True)[1].max()
    assert top > 1
    for n in (int(top), int(top) + 1, 1 << 30):
        pts, idx = voxel_downsample(P, 0.5, n)
        assert np.array_equal(idx, finite) and pts.tobytes() == np.ascontiguousarray(P[finite, :3]).tobytes()
    assert len(voxel_downsample(P, 0.5, int(top) - 1)[1]) < len(finite)


def test_bad_arguments():
    P = np.zeros((3, 3), np.float32)
    for bad in (0, -1, 2.0, 1.5, True, None, "2", 1 << 31):
        with pytest.raises(ValueError):
            voxel_downsample(P, 0.5, bad)
    assert list(voxel_downsample(P, 0.5, np.int64(2))[1]) == [0, 1]
    for v in (0.0, -1.0, np.inf, np.nan):
        with pytest.raises(ValueError):
            voxel_downsample(P, v, 4)
    with pytest.raises(ValueError):                                          # out of the voxel range, whatever the cap
        voxel_downsample(np.array([[2.0 ** 20, 0.0, 0.0]], np.float32), 1.0, 20)
    with pytest.raises(ValueError):
        voxel_downsample(np.zeros((3, 2), np.float32), 0.5, 2)
