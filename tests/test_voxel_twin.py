"""dcreg_b200.api.voxel_downsample, the NumPy twin of dcreg_voxel_downsample: against a direct per-point reading of the
rule (a dict of the first index per voxel, one point at a time), on the CPU."""
import math

import numpy as np
import pytest

from dcreg_b200.api import VOXEL_LIMIT, voxel_downsample


def direct(P, voxel):
    """The rule read literally: walk the points in order, the voxel of a finite point is floor(float64(c) * (1 / voxel))
    per axis, and the first point to reach a voxel keeps it."""
    inv = 1.0 / voxel
    first = {}
    for i, p in enumerate(np.asarray(P, dtype=np.float32)):
        c = [float(np.float64(v)) for v in p[:3]]
        if not all(math.isfinite(v) for v in c):
            continue
        key = tuple(math.floor(v * inv) for v in c)
        assert all(-VOXEL_LIMIT <= k < VOXEL_LIMIT for k in key)
        first.setdefault(key, i)
    return np.array(sorted(first.values()), dtype=np.int64)


def check(P, voxel):
    P = np.asarray(P, dtype=np.float32)
    pts, idx = voxel_downsample(P, voxel)
    ref = direct(P, voxel)
    assert idx.dtype == np.int64 and pts.dtype == np.float32 and pts.shape == (len(idx), 3)
    assert np.array_equal(idx, ref)
    assert pts.tobytes() == np.ascontiguousarray(P[ref, :3]).tobytes()       # kept rows bit for bit
    return pts, idx


@pytest.mark.parametrize("voxel", [0.05, 0.25, 0.3, 1.0, 7.5])
def test_random_clouds(voxel):
    rng = np.random.default_rng(int(voxel * 100))
    P = (rng.standard_normal((3000, 3)) * [10.0, 5.0, 1.0]).astype(np.float32)
    pts, idx = check(P, voxel)
    assert 0 < len(idx) <= len(P)


@pytest.mark.parametrize("voxel", [0.25, 0.5, 1.0, 0.1])
def test_lattice_on_voxel_boundaries(voxel):
    """Points exactly on voxel faces, on both sides of 0, where floor and truncation differ for negative coordinates;
    0.1 is not a binary fraction, so some products round across a face."""
    g = np.arange(-6, 6, dtype=np.float64) * voxel
    P = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    P = np.concatenate([P, np.nextafter(P, np.float32(-np.inf)), -P])
    pts, idx = check(P, voxel)
    keys = np.floor(pts.astype(np.float64) * (1.0 / voxel))
    assert len(np.unique(keys, axis=0)) == len(keys)
    assert (keys < 0).any()


def test_duplicates_keep_the_first():
    rng = np.random.default_rng(3)
    base = rng.uniform(-4, 4, (200, 3)).astype(np.float32)
    P = np.concatenate([base, base, base[::-1]])
    pts, idx = check(P, 0.5)
    assert idx.max() < 200


def test_non_finite_rows_are_dropped():
    rng = np.random.default_rng(4)
    P = rng.uniform(-3, 3, (500, 4)).astype(np.float32)
    P[::7, 0] = np.nan
    P[3::11, 1] = np.inf
    P[5::13, 2] = -np.inf
    P[::17, 3] = np.nan                                                      # a 4th column does not matter
    pts, idx = check(P, 0.4)
    assert np.isfinite(pts).all()
    assert not np.isin(idx, np.arange(0, 500, 7)).any()
    nan_only = np.full((4, 3), np.nan, np.float32)
    pts, idx = voxel_downsample(nan_only, 1.0)
    assert pts.shape == (0, 3) and idx.shape == (0,)


def test_one_point():
    pts, idx = check(np.array([[-0.5, 2.0, 1e-3]], np.float32), 0.3)
    assert list(idx) == [0]


def test_idempotent():
    rng = np.random.default_rng(5)
    P = rng.uniform(-20, 20, (4000, 3)).astype(np.float32)
    pts, idx = voxel_downsample(P, 0.75)
    again, idx2 = voxel_downsample(pts, 0.75)
    assert again.tobytes() == pts.tobytes() and np.array_equal(idx2, np.arange(len(pts)))


def test_key_range():
    ok = np.array([[-(2.0 ** 20), 0.0, 2.0 ** 20 - 1]], np.float32)
    assert list(voxel_downsample(ok, 1.0)[1]) == [0]
    for bad in ([2.0 ** 20, 0.0, 0.0], [0.0, -(2.0 ** 20) - 1, 0.0], [0.0, 0.0, 3e38]):
        with pytest.raises(ValueError):
            voxel_downsample(np.array([bad], np.float32), 1.0)
    with pytest.raises(ValueError):                                          # a tiny voxel moves ordinary points out
        voxel_downsample(np.array([[1.0, 0.0, 0.0]], np.float32), 1e-7)
    for v in (0.0, -1.0, np.inf, np.nan):
        with pytest.raises(ValueError):
            voxel_downsample(np.zeros((1, 3), np.float32), v)
