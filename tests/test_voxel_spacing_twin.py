"""dcreg_b200.api.voxel_downsample with min_spacing, the NumPy twin of dcreg_voxel_downsample_spaced, and
api.voxel_map_update with it: against a literal dict-of-lists reading of KISS-ICP's VoxelHashMap::AddPoints (points
inserted one at a time in order, a voxel taking a point while it holds fewer than max_points and no held point lies
closer than min_spacing), on the CPU.  The device is checked against these twins in tests/test_gpu_voxel_spacing.py."""
import math

import numpy as np
import pytest

from dcreg_b200 import api
from dcreg_b200.api import voxel_downsample
from harness import holes, voxel_lattice


def add_points(voxels, P, voxel, max_points, min_spacing, stamp0=0):
    """AddPoints, literally: voxel -> list of (stamp, float32 point).  Returns the stamps kept, in order."""
    inv = 1.0 / voxel
    s2 = min_spacing * min_spacing
    kept = []
    for i, p in enumerate(np.asarray(P, dtype=np.float32)):
        c = [float(v) for v in p[:3]]
        if not all(math.isfinite(v) for v in c):
            continue
        held = voxels.setdefault(tuple(math.floor(v * inv) for v in c), [])
        if len(held) >= max_points:
            continue
        far = True
        for _, q in held:
            dx, dy, dz = c[0] - float(q[0]), c[1] - float(q[1]), c[2] - float(q[2])
            if (dx * dx + dy * dy) + dz * dz < s2:
                far = False
                break
        if far:
            held.append((stamp0 + i, p[:3].copy()))
            kept.append(stamp0 + i)
    return kept


def insertion_loop(P, voxel, max_points, min_spacing):
    return np.array(add_points({}, P, voxel, max_points, min_spacing), dtype=np.int64)


def check(P, voxel, max_points, min_spacing):
    P = np.asarray(P, dtype=np.float32)
    pts, idx = voxel_downsample(P, voxel, max_points, min_spacing)
    ref = insertion_loop(P, voxel, max_points, min_spacing)
    assert idx.dtype == np.int64 and pts.dtype == np.float32 and pts.shape == (len(idx), 3)
    assert np.array_equal(idx, ref)
    assert pts.tobytes() == np.ascontiguousarray(P[ref, :3]).tobytes()
    return pts, idx


CAPS = [1, 4, 20]


@pytest.mark.parametrize("max_points", CAPS)
@pytest.mark.parametrize("voxel", [0.1, 0.5, 2.0])
def test_random_clouds(voxel, max_points):
    rng = np.random.default_rng(int(voxel * 10) + max_points)
    P = (rng.standard_normal((4000, 3)) * [6.0, 3.0, 1.0]).astype(np.float32)
    for s in (voxel / math.sqrt(max_points), 0.3 * voxel, 0.05 * voxel):
        check(P, voxel, max_points, s)


@pytest.mark.parametrize("max_points", CAPS)
def test_several_clouds_filter_alone(max_points):
    """Clouds do not see each other: each cloud's result is the loop over that cloud alone"""
    rng = np.random.default_rng(5)
    clouds = [rng.uniform(-1, 1, (n, 3)).astype(np.float32) for n in (1, 50, 700, 3000)]
    for P in clouds:
        check(P, 0.5, max_points, 0.5 / math.sqrt(max_points))


@pytest.mark.parametrize("max_points", [2, 4, 20])
def test_pairs_at_the_spacing_and_one_ulp_either_side(max_points):
    """A second point exactly s away along x is kept; one float32 ulp nearer is dropped, one ulp farther kept"""
    s = 0.125                                                               # exact in FP32 and FP64
    base = np.array([0.3, 0.2, 0.1], np.float32)
    x = np.float32(base[0] + np.float32(s))
    assert float(x) - float(base[0]) == s
    for x2, kept in ((x, True), (np.nextafter(x, np.float32(0)), False), (np.nextafter(x, np.float32(1)), True)):
        P = np.array([base, [x2, base[1], base[2]]], np.float32)
        pts, idx = check(P, 1.0, max_points, s)
        assert list(idx) == ([0, 1] if kept else [0])
    # a spacing that is not exact in FP32: the decision follows the FP64 d^2 against s * s
    rng = np.random.default_rng(7)
    for _ in range(200):
        p = rng.uniform(0.1, 0.4, 3).astype(np.float32)
        s = float(rng.uniform(0.01, 0.2))
        q = p.copy()
        q[0] = np.float32(float(p[0]) + s)
        check(np.stack([p, q, np.nextafter(q, np.float32(0)), np.nextafter(q, np.float32(1))]), 1.0, max_points, s)


@pytest.mark.parametrize("max_points", CAPS)
@pytest.mark.parametrize("voxel", [0.25, 0.1])
def test_points_on_voxel_faces(voxel, max_points):
    check(voxel_lattice(voxel), voxel, max_points, voxel / math.sqrt(max_points))
    check(voxel_lattice(voxel), voxel, max_points, 0.5 * voxel)


@pytest.mark.parametrize("max_points", CAPS)
def test_non_finite_rows(max_points):
    pts, idx = check(holes(np.random.default_rng(3), 3000), 0.4, max_points, 0.1)
    assert np.isfinite(pts).all() and not np.isin(idx, np.arange(0, 3000, 7)).any()


@pytest.mark.parametrize("max_points", CAPS)
def test_zero_spacing_is_the_cap_rule(max_points):
    rng = np.random.default_rng(11)
    for P in (rng.standard_normal((3000, 3)).astype(np.float32), voxel_lattice(0.25), holes(rng)):
        pts, idx = voxel_downsample(P, 0.25, max_points, 0.0)
        pts0, idx0 = voxel_downsample(P, 0.25, max_points)
        assert np.array_equal(idx, idx0) and pts.tobytes() == pts0.tobytes()


@pytest.mark.parametrize("max_points", [4, 20, 1 << 30])
def test_spacing_above_twice_the_voxel_is_cap_one(max_points):
    rng = np.random.default_rng(12)
    for voxel in (0.1, 0.5):
        P = np.concatenate([rng.standard_normal((3000, 3)).astype(np.float32), voxel_lattice(voxel), holes(rng)[:, :3]])
        idx1 = voxel_downsample(P, voxel, 1)[1]
        for s in (np.nextafter(2 * voxel, np.inf), 3 * voxel):
            assert np.array_equal(voxel_downsample(P, voxel, max_points, s)[1], idx1)


def test_first_point_of_every_voxel_is_kept():
    rng = np.random.default_rng(13)
    P = rng.standard_normal((5000, 3)).astype(np.float32)
    first = voxel_downsample(P, 0.3, 1)[1]
    for n, s in ((4, 0.15), (20, 0.067), (3, 0.29)):
        assert np.isin(first, voxel_downsample(P, 0.3, n, s)[1]).all()


@pytest.mark.parametrize("max_points", [4, 20])
def test_one_voxel_holding_thousands(max_points):
    rng = np.random.default_rng(14)
    crowd = rng.uniform(0.01, 0.49, (5000, 3)).astype(np.float32)
    background = rng.uniform(-20, 20, (800, 3)).astype(np.float32)
    P = np.concatenate([rng.permutation(np.concatenate([crowd, background])), crowd])
    for s in (0.5 / math.sqrt(max_points), 0.02):
        check(P, 0.5, max_points, s)


@pytest.mark.parametrize("max_points", CAPS)
def test_idempotent_and_prefix_closed(max_points):
    """spaced(spaced(X)) = spaced(X) and spaced(spaced(A) ++ B) = spaced(A ++ B)"""
    rng = np.random.default_rng(15 + max_points)
    A = (rng.standard_normal((3000, 3)) * 2).astype(np.float32)
    B = (rng.standard_normal((2000, 3)) * 2).astype(np.float32)
    for s in (0.5 / math.sqrt(max_points), 0.1):
        once = voxel_downsample(A, 0.5, max_points, s)[0]
        assert voxel_downsample(once, 0.5, max_points, s)[0].tobytes() == once.tobytes()
        whole = voxel_downsample(np.concatenate([A, B]), 0.5, max_points, s)[0]
        assert voxel_downsample(np.concatenate([once, B]), 0.5, max_points, s)[0].tobytes() == whole.tobytes()


@pytest.mark.parametrize("max_points", CAPS)
def test_voxel_map_update_against_add_points_and_prune(max_points):
    """Ten updates of the voxel map with spacing against AddPoints + RemovePointsFarFromLocation on one dict"""
    rng = np.random.default_rng(16 + max_points)
    voxel, max_distance = 0.5, 6.0
    s = voxel / math.sqrt(max_points)
    voxels, stamp = {}, 0
    M = np.zeros((0, 3), np.float32)
    for k in range(10):
        T = np.eye(4)
        T[:3, 3] = [0.7 * k, 0.2 * k, 0.0]
        a = 0.1 * k
        T[:2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
        P = rng.normal(0.0, 3.0, (1500, 3)).astype(np.float32)
        P[rng.integers(0, 1500, 300)] = P[rng.integers(0, 1500, 300)]
        M = api.voxel_map_update(M, P, T, voxel, max_points, max_distance, s)
        add_points(voxels, api.map_points(T, P), voxel, max_points, s, stamp)
        stamp += len(P)
        d2max = max_distance * max_distance
        for key in list(voxels):
            q = voxels[key][0][1]
            dx, dy, dz = (float(q[c]) - float(T[c, 3]) for c in range(3))
            if (dx * dx + dy * dy) + dz * dz >= d2max:
                del voxels[key]
        ref = np.array([p for _, p in sorted((st, tuple(p)) for b in voxels.values() for st, p in b)],
                       np.float32).reshape(-1, 3)
        assert M.tobytes() == ref.tobytes()


def test_bad_spacing():
    P = np.zeros((3, 3), np.float32)
    for bad in (-0.1, -0.0 - 1e-300, np.inf, -np.inf, np.nan):
        with pytest.raises(ValueError):
            voxel_downsample(P, 0.5, 4, bad)
        with pytest.raises(ValueError):
            api.voxel_map_update(P, P, np.eye(4), 0.5, 4, 10.0, bad)
    assert list(voxel_downsample(P, 0.5, 4, 0.0)[1]) == [0, 1, 2]
    assert list(voxel_downsample(P, 0.5, 4, 1e-3)[1]) == [0]
