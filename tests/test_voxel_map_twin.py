"""The voxel map's NumPy twins (api.voxel_map_update, api.voxel_map_prune) against a literal reading of KISS-ICP's
VoxelHashMap: a dict of per-voxel point lists, AddPoints keeping at most max_points points per voxel, then
RemovePointsFarFromLocation dropping every voxel whose first point lies max_distance or more from the origin.  CPU only;
the device is checked against these twins in tests/test_gpu_odometry_map.py."""
import math

import numpy as np
import pytest

from dcreg_b200 import api


class HashMap:
    """VoxelHashMap, literally: voxel -> list of (insertion stamp, point), the voxels in no particular order"""

    def __init__(self, voxel, max_points, max_distance):
        self.voxel, self.max_points, self.max_distance = voxel, max_points, max_distance
        self.voxels = {}
        self.stamp = 0

    def key(self, p):
        inv = 1.0 / self.voxel
        return tuple(math.floor(float(c) * inv) for c in p)

    def add_points(self, pts):
        for p in pts:
            self.stamp += 1
            if not np.isfinite(p).all():
                continue
            k = self.key(p)
            block = self.voxels.setdefault(k, [])
            if len(block) < self.max_points:
                block.append((self.stamp, p.copy()))

    def remove_far(self, t):
        d2max = self.max_distance * self.max_distance
        for k in list(self.voxels):
            q = self.voxels[k][0][1]
            dx, dy, dz = float(q[0]) - float(t[0]), float(q[1]) - float(t[1]), float(q[2]) - float(t[2])
            if (dx * dx + dy * dy) + dz * dz >= d2max:
                del self.voxels[k]

    def update(self, P, T):
        self.add_points(api.map_points(T, P))
        self.remove_far(np.asarray(T, dtype=np.float64)[:3, 3])

    def by_age(self):
        pts = sorted((s, tuple(p.view(np.uint32))) for b in self.voxels.values() for s, p in b)
        return np.array([p for _, p in pts], dtype=np.uint32).reshape(-1, 3)

    def lists(self):
        return {k: [tuple(p.view(np.uint32)) for _, p in b] for k, b in self.voxels.items()}


def twin_lists(M, voxel):
    out = {}
    inv = 1.0 / voxel
    for p in M:
        out.setdefault(tuple(math.floor(float(c) * inv) for c in p), []).append(tuple(p.view(np.uint32)))
    return out


def random_pose(rng, origin, yaw_span=math.pi):
    a = rng.uniform(-yaw_span, yaw_span)
    b = rng.uniform(-0.2, 0.2)
    Rz = np.array([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, math.cos(b), -math.sin(b)], [0, math.sin(b), math.cos(b)]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Rx
    T[:3, 3] = origin
    return T


def random_frame(rng, n, spread):
    P = rng.normal(0.0, spread, size=(n, 3)).astype(np.float32)
    P[rng.integers(0, n, size=n // 4)] = P[rng.integers(0, n, size=n // 4)]       # repeated points
    return P


@pytest.mark.parametrize("max_points", [1, 4, 20])
@pytest.mark.parametrize("seed", range(4))
def test_twin_matches_voxel_hash_map(max_points, seed):
    """Random frames at random poses along a path: after every update the twin's map holds the same points per voxel
    as the dict of lists (bit for bit, each voxel's oldest first), its array is in insertion order, and the max_distance
    is small enough that voxels really are pruned."""
    rng = np.random.default_rng(100 + seed)
    voxel, max_distance = 0.5, 6.0
    ref = HashMap(voxel, max_points, max_distance)
    M = np.zeros((0, 3), np.float32)
    pruned = 0
    origin = np.zeros(3)
    for k in range(12):
        origin = origin + rng.uniform(-2.0, 2.0, size=3) * np.array([1.0, 1.0, 0.1])
        T = random_pose(rng, origin)
        P = random_frame(rng, int(rng.integers(1, 400)), 4.0)
        before = len(ref.voxels)
        ref.add_points(api.map_points(T, P))
        added = len(ref.voxels)
        ref.remove_far(T[:3, 3])
        pruned += added - len(ref.voxels)
        assert before <= added
        M = api.voxel_map_update(M, P, T, voxel, max_points, max_distance)
        assert M.dtype == np.float32 and M.shape[1] == 3
        assert twin_lists(M, voxel) == ref.lists()
        np.testing.assert_array_equal(M.view(np.uint32), ref.by_age())
    assert pruned > 0


def test_point_at_exactly_max_distance_is_removed():
    """(3, 4, 0) lies exactly 5 from the origin: max_distance 5 removes its voxel (>=), a hair more keeps it"""
    P = np.array([[3.0, 4.0, 0.0], [0.1, 0.1, 0.1]], np.float32)
    out, idx = api.voxel_map_prune(P, 1.0, 5.0, np.zeros(3))
    np.testing.assert_array_equal(idx, [1])
    out, idx = api.voxel_map_prune(P, 1.0, np.nextafter(5.0, 6.0), np.zeros(3))
    np.testing.assert_array_equal(idx, [0, 1])
    # the whole voxel goes with its first point, even when a later point of it is near
    Q = np.array([[0.9, 0.9, 0.0], [0.1, 0.1, 0.0]], np.float32)
    _, idx = api.voxel_map_prune(Q, 1.0, 1.2, np.zeros(3))
    assert len(idx) == 0


def test_pruned_voxel_is_recreated_at_the_end():
    """A voxel pruned when the sensor moves away comes back when it returns: its new points go after every other"""
    voxel, cap, d = 1.0, 4, 3.0
    T0, T1 = np.eye(4), np.eye(4)
    T1[:3, 3] = [10.0, 0.0, 0.0]
    a = np.array([[0.5, 0.5, 0.5]], np.float32)
    b = np.array([[0.5, 0.5, 0.5]], np.float32)                # at T1: (10.5, 0.5, 0.5)
    M = api.voxel_map_update(np.zeros((0, 3), np.float32), a, T0, voxel, cap, d)
    M = api.voxel_map_update(M, b, T1, voxel, cap, d)          # the voxel of a is now 10 away: gone
    np.testing.assert_array_equal(M, [[10.5, 0.5, 0.5]])
    T2 = np.eye(4)
    T2[:3, 3] = [8.0, 0.0, 0.0]
    c = np.array([[-7.75, 0.25, 0.25], [2.25, 0.25, 0.25]], np.float32)   # (0.25, ...) and (10.25, ...) at T2
    M = api.voxel_map_update(M, c, T2, voxel, cap, 9.0)
    np.testing.assert_array_equal(M, [[10.5, 0.5, 0.5], [0.25, 0.25, 0.25], [10.25, 0.25, 0.25]])


def test_nonfinite_rows_and_negative_voxel_faces():
    """NaN and Inf rows have no voxel and are dropped; points on voxel faces at negative coordinates go to the voxel
    floor(x / voxel) gives, in the twin and in the dict of lists alike"""
    voxel = 0.25
    lat = np.array([[i * voxel, j * voxel, -k * voxel] for i in range(-3, 2) for j in range(-2, 1) for k in range(3)],
                   np.float32)
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]], np.float32)
    P = np.concatenate([bad[:1], lat, bad[1:], lat * 1.0001, lat])
    for cap in (1, 4, 20):
        ref = HashMap(voxel, cap, np.inf)
        ref.update(P, np.eye(4))
        M = api.voxel_map_update(np.zeros((0, 3), np.float32), P, np.eye(4), voxel, cap, np.inf)
        assert np.isfinite(M).all()
        assert twin_lists(M, voxel) == ref.lists()
        np.testing.assert_array_equal(M.view(np.uint32), ref.by_age())
    _, idx = api.voxel_map_prune(P, voxel, 100.0, np.zeros(3))
    assert 0 not in idx and len(lat) + 1 not in idx


@pytest.mark.parametrize("max_points", [1, 4, 20])
def test_cap_of_cap_is_cap(max_points):
    """cap(cap(A) ++ B) = cap(A ++ B) for the smallest-index rule: the identity that makes the map at max_distance = inf
    the window map of every frame so far"""
    rng = np.random.default_rng(max_points)
    for _ in range(5):
        A = np.round(rng.normal(0, 2, size=(500, 3)) * 3).astype(np.float32) / 3
        B = np.round(rng.normal(0, 2, size=(300, 3)) * 3).astype(np.float32) / 3
        A[rng.random(500) < 0.05] = np.nan
        capA, _ = api.voxel_downsample(A, 0.5, max_points)
        left, _ = api.voxel_downsample(np.concatenate([capA, B]), 0.5, max_points)
        right, _ = api.voxel_downsample(np.concatenate([A, B]), 0.5, max_points)
        np.testing.assert_array_equal(left.view(np.uint32), right.view(np.uint32))


def test_infinite_distance_never_prunes():
    """max_distance = inf: every update is the capped filter of everything so far"""
    rng = np.random.default_rng(9)
    M = np.zeros((0, 3), np.float32)
    every = []
    for k in range(6):
        T = random_pose(rng, rng.uniform(-1e4, 1e4, size=3))
        P = random_frame(rng, 200, 50.0)
        every.append(api.map_points(T, P))
        M = api.voxel_map_update(M, P, T, 0.5, 4, np.inf)
        want, _ = api.voxel_downsample(np.concatenate(every), 0.5, 4)
        np.testing.assert_array_equal(M.view(np.uint32), want.view(np.uint32))
    X = np.array([[1e30, -1e30, 3e38]], np.float32)
    _, idx = api.voxel_map_prune(X, 1e33, np.inf, np.zeros(3))
    np.testing.assert_array_equal(idx, [0])


def test_bad_arguments():
    P = np.zeros((2, 3), np.float32)
    for md in (0.0, -1.0, np.nan):
        with pytest.raises(ValueError):
            api.voxel_map_prune(P, 1.0, md, np.zeros(3))
    for v in (0.0, np.inf, np.nan):
        with pytest.raises(ValueError):
            api.voxel_map_prune(P, v, 1.0, np.zeros(3))
    with pytest.raises(ValueError):
        api.voxel_map_prune(np.array([[1e9, 0, 0]], np.float32), 1e-3, 1.0, np.zeros(3))
