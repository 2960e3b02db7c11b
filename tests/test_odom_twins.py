"""map_points and constant_velocity_increment: the NumPy twins of dcreg_icp_run_odometry's map assembly and its
constant-velocity prior.  Their bits are pinned by the documented order of operations (one rounding each, no FMA),
evaluated here with plain Python floats and an explicit float32 store; the GPU tests check the device against the same
functions."""
import numpy as np

from dcreg_b200.api import compose_prior, constant_velocity_increment, map_points
from dcreg_b200.scenes import pose6d_to_matrix


def poses(n, seed):
    rng = np.random.default_rng(seed)
    return [pose6d_to_matrix(*rng.uniform(-30, 30, 3), *rng.uniform(-np.pi, np.pi, 3)) for _ in range(n)]


def scalar_map(T, P):
    out = np.empty((len(P), 3), dtype=np.float32)
    for i, p in enumerate(P):
        x, y, z = float(p[0]), float(p[1]), float(p[2])
        for r in range(3):
            a = float(T[r][0]) * x
            b = float(T[r][1]) * y
            e = float(T[r][2]) * z
            out[i, r] = np.float32(((a + b) + e) + float(T[r][3]))      # one float32 rounding of the FP64 result
    return out


def scalar_cv(A, B):
    out = [[0.0] * 4 for _ in range(4)]
    dt = [float(B[m][3]) - float(A[m][3]) for m in range(3)]
    for r in range(3):
        for c in range(3):
            out[r][c] = (float(A[0][r]) * float(B[0][c]) + float(A[1][r]) * float(B[1][c])) + float(A[2][r]) * float(B[2][c])
        out[r][3] = (float(A[0][r]) * dt[0] + float(A[1][r]) * dt[1]) + float(A[2][r]) * dt[2]
    out[3][3] = 1.0
    return np.array(out)


def test_map_points_bits_follow_the_documented_order():
    rng = np.random.default_rng(7)
    for T in poses(20, 1):
        P = (rng.standard_normal((64, 3)) * 25).astype(np.float32)
        got = map_points(T, P)
        assert got.dtype == np.float32 and got.shape == (64, 3)
        assert got.tobytes() == scalar_map(T, P).tobytes()
        ref = (P.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        assert np.max(np.abs(got.astype(np.float64) - ref)) < 1e-4                # the transform, up to rounding


def test_map_points_takes_the_first_three_columns():
    P = np.random.default_rng(8).standard_normal((10, 4)).astype(np.float32)
    T = poses(1, 2)[0]
    assert map_points(T, P).tobytes() == map_points(T, P[:, :3]).tobytes()
    assert np.array_equal(map_points(np.eye(4), P), P[:, :3])                   # identity: the points themselves


def test_constant_velocity_increment_bits():
    for A, B in zip(poses(200, 3), poses(200, 4)):
        assert constant_velocity_increment(A, B).tobytes() == scalar_cv(A, B).tobytes()


def test_constant_velocity_increment_is_the_relative_pose():
    for A, B in zip(poses(50, 5), poses(50, 6)):
        D = constant_velocity_increment(A, B)
        assert np.allclose(D, np.linalg.inv(A) @ B, rtol=0, atol=1e-12)
        assert np.allclose(compose_prior(A, D), B, rtol=0, atol=1e-12)            # T_{k-2} D = T_{k-1}
    for A in poses(5, 7):
        assert np.allclose(constant_velocity_increment(A, A), np.eye(4), rtol=0, atol=1e-14)
