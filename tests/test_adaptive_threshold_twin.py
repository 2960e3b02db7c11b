"""The adaptive threshold of scan-to-map odometry (dcreg_icp_run_odometry_adaptive) on the CPU: the NumPy twin
(api.adaptive_threshold_*) against a literal per-frame reading of KISS-ICP's AdaptiveThreshold, its error against a
50-digit evaluation, the sample rule at min_motion, poses that are not finite, the radius rule, and
dcreg_b200/csrc/adaptive_threshold.cuh built as host C++ against the twin."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from dcreg_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INIT, MIN_MOTION, MAX_RANGE, CEILING = 2.0, 0.1, 100.0, 2.0


def rot(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    return api.se3_exp(np.concatenate([np.zeros(3), a / np.linalg.norm(a) * angle]))


def pose(rng, angle=None, shift=1.0):
    T = rot(rng.normal(size=3), rng.uniform(0, 3.0) if angle is None else angle)
    T[:3, 3] = rng.normal(size=3) * shift
    return T


def corrections(rng, n):
    """n (T_prior, T_out) pairs: a prior anywhere, the result a small correction of it (some below min_motion)"""
    out = []
    for k in range(n):
        Tp = pose(rng, shift=30.0)
        small = rot(rng.normal(size=3), 10.0 ** rng.uniform(-6, -2.3))
        small[:3, 3] = rng.normal(size=3) * 10.0 ** rng.uniform(-3, -0.3)
        out.append((Tp, Tp @ small))
    return out


class LiteralThreshold:
    """KISS-ICP's AdaptiveThreshold read frame by frame: a model error above min_motion joins the sum of squares; sigma
    is the initial threshold before any sample and the root mean square after; the radius is three sigma"""

    def __init__(self):
        self.sse, self.num = 0.0, 0

    def update(self, T_prior, T_out):
        dev = np.linalg.inv(T_prior) @ T_out
        theta = math.acos(min(1.0, max(-1.0, 0.5 * (np.trace(dev[:3, :3]) - 1.0))))
        err = 2.0 * MAX_RANGE * math.sin(theta / 2.0) + np.linalg.norm(dev[:3, 3])
        if err > MIN_MOTION:
            self.sse += err * err
            self.num += 1

    def sigma(self):
        return INIT if self.num == 0 else math.sqrt(self.sse / self.num)


def test_twin_follows_the_literal_rule():
    rng = np.random.default_rng(5)
    lit, state = LiteralThreshold(), (0.0, 0)
    samples = 0
    for Tp, To in corrections(rng, 300):
        lit.update(Tp, To)
        state = api.adaptive_threshold_update(state, Tp, To, MIN_MOTION, MAX_RANGE)
        assert state[1] == lit.num
        assert state[0] == pytest.approx(lit.sse, rel=1e-6)     # (acos of a trace loses half the digits of a small angle)
        want = min(3.0 * lit.sigma(), 1e9)
        assert api.adaptive_threshold_radius(state, INIT, 1e9) == pytest.approx(want, rel=1e-6)
        samples = lit.num
    assert 50 < samples < 300                                   # both sides of min_motion occurred


@pytest.mark.parametrize("theta", [0.0, 1e-12, 1e-6, 0.1, 1.0, math.pi - 1e-6])
def test_error_against_50_digits(theta):
    import mpmath as mp
    mp.mp.dps = 50
    rng = np.random.default_rng(11)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    # the exact rotation by theta about the axis, rounded to FP64, and a translation: T_prior = I, so D = T_out
    a = [mp.mpf(float(x)) for x in axis]
    nrm = mp.sqrt(sum(x * x for x in a))
    a = [x / nrm for x in a]
    c, s = mp.cos(mp.mpf(theta)), mp.sin(mp.mpf(theta))
    K = [[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]
    T = np.eye(4)
    for i in range(3):
        for j in range(3):
            T[i, j] = float((1 if i == j else 0) * c + s * K[i][j] + (1 - c) * a[i] * a[j])
    T[:3, 3] = [0.3, -0.2, 0.05]
    # reference: the angle of the ROUNDED matrix through its quaternion (Shepperd's well-conditioned branch) in 50 digits
    R = [[mp.mpf(float(T[i, j])) for j in range(3)] for i in range(3)]
    tr = R[0][0] + R[1][1] + R[2][2]
    if tr > 0:
        w = mp.sqrt(tr + 1) / 2
        vx, vy, vz = (R[2][1] - R[1][2]) / (4 * w), (R[0][2] - R[2][0]) / (4 * w), (R[1][0] - R[0][1]) / (4 * w)
    else:
        i = max(range(3), key=lambda d: R[d][d])
        j, k = (i + 1) % 3, (i + 2) % 3
        vi = mp.sqrt(R[i][i] - R[j][j] - R[k][k] + 1) / 2
        w = abs(R[k][j] - R[j][k]) / (4 * vi)
        vx, vy, vz = vi, (R[j][i] + R[i][j]) / (4 * vi), (R[k][i] + R[i][k]) / (4 * vi)
    th = 2 * mp.atan2(mp.sqrt(vx * vx + vy * vy + vz * vz), w)
    t = [mp.mpf(float(x)) for x in T[:3, 3]]
    want = 2 * mp.mpf(MAX_RANGE) * mp.sin(th / 2) + mp.sqrt(sum(x * x for x in t))
    got = api.adaptive_threshold_error(np.eye(4), T, MAX_RANGE)
    # a few FP64 roundings of |v| and w, times the 200 m that turn half the angle into metres
    assert abs(mp.mpf(got) - want) <= mp.mpf(2e-13), (theta, got, float(want))
    if theta == 0.0:
        assert got == math.sqrt((0.3 * 0.3 + (-0.2) * (-0.2)) + 0.05 * 0.05)


def test_sample_rule_at_min_motion():
    """e exactly at min_motion is no sample; one ulp above is, one ulp below is not"""
    T = np.eye(4)
    for e, sample in ((0.25, False), (np.nextafter(0.25, 1.0), True), (np.nextafter(0.25, 0.0), False)):
        T[0, 3] = e                                         # a pure translation along x: e = sqrt(x x) = x exactly
        assert api.adaptive_threshold_error(np.eye(4), T, MAX_RANGE) == e
        sse, n = api.adaptive_threshold_update((1.5, 2), np.eye(4), T, 0.25, MAX_RANGE)
        assert (n == 3) == sample
        assert sse == (1.5 + e * e if sample else 1.5)
    # min_motion = 0: an exact zero correction (an aborted frame returns its prior) is no sample, anything above is
    assert api.adaptive_threshold_update((0.0, 0), T, T, 0.0, MAX_RANGE) == (0.0, 0)


@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf])
def test_poses_that_are_not_finite_leave_the_state(bad):
    rng = np.random.default_rng(3)
    for where in ((0, 0), (1, 2), (2, 3)):
        Tp, To = pose(rng), pose(rng)
        To[where] = bad
        assert math.isnan(api.adaptive_threshold_error(Tp, To, MAX_RANGE))
        assert api.adaptive_threshold_update((2.0, 5), Tp, To, MIN_MOTION, MAX_RANGE) == (2.0, 5)
        assert api.adaptive_threshold_update((2.0, 5), To, Tp, MIN_MOTION, MAX_RANGE) == (2.0, 5)


def test_radius_rule():
    assert api.adaptive_threshold_radius((0.0, 0), 0.1, 2.0) == 3.0 * 0.1           # n = 0: the initial threshold
    assert api.adaptive_threshold_radius((0.0, 0), 2.0, 2.0) == 2.0                 # ... capped at the ceiling
    assert api.adaptive_threshold_radius((123.0, 0), 0.1, 2.0) == 3.0 * 0.1         # (sse is not read while n = 0)
    assert api.adaptive_threshold_radius((0.09, 4), 2.0, 2.0) == 3.0 * math.sqrt(0.09 / 4.0)
    assert api.adaptive_threshold_radius((4.0, 1), 2.0, 2.0) == 2.0
    assert api.adaptive_threshold_radius((4.0, 9), 2.0, 2.0) == 2.0                 # 3 sigma == ceiling exactly
    r = api.adaptive_threshold_radius((1e-30, 1), 2.0, 2.0)
    assert 0.0 < r < 1e-14


def test_chunked_replay_equals_the_straight_one():
    rng = np.random.default_rng(17)
    frames = corrections(rng, 60)
    straight = (0.0, 0)
    for Tp, To in frames:
        straight = api.adaptive_threshold_update(straight, Tp, To, MIN_MOTION, MAX_RANGE)
    for cuts in ([1] * 60, [7, 1, 30, 22], [59, 1]):
        state, at = (0.0, 0), 0
        for c in cuts:
            committed = state                               # a push starts from the committed state ...
            for Tp, To in frames[at:at + c]:
                committed = api.adaptive_threshold_update(committed, Tp, To, MIN_MOTION, MAX_RANGE)
            state, at = committed, at + c                   # ... and commits when it succeeds
        assert state == straight
    assert straight[1] > 10


def test_host_build_matches_the_twin(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if not cxx:
        pytest.skip("no host C++ compiler")
    exe = tmp_path / "test_adaptive_threshold"
    subprocess.run([cxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tools", "test_adaptive_threshold.cpp")],
                   check=True, capture_output=True, text=True)
    rng = np.random.default_rng(29)
    frames = corrections(rng, 400)
    for ang in (0.0, 1e-12, 1e-6, 0.1, 1.0, math.pi - 1e-6, math.pi - 1e-3):      # large corrections too
        Tp = pose(rng)
        frames.append((Tp, api.compose_prior(Tp, pose(rng, ang, 0.2))))
    frames.append((np.eye(4), np.eye(4)))
    bad = pose(rng)
    bad[1, 1] = math.nan
    frames.append((np.eye(4), bad))
    D = np.array([api.constant_velocity_increment(Tp, To) for Tp, To in frames])
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.array([INIT, MIN_MOTION, MAX_RANGE, CEILING]).tobytes() + np.int32(len(D)).tobytes() +
                np.ascontiguousarray(D).tobytes())
    res = subprocess.run([str(exe), str(inp), str(out)], capture_output=True, text=True)
    assert res.returncode == 0 and "ADAPTIVE_HOST_OK" in res.stdout, res.stdout + res.stderr
    host = np.fromfile(out, dtype=np.float64).reshape(-1, 4)
    state = (0.0, 0)
    for k, (Tp, To) in enumerate(frames):
        e = api.adaptive_threshold_error(Tp, To, MAX_RANGE)
        state = api.adaptive_threshold_update(state, Tp, To, MIN_MOTION, MAX_RANGE)
        # the same libm on both sides: the same bits
        assert (math.isnan(e) and math.isnan(host[k, 0])) or host[k, 0] == e, k
        assert host[k, 1] == state[0] and host[k, 2] == state[1], k
        assert host[k, 3] == api.adaptive_threshold_radius(state, INIT, CEILING), k
    assert state[1] > 100
