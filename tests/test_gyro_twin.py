"""The gyroscope rotation of dcreg_icp_run_odometry_gyro: the NumPy twin (api.gyro_rotation, gyro_knots,
deskew_points_gyro) against closed forms, a 50-digit evaluation, its clipping and bracketing rules and a scene whose gyro
matches its trajectory; and dcreg_b200/csrc/se3.cuh built as host C++ against the twin, bit for bit."""
import subprocess

import mpmath
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from dcreg_b200 import api, scenes
from harness import tool_program


def random_samples(rng, n=60, t0=-0.3, dt=0.01, scale=1.5):
    t = t0 + np.cumsum(rng.uniform(0.2, 1.8, n) * dt)
    return np.concatenate([t[:, None], rng.normal(0.0, scale, (n, 3))], axis=1)


def extrinsic(rng):
    return Rotation.from_rotvec(rng.normal(0.0, 1.0, 3)).as_matrix(), rng.normal(0.0, 0.05, 3)


def test_constant_rate_is_the_closed_form():
    w = np.array([0.3, -1.2, 0.7])
    S = np.concatenate([np.arange(0.0, 1.0, 0.005)[:, None], np.tile(w, (200, 1))], axis=1)
    for a, b in [(0.0, 0.5), (0.0123, 0.9871), (0.2, 0.2), (0.33, 0.3350001)]:
        G = api.gyro_rotation(S, a, b)
        assert np.abs(G - Rotation.from_rotvec(w * (b - a)).as_matrix()).max() < 1e-14


def test_rotation_against_50_digits():
    rng = np.random.default_rng(5)
    R, bias = extrinsic(rng)
    S = random_samples(rng)
    mpmath.mp.dps = 50

    def mexp(phi):
        th = mpmath.sqrt(sum(p * p for p in phi))
        K = mpmath.matrix([[0, -phi[2], phi[1]], [phi[2], 0, -phi[0]], [-phi[1], phi[0], 0]])
        if th == 0:
            return mpmath.eye(3)
        return mpmath.eye(3) + (mpmath.sin(th) / th) * K + ((1 - mpmath.cos(th)) / th ** 2) * (K * K)

    Rm = mpmath.matrix(R.tolist())
    for a, b in [(S[3, 0], S[40, 0]), (S[5, 0] + 1e-3, S[30, 0] - 2e-3), (S[0, 0], S[-1, 0])]:
        M = mpmath.eye(3)
        cur = mpmath.mpf(a)
        j = np.searchsorted(S[:, 0], a, side="right") - 1
        while cur < b:
            nxt = min(mpmath.mpf(S[j + 1, 0]), mpmath.mpf(b))
            w = Rm * mpmath.matrix([mpmath.mpf(S[j, c + 1]) - mpmath.mpf(bias[c]) for c in range(3)])
            M = M * mexp([w[c] * (nxt - cur) for c in range(3)])
            cur, j = nxt, j + 1
        G = api.gyro_rotation(S, a, b, R, bias)
        err = max(abs(float(M[r, c]) - G[r, c]) for r in range(3) for c in range(3))
        assert err < 1e-13, err


def test_clipping_at_arbitrary_ends():
    rng = np.random.default_rng(6)
    R, bias = extrinsic(rng)
    S = random_samples(rng)
    for _ in range(50):
        a, c, b = np.sort(rng.uniform(S[0, 0], S[-1, 0], 3))
        Gac, Gcb, Gab = (api.gyro_rotation(S, x, y, R, bias) for x, y in [(a, c), (c, b), (a, b)])
        assert np.abs(Gac @ Gcb - Gab).max() < 1e-14
        assert np.abs(api.gyro_rotation(S, b, a, R, bias) - Gab.T).max() == 0.0
    with pytest.raises(ValueError):
        api.gyro_rotation(S, S[0, 0] - 1e-9, S[1, 0])
    with pytest.raises(ValueError):
        api.gyro_rotation(S, S[0, 0], S[-1, 0] + 1e-9)


def test_only_the_bracketing_samples_count():
    rng = np.random.default_rng(7)
    S = random_samples(rng)
    i, j = 10, 35
    a, b = S[i, 0] + 1e-3, S[j, 0] - 1e-3
    G = api.gyro_rotation(S, a, b)
    inner = S[i:j + 1]
    assert api.gyro_rotation(inner, a, b).tobytes() == G.tobytes()
    other = S.copy()
    other[:i, 1:] = rng.normal(size=(i, 3))
    other[j + 1:, 1:] = rng.normal(size=(len(S) - j - 1, 3))
    assert api.gyro_rotation(other, a, b).tobytes() == G.tobytes()
    K = api.gyro_knots(S, a, b - a)
    assert api.gyro_knots(inner, a, b - a).tobytes() == K.tobytes()


def test_knots_are_the_walk_from_mid_sweep():
    rng = np.random.default_rng(8)
    R, bias = extrinsic(rng)
    S = random_samples(rng)
    start, span = S[12, 0] - 1e-4, S[30, 0] - S[12, 0]
    tm = start + 0.5 * span
    K = api.gyro_knots(S, start, span, R, bias)
    inside = S[(S[:, 0] > start) & (S[:, 0] < start + span) & (S[:, 0] != tm), 0]
    assert np.array_equal(K[:, 0], np.sort(np.append(inside, tm)))
    for k in K:
        Q = k[1:10].reshape(3, 3)
        if k[0] >= tm:
            assert Q.tobytes() == api.gyro_rotation(S, tm, k[0], R, bias).tobytes()
        else:
            assert np.abs(Q - api.gyro_rotation(S, k[0], tm, R, bias).T).max() < 1e-14


def test_pure_rotation_scene_deskews_to_the_unskewed_frames():
    sk, ts, ft, smp, T, fr = scenes.make_parking_imu(5, pure_rotation=True, n_map=100_000, n_scan=3_000)
    tm = ft[:, 0] + 0.5 * ft[:, 1]
    for k in range(1, 5):
        G = api.gyro_rotation(smp, tm[k - 1], tm[k])
        assert np.abs(G - (np.linalg.inv(T[k - 1]) @ T[k])[:3, :3]).max() < 1e-14
        d = api.deskew_points_gyro(sk[k], ts[k], ft[k], tm[k - 1], smp)
        assert np.abs(sk[k] - fr[k]).max() > 1.0                      # the sweep did skew the frame
        ulp = np.spacing(np.abs(fr[k]).max(axis=1, keepdims=True))
        assert (np.abs(d - fr[k]) <= ulp).all()


def test_scene_rates_carry_bias_noise_and_extrinsic():
    R = Rotation.from_rotvec([0.1, -0.2, 0.3]).as_matrix()
    _, _, ft, exact, _, _ = scenes.make_parking_imu(4, n_map=50_000, n_scan=500)
    _, _, _, moved, _, _ = scenes.make_parking_imu(4, n_map=50_000, n_scan=500, R_sensor_imu=R, bias=(0.01, 0, -0.02))
    assert np.array_equal(moved[:, 0], exact[:, 0])
    assert np.abs((moved[:, 1:] - [0.01, 0, -0.02]) @ R.T - exact[:, 1:]).max() < 1e-15
    tm = ft[:, 0] + 0.5 * ft[:, 1]
    assert np.isin(tm, exact[:, 0]).all()                              # every mid-sweep is a sample time
    assert exact[0, 0] <= ft[0, 0] and exact[-1, 0] >= ft[-1, 0] + ft[-1, 1]


def test_deskew_copies_what_does_not_move():
    rng = np.random.default_rng(9)
    S = random_samples(rng)
    P = rng.uniform(-30, 30, (200, 3)).astype(np.float32)
    P[0] = [np.nan, 1.0, 2.0]
    P[1] = [-0.0, 0.0, -0.0]
    tau = rng.uniform(0, 1, 200).astype(np.float32)
    tau[2] = 0.5
    d = api.deskew_points_gyro(P, tau, (S[10, 0], 0.1), S[10, 0] - 0.05, S)          # a rotation keeps zero at zero
    assert d[:3].tobytes() == P[:3].tobytes()
    assert (d[3:] != P[3:]).any(axis=1).all()


def test_host_build_matches_the_twin(tmp_path):
    exe = tool_program(tmp_path, "test_gyro.cpp", compiler="c++")
    rng = np.random.default_rng(2026)
    R, bias = extrinsic(rng)
    S = random_samples(rng, n=300, scale=3.0)
    S[50:60, 1:] = 1e-6 * rng.normal(size=(10, 3))                    # small angles: the series branch
    lo, hi = S[0, 0], S[-1, 0]
    ab = np.sort(rng.uniform(lo, hi, (200, 2)), axis=1)
    ab[:5] = [[S[3, 0], S[90, 0]], [S[7, 0], S[7, 0]], [lo, hi], [S[51, 0], S[58, 0]], [S[10, 0], S[10, 0] + 1e-9]]
    sweeps = []
    for _ in range(40):
        start = rng.uniform(lo + 0.05, hi - 0.3)
        span = rng.uniform(0.01, 0.2)
        sweeps.append([start, span, start + 0.5 * span - rng.uniform(0.01, 0.05), *rng.normal(0.0, 1.0, 3)])
    sweeps.append([S[100, 0] - 0.05, 0.1, S[100, 0] - 0.1, 0.0, 0.0, 0.0])   # mid-sweep on a sample
    sweeps = np.array(sweeps)
    m = 20_000
    rec = np.zeros(m, dtype=[("w", "<i4"), ("tau", "<f4"), ("p", "<f4", 3)])
    rec["w"] = rng.integers(0, len(sweeps), m)
    rec["tau"] = rng.uniform(0, 1, m).astype(np.float32)
    rec["tau"][:40] = [0.0, 1.0, 0.5, 0.25] * 10
    rec["p"] = rng.uniform(-40, 40, (m, 3)).astype(np.float32)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.concatenate([R.reshape(-1), bias]).tobytes() + np.int32(len(S)).tobytes() + S.tobytes() +
                np.int32(len(ab)).tobytes() + ab.tobytes() + np.int32(len(sweeps)).tobytes() + sweeps.tobytes() +
                np.int32(m).tobytes() + rec.tobytes())
    res = subprocess.run([str(exe), str(inp), str(out)], capture_output=True, text=True)
    assert res.returncode == 0 and "GYRO_HOST_OK" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, dtype=np.uint8)
    G_host = raw[:len(ab) * 72].view(np.float64).reshape(-1, 3, 3)
    at = len(ab) * 72
    count = raw[at:at + 4 * len(sweeps)].view(np.int32)
    at += 4 * len(sweeps)
    K_host = raw[at:at + 128 * int(count.sum())].view(np.float64).reshape(-1, 16)
    pts_host = raw[at + 128 * int(count.sum()):].view(np.float32).reshape(-1, 3)
    G_twin = np.array([api.gyro_rotation(S, a, b, R, bias) for a, b in ab])
    assert G_host.tobytes() == G_twin.tobytes()
    K_twin = np.concatenate([api.gyro_knots(S, s[0], s[1], R, bias) for s in sweeps])
    assert np.array_equal(count, [len(api.gyro_knots(S, s[0], s[1], R, bias)) for s in sweeps])
    assert K_host.tobytes() == K_twin.tobytes()
    twin = np.empty((m, 3), np.float32)
    for w, s in enumerate(sweeps):
        rows = np.nonzero(rec["w"] == w)[0]
        twin[rows] = api.deskew_points_gyro(rec["p"][rows], rec["tau"][rows], s[:2], s[2], S, s[3:], R, bias)
    assert pts_host.tobytes() == twin.tobytes()
