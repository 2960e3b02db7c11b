"""The accelerometer preintegration of dcreg_icp_run_odometry_imu: the NumPy twin (api.imu_preintegrate, imu_increment,
imu_velocity) against closed forms, a 50-digit evaluation of the same first-order rule, its clipping and bracketing
rules, the gyro's rotation, and a scene whose IMU matches its trajectory; and dcreg_b200/csrc/se3.cuh built as host C++
against the twin, bit for bit."""
import subprocess

import mpmath as mp
import numpy as np
from scipy.spatial.transform import Rotation

from dcreg_b200 import api, scenes
from dcreg_oracle_motion_mp import last_sample, mp_so3_exp
from harness import tool_program

GRAV = (0.0, 0.0, -9.80665)


def random_samples(rng, n=60, t0=-0.3, dt=0.01, scale=1.5, accel=9.0):
    t = t0 + np.cumsum(rng.uniform(0.2, 1.8, n) * dt)
    return np.concatenate([t[:, None], rng.normal(0.0, scale, (n, 3)), rng.normal(0.0, accel, (n, 3))], axis=1)


def extrinsic(rng):
    return Rotation.from_rotvec(rng.normal(0.0, 1.0, 3)).as_matrix(), rng.normal(0.0, 0.05, 3), rng.normal(0.0, 0.2, 3)


def mp_imu_preintegrate(S, a, b, R_si, gyro_bias, accel_bias):
    """(G, alpha, beta, gamma) at 50 digits: the same pieces with exact rates, forces, durations and weights"""
    with mp.workdps(50):
        times = [float(r[0]) for r in S]
        Rm = mp.matrix([[mp.mpf(float(R_si[r][c])) for c in range(3)] for r in range(3)])
        M, cur = mp.eye(3), mp.mpf(float(a))
        A, B = cur, mp.mpf(float(b))
        al, be, ga = mp.matrix(3, 1), mp.matrix(3, 1), mp.matrix(3, 1)
        j = last_sample(times, float(a), False)
        while cur < B:
            nxt = min(mp.mpf(times[j + 1]), B)
            d = nxt - cur
            w = Rm * mp.matrix([mp.mpf(float(S[j][c + 1])) - mp.mpf(float(gyro_bias[c])) for c in range(3)])
            f = Rm * mp.matrix([mp.mpf(float(S[j][c + 4])) - mp.mpf(float(accel_bias[c])) for c in range(3)])
            m = (M * f) * d
            al += m
            be += m * ((B - cur) - d / 2)
            ga += m * ((cur - A) + d / 2)
            M = M * mp_so3_exp([w[c] * d for c in range(3)])
            cur, j = nxt, j + 1
        return M, al, be, ga


def test_constant_force_without_rotation_is_the_closed_form():
    """Zero rate and a constant force f: alpha = f dt, beta = gamma = f dt^2 / 2"""
    f = np.array([0.3, -1.2, 9.7])
    S = np.concatenate([np.arange(0.0, 1.0, 0.005)[:, None], np.zeros((200, 3)), np.tile(f, (200, 1))], axis=1)
    for a, b in [(0.0, 0.5), (0.0123, 0.9871), (0.33, 0.3350001)]:
        G, al, be, ga = api.imu_preintegrate(S, a, b)
        dt = b - a
        assert (G == np.eye(3)).all()
        for got, want in ((al, f * dt), (be, f * dt * dt / 2), (ga, f * dt * dt / 2)):
            assert np.abs(got - want).max() <= 1e-13 * max(1.0, np.abs(want).max())


def test_constant_rate_and_body_force_integrate_a_rotating_vector():
    """A constant rate w about z and a constant body force f: alpha -> the integral of Exp(w u) f over [0, dt], to the
    first-order rule's O(h) as the sample interval h shrinks"""
    wz, f, dt = 2.0, np.array([1.0, 0.5, 9.8]), 0.4

    def exact():
        c, s = (np.sin(wz * dt)) / wz, (1 - np.cos(wz * dt)) / wz
        return np.array([c * f[0] - s * f[1], s * f[0] + c * f[1], f[2] * dt])

    errs = []
    for h in (1e-2, 1e-3):
        n = int(round(dt / h)) + 2
        S = np.concatenate([(np.arange(n) * h)[:, None], np.tile([0.0, 0.0, wz], (n, 1)), np.tile(f, (n, 1))], axis=1)
        _, al, _, _ = api.imu_preintegrate(S, 0.0, dt)
        errs.append(np.abs(al - exact()).max())
    assert errs[1] < errs[0] / 8 and errs[1] < 1e-2


def test_against_50_digits():
    rng = np.random.default_rng(7)
    R, bg, ba = extrinsic(rng)
    S = random_samples(rng)
    for a, b in [(S[3, 0], S[40, 0]), (S[5, 0] + 1e-3, S[30, 0] - 2e-3), (S[0, 0], S[-1, 0])]:
        M, al, be, ga = mp_imu_preintegrate(S, a, b, R, bg, ba)
        G, al2, be2, ga2 = api.imu_preintegrate(S, a, b, R, bg, ba)
        assert max(abs(float(M[r, c]) - G[r, c]) for r in range(3) for c in range(3)) < 1e-13
        for x, y in ((al, al2), (be, be2), (ga, ga2)):
            scale = max(1.0, max(abs(float(x[i])) for i in range(3)))
            assert max(abs(float(x[i]) - y[i]) for i in range(3)) < 1e-13 * scale * len(S)


def test_reads_only_the_bracketing_samples_and_splits_compose():
    rng = np.random.default_rng(9)
    R, bg, ba = extrinsic(rng)
    S = random_samples(rng)
    a, b = S[10, 0] + 1e-3, S[30, 0] + 2e-3
    ref = api.imu_preintegrate(S, a, b, R, bg, ba)
    lo = np.searchsorted(S[:, 0], a, side="right") - 1
    hi = np.searchsorted(S[:, 0], b, side="left")
    junk = S.copy()
    junk[:lo, 1:] = np.nan
    junk[hi + 1:, 1:] = np.nan
    got = api.imu_preintegrate(junk, a, b, R, bg, ba)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(ref, got))
    # split at a sample time m: G = G1 G2, alpha = a1 + G1 a2, gamma and beta with the shifted weights
    m = S[20, 0]
    G1, a1, b1, g1 = api.imu_preintegrate(S, a, m, R, bg, ba)
    G2, a2, b2, g2 = api.imu_preintegrate(S, m, b, R, bg, ba)
    G, al, be, ga = ref
    assert np.abs(G1 @ G2 - G).max() < 1e-13
    assert np.abs(a1 + G1 @ a2 - al).max() < 1e-12
    assert np.abs(b1 + a1 * (b - m) + G1 @ b2 - be).max() < 1e-12
    assert np.abs(g1 + G1 @ (g2 + a2 * (m - a)) - ga).max() < 1e-12
    for bad in ((S[0, 0] - 1.0, b), (a, S[-1, 0] + 1.0)):
        try:
            api.imu_preintegrate(S, *bad)
        except ValueError:
            continue
        raise AssertionError("unbracketed interval accepted")


def test_rotation_is_the_gyro_walk_bit_for_bit():
    rng = np.random.default_rng(11)
    R, bg, ba = extrinsic(rng)
    S = random_samples(rng)
    for a, b in [(S[3, 0], S[40, 0]), (S[5, 0] + 1e-3, S[30, 0] - 2e-3), (S[7, 0], S[7, 0])]:
        G = api.imu_preintegrate(S, a, b, R, bg, ba)[0]
        assert G.tobytes() == api.gyro_rotation(S[:, :4], a, b, R, bg).tobytes()


def scene_errors(rate):
    sk, _, ft, smp, T, v, _ = scenes.make_parking_imu_accel(10, rate_hz=rate, n_map=20_000, n_scan=300,
                                                             path_half_length=3.0)
    tm = ft[:, 0] + 0.5 * ft[:, 1]
    et, ev = 0.0, 0.0
    for k in range(1, len(T)):
        D = api.imu_increment(smp, tm[k - 1], tm[k], T[k - 1], v[k - 1], GRAV)
        P = api.compose_prior(T[k - 1], D)
        et = max(et, np.abs(P[:3, 3] - T[k][:3, 3]).max())
        ev = max(ev, np.abs(api.imu_velocity(smp, tm[k - 1], tm[k], T[k - 1], T[k], GRAV) - v[k]).max())
    return et, ev, tm[1] - tm[0]


def test_scene_truth_is_reproduced_to_the_sample_interval():
    """The twin from the true poses and velocities gives T_true[k] and v_k back.  Holding M f over a piece of h seconds
    errs by at most J h per unit time, J the largest rate of change of the world-frame acceleration (the scene's jerk,
    here about 0.05 (2 pi 3.9)^3 m/s^3 from the vertical shake), so over dt: |t| <= J h dt^2 and |v| <= J h dt, with a
    factor 2 for the rotation's own first-order error; and the error falls with h"""
    (t200, v200, dt), (t1k, v1k, _) = scene_errors(200), scene_errors(1000)
    J = 0.05 * (2 * np.pi * 3.9) ** 3 + 0.05 * (2 * np.pi * 3.0) ** 3
    for h, et, ev in ((1 / 200, t200, v200), (1 / 1000, t1k, v1k)):
        assert et <= 2 * J * h * dt * dt, (et, J * h * dt * dt)
        assert ev <= 2 * J * h * dt, (ev, J * h * dt)
    assert t1k * 3 <= t200 and v1k * 3 <= v200


def test_host_build_is_the_twin_bit_for_bit(tmp_path):
    exe = tool_program(tmp_path, "test_imu.cpp", compiler="c++")
    rng = np.random.default_rng(13)
    R, bg, ba = extrinsic(rng)
    S = random_samples(rng, n=80)
    queries = []
    for i in range(30):
        a = rng.uniform(S[1, 0], S[-20, 0])
        b = a + rng.uniform(0.0, S[-2, 0] - a) if i % 5 else float(S[rng.integers(2, 70), 0])
        a, b = min(a, b), max(a, b)
        Rp = Rotation.from_rotvec(rng.normal(0, 1, 3)).as_matrix()
        queries.append([a, b, *Rp.reshape(-1), *rng.normal(0, 5, 3), *rng.normal(0, 3, 3), *rng.normal(0, 5, 3),
                        *GRAV])
    Q = np.array(queries)
    blob = (np.concatenate([R.reshape(-1), bg, ba]).astype(np.float64).tobytes() + np.int32(len(S)).tobytes() +
            S.astype(np.float64).tobytes() + np.int32(len(Q)).tobytes() + Q.tobytes())
    (tmp_path / "in.bin").write_bytes(blob)
    subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
    out = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.float64).reshape(-1, 24)
    for q, o in zip(Q, out):
        a, b = q[0], q[1]
        G, al, be, ga = api.imu_preintegrate(S, a, b, R, bg, ba)
        Tp = np.eye(4); Tp[:3, :3] = q[2:11].reshape(3, 3); Tp[:3, 3] = q[11:14]
        T = np.eye(4); T[:3, 3] = q[17:20]
        tD = api.imu_translation(Tp, q[14:17], q[20:23], be, b - a)
        twin = np.concatenate([G.reshape(-1), al, be, ga, tD])
        assert twin.tobytes() == o[:21].tobytes()
        if b > a:
            v = api.imu_velocity_from(Tp, T, q[20:23], ga, b - a)
            assert v.tobytes() == o[21:].tobytes()
