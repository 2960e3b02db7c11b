"""The NumPy twin of the odometry's motion compensation (api.se3_log / se3_exp / deskew_points) on the CPU: against a
50-digit mpmath evaluation of the same maps, its exact-copy rules, and the geometry of make_parking_sweeps (a sign or
direction error that device-vs-twin parity cannot catch)."""
import math

import mpmath as mp
import numpy as np
import pytest

from dcreg_b200 import api
from dcreg_b200.scenes import make_parking_sweeps

mp.mp.dps = 50
THETAS = [0.0, 1e-12, 1e-6, 0.1, 1.0, math.pi - 1e-6]


def mp_cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def mp_exp_coeffs(theta):
    if theta == 0:
        return mp.mpf(1), mp.mpf(1) / 2, mp.mpf(1) / 6
    return mp.sin(theta) / theta, (1 - mp.cos(theta)) / theta ** 2, (theta - mp.sin(theta)) / theta ** 3


def mp_exp_apply(xi, s, p):
    """Exp(s xi) p in 50 digits"""
    rho = [s * x for x in xi[:3]]
    phi = [s * x for x in xi[3:]]
    A, B, C = mp_exp_coeffs(mp.sqrt(sum(x * x for x in phi)))
    a = mp_cross(phi, p)
    c = mp_cross(phi, rho)
    b, d = mp_cross(phi, a), mp_cross(phi, c)
    return [p[r] + A * a[r] + B * b[r] + rho[r] + B * c[r] + C * d[r] for r in range(3)]


def mp_exp(xi):
    """Exp(xi) as a 4x4 of mpf"""
    T = [[mp.mpf(int(r == c)) for c in range(4)] for r in range(4)]
    for c in range(3):
        e = [mp.mpf(int(r == c)) for r in range(3)]
        col = mp_exp_apply(xi, 1, e)
        t0 = mp_exp_apply(xi, 1, [mp.mpf(0)] * 3)
        for r in range(3):
            T[r][c] = col[r] - t0[r]
    t0 = mp_exp_apply(xi, 1, [mp.mpf(0)] * 3)
    for r in range(3):
        T[r][3] = t0[r]
    return T


def mp_log(D):
    """Log(D) in 50 digits: the rotation's quaternion (Shepperd, w >= 0), theta = 2 atan2(|v|, w), rho = V^-1 t"""
    R = [[mp.mpf(float(D[r, c])) for c in range(3)] for r in range(3)]
    t = [mp.mpf(float(D[r, 3])) for r in range(3)]
    tr = R[0][0] + R[1][1] + R[2][2]
    v = [mp.mpf(0)] * 3
    if tr > 0:
        r = mp.sqrt(tr + 1)
        w = r / 2
        v = [(R[2][1] - R[1][2]) / (2 * r), (R[0][2] - R[2][0]) / (2 * r), (R[1][0] - R[0][1]) / (2 * r)]
    else:
        i = max(range(3), key=lambda k: (R[k][k], -k))
        j, k = (i + 1) % 3, (i + 2) % 3
        r = mp.sqrt(R[i][i] - R[j][j] - R[k][k] + 1)
        v[i] = r / 2
        w = (R[k][j] - R[j][k]) / (2 * r)
        v[j] = (R[j][i] + R[i][j]) / (2 * r)
        v[k] = (R[k][i] + R[i][k]) / (2 * r)
    if w < 0:
        w, v = -w, [-x for x in v]
    n = mp.sqrt(sum(x * x for x in v))
    f = 2 / w if n == 0 else 2 * mp.atan2(n, w) / n
    phi = [f * x for x in v]
    theta = f * n
    c = mp.mpf(1) / 12 if theta == 0 else (1 - theta * mp.cos(theta / 2) / (2 * mp.sin(theta / 2))) / theta ** 2
    a = mp_cross(phi, t)
    b = mp_cross(phi, a)
    return [t[r] - a[r] / 2 + c * b[r] for r in range(3)] + phi


def motion(theta, seed):
    """A double rigid motion with rotation angle theta about a random axis and a ~1 m translation"""
    rng = np.random.default_rng(seed)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    xi = [mp.mpf(float(x)) for x in rng.uniform(-1, 1, 3)] + [mp.mpf(theta) * mp.mpf(float(a)) for a in axis]
    T = mp_exp(xi)
    return np.array([[float(T[r][c]) for c in range(4)] for r in range(4)])


def within_contract(got, exact):
    """|got - exact| <= max(one float32 ulp of the exact value, 1e-12 m), per coordinate"""
    ex = np.array([float(x) for x in exact])
    ulp = np.spacing(np.abs(ex).astype(np.float32)).astype(np.float64)
    err = np.array([abs(mp.mpf(float(g)) - e) for g, e in zip(got, exact)], dtype=float)
    return bool((err <= np.maximum(ulp, 1e-12)).all()), err, ulp


@pytest.mark.parametrize("theta", THETAS)
def test_log_and_deskew_against_mpmath(theta):
    D = motion(theta, 7)
    xi_mp = mp_log(D)
    xi = api.se3_log(D)
    scale = max(1.0, float(max(abs(x) for x in xi_mp)))
    assert max(abs(float(mp.mpf(float(a)) - b)) for a, b in zip(xi, xi_mp)) <= 8 * np.finfo(float).eps * scale
    rng = np.random.default_rng(11)
    P = rng.uniform(-30, 30, (40, 3)).astype(np.float32)
    tau = np.concatenate([[0.0, 1.0, 0.5 + 2 ** -24], rng.uniform(0, 1, 37)]).astype(np.float32)
    out = api.deskew_points(P, tau, D)
    for i in range(len(P)):
        s = mp.mpf(float(tau[i])) - mp.mpf(0.5)
        exact = mp_exp_apply(xi_mp, s, [mp.mpf(float(x)) for x in P[i]])
        ok, err, ulp = within_contract(out[i], exact)
        assert ok, (theta, i, err, ulp)


@pytest.mark.parametrize("theta", THETAS)
def test_exp_of_log_is_the_motion(theta):
    D = motion(theta, 3)
    assert np.abs(api.se3_exp(api.se3_log(D)) - D).max() <= 1e-14 * max(1.0, np.abs(D).max())
    Tmp = mp_exp(mp_log(D))
    E = api.se3_exp(np.array([float(x) for x in mp_log(D)]))
    assert max(abs(float(Tmp[r][c]) - E[r, c]) for r in range(3) for c in range(4)) <= 1e-15 * 8


def test_log_of_the_identity_is_exactly_zero():
    xi = api.se3_log(np.eye(4))
    assert (xi == 0.0).all()
    assert api.se3_exp(np.zeros(6)).tobytes() == np.eye(4).tobytes()


def test_exact_copy_rules():
    rng = np.random.default_rng(5)
    P = rng.uniform(-20, 20, (12, 3)).astype(np.float32)
    P[0] = [-0.0, 1.0, -0.0]
    P[1, 0] = np.frombuffer(np.uint32(0x7FC01234).tobytes(), np.float32)[0]      # a NaN with a payload
    P[2] = [np.inf, 0.0, 1.0]
    P[3] = [3.4e38, -3.4e38, 3.4e38]                                               # moving it may overflow float32
    tau = rng.uniform(0, 1, 12).astype(np.float32)
    tau[0] = 0.2
    tau[4] = 0.5
    D = motion(0.3, 1)
    out = api.deskew_points(P, tau, D)
    assert out[[1, 2, 4]].tobytes() == P[[1, 2, 4]].tobytes()                     # NaN row, inf row, tau = 0.5
    assert np.isfinite(out[3]).all()                                               # moved, or copied if it overflowed
    assert np.isfinite(out[[0] + list(range(3, 12))]).all()
    assert (out[5:] != P[5:]).any(axis=1).all()                                    # the others moved
    # tau = 0.5 everywhere, the identity, a non-finite increment: the frame comes back bit for bit, -0.0 included
    P[5] = [-0.0, -0.0, 2.0]
    assert api.deskew_points(P, np.full(12, 0.5, np.float32), D).tobytes() == P.tobytes()
    assert api.deskew_points(P, tau, np.eye(4)).tobytes() == P.tobytes()
    Dn = D.copy()
    Dn[0, 3] = np.nan
    assert api.deskew_points(P, tau, Dn).tobytes() == P.tobytes()
    Di = D.copy()
    Di[1, 1] = np.inf
    assert api.deskew_points(P, tau, Di).tobytes() == P.tobytes()


def test_sweep_geometry_has_teeth():
    """On make_parking_sweeps the skewed frame deskewed with the true increment is the unskewed frame to 1e-5 m; the
    inverse increment or the reversed sweep is off by at least 5 cm"""
    skewed, stamps, T_true, deltas, frames = make_parking_sweeps(16, n_map=120_000, n_scan=4_000)
    for k in range(1, 16):
        D = deltas[k - 1]
        assert np.allclose(D, np.linalg.inv(T_true[k - 1]) @ T_true[k])
        assert ((stamps[k] >= 0) & (stamps[k] <= 1)).all()
        good = api.deskew_points(skewed[k], stamps[k], D)
        assert np.abs(good.astype(np.float64) - frames[k]).max() <= 1e-5, k
        for wrong in (api.deskew_points(skewed[k], stamps[k], np.linalg.inv(D)),
                      api.deskew_points(skewed[k], (1.0 - stamps[k]).astype(np.float32), D)):
            assert np.abs(wrong.astype(np.float64) - frames[k]).max() >= 0.05, k
