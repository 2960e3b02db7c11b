"""The NumPy twin of the odometry's motion compensation (api.se3_log / se3_exp / deskew_points) on the CPU: against a
50-digit mpmath evaluation of the same maps (oracle/dcreg_oracle_motion_mp.py), its exact-copy rules, and the geometry of make_parking_sweeps (a sign or
direction error that device-vs-twin parity cannot catch)."""
import math

import mpmath as mp
import numpy as np
import pytest

from dcreg_b200 import api
from dcreg_b200.scenes import make_parking_sweeps
from dcreg_oracle_motion_mp import mp_exp, mp_exp_apply, mp_log

mp.mp.dps = 50
THETAS = [0.0, 1e-12, 1e-6, 0.1, 1.0, math.pi - 1e-6]


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
