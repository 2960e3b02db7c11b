"""The odometry's motion math on the device (dcreg_b200/csrc/se3.cuh, adaptive_threshold.cuh) record by record, at every
branch edge, against a 50-digit reference, against its host build, and against the bytes of the odometry kernels.

tools/test_motion_device.cu runs the production functions unchanged, built with the library's nvcc flags (sm_90a,
--fmad=true), on designed records written here: one kernel per function family, one thread per record, and the same
records on the host in the same binary.  The reference is oracle/dcreg_oracle_motion_mp.py: the exact value of every
output (mpmath, 50 digits, the inputs taken as the exact values of their FP64 / float32 numbers) and a bound on the
error of any FP64 evaluation of the header's formula there, derived from its operations and the conditioning at that
input (fused multiply-adds, CUDA's 2-ulp sin / cos / atan2 and both sides of a threshold the rounded predicate can
fall on included).

Held, per record:
  * every FP64 output (device and host) within its bound of the exact value; se3_log's bound is at least the twin
    test's 8 eps of the largest entry; deskewed points (deskew_point, deskew_point_gyro) within one float32 ulp of the
    exact value or 1e-12 m (DESIGN.md section 3, "Motion compensation"), and copied bit for bit where their rules copy;
  * device against host: bit for bit where the headers promise one IEEE operation per step and no transcendental runs
    (so3_exp in its series branch and the walks made only of such pieces, the knot times, rates and counts, fold,
    radius, rotation_angle's series branch); elsewhere the largest difference in ulps is printed per family;
  * the records take the branches they are named for: the test replays every predicate the device cannot round
    differently (Shepperd's tr > 0 and index, the sign of w, |phi'| against kSmallAngle in so3_exp) and asserts
    from the exact inputs which side the others are on.
And against production, bit for bit: se3_log + deskew_point of the program reproduce a deskew call's deskewed_xyz,
gyro_rotation + gyro_knots + deskew_point_gyro a gyro call's T_prior rotation and deskewed_xyz, model_error + fold +
radius an adaptive call's search_radius.
"""
import math
import subprocess

import mpmath as mp
import numpy as np
import pytest

import dcreg_oracle_motion_mp as M
from harness import ctx, params, tool_program  # noqa: F401
from odom_harness import CELL, split

EPS = np.finfo(np.float64).eps
F32 = np.float32
TH0 = 1e-3                                              # se3::kSmallAngle
SMALL3 = [np.nextafter(TH0, 0.0), TH0, np.nextafter(TH0, 1.0)]
POINT = np.dtype([("o", "<f4", 3), ("moved", "<i4")])
DESKEW_IN = np.dtype([("xi", "<f8", 6), ("tau", "<f4"), ("p", "<f4", 3)])
GYRO_IN = np.dtype([("tm_prev", "<f8"), ("tD", "<f8", 3), ("sweep", "<i4"), ("tau", "<f4"), ("p", "<f4", 3),
                    ("pad", "<i4")])
FOLD_IN = np.dtype([("sse", "<f8"), ("n", "<i8"), ("e", "<f8"), ("min_motion", "<f8")])
RADIUS_IN = np.dtype([("sse", "<f8"), ("n", "<i8"), ("initial", "<f8"), ("ceiling", "<f8")])
STATE = np.dtype([("sse", "<f8"), ("n", "<i8")])
BIAS = (0.002, -0.001, 0.003)                           # the gyro's bias (its extrinsic R_SI: below)
(LOG, EXP, DESKEW, SO3, SAMPLES, GYRO_ROT, KNOTS, GYRO_DESKEW, ANGLE, MODEL_ERROR, FOLD, RADIUS, CHAIN) = range(1, 14)


# ---- designed inputs ------------------------------------------------------------------------------------------------
def rot(axis, theta):
    """the exact rotation by theta (mp) about axis, rounded to FP64: (3, 3)"""
    a = [mp.mpf(float(x)) for x in axis]
    n = mp.sqrt(sum(x * x for x in a))
    a = [x / n for x in a]
    th = mp.mpf(theta)
    c, s = mp.cos(th), mp.sin(th)
    K = [[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]
    return np.array([[float((c if i == j else 0) + s * K[i][j] + (1 - c) * a[i] * a[j]) for j in range(3)]
                     for i in range(3)])


R_SI = rot((0.3, -0.5, 0.8), 1.1)


def about_x(s, c):
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def log_at_small_angle():
    """Rotations about x whose theta, as se3_log rounds it (the twin: one axis, no sum to contract), is kSmallAngle and
    one ulp either side"""
    from dcreg_b200 import api
    found = {}
    s0, c0 = math.sin(TH0), math.cos(TH0)
    for dc in (0, -1, 1):
        c = c0
        for _ in range(abs(dc)):
            c = np.nextafter(c, 2.0 * dc)
        for k in range(-60, 61):
            s = s0 + k * np.spacing(s0)
            D = np.eye(4)
            D[:3, :3] = about_x(s, c)
            th = abs(api.se3_log(D)[3])
            if th in SMALL3 and th not in found:
                found[th] = D[:3, :3].copy()
        if len(found) == 3:
            break
    assert len(found) == 3, sorted(found)
    return [found[t] for t in SMALL3]


def angle_at_log_small():
    """Rotations about x whose |v|^2, as rotation_angle rounds it, is 1e-10^2 and one ulp either side"""
    thr = M.K_LOG_SMALL2
    want = [np.nextafter(thr, 0.0), thr, np.nextafter(thr, 1.0)]
    found = {}
    s0 = 2.0 * math.sqrt(thr)
    for m in range(12):                                 # fl(v0^2) alone skips values: a small v1^2 fills them
        for k in range(-4, 5):
            s = s0 + k * np.spacing(s0)
            R = about_x(s, 1.0).reshape(-1)
            R[2], R[6] = m * 2e-19, -m * 2e-19
            r = 0.5 / math.sqrt(((R[0] + R[4]) + R[8]) + 1.0)
            v = [(R[7] - R[5]) * r, (R[2] - R[6]) * r, (R[3] - R[1]) * r]
            n2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
            if n2 in want and n2 not in found:
                found[n2] = R.reshape(3, 3)
    assert len(found) == 3, sorted(found)
    return [found[t] for t in want]


SHEPPERD_AXES = [(1.0, 0.2, 0.1), (0.1, 1.0, 0.3), (0.2, 0.1, 1.0)]


def rotations(rng):
    """(name, R) over [0, pi], Shepperd's every index with both signs of w, its ties, pi about x, y, z and diagonals"""
    out = [("identity", np.eye(3))]
    for th in (1e-12, 1e-9, 1.9e-10, 2.1e-10, 1e-6, 5e-4, 2e-3, 0.1, 1.0, 2.0, 2.2, 2.5, 3.0, 3.1, math.pi - 1e-6,
               math.pi - 1e-9):
        out.append((f"theta {th:g}", rot(rng.normal(size=3), th)))
    for i, ax in enumerate(SHEPPERD_AXES):
        for sign in (1.0, -1.0):
            for th in (2.3, 2.9, mp.pi):
                out.append((f"shepperd i={i} sign {sign:+g} theta {float(th):.3g}", rot(np.multiply(sign, ax), th)))
    R = rot((1.0, 1.0, 0.1), 2.8)
    R[1, 1] = R[0, 0]
    out.append(("tie R[4] == R[0]", R))
    R = rot((0.1, 1.0, 1.0), 2.8)
    R[2, 2] = R[1, 1]
    out.append(("tie R[8] == R[4]", R))
    out += [("pi about x", np.diag([1.0, -1.0, -1.0])), ("pi about y", np.diag([-1.0, 1.0, -1.0])),
            ("pi about z", np.diag([-1.0, -1.0, 1.0])), ("pi about (1,1,1)", rot((1, 1, 1), mp.pi)),
            ("pi about (1,-1,0)", rot((1, -1, 0), mp.pi)), ("2.5 about (-1,-1,-1)", rot((-1, -1, -1), 2.5))]
    return out


def log_records():
    rng = np.random.default_rng(1)
    recs = [("identity", np.eye(3), np.zeros(3)), ("translation", np.eye(3), np.array([1.5, -2.0, 0.25]))]
    for name, R in rotations(rng)[1:]:
        recs.append((name, R, rng.uniform(-2.0, 2.0, 3)))
    for R, th in zip(log_at_small_angle(), ("below", "at", "above")):
        recs.append((f"theta {th} kSmallAngle", R, np.array([0.4, -1.1, 2.0])))
    for th in (1.0, 3.0):
        recs.append((f"t 1e6 theta {th}", rot((0.3, 0.4, -0.2), th), np.array([1e6, -7e5, 3e5])))
    bad = [(0, 4, math.nan), (0, 0, -math.inf), (1, 1, math.inf), (1, 2, math.nan)]
    for where, i, v in bad:
        R, t = rot((1, 2, 3), 0.5), np.array([1.0, 2.0, 3.0])
        (R.reshape(-1) if where == 0 else t)[i] = v
        recs.append((f"not finite {'Rt'[where]}[{i}] = {v}", R, t))
    return recs


def exp_records():
    rng = np.random.default_rng(2)
    recs = []
    for ax in range(3):
        for th in SMALL3:
            xi = np.array([0.3, -0.2, 0.1, 0.0, 0.0, 0.0])
            xi[3 + ax] = th
            recs.append((f"theta {th!r} axis {ax}", xi, 1.0, np.array([1.5, -2.0, 3.0])))
    for th in (0.0, 1e-9, 1e-4, 9.99e-4, 1.001e-3, 0.1, 1.0, 3.0, math.pi):
        for s in (-0.5, 0.25, 0.5, 1.0):
            u = rng.normal(size=3)
            xi = np.concatenate([rng.uniform(-2, 2, 3), u / np.linalg.norm(u) * th])
            p = rng.choice([-1.0, 1.0], 3) * 10.0 ** rng.uniform(-3, 4, 3)
            recs.append((f"theta {th:g} s {s}", xi, s, p))
    return recs


def f32_bits(v):
    return np.frombuffer(np.uint32(v).tobytes(), F32)[0]


def deskew_records():
    from dcreg_b200 import api
    rng = np.random.default_rng(3)
    D = np.eye(4)
    D[:3, :3], D[:3, 3] = rot((0.2, -0.4, 1.0), 0.3), [1.2, -0.3, 0.1]
    xi_a = api.se3_log(D)
    D[:3, :3] = rot((0.7, 0.2, -0.3), 2.9)
    xi_b = api.se3_log(D)
    taus = [0.0, 1.0, 0.5, np.nextafter(F32(0.5), F32(0)), np.nextafter(F32(0.5), F32(1)), 0.25, 0.75]
    recs = []
    for name, xi in (("0.3 rad", xi_a), ("2.9 rad", xi_b)):
        for tau in taus + list(rng.uniform(0, 1, 6)):
            for scale in (1e-3, 1.0, 1e2, 1e4):
                recs.append((f"{name} tau {float(tau):.9g} scale {scale:g}", xi, tau,
                             rng.choice([-1.0, 1.0], 3) * scale * rng.uniform(0.5, 1.0, 3)))
    for th in SMALL3:
        for tau in (0.0, 1.0):
            recs.append((f"s theta {th!r} tau {tau}", np.array([0.1, 0.2, -0.3, 2.0 * th, 0.0, 0.0]), tau,
                         np.array([20.0, -30.0, 5.0])))
    p = np.array([3.0, -4.0, 5.0])
    recs += [("xi zero", np.zeros(6), 0.1, p), ("xi NaN", np.array([0.1, 0.0, 0.0, math.nan, 0.0, 0.0]), 0.1, p)]
    for name, q in (("NaN payload", [f32_bits(0x7FC01234), 1.0, 2.0]), ("+inf", [1.0, math.inf, 2.0]),
                    ("-inf", [1.0, 2.0, -math.inf]), ("-0.0", [-0.0, 1.0, -0.0]), ("all -0.0", [-0.0, -0.0, -0.0])):
        recs.append((name, xi_a, 0.1, np.array(q)))
    quarter = np.array([0.0, 0.0, 0.0, 0.0, 0.0, math.pi / 2.0])       # 45 degrees about z at tau = 1
    recs += [("overflow", quarter, 1.0, np.array([3.0e38, 3.0e38, 0.0])),
             ("near 3e38, moved", quarter, 1.0, np.array([3.0e38, 0.0, 1.0]))]
    return recs


# Series-branch rotation vectors whose diagonal term B (phi_r^2 - t2) rounds to a tie of 1 + B (phi_r^2 - t2): the
# unfused sum (so3_exp's SE3_ADD / SE3_MUL) and a fused multiply-add round it to different neighbours, so a contraction
# of that pair shows in the device-host comparison (found by a search over 2e7 random vectors, about one in 3e6)
FMA_TIES = [(2, ["0x1.8ca0933bdcafep-12", "-0x1.bffa01ed19bdap-12", "0x1.25fd0ce1949f7p-11"]),
            (1, ["-0x1.2cbd83c3f512fp-11", "-0x1.72c1073aa19b6p-13", "0x1.3421e38926de8p-13"]),
            (1, ["0x1.79208a721b906p-12", "0x1.432536827e742p-12", "-0x1.3898a9cc0ad85p-12"]),
            (1, ["0x1.243b6773d7160p-16", "0x1.35a7ac269ab40p-16", "-0x1.ab3dc94714772p-12"]),
            (0, ["0x1.6157b73081be4p-12", "0x1.9ea9992d509d0p-15", "-0x1.2fc627cfccc8dp-11"])]


def fused_diagonal_differs(phi, r):
    """whether fl(1 + B x) (one rounding) differs from fl(1 + fl(B x)) for so3_exp's diagonal entry r"""
    from fractions import Fraction
    t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2]
    B = 0.5 - (t2 / 24.0) * (1.0 - t2 / 30.0)
    x = phi[r] * phi[r] - t2
    return float(1 + Fraction(B) * Fraction(x)) != 1.0 + B * x


def so3_records():
    rng = np.random.default_rng(4)
    recs = [("zero", np.zeros(3))]
    recs += [(f"fused diagonal {r} rounds differently", np.array([float.fromhex(h) for h in phi])) for r, phi in FMA_TIES]
    for ax in range(3):
        for th in SMALL3:
            phi = np.zeros(3)
            phi[ax] = -th if ax == 1 else th
            recs.append((f"theta {th!r} axis {ax}", phi))
    for th in (1e-8, 1e-4, 9e-4, 1.1e-3, 0.5, 2.0, 3.1, math.pi):
        for _ in range(3):
            u = rng.normal(size=3)
            recs.append((f"theta {th:g}", u / np.linalg.norm(u) * th))
    return recs


# the gyro: 64 samples 1/64 s apart (exact binary times), rates per segment: series pieces (1e-3 rad/s), moderate
# (2 rad/s), up to ~pi per piece (200 rad/s), and 0.5 rad/s
def gyro_samples():
    rng = np.random.default_rng(5)
    t = (np.arange(64) - 4) / 64.0
    w = np.empty((64, 3))
    w[:16] = rng.normal(0.0, 1e-3, (16, 3))
    w[16:32] = rng.normal(0.0, 2.0, (16, 3))
    u = rng.normal(size=(16, 3))
    w[32:48] = u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(100.0, 200.0, (16, 1))
    w[36] *= 199.0 / np.linalg.norm(w[36])              # 3.11 rad over its 1/64 s
    w[48:] = rng.normal(0.0, 0.5, (16, 3))
    return np.concatenate([t[:, None], w], axis=1)


def gyro_queries(S):
    T = S[:, 0]
    return [("a = b", T[3], T[3]), ("series, both on samples", T[2], T[10]), ("a off", T[2] + 1 / 256, T[10]),
            ("b off", T[2], T[10] - 1 / 300), ("moderate", T[18], T[30]), ("up to pi per piece", T[33], T[40]),
            ("across every segment", T[5] + 0.001, T[60] - 0.002), ("everything", T[0], T[-1]),
            ("one piece of pi", T[36], T[37])]


def gyro_sweeps(S):
    T = S[:, 0]
    return [("tm on a sample, series", T[6], 1 / 16), ("tm on a sample, moderate", T[20], 4 / 64),
            ("tm on a sample, large", T[36], 4 / 64), ("off samples, series", T[4] + 1 / 1000, 0.1),
            ("off samples, moderate", T[17] + 0.2 / 64, 0.12), ("off samples, large", T[35] + 1 / 512, 0.07),
            ("large into slow", T[44] + 1 / 256, 0.1), ("start and end on samples", T[50], 5 / 64)]


def gyro_points(S, sweeps):
    """GYRO_IN records: tau 0, 1, 0.5 (t = tm: copied), 0.25 and 0.75 (on a knot before and after tm where the sweep
    is 4 samples long), random; coordinates from 1e-3 to 1e4 m; a NaN point; the origin with tD = 0 (a rotation
    keeps it: the equal-result copy)"""
    rng = np.random.default_rng(6)
    recs = []
    for w, (name, start, span) in enumerate(sweeps):
        tm = start + 0.5 * span
        for tau in [0.0, 1.0, 0.5, 0.25, 0.75] + list(rng.uniform(0, 1, 10)):
            for scale in (1e-3, 1.0, 1e2, 1e4):
                r = np.zeros(1, GYRO_IN)
                r["tm_prev"], r["tD"], r["sweep"], r["tau"] = tm - 0.1, rng.normal(0.0, 1.0, 3), w, tau
                r["p"] = rng.choice([-1.0, 1.0], 3) * scale * rng.uniform(0.5, 1.0, 3)
                recs.append(r)
        for p, tD in (([math.nan, 1.0, 2.0], [0.1, 0.2, 0.3]), ([0.0, 0.0, 0.0], [0.0, 0.0, 0.0])):
            r = np.zeros(1, GYRO_IN)
            r["tm_prev"], r["tD"], r["sweep"], r["tau"], r["p"] = tm - 0.1, tD, w, 0.3, p
            recs.append(r)
    return np.concatenate(recs)


def angle_records():
    rng = np.random.default_rng(7)
    recs = rotations(rng)
    for R, side in zip(angle_at_log_small(), ("below", "at", "above")):
        recs.append((f"|v|^2 {side} 1e-20", R))
    bad = rot((1, 2, 3), 0.5)
    bad[1, 1] = math.nan
    return recs + [("NaN", bad)]


def model_error_records():
    rng = np.random.default_rng(8)
    recs = []
    for th in list(np.linspace(0.0, math.pi, 13)) + [1e-12, 2e-10, 2.5]:
        for rng_max in (1.0, 100.0, 1000.0):
            D = np.eye(4)
            D[:3, :3] = rot(rng.normal(size=3), th) if th else np.eye(3)
            D[:3, 3] = rng.normal(0.0, 0.3, 3)
            recs.append((f"theta {th:.4g} max_range {rng_max:g}", D, rng_max))
    D = np.eye(4)
    D[2, 3] = math.inf
    return recs + [("inf t", D, 100.0)]


def fold_records():
    mm = 0.25
    es = [mm, np.nextafter(mm, 1.0), np.nextafter(mm, 0.0), math.nan, math.inf, -math.inf, 0.0, 3.7, 1e-300, 1e150]
    r = np.zeros(len(es) + 2, FOLD_IN)
    r["sse"], r["n"], r["min_motion"] = 1.5, 2, mm
    r["e"][:len(es)] = es
    r[len(es)] = (0.0, 0, 0.0, 0.0)                      # min_motion 0: an exact zero is no sample
    r[len(es) + 1] = (0.0, 0, 1e-300, 0.0)
    return r


def radius_records():
    rows = [(0.0, 0, 0.1, 2.0), (0.0, 0, 2.0, 2.0), (123.0, 0, 0.1, 2.0), (0.09, 4, 2.0, 2.0), (4.0, 1, 2.0, 2.0),
            (4.0, 9, 2.0, 2.0), (1e-30, 1, 2.0, 2.0), (7.3, 11, 0.5, 1.25), (2.0, 3, 0.5, 1e9)]
    return np.array(rows, RADIUS_IN)


# ---- running the program --------------------------------------------------------------------------------------------
class Program:
    """Sections for tools/test_motion_device.cu and the layout of what it writes"""

    def __init__(self):
        self.blob, self.outs = [], []

    def add(self, fam, n, payload, *outs):
        """outs: (dtype, count) of every output array of the section"""
        self.blob.append(np.array([fam, n], np.int32).tobytes() + payload)
        self.outs += list(outs)

    def run(self, exe, tmp):
        inp, out = tmp / "motion_in.bin", tmp / "motion_out.bin"
        inp.write_bytes(b"".join(self.blob))
        res = subprocess.run([str(exe), str(inp), str(out)], capture_output=True, text=True)
        assert res.returncode == 0 and "MOTION_DEVICE_OK" in res.stdout, res.stdout + res.stderr
        raw, at, got = out.read_bytes(), 0, []
        for dt, n in self.outs:
            dt = np.dtype(dt)
            pair = []
            for _ in range(2):
                pair.append(np.frombuffer(raw, dt, n, at).copy())
                at += dt.itemsize * n
            got.append(tuple(pair))
        assert at == len(raw)
        return got


def f8(a):
    return np.ascontiguousarray(a, np.float64).tobytes()


def ulps(a, b):
    """largest |a - b| in ulps of the larger magnitude, NaN = NaN"""
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    both = np.isnan(a) & np.isnan(b)
    with np.errstate(invalid="ignore"):
        d = np.where(both | (a == b), 0.0, np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b))))
    return float(d.max()) if len(d) else 0.0


def same_bits(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


class Tally:
    """worst |got - exact| / bound over a family.  The bounds are the reference's a-priori ones: tens of eps of the
    largest entry for se3_log's xi, more just above kSmallAngle, where c = (1 - theta cos(theta/2) / (2 sin(theta/2)))
    / theta^2 and C = (theta - sin(theta)) / theta^3 cancel to about theta^2 of their terms and keep ~eps / theta^2 of
    relative error (their products with phi x (phi x t) stay near eps of the result, and the bound says so)"""

    def __init__(self):
        self.worst, self.count = 0.0, 0

    def check(self, got, ref, what, floor=0.0):
        """every got (floats) within max(bound, floor) of its exact value (ref: X list)"""
        for g, x in zip(np.asarray(got, np.float64).ravel(), ref):
            bound = max(float(x.e), floor)
            err = float(abs(mp.mpf(float(g)) - x.v))
            assert math.isfinite(bound) and err <= bound, (what, float(g), float(x.v), err, bound)
            self.worst = max(self.worst, err / bound if bound else 0.0)
        self.count += 1


# ---- the checks against the reference (device, host or twin outputs alike) -------------------------------------------
def check_log(recs, xi, tally, branches):
    for (name, R, t), x in zip(recs, xi):
        ref, br = M.log(R.reshape(-1), t)
        if ref is None:
            assert np.isnan(x).all(), name
            branches.add("not finite")
            continue
        if name == "identity":
            assert (x == 0.0).all(), name
        scale = max(1.0, max(abs(float(v.v)) for v in ref))
        tally.check(x, ref, name, floor=8 * EPS * scale)
        branches.add("tr > 0" if br["pos"] else f"tr <= 0, i = {br['i']}" + (", w < 0" if br["flip"] else ""))
        branches.update({f"log {br['log_small']}", f"theta {br['small']}"})


def check_exp(recs, q, tally, branches):
    for (name, xi, s, p), got in zip(recs, q):
        ref, br = M.exp_apply(xi, s, p)
        tally.check(got, ref, name)
        branches.add(br)


def deskew_expect(xi, tau, p):
    kind, q = M.deskew_expected(xi, tau, p)
    assert kind is not None, (xi, tau, p)
    return kind, q


def check_deskew(recs, pts, tally):
    kinds = set()
    for (name, xi, tau, p), got in zip(recs, pts):
        p32 = np.asarray(p, F32)
        kind, q = deskew_expect(xi, F32(tau), p32)
        kinds.add(kind)
        if kind in ("copy", "overflow"):
            assert got["moved"] == 0 and same_bits(got["o"], p32), (name, got, p32)
        else:
            assert got["moved"] == 1, name
            ok, worst = M.within_contract(got["o"], [x.v for x in q])
            assert ok, (name, got["o"], [float(x.v) for x in q])
            tally.worst = max(tally.worst, worst)
        tally.count += 1
    return kinds


def so3_branch_fp64(phi):
    """so3_exp's theta < kSmallAngle as the device rounds it (SE3_MUL / SE3_ADD, IEEE sqrt: no other rounding)"""
    t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2]
    return "series" if math.sqrt(t2) < TH0 else "closed"


def check_so3(recs, R, tally, branches):
    for (name, phi), got in zip(recs, R):
        ref, br = M.so3_exp(phi)
        tally.check(got, ref, name)
        assert br == so3_branch_fp64([float(x) for x in phi]) or br == "either", name
        branches.add(so3_branch_fp64([float(x) for x in phi]))


def check_gyro_rot(S, queries, G, tally):
    walks = []
    for (name, a, b), got in zip(queries, G):
        ref, brs = M.gyro_rotation(S, a, b, R_SI, BIAS)
        tally.check(got, ref, name)
        walks.append(brs)
    return walks


def check_knots(S, sweeps, cnt, K, tally):
    """counts and times exactly, rates exactly (gyro_rate is one IEEE operation per step), Q within its bound"""
    from dcreg_b200 import api
    at = 0
    for w, (name, start, span) in enumerate(sweeps):
        tm, end = start + 0.5 * span, start + span
        ref, before = M.gyro_knots(S, start, tm, end, R_SI, BIAS)
        twin = api.gyro_knots(S, start, span, R_SI, BIAS)
        assert list(cnt[w]) == [len(ref), before], name
        k = K[at:at + len(ref)]
        assert same_bits(k[:, 0], twin[:, 0]) and same_bits(k[:, 10:], twin[:, 10:]), name
        for row, (t, Q, wa, wb) in zip(k, ref):
            assert row[0] == t
            tally.check(row[1:10], Q, name)
        at += len(ref)
    assert at == len(K)


def check_gyro_points(S, sweeps, recs, pts, tally):
    knots = {}
    kinds = set()
    for r, got in zip(recs, pts):
        name, start, span = sweeps[r["sweep"]]
        tm, end = start + 0.5 * span, start + span
        if r["sweep"] not in knots:
            knots[r["sweep"]] = M.gyro_knots(S, start, tm, end, R_SI, BIAS)[0]
        t = M.point_time(start, r["tau"], span)
        p = r["p"]
        if t == tm or not np.isfinite(p).all():
            kinds.add("copy")
            assert got["moved"] == 0 and same_bits(got["o"], p), (name, r)
            continue
        q, br = M.gyro_point(knots[r["sweep"]], t, tm, r["tm_prev"], r["tD"], p)
        kinds.add("on a knot" if t in [k[0] for k in knots[r["sweep"]]] else "between knots")
        ok, worst = M.within_contract(got["o"], [x.v for x in q])
        assert ok, (name, r, got, [float(x.v) for x in q])
        tally.worst = max(tally.worst, worst)
        if same_bits(np.array([float(x.v) for x in q], F32), p):
            kinds.add("equal result")
            assert got["moved"] == 0
        else:
            assert got["moved"] == 1, (name, r)
        tally.count += 1
    return kinds


def angle_branch_fp64(R):
    """rotation_angle's |v|^2 < 1e-20 as the device rounds it (ADT_MUL / ADT_ADD and Shepperd's IEEE steps)"""
    from dcreg_b200 import api
    th = api._rotation_angle(list(R))                   # the same steps: the twin's n2 is the device's
    R = [float(x) for x in R]
    pos, i, _ = M.shepperd(R)
    if pos:
        r = math.sqrt(((R[0] + R[4]) + R[8]) + 1.0)
        r = 0.5 / r
        v = [(R[7] - R[5]) * r, (R[2] - R[6]) * r, (R[3] - R[1]) * r]
    else:
        j, k = (i + 1) % 3, (i + 2) % 3
        r = math.sqrt(((R[4 * i] - R[4 * j]) - R[4 * k]) + 1.0)
        v = [0.0] * 3
        v[i] = 0.5 * r
        r = 0.5 / r
        v[j] = (R[3 * j + i] + R[3 * i + j]) * r
        v[k] = (R[3 * k + i] + R[3 * i + k]) * r
    n2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
    return ("series" if n2 < M.K_LOG_SMALL2 else "closed"), th


def check_angle(recs, th, tally, branches):
    for (name, R), got in zip(recs, th):
        ref, br = M.rotation_angle(R.reshape(-1))
        if ref is None:
            assert math.isnan(got), name
            continue
        tally.check([got], [ref], name)
        branches.add(angle_branch_fp64(R.reshape(-1))[0])


def check_model_error(recs, e, tally):
    for (name, D, mr), got in zip(recs, e):
        ref = M.model_error(D.reshape(-1), mr)
        if ref is None:                                 # NaN, or +inf from an infinite t_D: fold takes neither
            assert not math.isfinite(got), name
            continue
        tally.check([got], [ref], name)


def fold_expected(r):
    e = float(r["e"])
    if math.isfinite(e) and e > float(r["min_motion"]):
        return (float(r["sse"]) + e * e, int(r["n"]) + 1)
    return (float(r["sse"]), int(r["n"]))


def check_fold(recs, got):
    want = np.array([fold_expected(r) for r in recs], STATE)
    assert same_bits(got, want)
    mm = recs["min_motion"]
    assert (got["n"][recs["e"] == mm] == recs["n"][recs["e"] == mm]).all()          # e == min_motion: no sample
    above = recs["e"] == np.nextafter(0.25, 1.0)
    assert (got["n"][above] == recs["n"][above] + 1).all()


def check_radius(recs, got):
    from dcreg_b200 import api
    want = [api.adaptive_threshold_radius((float(r["sse"]), int(r["n"])), float(r["initial"]), float(r["ceiling"]))
            for r in recs]
    assert same_bits(got, np.array(want))
    assert got[5] == 2.0 and 3.0 * math.sqrt(4.0 / 9.0) == 2.0                       # 3 sigma == the ceiling


# ---- the reference against the twin (CPU) ---------------------------------------------------------------------------
def twin_deskew(xi, tau, p):
    """se3::deskew_point through the twin's se3_exp_apply and the header's copy rules"""
    from dcreg_b200 import api
    s = float(F32(tau)) - 0.5
    p = np.asarray(p, F32)
    if s == 0.0 or (np.asarray(xi) == 0).all() or not np.isfinite(xi).all() or not np.isfinite(p).all():
        return p, 0
    with np.errstate(over="ignore"):
        q = api.se3_exp_apply(np.asarray(xi, np.float64), [s], p[None].astype(np.float64))[0].astype(F32)
    return (q, 1) if np.isfinite(q).all() else (p, 0)


def test_reference_agrees_with_the_twin():
    """The 50-digit module holds the NumPy twin (the host build's formulas) to the same bounds it holds the device
    to, on every designed record: the reference is checked before any device output is"""
    from dcreg_b200 import api
    t, br = Tally(), set()
    recs = log_records()
    D = [np.vstack([np.column_stack([R, tt]), [0, 0, 0, 1]]) for _, R, tt in recs]
    check_log(recs, [api.se3_log(d) for d in D], t, br)
    recs = exp_records()
    check_exp(recs, [api.se3_exp_apply(xi, [s], np.asarray(p)[None])[0] for _, xi, s, p in recs], t, br)
    recs = deskew_records()
    pts = np.zeros(len(recs), POINT)
    for i, (_, xi, tau, p) in enumerate(recs):
        pts[i]["o"], pts[i]["moved"] = twin_deskew(xi, tau, p)
    assert check_deskew(recs, pts, Tally()) == {"copy", "move", "overflow"}
    recs = so3_records()
    check_so3(recs, [api._so3_exp([float(x) for x in phi]) for _, phi in recs], t, br)
    S = gyro_samples()
    q = gyro_queries(S)
    check_gyro_rot(S, q, [api.gyro_rotation(S, a, b, R_SI, BIAS) for _, a, b in q], t)
    sw = gyro_sweeps(S)
    K = [api.gyro_knots(S, s, sp, R_SI, BIAS) for _, s, sp in sw]
    cnt = [[len(k), int((k[:, 0] < s + 0.5 * sp).sum())] for k, (_, s, sp) in zip(K, sw)]
    check_knots(S, sw, np.array(cnt), np.concatenate(K), t)
    recs = gyro_points(S, sw)
    pts = np.zeros(len(recs), POINT)
    for i, r in enumerate(recs):
        _, s, sp = sw[r["sweep"]]
        pts[i]["o"] = api.deskew_points_gyro(r["p"][None], [r["tau"]], (s, sp), r["tm_prev"], S, r["tD"], R_SI, BIAS)[0]
        pts[i]["moved"] = int(not same_bits(pts[i]["o"], r["p"]))
    check_gyro_points(S, sw, recs, pts, Tally())
    recs = angle_records()
    check_angle(recs, [api._rotation_angle(list(R.reshape(-1))) for _, R in recs], t, br)
    recs = model_error_records()
    check_model_error(recs, [api.adaptive_threshold_error(np.eye(4), D, mr) for _, D, mr in recs], t)
    fr = fold_records()
    check_fold(fr, np.array([fold_expected(r) for r in fr], STATE))
    print(f"\nreference vs twin: {t.count} records, worst error {t.worst:.3g} of its bound")


def test_records_take_their_branches():
    """Every branch the families are named for is taken by some record, decided from the exact inputs"""
    log_br = set()
    for name, R, t in log_records():
        ref, br = M.log(R.reshape(-1), t)
        if ref is None:
            continue
        log_br.add("tr > 0" if br["pos"] else f"tr <= 0, i = {br['i']}")
        log_br.add(f"w < 0 {br['flip']}")
        log_br.update({f"log {br['log_small']}", f"theta {br['small']}"})
        if name.startswith("tie"):
            assert not br["pos"] and br["i"] == {"tie R[4] == R[0]": 0, "tie R[8] == R[4]": 1}[name], name
    assert {"tr > 0", "tr <= 0, i = 0", "tr <= 0, i = 1", "tr <= 0, i = 2", "w < 0 True", "w < 0 False",
            "log series", "log closed", "theta series", "theta closed", "theta either"} <= log_br, log_br
    exp_br = {M.exp_apply(xi, s, p)[1] for _, xi, s, p in exp_records()}
    assert {"series", "closed", "either"} <= exp_br, exp_br
    for r, phi in FMA_TIES:
        assert fused_diagonal_differs([float.fromhex(h) for h in phi], r)
    so3 = [(so3_branch_fp64(list(phi)), phi) for _, phi in so3_records()]
    assert {b for b, _ in so3} == {"series", "closed"}
    for ax in range(3):                                  # one ulp below kSmallAngle: series; at it and above: closed
        got = [b for b, phi in so3 if np.count_nonzero(phi) == 1 and abs(phi[ax]) in SMALL3]
        assert got == ["series", "closed", "closed"], (ax, got)
    ang = {angle_branch_fp64(R.reshape(-1))[0] for _, R in angle_records()[:-1]}
    assert ang == {"series", "closed"}
    S = gyro_samples()
    walks = [M.gyro_rotation(S, a, b, R_SI, BIAS)[1] for _, a, b in gyro_queries(S)]
    assert walks[0] == [] and set(walks[1]) == {"series"} and "closed" in walks[5]
    big = max(math.sqrt(sum(float(x.v) ** 2 for x in M.gyro_rate(R_SI, BIAS, S[j]))) / 64 for j in range(32, 48))
    assert 3.0 < big < math.pi                          # a piece of nearly pi
    sw = gyro_sweeps(S)
    T = list(S[:, 0])
    for name, start, span in sw:
        tm = start + 0.5 * span
        assert ("tm on a sample" in name) == (tm in T), name
        assert ("start and end on samples" not in name) or (start in T and start + span in T)


def test_harness_compiles_for_sm90a(tmp_path):
    """tools/test_motion_device.cu builds with the library's flags (no GPU needed to compile)."""
    tool_program(tmp_path, "test_motion_device.cu", compiler="device")


# ---- the device -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def program(tmp_path_factory):
    return tool_program(tmp_path_factory.mktemp("motion"), "test_motion_device.cu", compiler="device",
                        skip_missing=False)


def report(family, n, tally, dev_host_ulps, extra=""):
    print(f"\n{family}: {n} records, worst error {tally.worst:.3g} of its bound, device vs host "
          f"{dev_host_ulps:.3g} ulp{extra}")


@pytest.mark.gpu
def test_se3_log_exp_and_deskew(program, tmp_path):
    lr, er, dr = log_records(), exp_records(), deskew_records()
    P = Program()
    P.add(LOG, len(lr), b"".join(f8(R.reshape(-1)) + f8(t) for _, R, t in lr), ("<f8", 6 * len(lr)))
    P.add(EXP, len(er), b"".join(f8(xi) + f8([s]) + f8(p) for _, xi, s, p in er), ("<f8", 3 * len(er)))
    d = np.zeros(len(dr), DESKEW_IN)
    for i, (_, xi, tau, p) in enumerate(dr):
        d[i] = (xi, tau, np.asarray(p, F32))
    P.add(DESKEW, len(dr), d.tobytes(), (POINT, len(dr)))
    (xi_d, xi_h), (q_d, q_h), (p_d, p_h) = P.run(program, tmp_path)
    for fam, recs, dev, host, check in (("se3_log", lr, xi_d, xi_h, check_log), ("se3_exp_apply", er, q_d, q_h, check_exp)):
        t, br = Tally(), set()
        for got in (dev, host):
            check(recs, got.reshape(len(recs), -1), t, br)
        report(fam, len(recs), t, ulps(dev, host), f"; branches {sorted(br)}")
    t = Tally()
    kinds = check_deskew(dr, p_d, t) | check_deskew(dr, p_h, t)
    assert kinds == {"copy", "move", "overflow"}
    assert same_bits(p_d["moved"], p_h["moved"])
    report("deskew_point", len(dr), t, ulps(p_d["o"], p_h["o"]), " (error in float32 ulp or 1e-12 m)")


@pytest.mark.gpu
def test_so3_exp_and_the_gyro_walks(program, tmp_path):
    sr, S = so3_records(), gyro_samples()
    q, sw = gyro_queries(S), gyro_sweeps(S)
    gp = gyro_points(S, sw)
    from dcreg_b200 import api
    counts = [len(api.gyro_knots(S, s, sp, R_SI, BIAS)) for _, s, sp in sw]
    P = Program()
    P.add(SO3, len(sr), b"".join(f8(phi) for _, phi in sr), ("<f8", 9 * len(sr)))
    P.add(SAMPLES, len(S), f8(R_SI.reshape(-1)) + f8(BIAS) + f8(S))
    P.add(GYRO_ROT, len(q), b"".join(f8([a, b]) for _, a, b in q), ("<f8", 9 * len(q)))
    P.add(KNOTS, len(sw), b"".join(f8([s, sp, s + 0.5 * sp]) for _, s, sp in sw), ("<i4", 2 * len(sw)),
          ("<f8", 16 * sum(counts)))
    P.add(GYRO_DESKEW, len(gp), gp.tobytes(), (POINT, len(gp)))
    (R_d, R_h), (G_d, G_h), (c_d, c_h), (K_d, K_h), (p_d, p_h) = P.run(program, tmp_path)
    t, br = Tally(), set()
    R_d, R_h = R_d.reshape(-1, 9), R_h.reshape(-1, 9)
    for got in (R_d, R_h):
        check_so3(sr, got, t, br)
    series = np.array([so3_branch_fp64(list(phi)) == "series" for _, phi in sr])
    assert same_bits(R_d[series], R_h[series])                                     # one IEEE operation per step
    report("so3_exp", len(sr), t, ulps(R_d[~series], R_h[~series]), f" (series branch bit for bit: {series.sum()} records)")
    t = Tally()
    G_d, G_h = G_d.reshape(-1, 9), G_h.reshape(-1, 9)
    walks = check_gyro_rot(S, q, G_d, t)
    check_gyro_rot(S, q, G_h, t)
    exact = np.array([set(w) <= {"series"} for w in walks])                      # a = b, and series pieces only
    assert exact.sum() >= 2 and same_bits(G_d[exact], G_h[exact])
    report("gyro_rotation", len(q), t, ulps(G_d, G_h))
    t = Tally()
    for c, K in ((c_d, K_d), (c_h, K_h)):
        check_knots(S, sw, c.reshape(-1, 2), K.reshape(-1, 16), t)
    assert same_bits(c_d, c_h)
    K_d, K_h = K_d.reshape(-1, 16), K_h.reshape(-1, 16)
    assert same_bits(K_d[:, 0], K_h[:, 0]) and same_bits(K_d[:, 10:], K_h[:, 10:])
    slow = np.concatenate([np.full(n, "series" in name) for n, (name, _, _) in zip(counts, sw)])
    assert same_bits(K_d[slow], K_h[slow])                                          # walks of series pieces
    report("gyro_knots", len(K_d), t, ulps(K_d[:, 1:10], K_h[:, 1:10]))
    t = Tally()
    kinds = check_gyro_points(S, sw, gp, p_d, t) | check_gyro_points(S, sw, gp, p_h, t)
    assert {"copy", "on a knot", "between knots", "equal result"} <= kinds, kinds
    report("deskew_point_gyro", len(gp), t, ulps(p_d["o"], p_h["o"]), " (error in float32 ulp or 1e-12 m)")


@pytest.mark.gpu
def test_adaptive_threshold(program, tmp_path):
    ar, mr, fr, rr = angle_records(), model_error_records(), fold_records(), radius_records()
    P = Program()
    P.add(ANGLE, len(ar), b"".join(f8(R.reshape(-1)) for _, R in ar), ("<f8", len(ar)))
    P.add(MODEL_ERROR, len(mr), b"".join(f8(D.reshape(-1)) + f8([m]) for _, D, m in mr), ("<f8", len(mr)))
    P.add(FOLD, len(fr), fr.tobytes(), (STATE, len(fr)))
    P.add(RADIUS, len(rr), rr.tobytes(), ("<f8", len(rr)))
    (a_d, a_h), (e_d, e_h), (f_d, f_h), (r_d, r_h) = P.run(program, tmp_path)
    t, br = Tally(), set()
    for got in (a_d, a_h):
        check_angle(ar, got, t, br)
    series = np.array([angle_branch_fp64(R.reshape(-1))[0] == "series" for _, R in ar])
    assert series.sum() >= 3 and same_bits(a_d[series], a_h[series])
    report("rotation_angle", len(ar), t, ulps(a_d, a_h), f" (series branch bit for bit: {series.sum()} records)")
    t = Tally()
    for got in (e_d, e_h):
        check_model_error(mr, got, t)
    report("model_error", len(mr), t, ulps(e_d, e_h))
    for got in (f_d, f_h):
        check_fold(fr, got)
    for got in (r_d, r_h):
        check_radius(rr, got)
    print(f"\nfold: {len(fr)} records, radius: {len(rr)} records, bit for bit (device, host, twin)")


# ---- against production ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_deskew_call_is_log_then_deskew_point(ctx, program, tmp_path):  # noqa: F811
    """make_parking_sweeps, constant velocity: the program's se3_log of each frame's increment (the twin's
    constant_velocity_increment of the returned T_out) and deskew_point give the call's deskewed_xyz, bit for bit"""
    from dcreg_b200.api import constant_velocity_increment
    from odom_harness import parking_sweeps
    sw = parking_sweeps((5, 7), n_scan=8_000)
    res = ctx.icp_run_odometry(params(), sw["skewed"], sw["T_init"], None, cell_size=CELL, map_frames=3,
                               motion="constant_velocity", timestamps=sw["stamps"], want_deskewed=True)
    D, frames = [], []
    for s, rs in enumerate(split(res, sw["skewed"])):
        for j in range(2, len(rs)):
            D.append(constant_velocity_increment(rs[j - 2].T, rs[j - 1].T))
            frames.append((rs[j], sw["skewed"][s][j], sw["stamps"][s][j]))
    P = Program()
    P.add(LOG, len(D), b"".join(f8(d[:3, :3].reshape(-1)) + f8(d[:3, 3]) for d in D), ("<f8", 6 * len(D)))
    (xi_d, xi_h), = P.run(program, tmp_path)
    xi_d = xi_d.reshape(-1, 6)
    P = Program()
    recs = []
    for (r, pts, ts), xi in zip(frames, xi_d):
        d = np.zeros(len(pts), DESKEW_IN)
        d["xi"], d["tau"], d["p"] = xi, ts, pts[:, :3]
        recs.append(d)
    d = np.concatenate(recs)
    P.add(DESKEW, len(d), d.tobytes(), (POINT, len(d)))
    (p_d, _), = P.run(program, tmp_path)
    got = np.concatenate([r.deskewed for r, _, _ in frames])
    bad = np.nonzero((p_d["o"].view(np.uint32) != got.view(np.uint32)).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:10], p_d["o"][bad[:10]], got[bad[:10]])
    assert p_d["moved"].sum() > len(d) // 2
    print(f"\nproduction deskew: {len(D)} frames, {len(d)} points bit for bit ({p_d['moved'].sum()} moved)")


@pytest.mark.gpu
def test_gyro_call_is_rotation_knots_and_deskew_point_gyro(ctx, program, tmp_path):  # noqa: F811
    """make_parking_imu with an extrinsic and a bias: the program's gyro_rotation composed by the twin gives the call's
    T_prior, and gyro_knots + deskew_point_gyro its deskewed_xyz, bit for bit"""
    from dcreg_b200.api import AdaptiveThreshold, Gyro, compose_prior, constant_velocity_increment, gyro_knots
    from dcreg_b200.scenes import make_parking_imu
    R_imu = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    bias = (0.002, -0.001, 0.003)
    sk, ts, ft, smp, T, fr = make_parking_imu(7, n_scan=6_000, max_range=20.0, R_sensor_imu=R_imu, bias=bias)
    sk[0] = fr[0]
    res = ctx.icp_run_odometry(params(), [list(sk)], T[:1], None, map_frames=3, cell_size=CELL,
                               motion="constant_velocity", gyro=Gyro(R_imu, bias), frame_times=ft, gyro_samples=[smp],
                               timestamps=[list(ts)], want_deskewed=True, adaptive=AdaptiveThreshold(0.12, 0.01, 20.0))
    tm = ft[:, 0] + 0.5 * ft[:, 1]
    P = Program()
    P.add(SAMPLES, len(smp), f8(R_imu.reshape(-1)) + f8(bias) + f8(smp))
    P.add(GYRO_ROT, 6, b"".join(f8([tm[k - 1], tm[k]]) for k in range(1, 7)), ("<f8", 54))
    counts = np.array([len(gyro_knots(smp, ft[k, 0], ft[k, 1], R_imu, bias)) for k in range(1, 7)])
    P.add(KNOTS, 6, b"".join(f8([ft[k, 0], ft[k, 1], tm[k]]) for k in range(1, 7)), ("<i4", 12),
          ("<f8", 16 * int(counts.sum())))
    recs, tD = [], []
    for k in range(1, 7):
        t = np.zeros(3) if k == 1 else constant_velocity_increment(res[k - 2].T, res[k - 1].T)[:3, 3]
        g = np.zeros(len(sk[k]), GYRO_IN)
        g["tm_prev"], g["tD"], g["sweep"], g["tau"], g["p"] = tm[k - 1], t, k - 1, ts[k], sk[k][:, :3]
        recs.append(g)
        tD.append(t)
    g = np.concatenate(recs)
    P.add(GYRO_DESKEW, len(g), g.tobytes(), (POINT, len(g)))
    (G_d, _), (c_d, _), _, (p_d, _) = P.run(program, tmp_path)
    assert same_bits(c_d.reshape(-1, 2)[:, 0], counts.astype(np.int32))
    for k in range(1, 7):
        D = np.eye(4)
        D[:3, :3], D[:3, 3] = G_d[9 * (k - 1):9 * k].reshape(3, 3), tD[k - 1]
        P_k = compose_prior(res[k - 1].T, D)
        assert same_bits(res[k].T_prior, P_k), (k, np.abs(res[k].T_prior - P_k).max())
    got = np.concatenate([res[k].deskewed for k in range(1, 7)])
    bad = np.nonzero((p_d["o"].view(np.uint32) != got.view(np.uint32)).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:10], p_d["o"][bad[:10]], got[bad[:10]])
    assert p_d["moved"].sum() > len(g) // 2
    print(f"\nproduction gyro: 6 priors and {len(g)} points bit for bit ({int(counts.sum())} knots)")


@pytest.mark.gpu
def test_adaptive_call_is_model_error_fold_and_radius(ctx, program, tmp_path):  # noqa: F811
    """An adaptive call: the program's model_error + fold + radius, fed each frame's correction (the twin's
    constant_velocity_increment of the returned T_prior and T_out), give the call's search_radius, bit for bit"""
    from dcreg_b200.api import AdaptiveThreshold, constant_velocity_increment
    from odom_harness import parking
    seqs, T_init, deltas = parking((1, 7, 12), n_scan=8_000)[:3]
    thr = AdaptiveThreshold(0.12, 0.01, 20.0)
    res = ctx.icp_run_odometry(params(search_radius=2.0), seqs, T_init, deltas, map_frames=3, cell_size=CELL,
                               adaptive=thr, map_max_points=4)
    per = split(res, seqs)
    D, off, want = [], [0], []
    for rs in per:
        for r in rs[1:]:
            D.append(constant_velocity_increment(r.T_prior, r.T))
            want.append(r.search_radius)
        off.append(len(D))
    P = Program()
    P.add(CHAIN, len(D), f8([thr.initial_threshold, thr.min_motion, thr.max_range, 2.0]) +
          np.array([len(per)] + off, np.int32).tobytes() + b"".join(f8(d) for d in D), ("<f8", len(D)))
    (r_d, r_h), = P.run(program, tmp_path)
    want = np.array(want)
    assert same_bits(r_d, want), np.nonzero(r_d != want)
    assert len(set(want)) >= 4
    # (the host build's radii differ where libm's sin and atan2 round differently from CUDA's)
    print(f"\nproduction adaptive: {len(D)} radii bit for bit ({len(set(want))} distinct); host build "
          f"{ulps(r_h, want):.3g} ulp from them")
