"""50-digit reference of the odometry's motion math (dcreg_b200/csrc/se3.cuh, adaptive_threshold.cuh).  TEST
INFRASTRUCTURE ONLY.

Every input is taken as the exact value of the FP64 or float32 number the device sees.  The functions compute with X
numbers: X.v is the exact value (mpmath, DPS digits) of the quantity, X.e a bound on how far an FP64 evaluation of the
header's formula, on those inputs, can land from it:

  * one rounding per operation, u (|z| + e) with u = 2^-53, and the operands' errors carried through the operation
    (|y| e_x + |x| e_y + e_x e_y for a product, (e_x + |z| e_y) / (|y| - e_y) for a quotient, e_x / (sqrt(x) +
    sqrt(x - e_x)) for a square root); constants such as 2.0 / 3.0 are rounded like any other quotient;
  * a fused multiply-add rounds once where the pair rounds twice, so --fmad=true stays inside the bound of the unfused
    formula (the bound never assumes two roundings cancel);
  * sin, cos and atan2 add LIB_ULP ulp of their result (CUDA documents 2 ulp for the double-precision sin, cos, sincos
    and atan2; glibc is within 1), and carry their arguments' errors with their derivatives (the largest over the
    arguments' error box for atan2, plus the second-order term for sin and cos);
  * where the header takes a series below a threshold (pick), the value is the exact function and the bound that of the
    branch's formula plus its distance from the exact function (the series' truncation); where the rounded predicate can
    fall on either side of the threshold, the larger of the two branches' bounds;
  * Shepperd's choice of quaternion branch (tr > 0, the largest diagonal entry) and the sign of w are decided, as in the
    headers, by sums, differences, products, a quotient and a square root that nvcc cannot contract and IEEE rounds one
    way: they are replayed here in Python floats, and the reference follows the branch the device takes.

The bounds are first order in the rounding errors (products of two rounding errors are kept where an operation meets
them, nothing smaller is dropped silently), derived from the operation count and the conditioning at the input, not
from any device output.
"""
from __future__ import annotations

import math

import mpmath as mp

DPS = 50
mp.mp.dps = DPS
U = mp.mpf(2) ** -53                   # FP64 unit roundoff
EPS = 2.0 ** -52
LIB_ULP = 2                            # ulp of sin, cos, sincos, atan2 (CUDA's documented maximum)
K_LOG_SMALL = 1e-10                    # se3::kLogSmall
K_LOG_SMALL2 = K_LOG_SMALL * K_LOG_SMALL    # the rounded square the headers compare |v|^2 against
K_SMALL_ANGLE = 1e-3                   # se3::kSmallAngle


class X:
    """An exact value and a bound on the error of its FP64 evaluation"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0):
        self.v = v if isinstance(v, mp.mpf) else mp.mpf(v)
        self.e = e if isinstance(e, mp.mpf) else mp.mpf(e)

    @staticmethod
    def of(x):
        return x if isinstance(x, X) else X(x)

    def _round(v, e):                 # noqa: N805 - a plain function used below
        return X(v, e + U * (abs(v) + e))

    def __neg__(self):
        return X(-self.v, self.e)

    def __add__(self, o):
        o = X.of(o)
        return X._round(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = X.of(o)
        return X._round(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return X.of(o) - self

    def __mul__(self, o):
        o = X.of(o)
        return X._round(self.v * o.v, abs(self.v) * o.e + abs(o.v) * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = X.of(o)
        z = self.v / o.v
        room = abs(o.v) - o.e
        return X._round(z, (self.e + abs(z) * o.e) / room if room > 0 else mp.inf)

    def __rtruediv__(self, o):
        return X.of(o) / self

    def __repr__(self):
        return f"X({mp.nstr(self.v, 20)} +- {mp.nstr(self.e, 3)})"


def sqrt(x):
    v = mp.sqrt(x.v) if x.v > 0 else mp.mpf(0)
    lo = mp.sqrt(x.v - x.e) if x.v > x.e else mp.mpf(0)
    prop = x.e / (v + lo) if v + lo > 0 else mp.mpf(0)
    return X._round(v, prop)


def _lib(v, prop):
    """a library function's result: the propagated error and LIB_ULP ulp (ulp(y) <= 2 u |y|)"""
    return X(v, prop + LIB_ULP * 2 * U * (abs(v) + prop))


def sin(x):
    v = mp.sin(x.v)
    return _lib(v, x.e * (abs(mp.cos(x.v)) + x.e))      # |sin(x + d) - sin(x)| <= |cos(x)| |d| + d^2 / 2


def cos(x):
    v = mp.cos(x.v)
    return _lib(v, x.e * (abs(mp.sin(x.v)) + x.e))


def atan2(y, x):
    """|d atan2 / dy| = |x| / r^2, |d atan2 / dx| = |y| / r^2, taken at their largest over the inputs' error box"""
    v = mp.atan2(y.v, x.v)
    room = mp.sqrt(y.v * y.v + x.v * x.v) - y.e - x.e
    prop = (y.e * (abs(x.v) + x.e) + x.e * (abs(y.v) + y.e)) / room ** 2 if room > 0 else mp.pi
    return _lib(v, prop)


def pick(x, thr, series, closed, exact):
    """The header's `x < thr ? series : closed`, with x the X of the predicate's operand.  The value is the exact
    function (exact); the bound covers every branch the rounded x can take, each with its distance from the function"""
    got = []
    if x.v - x.e < thr:
        got.append(series())
    if x.v + x.e >= thr:
        got.append(closed())
    return X(exact, max(g.e + abs(g.v - exact) for g in got))


def branch(x, thr):
    """which branches of `x < thr` the rounded x can take: 'series', 'closed' or 'either'"""
    lo, hi = x.v - x.e < thr, x.v + x.e >= thr
    return "either" if lo and hi else ("series" if lo else "closed")


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _mp(x):
    return x.v if isinstance(x, X) else mp.mpf(x)


def _flat(M):
    """a 3x3 (nested or array) or 9 numbers as 9 floats"""
    import numpy as np
    return [float(x) for x in np.asarray(M, dtype=np.float64).reshape(-1)]


# ---- the exact coefficients ---------------------------------------------------------------------------------------
def _series(theta, first, n=24):
    """sum_k (-1)^k theta^(2k) / (2k + first)!"""
    t2 = theta * theta
    return mp.fsum((-1) ** k * t2 ** k / mp.factorial(2 * k + first) for k in range(n))


def exp_coeffs(theta):
    """A = sin(theta) / theta, B = (1 - cos(theta)) / theta^2, C = (theta - sin(theta)) / theta^3, exactly (their series
    below 1e-2, where the closed forms cancel)"""
    theta = mp.mpf(theta)
    if theta < mp.mpf("1e-2"):
        return _series(theta, 1), _series(theta, 2), _series(theta, 3)
    return mp.sin(theta) / theta, (1 - mp.cos(theta)) / theta ** 2, (theta - mp.sin(theta)) / theta ** 3


def log_c(theta):
    """c = (1 - theta cos(theta / 2) / (2 sin(theta / 2))) / theta^2 = sum_n |B_2n| theta^(2n - 2) / (2n)!, exactly"""
    theta = mp.mpf(theta)
    if theta < mp.mpf("1e-2"):
        return mp.fsum(abs(mp.bernoulli(2 * n)) * theta ** (2 * n - 2) / mp.factorial(2 * n) for n in range(1, 24))
    h = theta / 2
    return (1 - theta * mp.cos(h) / (2 * mp.sin(h))) / theta ** 2


# ---- se3_log --------------------------------------------------------------------------------------------------------
def shepperd(R):
    """Shepperd's branch as the headers take it, replayed in FP64: (tr > 0, i, w < 0).  R: 9 floats"""
    R = [float(x) for x in R]
    tr = (R[0] + R[4]) + R[8]
    if tr > 0.0:
        return True, -1, False
    i = 0
    if R[4] > R[0]:
        i = 1
    if R[8] > R[4 * i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    r = math.sqrt(((R[4 * i] - R[4 * j]) - R[4 * k]) + 1.0)
    w = (R[3 * k + j] - R[3 * j + k]) * (0.5 / r)
    return False, i, w < 0.0


def quaternion(R):
    """(w, v) of R (9 floats) as X, Shepperd's branch and the sign rule of the headers (w >= 0)"""
    pos, i, flip = shepperd(R)
    Rx = [X(float(x)) for x in R]
    v = [None] * 3
    if pos:
        tr = (Rx[0] + Rx[4]) + Rx[8]
        r = sqrt(tr + 1.0)
        w = 0.5 * r
        r = 0.5 / r
        v = [(Rx[7] - Rx[5]) * r, (Rx[2] - Rx[6]) * r, (Rx[3] - Rx[1]) * r]
    else:
        j, k = (i + 1) % 3, (i + 2) % 3
        r = sqrt(((Rx[4 * i] - Rx[4 * j]) - Rx[4 * k]) + 1.0)
        v[i] = 0.5 * r
        r = 0.5 / r
        w = (Rx[3 * k + j] - Rx[3 * j + k]) * r
        v[j] = (Rx[3 * j + i] + Rx[3 * i + j]) * r
        v[k] = (Rx[3 * k + i] + Rx[3 * i + k]) * r
    if flip:
        w, v = -w, [-x for x in v]
    return w, v


def _atan_factor(w, v):
    """f = 2 atan(|v| / w) / |v| (kLogSmall's series below) and theta = f |v|, as X"""
    n2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
    n_exact = mp.sqrt(n2.v)
    f_exact = 2 / w.v if n_exact == 0 else 2 * mp.atan2(n_exact, w.v) / n_exact

    def closed():
        n = sqrt(n2)
        return 2.0 * atan2(n, w) / n

    f = pick(n2, K_LOG_SMALL2, lambda: 2.0 / w - (X(2.0) / 3.0) * n2 / ((w * w) * w), closed, f_exact)
    return f, n2, f * sqrt(n2)


def log(R, t):
    """Log(D) of D = [R t] (R 9 floats row-major, t 3 floats): 6 X, (rho, phi), or None when an entry is not finite.
    Also the branches: dict(pos=tr > 0, i=Shepperd's index, flip=w < 0, log_small=branch of |v|^2 against kLogSmall^2,
    small=branch of theta against kSmallAngle)"""
    if not all(math.isfinite(float(x)) for x in list(R) + list(t)):
        return None, None
    pos, i, flip = shepperd(R)
    w, v = quaternion(R)
    f, n2, theta = _atan_factor(w, v)
    phi = [f * x for x in v]
    th = theta.v

    def closed():
        h = 0.5 * theta
        return (1.0 - theta * cos(h) / (2.0 * sin(h))) / (theta * theta)

    c = pick(theta, K_SMALL_ANGLE, lambda: X(1.0) / 12.0 + (theta * theta) / 720.0, closed, log_c(th))
    tx = [X(float(x)) for x in t]
    a = cross(phi, tx)
    b = cross(phi, a)
    xi = [(tx[r] - 0.5 * a[r]) + c * b[r] for r in range(3)] + phi
    return xi, dict(pos=pos, i=i, flip=flip, log_small=branch(n2, K_LOG_SMALL2), small=branch(theta, K_SMALL_ANGLE))


def mp_log(D):
    """Log(D) (4x4) in DPS digits: 6 mpf"""
    R = [float(D[r][c]) for r in range(3) for c in range(3)]
    xi, _ = log(R, [float(D[r][3]) for r in range(3)])
    return [x.v for x in xi]


# ---- se3_exp_apply, deskew_point ------------------------------------------------------------------------------------
def exp_apply(xi, s, p):
    """q = Exp(s xi) p (xi 6, s, p 3 exact inputs): 3 X, and the branch of theta = |s phi| against kSmallAngle"""
    s = X(float(s))
    rho = [s * X(float(x)) for x in xi[:3]]
    phi = [s * X(float(x)) for x in xi[3:]]
    t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2]
    theta = sqrt(t2)
    Ae, Be, Ce = exp_coeffs(theta.v)

    def closed(which):
        def f():
            sn, cs = sin(theta), cos(theta)
            return (sn / theta, (1.0 - cs) / t2, (theta - sn) / (t2 * theta))[which]
        return f

    series = (lambda: 1.0 - t2 / 6.0 * (1.0 - t2 / 20.0), lambda: 0.5 - t2 / 24.0 * (1.0 - t2 / 30.0),
              lambda: X(1.0) / 6.0 - t2 / 120.0 * (1.0 - t2 / 42.0))
    A, B, C = (pick(theta, K_SMALL_ANGLE, series[m], closed(m), ex) for m, ex in enumerate((Ae, Be, Ce)))
    px = [X(float(x)) for x in p]
    a, c = cross(phi, px), cross(phi, rho)
    b, d = cross(phi, a), cross(phi, c)
    q = [((px[r] + A * a[r]) + B * b[r]) + ((rho[r] + B * c[r]) + C * d[r]) for r in range(3)]
    return q, branch(theta, K_SMALL_ANGLE)


def mp_exp_apply(xi, s, p):
    """Exp(s xi) p in DPS digits from mpf (or float) inputs, no bound: the exact map"""
    rho = [s * _mp(x) for x in xi[:3]]
    phi = [s * _mp(x) for x in xi[3:]]
    A, B, C = exp_coeffs(mp.sqrt(sum(x * x for x in phi)))
    p = [_mp(x) for x in p]
    a, c = cross(phi, p), cross(phi, rho)
    b, d = cross(phi, a), cross(phi, c)
    return [p[r] + A * a[r] + B * b[r] + rho[r] + B * c[r] + C * d[r] for r in range(3)]


def mp_exp(xi):
    """Exp(xi) as a 4x4 of mpf"""
    T = [[mp.mpf(int(r == c)) for c in range(4)] for r in range(4)]
    t0 = mp_exp_apply(xi, 1, [0, 0, 0])
    for c in range(3):
        col = mp_exp_apply(xi, 1, [int(r == c) for r in range(3)])
        for r in range(3):
            T[r][c] = col[r] - t0[r]
    for r in range(3):
        T[r][3] = t0[r]
    return T


F32_MAX = mp.mpf(3.4028234663852886e38)


def deskew_expected(xi, tau, p):
    """What se3::deskew_point must return for (xi 6 floats, tau float32, p 3 float32): ('copy', None) when its rules
    copy the point, ('move', exact) with the exact Exp((tau - 0.5) xi) p otherwise, ('overflow', exact) when the exact
    value is out of float32's range by more than the FP64 error (copied too), None when that is not decidable"""
    s = float(tau) - 0.5
    xi = [float(x) for x in xi]
    if s == 0.0 or all(x == 0.0 for x in xi) or not all(math.isfinite(x) for x in xi) \
            or not all(math.isfinite(float(x)) for x in p):
        return "copy", None
    q, _ = exp_apply(xi, s, p)
    big = F32_MAX * (1 + mp.mpf(2) ** -25)          # past the last value float32 rounds to its largest finite number
    if any(abs(x.v) - x.e > big for x in q):
        return "overflow", q
    if any(abs(x.v) + x.e >= big for x in q):
        return None, q
    return "move", q


def within_contract(got, exact):
    """|got - exact| <= max(one float32 ulp of the exact value, 1e-12 m) per coordinate; returns (ok, worst error in
    units of that allowance)"""
    import numpy as np
    worst = 0.0
    for g, x in zip(got, exact):
        ex = float(x)
        allow = max(float(np.spacing(np.float32(abs(ex)))), 1e-12)
        worst = max(worst, float(abs(mp.mpf(float(g)) - x)) / allow)
    return worst <= 1.0, worst


# ---- so3_exp and the gyro walk --------------------------------------------------------------------------------------
def so3_exp(phi):
    """R = Exp(phi) (phi 3 X or floats) as 9 X, se3::so3_exp's formula; and the branch of theta against kSmallAngle"""
    phi = [X.of(x) if isinstance(x, X) else X(float(x)) for x in phi]
    t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2]
    theta = sqrt(t2)
    Ae, Be, _ = exp_coeffs(theta.v)
    A = pick(theta, K_SMALL_ANGLE, lambda: 1.0 - (t2 / 6.0) * (1.0 - t2 / 20.0), lambda: sin(theta) / theta, Ae)
    B = pick(theta, K_SMALL_ANGLE, lambda: 0.5 - (t2 / 24.0) * (1.0 - t2 / 30.0), lambda: (1.0 - cos(theta)) / t2, Be)
    K = [X(0), -phi[2], phi[1], phi[2], X(0), -phi[0], -phi[1], phi[0], X(0)]
    R = [1.0 + B * (phi[r] * phi[r] - t2) if r == c else A * K[3 * r + c] + B * (phi[r] * phi[c])
         for r in range(3) for c in range(3)]
    return R, branch(theta, K_SMALL_ANGLE)


def mat3_mul(M, E):
    return [(M[3 * r] * E[c] + M[3 * r + 1] * E[3 + c]) + M[3 * r + 2] * E[6 + c] for r in range(3) for c in range(3)]


def identity():
    return [X(1.0 if i % 4 == 0 else 0.0) for i in range(9)]


def gyro_rate(R_si, bias, row):
    """R_si (omega - bias) of a sample row (t, wx, wy, wz), as 3 X"""
    d = [X(float(row[1 + c])) - X(float(bias[c])) for c in range(3)]
    Rx = [X(float(x)) for x in _flat(R_si)]
    return [(Rx[3 * r] * d[0] + Rx[3 * r + 1] * d[1]) + Rx[3 * r + 2] * d[2] for r in range(3)]


def piece(M, w, d):
    """M Exp(w d), and the branch of that piece's so3_exp"""
    E, br = so3_exp([x * d for x in w])
    return mat3_mul(M, E), br


def last_sample(times, t, strict):
    """se3::gyro_last: the last j with times[j] <= t (strict: < t), or -1"""
    import bisect
    return (bisect.bisect_left(times, t) if strict else bisect.bisect_right(times, t)) - 1


def gyro_rotation(S, a, b, R_si, bias):
    """G(a -> b) (a <= b floats) over the samples S (rows (t, wx, wy, wz)): 9 X, and the branches of its pieces"""
    times = [float(r[0]) for r in S]
    j = last_sample(times, float(a), False)
    M, cur, brs = identity(), float(a), []
    while cur < float(b):
        nxt = min(times[j + 1], float(b))
        M, br = piece(M, gyro_rate(R_si, bias, S[j]), X(nxt) - X(cur))
        brs.append(br)
        cur = nxt
        j += 1
    return M, brs


def gyro_knots(S, start, tm, end, R_si, bias):
    """The knot table of the sweep [start, end] with mid-sweep tm (floats): a list of (time, Q 9 X, w_after 3 X,
    w_before 3 X), ascending, Q the walk from tm with se3::gyro_knots' pieces; and the number before tm"""
    times = [float(r[0]) for r in S]
    lo, m0 = last_sample(times, start, False), last_sample(times, tm, True)
    m1, hi = last_sample(times, tm, False), last_sample(times, end, True)
    mid = (tm, identity(), gyro_rate(R_si, bias, S[m1]), gyro_rate(R_si, bias, S[m0]))
    before, Q, cur, w = [], identity(), tm, mid[3]
    for jb in range(m0, lo, -1):
        Q, _ = piece(Q, w, X(times[jb]) - X(cur))
        cur = times[jb]
        k = (cur, Q, gyro_rate(R_si, bias, S[jb]), gyro_rate(R_si, bias, S[jb - 1]))
        before.append(k)
        w = k[3]
    after, Q, cur, w = [], identity(), tm, mid[2]
    for ja in range(m1 + 1, hi + 1):
        Q, _ = piece(Q, w, X(times[ja]) - X(cur))
        cur = times[ja]
        k = (cur, Q, gyro_rate(R_si, bias, S[ja]), gyro_rate(R_si, bias, S[ja - 1]))
        after.append(k)
        w = k[2]
    return before[::-1] + [mid] + after, m0 - lo


def point_time(start, tau, span):
    """t = start + tau span, one rounding per operation (se3::deskew_point_gyro), as a float"""
    return float(start) + float(tau) * float(span)


def gyro_point(knots, t, tm, tm_prev, tD, p):
    """G(tm -> t) p + s tD (s = (t - tm) / (tm - tm_prev)) from the knot table as deskew_point_gyro defines G: for
    t >= tm the last knot at or before t and its rate after, else the first knot at or after t and its rate before;
    t the point's FP64 time.  3 X, and the branch of the final piece"""
    kt = [k[0] for k in knots]
    import bisect
    if t >= tm:
        k = knots[bisect.bisect_right(kt, t) - 1]
        w = k[2]
    else:
        k = knots[bisect.bisect_left(kt, t)]
        w = k[3]
    G, br = piece(k[1], w, X(t) - X(k[0]))
    s = (X(t) - X(tm)) / (X(tm) - X(float(tm_prev)))
    px = [X(float(x)) for x in p]
    return [((G[3 * r] * px[0] + G[3 * r + 1] * px[1]) + G[3 * r + 2] * px[2]) + s * X(float(tD[r]))
            for r in range(3)], br


def mp_so3_exp(phi):
    """Exp(phi) as an mpmath 3x3 matrix, exactly"""
    phi = [_mp(x) for x in phi]
    A, B, _ = exp_coeffs(mp.sqrt(sum(x * x for x in phi)))
    K = mp.matrix([[0, -phi[2], phi[1]], [phi[2], 0, -phi[0]], [-phi[1], phi[0], 0]])
    return mp.eye(3) + A * K + B * (K * K)


def mp_gyro_rotation(S, a, b, R_si, bias):
    """G(a -> b) in DPS digits: the walk over the sample intervals clipped to [a, b] with exact rates and durations"""
    times = [float(r[0]) for r in S]
    Rf = _flat(R_si)
    Rm = mp.matrix([[mp.mpf(Rf[3 * r + c]) for c in range(3)] for r in range(3)])
    M, cur = mp.eye(3), mp.mpf(float(a))
    j = last_sample(times, float(a), False)
    while cur < float(b):
        nxt = min(mp.mpf(times[j + 1]), mp.mpf(float(b)))
        w = Rm * mp.matrix([mp.mpf(float(S[j][c + 1])) - mp.mpf(float(bias[c])) for c in range(3)])
        M = M * mp_so3_exp([w[c] * (nxt - cur) for c in range(3)])
        cur, j = nxt, j + 1
    return M


# ---- the adaptive threshold -----------------------------------------------------------------------------------------
def rotation_angle(R):
    """theta of R (9 floats) by adaptive::rotation_angle's route: X (None when an entry is not finite), and the branch
    of |v|^2 against 1e-10^2"""
    if not all(math.isfinite(float(x)) for x in R):
        return None, None
    w, v = quaternion(R)
    w = X(abs(w.v), w.e)
    f, n2, theta = _atan_factor(w, v)
    return theta, branch(n2, K_LOG_SMALL2)


def model_error(D, max_range):
    """e = 2 max_range sin(theta / 2) + |t_D| of D (16 floats row-major): X, or None when not finite"""
    theta, _ = rotation_angle([D[0], D[1], D[2], D[4], D[5], D[6], D[8], D[9], D[10]])
    t = [float(D[3]), float(D[7]), float(D[11])]
    if theta is None or not all(math.isfinite(x) for x in t):
        return None
    tx = [X(x) for x in t]
    t2 = (tx[0] * tx[0] + tx[1] * tx[1]) + tx[2] * tx[2]
    return (2.0 * X(float(max_range))) * sin(0.5 * theta) + sqrt(t2)


def mp_rotation_angle(R):
    """theta of R (9 floats) in DPS digits by Shepperd's quaternion, 2 atan2(|v|, |w|)"""
    theta, _ = rotation_angle(R)
    return None if theta is None else theta.v


def mp_model_error(D, max_range):
    e = model_error(D, max_range)
    return None if e is None else e.v
