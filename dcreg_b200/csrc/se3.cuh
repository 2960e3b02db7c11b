// se3.cuh - the SE(3) log / exp of the odometry's motion compensation (dcreg_icp_run_odometry_deskew), host and device.
//
// A twist is xi = (rho, phi), Sophus's order: rho the translational part, phi the rotation vector.  Everything is FP64;
// dcreg_b200.api.se3_log / se3_exp / deskew_points are the NumPy twin with the same formulas and branch thresholds.
// Plain C++ as well, so tools/test_se3.cpp checks the host build against the twin (tests/test_se3_host.py).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define SE3_HD __host__ __device__ __forceinline__
#else
#define SE3_HD inline
#endif

namespace se3 {

constexpr double kLogSmall = 1e-10;     // |quaternion vector| below which 2 atan(n / w) / n takes its series
constexpr double kSmallAngle = 1e-3;    // rotation angle below which A, B, C and the V^-1 factor take their series

SE3_HD void cross(const double* a, const double* b, double* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// xi = Log(D) of the rigid motion D = [R t] (R row-major 3x3, t 3).  The rotation goes through its quaternion (Eigen's
// Shepperd rule: the largest of w and the diagonal picks the well-conditioned branch, w >= 0 after it), then
// theta = 2 atan2(|v|, w), exact for every angle in [0, pi] (Sophus SO3::logAndTheta's form, no acos).  rho = V^-1 t
// with V^-1 = I - Omega / 2 + c Omega^2, c = (1 - theta cos(theta/2) / (2 sin(theta/2))) / theta^2.  The exact
// identity gives exactly zero; a D with an entry that is not finite gives a NaN twist.
SE3_HD void se3_log(const double* R, const double* t, double* xi) {
    bool finite = isfinite(t[0]) && isfinite(t[1]) && isfinite(t[2]);
    for (int i = 0; i < 9; ++i) finite = finite && isfinite(R[i]);
    if (!finite) {
        for (int i = 0; i < 6; ++i) xi[i] = NAN;
        return;
    }
    const double tr = (R[0] + R[4]) + R[8];
    double w, v[3];
    if (tr > 0.0) {
        double r = sqrt(tr + 1.0);
        w = 0.5 * r;
        r = 0.5 / r;
        v[0] = (R[7] - R[5]) * r;
        v[1] = (R[2] - R[6]) * r;
        v[2] = (R[3] - R[1]) * r;
    } else {
        int i = 0;
        if (R[4] > R[0]) i = 1;
        if (R[8] > R[4 * i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        double r = sqrt(((R[4 * i] - R[4 * j]) - R[4 * k]) + 1.0);
        v[i] = 0.5 * r;
        r = 0.5 / r;
        w = (R[3 * k + j] - R[3 * j + k]) * r;
        v[j] = (R[3 * j + i] + R[3 * i + j]) * r;
        v[k] = (R[3 * k + i] + R[3 * i + k]) * r;
    }
    if (w < 0.0) { w = -w; v[0] = -v[0]; v[1] = -v[1]; v[2] = -v[2]; }
    const double n2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2];
    double f;                                               // 2 atan(n / w) / n
    if (n2 < kLogSmall * kLogSmall) f = 2.0 / w - (2.0 / 3.0) * n2 / ((w * w) * w);
    else { const double n = sqrt(n2); f = 2.0 * atan2(n, w) / n; }
    const double theta = f * sqrt(n2);
    double* phi = xi + 3;
    phi[0] = f * v[0]; phi[1] = f * v[1]; phi[2] = f * v[2];
    double c;
    if (theta < kSmallAngle) c = 1.0 / 12.0 + (theta * theta) / 720.0;
    else {
        const double h = 0.5 * theta;
        c = (1.0 - theta * cos(h) / (2.0 * sin(h))) / (theta * theta);
    }
    double a[3], b[3];
    cross(phi, t, a);
    cross(phi, a, b);
    for (int r = 0; r < 3; ++r) xi[r] = (t[r] - 0.5 * a[r]) + c * b[r];
}

// q = Exp(s xi) p: phi' = s phi, rho' = s rho, theta = |phi'|, R p = p + A phi' x p + B phi' x (phi' x p) (Rodrigues)
// and V rho' = rho' + B phi' x rho' + C phi' x (phi' x rho') with A = sin(theta) / theta, B = (1 - cos(theta)) /
// theta^2, C = (theta - sin(theta)) / theta^3 (their series below kSmallAngle).  q = R p + V rho' in FP64.
SE3_HD void se3_exp_apply(const double* xi, double s, const double* p, double* q) {
    const double rho[3] = {s * xi[0], s * xi[1], s * xi[2]};
    const double phi[3] = {s * xi[3], s * xi[4], s * xi[5]};
    const double t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2];
    const double theta = sqrt(t2);
    double A, B, C;
    if (theta < kSmallAngle) {
        A = 1.0 - t2 / 6.0 * (1.0 - t2 / 20.0);
        B = 0.5 - t2 / 24.0 * (1.0 - t2 / 30.0);
        C = 1.0 / 6.0 - t2 / 120.0 * (1.0 - t2 / 42.0);
    } else {
        double sn, cs;
#ifdef __CUDA_ARCH__
        sincos(theta, &sn, &cs);
#else
        sn = sin(theta); cs = cos(theta);
#endif
        A = sn / theta;
        B = (1.0 - cs) / t2;
        C = (theta - sn) / (t2 * theta);
    }
    double a[3], b[3], c[3], d[3];
    cross(phi, p, a);
    cross(phi, a, b);
    cross(phi, rho, c);
    cross(phi, c, d);
    for (int r = 0; r < 3; ++r) q[r] = ((p[r] + A * a[r]) + B * b[r]) + ((rho[r] + B * c[r]) + C * d[r]);
}

// One point of a frame deskewed to mid-sweep: out = fl32(Exp((tau - 0.5) xi) p), or p itself, bit for bit (no
// arithmetic: -0.0 and NaN payloads stay), when tau = 0.5, when xi is zero or not finite, when p has a non-finite
// coordinate, or when the result would have one.  Returns whether it moved the point.
SE3_HD bool deskew_point(const double* xi, float tau, const float* p, float* out) {
    const double s = (double)tau - 0.5;
    bool zero = true, finite = true;
    for (int i = 0; i < 6; ++i) { zero = zero && xi[i] == 0.0; finite = finite && isfinite(xi[i]); }
    bool move = s != 0.0 && !zero && finite && isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
    float o[3] = {p[0], p[1], p[2]};
    if (move) {
        const double pd[3] = {(double)p[0], (double)p[1], (double)p[2]};
        double q[3];
        se3_exp_apply(xi, s, pd, q);
        for (int r = 0; r < 3; ++r) o[r] = (float)q[r];
        move = isfinite(o[0]) && isfinite(o[1]) && isfinite(o[2]);
    }
    for (int r = 0; r < 3; ++r) out[r] = move ? o[r] : p[r];
    return move;
}

// ---- gyroscope rotation (dcreg_icp_run_odometry_gyro) ------------------------------------------------------------
// Every product, sum and difference below is one IEEE operation (no FMA contraction on the device), so the host build
// and dcreg_b200.api.gyro_rotation / gyro_knots / deskew_points_gyro give the same bits; on the device only sin and cos
// (CUDA's sincos) may differ from libm in the last bit.
#ifdef __CUDA_ARCH__
#define SE3_MUL(x, y) __dmul_rn(x, y)
#define SE3_ADD(x, y) __dadd_rn(x, y)
#define SE3_SUB(x, y) __dsub_rn(x, y)
#else
#define SE3_MUL(x, y) ((x) * (y))
#define SE3_ADD(x, y) ((x) + (y))
#define SE3_SUB(x, y) ((x) - (y))
#endif

// The gyro's settings: R_si maps IMU-frame rates into the LiDAR frame (row-major), bias is subtracted first (rad/s)
struct Gyro {
    double R_si[9];
    double bias[3];
};

// Rows of a sample array: (t, wx, wy, wz), t strictly ascending; with an accelerometer (dcreg_icp_run_odometry_imu)
// (t, wx, wy, wz, ax, ay, az).  Every function below that reads samples takes the row stride, the gyro's by default
constexpr int kSampleStride = 4;
constexpr int kImuStride = 7;
// One knot of a sweep's table: time, Q = G(t_m -> time) row-major, the rate after the knot, the rate before it
constexpr int kKnotStride = 16;

// R = Exp(phi), row-major, by Rodrigues: R = I + A K + B K^2 with K = [phi]x and K^2 = phi phi^T - theta^2 I, so
// R_rr = 1 + B (phi_r^2 - t2) and R_rc = A K_rc + B phi_r phi_c, with se3_exp_apply's A, B and series threshold
SE3_HD void so3_exp(const double* phi, double* R) {
    const double t2 = SE3_ADD(SE3_ADD(SE3_MUL(phi[0], phi[0]), SE3_MUL(phi[1], phi[1])), SE3_MUL(phi[2], phi[2]));
    const double theta = sqrt(t2);
    double A, B;
    if (theta < kSmallAngle) {
        A = SE3_SUB(1.0, SE3_MUL(t2 / 6.0, SE3_SUB(1.0, t2 / 20.0)));
        B = SE3_SUB(0.5, SE3_MUL(t2 / 24.0, SE3_SUB(1.0, t2 / 30.0)));
    } else {
        double sn, cs;
#ifdef __CUDA_ARCH__
        sincos(theta, &sn, &cs);
#else
        sn = sin(theta); cs = cos(theta);
#endif
        A = sn / theta;
        B = SE3_SUB(1.0, cs) / t2;
    }
    const double K[9] = {0.0, -phi[2], phi[1], phi[2], 0.0, -phi[0], -phi[1], phi[0], 0.0};
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            R[3 * r + c] = r == c ? SE3_ADD(1.0, SE3_MUL(B, SE3_SUB(SE3_MUL(phi[r], phi[r]), t2)))
                                  : SE3_ADD(SE3_MUL(A, K[3 * r + c]), SE3_MUL(B, SE3_MUL(phi[r], phi[c])));
}

// M = M E, every entry ((m0 e0 + m1 e1) + m2 e2)
SE3_HD void mat3_mul_right(double* M, const double* E) {
    double o[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            o[3 * r + c] = SE3_ADD(SE3_ADD(SE3_MUL(M[3 * r], E[c]), SE3_MUL(M[3 * r + 1], E[3 + c])),
                                   SE3_MUL(M[3 * r + 2], E[6 + c]));
    for (int i = 0; i < 9; ++i) M[i] = o[i];
}

// The rate of sample j in the LiDAR frame: R_si (omega_j - bias), each entry ((r0 d0 + r1 d1) + r2 d2)
SE3_HD void gyro_rate(const Gyro& g, const double* smp, long long j, double* w, int stride = kSampleStride) {
    const double* s = smp + (size_t)j * stride;
    const double d[3] = {SE3_SUB(s[1], g.bias[0]), SE3_SUB(s[2], g.bias[1]), SE3_SUB(s[3], g.bias[2])};
    for (int r = 0; r < 3; ++r)
        w[r] = SE3_ADD(SE3_ADD(SE3_MUL(g.R_si[3 * r], d[0]), SE3_MUL(g.R_si[3 * r + 1], d[1])), SE3_MUL(g.R_si[3 * r + 2], d[2]));
}

// The specific force of IMU sample j (kImuStride rows) in the LiDAR frame: R_si (acc_j - acc_bias), gyro_rate's order
SE3_HD void accel_force(const Gyro& g, const double* acc_bias, const double* smp, long long j, double* f) {
    const double* s = smp + (size_t)j * kImuStride;
    const double d[3] = {SE3_SUB(s[4], acc_bias[0]), SE3_SUB(s[5], acc_bias[1]), SE3_SUB(s[6], acc_bias[2])};
    for (int r = 0; r < 3; ++r)
        f[r] = SE3_ADD(SE3_ADD(SE3_MUL(g.R_si[3 * r], d[0]), SE3_MUL(g.R_si[3 * r + 1], d[1])), SE3_MUL(g.R_si[3 * r + 2], d[2]));
}

// M = M Exp(w d): one zero-order-hold piece of d seconds (d < 0: walked backwards)
SE3_HD void gyro_piece(double* M, const double* w, double d) {
    const double phi[3] = {SE3_MUL(w[0], d), SE3_MUL(w[1], d), SE3_MUL(w[2], d)};
    double E[9];
    so3_exp(phi, E);
    mat3_mul_right(M, E);
}

// The last sample j in [0, n) with t_j <= t (strict: t_j < t), or -1
SE3_HD long long gyro_last(const double* smp, long long n, double t, bool strict, int stride = kSampleStride) {
    long long lo = 0, hi = n;           // the first sample past t is in [lo, hi]
    while (lo < hi) {
        const long long mid = lo + (hi - lo) / 2;
        const double tm = smp[(size_t)mid * stride];
        if (strict ? tm < t : tm <= t) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// G(a -> b), a <= b, over n samples: the walk from a to b in time order, M = I then M = M Exp(w_j d_j) for every sample
// interval [t_j, t_{j+1}) clipped to [a, b] with d_j > 0, w_j the rate of sample j (zero-order hold).  Needs a sample at
// or before a and one at or after b (the caller checks); it reads no sample outside them.
//
// With acc_bias (IMU samples, stride kImuStride) the same walk preintegrates the accelerometer into abg[9] = (alpha,
// beta, gamma): over every piece [u, u + d], M the walk's rotation at u (before the piece) and f = R_si (acc_j -
// acc_bias) (accel_force), both held over the piece (a first-order rule), m = M f d (each entry ((m0 f0 + m1 f1) + m2
// f2) d) and alpha += m, beta += m ((b - u) - 0.5 d), gamma += m ((u - a) + 0.5 d), from zero.  G is the gyro's walk,
// bit for bit.
SE3_HD void gyro_rotation(const Gyro& g, const double* smp, long long n, double a, double b, double* G,
                          int stride = kSampleStride, const double* acc_bias = nullptr, double* abg = nullptr) {
    for (int i = 0; i < 9; ++i) G[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (acc_bias)
        for (int i = 0; i < 9; ++i) abg[i] = 0.0;
    long long j = gyro_last(smp, n, a, false, stride);
    double cur = a;
    while (cur < b) {
        const double t1 = smp[(size_t)(j + 1) * stride];
        const double nxt = t1 < b ? t1 : b;
        const double d = SE3_SUB(nxt, cur);
        if (acc_bias) {
            double f[3];
            accel_force(g, acc_bias, smp, j, f);
            const double h = SE3_MUL(0.5, d);
            const double wb = SE3_SUB(SE3_SUB(b, cur), h), wg = SE3_ADD(SE3_SUB(cur, a), h);
            for (int r = 0; r < 3; ++r) {
                const double m = SE3_MUL(SE3_ADD(SE3_ADD(SE3_MUL(G[3 * r], f[0]), SE3_MUL(G[3 * r + 1], f[1])),
                                                 SE3_MUL(G[3 * r + 2], f[2])),
                                         d);
                abg[r] = SE3_ADD(abg[r], m);
                abg[3 + r] = SE3_ADD(abg[3 + r], SE3_MUL(m, wb));
                abg[6 + r] = SE3_ADD(abg[6 + r], SE3_MUL(m, wg));
            }
        }
        double w[3];
        gyro_rate(g, smp, j, w, stride);
        gyro_piece(G, w, d);
        cur = nxt;
        ++j;
    }
}

// The accelerometer's prior translation (dcreg_icp_run_odometry_imu) over [tm_prev, tm], dt = tm - tm_prev, from the
// previous frame's pose (R row-major) and velocity v, gravity grav (world frame) and beta: t_D = dt R^T v + (0.5 dt^2)
// R^T g + beta, every R^T x entry ((R_0r x0 + R_1r x1) + R_2r x2), summed in that order
SE3_HD void imu_translation(const double* R, const double* v, const double* grav, const double* beta, double dt,
                            double* tD) {
    const double c2 = SE3_MUL(0.5, SE3_MUL(dt, dt));
    for (int r = 0; r < 3; ++r) {
        const double rv = SE3_ADD(SE3_ADD(SE3_MUL(R[r], v[0]), SE3_MUL(R[3 + r], v[1])), SE3_MUL(R[6 + r], v[2]));
        const double rg = SE3_ADD(SE3_ADD(SE3_MUL(R[r], grav[0]), SE3_MUL(R[3 + r], grav[1])), SE3_MUL(R[6 + r], grav[2]));
        tD[r] = SE3_ADD(SE3_ADD(SE3_MUL(dt, rv), SE3_MUL(c2, rg)), beta[r]);
    }
}

// A frame's velocity once it has stopped: v = (t - t_prev) / dt + (R_prev gamma) / dt + (0.5 dt) g (world frame), the
// exact kinematic identity for the held inputs, every R gamma entry ((r0 g0 + r1 g1) + r2 g2)
SE3_HD void imu_velocity(const double* R_prev, const double* t_prev, const double* t, const double* grav,
                         const double* gamma, double dt, double* v) {
    const double h = SE3_MUL(0.5, dt);
    for (int r = 0; r < 3; ++r) {
        const double rg = SE3_ADD(SE3_ADD(SE3_MUL(R_prev[3 * r], gamma[0]), SE3_MUL(R_prev[3 * r + 1], gamma[1])),
                                  SE3_MUL(R_prev[3 * r + 2], gamma[2]));
        v[r] = SE3_ADD(SE3_ADD(SE3_SUB(t[r], t_prev[r]) / dt, rg / dt), SE3_MUL(h, grav[r]));
    }
}

// The knots of a sweep [start, end] with mid-sweep tm: tm, and every sample time strictly inside (start, end) other
// than tm.  Returns how many lie before tm (*before) and in all.
SE3_HD int gyro_knot_count(const double* smp, long long n, double start, double tm, double end, int* before,
                           int stride = kSampleStride) {
    const long long lo = gyro_last(smp, n, start, false, stride), m0 = gyro_last(smp, n, tm, true, stride),
                    m1 = gyro_last(smp, n, tm, false, stride), hi = gyro_last(smp, n, end, true, stride);
    *before = (int)(m0 - lo);
    return 1 + (int)(m0 - lo) + (int)(hi - m1);
}

// The knot table of that sweep, ascending in time, kKnotStride doubles per knot: the time, Q = G(tm -> time) as the walk
// from tm to the knot forms it (forwards: M = M Exp(w d); backwards: the same with d < 0, which is G(time -> tm)^T up
// to rounding), the rate after the knot (of the last sample at or before it) and the rate before it (of the last sample
// strictly before it).  Needs a sample at or before start and one at or after end.
SE3_HD void gyro_knots(const Gyro& g, const double* smp, long long n, double start, double tm, double end, double* K,
                       int stride = kSampleStride) {
    int nb = 0;
    gyro_knot_count(smp, n, start, tm, end, &nb, stride);
    double Q[9];
    double* k = K + (size_t)nb * kKnotStride;           // tm's knot
    for (int i = 0; i < 9; ++i) Q[i] = (i % 4 == 0) ? 1.0 : 0.0;
    long long ja = gyro_last(smp, n, tm, false, stride), jb = gyro_last(smp, n, tm, true, stride);
    k[0] = tm;
    for (int i = 0; i < 9; ++i) k[1 + i] = Q[i];
    gyro_rate(g, smp, ja, k + 10, stride);
    gyro_rate(g, smp, jb, k + 13, stride);
    double cur = tm;                                    // backwards: the samples in (start, tm), newest first
    for (int i = nb - 1; i >= 0; --i) {
        const double t = smp[(size_t)jb * stride];
        double* o = K + (size_t)i * kKnotStride;
        gyro_piece(Q, K + (size_t)(i + 1) * kKnotStride + 13, SE3_SUB(t, cur));
        cur = t;
        o[0] = t;
        for (int c = 0; c < 9; ++c) o[1 + c] = Q[c];
        gyro_rate(g, smp, jb, o + 10, stride);
        gyro_rate(g, smp, jb - 1, o + 13, stride);
        --jb;
    }
    for (int i = 0; i < 9; ++i) Q[i] = (i % 4 == 0) ? 1.0 : 0.0;
    cur = tm;                                           // forwards: the samples in (tm, end)
    for (double* o = k + kKnotStride; ja + 1 < n && smp[(size_t)(ja + 1) * stride] < end; o += kKnotStride) {
        const double t = smp[(size_t)(ja + 1) * stride];
        gyro_piece(Q, o - kKnotStride + 10, SE3_SUB(t, cur));
        cur = t;
        ++ja;
        o[0] = t;
        for (int c = 0; c < 9; ++c) o[1 + c] = Q[c];
        gyro_rate(g, smp, ja, o + 10, stride);
        gyro_rate(g, smp, ja - 1, o + 13, stride);
    }
}

// One point of a sweep deskewed to mid-sweep with the gyro: the point's time t = start + tau span; G = G(tm -> t) from
// the sweep's knot table K (nk knots): for t >= tm the last knot k at or before t, G = Q_k Exp(w_after (t - t_k)); for
// t < tm the first knot at or after t, G = Q_k Exp(w_before (t - t_k)) (the walk from tm to t, continued from the knot);
// out = fl32(G p + s tD), s = (t - tm) / (tm - tm_prev), every entry (((g0 x + g1 y) + g2 z) + s tD_r).  p itself, bit
// for bit, when t = tm, when p has a non-finite coordinate, or when the result would have one or equal p.  Returns
// whether it moved the point.
SE3_HD bool deskew_point_gyro(const double* K, int nk, double start, double span, double tm, double tm_prev,
                              const double* tD, float tau, const float* p, float* out) {
    const double t = SE3_ADD(start, SE3_MUL((double)tau, span));
    bool move = t != tm && isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
    float o[3] = {p[0], p[1], p[2]};
    if (move) {
        int lo = 0, hi = nk;            // the first knot past t (t >= tm), or at or past t (t < tm), is in [lo, hi]
        const bool fwd = t >= tm;
        while (lo < hi) {
            const int mid = (lo + hi) / 2;
            const double tk = K[(size_t)mid * kKnotStride];
            if (fwd ? tk <= t : tk < t) lo = mid + 1;
            else hi = mid;
        }
        const double* k = K + (size_t)(fwd ? lo - 1 : lo) * kKnotStride;
        double G[9];
        for (int i = 0; i < 9; ++i) G[i] = k[1 + i];
        gyro_piece(G, k + (fwd ? 10 : 13), SE3_SUB(t, k[0]));
        const double s = SE3_SUB(t, tm) / SE3_SUB(tm, tm_prev);
        const double x = p[0], y = p[1], z = p[2];
        for (int r = 0; r < 3; ++r)
            o[r] = (float)SE3_ADD(SE3_ADD(SE3_ADD(SE3_MUL(G[3 * r], x), SE3_MUL(G[3 * r + 1], y)), SE3_MUL(G[3 * r + 2], z)),
                                  SE3_MUL(s, tD[r]));
        move = isfinite(o[0]) && isfinite(o[1]) && isfinite(o[2]) && !(o[0] == p[0] && o[1] == p[1] && o[2] == p[2]);
    }
    for (int r = 0; r < 3; ++r) out[r] = move ? o[r] : p[r];
    return move;
}

#undef SE3_MUL
#undef SE3_ADD
#undef SE3_SUB

}  // namespace se3

#undef SE3_HD
