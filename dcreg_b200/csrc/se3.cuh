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

}  // namespace se3

#undef SE3_HD
