// adaptive_threshold.cuh - the adaptive search radius of scan-to-map odometry (dcreg_icp_run_odometry_adaptive), KISS-ICP's
// AdaptiveThreshold, host and device.
//
// Per sequence the state is (sse, n), the sum of squares and the count of the motion-model errors seen so far.  With
// sigma = initial_threshold before any sample and sqrt(sse / n) after, a frame registers with the search radius
// min(3 sigma, ceiling).  After a frame has stopped, D = inv(T_prior) T_out (constant_velocity_increment's rule) is how
// far registration corrected the prediction; its size in metres is e = 2 max_range sin(theta / 2) + |t_D|, theta the
// rotation angle of R_D, and e is a sample when it is finite and above min_motion.  Everything is FP64 with one
// rounding per operation; dcreg_b200.api.adaptive_threshold_* is the NumPy twin (the radius bit for bit, the error up to
// the last bits of sin and atan2).  Plain C++ as well, so tools/test_adaptive_threshold.cpp checks the host build
// against the twin (tests/test_adaptive_threshold_twin.py).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define ADT_HD __host__ __device__ __forceinline__
#else
#define ADT_HD inline
#endif
#ifdef __CUDA_ARCH__
#define ADT_MUL(x, y) __dmul_rn(x, y)
#define ADT_ADD(x, y) __dadd_rn(x, y)
#else
#define ADT_MUL(x, y) ((x) * (y))
#define ADT_ADD(x, y) ((x) + (y))
#endif

namespace adaptive {

struct Settings { double initial_threshold, min_motion, max_range; };
struct State { double sse; long long n; };

// the radius a sequence in state s registers its next frame with: sqrt, the division, 3 sigma and the min are single
// IEEE operations, so host and device agree bit for bit
ADT_HD double radius(State s, double initial_threshold, double ceiling) {
    const double sigma = s.n == 0 ? initial_threshold : sqrt(s.sse / (double)s.n);
    const double r = ADT_MUL(3.0, sigma);
    return r < ceiling ? r : ceiling;
}

// The rotation angle of R (row-major 3x3) by se3::se3_log's route: the quaternion by Shepperd's rule (w >= 0), then
// theta = 2 atan2(|v|, w), with its series below |v| = 1e-10.  NaN when an entry is not finite.
ADT_HD double rotation_angle(const double* R) {
    for (int i = 0; i < 9; ++i)
        if (!isfinite(R[i])) return NAN;
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
    if (w < 0.0) w = -w;
    const double n2 = ADT_ADD(ADT_ADD(ADT_MUL(v[0], v[0]), ADT_MUL(v[1], v[1])), ADT_MUL(v[2], v[2]));
    const double n = sqrt(n2);
    if (n2 < 1e-10 * 1e-10) return ADT_MUL(2.0 / w - (2.0 / 3.0) * n2 / ((w * w) * w), n);
    return 2.0 * atan2(n, w);
}

// e of the correction D (row-major 4x4): 2 max_range sin(theta / 2) + |t_D|
ADT_HD double model_error(const double* D, double max_range) {
    const double R[9] = {D[0], D[1], D[2], D[4], D[5], D[6], D[8], D[9], D[10]};
    const double theta = rotation_angle(R);
    const double t2 = ADT_ADD(ADT_ADD(ADT_MUL(D[3], D[3]), ADT_MUL(D[7], D[7])), ADT_MUL(D[11], D[11]));
    return ADT_ADD(ADT_MUL(ADT_MUL(2.0, max_range), sin(ADT_MUL(0.5, theta))), sqrt(t2));
}

// one frame's error folded into its sequence's state
ADT_HD void fold(State* s, double e, double min_motion) {
    if (isfinite(e) && e > min_motion) {
        s->sse = ADT_ADD(s->sse, ADT_MUL(e, e));
        s->n += 1;
    }
}

}  // namespace adaptive

#undef ADT_HD
#undef ADT_MUL
#undef ADT_ADD
