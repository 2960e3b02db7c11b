// Host build of the accelerometer preintegration in dcreg_b200/csrc/se3.cuh for tests/test_imu_twin.py: reads an
// IMU's settings, its samples and queries; writes every query's G, (alpha, beta, gamma), prior translation and velocity,
// so the test can hold them against the NumPy twin bit for bit.
// Input (argv[1]): 15 doubles (R_sensor_imu, gyro_bias, accel_bias); int32 n, n x 7 doubles (samples); int32 q, q x 23
// doubles (a, b, R_prev 9, t_prev 3, v_prev 3, t 3, gravity 3).
// Output (argv[2]): q x 24 doubles (G 9, alpha 3, beta 3, gamma 3, t_D 3, v 3).
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../dcreg_b200/csrc/se3.cuh"

template <class T>
static bool read(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: test_imu in.bin out.bin\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    se3::Gyro g;
    double acc_bias[3];
    int32_t n = 0, q = 0;
    if (!read(f, g.R_si, 9) || !read(f, g.bias, 3) || !read(f, acc_bias, 3) || !read(f, &n, 1)) return 2;
    std::vector<double> smp((size_t)n * se3::kImuStride);
    if (!read(f, smp.data(), smp.size()) || !read(f, &q, 1)) return 2;
    std::vector<double> in((size_t)q * 23);
    if (!read(f, in.data(), in.size())) return 2;
    std::fclose(f);
    std::vector<double> out((size_t)q * 24);
    for (int32_t i = 0; i < q; ++i) {
        const double* x = &in[(size_t)i * 23];
        double* o = &out[(size_t)i * 24];
        se3::gyro_rotation(g, smp.data(), n, x[0], x[1], o, se3::kImuStride, acc_bias, o + 9);
        const double dt = x[1] - x[0];
        se3::imu_translation(x + 2, x + 14, x + 20, o + 12, dt, o + 18);
        se3::imu_velocity(x + 2, x + 11, x + 17, x + 20, o + 15, dt, o + 21);
    }
    FILE* o = std::fopen(argv[2], "wb");
    if (!o) return 2;
    std::fwrite(out.data(), 8, out.size(), o);
    std::fclose(o);
    return 0;
}
