// Host build of the gyroscope rotation in dcreg_b200/csrc/se3.cuh for tests/test_gyro_twin.py: reads a gyro's settings,
// its samples, rotation queries, sweeps and points; writes G(a -> b) of every query, every sweep's knot table and every
// point deskewed by se3::deskew_point_gyro, so the test can hold them against the NumPy twin bit for bit.
// Input (argv[1]): 12 doubles (R_sensor_imu, bias); int32 n, n x 4 doubles (samples); int32 q, q x 2 doubles (a, b);
// int32 w, w x 6 doubles (start, span, tm_prev, tD); int32 m, m x (int32 sweep, float tau, 3 floats).
// Output (argv[2]): q x 9 doubles; w int32 knot counts, then their knots (16 doubles each); m x 3 floats.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../dcreg_b200/csrc/se3.cuh"

template <class T>
static bool read(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: test_gyro in.bin out.bin\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    se3::Gyro g;
    int32_t n = 0, q = 0, w = 0, m = 0;
    if (!read(f, g.R_si, 9) || !read(f, g.bias, 3) || !read(f, &n, 1)) return 2;
    std::vector<double> smp((size_t)n * 4);
    if (!read(f, smp.data(), smp.size()) || !read(f, &q, 1)) return 2;
    std::vector<double> ab((size_t)q * 2);
    if (!read(f, ab.data(), ab.size()) || !read(f, &w, 1)) return 2;
    std::vector<double> sw((size_t)w * 6);
    if (!read(f, sw.data(), sw.size()) || !read(f, &m, 1)) return 2;
    struct Pt { int32_t sweep; float tau, p[3]; };
    std::vector<Pt> P((size_t)m);
    if (!read(f, P.data(), P.size())) return 2;
    std::fclose(f);
    std::vector<double> G((size_t)q * 9);
    for (int32_t i = 0; i < q; ++i) se3::gyro_rotation(g, smp.data(), n, ab[2 * i], ab[2 * i + 1], &G[(size_t)i * 9]);
    std::vector<int32_t> count((size_t)w);
    std::vector<size_t> at((size_t)w + 1, 0);
    for (int32_t i = 0; i < w; ++i) {
        const double* s = &sw[(size_t)i * 6];
        int nb = 0;
        count[(size_t)i] = se3::gyro_knot_count(smp.data(), n, s[0], s[0] + 0.5 * s[1], s[0] + s[1], &nb);
        at[(size_t)i + 1] = at[(size_t)i] + (size_t)count[(size_t)i];
    }
    std::vector<double> K(at[(size_t)w] * se3::kKnotStride);
    for (int32_t i = 0; i < w; ++i) {
        const double* s = &sw[(size_t)i * 6];
        se3::gyro_knots(g, smp.data(), n, s[0], s[0] + 0.5 * s[1], s[0] + s[1], &K[at[(size_t)i] * se3::kKnotStride]);
    }
    std::vector<float> out((size_t)m * 3);
    for (int32_t i = 0; i < m; ++i) {
        const size_t b = (size_t)P[(size_t)i].sweep;
        const double* s = &sw[b * 6];
        se3::deskew_point_gyro(&K[at[b] * se3::kKnotStride], count[b], s[0], s[1], s[0] + 0.5 * s[1], s[2], s + 3,
                               P[(size_t)i].tau, P[(size_t)i].p, &out[(size_t)i * 3]);
    }
    FILE* o = std::fopen(argv[2], "wb");
    if (!o) return 2;
    std::fwrite(G.data(), 8, G.size(), o);
    std::fwrite(count.data(), 4, count.size(), o);
    std::fwrite(K.data(), 8, K.size(), o);
    std::fwrite(out.data(), 4, out.size(), o);
    std::fclose(o);
    std::printf("GYRO_HOST_OK %d queries %d sweeps %d points\n", q, w, m);
    return 0;
}
