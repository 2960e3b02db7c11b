// Host build of dcreg_b200/csrc/se3.cuh for tests/test_se3_host.py: reads motions and points, writes se3_log of every
// motion and se3::deskew_point of every point, so the test can hold them against the NumPy twin.
// Input (argv[1]): int32 n_mats, n_mats x 16 doubles (row-major 4x4); int32 n_pts, n_pts x (int32 motion, float tau,
// 3 floats).  Output (argv[2]): n_mats x 6 doubles, then n_pts x 3 floats.
#include <cstdio>
#include <cstdint>
#include <vector>

#include "../dcreg_b200/csrc/se3.cuh"

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: test_se3 in.bin out.bin\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    int32_t n_mats = 0, n_pts = 0;
    if (std::fread(&n_mats, 4, 1, f) != 1) return 2;
    std::vector<double> D((size_t)n_mats * 16);
    if (std::fread(D.data(), 8, D.size(), f) != D.size() || std::fread(&n_pts, 4, 1, f) != 1) return 2;
    struct Pt { int32_t m; float tau, p[3]; };
    std::vector<Pt> P((size_t)n_pts);
    if (std::fread(P.data(), sizeof(Pt), P.size(), f) != P.size()) return 2;
    std::fclose(f);
    std::vector<double> xi((size_t)n_mats * 6);
    for (int32_t m = 0; m < n_mats; ++m) {
        const double* T = &D[(size_t)m * 16];
        const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, t[3] = {T[3], T[7], T[11]};
        se3::se3_log(R, t, &xi[(size_t)m * 6]);
    }
    std::vector<float> out((size_t)n_pts * 3);
    for (int32_t i = 0; i < n_pts; ++i) se3::deskew_point(&xi[(size_t)P[i].m * 6], P[i].tau, P[i].p, &out[(size_t)i * 3]);
    FILE* g = std::fopen(argv[2], "wb");
    if (!g) return 2;
    std::fwrite(xi.data(), 8, xi.size(), g);
    std::fwrite(out.data(), 4, out.size(), g);
    std::fclose(g);
    std::printf("SE3_HOST_OK %d motions %d points\n", n_mats, n_pts);
    return 0;
}
