// Host build of dcreg_b200/csrc/adaptive_threshold.cuh for tests/test_adaptive_threshold_twin.py: one sequence's
// corrections folded one after another, so the test can hold errors, states and radii against the NumPy twin.
// Input (argv[1]): 4 doubles (initial_threshold, min_motion, max_range, ceiling); int32 n; n x 16 doubles, the
// corrections D = inv(T_prior) T_out (row-major 4x4).  Output (argv[2]): n x 4 doubles: e of D, then sse, n and the
// next radius after folding it.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../dcreg_b200/csrc/adaptive_threshold.cuh"

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: test_adaptive_threshold in.bin out.bin\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    double set[4];
    int32_t n = 0;
    if (std::fread(set, 8, 4, f) != 4 || std::fread(&n, 4, 1, f) != 1) return 2;
    std::vector<double> D((size_t)n * 16);
    if (std::fread(D.data(), 8, D.size(), f) != D.size()) return 2;
    std::fclose(f);
    std::vector<double> out((size_t)n * 4);
    adaptive::State s{0.0, 0};
    for (int32_t k = 0; k < n; ++k) {
        const double e = adaptive::model_error(&D[(size_t)k * 16], set[2]);
        adaptive::fold(&s, e, set[1]);
        out[(size_t)k * 4] = e; out[(size_t)k * 4 + 1] = s.sse; out[(size_t)k * 4 + 2] = (double)s.n;
        out[(size_t)k * 4 + 3] = adaptive::radius(s, set[0], set[3]);
    }
    FILE* g = std::fopen(argv[2], "wb");
    if (!g) return 2;
    std::fwrite(out.data(), 8, out.size(), g);
    std::fclose(g);
    std::printf("ADAPTIVE_HOST_OK %d corrections\n", n);
    return 0;
}
