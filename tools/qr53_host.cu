// dla::colpiv_qr_solve<5,3>(A, b = -1) as host code (no GPU needed), for the NumPy restatement in
// oracle/dcreg_oracle_rows.py:qr53.  Reads K row-major 5x3 systems (K x 15 doubles) from argv[1] and writes the K
// solutions (K x 3 doubles) to argv[2].   nvcc -O2 -o qr53_host tools/qr53_host.cu
#include <cstdio>
#include <vector>
#include "../dcreg_b200/csrc/small_la.cuh"

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: qr53_host systems.bin solutions.bin\n"); return 2; }
    std::FILE* in = std::fopen(argv[1], "rb");
    if (!in) { std::perror(argv[1]); return 1; }
    std::vector<double> a;
    double buf[15];
    while (std::fread(buf, sizeof(double), 15, in) == 15) a.insert(a.end(), buf, buf + 15);
    std::fclose(in);
    const size_t K = a.size() / 15;
    std::vector<double> x(3 * K);
    for (size_t k = 0; k < K; ++k) {
        double A[15], b[5] = {-1.0, -1.0, -1.0, -1.0, -1.0};
        for (int i = 0; i < 15; ++i) A[i] = a[15 * k + i];
        dla::colpiv_qr_solve<5, 3>(A, b, &x[3 * k]);
    }
    std::FILE* out = std::fopen(argv[2], "wb");
    if (!out || std::fwrite(x.data(), sizeof(double), x.size(), out) != x.size()) { std::perror(argv[2]); return 1; }
    std::fclose(out);
    std::printf("%zu systems\n", K);
    return 0;
}
