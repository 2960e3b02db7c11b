// Device program for tests/test_gpu_motion_math.py: the odometry's motion math (dcreg_b200/csrc/se3.cuh,
// adaptive_threshold.cuh, included unchanged) on records written by the test, one kernel launch per section and one
// thread per record, built with the library's nvcc flags (sm_90a, --fmad=true) so the compiler treats the headers as
// it does in the library.  Every record is evaluated twice, in the kernel and on the host in this binary, and both
// results are written: device against host on identical inputs.
//
// Input (argv[1]): sections, each int32 family, int32 count, then its payload:
//   1 LOG          count x (R 9, t 3 doubles)                        -> xi 6 doubles
//   2 EXP          count x (xi 6, s, p 3 doubles)                    -> q 3 doubles (se3_exp_apply)
//   3 DESKEW       count x DeskewIn                                  -> PointOut (deskew_point)
//   4 SO3          count x (phi 3 doubles)                           -> R 9 doubles
//   5 SAMPLES      R_si 9, bias 3 doubles, count x (t, wx, wy, wz)   -> nothing (the gyro sections that follow read them)
//   6 GYRO_ROT     count x (a, b doubles)                            -> G 9 doubles (gyro_rotation)
//   7 KNOTS        count x (start, span, tm doubles), end = start + span
//                  -> int32 (count, before) per sweep (gyro_knot_count), then the knot tables (gyro_knots) at the host's
//                     offsets; a sweep whose device count differs from the host's gets no device table
//   8 GYRO_DESKEW  count x GyroDeskewIn (a sweep of the last KNOTS)  -> PointOut (deskew_point_gyro)
//   9 ANGLE        count x (R 9 doubles)                             -> double (rotation_angle)
//  10 MODEL_ERROR  count x (D 16, max_range doubles)                 -> double (model_error)
//  11 FOLD         count x FoldIn                                    -> adaptive::State (fold)
//  12 RADIUS       count x RadiusIn                                  -> double (radius)
//  13 CHAIN        initial_threshold, min_motion, max_range, ceiling doubles, int32 sequences, int32 offsets
//                  [sequences + 1], then count x (D 16 doubles); one thread per sequence, state (0, 0): every frame's
//                  radius, then its error folded in (odom_threshold_kernel's order)  -> double per frame
// Output (argv[2]): per section, every output array as the device's bytes then the host's.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <deque>
#include <vector>

#include "../dcreg_b200/csrc/se3.cuh"
#include "../dcreg_b200/csrc/adaptive_threshold.cuh"

#define HD __host__ __device__

enum Family { kLog = 1, kExp, kDeskew, kSo3, kSamples, kGyroRot, kKnots, kGyroDeskew, kAngle, kModelError, kFold,
              kRadius, kChain };

struct DeskewIn { double xi[6]; float tau; float p[3]; };
struct PointOut { float o[3]; int32_t moved; };
struct GyroDeskewIn { double tm_prev; double tD[3]; int32_t sweep; float tau; float p[3]; int32_t pad; };
struct FoldIn { double sse; long long n; double e, min_motion; };
struct RadiusIn { double sse; long long n; double initial_threshold, ceiling; };

struct LogF {
    const double* in; double* out;
    HD void operator()(int i) const { se3::se3_log(in + 12 * i, in + 12 * i + 9, out + 6 * i); }
};
struct ExpF {
    const double* in; double* out;
    HD void operator()(int i) const { se3::se3_exp_apply(in + 10 * i, in[10 * i + 6], in + 10 * i + 7, out + 3 * i); }
};
struct DeskewF {
    const DeskewIn* in; PointOut* out;
    HD void operator()(int i) const { out[i].moved = se3::deskew_point(in[i].xi, in[i].tau, in[i].p, out[i].o); }
};
struct So3F {
    const double* in; double* out;
    HD void operator()(int i) const { se3::so3_exp(in + 3 * i, out + 9 * i); }
};
struct GyroRotF {
    se3::Gyro g; const double* smp; long long n; const double* in; double* out;
    HD void operator()(int i) const { se3::gyro_rotation(g, smp, n, in[2 * i], in[2 * i + 1], out + 9 * i); }
};
struct KnotsF {
    se3::Gyro g; const double* smp; long long n; const double* in; const long long* off; int32_t* cnt; double* K;
    HD void operator()(int i) const {
        const double start = in[3 * i], span = in[3 * i + 1], tm = in[3 * i + 2], end = start + span;
        int nb = 0;
        const int c = se3::gyro_knot_count(smp, n, start, tm, end, &nb);
        cnt[2 * i] = c;
        cnt[2 * i + 1] = nb;
        if (c == off[i + 1] - off[i]) se3::gyro_knots(g, smp, n, start, tm, end, K + off[i] * se3::kKnotStride);
    }
};
struct GyroDeskewF {
    const double* sweeps; const long long* off; const double* K; const GyroDeskewIn* in; PointOut* out;
    HD void operator()(int i) const {
        const GyroDeskewIn& r = in[i];
        const double* s = sweeps + 3 * r.sweep;
        out[i].moved = se3::deskew_point_gyro(K + off[r.sweep] * se3::kKnotStride, (int)(off[r.sweep + 1] - off[r.sweep]),
                                              s[0], s[1], s[2], r.tm_prev, r.tD, r.tau, r.p, out[i].o);
    }
};
struct AngleF {
    const double* in; double* out;
    HD void operator()(int i) const { out[i] = adaptive::rotation_angle(in + 9 * i); }
};
struct ModelErrorF {
    const double* in; double* out;
    HD void operator()(int i) const { out[i] = adaptive::model_error(in + 17 * i, in[17 * i + 16]); }
};
struct FoldF {
    const FoldIn* in; adaptive::State* out;
    HD void operator()(int i) const {
        adaptive::State s{in[i].sse, in[i].n};
        adaptive::fold(&s, in[i].e, in[i].min_motion);
        out[i] = s;
    }
};
struct RadiusF {
    const RadiusIn* in; double* out;
    HD void operator()(int i) const {
        out[i] = adaptive::radius(adaptive::State{in[i].sse, in[i].n}, in[i].initial_threshold, in[i].ceiling);
    }
};
struct ChainF {
    const double* set; const int32_t* off; const double* D; double* out;
    HD void operator()(int i) const {
        adaptive::State x{0.0, 0};
        for (int k = off[i]; k < off[i + 1]; ++k) {
            out[k] = adaptive::radius(x, set[0], set[3]);
            adaptive::fold(&x, adaptive::model_error(D + 16 * (size_t)k, set[2]), set[1]);
        }
    }
};

template <class F>
__global__ void each(F f, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) f(i);
}

static bool ok(cudaError_t e, const char* what) {
    if (e != cudaSuccess) std::fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e));
    return e == cudaSuccess;
}
#define CK(x) do { if (!ok((x), #x)) return 1; } while (0)

// one output array: the device's copy and the host's
struct Out { void* dev; std::vector<char> host; };

struct Reader {
    FILE* f;
    template <class T>
    bool take(std::vector<T>& v, size_t n) { v.resize(n); return n == 0 || std::fread(v.data(), sizeof(T), n, f) == n; }
};

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: test_motion_device in.bin out.bin\n"); return 2; }
    Reader rd{std::fopen(argv[1], "rb")};
    if (!rd.f) return 2;
    std::vector<void*> owned;
    auto dev_copy = [&](const void* h, size_t bytes) -> void* {
        void* d = nullptr;
        if (!ok(cudaMalloc(&d, bytes ? bytes : 8), "cudaMalloc")) d = nullptr;
        else if (bytes && !ok(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice), "cudaMemcpy")) d = nullptr;
        owned.push_back(d);                 // (a null entry ends the program after the section)
        return d;
    };
    std::deque<Out> outs;                   // (references stay valid as it grows)
    auto out = [&](size_t bytes) -> Out& {
        void* d = nullptr;
        if (!ok(cudaMalloc(&d, bytes ? bytes : 8), "cudaMalloc")) d = nullptr;
        else if (!ok(cudaMemset(d, 0xff, bytes ? bytes : 8), "cudaMemset")) d = nullptr;   // unwritten: all ones
        owned.push_back(d);
        outs.push_back(Out{d, std::vector<char>(bytes)});
        return outs.back();
    };
    auto launch = [&](auto fd, auto fh, int n) {
        if (n > 0) each<<<(n + 127) / 128, 128>>>(fd, n);
        for (int i = 0; i < n; ++i) fh(i);
    };
    // the gyro state the gyro sections read: settings, samples, and the last KNOTS section's sweeps and tables
    se3::Gyro g{};
    std::vector<double> smp, sweeps, K;
    std::vector<long long> off(1, 0);
    const double *d_smp = nullptr, *d_sweeps = nullptr, *d_K = nullptr;
    const long long* d_off = nullptr;
    int32_t head[2];
    while (std::fread(head, 4, 2, rd.f) == 2) {
        const int fam = head[0], n = head[1];
        std::vector<double> in;
        switch (fam) {
        case kLog: {
            if (!rd.take(in, 12 * (size_t)n)) return 2;
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 48);
            launch(LogF{d, (double*)o.dev}, LogF{in.data(), (double*)o.host.data()}, n);
            break;
        }
        case kExp: {
            if (!rd.take(in, 10 * (size_t)n)) return 2;
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 24);
            launch(ExpF{d, (double*)o.dev}, ExpF{in.data(), (double*)o.host.data()}, n);
            break;
        }
        case kDeskew: {
            std::vector<DeskewIn> r;
            if (!rd.take(r, (size_t)n)) return 2;
            const DeskewIn* d = (const DeskewIn*)dev_copy(r.data(), r.size() * sizeof(DeskewIn));
            Out& o = out((size_t)n * sizeof(PointOut));
            launch(DeskewF{d, (PointOut*)o.dev}, DeskewF{r.data(), (PointOut*)o.host.data()}, n);
            break;
        }
        case kSo3: {
            if (!rd.take(in, 3 * (size_t)n)) return 2;
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 72);
            launch(So3F{d, (double*)o.dev}, So3F{in.data(), (double*)o.host.data()}, n);
            break;
        }
        case kSamples: {
            if (std::fread(g.R_si, 8, 9, rd.f) != 9 || std::fread(g.bias, 8, 3, rd.f) != 3) return 2;
            if (!rd.take(smp, 4 * (size_t)n)) return 2;
            d_smp = (const double*)dev_copy(smp.data(), smp.size() * 8);
            break;
        }
        case kGyroRot: {
            if (!rd.take(in, 2 * (size_t)n)) return 2;
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 72);
            const long long ns = (long long)smp.size() / 4;
            launch(GyroRotF{g, d_smp, ns, d, (double*)o.dev}, GyroRotF{g, smp.data(), ns, in.data(), (double*)o.host.data()},
                   n);
            break;
        }
        case kKnots: {
            if (!rd.take(sweeps, 3 * (size_t)n)) return 2;
            const long long ns = (long long)smp.size() / 4;
            off.assign(1, 0);
            for (int i = 0; i < n; ++i) {
                int nb = 0;
                const double* s = &sweeps[3 * (size_t)i];
                off.push_back(off.back() + se3::gyro_knot_count(smp.data(), ns, s[0], s[2], s[0] + s[1], &nb));
            }
            d_sweeps = (const double*)dev_copy(sweeps.data(), sweeps.size() * 8);
            d_off = (const long long*)dev_copy(off.data(), off.size() * 8);
            Out& c = out((size_t)n * 8);
            Out& k = out((size_t)off.back() * se3::kKnotStride * 8);
            d_K = (const double*)k.dev;
            launch(KnotsF{g, d_smp, ns, d_sweeps, d_off, (int32_t*)c.dev, (double*)k.dev},
                   KnotsF{g, smp.data(), ns, sweeps.data(), off.data(), (int32_t*)c.host.data(), (double*)k.host.data()}, n);
            K.assign((const double*)k.host.data(), (const double*)k.host.data() + off.back() * se3::kKnotStride);
            break;
        }
        case kGyroDeskew: {
            std::vector<GyroDeskewIn> r;
            if (!rd.take(r, (size_t)n)) return 2;
            const GyroDeskewIn* d = (const GyroDeskewIn*)dev_copy(r.data(), r.size() * sizeof(GyroDeskewIn));
            Out& o = out((size_t)n * sizeof(PointOut));
            launch(GyroDeskewF{d_sweeps, d_off, d_K, d, (PointOut*)o.dev},
                   GyroDeskewF{sweeps.data(), off.data(), K.data(), r.data(), (PointOut*)o.host.data()}, n);
            break;
        }
        case kAngle: {
            if (!rd.take(in, 9 * (size_t)n)) return 2;
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 8);
            launch(AngleF{d, (double*)o.dev}, AngleF{in.data(), (double*)o.host.data()}, n);
            break;
        }
        case kModelError: {
            if (!rd.take(in, 17 * (size_t)n)) return 2;
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 8);
            launch(ModelErrorF{d, (double*)o.dev}, ModelErrorF{in.data(), (double*)o.host.data()}, n);
            break;
        }
        case kFold: {
            std::vector<FoldIn> r;
            if (!rd.take(r, (size_t)n)) return 2;
            const FoldIn* d = (const FoldIn*)dev_copy(r.data(), r.size() * sizeof(FoldIn));
            Out& o = out((size_t)n * sizeof(adaptive::State));
            launch(FoldF{d, (adaptive::State*)o.dev}, FoldF{r.data(), (adaptive::State*)o.host.data()}, n);
            break;
        }
        case kRadius: {
            std::vector<RadiusIn> r;
            if (!rd.take(r, (size_t)n)) return 2;
            const RadiusIn* d = (const RadiusIn*)dev_copy(r.data(), r.size() * sizeof(RadiusIn));
            Out& o = out((size_t)n * 8);
            launch(RadiusF{d, (double*)o.dev}, RadiusF{r.data(), (double*)o.host.data()}, n);
            break;
        }
        case kChain: {
            std::vector<double> set;
            std::vector<int32_t> seqs, offs;
            if (!rd.take(set, 4) || !rd.take(seqs, 1) || !rd.take(offs, (size_t)seqs[0] + 1) || !rd.take(in, 16 * (size_t)n))
                return 2;
            const double* d_set = (const double*)dev_copy(set.data(), 32);
            const int32_t* d_offs = (const int32_t*)dev_copy(offs.data(), offs.size() * 4);
            const double* d = (const double*)dev_copy(in.data(), in.size() * 8);
            Out& o = out((size_t)n * 8);
            launch(ChainF{d_set, d_offs, d, (double*)o.dev}, ChainF{set.data(), offs.data(), in.data(), (double*)o.host.data()},
                   seqs[0]);
            break;
        }
        default:
            std::fprintf(stderr, "unknown family %d\n", fam);
            return 2;
        }
        for (void* p : owned)
            if (!p) return 1;
    }
    std::fclose(rd.f);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    FILE* o = std::fopen(argv[2], "wb");
    if (!o) return 2;
    std::vector<char> buf;
    for (const Out& x : outs) {
        buf.resize(x.host.size());
        if (!buf.empty()) CK(cudaMemcpy(buf.data(), x.dev, buf.size(), cudaMemcpyDeviceToHost));
        std::fwrite(buf.data(), 1, buf.size(), o);
        std::fwrite(x.host.data(), 1, x.host.size(), o);
    }
    std::fclose(o);
    for (void* p : owned) cudaFree(p);
    std::printf("MOTION_DEVICE_OK %zu arrays\n", outs.size());
    return 0;
}
