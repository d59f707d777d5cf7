// CPU build of the anchor k-means' per-box arithmetic (tests/test_anchors_cpu.py compiles it with nvcc, -ffp-contract=off): the
// same csrc/anchors.cuh functions the device kernels call.
//   anchors_harness sim IN OUT             IN: M x (w, h, c_w, c_h) fp64 -> OUT: M similarities fp64
//   anchors_harness assign K IN OUT_A OUT_M IN: M x (w, h, then K centroids (c_w, c_h)) fp64 -> OUT_A: M argmin int32,
//                                          OUT_M: M builtin-max similarities fp64
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../yolo-fastestv2_b200/csrc/anchors.cuh"

static std::vector<double> read_all(const char* path) {
    std::vector<double> v;
    FILE* f = fopen(path, "rb");
    if (!f) exit(2);
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    v.resize(n / sizeof(double));
    if (fread(v.data(), sizeof(double), v.size(), f) != v.size()) exit(2);
    fclose(f);
    return v;
}

template <typename T>
static void write_all(const char* path, const std::vector<T>& v) {
    FILE* f = fopen(path, "wb");
    if (!f || fwrite(v.data(), sizeof(T), v.size(), f) != v.size()) exit(2);
    fclose(f);
}

int main(int argc, char** argv) {
    using namespace yfv2::anchors;
    if (argc == 4 && !strcmp(argv[1], "sim")) {
        const std::vector<double> in = read_all(argv[2]);
        std::vector<double> out(in.size() / 4);
        for (size_t i = 0; i < out.size(); ++i) out[i] = similarity(in[4 * i], in[4 * i + 1], in[4 * i + 2], in[4 * i + 3]);
        write_all(argv[3], out);
        return 0;
    }
    if (argc == 6 && !strcmp(argv[1], "assign")) {
        const int k = atoi(argv[2]);
        if (k < 1 || k > kMaxK) return 2;
        const std::vector<double> in = read_all(argv[3]);
        const size_t rec = 2 + 2 * (size_t)k, M = in.size() / rec;
        std::vector<int> a(M);
        std::vector<double> m(M);
        for (size_t i = 0; i < M; ++i) {
            const double* r = in.data() + i * rec;
            a[i] = assign(r[0], r[1], r + 2, k);
            m[i] = best_similarity(r[0], r[1], r + 2, k);
        }
        write_all(argv[4], a);
        write_all(argv[5], m);
        return 0;
    }
    fprintf(stderr, "usage: anchors_harness sim IN OUT | assign K IN OUT_A OUT_M\n");
    return 2;
}
