// Per-box arithmetic of the anchor k-means (reference genanchors.py), shared by the device kernels (k_anchors.cu) and a CPU build
// (tests/anchors_harness.cu).  Every operation is one IEEE fp64 operation rounded to nearest, in the order Python evaluates the
// reference's expressions, with no fused multiply-add: the device calls the _rn intrinsics, the host build is compiled with
// -ffp-contract=off.  Zero-size boxes give inf / NaN as numpy's float64 scalars do.
#pragma once

namespace yfv2 {
namespace anchors {

constexpr int kMaxK = 16;           // two levels x anchor_num <= 8 (yfv2_plan_create's limit)

__host__ __device__ __forceinline__ double mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ __forceinline__ double div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// IOU(x, centroid) of genanchors.py:17-32 for one centroid: the four branches in the reference's order, >= / <= as written
__host__ __device__ __forceinline__ double similarity(double w, double h, double cw, double ch) {
    if (cw >= w && ch >= h) return div(mul(w, h), mul(cw, ch));
    if (cw >= w && ch <= h) return div(mul(w, ch), add(mul(w, h), mul(sub(cw, w), ch)));
    if (cw <= w && ch >= h) return div(mul(cw, h), add(mul(w, h), mul(cw, sub(ch, h))));
    return div(mul(cw, ch), mul(w, h));
}

// np.argmin(1 - IOU(x, centroids)) (genanchors.py:80,87): the first minimum of d = 1 - s, or the first NaN.  c: k (w, h) pairs.
// The argmin of d, not the argmax of s: below about 1e-16, 1 - s rounds to 1.0 for every centroid and the first one wins.
__host__ __device__ __forceinline__ int assign(double w, double h, const double* c, int k) {
    int best = 0;
    double bd = sub(1.0, similarity(w, h, c[0], c[1]));
    if (bd != bd) return 0;
    for (int j = 1; j < k; ++j) {
        const double d = sub(1.0, similarity(w, h, c[2 * j], c[2 * j + 1]));
        if (d != d) return j;
        if (d < bd) { bd = d; best = j; }
    }
    return best;
}

// Python's builtin max over IOU(x, centroids) (genanchors.py:39): a NaN first element is the result, a later NaN is skipped.
__host__ __device__ __forceinline__ double best_similarity(double w, double h, const double* c, int k) {
    double m = similarity(w, h, c[0], c[1]);
    for (int j = 1; j < k; ++j) {
        const double s = similarity(w, h, c[2 * j], c[2 * j + 1]);
        if (s > m) m = s;
    }
    return m;
}

}  // namespace anchors
}  // namespace yfv2
