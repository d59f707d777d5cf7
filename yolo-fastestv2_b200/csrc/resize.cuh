// cv2.resize(INTER_LINEAR)'s per-pixel arithmetic (k_resize.cu states it): the coefficients of one target index and one output
// pixel computed over any source type with a fetch(c0, c1, p0, p1) of two pixels of a row.  k_resize.cu's kernels and k_jpeg.cu's
// fused decode + resize (JpegSource) share it.
#pragma once
#include <stdint.h>

namespace yfv2 {
namespace {

__device__ __forceinline__ int sat_u8(int v) { return min(max(v, 0), 255); }

// fractional source coordinate of target index d: returns the fraction, s = its floor
__device__ __forceinline__ float src_coord(int d, int n, int m, int& s) {
    const double scale = (double)n / (double)m;                                          // IEEE division
    const float f = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));   // no FMA contraction
    const float fl = floorf(f);
    s = (int)fl;
    return __fsub_rn(f, fl);
}
__device__ __forceinline__ int weight0(float f) { return __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f)); }
__device__ __forceinline__ int weight1(float f) { return __float2int_rn(__fmul_rn(f, 2048.f)); }

// Output pixel (x, y) of the resize of fr (w x h source pixels) to W x H: B, G, R in v.  resize_kernel's arithmetic, for the
// augmentation's nested resize and the fused JPEG decode (resize_kernel keeps its own copy of these lines so that its code stays
// as it was).
template <class Src>
__device__ __forceinline__ void resize_pixel(const typename Src::Desc& fr, int w, int h, int x, int y, int W, int H, int (&v)[3]) {
    int sx;
    float fx = src_coord(x, w, W, sx);
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= w - 1) { fx = 0.f; sx = w - 1; }
    const int a0 = weight0(fx), a1 = weight1(fx);
    const int x1 = min(sx + 1, w - 1);

    int sy;
    const float fy = src_coord(y, h, H, sy);
    const int b0 = weight0(fy), b1 = weight1(fy);
    const int r0 = min(max(sy, 0), h - 1), r1 = min(max(sy + 1, 0), h - 1);

    const Src row0(fr, r0), row1(fr, r1);
    int p00[3], p01[3], p10[3], p11[3];          // [row][column] source pixels, B G R
    row0.fetch(sx, x1, p00, p01);
    row1.fetch(sx, x1, p10, p11);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int S0 = p00[c] * a0 + p01[c] * a1;
        const int S1 = p10[c] * a0 + p11[c] * a1;
        v[c] = sat_u8(((((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16) + 2) >> 2);
    }
}

}  // namespace
}  // namespace yfv2
