// Raw-frame resize: cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR) on packed HWC uint8 BGR frames (the host step of
// test.py:35 and utils/datasets.py:107), written straight into the [N,3,H,W] planar uint8 batch yfv2_forward_u8 consumes
// (test.py:36-37: res_img.transpose(2, 0, 1)).  Bit-identical to OpenCV's x86 8-bit path, all integer after the coefficients:
//   coefficients per axis: f = fl32((d + 0.5) * (n / m) - 0.5) (product and difference rounded in double), s = floor(f),
//     f = fl32(f - s); weights rint(fl32(1 - f) * 2048), rint(f * 2048).  Along x, s < 0 -> (0, 0) then s >= w - 1 -> (w - 1, 0);
//     along y the weights keep the unclamped fraction and the two rows are clamped.
//   horizontal: S = src[sx] * a0 + src[min(sx + 1, w - 1)] * a1 (int32, per channel)
//   vertical:   out = sat_u8((((S0 >> 4) * b0 >> 16) + ((S1 >> 4) * b1 >> 16) + 2) >> 2)
// oracle/resize.py restates the same arithmetic in numpy.  One thread per output pixel (all three channels); a warp covers 32
// consecutive x of one row, so each plane store of a warp is one contiguous 32-byte run.  The coefficients are recomputed per
// thread (four double operations): cheaper than a table round trip, and the call needs no workspace.
#include "common.cuh"

namespace yfv2 {
namespace {

constexpr int kResizeChunk = 128;        // frames per launch: their descriptors travel as kernel parameters (3 KB)
constexpr int kResizeBx = 64, kResizeBy = 4;
constexpr int kResizeMaxSide = 32768;

struct ResizeChunk {
    yfv2_frame src[kResizeChunk];
    uint8_t* dst;                        // [n][3][H][W] of the chunk's first frame
    int H, W;
};

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

__global__ void __launch_bounds__(kResizeBx * kResizeBy)
resize_bgr_kernel(const __grid_constant__ ResizeChunk a) {
    const int x = blockIdx.x * kResizeBx + threadIdx.x;
    const int y = blockIdx.y * kResizeBy + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const yfv2_frame fr = a.src[blockIdx.z];
    const int w = fr.w, h = fr.h;

    int sx;
    float fx = src_coord(x, w, a.W, sx);
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= w - 1) { fx = 0.f; sx = w - 1; }
    const int a0 = weight0(fx), a1 = weight1(fx);
    const int x1 = min(sx + 1, w - 1);

    int sy;
    const float fy = src_coord(y, h, a.H, sy);
    const int b0 = weight0(fy), b1 = weight1(fy);
    const int r0 = min(max(sy, 0), h - 1), r1 = min(max(sy + 1, 0), h - 1);

    const uint8_t* row0 = fr.data + (long long)r0 * fr.pitch;
    const uint8_t* row1 = fr.data + (long long)r1 * fr.pitch;
    const size_t plane = (size_t)a.H * a.W;
    uint8_t* out = a.dst + (size_t)blockIdx.z * 3 * plane + (size_t)y * a.W + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int S0 = __ldg(row0 + 3 * sx + c) * a0 + __ldg(row0 + 3 * x1 + c) * a1;
        const int S1 = __ldg(row1 + 3 * sx + c) * a0 + __ldg(row1 + 3 * x1 + c) * a1;
        const int v = ((((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16) + 2) >> 2;
        out[c * plane] = (uint8_t)min(max(v, 0), 255);
    }
}

}  // namespace
}  // namespace yfv2

extern "C" int yfv2_resize_bgr_u8(const yfv2_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    using namespace yfv2;
    if (!frames || !dst || N <= 0) { set_error("resize_bgr_u8: null frames / dst or N <= 0"); return YFV2_EINVAL; }
    if (H <= 0 || W <= 0 || H > kResizeMaxSide || W > kResizeMaxSide) {
        set_error("resize_bgr_u8: target %dx%d outside 1..%d", W, H, kResizeMaxSide);
        return YFV2_EINVAL;
    }
    for (int n = 0; n < N; ++n) {
        const yfv2_frame& f = frames[n];
        if (!f.data || f.w <= 0 || f.h <= 0 || f.pitch < 3LL * f.w) {
            set_error("resize_bgr_u8: frame %d: data %p, %dx%d, pitch %lld (need data, w, h > 0, pitch >= 3*w)", n, (const void*)f.data,
                      f.w, f.h, f.pitch);
            return YFV2_EINVAL;
        }
    }
    const dim3 block(kResizeBx, kResizeBy);
    for (int n0 = 0; n0 < N; n0 += kResizeChunk) {
        const int cnt = N - n0 < kResizeChunk ? N - n0 : kResizeChunk;
        ResizeChunk a{};
        for (int i = 0; i < cnt; ++i) a.src[i] = frames[n0 + i];
        a.dst = dst + (size_t)n0 * 3 * H * W;
        a.H = H; a.W = W;
        const dim3 grid((unsigned)((W + kResizeBx - 1) / kResizeBx), (unsigned)((H + kResizeBy - 1) / kResizeBy), (unsigned)cnt);
        resize_bgr_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(a);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}
