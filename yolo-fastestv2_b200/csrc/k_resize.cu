// Raw-frame resize: cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR) (the host step of test.py:35 and
// utils/datasets.py:107), written straight into the [N,3,H,W] planar uint8 batch yfv2_forward_u8 consumes (test.py:36-37:
// res_img.transpose(2, 0, 1)).  Four sources share one kernel body, a template over the source-pixel fetch:
//   packed HWC BGR frames (yfv2_resize_bgr_u8);
//   strided frames (yfv2_resize_strided_u8): channel k of pixel (r, c) at ch_k + r * pitch + c * step, which states packed
//   RGB / BGRA / RGBA, grey and planar RGB alike (each a channel move away from BGR, and channel moves commute with the resize);
//   YUV 4:2:0 frames (yfv2_resize_yuv420_u8: NV12 / NV21 / I420 / YV12) and packed YUV 4:2:2 frames (yfv2_resize_yuv422_u8:
//   YUYV / UYVY / YVYU), each source pixel converted to BGR exactly as cv2.cvtColor(COLOR_YUV2BGR_*) does (OpenCV's ITUR_BT_601
//   fixed point, limited range, chroma not interpolated; (U, V) is the sample of the pixel's 2x2 block for 4:2:0, of its
//   two-pixel macropixel for 4:2:2):
//     uu = U - 128, vv = V - 128, y = max(0, Y[r][c] - 16) * 1220542 + (1 << 19)
//     B = sat_u8((y + 2116026 uu) >> 20), G = sat_u8((y - 852492 vv - 409993 uu) >> 20), R = sat_u8((y + 1673527 vv) >> 20).
// The resize is bit-identical to OpenCV's x86 8-bit path, all integer after the coefficients:
//   coefficients per axis: f = fl32((d + 0.5) * (n / m) - 0.5) (product and difference rounded in double), s = floor(f),
//     f = fl32(f - s); weights rint(fl32(1 - f) * 2048), rint(f * 2048).  Along x, s < 0 -> (0, 0) then s >= w - 1 -> (w - 1, 0);
//     along y the weights keep the unclamped fraction and the two rows are clamped.
//   horizontal: S = src[sx] * a0 + src[min(sx + 1, w - 1)] * a1 (int32, per channel)
//   vertical:   out = sat_u8((((S0 >> 4) * b0 >> 16) + ((S1 >> 4) * b1 >> 16) + 2) >> 2)
// oracle/resize.py restates the resize in numpy, tests/yuv_oracle.py the colour conversion and tests/layout_oracle.py the channel
// moves.  One thread per output pixel (all three channels); a warp covers 32 consecutive x of one row, so each plane store of a
// warp is one contiguous 32-byte run.  The coefficients are recomputed per thread (four double operations): cheaper than a table
// round trip, and the call needs no workspace.
#include <climits>

#include "common.cuh"

namespace yfv2 {
namespace {

constexpr int kResizeBx = 64, kResizeBy = 4;
constexpr int kResizeMaxSide = 32768;

// Packed HWC BGR: pixel (r, c) is the three bytes at data + r * pitch + 3c.  StridedSource states this layout too, but is 2.5 %
// slower on it (DESIGN.md §7), so BGR keeps its own fetch.
struct BgrSource {
    using Desc = yfv2_frame;
    static constexpr int kChunk = 128;   // frames per launch: their 24-byte descriptors travel as kernel parameters (3 KB)
    static constexpr int kMinBlocks = 0;
    const uint8_t* row;
    __device__ __forceinline__ BgrSource(const yfv2_frame& f, int r) : row(f.data + (long long)r * f.pitch) {}
    // B, G, R of pixels (r, c0) and (r, c1)
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p0[c] = __ldg(row + 3 * c0 + c);
            p1[c] = __ldg(row + 3 * c1 + c);
        }
    }
};

// Strided: channel k of pixel (r, c) at ch_k + r * pitch + c * step (B, G, R).  Packed BGR / RGB / BGRA / RGBA, grey and planar
// RGB differ only in the descriptor's values, so nothing here branches on the layout.
struct StridedSource {
    using Desc = yfv2_strided_frame;
    static constexpr int kChunk = 80;    // 48-byte descriptors: 3.75 KB of kernel parameters, under the 4 KB launch limit
    static constexpr int kMinBlocks = 8;
    const uint8_t* ch[3];
    int step;
    __device__ __forceinline__ StridedSource(const yfv2_strided_frame& f, int r) : step(f.step) {
        const long long off = (long long)r * f.pitch;
        ch[0] = f.b + off; ch[1] = f.g + off; ch[2] = f.r + off;
    }
    // B, G, R of pixels (r, c0) and (r, c1)
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        const int k0 = c0 * step, k1 = c1 * step;     // step * w < 2^31, checked on the host
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p0[c] = __ldg(ch[c] + k0);
            p1[c] = __ldg(ch[c] + k1);
        }
    }
};

__device__ __forceinline__ int sat_u8(int v) { return min(max(v, 0), 255); }

// cv2.cvtColor's YUV -> BGR of one pixel, 4:2:0 and 4:2:2 alike (OpenCV ITUR_BT_601: 20-bit fixed point, limited range)
__device__ __forceinline__ void yuv_to_bgr(int y, int uu, int vv, int (&bgr)[3]) {
    const int yy = max(0, y - 16) * 1220542 + (1 << 19);
    bgr[0] = sat_u8((yy + 2116026 * uu) >> 20);
    bgr[1] = sat_u8((yy - 852492 * vv - 409993 * uu) >> 20);
    bgr[2] = sat_u8((yy + 1673527 * vv) >> 20);
}

// YUV 4:2:0: luma Y[r][c] at y + r * y_pitch + c; the chroma of pixel (r, c) at u / v + (r >> 1) * uv_pitch + (c >> 1) * uv_step.
// The descriptor states every layout, so nothing here branches on it.
struct Yuv420Source {
    using Desc = yfv2_yuv420_frame;
    static constexpr int kChunk = 64;    // 56-byte descriptors: 3.5 KB of kernel parameters, under the 4 KB launch limit
    static constexpr int kMinBlocks = 0;
    const uint8_t* luma;
    const uint8_t* u;
    const uint8_t* v;
    int step;
    __device__ __forceinline__ Yuv420Source(const yfv2_yuv420_frame& f, int r)
        : luma(f.y + (long long)r * f.y_pitch), u(f.u + (long long)(r >> 1) * f.uv_pitch), v(f.v + (long long)(r >> 1) * f.uv_pitch),
          step(f.uv_step) {}
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        const int k0 = (c0 >> 1) * step, k1 = (c1 >> 1) * step;
        const int u0 = __ldg(u + k0) - 128, v0 = __ldg(v + k0) - 128;
        int u1 = u0, v1 = v0;
        if (k1 != k0) { u1 = __ldg(u + k1) - 128; v1 = __ldg(v + k1) - 128; }   // c0, c1 in different chroma columns
        yuv_to_bgr(__ldg(luma + c0), u0, v0, p0);
        yuv_to_bgr(__ldg(luma + c1), u1, v1, p1);
    }
};

// Packed YUV 4:2:2: luma of (r, c) at y + r * pitch + 2c; U and V of the macropixel (r, 2j), (r, 2j + 1) at u / v + r * pitch + 4j.
// YUYV, UYVY and YVYU differ only in the three pointers.
struct Yuv422Source {
    using Desc = yfv2_yuv422_frame;
    static constexpr int kChunk = 96;    // 40-byte descriptors: 3.75 KB of kernel parameters
    static constexpr int kMinBlocks = 8;
    const uint8_t* luma;
    const uint8_t* u;
    const uint8_t* v;
    __device__ __forceinline__ Yuv422Source(const yfv2_yuv422_frame& f, int r) {
        const long long off = (long long)r * f.pitch;
        luma = f.y + off; u = f.u + off; v = f.v + off;
    }
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        const int k0 = (c0 >> 1) * 4, k1 = (c1 >> 1) * 4;
        const int u0 = __ldg(u + k0) - 128, v0 = __ldg(v + k0) - 128;
        int u1 = u0, v1 = v0;
        if (k1 != k0) { u1 = __ldg(u + k1) - 128; v1 = __ldg(v + k1) - 128; }   // c0, c1 in different macropixels
        yuv_to_bgr(__ldg(luma + 2 * c0), u0, v0, p0);
        yuv_to_bgr(__ldg(luma + 2 * c1), u1, v1, p1);
    }
};

template <class Src>
struct ResizeChunk {
    typename Src::Desc src[Src::kChunk];
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

// Src::kMinBlocks 8 holds a fetch to 32 registers (the strided fetch's three row pointers take 34 unbounded), so an SM keeps its
// full 2048 threads in flight: the kernel waits on DRAM, not on issue.  BGR and 4:2:0 use 32 registers unbounded (0: no bound).
template <class Src>
__global__ void __launch_bounds__(kResizeBx * kResizeBy, Src::kMinBlocks)
resize_kernel(const __grid_constant__ ResizeChunk<Src> a) {
    const int x = blockIdx.x * kResizeBx + threadIdx.x;
    const int y = blockIdx.y * kResizeBy + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const typename Src::Desc fr = a.src[blockIdx.z];
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

    const Src row0(fr, r0), row1(fr, r1);
    const size_t plane = (size_t)a.H * a.W;
    uint8_t* out = a.dst + (size_t)blockIdx.z * 3 * plane + (size_t)y * a.W + x;
    int p00[3], p01[3], p10[3], p11[3];          // [row][column] source pixels, B G R
    row0.fetch(sx, x1, p00, p01);
    row1.fetch(sx, x1, p10, p11);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int S0 = p00[c] * a0 + p01[c] * a1;
        const int S1 = p10[c] * a0 + p11[c] * a1;
        const int v = ((((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16) + 2) >> 2;
        out[c * plane] = (uint8_t)sat_u8(v);
    }
}

// Launches the checked descriptors Src::kChunk frames at a time.
template <class Src>
int launch_resize(const typename Src::Desc* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    const dim3 block(kResizeBx, kResizeBy);
    for (int n0 = 0; n0 < N; n0 += Src::kChunk) {
        const int cnt = N - n0 < Src::kChunk ? N - n0 : Src::kChunk;
        ResizeChunk<Src> a{};
        for (int i = 0; i < cnt; ++i) a.src[i] = frames[n0 + i];
        a.dst = dst + (size_t)n0 * 3 * H * W;
        a.H = H; a.W = W;
        const dim3 grid((unsigned)((W + kResizeBx - 1) / kResizeBx), (unsigned)((H + kResizeBy - 1) / kResizeBy), (unsigned)cnt);
        resize_kernel<Src><<<grid, block, 0, (cudaStream_t)stream>>>(a);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}

// The checks every entry makes on its call before it looks at the frames.
bool bad_call(const char* fn, const void* frames, int N, int H, int W, const uint8_t* dst) {
    if (!frames || !dst || N <= 0) { set_error("%s: null frames / dst or N <= 0", fn); return true; }
    if (H <= 0 || W <= 0 || H > kResizeMaxSide || W > kResizeMaxSide) {
        set_error("%s: target %dx%d outside 1..%d", fn, W, H, kResizeMaxSide);
        return true;
    }
    return false;
}

}  // namespace
}  // namespace yfv2

extern "C" int yfv2_resize_bgr_u8(const yfv2_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    using namespace yfv2;
    if (bad_call("resize_bgr_u8", frames, N, H, W, dst)) return YFV2_EINVAL;
    for (int n = 0; n < N; ++n) {
        const yfv2_frame& f = frames[n];
        if (!f.data || f.w <= 0 || f.h <= 0 || f.pitch < 3LL * f.w) {
            set_error("resize_bgr_u8: frame %d: data %p, %dx%d, pitch %lld (need data, w, h > 0, pitch >= 3*w)", n, (const void*)f.data,
                      f.w, f.h, f.pitch);
            return YFV2_EINVAL;
        }
    }
    return launch_resize<BgrSource>(frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_yuv420_u8(const yfv2_yuv420_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    using namespace yfv2;
    if (bad_call("resize_yuv420_u8", frames, N, H, W, dst)) return YFV2_EINVAL;
    for (int n = 0; n < N; ++n) {
        const yfv2_yuv420_frame& f = frames[n];
        const char* why = nullptr;
        if (!f.y || !f.u || !f.v) why = "null plane";
        else if (f.w <= 0 || f.h <= 0 || (f.w & 1) || (f.h & 1)) why = "w and h must be even and > 0";
        else if (f.y_pitch < f.w) why = "y_pitch < w";
        else if (f.uv_step != 1 && f.uv_step != 2) why = "uv_step must be 1 (planar) or 2 (interleaved)";
        else if (f.uv_pitch < (f.uv_step == 2 ? (long long)f.w : (long long)(f.w / 2))) why = "uv_pitch < w / 2 * uv_step";
        if (why) {
            set_error("resize_yuv420_u8: frame %d: %s (y %p, u %p, v %p, %dx%d, y_pitch %lld, uv_pitch %lld, uv_step %d)", n, why,
                      (const void*)f.y, (const void*)f.u, (const void*)f.v, f.w, f.h, f.y_pitch, f.uv_pitch, f.uv_step);
            return YFV2_EINVAL;
        }
    }
    return launch_resize<Yuv420Source>(frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_strided_u8(const yfv2_strided_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    using namespace yfv2;
    if (bad_call("resize_strided_u8", frames, N, H, W, dst)) return YFV2_EINVAL;
    for (int n = 0; n < N; ++n) {
        const yfv2_strided_frame& f = frames[n];
        const char* why = nullptr;
        if (!f.b || !f.g || !f.r) why = "null channel pointer";
        else if (f.w <= 0 || f.h <= 0) why = "w and h must be > 0";
        else if (f.step < 1) why = "step must be >= 1";
        else if ((long long)f.step * f.w > INT_MAX) why = "step * w must be < 2^31";
        else if (f.pitch < (long long)f.step * f.w) why = "pitch < step * w";
        if (why) {
            set_error("resize_strided_u8: frame %d: %s (b %p, g %p, r %p, %dx%d, pitch %lld, step %d)", n, why, (const void*)f.b,
                      (const void*)f.g, (const void*)f.r, f.w, f.h, f.pitch, f.step);
            return YFV2_EINVAL;
        }
    }
    return launch_resize<StridedSource>(frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_yuv422_u8(const yfv2_yuv422_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    using namespace yfv2;
    if (bad_call("resize_yuv422_u8", frames, N, H, W, dst)) return YFV2_EINVAL;
    for (int n = 0; n < N; ++n) {
        const yfv2_yuv422_frame& f = frames[n];
        const char* why = nullptr;
        if (!f.y || !f.u || !f.v) why = "null plane pointer";
        else if (f.w <= 0 || f.h <= 0 || (f.w & 1)) why = "w must be even and > 0, h > 0";
        else if (f.pitch < 2LL * f.w) why = "pitch < 2 * w";
        if (why) {
            set_error("resize_yuv422_u8: frame %d: %s (y %p, u %p, v %p, %dx%d, pitch %lld)", n, why, (const void*)f.y,
                      (const void*)f.u, (const void*)f.v, f.w, f.h, f.pitch);
            return YFV2_EINVAL;
        }
    }
    return launch_resize<Yuv422Source>(frames, N, H, W, dst, stream);
}
