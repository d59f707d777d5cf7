// cv2.resize(INTER_LINEAR)'s per-pixel arithmetic (k_resize.cu states it): the coefficients of one target index and one output
// pixel computed over any source type with a fetch(c0, c1, p0, p1) of two pixels of a row.  k_resize.cu's kernels and k_jpeg.cu's
// fused decode + resize (JpegSource) share it.  The frame fetches (BGR, strided, YUV 4:2:0, packed YUV 4:2:2: cv2.cvtColor's BGR
// bytes of any layout) are here too, shared by k_resize.cu and the JPEG encoder (k_jpeg_enc.cu), with the host checks of their
// descriptors.
#pragma once
#include <climits>
#include <stdint.h>

namespace yfv2 {
namespace {

// Host checks of one frame descriptor: nullptr, or why it is refused.  The resize entries and yfv2_jpeg_encode_plan accept exactly
// the descriptors these accept.
inline const char* frame_fault(const yfv2_frame& f) {
    if (!f.data) return "null data";
    if (f.w <= 0 || f.h <= 0) return "w and h must be > 0";
    if (f.pitch < 3LL * f.w) return "pitch < 3 * w";
    return nullptr;
}
// grey (YFV2_JPEG_SRC_GRAY) reads the byte at b only
inline const char* frame_fault(const yfv2_strided_frame& f, bool grey = false) {
    if (!f.b || (!grey && (!f.g || !f.r))) return "null channel pointer";
    if (f.w <= 0 || f.h <= 0) return "w and h must be > 0";
    if (f.step < 1) return "step must be >= 1";
    if ((long long)f.step * f.w > INT_MAX) return "step * w must be < 2^31";
    if (f.pitch < (long long)f.step * f.w) return "pitch < step * w";
    return nullptr;
}
inline const char* frame_fault(const yfv2_yuv420_frame& f) {
    if (!f.y || !f.u || !f.v) return "null plane";
    if (f.w <= 0 || f.h <= 0 || (f.w & 1) || (f.h & 1)) return "w and h must be even and > 0";
    if (f.y_pitch < f.w) return "y_pitch < w";
    if (f.uv_step != 1 && f.uv_step != 2) return "uv_step must be 1 (planar) or 2 (interleaved)";
    if (f.uv_pitch < (f.uv_step == 2 ? (long long)f.w : (long long)(f.w / 2))) return "uv_pitch < w / 2 * uv_step";
    return nullptr;
}
inline const char* frame_fault(const yfv2_yuv422_frame& f) {
    if (!f.y || !f.u || !f.v) return "null plane pointer";
    if (f.w <= 0 || f.h <= 0 || (f.w & 1)) return "w must be even and > 0, h > 0";
    if (f.pitch < 2LL * f.w) return "pitch < 2 * w";
    return nullptr;
}

__device__ __forceinline__ int sat_u8(int v) { return min(max(v, 0), 255); }

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
