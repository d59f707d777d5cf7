// cv2.resize(INTER_LINEAR)'s per-pixel arithmetic (k_resize.cu states it): the coefficients of one target index and one output
// pixel computed over any source type with a fetch(c0, c1, p0, p1) of two pixels of a row.  k_resize.cu's kernels and k_jpeg.cu's
// fused decode + resize (JpegSource) share it.  The frame fetches (BGR, strided, YUV 4:2:0, packed YUV 4:2:2, raw Bayer:
// cv2.cvtColor's BGR bytes of any layout) are here too, shared by k_resize.cu and the JPEG encoder (k_jpeg_enc.cu), with the host
// checks of their descriptors.
#pragma once
#include <climits>
#include <cmath>
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
inline const char* frame_fault(const yfv2_bayer_frame& f) {
    if (!f.data) return "null data";
    if (f.fw < 1 || f.fh < 1) return "fw and fh must be >= 1";
    if (f.pitch < f.fw) return "pitch < fw";
    if (f.w < 1 || f.h < 1 || f.x0 < 0 || f.y0 < 0 || (long long)f.x0 + f.w > f.fw || (long long)f.y0 + f.h > f.fh)
        return "window empty or outside the frame";
    if ((f.red_x | f.red_y) & ~1) return "red_x and red_y must be 0 or 1";
    if (f.edge_aware & ~1) return "edge_aware must be 0 or 1";
    return nullptr;
}
inline const char* frame_fault(const yfv2_remap_map& m) {
    if (!m.xy || !m.code) return "null map plane";
    if (m.mw < 1 || m.mh < 1 || m.mw > 32767 || m.mh > 32767) return "map sides must be in 1..32767";
    if (((uintptr_t)m.xy & 3) || (m.xy_pitch & 3) || m.xy_pitch < 4LL * m.mw) return "xy must be 4-byte aligned, xy_pitch >= 4 * mw";
    if (((uintptr_t)m.code & 1) || (m.code_pitch & 1) || m.code_pitch < 2LL * m.mw)
        return "code must be 2-byte aligned, code_pitch >= 2 * mw";
    return nullptr;
}
inline const char* frame_fault(const yfv2_remap_frame& f) {
    const char* why = "kind must be YFV2_JPEG_SRC_BGR, _STRIDED, _YUV420, _YUV422 or _BAYER";
    switch (f.kind) {
        case YFV2_JPEG_SRC_BGR: why = frame_fault(f.f.bgr); break;
        case YFV2_JPEG_SRC_STRIDED: why = frame_fault(f.f.strided); break;
        case YFV2_JPEG_SRC_YUV420: why = frame_fault(f.f.yuv420); break;
        case YFV2_JPEG_SRC_YUV422: why = frame_fault(f.f.yuv422); break;
        case YFV2_JPEG_SRC_BAYER: why = frame_fault(f.f.bayer); break;
        default: break;
    }
    if (why) return why;
    if ((why = frame_fault(f.map))) return why;
    if (f.w < 1 || f.h < 1 || f.x0 < 0 || f.y0 < 0 || (long long)f.x0 + f.w > f.map.mw || (long long)f.y0 + f.h > f.map.mh)
        return "window empty or outside the map";
    return nullptr;
}

// The destination -> source matrix of a warp descriptor in m (9 values), inverted as cv2 inverts it, or why the descriptor is
// refused; its inner frame is not checked.  Host code: each line is one IEEE double operation (no x86-64 host compiler fuses
// them without FMA enabled, and tests/test_warp_cpu.py pins the results to cv2's own bits).
inline const char* warp_matrix_fault(const yfv2_warp_frame& f, double (&m)[9]) {
    if (f.perspective & ~1) return "perspective must be 0 or 1";
    if (f.inverse & ~1) return "inverse must be 0 or 1";
    if (f.dw < 1 || f.dh < 1 || f.dw > 32767 || f.dh > 32767) return "dw and dh must be in 1..32767";
    const int n = f.perspective ? 9 : 6;
    for (int k = 0; k < n; ++k)
        if (!std::isfinite(f.m[k])) return "matrix entries must be finite";
    for (int k = 0; k < 9; ++k) m[k] = k < n ? f.m[k] : k == 8 ? 1.0 : 0.0;
    if (!f.inverse && !f.perspective) {                       // warpAffine's inversion
        double D = m[0] * m[4] - m[1] * m[3];
        if (D == 0) return "singular matrix (determinant 0)";
        D = 1. / D;
        const double A11 = m[4] * D, A22 = m[0] * D;
        m[0] = A11; m[1] *= -D;
        m[3] *= -D; m[4] = A22;
        const double b1 = -m[0] * m[2] - m[1] * m[5];
        const double b2 = -m[3] * m[2] - m[4] * m[5];
        m[2] = b1; m[5] = b2;
    } else if (!f.inverse) {                                  // cv2.invert(M, DECOMP_LU) of a 3x3 matrix
        const double* a = f.m;
        double d = a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) + a[2] * (a[3] * a[7] - a[4] * a[6]);
        if (d == 0) return "singular matrix (determinant 0)";
        d = 1. / d;
        m[0] = (a[4] * a[8] - a[5] * a[7]) * d; m[1] = (a[2] * a[7] - a[1] * a[8]) * d; m[2] = (a[1] * a[5] - a[2] * a[4]) * d;
        m[3] = (a[5] * a[6] - a[3] * a[8]) * d; m[4] = (a[0] * a[8] - a[2] * a[6]) * d; m[5] = (a[2] * a[3] - a[0] * a[5]) * d;
        m[6] = (a[3] * a[7] - a[4] * a[6]) * d; m[7] = (a[1] * a[6] - a[0] * a[7]) * d; m[8] = (a[0] * a[4] - a[1] * a[3]) * d;
    }
    for (int k = 0; k < 9; ++k)
        if (!std::isfinite(m[k])) return "the inverse has non-finite entries";
    if (!f.perspective) {                                     // every scaled term below 2^30: the int32 sums cannot overflow
        const double lim = 1073741824.0;
        for (int e = 0; e < 2; ++e) {
            const double x = e ? f.dw - 1 : 0, y = e ? f.dh - 1 : 0;
            if (std::fabs((m[0] * x) * 1024) >= lim || std::fabs((m[3] * x) * 1024) >= lim ||
                std::fabs((m[1] * y + m[2]) * 1024) >= lim || std::fabs((m[4] * y + m[5]) * 1024) >= lim)
                return "affine coordinates reach 2^30 / 1024 pixels (cv2's int32 sums would overflow)";
        }
    }
    return nullptr;
}
inline const char* frame_fault(const yfv2_warp_frame& f) {
    const char* why = "kind must be YFV2_JPEG_SRC_BGR, _STRIDED, _YUV420, _YUV422 or _BAYER";
    switch (f.kind) {
        case YFV2_JPEG_SRC_BGR: why = frame_fault(f.f.bgr); break;
        case YFV2_JPEG_SRC_STRIDED: why = frame_fault(f.f.strided); break;
        case YFV2_JPEG_SRC_YUV420: why = frame_fault(f.f.yuv420); break;
        case YFV2_JPEG_SRC_YUV422: why = frame_fault(f.f.yuv422); break;
        case YFV2_JPEG_SRC_BAYER: why = frame_fault(f.f.bayer); break;
        default: break;
    }
    if (why) return why;
    double m[9];
    if ((why = warp_matrix_fault(f, m))) return why;
    if (f.w < 1 || f.h < 1 || f.x0 < 0 || f.y0 < 0 || (long long)f.x0 + f.w > f.dw || (long long)f.y0 + f.h > f.dh)
        return "window empty or outside the output";
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

// cv2.cvtColor's COLOR_Bayer??2BGR (_EA) of one interior pixel from its 3x3 raw neighbourhood (row-major: up, centre, down),
// into B, G, R.  red_row / red_col: the pixel's row / column holds red sites; both or neither: an R or B site, else a G site.
__device__ __forceinline__ void demosaic(int ul, int u, int ur, int l, int c, int r, int dl, int d, int dr, bool red_row,
                                         bool red_col, bool ea, int (&p)[3]) {
    const int hor = (l + r + 1) >> 1, ver = (u + d + 1) >> 1;
    if (red_row == red_col) {
        const int diag = (ul + ur + dl + dr + 2) >> 2;
        p[1] = ea ? (abs(l - r) <= abs(u - d) ? hor : ver) : (u + d + l + r + 2) >> 2;
        p[0] = red_row ? diag : c;
        p[2] = red_row ? c : diag;
    } else {
        p[1] = c;
        p[0] = red_row ? ver : hor;
        p[2] = red_row ? hor : ver;
    }
}

// Raw Bayer: the window (x0, y0, w, h) of cv2.cvtColor(raw, COLOR_Bayer??2BGR / _EA) of the whole fw x fh frame.  Pixel (r, c) of
// the window is demosaiced where it is read, at the frame's interior pixel (clamp(y0 + r, 1, fh - 2), clamp(x0 + c, 1, fw - 2));
// frames under 3 pixels on a side are zeros.  The pattern (red_x, red_y) and the method are descriptor values, so nothing here
// branches on the layout.  The two columns of a fetch are adjacent or equal after the clamp, so they share one 3 x 4 raw window.
struct BayerSource {
    using Desc = yfv2_bayer_frame;
    static constexpr int kChunk = 64;    // 56-byte descriptors: 3.5 KB of kernel parameters, under the 4 KB launch limit
    static constexpr int kMinBlocks = 0;
    const yfv2_bayer_frame& f;           // the rest is read from the descriptor where it is used: no registers held across fetches
    const uint8_t* mid;                  // the clamped row
    bool red_row;
    __device__ __forceinline__ BayerSource(const yfv2_bayer_frame& f_, int r) : f(f_) {
        const int R = min(max(f.y0 + r, 1), f.fh - 2);
        mid = f.data + (long long)R * f.pitch;
        red_row = ((R ^ f.red_y) & 1) == 0;
    }
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        if (f.fw < 3 || f.fh < 3) {
#pragma unroll
            for (int c = 0; c < 3; ++c) p0[c] = p1[c] = 0;
            return;
        }
        const int C0 = min(max(f.x0 + c0, 1), f.fw - 2), C1 = min(max(f.x0 + c1, 1), f.fw - 2);
        const bool d = C1 != C0;                                  // C1 == C0 + 1
        const bool ea = f.edge_aware;
        int a[3][4];                                              // raw columns C0 - 1 .. C0 + 1, C1 + 1 of rows R - 1 .. R + 1
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const uint8_t* row = mid + (k - 1) * f.pitch + C0;
            a[k][0] = __ldg(row - 1); a[k][1] = __ldg(row); a[k][2] = __ldg(row + 1); a[k][3] = __ldg(row + d + 1);
        }
        const bool red_col0 = ((C0 ^ f.red_x) & 1) == 0;
        demosaic(a[0][0], a[0][1], a[0][2], a[1][0], a[1][1], a[1][2], a[2][0], a[2][1], a[2][2], red_row, red_col0, ea, p0);
        int b[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int j = 0; j < 3; ++j) b[k][j] = d ? a[k][j + 1] : a[k][j];
        demosaic(b[0][0], b[0][1], b[0][2], b[1][0], b[1][1], b[1][2], b[2][0], b[2][1], b[2][2], red_row, red_col0 != d, ea, p1);
    }
};

// cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0)'s sampling of an Inner frame at one fixed-point entry: integer source pixel (X, Y)
// and interpolation code k (0..1023), B, G, R in v.  cv2's weights for code (i, j) are rint(fl32(fl32(1 - i/32) *
// fl32(1 - j/32)) * 32768) and so on; every factor is a multiple of 1/32, so each product is exact and the weights are the
// integers 32 (32 - i)(32 - j) ..., already summing to 32768 (initInterTab2D's correction never fires; tests/remap_oracle.py
// computes the table cv2's way and checks this).  A tap outside the inner frame's w x h weighs 0, and its fetch reads the clamped
// coordinate, so Inner is never read out of range; the two columns of a fetch stay equal or adjacent, as BayerSource needs.
// remap_pixel (a map entry) and warp_pixel (a computed coordinate) share it.
// Border != 0 is BORDER_CONSTANT with that value instead (YOLOv5's borderValue 114): a tap outside weighs as it would inside and
// reads Border, so a pixel with all four taps outside is Border.  Border 0, the default, is the rule above.
template <class Inner, int Border = 0>
__device__ __forceinline__ void sample_fixed(const typename Inner::Desc& f, int X, int Y, int k, int (&v)[3]) {
    const int i = k >> 5, j = k & 31;
    const int w = f.w, h = f.h;
    const bool x0in = (unsigned)X < (unsigned)w, x1in = (unsigned)(X + 1) < (unsigned)w;
    const bool y0in = (unsigned)Y < (unsigned)h, y1in = (unsigned)(Y + 1) < (unsigned)h;
    if (!((x0in || x1in) && (y0in || y1in))) {
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = Border;
        return;
    }
    const int ax0 = x0in || Border ? 32 - j : 0, ax1 = x1in || Border ? j : 0;
    const int by0 = y0in || Border ? 32 - i : 0, by1 = y1in || Border ? i : 0;
    const int cx0 = min(max(X, 0), w - 1), cx1 = min(max(X + 1, 0), w - 1);
    const Inner row0(f, min(max(Y, 0), h - 1)), row1(f, min(max(Y + 1, 0), h - 1));
    int p00[3], p01[3], p10[3], p11[3];          // [row][column] taps, B G R
    row0.fetch(cx0, cx1, p00, p01);
    row1.fetch(cx0, cx1, p10, p11);
    if (Border) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p00[c] = y0in && x0in ? p00[c] : Border; p01[c] = y0in && x1in ? p01[c] : Border;
            p10[c] = y1in && x0in ? p10[c] : Border; p11[c] = y1in && x1in ? p11[c] : Border;
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
        v[c] = sat_u8(((by0 * (p00[c] * ax0 + p01[c] * ax1) + by1 * (p10[c] * ax0 + p11[c] * ax1)) * 32 + 16384) >> 15);
}

// cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) of an Inner frame through fixed maps: pixel (mx, my) of the remapped image, B, G,
// R in v
template <class Inner>
__device__ __forceinline__ void remap_pixel(const typename Inner::Desc& f, const yfv2_remap_map& m, int mx, int my, int (&v)[3]) {
    const int xy = __ldg((const int*)((const uint8_t*)m.xy + (long long)my * m.xy_pitch) + mx);    // 4-byte aligned: checked
    const int k = __ldg((const uint16_t*)((const uint8_t*)m.code + (long long)my * m.code_pitch) + mx) & 1023;
    sample_fixed<Inner>(f, (int)(int16_t)(xy & 0xffff), xy >> 16, k, v);
}

// A warped view's descriptor on the device: the inner frame, the destination -> source matrix (inverted on the host), whether
// it is a perspective one, and the window of the warped image (w, h: the resize's source size)
template <class Inner>
struct WarpDesc {
    typename Inner::Desc f;
    double m[9];
    int perspective;
    int x0, y0, w, h;
};

// cvRound of a perspective coordinate: std::max(INT_MIN, std::min(INT_MAX, v)) as cv2 writes it (a NaN becomes INT_MAX), then
// half to even
__device__ __forceinline__ int clamp_round(double v) {
    v = v < 2147483647.0 ? v : 2147483647.0;
    v = -2147483648.0 < v ? v : -2147483648.0;
    return __double2int_rn(v);
}

// cv2.warpAffine / cv2.warpPerspective(INTER_LINEAR, BORDER_CONSTANT 0) of an Inner frame: pixel (x, y) of the warped image, B,
// G, R in v.  The fixed-point coordinate is computed here in cv2's order of fp64 operations (yfv2.h states them), each rounded
// on its own (__dmul_rn / __dadd_rn: no FMA contraction), then sampled as a remap map entry (with Border: sample_fixed's).
template <class Inner, int Border = 0>
__device__ __forceinline__ void warp_pixel(const WarpDesc<Inner>& d, int x, int y, int (&v)[3]) {
    const double* m = d.m;
    const double dx = (double)x, dy = (double)y;
    int X, Y;
    if (!d.perspective) {                     // cvRound((m1 y + m2) 1024) + 16 + cvRound((m0 x) 1024), >> 5; |terms| < 2^30
        X = (__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], dy), m[2]), 1024.0)) + 16 +
             __double2int_rn(__dmul_rn(__dmul_rn(m[0], dx), 1024.0))) >> 5;
        Y = (__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], dy), m[5]), 1024.0)) + 16 +
             __double2int_rn(__dmul_rn(__dmul_rn(m[3], dx), 1024.0))) >> 5;
    } else {
        double W = __dadd_rn(__dadd_rn(__dmul_rn(m[7], dy), m[8]), __dmul_rn(m[6], dx));
        W = W != 0.0 ? __ddiv_rn(32.0, W) : 0.0;
        X = clamp_round(__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[1], dy), m[2]), __dmul_rn(m[0], dx)), W));
        Y = clamp_round(__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4], dy), m[5]), __dmul_rn(m[3], dx)), W));
    }
    const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
    sample_fixed<Inner, Border>(d.f, sx, sy, ((Y & 31) << 5) + (X & 31), v);
}

// Pixels of the window of cv2.warpAffine / cv2.warpPerspective(inner frame), each computed from the inner frame where it is read
template <class Inner>
struct WarpSource {
    using Desc = WarpDesc<Inner>;
    // frames per launch: each descriptor, plus yfv2_warp_u8's output pointer, under the 4 KB launch limit with the chunk's rest
    static constexpr int kChunk = 4000 / (int)(sizeof(Desc) + sizeof(void*));
    static constexpr int kMinBlocks = 0;
    const Desc& f;
    int y;
    __device__ __forceinline__ WarpSource(const Desc& f_, int r) : f(f_), y(f_.y0 + r) {}
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        warp_pixel<Inner>(f, f.x0 + c0, y, p0);
        warp_pixel<Inner>(f, f.x0 + c1, y, p1);
    }
};

// A remapped view's descriptor on the device: the inner frame, the map and the window (w, h: the resize's source size)
template <class Inner>
struct RemapDesc {
    typename Inner::Desc f;
    yfv2_remap_map m;
    int x0, y0, w, h;
};

// Pixels of the window of cv2.remap(inner frame), each computed from the inner frame where it is read
template <class Inner>
struct RemapSource {
    using Desc = RemapDesc<Inner>;
    // frames per launch: each descriptor, plus yfv2_remap_u8's output pointer, under the 4 KB launch limit with the chunk's rest
    static constexpr int kChunk = 4000 / (int)(sizeof(Desc) + sizeof(void*));
    static constexpr int kMinBlocks = 0;
    const Desc& f;
    int my;
    __device__ __forceinline__ RemapSource(const Desc& f_, int r) : f(f_), my(f_.y0 + r) {}
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        remap_pixel<Inner>(f.f, f.m, f.x0 + c0, my, p0);
        remap_pixel<Inner>(f.f, f.m, f.x0 + c1, my, p1);
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
