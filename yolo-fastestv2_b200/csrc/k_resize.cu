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
//     B = sat_u8((y + 2116026 uu) >> 20), G = sat_u8((y - 852492 vv - 409993 uu) >> 20), R = sat_u8((y + 1673527 vv) >> 20);
//   raw Bayer frames (yfv2_resize_bayer_u8), each source pixel demosaiced as cv2.cvtColor(COLOR_Bayer??2BGR / _EA) does, in
//   integers on the 3x3 raw neighbourhood of its clamped frame coordinate (resize.cuh's BayerSource, tests/bayer_oracle.py);
//   lens-corrected views of any of these (yfv2_resize_remap_u8): each source pixel is cv2.remap(INTER_LINEAR)'s pixel of the
//   inner frame (resize.cuh's RemapSource over the inner fetch, remap_pixel), one instantiation per inner kind;
//   rotated, de-skewed and bird's-eye views of any of these (yfv2_resize_warp_u8): each source pixel is cv2.warpAffine's or
//   cv2.warpPerspective's pixel of the inner frame, its fixed-point coordinate computed from the descriptor's matrix where it is
//   read (resize.cuh's WarpSource, warp_pixel), sampled by remap_pixel's own sample_fixed.
// yfv2_remap_u8 and yfv2_warp_u8 write the views' windows alone (remap_kernel, warp_kernel), with the same per-pixel functions.
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
// aug_resize_kernel (yfv2_aug_batch, k_aug.cu) runs random_resize as the second resize over a fetch that computes the pixels of
// the first from the planar source where they are read (DESIGN.md §9).
// The per-pixel arithmetic is in resize.cuh, shared with the fused JPEG decode + resize (k_jpeg.cu).
#include "aug.cuh"
#include "resize.cuh"

namespace yfv2 {
namespace {

constexpr int kResizeBx = 64, kResizeBy = 4;
constexpr int kResizeMaxSide = 32768;

template <class Src>
struct ResizeChunk {
    typename Src::Desc src[Src::kChunk];
    uint8_t* dst;                        // [n][3][H][W] of the chunk's first frame
    int H, W;
};

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

// Image n of an augmentation chunk: its planar [3][H][W] source bytes and parameters
struct AugFrame {
    const uint8_t* img;
    int W, H;
    yfv2_aug_params p;
};

// Source pixels of the augmentation, through contrast_and_brightness (alpha 1, beta 0 leave them unchanged)
struct PlanarSource {
    using Desc = AugFrame;
    const uint8_t* row;
    size_t plane;
    float alpha, beta;
    __device__ __forceinline__ PlanarSource(const AugFrame& f, int r)
        : row(f.img + (size_t)r * f.W), plane((size_t)f.H * f.W), alpha(f.p.alpha), beta(f.p.beta) {}
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p0[c] = (int)aug_byte(__ldg(row + c * plane + c0), alpha, beta);
            p1[c] = (int)aug_byte(__ldg(row + c * plane + c1), alpha, beta);
        }
    }
};

// motion_blur's output in the workspace, read through the image's normalize map (staged in shared memory)
struct MapFrame : AugFrame {
    const uint8_t* map;
};
struct MappedSource {
    using Desc = MapFrame;
    const uint8_t* row;
    size_t plane;
    const uint8_t* map;
    __device__ __forceinline__ MappedSource(const MapFrame& f, int r)
        : row(f.img + (size_t)r * f.W), plane((size_t)f.H * f.W), map(f.map) {}
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p0[c] = map[__ldg(row + c * plane + c0)];
            p1[c] = map[__ldg(row + c * plane + c1)];
        }
    }
};

// Pixels of random_resize's rw x rh intermediate cv2.resize(img, (rw, rh)), each computed from the source where it is read,
// so the intermediate image is never stored
template <class Inner>
struct NestedSource {
    using Desc = typename Inner::Desc;
    const Desc& f;
    int r;
    __device__ __forceinline__ NestedSource(const Desc& f_, int r_) : f(f_), r(r_) {}
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        resize_pixel<Inner>(f, f.W, f.H, c0, r, f.p.rw, f.p.rh, p0);
        resize_pixel<Inner>(f, f.W, f.H, c1, r, f.p.rw, f.p.rh, p1);
    }
};

// yfv2_aug_batch with the resize: one thread per output pixel of image blockIdx.z, the second resize over NestedSource, then
// augment_hsv on the pixel when the chunk has LUTs.  With an AugBlurChunk the source bytes go through the image's byte map
// (MappedSource), read from the workspace for a blurred image.
template <class Chunk>
__global__ void __launch_bounds__(kResizeBx * kResizeBy)
aug_resize_kernel(const __grid_constant__ Chunk a) {
    __shared__ typename AugTraits<Chunk>::Smem t;
    const bool hsv = a.luts != nullptr;
    if (hsv) {
        stage_hsv(t, a.luts + (size_t)blockIdx.z * 768);
        __syncthreads();
    }
    const uint8_t* img = nullptr;                      // with an AugBlurChunk: where the image's bytes are read
    if constexpr (AugTraits<Chunk>::kBlur) {
        img = stage_map(t, a, blockIdx.z, 3 * (size_t)a.H * a.W);
        __syncthreads();
    }
    const int x = blockIdx.x * kResizeBx + threadIdx.x;
    const int y = blockIdx.y * kResizeBy + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const size_t plane = (size_t)a.H * a.W;
    int v[3];
    if constexpr (AugTraits<Chunk>::kBlur) {
        const MapFrame f{{img, a.W, a.H, a.im[blockIdx.z]}, t.map};
        resize_pixel<NestedSource<MappedSource>>(f, f.p.rw, f.p.rh, x, y, a.W, a.H, v);
    } else {
        const AugFrame f{a.img + (size_t)blockIdx.z * 3 * plane, a.W, a.H, a.im[blockIdx.z]};
        resize_pixel<NestedSource<PlanarSource>>(f, f.p.rw, f.p.rh, x, y, a.W, a.H, v);
    }
    if (hsv) hsv_lut_pixel(v[0], v[1], v[2], x, a.W, t);
    uint8_t* out = a.out + (size_t)blockIdx.z * 3 * plane + (size_t)y * a.W + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * plane] = (uint8_t)v[c];
}

// Every resize entry: the call's checks, each frame's (frame_fault), then the launches; a refusal names the entry and the frame.
template <class Src>
int resize_entry(const char* fn, const typename Src::Desc* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    if (!frames || !dst || N <= 0) { set_error("%s: null frames / dst or N <= 0", fn); return YFV2_EINVAL; }
    if (H <= 0 || W <= 0 || H > kResizeMaxSide || W > kResizeMaxSide) {
        set_error("%s: target %dx%d outside 1..%d", fn, W, H, kResizeMaxSide);
        return YFV2_EINVAL;
    }
    for (int n = 0; n < N; ++n) {
        if (const char* why = frame_fault(frames[n])) {
            set_error("%s: frame %d: %s (%dx%d)", fn, n, why, frames[n].w, frames[n].h);
            return YFV2_EINVAL;
        }
    }
    return launch_resize<Src>(frames, N, H, W, dst, stream);
}

// A view alone (yfv2_remap_u8, yfv2_warp_u8): one thread per pixel of the window of frame blockIdx.z's view, written as packed
// HWC BGR to its own dst
template <class Src>
struct ViewChunk {
    typename Src::Desc src[Src::kChunk];
    uint8_t* dst[Src::kChunk];
};

// cv2.remap alone
template <class Inner>
__global__ void __launch_bounds__(kResizeBx * kResizeBy)
remap_kernel(const __grid_constant__ ViewChunk<RemapSource<Inner>> a) {
    const RemapDesc<Inner>& fr = a.src[blockIdx.z];
    const int x = blockIdx.x * kResizeBx + threadIdx.x;
    const int y = blockIdx.y * kResizeBy + threadIdx.y;
    if (x >= fr.w || y >= fr.h) return;
    int v[3];
    remap_pixel<Inner>(fr.f, fr.m, fr.x0 + x, fr.y0 + y, v);
    uint8_t* out = a.dst[blockIdx.z] + 3 * ((size_t)y * fr.w + x);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = (uint8_t)v[c];
}

// cv2.warpAffine / cv2.warpPerspective alone
template <class Inner>
__global__ void __launch_bounds__(kResizeBx * kResizeBy)
warp_kernel(const __grid_constant__ ViewChunk<WarpSource<Inner>> a) {
    const WarpDesc<Inner>& fr = a.src[blockIdx.z];
    const int x = blockIdx.x * kResizeBx + threadIdx.x;
    const int y = blockIdx.y * kResizeBy + threadIdx.y;
    if (x >= fr.w || y >= fr.h) return;
    int v[3];
    warp_pixel<Inner>(fr, fr.x0 + x, fr.y0 + y, v);
    uint8_t* out = a.dst[blockIdx.z] + 3 * ((size_t)y * fr.w + x);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = (uint8_t)v[c];
}

// The inner frame of a checked view descriptor (remap or warp), as Inner's descriptor
template <class Inner> struct InnerOf;
template <> struct InnerOf<BgrSource> { template <class F> static const yfv2_frame& get(const F& f) { return f.f.bgr; } };
template <> struct InnerOf<StridedSource> { template <class F> static const yfv2_strided_frame& get(const F& f) { return f.f.strided; } };
template <> struct InnerOf<Yuv420Source> { template <class F> static const yfv2_yuv420_frame& get(const F& f) { return f.f.yuv420; } };
template <> struct InnerOf<Yuv422Source> { template <class F> static const yfv2_yuv422_frame& get(const F& f) { return f.f.yuv422; } };
template <> struct InnerOf<BayerSource> { template <class F> static const yfv2_bayer_frame& get(const F& f) { return f.f.bayer; } };

// What the two view entries differ in: the source of the fused resize, the device descriptor of a checked host one, the kernel of
// the view alone, and how a refused descriptor is described
template <class Frame> struct ViewOf;
template <> struct ViewOf<yfv2_remap_frame> {
    template <class Inner> using Src = RemapSource<Inner>;
    template <class Inner> static RemapDesc<Inner> desc(const yfv2_remap_frame& fr) {
        return RemapDesc<Inner>{InnerOf<Inner>::get(fr), fr.map, fr.x0, fr.y0, fr.w, fr.h};
    }
    template <class Inner> static void launch_alone(dim3 grid, dim3 block, cudaStream_t s, const ViewChunk<Src<Inner>>& a) {
        remap_kernel<Inner><<<grid, block, 0, s>>>(a);
    }
    static void refuse(const char* fn, int n, const char* why, const yfv2_remap_frame& f) {
        set_error("%s: frame %d: %s (window %dx%d of a %dx%d map)", fn, n, why, f.w, f.h, f.map.mw, f.map.mh);
    }
};
template <> struct ViewOf<yfv2_warp_frame> {
    template <class Inner> using Src = WarpSource<Inner>;
    template <class Inner> static WarpDesc<Inner> desc(const yfv2_warp_frame& fr) {
        WarpDesc<Inner> d{InnerOf<Inner>::get(fr), {}, fr.perspective, fr.x0, fr.y0, fr.w, fr.h};
        warp_matrix_fault(fr, d.m);                             // checked: the destination -> source matrix
        return d;
    }
    template <class Inner> static void launch_alone(dim3 grid, dim3 block, cudaStream_t s, const ViewChunk<Src<Inner>>& a) {
        warp_kernel<Inner><<<grid, block, 0, s>>>(a);
    }
    static void refuse(const char* fn, int n, const char* why, const yfv2_warp_frame& f) {
        set_error("%s: frame %d: %s (window (%d, %d) %dx%d of a %dx%d %s warp)", fn, n, why, f.x0, f.y0, f.w, f.h, f.dw, f.dh,
                  f.perspective == 1 ? "perspective" : "affine");
    }
};

// frames[0, n), all of Inner's kind, Src<Inner>::kChunk per launch: with dst the fused resize into dst's H x W images, else the
// view alone into dst_each[i]
template <class Frame, class Inner>
int launch_view(const Frame* frames, int n, int H, int W, uint8_t* dst, uint8_t* const* dst_each, cudaStream_t stream) {
    using V = ViewOf<Frame>;
    using Src = typename V::template Src<Inner>;
    constexpr int kChunk = Src::kChunk;
    const dim3 block(kResizeBx, kResizeBy);
    for (int n0 = 0; n0 < n; n0 += kChunk) {
        const int cnt = n - n0 < kChunk ? n - n0 : kChunk;
        typename Src::Desc d[kChunk];
        int mw = 1, mh = 1;
        for (int i = 0; i < cnt; ++i) {
            const Frame& fr = frames[n0 + i];
            d[i] = V::template desc<Inner>(fr);
            mw = fr.w > mw ? fr.w : mw;
            mh = fr.h > mh ? fr.h : mh;
        }
        if (dst) {
            ResizeChunk<Src> a{};
            for (int i = 0; i < cnt; ++i) a.src[i] = d[i];
            a.dst = dst + (size_t)n0 * 3 * H * W;
            a.H = H; a.W = W;
            const dim3 grid((unsigned)((W + kResizeBx - 1) / kResizeBx), (unsigned)((H + kResizeBy - 1) / kResizeBy), (unsigned)cnt);
            resize_kernel<Src><<<grid, block, 0, stream>>>(a);
        } else {
            ViewChunk<Src> a{};
            for (int i = 0; i < cnt; ++i) {
                a.src[i] = d[i];
                a.dst[i] = dst_each[n0 + i];
            }
            const dim3 grid((unsigned)((mw + kResizeBx - 1) / kResizeBx), (unsigned)((mh + kResizeBy - 1) / kResizeBy), (unsigned)cnt);
            V::template launch_alone<Inner>(grid, block, stream, a);
        }
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}

// The remap and warp entries: the call's checks, each frame's (frame_fault), then one launch_view per run of consecutive frames
// of one kind, so that no kernel branches on the kind.  dst (the fused resize, H x W) or dst_each (the view alone) is non-null.
template <class Frame>
int view_entry(const char* fn, const Frame* frames, int N, int H, int W, uint8_t* dst, uint8_t* const* dst_each, void* stream) {
    if (!frames || (!dst && !dst_each) || N <= 0) { set_error("%s: null frames / dst or N <= 0", fn); return YFV2_EINVAL; }
    if (dst && (H <= 0 || W <= 0 || H > kResizeMaxSide || W > kResizeMaxSide)) {
        set_error("%s: target %dx%d outside 1..%d", fn, W, H, kResizeMaxSide);
        return YFV2_EINVAL;
    }
    for (int n = 0; n < N; ++n) {
        if (const char* why = frame_fault(frames[n])) {
            ViewOf<Frame>::refuse(fn, n, why, frames[n]);
            return YFV2_EINVAL;
        }
        if (dst_each && !dst_each[n]) { set_error("%s: frame %d: null dst", fn, n); return YFV2_EINVAL; }
    }
    const cudaStream_t s = (cudaStream_t)stream;
    for (int i = 0; i < N;) {
        int j = i + 1;
        while (j < N && frames[j].kind == frames[i].kind) ++j;
        uint8_t* d = dst ? dst + (size_t)i * 3 * H * W : nullptr;
        uint8_t* const* de = dst_each ? dst_each + i : nullptr;
        int rc = YFV2_OK;
        switch (frames[i].kind) {
            case YFV2_JPEG_SRC_BGR: rc = launch_view<Frame, BgrSource>(frames + i, j - i, H, W, d, de, s); break;
            case YFV2_JPEG_SRC_STRIDED: rc = launch_view<Frame, StridedSource>(frames + i, j - i, H, W, d, de, s); break;
            case YFV2_JPEG_SRC_YUV420: rc = launch_view<Frame, Yuv420Source>(frames + i, j - i, H, W, d, de, s); break;
            case YFV2_JPEG_SRC_YUV422: rc = launch_view<Frame, Yuv422Source>(frames + i, j - i, H, W, d, de, s); break;
            default: rc = launch_view<Frame, BayerSource>(frames + i, j - i, H, W, d, de, s); break;   // kinds checked above
        }
        if (rc != YFV2_OK) return rc;
        i = j;
    }
    return YFV2_OK;
}

}  // namespace
}  // namespace yfv2


extern "C" int yfv2_resize_bgr_u8(const yfv2_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::resize_entry<yfv2::BgrSource>("resize_bgr_u8", frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_yuv420_u8(const yfv2_yuv420_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::resize_entry<yfv2::Yuv420Source>("resize_yuv420_u8", frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_strided_u8(const yfv2_strided_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::resize_entry<yfv2::StridedSource>("resize_strided_u8", frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_yuv422_u8(const yfv2_yuv422_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::resize_entry<yfv2::Yuv422Source>("resize_yuv422_u8", frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_bayer_u8(const yfv2_bayer_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::resize_entry<yfv2::BayerSource>("resize_bayer_u8", frames, N, H, W, dst, stream);
}

extern "C" int yfv2_resize_remap_u8(const yfv2_remap_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::view_entry("resize_remap_u8", frames, N, H, W, dst, nullptr, stream);
}

extern "C" int yfv2_remap_u8(const yfv2_remap_frame* frames, int N, uint8_t* const* dst, void* stream) {
    return yfv2::view_entry("remap_u8", frames, N, 0, 0, nullptr, dst, stream);
}

extern "C" int yfv2_resize_warp_u8(const yfv2_warp_frame* frames, int N, int H, int W, uint8_t* dst, void* stream) {
    return yfv2::view_entry("resize_warp_u8", frames, N, H, W, dst, nullptr, stream);
}

extern "C" int yfv2_warp_u8(const yfv2_warp_frame* frames, int N, uint8_t* const* dst, void* stream) {
    return yfv2::view_entry("warp_u8", frames, N, 0, 0, nullptr, dst, stream);
}

extern "C" int yfv2_warp_matrix(const yfv2_warp_frame* frame, double* m_out) {
    if (!frame || !m_out) { yfv2::set_error("warp_matrix: null frame or m_out"); return YFV2_EINVAL; }
    double m[9];
    if (const char* why = yfv2::warp_matrix_fault(*frame, m)) { yfv2::set_error("warp_matrix: %s", why); return YFV2_EINVAL; }
    for (int k = 0; k < 9; ++k) m_out[k] = m[k];
    return YFV2_OK;
}

namespace yfv2 {

template <class Chunk>
int launch_aug_resize(const Chunk& a, int cnt, cudaStream_t stream) {
    const dim3 grid((unsigned)((a.W + kResizeBx - 1) / kResizeBx), (unsigned)((a.H + kResizeBy - 1) / kResizeBy), (unsigned)cnt);
    aug_resize_kernel<Chunk><<<grid, dim3(kResizeBx, kResizeBy), 0, stream>>>(a);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
template int launch_aug_resize<AugChunk>(const AugChunk&, int, cudaStream_t);
template int launch_aug_resize<AugBlurChunk>(const AugBlurChunk&, int, cudaStream_t);

}  // namespace yfv2
