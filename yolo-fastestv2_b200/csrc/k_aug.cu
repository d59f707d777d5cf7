// Device-side `contrast_and_brightness` (reference utils/datasets.py:10-16, the only augmentation img_aug applies, :63-68):
//   dst = cv2.addWeighted(img, alpha, zeros, 1 - alpha, beta)  on uint8 images
// i.e. per element  saturate_cast<uint8>( round_half_even( fl32(fl32(x * alpha) + beta) ) )  (the zero image contributes
// exactly 0; OpenCV evaluates the weighted sum in fp32 and rounds with cvRound).  One (alpha, beta) pair per image, drawn by
// the caller (the reference draws them with random.uniform on the host).  Pure byte streaming: 16 bytes per thread and trip.
//
// yfv2_aug_batch adds random_resize and augment_hsv (:54-61, :39-51) in img_aug's order; without the resize this file's
// aug_pixel_kernel runs it elementwise, with it k_resize.cu's aug_resize_kernel (aug.cuh holds the shared pixel arithmetic).
// yfv2_aug_batch_blur adds motion_blur (:18-37) between contrast and the resize: blur_kernel filters each blurred image into the
// workspace and reduces its byte range, then the same two kernels read it there through cv2.normalize's byte map.
// yfv2_aug_geometric (geom_kernel) runs YOLOv5's geometric steps before all of these: load_mosaic's canvas, random_perspective's
// warp with border 114 and fliplr, one output pixel per thread through resize.cuh's warp_pixel.
#include <cmath>
#include <vector>

#include "aug.cuh"
#include "resize.cuh"

namespace yfv2 {
namespace {

__device__ __forceinline__ unsigned aug_word(unsigned w, float alpha, float beta) {
    return aug_byte(w & 0xffu, alpha, beta) | (aug_byte((w >> 8) & 0xffu, alpha, beta) << 8) |
           (aug_byte((w >> 16) & 0xffu, alpha, beta) << 16) | (aug_byte(w >> 24, alpha, beta) << 24);
}

// img / out: [N][per_image] bytes; alpha / beta: [N]
__global__ void __launch_bounds__(256)
contrast_brightness_kernel(const uint8_t* __restrict__ img, uint8_t* __restrict__ out, const float* __restrict__ alpha,
                           const float* __restrict__ beta, long long per_image, int vec_ok) {
    const int n = blockIdx.y;
    const float a = __ldg(alpha + n), b = __ldg(beta + n);
    const uint8_t* src = img + (long long)n * per_image;
    uint8_t* dst = out + (long long)n * per_image;
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec_ok) {
        const long long nv = per_image >> 4;
        for (long long v = i; v < nv; v += stride) {
            uint4 q = __ldg(reinterpret_cast<const uint4*>(src) + v);
            q.x = aug_word(q.x, a, b); q.y = aug_word(q.y, a, b); q.z = aug_word(q.z, a, b); q.w = aug_word(q.w, a, b);
            reinterpret_cast<uint4*>(dst)[v] = q;
        }
        for (long long e = (nv << 4) + i; e < per_image; e += stride) dst[e] = (uint8_t)aug_byte(src[e], a, b);
    } else {
        for (long long e = i; e < per_image; e += stride) dst[e] = (uint8_t)aug_byte(src[e], a, b);
    }
}

// contrast (with kMap: the image's byte map instead), then augment_hsv when hsv is set, on the B, G, R of plane pixel e (row
// width W)
template <bool kMap>
__device__ __forceinline__ void aug_pixel(unsigned& b, unsigned& g, unsigned& r, float al, float be, const uint8_t* map, bool hsv,
                                          int e, int W, const HsvSmem& t) {
    if (kMap) {
        b = map[b]; g = map[g]; r = map[r];
    } else {
        b = aug_byte(b, al, be); g = aug_byte(g, al, be); r = aug_byte(r, al, be);
    }
    if (hsv) {
        int ib = (int)b, ig = (int)g, ir = (int)r;
        hsv_lut_pixel(ib, ig, ir, (W & 31) ? e % W : 0, W, t);          // only rows with a tail need the column
        b = (unsigned)ib; g = (unsigned)ig; r = (unsigned)ir;
    }
}

// yfv2_aug_batch without the resize: image blockIdx.y of the chunk, elementwise over its plane-sized B, G and R planes; 16
// pixels per thread and trip (one uint4 per plane) when vec_ok.  Each pixel is read before it is written by the same thread,
// so img == out is allowed.  With an AugBlurChunk a blurred image is read from the workspace through its normalize map.
template <class Chunk>
__global__ void __launch_bounds__(256)
aug_pixel_kernel(const __grid_constant__ Chunk a, long long plane, int vec_ok) {
    constexpr bool kBlur = AugTraits<Chunk>::kBlur;
    __shared__ typename AugTraits<Chunk>::Smem t;
    const int n = blockIdx.y;
    const bool hsv = a.luts != nullptr;
    if (hsv) {
        stage_hsv(t, a.luts + (size_t)n * 768);
        __syncthreads();
    }
    const float al = a.im[n].alpha, be = a.im[n].beta;
    const uint8_t* src = a.img + (size_t)n * 3 * plane;
    const uint8_t* map = nullptr;
    if constexpr (kBlur) {
        src = stage_map(t, a, n, 3 * plane);
        map = t.map;
        __syncthreads();
    }
    uint8_t* dst = a.out + (size_t)n * 3 * plane;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long e0 = 0;
    if (vec_ok) {
        const long long nv = plane >> 4;
        for (long long v = i; v < nv; v += stride) {
            const uint4 qb = __ldg(reinterpret_cast<const uint4*>(src) + v);
            const uint4 qg = __ldg(reinterpret_cast<const uint4*>(src + plane) + v);
            const uint4 qr = __ldg(reinterpret_cast<const uint4*>(src + 2 * plane) + v);
            const unsigned wb[4] = {qb.x, qb.y, qb.z, qb.w}, wg[4] = {qg.x, qg.y, qg.z, qg.w}, wr[4] = {qr.x, qr.y, qr.z, qr.w};
            unsigned ob[4] = {0, 0, 0, 0}, og[4] = {0, 0, 0, 0}, orr[4] = {0, 0, 0, 0};
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const int w = k >> 2, sh = 8 * (k & 3);
                unsigned b = (wb[w] >> sh) & 0xffu, g = (wg[w] >> sh) & 0xffu, r = (wr[w] >> sh) & 0xffu;
                aug_pixel<kBlur>(b, g, r, al, be, map, hsv, (int)(v * 16 + k), a.W, t);
                ob[w] |= b << sh; og[w] |= g << sh; orr[w] |= r << sh;
            }
            reinterpret_cast<uint4*>(dst)[v] = make_uint4(ob[0], ob[1], ob[2], ob[3]);
            reinterpret_cast<uint4*>(dst + plane)[v] = make_uint4(og[0], og[1], og[2], og[3]);
            reinterpret_cast<uint4*>(dst + 2 * plane)[v] = make_uint4(orr[0], orr[1], orr[2], orr[3]);
        }
        e0 = nv << 4;
    }
    for (long long e = e0 + i; e < plane; e += stride) {
        unsigned b = src[e], g = src[plane + e], r = src[2 * plane + e];
        aug_pixel<kBlur>(b, g, r, al, be, map, hsv, (int)e, a.W, t);
        dst[e] = (uint8_t)b; dst[plane + e] = (uint8_t)g; dst[2 * plane + e] = (uint8_t)r;
    }
}

// ---- motion_blur's first pass: contrast -> cv2.filter2D into the workspace, and the image's byte minimum and maximum ----------
// One CTA of 32 x 8 threads per 32 x 32 output tile of one blurred image (blockIdx.z).  The tile and a one-pixel
// BORDER_REFLECT_101 halo, through contrast, are staged as fp32 in shared memory; each thread runs the fused chain over the
// taps for 4 rows x 3 channels.  A 2 x 2 kernel (anchor (1, 1): offsets -1..0) travels in the upper left of a 3 x 3 over
// offsets -1..1 with zeros elsewhere: an fma with a zero tap adds +0 to a sum that is >= 0, so the chain is unchanged.
constexpr int kBlurMax = 64;                        // blurred images per launch (their taps travel as kernel parameters)
constexpr int kBlurTx = 32, kBlurTy = 8, kBlurRows = 4;
struct BlurImage {
    int n;                                          // image index in the batch
    float alpha, beta;                              // contrast (1, 0 when off)
    float taps[9];                                  // 3 x 3 row-major over offsets -1..1
};
struct BlurPass {
    BlurImage im[kBlurMax];
    const uint8_t* img;                             // image 0 of the batch
    uint8_t* ws;                                    // image 0 of the batch; mm = the min / max slots, 2 per image
    unsigned* mm;
    int H, W;
};

// BORDER_REFLECT_101 of index i in -1..n (cv2 maps every index of a 1-long axis to 0)
__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    i = i < 0 ? -i : i;
    return i >= n ? 2 * n - 2 - i : i;
}

__global__ void __launch_bounds__(kBlurTx * kBlurTy)
blur_kernel(const __grid_constant__ BlurPass p) {
    constexpr int TW = kBlurTx + 2, TH = kBlurTy * kBlurRows + 2, NT = kBlurTx * kBlurTy;
    __shared__ float s[3][TH][TW];
    __shared__ unsigned red[2][NT / 32];
    const BlurImage& im = p.im[blockIdx.z];
    const int H = p.H, W = p.W, tid = threadIdx.y * kBlurTx + threadIdx.x;
    const size_t plane = (size_t)H * W;
    const uint8_t* src = p.img + (size_t)im.n * 3 * plane;
    const int x0 = blockIdx.x * kBlurTx, y0 = blockIdx.y * (kBlurTy * kBlurRows);
    for (int i = tid; i < 3 * TH * TW; i += NT) {
        const int c = i / (TH * TW), r = (i / TW) % TH, q = i % TW;
        const int y = reflect101(min(y0 + r - 1, H), H), x = reflect101(min(x0 + q - 1, W), W);   // beyond W or H: never used
        s[c][r][q] = (float)aug_byte(__ldg(src + c * plane + (size_t)y * W + x), im.alpha, im.beta);
    }
    float k[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) k[j] = im.taps[j];
    __syncthreads();
    unsigned lo = 255u, hi = 0u;
    uint8_t* dst = p.ws + (size_t)im.n * 3 * plane;
    const int x = x0 + threadIdx.x;
#pragma unroll
    for (int rr = 0; rr < kBlurRows; ++rr) {
        const int ty = threadIdx.y + rr * kBlurTy, y = y0 + ty;
        if (x < W && y < H) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float acc = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) acc = __fmaf_rn(s[c][ty + i][threadIdx.x + j], k[3 * i + j], acc);
                const unsigned v = (unsigned)fminf(fmaxf(rintf(acc), 0.f), 255.f);
                dst[c * plane + (size_t)y * W + x] = (uint8_t)v;
                lo = min(lo, v);
                hi = max(hi, v);
            }
        }
    }
    lo = __reduce_min_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    if ((tid & 31) == 0) { red[0][tid >> 5] = lo; red[1][tid >> 5] = hi; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < NT / 32; ++w) { lo = min(lo, red[0][w]); hi = max(hi, red[1][w]); }
        atomicMax(p.mm + 2 * im.n, hi);
        atomicMax(p.mm + 2 * im.n + 1, 255u - lo);
    }
}

// yfv2_debug_bgr2hsv / _hsv2bgr: n packed 3-byte pixels in rows of row_w (HSV -> BGR depends on the column)
__global__ void __launch_bounds__(256) hsv_debug_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, long long n,
                                                        int row_w, int to_hsv) {
    __shared__ HsvSmem t;
    stage_hsv(t, nullptr);
    __syncthreads();
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
        const int x0 = in[3 * p], x1 = in[3 * p + 1], x2 = in[3 * p + 2];
        int y0, y1, y2;
        if (to_hsv) bgr_to_hsv(x0, x1, x2, t, y0, y1, y2);
        else hsv_to_bgr(x0, x1, x2, (int)(p % row_w) >= (row_w & ~31), y0, y1, y2);
        out[3 * p] = (uint8_t)y0; out[3 * p + 1] = (uint8_t)y1; out[3 * p + 2] = (uint8_t)y2;
    }
}

int debug_hsv(const uint8_t* in, uint8_t* out, long long n, int row_w, int to_hsv, void* stream) {
    if (!in || !out || n <= 0 || row_w <= 0) {
        set_error("debug_%s: null in / out, n <= 0 or row_w <= 0", to_hsv ? "bgr2hsv" : "hsv2bgr");
        return YFV2_EINVAL;
    }
    long long blocks = (n + 255) / 256;
    if (blocks > 8 * sm_count()) blocks = 8 * sm_count();
    hsv_debug_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(in, out, n, row_w, to_hsv);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

constexpr int kAugMaxSide = 32768;

// The blur workspace: [N][3][H][W] filtered bytes, then (256-byte aligned) the [N][2] min / max slots
size_t blur_ws_mm_offset(int N, int H, int W) { return ((size_t)N * 3 * H * W + 255) & ~(size_t)255; }
size_t blur_ws_bytes(int N, int H, int W) { return blur_ws_mm_offset(N, H, W) + (size_t)N * 2 * sizeof(unsigned); }

bool overlaps(uintptr_t a, size_t na, uintptr_t b, size_t nb) { return a < b + nb && b < a + na; }

// yfv2_aug_batch (allowed = YFV2_AUG_ALL, blur null) and yfv2_aug_batch_blur: every check, then the launches
int aug_batch(const char* fn, int allowed, const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_params* params,
              const uint8_t* luts, const yfv2_aug_blur* blur, int flags, uint8_t* ws, size_t ws_bytes, void* stream) {
    if (!img || !out || !params || N <= 0) { set_error("%s: null img / out / params or N <= 0", fn); return YFV2_EINVAL; }
    if (H <= 0 || W <= 0 || H > kAugMaxSide || W > kAugMaxSide) {
        set_error("%s: image %dx%d outside 1..%d", fn, W, H, kAugMaxSide);
        return YFV2_EINVAL;
    }
    if (flags & ~allowed) { set_error("%s: unknown flags 0x%x", fn, flags & ~allowed); return YFV2_EINVAL; }
    const bool resize = flags & YFV2_AUG_RESIZE, hsv = flags & YFV2_AUG_HSV, contrast = flags & YFV2_AUG_CONTRAST;
    const bool blurring = flags & YFV2_AUG_BLUR;
    if (hsv && !luts) { set_error("%s: YFV2_AUG_HSV needs luts", fn); return YFV2_EINVAL; }
    const size_t plane = (size_t)H * W, bytes = (size_t)N * 3 * plane;
    int nblur = 0;
    if (blurring) {
        if (!blur) { set_error("%s: YFV2_AUG_BLUR needs blur descriptors", fn); return YFV2_EINVAL; }
        if (!ws || ws_bytes < blur_ws_bytes(N, H, W)) {
            set_error("%s: YFV2_AUG_BLUR needs a workspace of %zu bytes (got %zu%s)", fn, blur_ws_bytes(N, H, W), ws_bytes,
                      ws ? "" : ", null");
            return YFV2_EINVAL;
        }
        for (int n = 0; n < N; ++n) {
            const int k = blur[n].ksize;
            if (k != 0 && k != 2 && k != 3) { set_error("%s: image %d: blur ksize %d not 0, 2 or 3", fn, n, k); return YFV2_EINVAL; }
            for (int j = 0; j < k * k; ++j) {
                if (!std::isfinite(blur[n].taps[j])) { set_error("%s: image %d: blur tap %d is not finite", fn, n, j); return YFV2_EINVAL; }
            }
            nblur += k != 0;
        }
    }
    const uintptr_t pi = reinterpret_cast<uintptr_t>(img), po = reinterpret_cast<uintptr_t>(out);
    if (pi < po + bytes && po < pi + bytes && (resize || pi != po)) {
        set_error("%s: img and out overlap (%s)", fn, resize ? "YFV2_AUG_RESIZE reads neighbours: use another buffer"
                                                            : "only img == out is allowed");
        return YFV2_EINVAL;
    }
    const uintptr_t pw = reinterpret_cast<uintptr_t>(ws);
    if (blurring && (overlaps(pw, ws_bytes, pi, bytes) || overlaps(pw, ws_bytes, po, bytes))) {
        set_error("%s: the workspace overlaps img or out", fn);
        return YFV2_EINVAL;
    }
    if (resize) {
        for (int n = 0; n < N; ++n) {
            if (params[n].rw < 1 || params[n].rw > W || params[n].rh < 1 || params[n].rh > H) {
                set_error("%s: image %d: random_resize size %dx%d outside 1..%d x 1..%d", fn, n, params[n].rw, params[n].rh, W, H);
                return YFV2_EINVAL;
            }
        }
    }
    unsigned* mm = nblur ? reinterpret_cast<unsigned*>(ws + blur_ws_mm_offset(N, H, W)) : nullptr;
    if (nblur) {                                     // first pass: every blurred image into the workspace
        YFV2_CUDA(cudaMemsetAsync(mm, 0, (size_t)N * 2 * sizeof(unsigned), (cudaStream_t)stream));
        BlurPass bp{};
        bp.img = img; bp.ws = ws; bp.mm = mm; bp.H = H; bp.W = W;
        const dim3 block(kBlurTx, kBlurTy);
        int cnt = 0;
        for (int n = 0; n < N; ++n) {
            const int k = blur[n].ksize;
            if (k) {
                BlurImage& b = bp.im[cnt++];
                b.n = n;
                b.alpha = contrast ? params[n].alpha : 1.f;
                b.beta = contrast ? params[n].beta : 0.f;
                for (int j = 0; j < 9; ++j) b.taps[j] = 0.f;
                for (int i = 0; i < k; ++i)
                    for (int j = 0; j < k; ++j) b.taps[3 * i + j] = blur[n].taps[k * i + j];
            }
            if (cnt == kBlurMax || (cnt && n == N - 1)) {
                const dim3 grid((unsigned)((W + kBlurTx - 1) / kBlurTx), (unsigned)((H + kBlurTy * kBlurRows - 1) / (kBlurTy * kBlurRows)),
                                (unsigned)cnt);
                blur_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(bp);
                YFV2_LAUNCH_CHECK();
                cnt = 0;
            }
        }
    }
    const int vec_ok = pi % 16 == 0 && po % 16 == 0 && plane % 16 == 0;
    long long blocks = ((long long)(plane / 16) + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
    for (int n0 = 0; n0 < N; n0 += kAugChunk) {
        const int cnt = N - n0 < kAugChunk ? N - n0 : kAugChunk;
        AugBlurChunk a{};
        for (int i = 0; i < cnt; ++i) {
            a.im[i] = params[n0 + i];
            if (!contrast) { a.im[i].alpha = 1.f; a.im[i].beta = 0.f; }
            if (nblur && blur[n0 + i].ksize) a.blurred[i >> 5] |= 1u << (i & 31);
        }
        a.img = img + (size_t)n0 * 3 * plane;
        a.out = out + (size_t)n0 * 3 * plane;
        a.luts = hsv ? luts + (size_t)n0 * 768 : nullptr;
        a.H = H; a.W = W;
        bool any = false;
        for (unsigned m : a.blurred) any |= m != 0;
        if (any) {                                   // second pass with the workspace: only chunks with a blurred image
            a.ws = ws + (size_t)n0 * 3 * plane;
            a.mm = mm + 2 * n0;
            if (resize) {
                const int rc = launch_aug_resize(a, cnt, (cudaStream_t)stream);
                if (rc != YFV2_OK) return rc;
            } else {
                aug_pixel_kernel<AugBlurChunk><<<dim3((unsigned)blocks, (unsigned)cnt), 256, 0, (cudaStream_t)stream>>>(
                    a, (long long)plane, vec_ok && pw % 16 == 0);
                YFV2_LAUNCH_CHECK();
            }
        } else if (resize) {
            const int rc = launch_aug_resize(static_cast<const AugChunk&>(a), cnt, (cudaStream_t)stream);
            if (rc != YFV2_OK) return rc;
        } else {
            aug_pixel_kernel<AugChunk><<<dim3((unsigned)blocks, (unsigned)cnt), 256, 0, (cudaStream_t)stream>>>(
                static_cast<const AugChunk&>(a), (long long)plane, vec_ok);
            YFV2_LAUNCH_CHECK();
        }
    }
    return YFV2_OK;
}

// ---- yfv2_aug_geometric: load_mosaic's canvas -> random_perspective's warp (border 114) -> fliplr ---------------------------------
constexpr int kGeomBorder = 114;                    // load_mosaic's fill and random_perspective's borderValue
constexpr int kGeomBx = 64, kGeomBy = 4;
constexpr int kGeomMaxCanvas = 32767;               // SHRT_MAX: cv2.remap refuses sources this large, warp_pixel saturates there

// load_mosaic's 2W x 2H canvas of four W x H planar images of the batch around (xc, yc)
struct MosaicFrame {
    const uint8_t* img;                             // image 0 of the batch, [N][3][th][tw]
    int src[4];                                     // top-left, top-right, bottom-left, bottom-right
    int xc, yc;
    int w, h;                                       // the canvas, 2 tw x 2 th: sample_fixed's bounds
    int tw, th;                                     // one tile (a batch image)
};

// Canvas pixel (r, c) is tile 2 (r >= yc) + (c >= xc) at local (c - xc + tw (c < xc), r - yc + th (r < yc)), and kGeomBorder
// where that falls outside the tile.  The row's two tiles are found once per row.
struct MosaicSource {
    using Desc = MosaicFrame;
    const uint8_t* left;                            // the row's left and right tiles at the local row
    const uint8_t* right;
    long long plane;
    int xc, tw;
    bool row_in;
    __device__ __forceinline__ MosaicSource(const MosaicFrame& f, int r) : plane((long long)f.tw * f.th), xc(f.xc), tw(f.tw) {
        const int below = r >= f.yc;
        const int lr = r - f.yc + (below ? 0 : f.th);
        row_in = (unsigned)lr < (unsigned)f.th;
        const long long off = row_in ? (long long)lr * f.tw : 0;
        left = f.img + 3 * plane * f.src[2 * below] + off;
        right = f.img + 3 * plane * f.src[2 * below + 1] + off;
    }
    __device__ __forceinline__ void pixel(int c, int (&p)[3]) const {
        const bool r = c >= xc;
        const int lc = c - xc + (r ? 0 : tw);
        const bool in = row_in && (unsigned)lc < (unsigned)tw;
        const uint8_t* q = (r ? right : left) + (in ? lc : 0);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) p[ch] = in ? __ldg(q + ch * plane) : kGeomBorder;
    }
    __device__ __forceinline__ void fetch(int c0, int c1, int (&p0)[3], int (&p1)[3]) const {
        pixel(c0, p0);
        pixel(c1, p1);
    }
};

// Images of one canvas kind (MosaicSource, or StridedSource over one planar batch image): each warp descriptor (the canvas, M
// inverted, the window (0, 0, W, H)), its output image and flip, under the 4 KB launch limit with the chunk's rest
template <class Inner>
struct GeomChunk {
    static constexpr int kChunk = 3968 / (int)(sizeof(WarpDesc<Inner>) + sizeof(int) + 1);
    WarpDesc<Inner> d[kChunk];
    int n[kChunk];
    uint8_t flip[kChunk];
    uint8_t* out;                                   // image 0 of the batch
    int H, W;
};
static_assert(sizeof(GeomChunk<MosaicSource>) <= 4000 && sizeof(GeomChunk<StridedSource>) <= 4000, "kernel parameters over 4 KB");

// One thread per output pixel of image a.n[blockIdx.z]: the warp's pixel at the flipped column, written to the three planes
template <class Inner>
__global__ void __launch_bounds__(kGeomBx * kGeomBy)
geom_kernel(const __grid_constant__ GeomChunk<Inner> a) {
    const int x = blockIdx.x * kGeomBx + threadIdx.x;
    const int y = blockIdx.y * kGeomBy + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const int i = blockIdx.z;
    int v[3];
    warp_pixel<Inner, kGeomBorder>(a.d[i], a.flip[i] ? a.W - 1 - x : x, y, v);
    const size_t plane = (size_t)a.H * a.W;
    uint8_t* out = a.out + (size_t)a.n[i] * 3 * plane + (size_t)y * a.W + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * plane] = (uint8_t)v[c];
}

// The canvas of a checked image: the mosaic, or the planar image src[0] as a strided frame
inline void geom_canvas(MosaicFrame& f, const yfv2_aug_geom& p, const uint8_t* img, int H, int W) {
    f = MosaicFrame{img, {p.src[0], p.src[1], p.src[2], p.src[3]}, p.xc, p.yc, 2 * W, 2 * H, W, H};
}
inline void geom_canvas(yfv2_strided_frame& f, const yfv2_aug_geom& p, const uint8_t* img, int H, int W) {
    const size_t plane = (size_t)H * W;
    const uint8_t* b = img + 3 * plane * p.src[0];
    f = yfv2_strided_frame{b, b + plane, b + 2 * plane, W, 1, W, H};
}

// The matrix check of yfv2_warp_matrix (warp_matrix_fault) for M with dsize (W, H); m gets the output -> canvas matrix
inline const char* geom_matrix_fault(const yfv2_aug_geom& p, int H, int W, double (&m)[9]) {
    yfv2_warp_frame wf{};
    for (int k = 0; k < 9; ++k) wf.m[k] = p.m[k];
    wf.perspective = p.perspective;
    wf.dw = W;
    wf.dh = H;
    return warp_matrix_fault(wf, m);
}

// The images idx[0, cnt), all of Inner's canvas kind, GeomChunk<Inner>::kChunk per launch
template <class Inner>
int launch_geom(const yfv2_aug_geom* params, const int* idx, int cnt, const uint8_t* img, uint8_t* out, int H, int W,
                cudaStream_t stream) {
    using Chunk = GeomChunk<Inner>;
    for (int i0 = 0; i0 < cnt; i0 += Chunk::kChunk) {
        const int k = cnt - i0 < Chunk::kChunk ? cnt - i0 : Chunk::kChunk;
        Chunk a{};
        for (int i = 0; i < k; ++i) {
            const yfv2_aug_geom& p = params[idx[i0 + i]];
            WarpDesc<Inner>& d = a.d[i];
            geom_canvas(d.f, p, img, H, W);
            geom_matrix_fault(p, H, W, d.m);                // checked
            d.perspective = p.perspective;
            d.x0 = 0; d.y0 = 0; d.w = W; d.h = H;
            a.n[i] = idx[i0 + i];
            a.flip[i] = (uint8_t)p.flip;
        }
        a.out = out;
        a.H = H; a.W = W;
        const dim3 grid((unsigned)((W + kGeomBx - 1) / kGeomBx), (unsigned)((H + kGeomBy - 1) / kGeomBy), (unsigned)k);
        geom_kernel<Inner><<<grid, dim3(kGeomBx, kGeomBy), 0, stream>>>(a);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}

// yfv2_aug_geometric: every check, then one launch sequence for the mosaic images and one for the others
int aug_geometric(const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_geom* params, void* stream) {
    const char* fn = "aug_geometric";
    if (!img || !out || !params || N <= 0) { set_error("%s: null img / out / params or N <= 0", fn); return YFV2_EINVAL; }
    if (H <= 0 || W <= 0 || H > kAugMaxSide || W > kAugMaxSide) {
        set_error("%s: image %dx%d outside 1..%d", fn, W, H, kAugMaxSide);
        return YFV2_EINVAL;
    }
    const size_t bytes = (size_t)N * 3 * H * W;
    if (overlaps(reinterpret_cast<uintptr_t>(img), bytes, reinterpret_cast<uintptr_t>(out), bytes)) {
        set_error("%s: img and out overlap (a mosaic reads other images: use another buffer)", fn);
        return YFV2_EINVAL;
    }
    for (int n = 0; n < N; ++n) {
        const yfv2_aug_geom& p = params[n];
        if ((p.perspective | p.mosaic | p.flip) & ~1) {
            set_error("%s: image %d: perspective, mosaic and flip must be 0 or 1 (got %d, %d, %d)", fn, n, p.perspective, p.mosaic,
                      p.flip);
            return YFV2_EINVAL;
        }
        for (int t = 0; t < (p.mosaic ? 4 : 1); ++t) {
            if (p.src[t] < 0 || p.src[t] >= N) {
                set_error("%s: image %d: src[%d] = %d outside [0, %d)", fn, n, t, p.src[t], N);
                return YFV2_EINVAL;
            }
        }
        const int cw = p.mosaic ? 2 * W : W, ch = p.mosaic ? 2 * H : H;
        if (cw >= kGeomMaxCanvas || ch >= kGeomMaxCanvas) {
            set_error("%s: image %d: %s canvas %dx%d: its sides must be below %d (cv2.remap's limit; the fixed-point source "
                      "coordinate saturates there)", fn, n, p.mosaic ? "mosaic" : "image", cw, ch, kGeomMaxCanvas);
            return YFV2_EINVAL;
        }
        if (p.mosaic) {
            if ((H | W) & 1) { set_error("%s: image %d: mosaic needs even H and W (got %dx%d)", fn, n, W, H); return YFV2_EINVAL; }
            if (p.xc < W / 2 || p.xc > 2 * W - W / 2 || p.yc < H / 2 || p.yc > 2 * H - H / 2) {
                set_error("%s: image %d: mosaic centre (%d, %d) outside [%d, %d] x [%d, %d]", fn, n, p.xc, p.yc, W / 2,
                          2 * W - W / 2, H / 2, 2 * H - H / 2);
                return YFV2_EINVAL;
            }
        }
        double m[9];
        if (const char* why = geom_matrix_fault(p, H, W, m)) {
            set_error("%s: image %d: %s (%s M, dsize %dx%d)", fn, n, why, p.perspective ? "perspective" : "affine", W, H);
            return YFV2_EINVAL;
        }
    }
    std::vector<int> idx;
    for (int mosaic = 0; mosaic < 2; ++mosaic) {
        idx.clear();
        for (int n = 0; n < N; ++n)
            if (params[n].mosaic == mosaic) idx.push_back(n);
        if (idx.empty()) continue;
        const int cnt = (int)idx.size();
        const int rc = mosaic ? launch_geom<MosaicSource>(params, idx.data(), cnt, img, out, H, W, (cudaStream_t)stream)
                              : launch_geom<StridedSource>(params, idx.data(), cnt, img, out, H, W, (cudaStream_t)stream);
        if (rc != YFV2_OK) return rc;
    }
    return YFV2_OK;
}

}  // namespace
}  // namespace yfv2

extern "C" int yfv2_aug_geometric(const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_geom* params,
                                  void* stream) {
    return yfv2::aug_geometric(img, out, N, H, W, params, stream);
}

extern "C" int yfv2_aug_contrast_brightness(const uint8_t* img, uint8_t* out, const float* alpha, const float* beta, int N,
                                            long long bytes_per_image, void* stream) {
    using namespace yfv2;
    if (!img || !out || !alpha || !beta || N <= 0 || bytes_per_image <= 0) { set_error("aug_contrast_brightness: bad argument"); return YFV2_EINVAL; }
    const int vec_ok = (reinterpret_cast<uintptr_t>(img) % 16 == 0) && (reinterpret_cast<uintptr_t>(out) % 16 == 0) && (bytes_per_image % 16 == 0);
    long long blocks = (bytes_per_image / 16 + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
    contrast_brightness_kernel<<<dim3((unsigned)blocks, (unsigned)N), 256, 0, (cudaStream_t)stream>>>(img, out, alpha, beta, bytes_per_image, vec_ok);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_aug_batch(const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_params* params,
                              const uint8_t* luts, int flags, void* stream) {
    return yfv2::aug_batch("aug_batch", YFV2_AUG_ALL, img, out, N, H, W, params, luts, nullptr, flags, nullptr, 0, stream);
}

extern "C" int yfv2_aug_blur_workspace_bytes(int N, int H, int W, size_t* bytes) {
    using namespace yfv2;
    if (!bytes || N <= 0 || H <= 0 || W <= 0 || H > kAugMaxSide || W > kAugMaxSide) {
        set_error("aug_blur_workspace_bytes: null bytes, N <= 0 or image %dx%d outside 1..%d", W, H, kAugMaxSide);
        return YFV2_EINVAL;
    }
    *bytes = blur_ws_bytes(N, H, W);
    return YFV2_OK;
}

extern "C" int yfv2_aug_batch_blur(const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_params* params,
                                   const uint8_t* luts, const yfv2_aug_blur* blur, int flags, void* workspace,
                                   size_t workspace_bytes, void* stream) {
    return yfv2::aug_batch("aug_batch_blur", YFV2_AUG_ALL | YFV2_AUG_BLUR, img, out, N, H, W, params, luts, blur, flags,
                           static_cast<uint8_t*>(workspace), workspace_bytes, stream);
}

extern "C" int yfv2_debug_bgr2hsv(const uint8_t* in, uint8_t* out, long long n, void* stream) {
    return yfv2::debug_hsv(in, out, n, 1, 1, stream);
}

extern "C" int yfv2_debug_hsv2bgr(const uint8_t* in, uint8_t* out, long long n, int row_w, void* stream) {
    return yfv2::debug_hsv(in, out, n, row_w, 0, stream);
}
