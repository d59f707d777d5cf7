// Device-side `contrast_and_brightness` (reference utils/datasets.py:10-16, the only augmentation img_aug applies, :63-68):
//   dst = cv2.addWeighted(img, alpha, zeros, 1 - alpha, beta)  on uint8 images
// i.e. per element  saturate_cast<uint8>( round_half_even( fl32(fl32(x * alpha) + beta) ) )  (the zero image contributes
// exactly 0; OpenCV evaluates the weighted sum in fp32 and rounds with cvRound).  One (alpha, beta) pair per image, drawn by
// the caller (the reference draws them with random.uniform on the host).  Pure byte streaming: 16 bytes per thread and trip.
//
// yfv2_aug_batch adds random_resize and augment_hsv (:54-61, :39-51) in img_aug's order; without the resize this file's
// aug_pixel_kernel runs it elementwise, with it k_resize.cu's aug_resize_kernel (aug.cuh holds the shared pixel arithmetic).
#include "aug.cuh"

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

// contrast, then augment_hsv when hsv is set, on the B, G, R of plane pixel e (row width W)
__device__ __forceinline__ void aug_pixel(unsigned& b, unsigned& g, unsigned& r, float al, float be, bool hsv, int e, int W,
                                          const HsvSmem& t) {
    b = aug_byte(b, al, be); g = aug_byte(g, al, be); r = aug_byte(r, al, be);
    if (hsv) {
        int ib = (int)b, ig = (int)g, ir = (int)r;
        hsv_lut_pixel(ib, ig, ir, (W & 31) ? e % W : 0, W, t);          // only rows with a tail need the column
        b = (unsigned)ib; g = (unsigned)ig; r = (unsigned)ir;
    }
}

// yfv2_aug_batch without the resize: image blockIdx.y of the chunk, elementwise over its plane-sized B, G and R planes; 16
// pixels per thread and trip (one uint4 per plane) when vec_ok.  Each pixel is read before it is written by the same thread,
// so img == out is allowed.
__global__ void __launch_bounds__(256)
aug_pixel_kernel(const __grid_constant__ AugChunk a, long long plane, int vec_ok) {
    __shared__ HsvSmem t;
    const int n = blockIdx.y;
    const bool hsv = a.luts != nullptr;
    if (hsv) {
        stage_hsv(t, a.luts + (size_t)n * 768);
        __syncthreads();
    }
    const float al = a.im[n].alpha, be = a.im[n].beta;
    const uint8_t* src = a.img + (size_t)n * 3 * plane;
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
                aug_pixel(b, g, r, al, be, hsv, (int)(v * 16 + k), a.W, t);
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
        aug_pixel(b, g, r, al, be, hsv, (int)e, a.W, t);
        dst[e] = (uint8_t)b; dst[plane + e] = (uint8_t)g; dst[2 * plane + e] = (uint8_t)r;
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

}  // namespace
}  // namespace yfv2

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
    using namespace yfv2;
    if (!img || !out || !params || N <= 0) { set_error("aug_batch: null img / out / params or N <= 0"); return YFV2_EINVAL; }
    if (H <= 0 || W <= 0 || H > kAugMaxSide || W > kAugMaxSide) {
        set_error("aug_batch: image %dx%d outside 1..%d", W, H, kAugMaxSide);
        return YFV2_EINVAL;
    }
    if (flags & ~YFV2_AUG_ALL) { set_error("aug_batch: unknown flags 0x%x", flags & ~YFV2_AUG_ALL); return YFV2_EINVAL; }
    const bool resize = flags & YFV2_AUG_RESIZE, hsv = flags & YFV2_AUG_HSV, contrast = flags & YFV2_AUG_CONTRAST;
    if (hsv && !luts) { set_error("aug_batch: YFV2_AUG_HSV needs luts"); return YFV2_EINVAL; }
    const size_t plane = (size_t)H * W, bytes = (size_t)N * 3 * plane;
    const uintptr_t pi = reinterpret_cast<uintptr_t>(img), po = reinterpret_cast<uintptr_t>(out);
    if (pi < po + bytes && po < pi + bytes && (resize || pi != po)) {
        set_error("aug_batch: img and out overlap (%s)", resize ? "YFV2_AUG_RESIZE reads neighbours: use another buffer"
                                                               : "only img == out is allowed");
        return YFV2_EINVAL;
    }
    if (resize) {
        for (int n = 0; n < N; ++n) {
            if (params[n].rw < 1 || params[n].rw > W || params[n].rh < 1 || params[n].rh > H) {
                set_error("aug_batch: image %d: random_resize size %dx%d outside 1..%d x 1..%d", n, params[n].rw, params[n].rh, W, H);
                return YFV2_EINVAL;
            }
        }
    }
    const int vec_ok = pi % 16 == 0 && po % 16 == 0 && plane % 16 == 0;
    long long blocks = ((long long)(plane / 16) + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
    for (int n0 = 0; n0 < N; n0 += kAugChunk) {
        const int cnt = N - n0 < kAugChunk ? N - n0 : kAugChunk;
        AugChunk a{};
        for (int i = 0; i < cnt; ++i) {
            a.im[i] = params[n0 + i];
            if (!contrast) { a.im[i].alpha = 1.f; a.im[i].beta = 0.f; }
        }
        a.img = img + (size_t)n0 * 3 * plane;
        a.out = out + (size_t)n0 * 3 * plane;
        a.luts = hsv ? luts + (size_t)n0 * 768 : nullptr;
        a.H = H; a.W = W;
        if (resize) {
            const int rc = launch_aug_resize(a, cnt, (cudaStream_t)stream);
            if (rc != YFV2_OK) return rc;
        } else {
            aug_pixel_kernel<<<dim3((unsigned)blocks, (unsigned)cnt), 256, 0, (cudaStream_t)stream>>>(a, (long long)plane, vec_ok);
            YFV2_LAUNCH_CHECK();
        }
    }
    return YFV2_OK;
}

extern "C" int yfv2_debug_bgr2hsv(const uint8_t* in, uint8_t* out, long long n, void* stream) {
    return yfv2::debug_hsv(in, out, n, 1, 1, stream);
}

extern "C" int yfv2_debug_hsv2bgr(const uint8_t* in, uint8_t* out, long long n, int row_w, void* stream) {
    return yfv2::debug_hsv(in, out, n, row_w, 0, stream);
}
