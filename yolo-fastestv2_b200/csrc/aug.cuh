// Per-pixel arithmetic of the reference's img_aug (utils/datasets.py:10-16, :39-51) shared by the augmentation kernels of
// k_aug.cu (elementwise) and k_resize.cu (with the nested random_resize).
#pragma once
#include "common.cuh"

#define YFV2_AUG_ALL (YFV2_AUG_CONTRAST | YFV2_AUG_RESIZE | YFV2_AUG_HSV)

namespace yfv2 {

// contrast_and_brightness of one byte: cv2.addWeighted(img, alpha, zeros, 1 - alpha, beta) on uint8 (k_aug.cu's header)
__device__ __forceinline__ unsigned aug_byte(unsigned b, float alpha, float beta) {
    const float t = __fadd_rn(__fmul_rn((float)b, alpha), beta);
    const float r = fminf(fmaxf(rintf(t), 0.f), 255.f);      // rintf: round half to even (cvRound)
    return (unsigned)r;
}

// augment_hsv's per-image state in shared memory: cv2's BGR2HSV division tables and the image's three LUTs
struct HsvSmem {
    int sdiv[256], hdiv[256];
    uint8_t lut[3][256];   // H, S, V
};

// Fills t's tables and, when luts is set, its LUTs from the image's [3][256] bytes (global memory).  Needs at least 256 threads
// per block; the caller synchronises.
__device__ __forceinline__ void stage_hsv(HsvSmem& t, const uint8_t* __restrict__ luts) {
    const int i = threadIdx.x + threadIdx.y * blockDim.x;
    if (i < 256) {
        // cv2's 8-bit tables (hsv_shift 12): cvRound((255 << 12) / i), cvRound((180 << 12) / (6 i)); entry 0 is 0
        t.sdiv[i] = i ? __double2int_rn(1044480.0 / (double)i) : 0;
        t.hdiv[i] = i ? __double2int_rn(737280.0 / (6.0 * (double)i)) : 0;
        if (luts) {
            t.lut[0][i] = __ldg(luts + i);
            t.lut[1][i] = __ldg(luts + 256 + i);
            t.lut[2][i] = __ldg(luts + 512 + i);
        }
    }
}

// cv2.cvtColor(COLOR_BGR2HSV) of one 8-bit pixel (OpenCV's integer path, hsv_shift 12, H in 0..179)
__device__ __forceinline__ void bgr_to_hsv(int b, int g, int r, const HsvSmem& t, int& h, int& s, int& v) {
    v = max(max(b, g), r);
    const int diff = v - min(min(b, g), r);
    s = (diff * t.sdiv[v] + 2048) >> 12;
    const int hh = v == r ? g - b : v == g ? b - r + 2 * diff : r - g + 4 * diff;
    h = (hh * t.hdiv[diff] + 2048) >> 12;
    if (h < 0) h += 180;
}

// cv2.cvtColor(COLOR_HSV2BGR) of one 8-bit pixel, any H in 0..255: fp32 with s and v scaled by fl(1/255), h by fl(6/180);
// 1 - s*h and 1 - s*(1 - h) are single fused roundings; the channel is x * 255 truncated, or rounded to nearest even in a row's
// tail.  OpenCV 4.13 (x86, AVX2) converts each row 32 pixels at a time with vector code that truncates, and the last W mod 32
// pixels of a row with scalar code that rounds: `tail` is column >= W - W mod 32.  Bit-identical over all 2^24 triples on both
// paths (tests/golden/aug_hsv_cases.npz).
__device__ __forceinline__ int hsv_channel(float x, bool tail) {
    const float y = __fmul_rn(x, 255.f);
    return min(max(tail ? __float2int_rn(y) : __float2int_rz(y), 0), 255);
}
__device__ __forceinline__ float pick(unsigned sel, float t0, float t1, float t2, float t3) {
    return sel == 0 ? t0 : sel == 1 ? t1 : sel == 2 ? t2 : t3;
}
__device__ __forceinline__ void hsv_to_bgr(int h, int s, int v, bool tail, int& b, int& g, int& r) {
    const float hf = __fmul_rn((float)h, (float)(6.0 / 180.0));
    const float sf = __fmul_rn((float)s, (float)(1.0 / 255.0));
    const float vf = __fmul_rn((float)v, (float)(1.0 / 255.0));
    const float fl = floorf(hf);
    const float f = __fsub_rn(hf, fl);
    int sector = (int)fl;                                          // 0..8
    if (sector >= 6) sector -= 6;
    const float t1 = __fmul_rn(vf, __fsub_rn(1.f, sf));
    const float t2 = __fmul_rn(vf, __fmaf_rn(-sf, f, 1.f));
    const float t3 = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.f, f), 1.f));
    // OpenCV's sector table {{1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}} (B, G, R), 2 bits per sector
    const unsigned sh = 2u * (unsigned)sector;
    b = hsv_channel(pick((0x835u >> sh) & 3u, vf, t1, t2, t3), tail);
    g = hsv_channel(pick((0x583u >> sh) & 3u, vf, t1, t2, t3), tail);
    r = hsv_channel(pick((0x358u >> sh) & 3u, vf, t1, t2, t3), tail);
}

// augment_hsv's device part on one pixel of column col of a W-wide row: BGR -> HSV, the three LUTs, HSV -> BGR
__device__ __forceinline__ void hsv_lut_pixel(int& b, int& g, int& r, int col, int W, const HsvSmem& t) {
    int h, s, v;
    bgr_to_hsv(b, g, r, t, h, s, v);
    hsv_to_bgr(t.lut[0][h], t.lut[1][s], t.lut[2][v], col >= (W & ~31), b, g, r);
}

// One launch of yfv2_aug_batch: up to kAugChunk [3][H][W] planar images.  Per image (alpha, beta, rw, rh) as the host
// checked them; contrast off is alpha 1, beta 0, for which aug_byte is the identity.  luts: the chunk's [n][3][256] LUTs, or
// null for no augment_hsv.  The parameters travel as kernel parameters (2 KB).
constexpr int kAugChunk = 128;
struct AugChunk {
    yfv2_aug_params im[kAugChunk];
    const uint8_t* img;    // image 0 of the chunk
    uint8_t* out;
    const uint8_t* luts;
    int H, W;
};

// A chunk with motion_blur: image n of the chunk with bit n of `blurred` set was filtered by the first pass into
// ws + n * 3 * H * W, whose byte minimum and maximum are mm[2 n + 1] = 255 - min and mm[2 n] = max; the second pass reads it
// there through cv2.normalize's byte map instead of reading img through contrast.  The other images take the AugChunk path.
struct AugBlurChunk : AugChunk {
    const uint8_t* ws;     // image 0 of the chunk
    const unsigned* mm;    // image 0 of the chunk
    unsigned blurred[kAugChunk / 32];
};

// augment_hsv's state plus the image's 256-byte map from source byte to the byte the later steps see: contrast for an image
// without blur, normalize for a blurred one (both are functions of the byte alone)
struct BlurSmem : HsvSmem {
    uint8_t map[256];
};

template <class Chunk> struct AugTraits {
    static constexpr bool kBlur = false;
    using Smem = HsvSmem;
};
template <> struct AugTraits<AugBlurChunk> {
    static constexpr bool kBlur = true;
    using Smem = BlurSmem;
};

// cv2.normalize(NORM_MINMAX, 0..255) of byte x in an image whose bytes span smin..smax
__device__ __forceinline__ unsigned normalize_byte(unsigned x, unsigned smin, unsigned smax) {
    const double d = (double)smax - (double)smin;
    const double scale = d > 2.220446049250313e-16 ? 255.0 * (1.0 / d) : 0.0;
    const double shift = 0.0 - (double)smin * scale;
    const float y = __fmaf_rn((float)x, (float)scale, (float)shift);
    return (unsigned)fminf(fmaxf(rintf(y), 0.f), 255.f);
}

// Fills t.map for image n of the chunk (256 threads or more; the caller synchronises) and returns where its bytes are read
__device__ __forceinline__ const uint8_t* stage_map(BlurSmem& t, const AugBlurChunk& a, int n, size_t image_bytes) {
    const int i = threadIdx.x + threadIdx.y * blockDim.x;
    const bool bl = (a.blurred[n >> 5] >> (n & 31)) & 1u;
    if (i < 256) t.map[i] = (uint8_t)(bl ? normalize_byte(i, 255u - a.mm[2 * n + 1], a.mm[2 * n]) : aug_byte(i, a.im[n].alpha, a.im[n].beta));
    return (bl ? a.ws : a.img) + (size_t)n * image_bytes;
}

// k_resize.cu: contrast -> random_resize -> (augment_hsv) on the chunk's cnt images; img and out do not overlap.  With an
// AugBlurChunk the blurred images are read from the workspace through their normalize map.
template <class Chunk>
int launch_aug_resize(const Chunk& a, int cnt, cudaStream_t stream);

}  // namespace yfv2
