// Baseline JPEG decode: the decode tables the host parser (k_jpeg.cu) packs into the metadata blob, and the per-segment, per-block
// and per-pixel functions of the three device phases.  Everything below is __host__ __device__, so tests/jpeg_harness.cu runs the
// same functions on the CPU.  The arithmetic is libjpeg-turbo's (what cv2.imread decodes with): jdhuff's bit reader and Huffman
// decode, jidctint's jpeg_idct_islow with its range-limit table, jdsample's fancy upsampling and jdcolor's YCbCr -> RGB tables.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define JPEG_HD __host__ __device__ __forceinline__
#else
#define JPEG_HD inline
#endif

namespace yfv2 {
namespace jpeg {

constexpr uint32_t kMagic = 0x3147504a;   // "JPG1": a blob yfv2_jpeg_parse wrote
constexpr int kMaxSide = 32768;           // the resize's limit
constexpr int kFastBits = 9;              // first-level Huffman lookup
constexpr int kErrShort = 1;              // an entropy-coded segment ran out of data (zero bits were decoded)
constexpr int kErrCode = 2;               // a bit pattern that is no Huffman code of its table

struct alignas(16) Huff {           // 16-byte aligned: the entropy kernel copies tables with 16-byte accesses
    uint16_t fast[1 << kFastBits];   // (length << 8) | symbol of the code the next kFastBits bits start with; 0: a longer code
    int32_t maxcode[18];             // largest code of each length, -1 when there is none
    int32_t valoff[18];              // vals index of a code of that length, minus the code
    uint8_t vals[256];
};

struct Comp {
    int h, v;            // sampling factors (1, 1 for a one-component image, which is one non-interleaved scan)
    int bw, bh;          // block grid, MCU-padded
    int dw, dh;          // downsampled size: ceil(w * h / hmax) x ceil(h * v / vmax), what jdsample's edges are at
    int pitch;           // bytes between plane rows: 8 * bw
    int pad_;
    long long coef;      // workspace byte offset of the [bh][bw][64] int16 coefficient blocks, natural order
    long long plane;     // workspace byte offset of the [8 * bh][pitch] uint8 sample plane
    uint16_t q[64];      // dequantisation, natural order
};

struct Image {
    int w, h;            // coded size
    int ow, oh;          // oriented size: the frame's
    int orient;          // EXIF orientation 1..8
    int ncomp;           // 1 (grey) or 3 (YCbCr)
    int hmax, vmax;
    int mcux, mcuy;      // MCUs per row and column
    int restart;         // MCUs per restart interval, 0: none
    int nseg, seg0;      // its entropy-coded segments in the blob's segment array
    int pad_;
    long long blocks;    // blocks of all components
    long long frame;     // byte offset of the [oh][ow][3] BGR frame in the arena
    Comp comp[3];
    Huff dc[3], ac[3];   // each component's tables
};

struct Seg {
    int img, mcu0, nmcu, pad_;
    long long begin, end;   // bytes of the file arena, RSTn / end-of-scan markers excluded
};

struct Header {
    uint32_t magic;
    int n, nseg, max_blocks;     // images, segments, most blocks of one image
    long long max_pixels;        // most pixels of one frame
    long long img_off, seg_off;  // byte offsets of Image[n] and Seg[nseg] in the blob
    long long bytes;             // blob size
    long long workspace;         // workspace bytes the decode needs
    long long frames;            // arena bytes
    long long files;             // bytes of the file arena the segments point into
};

// jpeg_natural_order with libjpeg's 16 extra entries, so a corrupt run past coefficient 63 lands on 63
#define YFV2_JPEG_NATURAL_ORDER                                                                                              \
    {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, \
     21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, \
     47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63}
#ifdef __CUDACC__
static __constant__ uint8_t kNaturalDev[80] = YFV2_JPEG_NATURAL_ORDER;
#endif
static const uint8_t kNaturalHost[80] = YFV2_JPEG_NATURAL_ORDER;

JPEG_HD int natural(int k) {
#ifdef __CUDA_ARCH__
    return kNaturalDev[k];
#else
    return kNaturalHost[k];
#endif
}

// ---- entropy decode ---------------------------------------------------------------------------------------------------------
// MSB-first bit buffer over one segment.  FF 00 stuffing is removed; past the segment's end zero bits are shifted in (as
// libjpeg-turbo does at a marker or the end of data) and counted, and no byte at or past `end` is ever read.
struct Bits {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc;    // the low n bits are the next bits of the stream
    int n;
    int zeros;       // zero bits shifted in past the end

    JPEG_HD void fill() {
        while (n <= 56) {
            uint32_t b = 0;
            if (p < end) {
                b = *p++;
                if (b == 0xFF && p < end && *p == 0x00) ++p;
            } else {
                zeros += 8;
            }
            acc = (acc << 8) | b;
            n += 8;
        }
    }
    JPEG_HD int peek(int k) const { return (int)(acc >> (n - k)) & ((1 << k) - 1); }
};

// One Huffman symbol (jdhuff.c HUFF_DECODE): the caller has made n >= 16.  A pattern no code matches flags kErrCode and gives 0.
JPEG_HD int huff_decode(Bits& b, const Huff& t, int& err) {
    const int e = t.fast[b.peek(kFastBits)];
    if (e) {
        b.n -= e >> 8;
        return e & 255;
    }
    for (int l = kFastBits + 1; l <= 16; ++l) {
        const int code = b.peek(l);
        if (code <= t.maxcode[l]) {
            b.n -= l;
            return t.vals[(code + t.valoff[l]) & 255];
        }
    }
    err |= kErrCode;
    b.n -= 16;
    return 0;
}

// s more bits as a signed coefficient (HUFF_EXTEND); the caller has made n >= s
JPEG_HD int receive_extend(Bits& b, int s) {
    const int x = b.peek(s);
    b.n -= s;
    return x < (1 << (s - 1)) ? x - (1 << s) + 1 : x;
}

// One block: the DC difference onto the component's predictor, then the AC run/size symbols, de-zigzagged into blk
JPEG_HD void decode_block(Bits& b, const Huff& dc, const Huff& ac, int& pred, int16_t* blk, int& err) {
    uint64_t* z = reinterpret_cast<uint64_t*>(blk);
    for (int i = 0; i < 16; ++i) z[i] = 0;
    if (b.n < 32) b.fill();
    const int s = huff_decode(b, dc, err);
    if (s) pred += receive_extend(b, s);
    blk[0] = (int16_t)pred;
    for (int k = 1; k < 64; ++k) {
        if (b.n < 32) b.fill();
        const int rs = huff_decode(b, ac, err);
        const int r = rs >> 4, sz = rs & 15;
        if (sz) {
            k += r;
            blk[natural(k)] = (int16_t)receive_extend(b, sz);
        } else {
            if (r != 15) break;
            k += 15;
        }
    }
}

// Phase 1: every MCU of segment s into the coefficient blocks of the workspace, with component c's tables dc[c], ac[c] (the
// image's own, or a copy of them); returns kErr* flags
JPEG_HD int decode_segment(const Image& im, const Seg& s, const uint8_t* files, uint8_t* ws, const Huff* dc, const Huff* ac) {
    Bits b{files + s.begin, files + s.end, 0, 0, 0};
    int pred[3] = {0, 0, 0};
    int err = 0;
    for (int m = s.mcu0; m < s.mcu0 + s.nmcu; ++m) {
        const int mx = m % im.mcux, my = m / im.mcux;
        for (int c = 0; c < im.ncomp; ++c) {
            const Comp& cp = im.comp[c];
            int16_t* coef = reinterpret_cast<int16_t*>(ws + cp.coef);
            for (int bv = 0; bv < cp.v; ++bv)
                for (int bh = 0; bh < cp.h; ++bh) {
                    const long long blk = (long long)(my * cp.v + bv) * cp.bw + mx * cp.h + bh;
                    decode_block(b, dc[c], ac[c], pred[c], coef + blk * 64, err);
                }
        }
    }
    if (b.n < b.zeros) err |= kErrShort;   // some of the shifted-in zeros were decoded
    return err;
}

// ---- dequantise + IDCT --------------------------------------------------------------------------------------------------------
// jidctint.c's post-IDCT range limit: the index is masked with 1023, so values far outside 0..255 wrap instead of clamping
JPEG_HD int idct_range_limit(long long x) {
    const int t = (int)(x & 1023);
    return t < 128 ? t + 128 : t < 512 ? 255 : t < 896 ? 0 : t - 896;
}

// jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) in 64-bit arithmetic like its JLONG.  The zero-AC shortcuts of both passes give
// the same values as the full computation, so they are not restated.
JPEG_HD void idct_islow(const int16_t* coef, const uint16_t* q, uint8_t* out, int pitch) {
    constexpr int CB = 13, P1 = 2;
    constexpr long long F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                        F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    int ws[64];
    for (int c = 0; c < 8; ++c) {
        long long in[8];
        for (int r = 0; r < 8; ++r) in[r] = (long long)(coef[r * 8 + c] * (int)q[r * 8 + c]);
        long long z2 = in[2], z3 = in[6];
        long long z1 = (z2 + z3) * F0541;
        long long tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
        long long tmp0 = (in[0] + in[4]) * (1LL << CB), tmp1 = (in[0] - in[4]) * (1LL << CB);
        const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = in[7]; tmp1 = in[5]; tmp2 = in[3]; tmp3 = in[1];
        z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
        long long z4 = tmp1 + tmp3;
        const long long z5 = (z3 + z4) * F1175;
        tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
        constexpr int S = CB - P1;
        constexpr long long R = 1LL << (S - 1);
        ws[0 * 8 + c] = (int)((tmp10 + tmp3 + R) >> S);
        ws[7 * 8 + c] = (int)((tmp10 - tmp3 + R) >> S);
        ws[1 * 8 + c] = (int)((tmp11 + tmp2 + R) >> S);
        ws[6 * 8 + c] = (int)((tmp11 - tmp2 + R) >> S);
        ws[2 * 8 + c] = (int)((tmp12 + tmp1 + R) >> S);
        ws[5 * 8 + c] = (int)((tmp12 - tmp1 + R) >> S);
        ws[3 * 8 + c] = (int)((tmp13 + tmp0 + R) >> S);
        ws[4 * 8 + c] = (int)((tmp13 - tmp0 + R) >> S);
    }
    for (int r = 0; r < 8; ++r) {
        const int* w = ws + r * 8;
        long long z2 = w[2], z3 = w[6];
        long long z1 = (z2 + z3) * F0541;
        long long tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
        long long tmp0 = ((long long)w[0] + w[4]) * (1LL << CB), tmp1 = ((long long)w[0] - w[4]) * (1LL << CB);
        const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = w[7]; tmp1 = w[5]; tmp2 = w[3]; tmp3 = w[1];
        z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
        long long z4 = tmp1 + tmp3;
        const long long z5 = (z3 + z4) * F1175;
        tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
        constexpr int S = CB + P1 + 3;
        constexpr long long R = 1LL << (S - 1);
        uint8_t* o = out + (long long)r * pitch;
        o[0] = (uint8_t)idct_range_limit((tmp10 + tmp3 + R) >> S);
        o[7] = (uint8_t)idct_range_limit((tmp10 - tmp3 + R) >> S);
        o[1] = (uint8_t)idct_range_limit((tmp11 + tmp2 + R) >> S);
        o[6] = (uint8_t)idct_range_limit((tmp11 - tmp2 + R) >> S);
        o[2] = (uint8_t)idct_range_limit((tmp12 + tmp1 + R) >> S);
        o[5] = (uint8_t)idct_range_limit((tmp12 - tmp1 + R) >> S);
        o[3] = (uint8_t)idct_range_limit((tmp13 + tmp0 + R) >> S);
        o[4] = (uint8_t)idct_range_limit((tmp13 - tmp0 + R) >> S);
    }
}

// Phase 2: block k (0 <= k < im.blocks, component-major) of an image from the workspace's coefficients into its plane
JPEG_HD void idct_block(const Image& im, long long k, uint8_t* ws) {
    int c = 0;
    while (c + 1 < im.ncomp && k >= (long long)im.comp[c].bw * im.comp[c].bh) {
        k -= (long long)im.comp[c].bw * im.comp[c].bh;
        ++c;
    }
    const Comp& cp = im.comp[c];
    const int by = (int)(k / cp.bw), bx = (int)(k % cp.bw);
    idct_islow(reinterpret_cast<const int16_t*>(ws + cp.coef) + k * 64, cp.q,
               ws + cp.plane + (long long)by * 8 * cp.pitch + bx * 8, cp.pitch);
}

// ---- upsample + colour + orientation -------------------------------------------------------------------------------------------
JPEG_HD int sample(const uint8_t* ws, const Comp& c, int x, int y) { return ws[c.plane + (long long)y * c.pitch + x]; }

// The chroma value jdsample gives full-resolution pixel (x, y).  Fancy (triangle) upsampling for h2v1 and h2v2 planes wider than
// 2 samples and for h1v2; plain replication otherwise.  Neighbours past the plane's downsampled edge are the edge sample itself,
// which is what the edge cases of h2v1_fancy_upsample / h2v2_fancy_upsample compute and what jdmainct's context rows hold.
JPEG_HD int chroma(const Image& im, const Comp& c, const uint8_t* ws, int x, int y) {
    const int fh = im.hmax / c.h, fv = im.vmax / c.v;
    if (fh == 1 && fv == 1) return sample(ws, c, x, y);
    if (fh == 2 && fv == 1 && c.dw > 2) {
        const int i = x >> 1, j = (x & 1) ? (i + 1 < c.dw ? i + 1 : i) : (i > 0 ? i - 1 : 0);
        return (3 * sample(ws, c, i, y) + sample(ws, c, j, y) + ((x & 1) ? 2 : 1)) >> 2;
    }
    if (fh == 1 && fv == 2) {
        const int r = y >> 1, rn = (y & 1) ? (r + 1 < c.dh ? r + 1 : r) : (r > 0 ? r - 1 : 0);
        return (3 * sample(ws, c, x, r) + sample(ws, c, x, rn) + ((y & 1) ? 2 : 1)) >> 2;
    }
    if (fh == 2 && fv == 2 && c.dw > 2) {
        const int r = y >> 1, rn = (y & 1) ? (r + 1 < c.dh ? r + 1 : r) : (r > 0 ? r - 1 : 0);
        const int i = x >> 1, j = (x & 1) ? (i + 1 < c.dw ? i + 1 : i) : (i > 0 ? i - 1 : 0);
        const int ci = 3 * sample(ws, c, i, r) + sample(ws, c, i, rn);
        const int cj = 3 * sample(ws, c, j, r) + sample(ws, c, j, rn);
        return (3 * ci + cj + ((x & 1) ? 7 : 8)) >> 4;
    }
    return sample(ws, c, x / fh, y / fv);
}

JPEG_HD int clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

// Source pixel of oriented pixel (ox, oy): the inverse of the EXIF transform cv2 applies (ExifTransform)
JPEG_HD void orient_source(const Image& im, int ox, int oy, int& x, int& y) {
    switch (im.orient) {
        case 2: x = im.w - 1 - ox; y = oy; break;
        case 3: x = im.w - 1 - ox; y = im.h - 1 - oy; break;
        case 4: x = ox; y = im.h - 1 - oy; break;
        case 5: x = oy; y = ox; break;
        case 6: x = oy; y = im.h - 1 - ox; break;
        case 7: x = im.w - 1 - oy; y = im.h - 1 - ox; break;
        case 8: x = im.w - 1 - oy; y = ox; break;
        default: x = ox; y = oy; break;
    }
}

// Phase 3: B, G, R of oriented pixel (ox, oy), jdcolor's ycc_rgb_convert (16-bit fixed point) or grey replicated
JPEG_HD void bgr_pixel(const Image& im, const uint8_t* ws, int ox, int oy, uint8_t* o) {
    int x, y;
    orient_source(im, ox, oy, x, y);
    const int Y = sample(ws, im.comp[0], x, y);
    if (im.ncomp == 1) {
        o[0] = o[1] = o[2] = (uint8_t)Y;
        return;
    }
    const long long cb = chroma(im, im.comp[1], ws, x, y) - 128, cr = chroma(im, im.comp[2], ws, x, y) - 128;
    constexpr long long HALF = 1LL << 15;
    o[0] = (uint8_t)clamp255(Y + (int)((116130 * cb + HALF) >> 16));
    o[1] = (uint8_t)clamp255(Y + (int)((-22554 * cb + HALF + -46802 * cr) >> 16));
    o[2] = (uint8_t)clamp255(Y + (int)((91881 * cr + HALF) >> 16));
}

}  // namespace jpeg
}  // namespace yfv2
