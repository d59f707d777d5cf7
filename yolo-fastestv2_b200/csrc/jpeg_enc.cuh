// Baseline JPEG encode: the per-pixel, per-block and per-unit functions of the encoder (k_jpeg_enc.cu), each __host__ __device__
// so tests/jpeg_enc_harness.cu composes the same functions on the CPU.  The arithmetic is libjpeg-turbo 3.1's, what cv2.imencode
// runs: jccolor's 16-bit fixed-point RGB -> YCbCr, jcprepro / jcsample's edge replication and h2v1 / h2v2 downsampling with
// alternating bias, jpeg_fdct_islow, jcdctmgr's reciprocal quantiser, jccoefct's dummy blocks and jchuff's baseline coding with
// the ITU-T T.81 Annex K tables.
#pragma once
#include <stdint.h>

#include "jpeg.cuh"

namespace yfv2 {
namespace jpege {

using jpeg::natural;

constexpr uint32_t kMagic = 0x31434e45;   // "ENC1": a blob yfv2_jpeg_encode_plan wrote
// Most bits one block can take: DC code + value (16 + 11), then 63 AC symbols of 16-bit code + 10 value bits.  ZRL and EOB only
// appear where coefficients are zero, each of which saves more than they cost.
constexpr int kMaxBlockBits = 27 + 63 * 26;

struct HuffEnc {          // jchuff's derived table: code and length of each symbol (length 0: no code)
    uint16_t code[256];
    uint8_t size[256];
};

struct Quant {            // jcdctmgr's divisors of one table (natural order), for the islow FDCT's output scaled by 8
    uint16_t recip[64];
    uint16_t corr[64];
    uint8_t shift[64];    // r: the product is shifted right by r
};

// Geometry of one output: the region size and the scan's block layout
struct Geom {
    int w, h;             // image size
    int ncomp;            // 1 (grey) or 3 (YCbCr)
    int hs, vs;           // luma sampling factors (chroma is 1x1)
    int mcux, mcuy;       // MCUs per row and column
    int upm;              // units (blocks) per MCU: hs * vs + 2, or 1 for grey
    int restart;          // MCUs per restart interval, 0: none
    int wb0, hb0;         // luma blocks that hold image data (past them: jccoefct's dummy blocks)
};

// ---- colour and sampling -------------------------------------------------------------------------------------------------------
// jccolor.c rgb_ycc_convert (SCALEBITS 16): Y rounds to nearest, Cb and Cr with the 0.5 - epsilon fudge and CBCR_OFFSET
JPEG_HD void rgb_ycc(int b, int g, int r, int (&ycc)[3]) {
    constexpr int HALF = 1 << 15, CBCR = 128 << 16;
    ycc[0] = (19595 * r + 38470 * g + 7471 * b + HALF) >> 16;
    ycc[1] = (-11059 * r - 21709 * g + 32768 * b + CBCR + HALF - 1) >> 16;
    ycc[2] = (32768 * r - 27439 * g - 5329 * b + CBCR + HALF - 1) >> 16;
}

// Sample (i, j) of component c, its plane padded to whole blocks.  px(x, y, bgr) gives the B, G, R (or for grey the byte in bgr[0])
// of image pixel (x, y), 0 <= x < w, 0 <= y < h.  Image rows and columns past the edge repeat the last one (expand_right_edge,
// expand_bottom_edge of jcprepro); a downsampled component's rows past ceil(h / vs) repeat its last row (jcprepro pads the
// downsampled rows of the last iMCU row); h2v1 adds bias 0, 1, 0, 1, ... and h2v2 1, 2, 1, 2, ... along the row (jcsample).
template <class Px>
JPEG_HD int comp_sample(const Px& px, const Geom& g, int c, int i, int j) {
    int p[3], ycc[3];
    if (g.ncomp == 1) {
        px(i < g.w ? i : g.w - 1, j < g.h ? j : g.h - 1, p);
        return p[0];
    }
    const int fh = c == 0 ? 1 : g.hs, fv = c == 0 ? 1 : g.vs;
    if (fv == 2) {
        const int last = (g.h + 1) / 2 - 1;
        if (j > last) j = last;
    }
    int sum = 0;
    for (int dy = 0; dy < fv; ++dy)
        for (int dx = 0; dx < fh; ++dx) {
            const int x = i * fh + dx, y = j * fv + dy;
            px(x < g.w ? x : g.w - 1, y < g.h ? y : g.h - 1, p);
            rgb_ycc(p[0], p[1], p[2], ycc);
            sum += c == 0 ? ycc[0] : c == 1 ? ycc[1] : ycc[2];   // no dynamic index: the array stays in registers
        }
    if (fh * fv == 1) return sum;
    if (fv == 1) return (sum + (i & 1)) >> 1;   // h2v1
    return (sum + 1 + (i & 1)) >> 2;            // h2v2
}

// ---- forward DCT and quantisation ------------------------------------------------------------------------------------------------
// One 1-D pass of jpeg_fdct_islow (CONST_BITS 13, PASS1_BITS 2) over d[0], d[st], ..., d[7 st]: pass 0 over a row of centred
// samples, pass 1 over a column of pass 0's output.  The result is the DCT scaled by 8.
template <int PASS>
JPEG_HD void fdct_1d(int* d, int st) {
    constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    constexpr int S = PASS == 0 ? 13 - 2 : 13 + 2;
    constexpr int R = 1 << (S - 1);
    const int tmp0 = d[0] + d[7 * st], tmp7 = d[0] - d[7 * st];
    const int tmp1 = d[st] + d[6 * st], tmp6 = d[st] - d[6 * st];
    const int tmp2 = d[2 * st] + d[5 * st], tmp5 = d[2 * st] - d[5 * st];
    const int tmp3 = d[3 * st] + d[4 * st], tmp4 = d[3 * st] - d[4 * st];
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    if (PASS == 0) {
        d[0] = (tmp10 + tmp11) * 4;
        d[4 * st] = (tmp10 - tmp11) * 4;
    } else {
        d[0] = (tmp10 + tmp11 + 2) >> 2;
        d[4 * st] = (tmp10 - tmp11 + 2) >> 2;
    }
    const int z1 = (tmp12 + tmp13) * F0541;
    d[2 * st] = (z1 + tmp13 * F0765 + R) >> S;
    d[6 * st] = (z1 - tmp12 * F1847 + R) >> S;
    const int z5 = (tmp4 + tmp6 + tmp5 + tmp7) * F1175;
    const int o1 = (tmp4 + tmp7) * -F0899, o2 = (tmp5 + tmp6) * -F2562;
    const int o3 = (tmp4 + tmp6) * -F1961 + z5, o4 = (tmp5 + tmp7) * -F0390 + z5;
    d[7 * st] = (tmp4 * F0298 + o1 + o3 + R) >> S;
    d[5 * st] = (tmp5 * F2053 + o2 + o4 + R) >> S;
    d[3 * st] = (tmp6 * F3072 + o2 + o3 + R) >> S;
    d[st] = (tmp7 * F1501 + o1 + o4 + R) >> S;
}

// jcdctmgr.c quantize: |v| + correction times the reciprocal, shifted, the sign put back
JPEG_HD int quantize(int v, const Quant& q, int k) {
    const uint32_t a = (uint32_t)(v < 0 ? -v : v);
    const int m = (int)(((a + q.corr[k]) * (uint64_t)q.recip[k]) >> q.shift[k]);
    return v < 0 ? -m : m;
}

// ---- scan order ----------------------------------------------------------------------------------------------------------------
// Unit u (a block in scan order) of an output: its MCU, component and block coordinates.  src_x, src_y is the block whose samples
// it codes: itself, or for a dummy block of the interleaved scan the block whose DC it repeats (jccoefct compress_data: a dummy at
// the right edge repeats the DC of the block to its left, one in the bottom dummy row that of the last block of the row above in
// its MCU; both are AC zero).
struct Unit {
    int mcu, c, bx, by;
    int src_x, src_y;
    bool dummy;
};

JPEG_HD Unit unit_of(const Geom& g, long long u) {
    Unit r;
    r.mcu = (int)(u / g.upm);
    const int k = (int)(u - (long long)r.mcu * g.upm);
    const int mx = r.mcu % g.mcux, my = r.mcu / g.mcux;
    if (g.ncomp == 1) {
        r.c = 0; r.bx = mx; r.by = my;
    } else if (k < g.hs * g.vs) {
        r.c = 0; r.bx = mx * g.hs + k % g.hs; r.by = my * g.vs + k / g.hs;
    } else {
        r.c = 1 + k - g.hs * g.vs; r.bx = mx; r.by = my;
    }
    r.src_x = r.bx; r.src_y = r.by;
    r.dummy = false;
    if (g.ncomp == 3 && r.c == 0) {
        if (r.by >= g.hb0) {
            r.dummy = true;
            r.src_y = g.hb0 - 1;
            r.src_x = mx * g.hs + g.hs - 1 < g.wb0 - 1 ? mx * g.hs + g.hs - 1 : g.wb0 - 1;
        } else if (r.bx >= g.wb0) {
            r.dummy = true;
            r.src_x = g.wb0 - 1;
        }
    }
    return r;
}

JPEG_HD bool segment_start(const Geom& g, int mcu) { return g.restart ? mcu % g.restart == 0 : mcu == 0; }

// The unit whose DC predicts unit u's (the previous block of its component in the same restart interval), -1: predictor 0
JPEG_HD long long dc_pred_unit(const Geom& g, long long u) {
    const int mcu = (int)(u / g.upm), k = (int)(u - (long long)mcu * g.upm);
    if (g.ncomp == 3 && k > 0 && k < g.hs * g.vs) return u - 1;
    if (segment_start(g, mcu)) return -1;
    if (g.ncomp == 3 && k == 0) return u - g.upm + g.hs * g.vs - 1;
    return u - g.upm;
}

// ---- Huffman coding ------------------------------------------------------------------------------------------------------------
JPEG_HD int nbits(int a) {   // bits of |v| (jchuff's JPEG_NBITS)
    int n = 0;
    while (a) { ++n; a >>= 1; }
    return n;
}

// jchuff.c encode_one_block: the DC difference, then the AC coefficients in zigzag order as run/size symbols, ZRL for runs of 16
// zeros before a nonzero coefficient, EOB after the last one.  coef is natural order.  Sink::put(code, size) takes the bits.
template <class Sink>
JPEG_HD void encode_block(const int16_t* coef, int diff, const HuffEnc& dc, const HuffEnc& ac, Sink& s) {
    int a = diff < 0 ? -diff : diff;
    int n = nbits(a);
    s.put(dc.code[n], dc.size[n]);
    if (n) s.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = coef[natural(k)];
        if (v == 0) { ++run; continue; }
        while (run > 15) {
            s.put(ac.code[0xF0], ac.size[0xF0]);
            run -= 16;
        }
        a = v < 0 ? -v : v;
        n = nbits(a);
        const int sym = (run << 4) + n;
        s.put(ac.code[sym], ac.size[sym]);
        s.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1), n);
        run = 0;
    }
    if (run > 0) s.put(ac.code[0], ac.size[0]);
}

struct CountSink {
    int n = 0;
    JPEG_HD void put(uint32_t, int size) { n += size; }
};

}  // namespace jpege
}  // namespace yfv2
