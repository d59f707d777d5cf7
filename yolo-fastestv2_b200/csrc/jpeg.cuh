// Baseline JPEG decode: the decode tables the host parser (k_jpeg.cu) packs into the metadata blob, and the per-segment, per-block
// and per-pixel functions of the three device phases.  Everything below is __host__ __device__, so tests/jpeg_harness.cu runs the
// same functions on the CPU.  The arithmetic is libjpeg-turbo's (what cv2.imread decodes with): jdhuff's bit reader and Huffman
// decode, jpeg_idct_islow as its x86 SIMD code computes it, jdsample's fancy upsampling and jdcolor's YCbCr -> RGB tables.
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
constexpr int kErrShort = 1;              // a segment ran out of data (zero bits were decoded), or the file ends inside the scan
constexpr int kErrCode = 2;               // a bit pattern that is no Huffman code of its table
constexpr int kErrRestart = 4;            // RSTn markers out of sequence: libjpeg resyncs and its intervals get other data

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
    int img, mcu0, nmcu;
    int err;                // kErr* flags the parse found: kErrShort when the file ends inside the scan, kErrRestart
    long long begin, end;   // bytes of the file arena, RSTn / end-of-scan markers excluded
};

// ---- progressive images (yfv2_jpeg_parse_ex with YFV2_JPEG_PROGRESSIVE) ----------------------------------------------------
// A progressive image's Image record has nseg = 0; its scans, their tables and their segments are in the arrays below.  Each scan
// has a level: 1 + the highest level of the image's earlier scans whose (component, coefficient) sets it overlaps, so the scans of
// one level write disjoint coefficients and read only what lower levels wrote.  The decode runs one launch per level.
constexpr int kMaxScans = 128;            // scans per progressive file (libjpeg's default script, cv2's and Pillow's: 10, 6 for grey)

struct Scan {
    int ncomp, comp[3];   // the scan's components (indices into Image::comp, frame order); an AC scan has one
    int ss, se, ah, al;   // spectral selection and successive approximation
    int tab[3];           // Huff pool index of scan component k's DC table (DC first scans) or tab[0] the AC table; -1: none
    int upr, units;       // units per row and units: MCUs when interleaved, else the component's ceil(dw / 8) x ceil(dh / 8) blocks
    int level;
};

struct PSeg {
    int img, scan, level;   // image, Scan index, the scan's level
    int unit0, nunit;       // its MCUs (interleaved) or blocks (one component) in scan order
    int err;                // kErr* flags the parse found (kErrShort also when the file ends before its EOI)
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
    // progressive images; all zero when the batch has none
    int nscan, nhuff, npseg, nlevel;                  // scans, pooled Huffman tables, segments, levels
    long long scan_off, huff_off, pseg_off, lvl_off;  // Scan[nscan], Huff[nhuff], PSeg[npseg] (sorted by level), int[nlevel + 1]
    long long prog_coef;         // workspace bytes [0, prog_coef) hold the progressive images' coefficients, zeroed before decode
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
    int err = s.err;
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

// ---- progressive entropy decode (libjpeg-turbo's jdphuff.c) -------------------------------------------------------------------
// Each function decodes one block of one scan into coefficients earlier scans may have set; none zeroes a block (the decode zeroes
// every progressive image's coefficients once, before its first scan).  A run that carries an AC symbol past the scan's band
// (never in an encoder's output) writes outside the band, as libjpeg does, and sets kErrCode: scans of one level are decoded in
// parallel on the premise that their bands are disjoint, so such a frame is not promised to be cv2's.
JPEG_HD void prog_dc_first(Bits& b, const Huff& t, int al, int& pred, int16_t* blk, int& err) {
    if (b.n < 32) b.fill();
    const int s = huff_decode(b, t, err);
    if (s) pred += receive_extend(b, s);
    blk[0] = (int16_t)((uint32_t)pred << al);
}

JPEG_HD void prog_dc_refine(Bits& b, int al, int16_t* blk) {
    if (b.n < 32) b.fill();
    if (b.peek(1)) blk[0] = (int16_t)(blk[0] | (1 << al));
    b.n -= 1;
}

JPEG_HD void prog_ac_first(Bits& b, const Huff& t, int ss, int se, int al, int& eobrun, int16_t* blk, int& err) {
    if (eobrun > 0) {
        --eobrun;
        return;
    }
    for (int k = ss; k <= se; ++k) {
        if (b.n < 32) b.fill();
        const int rs = huff_decode(b, t, err);
        const int r = rs >> 4, s = rs & 15;
        if (s) {
            k += r;
            if (k > se) err |= kErrCode;
            blk[natural(k)] = (int16_t)((uint32_t)receive_extend(b, s) << al);
        } else if (r == 15) {
            k += 15;
        } else {
            eobrun = 1 << r;                     // EOBr: this block and 2^r - 1 + r more bits' worth of blocks end here
            if (r) {
                eobrun += b.peek(r);
                b.n -= r;
            }
            --eobrun;
            break;
        }
    }
}

// One correction bit onto a coefficient already nonzero: its magnitude gains 1 << al unless that bit is already set
JPEG_HD void prog_correct(Bits& b, int16_t& c, int p1) {
    if (b.n < 32) b.fill();
    if (b.peek(1) && (c & p1) == 0) c = (int16_t)(c >= 0 ? c + p1 : c - p1);
    b.n -= 1;
}

// A symbol's size other than 1 is taken as 1 (libjpeg-turbo warns and goes on), so it is not flagged
JPEG_HD void prog_ac_refine(Bits& b, const Huff& t, int ss, int se, int al, int& eobrun, int16_t* blk, int& err) {
    const int p1 = 1 << al;
    int k = ss;
    if (eobrun == 0) {
        for (; k <= se; ++k) {
            if (b.n < 32) b.fill();
            const int rs = huff_decode(b, t, err);
            int r = rs >> 4, s = rs & 15;
            if (s) {
                s = b.peek(1) ? p1 : -p1;
                b.n -= 1;
            } else if (r != 15) {
                eobrun = 1 << r;
                if (r) {
                    eobrun += b.peek(r);
                    b.n -= r;
                }
                break;
            }
            do {                                 // skip r zero-history coefficients, correcting the nonzero ones passed
                int16_t& c = blk[natural(k)];
                if (c != 0) prog_correct(b, c, p1);
                else if (--r < 0) break;
                ++k;
            } while (k <= se);
            if (s) {
                if (k > se) err |= kErrCode;
                blk[natural(k)] = (int16_t)s;
            }
        }
    }
    if (eobrun > 0) {                            // in an EOB run: correction bits for the rest of the band
        for (; k <= se; ++k) {
            int16_t& c = blk[natural(k)];
            if (c != 0) prog_correct(b, c, p1);
        }
        --eobrun;
    }
}

// Every unit of progressive segment s of scan sc into the workspace's coefficients; tabs[k] is the table of scan component k (DC
// first scans) or tabs[0] the AC table (the pool's, or a copy).  Restarts reset the DC predictors and the EOB run; returns kErr*.
JPEG_HD int decode_prog_segment(const Image& im, const Scan& sc, const PSeg& s, const uint8_t* files, uint8_t* ws, const Huff* tabs) {
    Bits b{files + s.begin, files + s.end, 0, 0, 0};
    int pred[3] = {0, 0, 0}, eobrun = 0;
    int err = s.err;
    for (int u = s.unit0; u < s.unit0 + s.nunit; ++u) {
        if (sc.ncomp > 1) {                      // interleaved (DC only): MCUs as in a baseline scan
            const int mx = u % im.mcux, my = u / im.mcux;
            for (int k = 0; k < sc.ncomp; ++k) {
                const Comp& cp = im.comp[sc.comp[k]];
                int16_t* coef = reinterpret_cast<int16_t*>(ws + cp.coef);
                for (int bv = 0; bv < cp.v; ++bv)
                    for (int bh = 0; bh < cp.h; ++bh) {
                        int16_t* blk = coef + ((long long)(my * cp.v + bv) * cp.bw + mx * cp.h + bh) * 64;
                        if (sc.ah == 0) prog_dc_first(b, tabs[k], sc.al, pred[k], blk, err);
                        else prog_dc_refine(b, sc.al, blk);
                    }
            }
            continue;
        }
        const Comp& cp = im.comp[sc.comp[0]];    // one component: its blocks in raster order, whatever the sampling
        int16_t* blk = reinterpret_cast<int16_t*>(ws + cp.coef) + ((long long)(u / sc.upr) * cp.bw + u % sc.upr) * 64;
        if (sc.ss == 0) {
            if (sc.ah == 0) prog_dc_first(b, tabs[0], sc.al, pred[0], blk, err);
            else prog_dc_refine(b, sc.al, blk);
        } else if (sc.ah == 0) {
            prog_ac_first(b, tabs[0], sc.ss, sc.se, sc.al, eobrun, blk, err);
        } else {
            prog_ac_refine(b, tabs[0], sc.ss, sc.se, sc.al, eobrun, blk, err);
        }
    }
    if (b.n < b.zeros) err |= kErrShort;
    return err;
}

// Tables of scan sc in use: 0 (DC refinement), ncomp (DC first) or 1 (AC)
JPEG_HD int prog_ntabs(const Scan& sc) { return sc.ss == 0 ? (sc.ah == 0 ? sc.ncomp : 0) : 1; }

// ---- dequantise + IDCT --------------------------------------------------------------------------------------------------------
// jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) as libjpeg-turbo's x86 SIMD code computes it (jsimd_idct_islow, jidctint-sse2.asm
// and jidctint-avx2.asm), which is what cv2.imread runs on x86-64.  It equals jidctint.c while every value fits in int16, which
// encoder output always does.  Corrupt or hand-made coefficients do not, and then the SIMD arithmetic decides the pixels:
//  - dequantisation keeps the low 16 bits of coef * q (pmullw);
//  - in0 + in4, in0 - in4, in7 + in3 and in5 + in1 are 16-bit sums that wrap (paddw / psubw);
//  - the products and their sums are 32-bit and wrap (pmaddwd / paddd), so they are computed here in uint32_t;
//  - each pass's descaled outputs saturate to int16 (packssdw); pass 2's then saturate to -128..127 (packsswb) before + 128,
//    which clamps where jidctint.c's range-limit table (indexed & 1023) would wrap;
//  - when rows 1-7 of the block's coefficients are all zero, pass 1 writes the dequantised row 0 shifted left by 2 in 16 bits
//    (psllw), which wraps where the full pass would saturate.
JPEG_HD int wrap16(uint32_t x) { return (int16_t)(uint16_t)x; }
JPEG_HD int clampi(int x, int lo, int hi) { return x < lo ? lo : x > hi ? hi : x; }

// One 1-D transform of 8 int16 inputs in[0], in[st], ..., in[7 * st]; out[k] = the descaled output k (>> S) in 32 bits
template <int S>
JPEG_HD void islow_1d(const int* in, int st, int* out) {
    using u = uint32_t;
    constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    const u i0 = (u)in[0], i1 = (u)in[st], i2 = (u)in[2 * st], i3 = (u)in[3 * st], i4 = (u)in[4 * st], i5 = (u)in[5 * st],
            i6 = (u)in[6 * st], i7 = (u)in[7 * st];
    const u tmp3 = i2 * (u)(F0541 + F0765) + i6 * (u)F0541, tmp2 = i2 * (u)F0541 + i6 * (u)(F0541 - F1847);
    const u tmp0 = (u)wrap16(i0 + i4) << 13, tmp1 = (u)wrap16(i0 - i4) << 13;
    const u t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    const u z3 = (u)wrap16(i7 + i3), z4 = (u)wrap16(i5 + i1);
    const u za = z3 * (u)(F1175 - F1961) + z4 * (u)F1175, zb = z3 * (u)F1175 + z4 * (u)(F1175 - F0390);
    const u o0 = i7 * (u)(F0298 - F0899) + i1 * (u)-F0899 + za, o3 = i7 * (u)-F0899 + i1 * (u)(F1501 - F0899) + zb;
    const u o1 = i5 * (u)(F2053 - F2562) + i3 * (u)-F2562 + zb, o2 = i5 * (u)-F2562 + i3 * (u)(F3072 - F2562) + za;
    constexpr u R = 1u << (S - 1);
    out[0] = (int)(t10 + o3 + R) >> S; out[7] = (int)(t10 - o3 + R) >> S;
    out[1] = (int)(t11 + o2 + R) >> S; out[6] = (int)(t11 - o2 + R) >> S;
    out[2] = (int)(t12 + o1 + R) >> S; out[5] = (int)(t12 - o1 + R) >> S;
    out[3] = (int)(t13 + o0 + R) >> S; out[4] = (int)(t13 - o0 + R) >> S;
}

JPEG_HD void idct_islow(const int16_t* coef, const uint16_t* q, uint8_t* out, int pitch) {
    int in[64], ws[64], o[8];
    bool ac = false;                                       // any coefficient in rows 1-7 (the SIMD's zero-column test)
    for (int k = 0; k < 64; ++k) {
        in[k] = wrap16((uint32_t)(coef[k] * (int)q[k]));
        ac = ac || (k >= 8 && coef[k] != 0);
    }
    for (int c = 0; c < 8; ++c) {
        if (!ac) {
            for (int r = 0; r < 8; ++r) ws[r * 8 + c] = wrap16((uint32_t)in[c] << 2);
            continue;
        }
        islow_1d<11>(in + c, 8, o);
        for (int r = 0; r < 8; ++r) ws[r * 8 + c] = clampi(o[r], -32768, 32767);
    }
    for (int r = 0; r < 8; ++r) {
        islow_1d<18>(ws + r * 8, 1, o);
        for (int c = 0; c < 8; ++c) out[(long long)r * pitch + c] = (uint8_t)(clampi(o[c], -128, 127) + 128);
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
