// Baseline JPEG encode on the device: output i is, byte for byte, cv2.imencode('.jpg', img_i, params_i)[1] of OpenCV 4.13
// (libjpeg-turbo 3.1), img_i the BGR (or grey) image cv2.cvtColor gives the frame, cropped to the output's region.  The per-pixel,
// per-block and per-unit arithmetic is in jpeg_enc.cuh (shared with tests/jpeg_enc_harness.cu); the frames are read through the
// resize's Source fetches (resize.cuh), so no converted or cropped frame is ever stored.
//
// yfv2_jpeg_encode_plan (host only) checks every output, writes each one's headers (SOI, JFIF APP0, DQT, SOF0, DHT, DRI, SOS, as
// jcmarker writes them) into a blob with the geometry and quantiser tables, and sizes the workspace and the output arena from a
// worst-case bound.  yfv2_jpeg_encode then runs five stages over every block ("unit") of the batch, in scan order:
//   transform  64 threads per unit: fetch + colour + edge replication + downsampling of its 64 samples, islow FDCT, quantise,
//              int16 coefficients (dummy blocks: AC zero, the DC of the block they repeat);
//   scan       each unit's Huffman bit count (its DC difference against the previous block of its component, reset at every
//              restart), then an exclusive scan over all units of the batch (tile sums, one CTA over the sums, tile rescans);
//   pack       each unit writes its codes at its offset into 32-bit words of a staging area where every segment (the scan, or one
//              restart interval) starts on a word; words shared with the neighbours are merged with atomicOr; a segment's last unit
//              pads it with 1-bits to a byte (jchuff flush_bits);
//   stuff      each unit counts the output bytes it owns (staging bytes whose first bit is its, 0xFF counted twice, plus the header,
//              RSTn or EOI it writes), a scan of the counts places them, and each unit writes its bytes with 0xFF 0x00 stuffing.
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "jpeg_enc.cuh"
#include "resize.cuh"

namespace yfv2 {
namespace jpege {

constexpr int kScanThreads = 256, kScanItems = 8, kTile = kScanThreads * kScanItems;
constexpr int kUnitsPerCta = 4;                 // transform: 4 units of 64 threads

struct alignas(16) EncImage {
    int kind;                  // YFV2_JPEG_SRC_*
    int x0, y0;                // region origin in the frame
    int nseg, seg0;            // segments of this output, index of its first one in the batch
    Geom g;
    long long unit0, nunits;   // its units in the batch's scan-order unit array
    long long hdr, hdr_len;    // header bytes in the blob
    long long out_off;         // arena offset
    Quant q[2];                // luma, chroma
    union {
        yfv2_frame bgr;
        yfv2_strided_frame strided;
        yfv2_yuv420_frame yuv420;
        yfv2_yuv422_frame yuv422;
        yfv2_bayer_frame bayer;
    } f;
};

struct EncHeader {
    uint32_t magic;
    int n, nseg, ntiles;
    long long units;
    long long img_off, bytes;
    long long ws_coef, ws_cnt, ws_boff, ws_pos, ws_tsum, ws_stage, workspace, stage_words;
    long long arena;
    HuffEnc huff[4];           // DC luma, AC luma, DC chroma, AC chroma
};

// ---- host: tables and headers ---------------------------------------------------------------------------------------------------
// ITU-T T.81 Annex K: K.1 / K.2 quantisation tables (natural order) and K.3 / K.5 Huffman tables (jcparam's std_huff_tables)
const uint8_t kBaseQ[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112,
     100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
const uint8_t kBitsDcL[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kBitsDcC[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kValsDc[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kBitsAcL[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
const uint8_t kValsAcL[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kBitsAcC[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
const uint8_t kValsAcC[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t* const kBits[4] = {kBitsDcL, kBitsAcL, kBitsDcC, kBitsAcC};
const uint8_t* const kVals[4] = {kValsDc, kValsAcL, kValsDc, kValsAcC};

// jcomapi / jchuff jpeg_make_c_derived_tbl: canonical codes from the counts per length
void make_huff(const uint8_t* bits, const uint8_t* vals, HuffEnc& t) {
    memset(&t, 0, sizeof(t));
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < bits[l - 1]; ++i, ++k) {
            t.code[vals[k]] = (uint16_t)code++;
            t.size[vals[k]] = (uint8_t)l;
        }
        code <<= 1;
    }
}

// jcparam jpeg_set_quality(quality, force_baseline TRUE): jpeg_quality_scaling, then each entry scaled, rounded and clamped to
// 1..255.  cv2 has already clamped the quality to 0..100; 0 scales as 1.
void quant_table(int quality, int t, uint16_t* q) {
    if (quality <= 0) quality = 1;
    if (quality > 100) quality = 100;
    const long scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    for (int k = 0; k < 64; ++k) {
        long v = (kBaseQ[t][k] * scale + 50) / 100;
        q[k] = (uint16_t)(v < 1 ? 1 : v > 255 ? 255 : v);
    }
}

// jcdctmgr compute_reciprocal for divisor q << 3 (the islow FDCT's output is 8x the DCT), with 16-bit DCTELEMs (the SIMD build)
void make_quant(const uint16_t* q, Quant& d) {
    for (int k = 0; k < 64; ++k) {
        const uint32_t div = (uint32_t)q[k] << 3;
        int b = 0;
        while ((div >> (b + 1)) != 0) ++b;
        int r = 16 + b;
        uint32_t fq = (1u << r) / div;
        const uint32_t fr = (1u << r) % div;
        uint32_t c = div / 2;
        if (fr == 0) {
            fq >>= 1;
            --r;
        } else if (fr <= div / 2) {
            ++c;
        } else {
            ++fq;
        }
        d.recip[k] = (uint16_t)fq;
        d.corr[k] = (uint16_t)c;
        d.shift[k] = (uint8_t)r;
    }
}

// The bytes jcmarker writes before the scan data: SOI, APP0 (JFIF 1.01, no density, no thumbnail), DQT per table, SOF0, DHT
// per table (DC0 AC0 [DC1 AC1]), DRI when restarting, SOS
std::vector<uint8_t> make_headers(int w, int h, int ncomp, int hs, int vs, const uint16_t (*q)[64], int restart) {
    std::vector<uint8_t> o = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    auto u16 = [&](int v) { o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); };
    const int ntab = ncomp == 1 ? 1 : 2;
    for (int t = 0; t < ntab; ++t) {
        o.push_back(0xFF); o.push_back(0xDB); u16(67); o.push_back((uint8_t)t);
        for (int k = 0; k < 64; ++k) o.push_back((uint8_t)q[t][natural(k)]);
    }
    o.push_back(0xFF); o.push_back(0xC0); u16(8 + 3 * ncomp); o.push_back(8); u16(h); u16(w); o.push_back((uint8_t)ncomp);
    for (int c = 0; c < ncomp; ++c) {
        o.push_back((uint8_t)(c + 1));
        o.push_back((uint8_t)(c == 0 ? (hs << 4) | vs : 0x11));
        o.push_back((uint8_t)(c == 0 ? 0 : 1));
    }
    for (int t = 0; t < 2 * ntab; ++t) {
        int nv = 0;
        for (int l = 0; l < 16; ++l) nv += kBits[t][l];
        o.push_back(0xFF); o.push_back(0xC4); u16(3 + 16 + nv); o.push_back((uint8_t)(((t & 1) << 4) | (t >> 1)));
        for (int l = 0; l < 16; ++l) o.push_back(kBits[t][l]);
        for (int i = 0; i < nv; ++i) o.push_back(kVals[t][i]);
    }
    if (restart) { o.push_back(0xFF); o.push_back(0xDD); u16(4); u16(restart); }
    o.push_back(0xFF); o.push_back(0xDA); u16(6 + 2 * ncomp); o.push_back((uint8_t)ncomp);
    for (int c = 0; c < ncomp; ++c) {
        o.push_back((uint8_t)(c + 1));
        o.push_back((uint8_t)(c == 0 ? 0x00 : 0x11));
    }
    o.push_back(0); o.push_back(63); o.push_back(0);
    return o;
}

Geom make_geom(int w, int h, int ncomp, int hs, int vs, int restart) {
    Geom g{};
    g.w = w; g.h = h; g.ncomp = ncomp; g.restart = restart;
    g.hs = ncomp == 1 ? 1 : hs; g.vs = ncomp == 1 ? 1 : vs;
    g.mcux = (w + 8 * g.hs - 1) / (8 * g.hs);
    g.mcuy = (h + 8 * g.vs - 1) / (8 * g.vs);
    g.upm = ncomp == 1 ? 1 : g.hs * g.vs + 2;
    g.wb0 = (w + 7) / 8;
    g.hb0 = (h + 7) / 8;
    return g;
}

// cv2.imencode's JPEG parameters of one output (imwrite IMWRITE_JPEG_*), checked
struct Params {
    int quality = 95, hs = 2, vs = 2, restart = 0;
};

int parse_params(int i, const int* p, int np, Params& o) {
    if (np < 0 || (np & 1) || (np && !p)) {
        set_error("jpeg_encode_plan: output %d: params must be (id, value) pairs, got %d ints", i, np);
        return YFV2_EINVAL;
    }
    for (int k = 0; k < np; k += 2) {
        const int id = p[k], v = p[k + 1];
        switch (id) {
            case 1: o.quality = std::min(std::max(v, 0), 100); break;                      // IMWRITE_JPEG_QUALITY, cv2 clamps
            case 4: o.restart = std::min(std::max(v, 0), 65535); break;                    // IMWRITE_JPEG_RST_INTERVAL, cv2 clamps
            case 7:                                                                        // IMWRITE_JPEG_SAMPLING_FACTOR
                if (v == 0x221111) { o.hs = 2; o.vs = 2; }
                else if (v == 0x211111) { o.hs = 2; o.vs = 1; }
                else if (v == 0x111111) { o.hs = 1; o.vs = 1; }
                else if (v == 0x121111 || v == 0x411111) {
                    set_error("jpeg_encode_plan: output %d: sampling factor 0x%x (4:4:0 / 4:1:1) is not supported; 4:2:0, 4:2:2 and "
                              "4:4:4 are", i, v);
                    return YFV2_EUNSUPPORTED;
                } else {
                    set_error("jpeg_encode_plan: output %d: sampling factor 0x%x is none of cv2's IMWRITE_JPEG_SAMPLING_FACTOR_*", i, v);
                    return YFV2_EINVAL;
                }
                break;
            case 2: case 3:                                                                // PROGRESSIVE, OPTIMIZE
                if (v) {
                    set_error("jpeg_encode_plan: output %d: %s is not supported (baseline with the standard Huffman tables only)", i,
                              id == 2 ? "IMWRITE_JPEG_PROGRESSIVE" : "IMWRITE_JPEG_OPTIMIZE");
                    return YFV2_EUNSUPPORTED;
                }
                break;
            case 5: case 6:                                                                // LUMA_QUALITY, CHROMA_QUALITY
                if (v >= 0) {
                    set_error("jpeg_encode_plan: output %d: %s is not supported (one quality for both tables only)", i,
                              id == 5 ? "IMWRITE_JPEG_LUMA_QUALITY" : "IMWRITE_JPEG_CHROMA_QUALITY");
                    return YFV2_EUNSUPPORTED;
                }
                break;
            default: break;                                                                // other formats' ids: cv2 ignores them
        }
    }
    return YFV2_OK;
}

// The frame's size and a reason when its descriptor is unusable (the resize entries' checks, frame_fault)
const char* check_frame(const yfv2_jpeg_enc_src& s, int& fw, int& fh) {
    const auto fault = [&](const auto& f, const char* why) { fw = f.w; fh = f.h; return why; };
    switch (s.kind) {
        case YFV2_JPEG_SRC_BGR: return fault(s.f.bgr, frame_fault(s.f.bgr));
        case YFV2_JPEG_SRC_STRIDED: case YFV2_JPEG_SRC_GRAY:
            return fault(s.f.strided, frame_fault(s.f.strided, s.kind == YFV2_JPEG_SRC_GRAY));
        case YFV2_JPEG_SRC_YUV420: return fault(s.f.yuv420, frame_fault(s.f.yuv420));
        case YFV2_JPEG_SRC_YUV422: return fault(s.f.yuv422, frame_fault(s.f.yuv422));
        case YFV2_JPEG_SRC_BAYER: return fault(s.f.bayer, frame_fault(s.f.bayer));
        default: fw = fh = 0; return "unknown kind";
    }
}

long long align256(long long v) { return (v + 255) & ~255LL; }

// ---- device ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ const EncImage& image_of(const EncHeader& hd, const EncImage* im, long long u) {
    int lo = 0, hi = hd.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (im[mid].unit0 <= u) lo = mid; else hi = mid - 1;
    }
    return im[lo];
}

template <class Src>
struct FramePx {
    const typename Src::Desc& d;
    int x0, y0;
    __device__ __forceinline__ void operator()(int x, int y, int (&p)[3]) const {
        const Src row(d, y0 + y);
        int q[3];
        row.fetch(x0 + x, x0 + x, p, q);
    }
};

__device__ __forceinline__ int enc_sample(const EncImage& im, int c, int i, int j) {
    switch (im.kind) {
        case YFV2_JPEG_SRC_BGR: return comp_sample(FramePx<BgrSource>{im.f.bgr, im.x0, im.y0}, im.g, c, i, j);
        case YFV2_JPEG_SRC_YUV420: return comp_sample(FramePx<Yuv420Source>{im.f.yuv420, im.x0, im.y0}, im.g, c, i, j);
        case YFV2_JPEG_SRC_YUV422: return comp_sample(FramePx<Yuv422Source>{im.f.yuv422, im.x0, im.y0}, im.g, c, i, j);
        case YFV2_JPEG_SRC_BAYER: return comp_sample(FramePx<BayerSource>{im.f.bayer, im.x0, im.y0}, im.g, c, i, j);
        default: return comp_sample(FramePx<StridedSource>{im.f.strided, im.x0, im.y0}, im.g, c, i, j);
    }
}

// Stage 1: one unit per 64 threads; thread t is sample / coefficient t (row t / 8, column t % 8)
__global__ void __launch_bounds__(64 * kUnitsPerCta) enc_transform_kernel(const uint8_t* __restrict__ meta, int16_t* __restrict__ coef) {
    __shared__ int s[kUnitsPerCta][64];
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(meta);
    const EncImage* ims = reinterpret_cast<const EncImage*>(meta + hd.img_off);
    const int t = threadIdx.x, slot = threadIdx.y;
    const long long u = (long long)blockIdx.x * kUnitsPerCta + slot;
    const bool live = u < hd.units;
    const EncImage& im = image_of(hd, ims, live ? u : hd.units - 1);
    const Unit un = unit_of(im.g, (live ? u : hd.units - 1) - im.unit0);
    int* d = s[slot];
    d[t] = enc_sample(im, un.c, un.src_x * 8 + (t & 7), un.src_y * 8 + (t >> 3)) - 128;
    __syncthreads();
    if (t < 8) fdct_1d<0>(d + 8 * t, 1);
    __syncthreads();
    if (t < 8) fdct_1d<1>(d + t, 8);
    __syncthreads();
    if (!live) return;
    const int v = un.dummy && t ? 0 : quantize(d[t], im.q[un.c ? 1 : 0], t);
    coef[u * 64 + t] = (int16_t)v;
}

__device__ __forceinline__ int unit_diff(const EncImage& im, const int16_t* coef, long long u) {
    const long long p = dc_pred_unit(im.g, u - im.unit0);
    return coef[u * 64] - (p < 0 ? 0 : coef[(im.unit0 + p) * 64]);
}

// Stage 2a: each unit's Huffman bit count
__global__ void __launch_bounds__(256) enc_bits_kernel(const uint8_t* __restrict__ meta, const int16_t* __restrict__ coef,
                                                       int* __restrict__ bits) {
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(meta);
    const EncImage* ims = reinterpret_cast<const EncImage*>(meta + hd.img_off);
    const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= hd.units) return;
    const EncImage& im = image_of(hd, ims, u);
    const int c = unit_of(im.g, u - im.unit0).c ? 1 : 0;
    CountSink cs;
    encode_block(coef + u * 64, unit_diff(im, coef, u), hd.huff[2 * c], hd.huff[2 * c + 1], cs);
    bits[u] = cs.n;
}

// Exclusive scan of x over the CTA (blockDim.x a multiple of 32); total gets the sum
__device__ __forceinline__ long long cta_exclusive_scan(long long x, long long& total) {
    __shared__ long long warp[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    long long inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        long long w = lane < nw ? warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < nw) warp[lane] = w;
    }
    __syncthreads();
    const long long base = wid ? warp[wid - 1] : 0;
    total = warp[nw - 1];
    __syncthreads();
    return base + inc - x;
}

// Stage 2b / 4b: the exclusive scan of n int32 values into out[n + 1] (out[n]: the total), in three launches
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(const int* __restrict__ v, long long n, long long* __restrict__ tsum) {
    const long long i0 = (long long)blockIdx.x * kTile + threadIdx.x * kScanItems;
    long long s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k)
        if (i0 + k < n) s += v[i0 + k];
    long long total;
    cta_exclusive_scan(s, total);
    if (threadIdx.x == 0) tsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) scan_tiles_kernel(long long* __restrict__ tsum, int ntiles) {
    long long carry = 0;
    for (int b = 0; b < ntiles; b += blockDim.x) {
        const int i = b + threadIdx.x;
        const long long x = i < ntiles ? tsum[i] : 0;
        long long total;
        const long long e = cta_exclusive_scan(x, total);
        if (i < ntiles) tsum[i] = carry + e;
        carry += total;
    }
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const int* __restrict__ v, long long n, const long long* __restrict__ tsum,
                                                                  long long* __restrict__ out) {
    const long long i0 = (long long)blockIdx.x * kTile + threadIdx.x * kScanItems;
    long long s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k)
        if (i0 + k < n) s += v[i0 + k];
    long long total;
    long long e = cta_exclusive_scan(s, total) + tsum[blockIdx.x];
    for (int k = 0; k < kScanItems && i0 + k < n; ++k) {   // the values again (from L1): holding them costs more registers
        out[i0 + k] = e;
        e += v[i0 + k];
    }
    if (i0 <= n - 1 && n - 1 < i0 + kScanItems) out[n] = e;
}

// The segment of unit u: its first unit, one past its last, its index within the output and its first staging word
struct SegOf {
    long long ub, ue, word;
    int sidx;
};
__device__ __forceinline__ SegOf seg_of(const EncImage& im, const long long* boff, long long u) {
    SegOf s;
    const int mcu = (int)((u - im.unit0) / im.g.upm);
    s.sidx = im.g.restart ? mcu / im.g.restart : 0;
    const long long per = (long long)im.g.restart * im.g.upm;
    s.ub = im.unit0 + (im.g.restart ? s.sidx * per : 0);
    s.ue = im.g.restart ? min(s.ub + per, im.unit0 + im.nunits) : im.unit0 + im.nunits;
    s.word = (boff[s.ub] + 31) / 32 + im.seg0 + s.sidx;
    return s;
}

__global__ void enc_zero_kernel(const uint8_t* __restrict__ meta, const long long* __restrict__ boff, uint32_t* __restrict__ stage) {
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(meta);
    const long long words = (boff[hd.units] + 31) / 32 + hd.nseg + 1;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (long long)gridDim.x * blockDim.x) stage[i] = 0;
}

// MSB-first bits into staging words from bit position p on: the first word and the last partial one may hold a neighbour's bits
// and are merged with atomicOr; the words between are this unit's alone.  Bytes are in stream order in memory.
struct WordSink {
    uint32_t* stage;
    long long word;
    uint64_t acc;
    int n;
    bool first;
    __device__ __forceinline__ void emit(uint32_t x) {
        const uint32_t be = __byte_perm(x, 0, 0x0123);
        if (first) { atomicOr(stage + word, be); first = false; }
        else stage[word] = be;
        ++word;
    }
    __device__ __forceinline__ void put(uint32_t code, int size) {
        acc = (acc << size) | code;
        n += size;
        if (n >= 32) {
            emit((uint32_t)(acc >> (n - 32)));
            n -= 32;
        }
    }
    __device__ __forceinline__ void finish() {
        if (n > 0) atomicOr(stage + word, __byte_perm((uint32_t)(acc << (32 - n)), 0, 0x0123));
    }
};

// Stage 3: each unit's codes at its offset in its segment; the segment's last unit pads it with 1-bits to a byte
__global__ void __launch_bounds__(256) enc_pack_kernel(const uint8_t* __restrict__ meta, const int16_t* __restrict__ coef,
                                                       const long long* __restrict__ boff, uint32_t* __restrict__ stage) {
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(meta);
    const EncImage* ims = reinterpret_cast<const EncImage*>(meta + hd.img_off);
    const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= hd.units) return;
    const EncImage& im = image_of(hd, ims, u);
    const SegOf sg = seg_of(im, boff, u);
    const long long p = 32 * sg.word + boff[u] - boff[sg.ub];
    WordSink ws{stage, p >> 5, 0, (int)(p & 31), true};
    const int c = unit_of(im.g, u - im.unit0).c ? 1 : 0;
    encode_block(coef + u * 64, unit_diff(im, coef, u), hd.huff[2 * c], hd.huff[2 * c + 1], ws);
    if (u == sg.ue - 1) {
        const int pad = (int)((8 - (boff[sg.ue] - boff[sg.ub]) % 8) % 8);
        if (pad) ws.put((1u << pad) - 1, pad);
    }
    ws.finish();
}

// The staging bytes unit u owns: those whose first bit is in its bit range (the segment's last unit: up to the padded end)
__device__ __forceinline__ void owned_bytes(const SegOf& sg, const long long* boff, long long u, long long& b0, long long& b1) {
    const long long a = boff[u] - boff[sg.ub];
    const long long e = boff[u + 1] - boff[sg.ub];
    b0 = 4 * sg.word + (a + 7) / 8;
    b1 = 4 * sg.word + (e + 7) / 8;   // the last unit: e is the segment's length, and the padding fills its last byte
}

// Stage 4a: the output bytes each unit writes: its header (first unit), RSTn (first unit of a later segment), its bytes with
// every 0xFF doubled, EOI (last unit)
__global__ void __launch_bounds__(256) enc_count_kernel(const uint8_t* __restrict__ meta, const long long* __restrict__ boff,
                                                        const uint8_t* __restrict__ stage, int* __restrict__ cnt) {
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(meta);
    const EncImage* ims = reinterpret_cast<const EncImage*>(meta + hd.img_off);
    const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= hd.units) return;
    const EncImage& im = image_of(hd, ims, u);
    const SegOf sg = seg_of(im, boff, u);
    long long b0, b1;
    owned_bytes(sg, boff, u, b0, b1);
    int n = (int)(b1 - b0);
    for (long long b = b0; b < b1; ++b) n += stage[b] == 0xFF;
    if (u == im.unit0) n += (int)im.hdr_len;
    if (u == sg.ub && sg.sidx > 0) n += 2;
    if (u == im.unit0 + im.nunits - 1) n += 2;
    cnt[u] = n;
}

// Stage 4b: each unit's bytes at their place in the output; the first unit also writes the header and the output's length
__global__ void __launch_bounds__(256) enc_stuff_kernel(const uint8_t* __restrict__ meta, const long long* __restrict__ boff,
                                                        const uint8_t* __restrict__ stage, const long long* __restrict__ pos,
                                                        uint8_t* __restrict__ arena, long long* __restrict__ lengths) {
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(meta);
    const EncImage* ims = reinterpret_cast<const EncImage*>(meta + hd.img_off);
    const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= hd.units) return;
    const int i = (int)(&image_of(hd, ims, u) - ims);
    const EncImage& im = ims[i];
    const SegOf sg = seg_of(im, boff, u);
    uint8_t* o = arena + im.out_off + (pos[u] - pos[im.unit0]);
    if (u == im.unit0) {
        for (long long k = 0; k < im.hdr_len; ++k) o[k] = meta[im.hdr + k];
        o += im.hdr_len;
        lengths[i] = pos[im.unit0 + im.nunits] - pos[im.unit0];
    }
    if (u == sg.ub && sg.sidx > 0) {
        *o++ = 0xFF;
        *o++ = (uint8_t)(0xD0 + ((sg.sidx - 1) & 7));
    }
    long long b0, b1;
    owned_bytes(sg, boff, u, b0, b1);
    for (long long b = b0; b < b1; ++b) {
        const uint8_t x = stage[b];
        *o++ = x;
        if (x == 0xFF) *o++ = 0;
    }
    if (u == im.unit0 + im.nunits - 1) {
        o[0] = 0xFF;
        o[1] = 0xD9;
    }
}

int launch_scan(const int* v, long long n, long long* tsum, long long* out, cudaStream_t st) {
    const unsigned tiles = (unsigned)((n + kTile - 1) / kTile);
    scan_reduce_kernel<<<tiles, kScanThreads, 0, st>>>(v, n, tsum);
    YFV2_LAUNCH_CHECK();
    scan_tiles_kernel<<<1, 1024, 0, st>>>(tsum, (int)tiles);
    YFV2_LAUNCH_CHECK();
    scan_apply_kernel<<<tiles, kScanThreads, 0, st>>>(v, n, tsum, out);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

}  // namespace jpege
}  // namespace yfv2

extern "C" int yfv2_jpeg_encode_plan(const yfv2_jpeg_enc_src* srcs, int N, void* meta_host, size_t meta_cap, size_t* meta_bytes,
                                     size_t* workspace_bytes, long long* out_offsets, size_t* arena_bytes) {
    using namespace yfv2;
    using namespace yfv2::jpege;
    if (!srcs || N <= 0 || !meta_bytes || !workspace_bytes || !arena_bytes) {
        set_error("jpeg_encode_plan: null srcs / meta_bytes / workspace_bytes / arena_bytes or N <= 0");
        return YFV2_EINVAL;
    }
    std::vector<EncImage> ims(N);
    std::vector<std::vector<uint8_t>> hdrs(N);
    long long units = 0, arena = 0, stage_bits = 0;
    int nseg = 0;
    for (int i = 0; i < N; ++i) {
        const yfv2_jpeg_enc_src& s = srcs[i];
        Params p;
        const int rc = parse_params(i, s.params, s.nparams, p);
        if (rc) return rc;
        int fw, fh;
        if (const char* why = check_frame(s, fw, fh)) {
            set_error("jpeg_encode_plan: output %d: frame: %s (%dx%d)", i, why, fw, fh);
            return YFV2_EINVAL;
        }
        if (s.w <= 0 || s.h <= 0 || s.x0 < 0 || s.y0 < 0 || (long long)s.x0 + s.w > fw || (long long)s.y0 + s.h > fh) {
            set_error("jpeg_encode_plan: output %d: region (%d, %d) %dx%d is empty or outside the %dx%d frame", i, s.x0, s.y0, s.w, s.h,
                      fw, fh);
            return YFV2_EINVAL;
        }
        if (s.w > jpeg::kMaxSide || s.h > jpeg::kMaxSide) {
            set_error("jpeg_encode_plan: output %d: %dx%d is larger than %d on a side", i, s.w, s.h, jpeg::kMaxSide);
            return YFV2_EUNSUPPORTED;
        }
        const int ncomp = s.kind == YFV2_JPEG_SRC_GRAY ? 1 : 3;
        EncImage& im = ims[i];
        memset(&im, 0, sizeof(im));
        im.kind = s.kind;
        im.x0 = s.x0; im.y0 = s.y0;
        im.g = make_geom(s.w, s.h, ncomp, p.hs, p.vs, p.restart);
        const long long mcus = (long long)im.g.mcux * im.g.mcuy;
        im.nseg = p.restart ? (int)((mcus + p.restart - 1) / p.restart) : 1;
        im.seg0 = nseg;
        im.unit0 = units;
        im.nunits = mcus * im.g.upm;
        uint16_t q[2][64];
        quant_table(p.quality, 0, q[0]);
        quant_table(p.quality, 1, q[1]);
        make_quant(q[0], im.q[0]);
        make_quant(q[1], im.q[1]);
        memcpy(&im.f, &s.f, sizeof(im.f));
        hdrs[i] = make_headers(s.w, s.h, ncomp, im.g.hs, im.g.vs, q, p.restart);
        im.hdr_len = (long long)hdrs[i].size();
        // worst case: every block at kMaxBlockBits, every segment padded by a byte, every byte stuffed, RSTn and EOI
        const long long raw = im.nunits * ((kMaxBlockBits + 7) / 8) + im.nseg;
        im.out_off = arena;
        if (out_offsets) out_offsets[i] = arena;
        arena += align256(im.hdr_len + 2 * raw + 2LL * im.nseg + 2);
        units += im.nunits;
        stage_bits += im.nunits * (long long)kMaxBlockBits;
        nseg += im.nseg;
    }
    if (out_offsets) out_offsets[N] = arena;
    const long long img_off = align256(sizeof(EncHeader));
    long long bytes = img_off + (long long)N * sizeof(EncImage);
    for (int i = 0; i < N; ++i) {
        ims[i].hdr = bytes;
        bytes += ims[i].hdr_len;
    }
    bytes = align256(bytes);
    EncHeader hd;
    memset(&hd, 0, sizeof(hd));
    hd.magic = kMagic;
    hd.n = N;
    hd.nseg = nseg;
    hd.units = units;
    hd.ntiles = (int)((units + kTile - 1) / kTile);
    hd.img_off = img_off;
    hd.bytes = bytes;
    hd.stage_words = stage_bits / 32 + 2LL * nseg + 2;
    long long w = 0;
    hd.ws_coef = w;  w += align256(units * 64 * 2);
    hd.ws_cnt = w;   w += align256(units * 4);
    hd.ws_boff = w;  w += align256((units + 1) * 8);
    hd.ws_pos = w;   w += align256((units + 1) * 8);
    hd.ws_tsum = w;  w += align256((long long)hd.ntiles * 8);
    hd.ws_stage = w; w += align256(hd.stage_words * 4);
    hd.workspace = w;
    hd.arena = arena;
    for (int t = 0; t < 4; ++t) make_huff(kBits[t], kVals[t], hd.huff[t]);
    *meta_bytes = (size_t)bytes;
    *workspace_bytes = (size_t)w;
    *arena_bytes = (size_t)arena;
    if (!meta_host) return YFV2_OK;
    if (meta_cap < (size_t)bytes) {
        set_error("jpeg_encode_plan: meta_cap %zu < %lld bytes", meta_cap, bytes);
        return YFV2_ENOMEM;
    }
    uint8_t* m = static_cast<uint8_t*>(meta_host);
    memset(m, 0, (size_t)bytes);
    memcpy(m, &hd, sizeof(hd));
    memcpy(m + img_off, ims.data(), (size_t)N * sizeof(EncImage));
    for (int i = 0; i < N; ++i) memcpy(m + ims[i].hdr, hdrs[i].data(), hdrs[i].size());
    return YFV2_OK;
}

extern "C" int yfv2_jpeg_encode(const void* meta_host, const void* meta_dev, size_t meta_bytes, void* workspace, size_t workspace_bytes,
                                uint8_t* arena, size_t arena_bytes, long long* lengths, int phases, void* stream) {
    using namespace yfv2;
    using namespace yfv2::jpege;
    if (!meta_host || !meta_dev || !workspace || !arena || !lengths) {
        set_error("jpeg_encode: null meta_host / meta_dev / workspace / arena / lengths");
        return YFV2_EINVAL;
    }
    const EncHeader& hd = *static_cast<const EncHeader*>(meta_host);
    if (meta_bytes < sizeof(EncHeader) || hd.magic != kMagic || (size_t)hd.bytes != meta_bytes) {
        set_error("jpeg_encode: meta is not a blob yfv2_jpeg_encode_plan wrote (or meta_bytes differs)");
        return YFV2_EINVAL;
    }
    if (workspace_bytes < (size_t)hd.workspace || arena_bytes < (size_t)hd.arena) {
        set_error("jpeg_encode: workspace %zu / arena %zu bytes, the plan needs %lld / %lld", workspace_bytes, arena_bytes, hd.workspace,
                  hd.arena);
        return YFV2_ENOMEM;
    }
    if (phases <= 0 || (phases & ~YFV2_JPEG_ENC_ALL)) {
        set_error("jpeg_encode: phases %d: a nonzero subset of YFV2_JPEG_ENC_ALL", phases);
        return YFV2_EINVAL;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const uint8_t* meta = static_cast<const uint8_t*>(meta_dev);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    int16_t* coef = reinterpret_cast<int16_t*>(ws + hd.ws_coef);
    int* cnt = reinterpret_cast<int*>(ws + hd.ws_cnt);
    long long* boff = reinterpret_cast<long long*>(ws + hd.ws_boff);
    long long* pos = reinterpret_cast<long long*>(ws + hd.ws_pos);
    long long* tsum = reinterpret_cast<long long*>(ws + hd.ws_tsum);
    uint32_t* stage = reinterpret_cast<uint32_t*>(ws + hd.ws_stage);
    const unsigned unit_ctas = (unsigned)((hd.units + 255) / 256);
    if (phases & YFV2_JPEG_ENC_TRANSFORM) {
        enc_transform_kernel<<<(unsigned)((hd.units + kUnitsPerCta - 1) / kUnitsPerCta), dim3(64, kUnitsPerCta), 0, st>>>(meta, coef);
        YFV2_LAUNCH_CHECK();
    }
    if (phases & YFV2_JPEG_ENC_SCAN) {
        enc_bits_kernel<<<unit_ctas, 256, 0, st>>>(meta, coef, cnt);
        YFV2_LAUNCH_CHECK();
        if (int rc = launch_scan(cnt, hd.units, tsum, boff, st)) return rc;
    }
    if (phases & YFV2_JPEG_ENC_PACK) {
        enc_zero_kernel<<<1056, 256, 0, st>>>(meta, boff, stage);
        YFV2_LAUNCH_CHECK();
        enc_pack_kernel<<<unit_ctas, 256, 0, st>>>(meta, coef, boff, stage);
        YFV2_LAUNCH_CHECK();
    }
    if (phases & YFV2_JPEG_ENC_STUFF) {
        const uint8_t* sb = reinterpret_cast<const uint8_t*>(stage);
        enc_count_kernel<<<unit_ctas, 256, 0, st>>>(meta, boff, sb, cnt);
        YFV2_LAUNCH_CHECK();
        if (int rc = launch_scan(cnt, hd.units, tsum, pos, st)) return rc;
        enc_stuff_kernel<<<unit_ctas, 256, 0, st>>>(meta, boff, sb, pos, arena, lengths);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}
