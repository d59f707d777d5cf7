// Baseline JPEG files -> packed HWC BGR frames, the bytes cv2.imread returns (yfv2_jpeg_parse / yfv2_jpeg_decode).
//
// The host parser walks each file's markers, refuses what is out of scope with a reason, builds the decode tables and finds the
// byte range of every entropy-coded segment (the whole scan, or one restart interval), all into a blob the caller copies to the
// device.  The decode then runs three launches on the caller's stream, each over functions of jpeg.cuh:
//   1. entropy_kernel: one thread per segment, Huffman decode into int16 coefficient blocks in the workspace;
//   2. idct_kernel:    one thread per block, jpeg_idct_islow into one uint8 plane per component;
//   3. color_kernel:   one thread per output pixel, upsampling, YCbCr -> BGR and the EXIF orientation into the frame arena.
// Progressive files (yfv2_jpeg_parse_ex with YFV2_JPEG_PROGRESSIVE) have no baseline segments: phase 1 zeroes their coefficients
// and runs prog_entropy_kernel once per level of their scans, one thread per segment of a scan (or of one restart interval).
#include <algorithm>
#include <climits>
#include <cstddef>
#include <cstdarg>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "jpeg.cuh"

namespace yfv2 {
namespace {

using namespace jpeg;

constexpr int kEntropyThreads = 32;
constexpr int kIdctThreads = 128;
constexpr int kColorThreads = 256;

// ---- host parser --------------------------------------------------------------------------------------------------------------
struct RawHuff {
    bool defined = false;
    uint8_t bits[17] = {};
    uint8_t vals[256] = {};
};

struct Parsed {
    int w = 0, h = 0, ncomp = 0, orient = 1, restart = 0;
    int id[3] = {}, hs[3] = {}, vs[3] = {}, tq[3] = {};
    Image* im = nullptr;                 // filled at SOS (tables latched there), when the caller wants the blob
    std::vector<Seg> segs;
    // a progressive file (SOF2 under YFV2_JPEG_PROGRESSIVE): its scans, their tables (Scan::tab indexes huffs) and segments
    bool prog = false, eoi = false;
    int restart0 = 0;                    // the first scan's restart interval
    std::vector<Scan> scans;
    std::vector<Huff> huffs;
    std::vector<PSeg> psegs;             // PSeg::scan indexes scans
};

// One entropy-coded segment of a scan: units [u0, u0 + nu) of the scan, its bytes and the flags found while cutting it
struct Piece {
    int u0, nu, err;
    long long begin, end;
};

// The segments of a scan of `units` MCUs (or blocks) with restart interval `restart`, from the RSTn-delimited byte ranges
// scan_entropy found and the marker after each
std::vector<Piece> cut_scan(long long units, int restart, const std::vector<std::pair<long long, long long>>& ranges,
                            const std::vector<int>& ends) {
    const long long nseg = restart ? (units + restart - 1) / restart : 1;
    std::vector<Piece> out;
    for (long long k = 0; k < nseg; ++k) {
        Piece g{};
        g.u0 = (int)(k * (restart ? restart : units));
        g.nu = (int)(restart ? (units - g.u0 < restart ? units - g.u0 : restart) : units);
        if (k < (long long)ranges.size()) {
            g.begin = ranges[k].first;
            g.end = ranges[k].second;
            // cv2.imdecode returns no image when the file ends inside the scan
            if (ends[k] < 0) g.err |= kErrShort;
            // The interval ends at RST(k mod 8).  libjpeg's jpeg_resync_to_restart takes a marker 1 or 2 numbers ahead as a
            // missing one (this interval decodes from no data) and 1 or 2 behind as a stale one (the data after it is skipped):
            // its intervals then hold other data than these segments.  A marker 3 to 5 away it takes as the expected one, as the
            // segments here do.
            const int d = (ends[k] - 0xD0 - (int)k) & 7;
            if (k + 1 < nseg && ends[k] >= 0xD0 && ends[k] <= 0xD7 && (d == 1 || d == 2 || d == 6 || d == 7)) g.err |= kErrRestart;
        } else {
            g.begin = g.end = ranges.back().second;      // a missing interval decodes from no data (flagged)
        }
        out.push_back(g);
    }
    return out;
}

struct Refuse {
    int code;
    char why[96];
};

[[noreturn]] void refuse(int code, const char* fmt, ...) {
    Refuse r;
    r.code = code;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(r.why, sizeof r.why, fmt, ap);
    va_end(ap);
    throw r;
}

int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// jdhuff.c jpeg_make_d_derived_tbl
void build_huff(const RawHuff& raw, bool dc, Huff& t) {
    int size[257], code[257];
    int p = 0;
    for (int l = 1; l <= 16; ++l)
        for (int i = 0; i < raw.bits[l]; ++i) {
            if (p >= 256) refuse(YFV2_EINVAL, "bad Huffman table (more than 256 codes)");
            size[p++] = l;
        }
    size[p] = 0;
    const int nsym = p;
    int c = 0, si = size[0];
    p = 0;
    while (size[p]) {
        while (size[p] == si) code[p++] = c++;
        if (c >= (1 << si)) refuse(YFV2_EINVAL, "bad Huffman table (code lengths overflow)");
        c <<= 1;
        ++si;
    }
    p = 0;
    for (int l = 1; l <= 16; ++l) {
        if (raw.bits[l]) {
            t.valoff[l] = p - code[p];
            p += raw.bits[l];
            t.maxcode[l] = code[p - 1];
        } else {
            t.maxcode[l] = -1;
            t.valoff[l] = 0;
        }
    }
    t.maxcode[0] = -1; t.valoff[0] = 0;
    t.maxcode[17] = 0xFFFFF; t.valoff[17] = 0;
    memset(t.fast, 0, sizeof t.fast);
    p = 0;
    for (int l = 1; l <= kFastBits; ++l)
        for (int i = 0; i < raw.bits[l]; ++i, ++p) {
            const int look = code[p] << (kFastBits - l);
            for (int k = 0; k < (1 << (kFastBits - l)); ++k) t.fast[look + k] = (uint16_t)((l << 8) | raw.vals[p]);
        }
    memcpy(t.vals, raw.vals, sizeof t.vals);
    if (dc)
        for (int i = 0; i < nsym; ++i)
            if (raw.vals[i] > 15) refuse(YFV2_EINVAL, "bad Huffman table (DC symbol %d)", raw.vals[i]);
}

// EXIF orientation (tag 0x0112 of IFD0) from an APP1 payload starting "Exif\0\0"; 1 when absent or out of range
int exif_orientation(const uint8_t* p, int n) {
    if (n < 14 || memcmp(p, "Exif\0\0", 6) != 0) return 1;
    const uint8_t* t = p + 6;
    const int tn = n - 6;
    bool le;
    if (t[0] == 'I' && t[1] == 'I') le = true;
    else if (t[0] == 'M' && t[1] == 'M') le = false;
    else return 1;
    auto u16 = [&](int o) { return le ? t[o] | (t[o + 1] << 8) : (t[o] << 8) | t[o + 1]; };
    auto u32 = [&](int o) {
        return le ? (uint32_t)t[o] | ((uint32_t)t[o + 1] << 8) | ((uint32_t)t[o + 2] << 16) | ((uint32_t)t[o + 3] << 24)
                  : ((uint32_t)t[o] << 24) | ((uint32_t)t[o + 1] << 16) | ((uint32_t)t[o + 2] << 8) | (uint32_t)t[o + 3];
    };
    if (u16(2) != 42) return 1;
    const uint32_t ifd = u32(4);
    if (ifd > (uint32_t)tn - 2) return 1;
    const int cnt = u16((int)ifd);
    for (int i = 0; i < cnt; ++i) {
        const long long e = (long long)ifd + 2 + 12LL * i;
        if (e + 10 > tn) break;   // OpenCV reads an entry whose last 2 bytes (past the 16-bit value) are cut off
        if (u16((int)e) == 0x0112) {
            const int v = u16((int)e + 8);   // OpenCV's ExifReader: a 16-bit word at the value offset, whatever the type and count
            return v >= 1 && v <= 8 ? v : 1;
        }
    }
    return 1;
}

const char* sof_name(int m) {
    switch (m) {
        case 0xC2: return "progressive DCT (SOF2)";
        case 0xC3: return "lossless (SOF3)";
        case 0xC5: return "hierarchical sequential (SOF5)";
        case 0xC6: return "hierarchical progressive (SOF6)";
        case 0xC7: return "hierarchical lossless (SOF7)";
        case 0xC9: return "arithmetic-coded sequential (SOF9)";
        case 0xCA: return "arithmetic-coded progressive (SOF10)";
        case 0xCB: return "arithmetic-coded lossless (SOF11)";
        case 0xCD: return "hierarchical arithmetic-coded (SOF13)";
        case 0xCE: return "hierarchical arithmetic-coded (SOF14)";
        case 0xCF: return "hierarchical arithmetic-coded (SOF15)";
        default: return nullptr;
    }
}

// Offset just past the entropy-coded data starting at `pos`; appends one [begin, end) range per RSTn-delimited piece, and to
// `ends` the marker byte after it (-1: the file ends first)
size_t scan_entropy(const uint8_t* f, size_t size, size_t pos, long long file_off, std::vector<std::pair<long long, long long>>& r,
                    std::vector<int>& ends) {
    size_t begin = pos, i = pos;
    while (true) {
        const void* q = i < size ? memchr(f + i, 0xFF, size - i) : nullptr;
        if (!q) {                                            // no end-of-scan marker: a truncated file, the last piece ends there
            r.emplace_back(file_off + (long long)begin, file_off + (long long)size);
            ends.push_back(-1);
            return size;
        }
        i = (const uint8_t*)q - f;
        size_t j = i + 1;
        while (j < size && f[j] == 0xFF) ++j;
        if (j >= size) {
            r.emplace_back(file_off + (long long)begin, file_off + (long long)i);
            ends.push_back(-1);
            return size;
        }
        if (f[j] == 0x00) { i = j + 1; continue; }
        r.emplace_back(file_off + (long long)begin, file_off + (long long)i);
        ends.push_back(f[j]);
        if (f[j] >= 0xD0 && f[j] <= 0xD7) { begin = i = j + 1; continue; }
        return i;                                            // the marker that ends the scan
    }
}

// The frame's geometry into P.im at its first scan: size, sampling, MCU and block grids (tables and quantisation are latched apart)
void frame_geometry(const Parsed& P, Image* im) {
    const bool grey = P.ncomp == 1;
    const int hmax = grey ? 1 : P.hs[0], vmax = grey ? 1 : P.vs[0];
    im->w = P.w; im->h = P.h; im->ncomp = P.ncomp; im->hmax = hmax; im->vmax = vmax;
    im->mcux = (P.w + 8 * hmax - 1) / (8 * hmax);
    im->mcuy = (P.h + 8 * vmax - 1) / (8 * vmax);
    im->restart = P.restart; im->orient = P.orient;
    for (int c = 0; c < P.ncomp; ++c) {
        Comp& cp = im->comp[c];
        cp.h = grey ? 1 : P.hs[c];
        cp.v = grey ? 1 : P.vs[c];
        cp.bw = im->mcux * cp.h;
        cp.bh = im->mcuy * cp.v;
        cp.dw = (int)(((long long)P.w * cp.h + hmax - 1) / hmax);
        cp.dh = (int)(((long long)P.h * cp.v + vmax - 1) / vmax);
        cp.pitch = 8 * cp.bw;
    }
}

// Refusals of a colour space outside the subset, made at the first scan (where libjpeg settles it)
void check_colour(const Parsed& P, bool jfif, bool adobe, int adobe_transform) {
    if (P.ncomp == 3 && !jfif) {
        if (adobe && adobe_transform == 0) refuse(YFV2_EUNSUPPORTED, "RGB-coded (Adobe APP14 transform 0)");
        if (!adobe && P.id[0] == 'R' && P.id[1] == 'G' && P.id[2] == 'B') refuse(YFV2_EUNSUPPORTED, "RGB-coded (component ids R, G, B)");
    }
}

// Per-file state of a progressive parse: libjpeg's coef_bits (the lowest bit known of each coefficient, -1: none yet) and
// which components have latched their quantisation table
struct Progress {
    int bits[3][64];
    bool latched[3] = {};
    Progress() { memset(bits, 0xFF, sizeof bits); }
};

// One SOS of a progressive file (payload s[n], entropy-coded data from pos): validates the scan the way libjpeg-turbo's
// start_pass_phuff_decoder and latch_quant_tables do, builds its tables, gives it a level and cuts its segments.  Returns the
// offset past its entropy-coded data.
size_t prog_scan(const uint8_t* f, size_t size, size_t pos, long long file_off, const uint8_t* s, int n, Parsed& P, Progress& G,
                 const RawHuff* hdc, const RawHuff* hac, const uint16_t (*qt)[64], const bool* qdef) {
    const int si = (int)P.scans.size();
    if (n < 1 || n < 4 + 2 * s[0]) refuse(YFV2_EINVAL, "short scan header");
    const int ns = s[0];
    if (ns < 1 || ns > P.ncomp) refuse(YFV2_EINVAL, "progressive scan %d has %d components", si, ns);
    if (si == kMaxScans) refuse(YFV2_EUNSUPPORTED, "progressive file with more than %d scans", kMaxScans);
    Scan sc{};
    sc.ncomp = ns;
    sc.ss = s[1 + 2 * ns];
    sc.se = s[2 + 2 * ns];
    sc.ah = s[3 + 2 * ns] >> 4;
    sc.al = s[3 + 2 * ns] & 15;
    sc.tab[0] = sc.tab[1] = sc.tab[2] = -1;
    int td[3], ta[3];
    for (int k = 0; k < ns; ++k) {
        int c = 0;
        while (c < P.ncomp && P.id[c] != s[1 + 2 * k]) ++c;
        if (c == P.ncomp) refuse(YFV2_EINVAL, "progressive scan %d: component id %d is not in the frame", si, s[1 + 2 * k]);
        if (k && c <= sc.comp[k - 1]) refuse(YFV2_EUNSUPPORTED, "progressive scan %d: components not in frame order", si);
        sc.comp[k] = c;
        td[k] = s[2 + 2 * k] >> 4;
        ta[k] = s[2 + 2 * k] & 15;
    }
    // libjpeg's JERR_BAD_PROGRESSION: cv2 returns no image
    const bool dc = sc.ss == 0;
    if (dc && sc.se != 0) refuse(YFV2_EINVAL, "bad progressive scan %d: a DC scan with Se = %d", si, sc.se);
    if (!dc && (sc.ss > sc.se || sc.se > 63)) refuse(YFV2_EINVAL, "bad progressive scan %d: coefficients %d..%d", si, sc.ss, sc.se);
    if (!dc && ns != 1) refuse(YFV2_EINVAL, "bad progressive scan %d: an AC scan of %d components", si, ns);
    if (sc.ah != 0 && sc.al != sc.ah - 1) refuse(YFV2_EINVAL, "bad progressive scan %d: Ah %d with Al %d", si, sc.ah, sc.al);
    if (sc.al > 13) refuse(YFV2_EINVAL, "bad progressive scan %d: Al %d", si, sc.al);
    // libjpeg's JWRN_BOGUS_PROGRESSION: cv2 decodes what the scans say, and this decoder does not follow it there
    for (int k = 0; k < ns; ++k) {
        const int c = sc.comp[k];
        if (!dc && G.bits[c][0] < 0) refuse(YFV2_EUNSUPPORTED, "bogus progressive scan %d: AC of component %d before its DC", si, c);
        for (int q = sc.ss; q <= sc.se; ++q) {
            const int expect = G.bits[c][q] < 0 ? 0 : G.bits[c][q];
            if (sc.ah != expect)
                refuse(YFV2_EUNSUPPORTED, "bogus progressive scan %d: component %d coefficient %d has Ah %d, %d expected", si, c, q, sc.ah, expect);
            G.bits[c][q] = sc.al;
        }
    }
    // Huffman tables latched here; a DC refinement reads raw bits and needs none
    for (int k = 0; k < prog_ntabs(sc); ++k) {
        const int t = dc ? td[k] : ta[k];
        const RawHuff* raw = dc ? hdc : hac;
        if (t > 3 || !raw[t].defined) refuse(YFV2_EINVAL, "scan uses an undefined Huffman table");
        sc.tab[k] = (int)P.huffs.size();
        P.huffs.emplace_back();
        build_huff(raw[t], dc, P.huffs.back());
    }
    // a component's quantisation table is latched at its first scan: a later DQT does not change it
    for (int k = 0; k < ns; ++k) {
        const int c = sc.comp[k];
        if (G.latched[c]) continue;
        if (!qdef[P.tq[c]]) refuse(YFV2_EINVAL, "component %d uses an undefined quantisation table", c);
        memcpy(P.im->comp[c].q, qt[P.tq[c]], sizeof P.im->comp[c].q);
        G.latched[c] = true;
    }
    for (const Scan& o : P.scans) {                   // a level above every earlier scan it shares a coefficient with
        bool overlap = o.ss <= sc.se && sc.ss <= o.se;
        bool shared = false;
        for (int a = 0; a < o.ncomp; ++a)
            for (int b = 0; b < ns; ++b) shared = shared || o.comp[a] == sc.comp[b];
        if (overlap && shared && o.level + 1 > sc.level) sc.level = o.level + 1;
    }
    const Image& im = *P.im;
    if (ns > 1) {
        sc.upr = im.mcux;
        sc.units = im.mcux * im.mcuy;
    } else {
        const Comp& cp = im.comp[sc.comp[0]];
        sc.upr = (cp.dw + 7) / 8;
        sc.units = sc.upr * ((cp.dh + 7) / 8);
    }
    if (si == 0) P.restart0 = P.restart;
    std::vector<std::pair<long long, long long>> ranges;
    std::vector<int> ends;
    pos = scan_entropy(f, size, pos, file_off, ranges, ends);
    for (const Piece& p : cut_scan(sc.units, P.restart, ranges, ends)) {
        PSeg g{};
        g.scan = si;
        g.level = sc.level;
        g.unit0 = p.u0;
        g.nunit = p.nu;
        g.err = p.err;
        g.begin = p.begin;
        g.end = p.end;
        P.psegs.push_back(g);
    }
    P.scans.push_back(sc);
    return pos;
}

// The end of a progressive file: without its EOI cv2.imdecode returns no image, so the file is flagged; with it, every coefficient
// must have been refined to its last bit (libjpeg would smooth the blocks of an incomplete one, which is not reproduced)
void prog_finish(Parsed& P, const Progress& G) {
    if (!P.eoi) {
        P.psegs[0].err |= kErrShort;
        return;
    }
    for (int c = 0; c < P.ncomp; ++c)
        for (int q = 0; q < 64; ++q) {
            if (G.bits[c][q] < 0) refuse(YFV2_EUNSUPPORTED, "incomplete progressive file: component %d coefficient %d is never sent", c, q);
            if (G.bits[c][q] > 0)
                refuse(YFV2_EUNSUPPORTED, "incomplete progressive refinement: component %d coefficient %d ends at Al %d", c, q, G.bits[c][q]);
        }
}

// One file: validates it against the supported subset, fills P (and P.im's tables when non-null); throws Refuse.  flags:
// YFV2_JPEG_PROGRESSIVE accepts progressive (SOF2) files.
void parse_markers(const uint8_t* f, size_t size, long long file_off, Parsed& P, int flags, Progress& G);

void parse_file(const uint8_t* f, size_t size, long long file_off, Parsed& P, int flags) {
    Progress G;
    parse_markers(f, size, file_off, P, flags, G);
    if (P.prog) prog_finish(P, G);
}

void parse_markers(const uint8_t* f, size_t size, long long file_off, Parsed& P, int flags, Progress& G) {
    if (size < 2 || f[0] != 0xFF || f[1] != 0xD8) {
        if (size >= 8 && memcmp(f, "\x89PNG\r\n\x1a\n", 8) == 0) refuse(YFV2_EUNSUPPORTED, "not a JPEG (a PNG file)");
        refuse(YFV2_EUNSUPPORTED, "not a JPEG (no SOI marker)");
    }
    uint16_t qt[4][64];
    bool qdef[4] = {};
    RawHuff hdc[4], hac[4];
    bool sof = false, jfif = false, adobe = false, scanned = false;
    int adobe_transform = -1;
    bool exif_seen = false;
    size_t pos = 2;
    while (true) {
        if (pos >= size) {
            if (scanned) return;                           // no EOI after the scan: libjpeg warns and decodes what is there
            refuse(YFV2_EINVAL, "truncated header (end of file before the scan)");
        }
        if (f[pos] != 0xFF) {
            if (scanned) return;
            refuse(YFV2_EINVAL, "corrupt header (0x%02x where a marker should be, offset %zu)", f[pos], pos);
        }
        while (pos < size && f[pos] == 0xFF) ++pos;
        if (pos >= size) {
            if (scanned) return;
            refuse(YFV2_EINVAL, "truncated header");
        }
        const int m = f[pos++];
        if (m == 0xD9) {
            if (!scanned) refuse(YFV2_EINVAL, "no scan before EOI");
            P.eoi = true;
            return;
        }
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;   // markers without a length
        if (pos + 2 > size) {
            if (scanned) return;
            refuse(YFV2_EINVAL, "truncated header (marker 0x%02x)", m);
        }
        const int len = be16(f + pos);
        if (len < 2 || pos + len > size) {
            if (scanned) return;
            refuse(YFV2_EINVAL, "truncated header (marker 0x%02x, %d bytes)", m, len);
        }
        const uint8_t* s = f + pos + 2;
        const int n = len - 2;
        pos += len;
        if (scanned && !P.prog) {                          // a progressive file's tables and scans go on after its first scan
            if (m == 0xDA) refuse(YFV2_EUNSUPPORTED, "more than one scan");
            continue;
        }
        const bool prog_sof = m == 0xC2 && (flags & YFV2_JPEG_PROGRESSIVE);
        if (const char* nm = sof_name(m); nm && !prog_sof) refuse(YFV2_EUNSUPPORTED, "%s", nm);
        if (m == 0xCC) refuse(YFV2_EUNSUPPORTED, "arithmetic coding (DAC)");
        if (m == 0xC0 || m == 0xC1 || prog_sof) {
            if (sof) refuse(YFV2_EINVAL, "two frame headers");
            sof = true;
            P.prog = prog_sof;
            if (n < 6) refuse(YFV2_EINVAL, "short frame header");
            if (s[0] != 8) refuse(YFV2_EUNSUPPORTED, "%d-bit samples", s[0]);
            P.h = be16(s + 1);
            P.w = be16(s + 3);
            P.ncomp = s[5];
            if (P.ncomp != 1 && P.ncomp != 3) refuse(YFV2_EUNSUPPORTED, "%d components", P.ncomp);
            if (n < 6 + 3 * P.ncomp) refuse(YFV2_EINVAL, "short frame header");
            if (P.h == 0) refuse(YFV2_EUNSUPPORTED, "height defined by a DNL marker");
            if (P.w == 0) refuse(YFV2_EINVAL, "zero width");
            if (P.w > kMaxSide || P.h > kMaxSide) refuse(YFV2_EUNSUPPORTED, "%dx%d is larger than %d on a side", P.w, P.h, kMaxSide);
            for (int c = 0; c < P.ncomp; ++c) {
                P.id[c] = s[6 + 3 * c];
                P.hs[c] = s[7 + 3 * c] >> 4;
                P.vs[c] = s[7 + 3 * c] & 15;
                P.tq[c] = s[8 + 3 * c];
                if (P.tq[c] > 3) refuse(YFV2_EINVAL, "quantisation table %d", P.tq[c]);
            }
            const int h0 = P.hs[0], v0 = P.vs[0];
            const bool luma = (h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 2 && v0 == 2) || (h0 == 1 && v0 == 2) ||
                              (h0 == 4 && v0 == 1);
            bool ok = luma;
            for (int c = 1; c < P.ncomp; ++c) ok = ok && P.hs[c] == 1 && P.vs[c] == 1;
            if (!ok) {
                if (P.ncomp == 3)
                    refuse(YFV2_EUNSUPPORTED, "sampling %dx%d,%dx%d,%dx%d", P.hs[0], P.vs[0], P.hs[1], P.vs[1], P.hs[2], P.vs[2]);
                refuse(YFV2_EUNSUPPORTED, "sampling %dx%d", P.hs[0], P.vs[0]);
            }
        } else if (m == 0xC4) {
            int o = 0;
            while (o < n) {
                const int tc = s[o] >> 4, th = s[o] & 15;
                if (tc > 1 || th > 3 || o + 17 > n) refuse(YFV2_EINVAL, "bad DHT segment");
                RawHuff& t = tc ? hac[th] : hdc[th];
                t = RawHuff{};
                int cnt = 0;
                for (int l = 1; l <= 16; ++l) cnt += (t.bits[l] = s[o + l]);
                if (cnt > 256 || o + 17 + cnt > n) refuse(YFV2_EINVAL, "bad DHT segment");
                memcpy(t.vals, s + o + 17, cnt);
                t.defined = true;
                o += 17 + cnt;
            }
        } else if (m == 0xDB) {
            int o = 0;
            while (o < n) {
                const int pq = s[o] >> 4, tq = s[o] & 15;
                if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > n) refuse(YFV2_EINVAL, "bad DQT segment");
                for (int k = 0; k < 64; ++k)
                    qt[tq][kNaturalHost[k]] = (uint16_t)(pq ? be16(s + o + 1 + 2 * k) : s[o + 1 + k]);
                qdef[tq] = true;
                o += 1 + 64 * (pq + 1);
            }
        } else if (m == 0xDD) {
            if (n < 2) refuse(YFV2_EINVAL, "bad DRI segment");
            P.restart = be16(s);
        } else if (m == 0xE0) {
            if (n >= 14 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;   // jdmarker's examine_app0 ignores a shorter one
        } else if (m == 0xE1) {
            if (!exif_seen && n >= 6 && memcmp(s, "Exif\0\0", 6) == 0) {
                exif_seen = true;
                P.orient = exif_orientation(s, n);
            }
        } else if (m == 0xEE) {
            if (n >= 12 && memcmp(s, "Adobe", 5) == 0) {
                adobe = true;
                adobe_transform = s[11];
            }
        } else if (m == 0xDA) {
            if (!sof) refuse(YFV2_EINVAL, "scan before the frame header");
            if (P.prog) {
                if (!scanned) {
                    check_colour(P, jfif, adobe, adobe_transform);
                    frame_geometry(P, P.im);
                }
                scanned = true;
                pos = prog_scan(f, size, pos, file_off, s, n, P, G, hdc, hac, qt, qdef);
                continue;
            }
            if (n < 1) refuse(YFV2_EINVAL, "short scan header");
            const int ns = s[0];
            if (n < 4 + 2 * ns) refuse(YFV2_EINVAL, "short scan header");
            if (ns != P.ncomp) refuse(YFV2_EUNSUPPORTED, "more than one scan (this one has %d of %d components)", ns, P.ncomp);
            check_colour(P, jfif, adobe, adobe_transform);
            int td[3], ta[3];
            for (int k = 0; k < ns; ++k) {
                if (s[1 + 2 * k] != P.id[k]) refuse(YFV2_EUNSUPPORTED, "scan components not in frame order");
                td[k] = s[2 + 2 * k] >> 4;
                ta[k] = s[2 + 2 * k] & 15;
                if (td[k] > 3 || ta[k] > 3 || !hdc[td[k]].defined || !hac[ta[k]].defined)
                    refuse(YFV2_EINVAL, "scan uses an undefined Huffman table");
                if (!qdef[P.tq[k]]) refuse(YFV2_EINVAL, "component %d uses an undefined quantisation table", k);
            }
            scanned = true;
            Image* im = P.im;
            frame_geometry(P, im);
            std::vector<std::pair<long long, long long>> ranges;
            std::vector<int> ends;
            pos = scan_entropy(f, size, pos, file_off, ranges, ends);
            P.segs.clear();
            for (const Piece& p : cut_scan((long long)im->mcux * im->mcuy, P.restart, ranges, ends)) {
                Seg g{};
                g.mcu0 = p.u0;
                g.nmcu = p.nu;
                g.err = p.err;
                g.begin = p.begin;
                g.end = p.end;
                P.segs.push_back(g);
            }
            for (int c = 0; c < P.ncomp; ++c) {
                memcpy(im->comp[c].q, qt[P.tq[c]], sizeof im->comp[c].q);
                build_huff(hdc[td[c]], true, im->dc[c]);
                build_huff(hac[ta[c]], false, im->ac[c]);
            }
        }
    }
}

long long align16(long long x) { return (x + 15) & ~15LL; }

// ---- device phases ------------------------------------------------------------------------------------------------------------
// One segment per CTA: the warp copies the image's Huffman tables (6 x 1.4 KB) into shared memory, then lane 0 decodes.  Read
// from global memory, the tables of the images a SM decodes at once do not fit its L1, and every symbol waited on a miss.
__global__ void __launch_bounds__(kEntropyThreads) entropy_kernel(const Header* hd, const uint8_t* files, uint8_t* ws, int* errors) {
    __shared__ Huff tabs[6];
    const uint8_t* blob = reinterpret_cast<const uint8_t*>(hd);
    const Seg& s = reinterpret_cast<const Seg*>(blob + hd->seg_off)[blockIdx.x];
    const Image& im = reinterpret_cast<const Image*>(blob + hd->img_off)[s.img];
    static_assert(sizeof(Huff) % 16 == 0 && sizeof(Image) % 16 == 0 && offsetof(Image, dc) % 16 == 0 &&
                  offsetof(Image, ac) == offsetof(Image, dc) + 3 * sizeof(Huff), "dc[3], ac[3] are copied as one aligned run");
    const uint4* src = reinterpret_cast<const uint4*>(im.dc);
    uint4* dst = reinterpret_cast<uint4*>(tabs);
    for (int i = threadIdx.x; i < 6 * (int)sizeof(Huff) / 16; i += kEntropyThreads) {
        const int t = i / ((int)sizeof(Huff) / 16);                  // table t: dc 0..2, then ac 0..2
        if (t % 3 < im.ncomp) dst[i] = src[i];
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int err = decode_segment(im, s, files, ws, tabs, tabs + 3);
    if (err) atomicOr(errors + s.img, err);
}

__global__ void __launch_bounds__(kIdctThreads) idct_kernel(const Header* hd, uint8_t* ws) {
    const uint8_t* blob = reinterpret_cast<const uint8_t*>(hd);
    const Image& im = reinterpret_cast<const Image*>(blob + hd->img_off)[blockIdx.y];
    for (long long k = (long long)blockIdx.x * kIdctThreads + threadIdx.x; k < im.blocks; k += (long long)gridDim.x * kIdctThreads)
        idct_block(im, k, ws);
}

__global__ void __launch_bounds__(kColorThreads) color_kernel(const Header* hd, const uint8_t* ws, uint8_t* frames) {
    const uint8_t* blob = reinterpret_cast<const uint8_t*>(hd);
    const Image& im = reinterpret_cast<const Image*>(blob + hd->img_off)[blockIdx.y];
    const long long npix = (long long)im.ow * im.oh;
    uint8_t* out = frames + im.frame;
    for (long long p = (long long)blockIdx.x * kColorThreads + threadIdx.x; p < npix; p += (long long)gridDim.x * kColorThreads) {
        const int oy = (int)(p / im.ow), ox = (int)(p % im.ow);
        bgr_pixel(im, ws, ox, oy, out + 3 * p);
    }
}

// Progressive segment first + blockIdx.x per CTA, all of one level: the warp copies the scan's tables (up to 3 DC or 1 AC) from
// the blob's pool into shared memory, then lane 0 decodes onto the coefficients lower levels wrote
__global__ void __launch_bounds__(kEntropyThreads) prog_entropy_kernel(const Header* hd, const uint8_t* files, uint8_t* ws,
                                                                       int* errors, int first) {
    __shared__ Huff tabs[3];
    const uint8_t* blob = reinterpret_cast<const uint8_t*>(hd);
    const PSeg& s = reinterpret_cast<const PSeg*>(blob + hd->pseg_off)[first + blockIdx.x];
    const Scan& sc = reinterpret_cast<const Scan*>(blob + hd->scan_off)[s.scan];
    const Image& im = reinterpret_cast<const Image*>(blob + hd->img_off)[s.img];
    const Huff* pool = reinterpret_cast<const Huff*>(blob + hd->huff_off);
    constexpr int kVec = (int)sizeof(Huff) / 16;
    const int nt = prog_ntabs(sc);
    for (int i = threadIdx.x; i < nt * kVec; i += kEntropyThreads)
        reinterpret_cast<uint4*>(tabs)[i] = reinterpret_cast<const uint4*>(pool + sc.tab[i / kVec])[i % kVec];
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int err = decode_prog_segment(im, sc, s, files, ws, tabs);
    if (err) atomicOr(errors + s.img, err);
}

// The checks yfv2_jpeg_decode makes on a host blob before anything is launched; returns the reason or nullptr
const char* bad_blob(const uint8_t* blob, size_t bytes, size_t files_bytes, size_t frames_bytes, size_t workspace_bytes) {
    if (bytes < sizeof(Header)) return "meta_bytes smaller than the blob header";
    const Header& hd = *reinterpret_cast<const Header*>(blob);
    if (hd.magic != kMagic) return "meta_host is not a blob yfv2_jpeg_parse wrote";
    if ((size_t)hd.bytes != bytes || hd.n < 1 || hd.n > 65535 || hd.nseg < 0 || hd.img_off != align16(sizeof(Header)) ||
        hd.seg_off != align16(hd.img_off + (long long)hd.n * sizeof(Image)) || hd.seg_off + (long long)hd.nseg * (long long)sizeof(Seg) > hd.bytes)
        return "inconsistent blob header (or meta_bytes is not the blob's size)";
    if (hd.npseg == 0) {
        if (hd.nscan || hd.nhuff || hd.nlevel || hd.prog_coef) return "inconsistent blob header (progressive arrays)";
    } else if (hd.nscan < 1 || hd.nhuff < 0 || hd.npseg < 0 || hd.nlevel < 1 || hd.nlevel > kMaxScans ||
               hd.scan_off != align16(hd.seg_off + (long long)hd.nseg * sizeof(Seg)) ||
               hd.huff_off != align16(hd.scan_off + (long long)hd.nscan * sizeof(Scan)) ||
               hd.pseg_off != align16(hd.huff_off + (long long)hd.nhuff * sizeof(Huff)) ||
               hd.lvl_off != align16(hd.pseg_off + (long long)hd.npseg * sizeof(PSeg)) ||
               hd.lvl_off + 4LL * (hd.nlevel + 1) != hd.bytes || hd.prog_coef < 0 || hd.prog_coef > hd.workspace) {
        return "inconsistent blob header (progressive arrays)";
    }
    if ((size_t)hd.files > files_bytes) return "files_bytes smaller than the files the blob was parsed from";
    if ((size_t)hd.frames > frames_bytes) return "frames_bytes smaller than the blob's frames";
    if ((size_t)hd.workspace > workspace_bytes) return "workspace_bytes smaller than the blob needs";
    const Image* ims = reinterpret_cast<const Image*>(blob + hd.img_off);
    const Seg* segs = reinterpret_cast<const Seg*>(blob + hd.seg_off);
    for (int i = 0; i < hd.n; ++i) {
        const Image& im = ims[i];
        if (im.frame < 0 || im.frame + 3LL * im.ow * im.oh > hd.frames) return "a frame outside the arena";
        long long blocks = 0;
        for (int c = 0; c < im.ncomp; ++c) {
            const Comp& cp = im.comp[c];
            const long long nb = (long long)cp.bw * cp.bh;
            if (cp.coef < 0 || cp.plane < 0 || cp.coef + nb * 128 > hd.workspace || cp.plane + nb * 64 > hd.workspace)
                return "a component outside the workspace";
            blocks += nb;
        }
        if (blocks != im.blocks || im.seg0 < 0 || im.seg0 + im.nseg > hd.nseg) return "inconsistent image record";
    }
    for (int k = 0; k < hd.nseg; ++k)
        if (segs[k].img < 0 || segs[k].img >= hd.n || segs[k].begin < 0 || segs[k].begin > segs[k].end || segs[k].end > hd.files)
            return "a segment outside the files";
    if (hd.npseg == 0) return nullptr;
    const Scan* scans = reinterpret_cast<const Scan*>(blob + hd.scan_off);
    const PSeg* ps = reinterpret_cast<const PSeg*>(blob + hd.pseg_off);
    const int* lvl = reinterpret_cast<const int*>(blob + hd.lvl_off);
    if (lvl[0] != 0 || lvl[hd.nlevel] != hd.npseg) return "inconsistent level starts";
    for (int l = 0; l < hd.nlevel; ++l)
        if (lvl[l + 1] < lvl[l]) return "inconsistent level starts";
    for (int k = 0; k < hd.nscan; ++k) {
        const Scan& sc = scans[k];
        if (sc.ncomp < 1 || sc.ncomp > 3 || sc.ss < 0 || sc.se > 63 || sc.ss > sc.se || (sc.ncomp > 1 && sc.ss != 0) || sc.al < 0 ||
            sc.al > 13 || sc.upr < 1 || sc.units < 0)
            return "a bad progressive scan record";
        for (int t = 0; t < prog_ntabs(sc); ++t)
            if (sc.tab[t] < 0 || sc.tab[t] >= hd.nhuff) return "a progressive scan's table outside the pool";
    }
    for (int k = 0; k < hd.npseg; ++k) {
        const PSeg& g = ps[k];
        if (g.img < 0 || g.img >= hd.n || g.scan < 0 || g.scan >= hd.nscan || g.begin < 0 || g.begin > g.end || g.end > hd.files)
            return "a progressive segment outside the files";
        if (g.level < 0 || g.level >= hd.nlevel || k < lvl[g.level] || k >= lvl[g.level + 1]) return "a progressive segment off its level";
        const Image& im = ims[g.img];
        const Scan& sc = scans[g.scan];
        if (g.unit0 < 0 || g.nunit < 0 || (long long)g.unit0 + g.nunit > sc.units) return "a progressive segment outside its scan";
        for (int q = 0; q < sc.ncomp; ++q) {
            if (sc.comp[q] < 0 || sc.comp[q] >= im.ncomp) return "a progressive scan's component outside its image";
            const Comp& cp = im.comp[sc.comp[q]];
            if (cp.coef + (long long)cp.bw * cp.bh * 128 > hd.prog_coef) return "a progressive image's coefficients outside their range";
            const bool fits = sc.ncomp > 1 ? sc.upr == im.mcux && sc.units <= (long long)im.mcux * im.mcuy &&
                                                 cp.bw >= (long long)im.mcux * cp.h && cp.bh >= (long long)im.mcuy * cp.v
                                           : sc.upr <= cp.bw && (sc.units + sc.upr - 1) / sc.upr <= cp.bh;
            if (!fits) return "a progressive scan outside its component's blocks";
        }
    }
    return nullptr;
}

}  // namespace
}  // namespace yfv2

extern "C" int yfv2_jpeg_parse_ex(const uint8_t* files_host, const long long* offsets_host, int N, int flags, yfv2_jpeg_info* info_host,
                                  void* meta_host, size_t meta_cap, size_t* meta_bytes, size_t* workspace_bytes, size_t* frames_bytes) {
    using namespace yfv2;
    using namespace yfv2::jpeg;
    if (!files_host || !offsets_host || !info_host || N < 1 || N > 65535) {
        set_error("jpeg_parse: null files_host / offsets_host / info_host, or N = %d outside 1..65535", N);
        return YFV2_EINVAL;
    }
    if (flags & ~YFV2_JPEG_PROGRESSIVE) {
        set_error("jpeg_parse: flags 0x%x has bits other than YFV2_JPEG_PROGRESSIVE", (unsigned)flags);
        return YFV2_EINVAL;
    }
    for (int i = 0; i < N; ++i)
        if (offsets_host[i] < 0 || offsets_host[i + 1] < offsets_host[i]) {
            set_error("jpeg_parse: offsets_host[%d..%d] = %lld, %lld are not ascending from 0", i, i + 1, offsets_host[i], offsets_host[i + 1]);
            return YFV2_EINVAL;
        }
    std::vector<Image> ims(meta_host ? N : 1);          // without meta_host one scratch record: the tables are still checked
    int rc = YFV2_OK, first_bad = -1;
    long long nseg = 0, frames = 0, blocks = 0, max_blocks = 0, max_pixels = 0;
    long long nscan = 0, nhuff = 0, npseg = 0, prog_blocks = 0;
    int nlevel = 0;
    std::vector<std::vector<Seg>> segs(N);
    std::vector<Scan> scans;                            // every progressive image's, in file order (when meta_host)
    std::vector<Huff> huffs;
    std::vector<PSeg> psegs;
    for (int i = 0; i < N; ++i) {
        yfv2_jpeg_info& inf = info_host[i];
        memset(&inf, 0, sizeof inf);
        Parsed P;
        P.im = &ims[meta_host ? i : 0];
        memset(P.im, 0, sizeof(Image));
        try {
            parse_file(files_host + offsets_host[i], (size_t)(offsets_host[i + 1] - offsets_host[i]), offsets_host[i], P, flags);
        } catch (const Refuse& r) {
            inf.status = r.code;
            snprintf(inf.reason, sizeof inf.reason, "%s", r.why);
            if (first_bad < 0) { first_bad = i; rc = r.code; }
            continue;
        }
        const bool swap = P.orient >= 5;
        inf.w = swap ? P.h : P.w;
        inf.h = swap ? P.w : P.h;
        inf.components = P.ncomp;
        inf.h_samp = P.ncomp == 1 ? 1 : P.hs[0];
        inf.v_samp = P.ncomp == 1 ? 1 : P.vs[0];
        inf.orientation = P.orient;
        inf.restart_interval = P.prog ? P.restart0 : P.restart;
        inf.segments = (int)(P.prog ? P.psegs.size() : P.segs.size());
        inf.scans = P.prog ? (int)P.scans.size() : 1;
        inf.frame_offset = frames;
        const int hm = inf.h_samp, vm = inf.v_samp;
        const long long mcus = (long long)((P.w + 8 * hm - 1) / (8 * hm)) * ((P.h + 8 * vm - 1) / (8 * vm));
        const long long nb = mcus * (hm * vm + (P.ncomp == 3 ? 2 : 0));
        if (meta_host) {
            Image& im = ims[i];
            im.ow = inf.w; im.oh = inf.h;
            im.frame = frames;
            im.seg0 = (int)nseg;
            im.nseg = P.prog ? 0 : inf.segments;
            im.restart = inf.restart_interval;
            im.blocks = nb;
            if (P.prog) {
                for (Scan& sc : P.scans)
                    for (int t = 0; t < prog_ntabs(sc); ++t) sc.tab[t] += (int)huffs.size();
                for (PSeg& g : P.psegs) {
                    g.img = i;
                    g.scan += (int)scans.size();
                }
                scans.insert(scans.end(), P.scans.begin(), P.scans.end());
                huffs.insert(huffs.end(), P.huffs.begin(), P.huffs.end());
                psegs.insert(psegs.end(), P.psegs.begin(), P.psegs.end());
            } else {
                for (Seg& g : P.segs) g.img = i;
                segs[i] = std::move(P.segs);
            }
        }
        if (P.prog) {
            nscan += (long long)P.scans.size();
            nhuff += (long long)P.huffs.size();
            npseg += (long long)P.psegs.size();
            prog_blocks += nb;
            for (const Scan& sc : P.scans) nlevel = sc.level + 1 > nlevel ? sc.level + 1 : nlevel;
        } else {
            nseg += inf.segments;
        }
        blocks += nb;
        max_blocks = nb > max_blocks ? nb : max_blocks;
        max_pixels = (long long)P.w * P.h > max_pixels ? (long long)P.w * P.h : max_pixels;
        frames = align16(frames + 3LL * P.w * P.h);
    }
    if (first_bad >= 0) {
        set_error("jpeg_parse: file %d: %s", first_bad, info_host[first_bad].reason);
        return rc;
    }
    if (nseg > INT_MAX || npseg > INT_MAX || nscan > INT_MAX || nhuff > INT_MAX || max_blocks > INT_MAX) {
        set_error("jpeg_parse: %lld segments / %lld blocks in one image are too many", nseg + npseg, max_blocks);
        return YFV2_EUNSUPPORTED;
    }
    // Header, Image[N], Seg[nseg]; with progressive images also Scan[nscan], Huff[nhuff], PSeg[npseg] and int[nlevel + 1]
    const long long img_off = align16(sizeof(Header));
    const long long seg_off = align16(img_off + (long long)N * sizeof(Image));
    long long bytes = seg_off + nseg * (long long)sizeof(Seg);
    long long scan_off = 0, huff_off = 0, pseg_off = 0, lvl_off = 0;
    if (npseg) {
        scan_off = align16(bytes);
        huff_off = align16(scan_off + nscan * (long long)sizeof(Scan));
        pseg_off = align16(huff_off + nhuff * (long long)sizeof(Huff));
        lvl_off = align16(pseg_off + npseg * (long long)sizeof(PSeg));
        bytes = lvl_off + 4LL * (nlevel + 1);
    }
    const long long ws_bytes = blocks * (128 + 64);
    if (meta_bytes) *meta_bytes = (size_t)bytes;
    if (workspace_bytes) *workspace_bytes = (size_t)ws_bytes;
    if (frames_bytes) *frames_bytes = (size_t)frames;
    if (!meta_host) return YFV2_OK;
    if (meta_cap < (size_t)bytes) {
        set_error("jpeg_parse: meta_cap %zu < %lld bytes needed", meta_cap, bytes);
        return YFV2_ENOMEM;
    }
    uint8_t* blob = static_cast<uint8_t*>(meta_host);
    memset(blob, 0, (size_t)bytes);
    Header& hd = *reinterpret_cast<Header*>(blob);
    hd.magic = kMagic;
    hd.n = N;
    hd.nseg = (int)nseg;
    hd.max_blocks = (int)max_blocks;
    hd.max_pixels = max_pixels;
    hd.img_off = img_off;
    hd.seg_off = seg_off;
    hd.bytes = bytes;
    hd.workspace = ws_bytes;
    hd.frames = frames;
    hd.files = offsets_host[N];
    // The progressive images' coefficient blocks first (one range the decode zeroes), then the others', then all planes
    long long coef[2] = {0, prog_blocks * 128}, plane = blocks * 128;
    Seg* sp = reinterpret_cast<Seg*>(blob + seg_off);
    std::vector<bool> prog(N, false);
    for (const PSeg& g : psegs) prog[g.img] = true;
    for (int i = 0; i < N; ++i) {
        Image& im = ims[i];
        for (int c = 0; c < im.ncomp; ++c) {
            const long long nb = (long long)im.comp[c].bw * im.comp[c].bh;
            im.comp[c].coef = coef[prog[i] ? 0 : 1];
            im.comp[c].plane = plane;
            coef[prog[i] ? 0 : 1] += nb * 128;
            plane += nb * 64;
        }
        for (const Seg& g : segs[i]) *sp++ = g;
    }
    memcpy(blob + img_off, ims.data(), (size_t)N * sizeof(Image));
    if (npseg) {
        hd.nscan = (int)nscan;
        hd.nhuff = (int)nhuff;
        hd.npseg = (int)npseg;
        hd.nlevel = nlevel;
        hd.scan_off = scan_off;
        hd.huff_off = huff_off;
        hd.pseg_off = pseg_off;
        hd.lvl_off = lvl_off;
        hd.prog_coef = prog_blocks * 128;
        std::stable_sort(psegs.begin(), psegs.end(), [](const PSeg& a, const PSeg& b) { return a.level < b.level; });
        int* lvl = reinterpret_cast<int*>(blob + lvl_off);
        for (const PSeg& g : psegs) ++lvl[g.level + 1];
        for (int l = 0; l < nlevel; ++l) lvl[l + 1] += lvl[l];
        memcpy(blob + scan_off, scans.data(), (size_t)nscan * sizeof(Scan));
        memcpy(blob + huff_off, huffs.data(), (size_t)nhuff * sizeof(Huff));
        memcpy(blob + pseg_off, psegs.data(), (size_t)npseg * sizeof(PSeg));
    }
    return YFV2_OK;
}

extern "C" int yfv2_jpeg_parse(const uint8_t* files_host, const long long* offsets_host, int N, yfv2_jpeg_info* info_host,
                               void* meta_host, size_t meta_cap, size_t* meta_bytes, size_t* workspace_bytes, size_t* frames_bytes) {
    return yfv2_jpeg_parse_ex(files_host, offsets_host, N, 0, info_host, meta_host, meta_cap, meta_bytes, workspace_bytes, frames_bytes);
}

extern "C" int yfv2_jpeg_decode(const void* meta_host, const void* meta_dev, size_t meta_bytes, const uint8_t* files, size_t files_bytes,
                                uint8_t* frames, size_t frames_bytes, int* errors, void* workspace, size_t workspace_bytes, int phases,
                                void* stream) {
    using namespace yfv2;
    using namespace yfv2::jpeg;
    if (!meta_host || !meta_dev || !files || !frames || !errors || !workspace) {
        set_error("jpeg_decode: null meta_host / meta_dev / files / frames / errors / workspace");
        return YFV2_EINVAL;
    }
    if (phases < 1 || phases > YFV2_JPEG_ALL) {
        set_error("jpeg_decode: phases %d is not a non-empty mask of YFV2_JPEG_ENTROPY | _IDCT | _COLOR", phases);
        return YFV2_EINVAL;
    }
    const uint8_t* blob = static_cast<const uint8_t*>(meta_host);
    if (const char* why = bad_blob(blob, meta_bytes, files_bytes, frames_bytes, workspace_bytes)) {
        set_error("jpeg_decode: %s", why);
        return YFV2_EINVAL;
    }
    const Header& hd = *reinterpret_cast<const Header*>(blob);
    const Header* dhd = static_cast<const Header*>(meta_dev);
    cudaStream_t s = (cudaStream_t)stream;
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    if (phases & YFV2_JPEG_ENTROPY) {
        YFV2_CUDA(cudaMemsetAsync(errors, 0, sizeof(int) * hd.n, s));
        if (hd.nseg) {
            entropy_kernel<<<hd.nseg, kEntropyThreads, 0, s>>>(dhd, files, ws, errors);
            YFV2_LAUNCH_CHECK();
        }
        if (hd.npseg) {                                  // progressive images: zeroed once, then one launch per level
            YFV2_CUDA(cudaMemsetAsync(ws, 0, (size_t)hd.prog_coef, s));
            const int* lvl = reinterpret_cast<const int*>(blob + hd.lvl_off);
            for (int l = 0; l < hd.nlevel; ++l) {
                if (lvl[l + 1] == lvl[l]) continue;
                prog_entropy_kernel<<<lvl[l + 1] - lvl[l], kEntropyThreads, 0, s>>>(dhd, files, ws, errors, lvl[l]);
                YFV2_LAUNCH_CHECK();
            }
        }
    }
    if (phases & YFV2_JPEG_IDCT) {
        const long long gx = (hd.max_blocks + kIdctThreads - 1) / kIdctThreads;
        idct_kernel<<<dim3((unsigned)(gx < 4096 ? gx : 4096), (unsigned)hd.n), kIdctThreads, 0, s>>>(dhd, ws);
        YFV2_LAUNCH_CHECK();
    }
    if (phases & YFV2_JPEG_COLOR) {
        const long long gx = (hd.max_pixels + kColorThreads - 1) / kColorThreads;
        color_kernel<<<dim3((unsigned)(gx < 8192 ? gx : 8192), (unsigned)hd.n), kColorThreads, 0, s>>>(dhd, ws, frames);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}
