// CPU build of the JPEG encode (tests/test_jpeg_encode_cpu.py compiles it with nvcc): yfv2_jpeg_encode_plan for the headers and
// the geometry, then every block through the same jpeg_enc.cuh functions the device kernels call, one output at a time, and the
// entropy-coded segments written sequentially as jchuff writes them (stuffing, 1-bit padding, RSTn, EOI).
//   jpeg_enc_harness IN W H C OUT [ID VALUE ...]  -> IN holds h*w*C bytes (C = 3: BGR, C = 1: grey); OUT receives the JPEG file;
//   prints "<plan status> <bytes>", or the status and the reason of a refusal.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../yolo-fastestv2_b200/csrc/k_jpeg_enc.cu"

namespace yfv2 {
static char g_err[512];
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace yfv2

using namespace yfv2::jpege;

struct HostPx {
    const uint8_t* img;
    int w, ch;
    void operator()(int x, int y, int (&p)[3]) const {
        const uint8_t* q = img + ((long long)y * w + x) * ch;
        p[0] = q[0];
        p[1] = ch == 3 ? q[1] : q[0];
        p[2] = ch == 3 ? q[2] : q[0];
    }
};

// jchuff's output: bytes with 0xFF stuffed, flushed with 1-bits at every restart and at the end
struct ByteSink {
    std::vector<uint8_t>& out;
    uint64_t acc = 0;
    int n = 0;
    void put(uint32_t code, int size) {
        acc = (acc << size) | code;
        n += size;
        while (n >= 8) {
            const uint8_t b = (uint8_t)(acc >> (n - 8));
            out.push_back(b);
            if (b == 0xFF) out.push_back(0);
            n -= 8;
        }
    }
    void flush() {
        if (n) put((1u << (8 - n)) - 1, 8 - n);
    }
};

int main(int argc, char** argv) {
    if (argc < 6) return 2;
    const int w = atoi(argv[2]), h = atoi(argv[3]), ch = atoi(argv[4]);
    std::vector<uint8_t> img((size_t)w * h * ch);
    FILE* fp = fopen(argv[1], "rb");
    if (!fp || fread(img.data(), 1, img.size(), fp) != img.size()) return 2;
    fclose(fp);
    std::vector<int> params;
    for (int k = 6; k < argc; ++k) params.push_back(atoi(argv[k]));
    yfv2_jpeg_enc_src s;
    memset(&s, 0, sizeof(s));
    s.kind = ch == 3 ? YFV2_JPEG_SRC_BGR : YFV2_JPEG_SRC_GRAY;
    if (ch == 3) s.f.bgr = yfv2_frame{img.data(), w, h, 3LL * w};
    else s.f.strided = yfv2_strided_frame{img.data(), img.data(), img.data(), (long long)w, 1, w, h};
    s.w = w; s.h = h;
    s.params = params.data();
    s.nparams = (int)params.size();
    size_t meta = 0, ws = 0, arena = 0;
    int rc = yfv2_jpeg_encode_plan(&s, 1, nullptr, 0, &meta, &ws, nullptr, &arena);
    if (rc) {
        printf("%d %s\n", rc, yfv2::g_err);
        return 0;
    }
    std::vector<uint8_t> blob(meta);
    if (yfv2_jpeg_encode_plan(&s, 1, blob.data(), blob.size(), &meta, &ws, nullptr, &arena)) return 3;
    const EncHeader& hd = *reinterpret_cast<const EncHeader*>(blob.data());
    const EncImage& im = *reinterpret_cast<const EncImage*>(blob.data() + hd.img_off);
    const HostPx px{img.data(), w, ch};
    std::vector<int16_t> coef(im.nunits * 64);
    for (long long u = 0; u < im.nunits; ++u) {
        const Unit un = unit_of(im.g, u);
        int d[64];
        for (int t = 0; t < 64; ++t) d[t] = comp_sample(px, im.g, un.c, un.src_x * 8 + (t & 7), un.src_y * 8 + (t >> 3)) - 128;
        for (int r = 0; r < 8; ++r) fdct_1d<0>(d + 8 * r, 1);
        for (int c = 0; c < 8; ++c) fdct_1d<1>(d + c, 8);
        for (int t = 0; t < 64; ++t) coef[u * 64 + t] = (int16_t)(un.dummy && t ? 0 : quantize(d[t], im.q[un.c ? 1 : 0], t));
    }
    std::vector<uint8_t> out(blob.data() + im.hdr, blob.data() + im.hdr + im.hdr_len);
    ByteSink bs{out};
    for (long long u = 0; u < im.nunits; ++u) {
        const int mcu = (int)(u / im.g.upm);
        if (u % im.g.upm == 0 && mcu > 0 && segment_start(im.g, mcu)) {
            bs.flush();
            out.push_back(0xFF);
            out.push_back((uint8_t)(0xD0 + ((mcu / im.g.restart - 1) & 7)));
        }
        const long long p = dc_pred_unit(im.g, u);
        const int c = unit_of(im.g, u).c ? 1 : 0;
        encode_block(&coef[u * 64], coef[u * 64] - (p < 0 ? 0 : coef[p * 64]), hd.huff[2 * c], hd.huff[2 * c + 1], bs);
    }
    bs.flush();
    out.push_back(0xFF);
    out.push_back(0xD9);
    FILE* fo = fopen(argv[5], "wb");
    if (!fo) return 2;
    fwrite(out.data(), 1, out.size(), fo);
    fclose(fo);
    printf("0 %zu\n", out.size());
    return 0;
}
