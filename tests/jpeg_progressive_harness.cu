// CPU build of the JPEG decode with progressive files accepted (tests/test_jpeg_progressive_cpu.py compiles it with nvcc):
// yfv2_jpeg_parse_ex(YFV2_JPEG_PROGRESSIVE), then the phases through the same jpeg.cuh functions the device kernels call, one file
// at a time: a baseline file's segments, or a progressive file's zeroed coefficients and its segments level by level, each with
// its scan's tables copied out of the pool as the kernel stages them.
//   jpeg_progressive_harness IN OUT [IN OUT ...]
//     -> one line per file: "<parse status> <w> <h> <error flags> <scans> <levels>"; OUT receives the BGR bytes.
// Each file is read into a buffer of exactly its size and the parser is compiled in, so an address-sanitised build sees any read
// past a file's end, by the parse or by the decode.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../yolo-fastestv2_b200/csrc/k_jpeg.cu"

namespace yfv2 {
void set_error(const char*, ...) {}
}  // namespace yfv2

using namespace yfv2::jpeg;

static int decode_file(const char* in, const char* out) {
    FILE* fp = fopen(in, "rb");
    if (!fp) return 2;
    fseek(fp, 0, SEEK_END);
    const long size = ftell(fp);
    fseek(fp, 0, SEEK_SET);
    uint8_t* file = static_cast<uint8_t*>(malloc(size > 0 ? size : 1));
    if (fread(file, 1, size, fp) != (size_t)size) return 2;
    fclose(fp);
    const long long off[2] = {0, size};
    yfv2_jpeg_info info;
    size_t meta = 0, ws_bytes = 0, frames_bytes = 0;
    int rc = yfv2_jpeg_parse_ex(file, off, 1, YFV2_JPEG_PROGRESSIVE, &info, nullptr, 0, &meta, &ws_bytes, &frames_bytes);
    if (rc != 0) {
        printf("%d 0 0 0 0 0 %s\n", rc, info.reason);
        free(file);
        return 0;
    }
    std::vector<uint8_t> blob(meta), ws(ws_bytes, 0x5A), frames(frames_bytes);   // the workspace starts dirty, as on the device
    rc = yfv2_jpeg_parse_ex(file, off, 1, YFV2_JPEG_PROGRESSIVE, &info, blob.data(), blob.size(), &meta, &ws_bytes, &frames_bytes);
    if (rc != 0) return 3;
    if (yfv2::bad_blob(blob.data(), blob.size(), (size_t)size, frames.size(), ws.size())) return 4;
    const Header& hd = *reinterpret_cast<const Header*>(blob.data());
    const Image& im = *reinterpret_cast<const Image*>(blob.data() + hd.img_off);
    const Seg* segs = reinterpret_cast<const Seg*>(blob.data() + hd.seg_off);
    int err = 0;
    for (int s = 0; s < hd.nseg; ++s) err |= decode_segment(im, segs[s], file, ws.data(), im.dc, im.ac);
    if (hd.npseg) {
        memset(ws.data(), 0, (size_t)hd.prog_coef);
        const Scan* scans = reinterpret_cast<const Scan*>(blob.data() + hd.scan_off);
        const Huff* pool = reinterpret_cast<const Huff*>(blob.data() + hd.huff_off);
        const PSeg* ps = reinterpret_cast<const PSeg*>(blob.data() + hd.pseg_off);
        const int* lvl = reinterpret_cast<const int*>(blob.data() + hd.lvl_off);
        std::vector<Huff> tabs(3);
        for (int l = 0; l < hd.nlevel; ++l)
            for (int k = lvl[l]; k < lvl[l + 1]; ++k) {
                const Scan& sc = scans[ps[k].scan];
                for (int t = 0; t < prog_ntabs(sc); ++t) tabs[t] = pool[sc.tab[t]];
                err |= decode_prog_segment(im, sc, ps[k], file, ws.data(), tabs.data());
            }
    }
    for (long long k = 0; k < im.blocks; ++k) idct_block(im, k, ws.data());
    for (int y = 0; y < im.oh; ++y)
        for (int x = 0; x < im.ow; ++x) bgr_pixel(im, ws.data(), x, y, frames.data() + im.frame + 3LL * ((long long)y * im.ow + x));
    FILE* fo = fopen(out, "wb");
    if (!fo) return 2;
    fwrite(frames.data() + im.frame, 1, 3LL * im.ow * im.oh, fo);
    fclose(fo);
    printf("0 %d %d %d %d %d\n", im.ow, im.oh, err, info.scans, hd.nlevel);
    free(file);
    return 0;
}

int main(int argc, char** argv) {
    for (int i = 1; i + 1 < argc; i += 2) {
        const int rc = decode_file(argv[i], argv[i + 1]);
        if (rc) {
            fprintf(stderr, "%s: harness error %d\n", argv[i], rc);
            return rc;
        }
    }
    return 0;
}
