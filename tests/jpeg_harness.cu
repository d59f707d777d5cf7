// CPU build of the JPEG decode (tests/test_jpeg_cpu.py compiles it with nvcc): yfv2_jpeg_parse, then the three phases through the
// same jpeg.cuh functions the device kernels call, one file at a time.
//   jpeg_harness IN OUT [IN OUT ...]  -> one line per file: "<parse status> <w> <h> <error flags>"; OUT receives the BGR bytes.
// Each file is read into a buffer of exactly its size, and the parser (k_jpeg.cu) is compiled into this program rather than taken
// from libyfv2.so, so an address-sanitised build sees any read past a file's end, by the parse or by the decode.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../yolo-fastestv2_b200/csrc/k_jpeg.cu"

namespace yfv2 {
void set_error(const char*, ...) {}   // the library keeps the message for yfv2_last_error; the harness prints info.reason
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
    int rc = yfv2_jpeg_parse(file, off, 1, &info, nullptr, 0, &meta, &ws_bytes, &frames_bytes);
    if (rc != 0) {
        printf("%d 0 0 0 %s\n", rc, info.reason);
        free(file);
        return 0;
    }
    std::vector<uint8_t> blob(meta), ws(ws_bytes), frames(frames_bytes);
    rc = yfv2_jpeg_parse(file, off, 1, &info, blob.data(), blob.size(), &meta, &ws_bytes, &frames_bytes);
    if (rc != 0) return 3;
    const Header& hd = *reinterpret_cast<const Header*>(blob.data());
    const Image& im = *reinterpret_cast<const Image*>(blob.data() + hd.img_off);
    const Seg* segs = reinterpret_cast<const Seg*>(blob.data() + hd.seg_off);
    int err = 0;
    for (int s = 0; s < hd.nseg; ++s) err |= decode_segment(im, segs[s], file, ws.data(), im.dc, im.ac);
    for (long long k = 0; k < im.blocks; ++k) idct_block(im, k, ws.data());
    for (int y = 0; y < im.oh; ++y)
        for (int x = 0; x < im.ow; ++x) bgr_pixel(im, ws.data(), x, y, frames.data() + im.frame + 3LL * ((long long)y * im.ow + x));
    FILE* fo = fopen(out, "wb");
    if (!fo) return 2;
    fwrite(frames.data() + im.frame, 1, 3LL * im.ow * im.oh, fo);
    fclose(fo);
    printf("0 %d %d %d\n", im.ow, im.oh, err);
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
