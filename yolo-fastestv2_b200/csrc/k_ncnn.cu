// Deploy-path post-process (SURVEY 8f.4): the decode + per-class greedy NMS that the reference's ncnn sample runs on the
// export_onnx head tensors, on the device, bit for bit.
//
//   getCategory        <- reference sample/ncnn/src/yolo-fastestv2.cpp:113-131  first strict maximum of cls*obj above 0
//   predHandle         <- :134-183  ((v*2 - 0.5) + cell) * stride and (v*2)^2 * anchor in DOUBLE, rounded to float, box corners
//                         (c -/+ 0.5 w) * scale in double, TRUNCATED to int (TargetBox has int coordinates, include/yolo-fastestv2.h:16-19)
//                         by yfv2_ncnn_corner (include/yfv2.h): INT_MIN for NaN and out-of-range values, as x86-64's cvttsd2si
//   intersection_area  <- :58-71    on the int corners
//   nmsHandle          <- :78-110   descending score, greedy, a box is dropped iff IoU > thr with an earlier kept box OF ITS CLASS
//
// Input: the two [N,h,w,5A+C] tensors yfv2_export_heads writes (sigmoid reg | sigmoid obj | softmax cls, model/detector.py:33-44).
// One CTA per image.  Candidates are scored a warp per cell (coalesced reads of the cell's 5A+C floats, shuffle arg-max with the
// smaller class winning ties = the reference's strict '>' scan), keyed (score, push order) and sorted by nms.cuh's bitonic networks,
// then suppressed by its greedy_pass in blocks of 64 sorted candidates: block vs everything kept so far, 64x64 pairs inside the
// block, an in-order resolve over bit masks.  Every floating-point step is the reference's operation with round-to-nearest
// intrinsics (no contraction).
// The reference sorts with std::sort (order among equal scores unspecified); ties here keep push order (level, row, column, anchor).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "nms.cuh"

namespace yfv2 {
namespace {

struct NcnnArgs {
    const float* out[2];
    int h[2], w[2];
    int stride[2];
    int A, C, ch;
    int M, MCp;
    float anchors[2][kMaxA][2];
    float thresh, nms_thresh, scale_w, scale_h;
    int max_out;
    int* boxes; float* scores; int* cates; int* counts;
};

struct Smem {
    unsigned long long* keys;   // [MCp]  (sortable score << 32) | (0xFFFF - push order) << 16 | slot
    int4* box;                  // [M]
    float* area;                // [M]
    short* cate;                // [M]
    unsigned short* picked;     // [M] slots of kept boxes, in kept order
    int4* chbox;                // [64]
    float* charea;              // [64]
    short* chcate;              // [64]
    unsigned int* cmask;        // [64][2]
    unsigned int* misc;         // [0] candidate count, [1..2] dead bits, [3..4] kept bits
};

// The shared memory of one CTA, laid out from `base` (16-byte aligned).  Returns the end of the layout.
__host__ __device__ __forceinline__ unsigned char* ncnn_layout(Smem& s, unsigned char* base, int M, int MCp) {
    s.keys = take<unsigned long long>(base, MCp);
    s.box = take<int4>(base, M);
    s.area = take<float>(base, M);
    s.cate = take<short>(base, M);
    s.picked = take<unsigned short>(base, M);
    s.chbox = take<int4>(base, kChunk);
    s.charea = take<float>(base, kChunk);
    s.chcate = take<short>(base, kChunk);
    s.cmask = take<unsigned int>(base, 2 * kChunk);
    s.misc = take<unsigned int>(base, 8);
    return base;
}

// IoU of two int boxes exactly as nmsHandle computes it (:91-96): float(inter) / (area_a + area_b - float(inter)) > thr
__device__ __forceinline__ bool iou_gt(const int4& a, float aa, const int4& b, float ab, float thr) {
    float ia = 0.f;
    if (!(a.x > b.z || a.z < b.x || a.y > b.w || a.w < b.y))
        ia = __fmul_rn((float)(min(a.z, b.z) - max(a.x, b.x)), (float)(min(a.w, b.w) - max(a.y, b.y)));
    const float ua = __fsub_rn(__fadd_rn(aa, ab), ia);
    return __fdiv_rn(ia, ua) > thr;
}

// nmsHandle's side of greedy_pass: a box suppresses only boxes of its category, and every kept box is recorded, the first max_out
// of them in the outputs.
struct NcnnPass {
    const NcnnArgs& p;
    const Smem& s;
    int* oboxes;
    float* oscores;
    int* ocates;

    __device__ __forceinline__ void stage(int j, unsigned long long key) const {
        const unsigned int slot = (unsigned int)(key & 0xFFFFull);
        s.chbox[j] = s.box[slot]; s.charea[j] = s.area[slot]; s.chcate[j] = s.cate[slot];
    }
    struct Cand {
        int4 box;
        float area;
        short cate;
    };
    __device__ __forceinline__ Cand cand(int j) const { return {s.chbox[j], s.charea[j], s.chcate[j]}; }
    __device__ __forceinline__ bool kept_other_source(int, const Cand&) const { return true; }
    __device__ __forceinline__ bool kept_same_class(int i, const Cand& c) const { return s.cate[s.picked[i]] == c.cate; }
    __device__ __forceinline__ bool kept_kills(int i, const Cand& c) const {
        const unsigned int ks = s.picked[i];
        return iou_gt(c.box, c.area, s.box[ks], s.area[ks], p.nms_thresh);
    }
    __device__ __forceinline__ bool other_source(const Cand&, int) const { return true; }
    __device__ __forceinline__ bool same_class(const Cand& c, int j) const { return s.chcate[j] == c.cate; }
    __device__ __forceinline__ bool kills(const Cand& c, int j) const {
        return iou_gt(s.chbox[j], s.charea[j], c.box, c.area, p.nms_thresh);
    }
    __device__ __forceinline__ void append(int pos, int j, const unsigned long long& key) const {
        s.picked[pos] = (unsigned short)(key & 0xFFFFull);
        if (pos < p.max_out) {
            const int4 b = s.chbox[j];
            oboxes[4 * pos] = b.x; oboxes[4 * pos + 1] = b.y; oboxes[4 * pos + 2] = b.z; oboxes[4 * pos + 3] = b.w;
            oscores[pos] = sortable2f((unsigned int)(key >> 32));
            ocates[pos] = (int)s.chcate[j];
        }
    }
};

__global__ void __launch_bounds__(NT)
ncnn_post_kernel(const NcnnArgs p) {
    extern __shared__ __align__(16) unsigned char smraw[];
    Smem s;
    ncnn_layout(s, smraw, p.M, p.MCp);
    const int n = blockIdx.x, t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    if (t == 0) s.misc[0] = 0u;
    __syncthreads();
    const int A = p.A, C = p.C;
    // ---- candidates (predHandle): one warp per cell --------------------------------------------------------------
    int row0 = 0;
    for (int lv = 0; lv < 2; ++lv) {
        const int hw = p.h[lv] * p.w[lv];
        const float* base = p.out[lv] + (long long)n * hw * p.ch;
        for (int cell = warp; cell < hw; cell += NT / 32) {
            const float* v = base + (long long)cell * p.ch;
            const int y = cell / p.w[lv], x = cell - y * p.w[lv];
            for (int b = 0; b < A; ++b) {
                const float obj = __ldg(v + 4 * A + b);
                float best = 0.f;                                 // getCategory: tmp = 0, strict '>' (:115-127)
                int bi = 0x7fffffff;
                for (int k = lane; k < C; k += 32) {
                    const float cs = __fmul_rn(__ldg(v + 5 * A + k), obj);
                    if (cs > best) { best = cs; bi = k; }
                }
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
                }
                const float score = bi == 0x7fffffff ? -1.f : best;             // nothing above 0: score = -1, category = -1 (:156-157)
                const int cate = bi == 0x7fffffff ? -1 : bi;
                if (lane == 0 && score > p.thresh) {                              // :161
                    const double st = (double)p.stride[lv];
                    const float bcx = (float)__dmul_rn(__dadd_rn(__dsub_rn(__dmul_rn((double)__ldg(v + b * 4 + 0), 2.0), 0.5), (double)x), st);
                    const float bcy = (float)__dmul_rn(__dadd_rn(__dsub_rn(__dmul_rn((double)__ldg(v + b * 4 + 1), 2.0), 0.5), (double)y), st);
                    const double tw = __dmul_rn((double)__ldg(v + b * 4 + 2), 2.0), th = __dmul_rn((double)__ldg(v + b * 4 + 3), 2.0);
                    const float bw = (float)__dmul_rn(__dmul_rn(tw, tw), (double)p.anchors[lv][b][0]);      // pow(x, 2) == x*x exactly
                    const float bh = (float)__dmul_rn(__dmul_rn(th, th), (double)p.anchors[lv][b][1]);
                    const double hx = __dmul_rn(0.5, (double)bw), hy = __dmul_rn(0.5, (double)bh);
                    int4 bb;                                          // :170-173, double -> int: truncates, INT_MIN for NaN / out of range
                    bb.x = yfv2_ncnn_corner(__dmul_rn(__dsub_rn((double)bcx, hx), (double)p.scale_w));
                    bb.y = yfv2_ncnn_corner(__dmul_rn(__dsub_rn((double)bcy, hy), (double)p.scale_h));
                    bb.z = yfv2_ncnn_corner(__dmul_rn(__dadd_rn((double)bcx, hx), (double)p.scale_w));
                    bb.w = yfv2_ncnn_corner(__dmul_rn(__dadd_rn((double)bcy, hy), (double)p.scale_h));
                    const unsigned int slot = atomicAdd(&s.misc[0], 1u);
                    s.box[slot] = bb;
                    s.area[slot] = __fmul_rn((float)(bb.z - bb.x), (float)(bb.w - bb.y));                     // TargetBox::area()
                    s.cate[slot] = (short)cate;
                    const unsigned int order = (unsigned int)(row0 + cell * A + b);
                    s.keys[slot] = ((unsigned long long)f2sortable(score) << 32) | ((unsigned long long)(0xFFFFu - order) << 16) | slot;
                }
            }
        }
        row0 += hw * A;
    }
    __syncthreads();
    const int cnt = (int)s.misc[0];
    sort_keys_desc(s.keys, cnt);                                             // nmsHandle :84

    // ---- greedy per-class suppression (:86-103), 64 sorted candidates at a time; counts[n] reports every kept box ----------
    int* oboxes = p.boxes + (long long)n * p.max_out * 4;
    float* oscores = p.scores + (long long)n * p.max_out;
    int* ocates = p.cates + (long long)n * p.max_out;
    const int np = greedy_pass(s.keys, cnt, cnt, s.cmask, s.misc + 1, NcnnPass{p, s, oboxes, oscores, ocates});
    if (t == 0) p.counts[n] = np;
    for (int i = min(np, p.max_out) + t; i < p.max_out; i += NT) {
        oboxes[4 * i] = 0; oboxes[4 * i + 1] = 0; oboxes[4 * i + 2] = 0; oboxes[4 * i + 3] = 0;
        oscores[i] = 0.f; ocates[i] = -1;
    }
}

}  // namespace
}  // namespace yfv2

using namespace yfv2;

extern "C" int yfv2_ncnn_post(const float* out2, const float* out3, int N, int H, int W, int A, int C, const float* anchors_host,
                              float thresh, float nms_thresh, float scale_w, float scale_h, int max_out, int* boxes, float* scores,
                              int* cates, int* counts, void* stream) {
    if (!out2 || !out3 || !anchors_host || !boxes || !scores || !cates || !counts || N <= 0 || A <= 0 || A > kMaxA || C <= 0 || C > 32767 ||
        H <= 0 || W <= 0 || H % 32 || W % 32 || max_out <= 0) {
        set_error("ncnn_post: bad arguments (N=%d H=%d W=%d A=%d C=%d max_out=%d; need A<=%d, H,W multiples of 32)", N, H, W, A, C, max_out, kMaxA);
        return YFV2_EINVAL;
    }
    NcnnArgs p{};
    p.out[0] = out2; p.out[1] = out3;
    for (int lv = 0; lv < 2; ++lv) {
        const int s = lv ? 32 : 16;
        p.h[lv] = H / s; p.w[lv] = W / s;
        p.stride[lv] = H / p.h[lv];                       // predHandle :146-147 (inputHeight / outH)
        for (int a = 0; a < A; ++a) { p.anchors[lv][a][0] = anchors_host[(lv * A + a) * 2]; p.anchors[lv][a][1] = anchors_host[(lv * A + a) * 2 + 1]; }
    }
    p.A = A; p.C = C; p.ch = 5 * A + C;
    p.M = A * (p.h[0] * p.w[0] + p.h[1] * p.w[1]);
    p.MCp = pow2_at_least(p.M);
    p.thresh = thresh; p.nms_thresh = nms_thresh; p.scale_w = scale_w; p.scale_h = scale_h;
    p.max_out = max_out; p.boxes = boxes; p.scores = scores; p.cates = cates; p.counts = counts;
    Smem s;
    const size_t bytes = reinterpret_cast<size_t>(ncnn_layout(s, nullptr, p.M, p.MCp));
    if (p.M > 0xFFFF || bytes > kSmemCap) { set_error("ncnn_post: %d candidates per image need %zu bytes of shared memory", p.M, bytes); return YFV2_EUNSUPPORTED; }
    YFV2_CUDA(cudaFuncSetAttribute(ncnn_post_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    ncnn_post_kernel<<<N, NT, bytes, (cudaStream_t)stream>>>(p);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
