// Evaluation bookkeeping on the device: get_batch_statistics (reference utils/utils.py:184-230), the per-image greedy
// marking of NMS output rows as true positives.  The reference walks every predicted box in a Python loop and calls
// bbox_iou once per box (SURVEY 8f.2: after NMS moved to the GPU this loop is the evaluation bottleneck); here one warp
// owns an image and keeps the same sequential semantics:
//   for each prediction in (descending-confidence) order, stop once every annotation of the image has been matched;
//   skip it if its label is not among the image's target labels; otherwise take the annotation with the largest IoU
//   (ALL annotations of the image compete, whatever their label; first maximum wins, and a NaN IoU is the maximum as in
//   torch's max(0)) and mark the prediction a true positive iff that IoU >= threshold and that annotation has not been
//   claimed before.
// IoU is the reference's bbox_iou (utils/utils.py:76-108, the +1 pixel convention) evaluated with the same sequence of
// individually rounded fp32 operations, so the flags are bit-identical to the reference's.
#include "common.cuh"

namespace yfv2 {
namespace {

constexpr int kEvalWarps = 4;                   // images per CTA
constexpr int kNoTarget = 0x7fffffff;

__device__ __forceinline__ float ref_iou(float ax1, float ay1, float ax2, float ay2, float bx1, float by1, float bx2, float by2) {
    const float ix1 = fmaxf(ax1, bx1), iy1 = fmaxf(ay1, by1), ix2 = fminf(ax2, bx2), iy2 = fminf(ay2, by2);
    const float iw = fmaxf(__fadd_rn(__fsub_rn(ix2, ix1), 1.0f), 0.0f);
    const float ih = fmaxf(__fadd_rn(__fsub_rn(iy2, iy1), 1.0f), 0.0f);
    const float inter = __fmul_rn(iw, ih);
    const float a1 = __fmul_rn(__fadd_rn(__fsub_rn(ax2, ax1), 1.0f), __fadd_rn(__fsub_rn(ay2, ay1), 1.0f));
    const float a2 = __fmul_rn(__fadd_rn(__fsub_rn(bx2, bx1), 1.0f), __fadd_rn(__fsub_rn(by2, by1), 1.0f));
    const float den = __fadd_rn(__fsub_rn(__fadd_rn(a1, a2), inter), 1e-16f);
    return __fdiv_rn(inter, den);
}

// torch's max(0) order on (IoU, annotation index): NaN above every number, then the larger value, then the smaller index.
// (fmaxf / fminf in ref_iou drop a NaN operand where torch.max / torch.min keep it, but a NaN coordinate also makes an area
// and so the IoU NaN: the result is the same.)  kNoTarget marks a lane that saw no annotation of the image.
__device__ __forceinline__ bool iou_before(float v, int i, float best, int besti) {
    if (i == kNoTarget) return false;
    if (besti == kNoTarget) return true;
    const bool vn = isnan(v), bn = isnan(best);
    if (vn || bn) return vn && (!bn || i < besti);
    return v > best || (v == best && i < besti);
}

// dets [N,max_det,6], counts [N]; targets [nt,6] = (image, class, x1, y1, x2, y2) in pixels; tp [N,max_det] (0 / 1).
// Dynamic shared memory: per warp the annotation index of each true positive so far (at most max_det of them).
__global__ void __launch_bounds__(32 * kEvalWarps)
batch_stats_kernel(const float* __restrict__ dets, const int* __restrict__ counts, int N, int max_det,
                   const float* __restrict__ targets, int nt, float thr, float* __restrict__ tp) {
    extern __shared__ int claimed_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int img = blockIdx.x * kEvalWarps + warp;
    if (img >= N) return;
    int* cl = claimed_all + (size_t)warp * max_det;
    int n_ann = 0;
    for (int t0 = 0; t0 < nt; t0 += 32) {
        const int t = t0 + lane;
        n_ann += __popc(__ballot_sync(0xffffffffu, t < nt && targets[(size_t)t * 6] == (float)img));
    }
    const int cnt = min(counts[img], max_det);
    float* tpo = tp + (size_t)img * max_det;
    for (int i = lane; i < max_det; i += 32) tpo[i] = 0.f;
    __syncwarp();
    int n_det = 0;
    for (int pi = 0; pi < cnt && n_det < n_ann; ++pi) {
        const float* d = dets + ((size_t)img * max_det + pi) * 6;
        const float px1 = d[0], py1 = d[1], px2 = d[2], py2 = d[3], plabel = d[5];
        float best = -INFINITY;
        int besti = kNoTarget;
        bool label_seen = false;
        for (int t0 = 0; t0 < nt; t0 += 32) {
            const int t = t0 + lane;
            if (t < nt) {
                const float* a = targets + (size_t)t * 6;
                if (a[0] == (float)img) {
                    label_seen |= (a[1] == plabel);
                    const float v = ref_iou(px1, py1, px2, py2, a[2], a[3], a[4], a[5]);
                    if (iou_before(v, t, best, besti)) { best = v; besti = t; }
                }
            }
        }
        label_seen = __any_sync(0xffffffffu, label_seen);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (iou_before(ob, oi, best, besti)) { best = ob; besti = oi; }
        }
        if (!label_seen || !(best >= thr)) continue;
        bool taken = false;
        for (int k = lane; k < n_det; k += 32) taken |= cl[k] == besti;
        if (__any_sync(0xffffffffu, taken)) continue;
        if (lane == 0) { tpo[pi] = 1.f; cl[n_det] = besti; }
        __syncwarp();
        ++n_det;
    }
}

}  // namespace
}  // namespace yfv2

extern "C" int yfv2_batch_statistics(const float* dets, const int* counts, int N, int max_det, const float* targets, int nt,
                                     float iou_threshold, float* tp, void* stream) {
    using namespace yfv2;
    if (!dets || !counts || !tp || N <= 0 || max_det <= 0 || nt < 0 || (nt > 0 && !targets)) { set_error("batch_statistics: bad argument"); return YFV2_EINVAL; }
    if (max_det > YFV2_EVAL_MAX_DET) { set_error("batch_statistics: %d rows per image (limit %d)", max_det, YFV2_EVAL_MAX_DET); return YFV2_EUNSUPPORTED; }
    const size_t bytes = (size_t)kEvalWarps * max_det * sizeof(int);
    if (bytes > 48 * 1024) YFV2_CUDA(cudaFuncSetAttribute(batch_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    batch_stats_kernel<<<(N + kEvalWarps - 1) / kEvalWarps, 32 * kEvalWarps, bytes, (cudaStream_t)stream>>>(dets, counts, N, max_det,
                                                                                                         targets, nt, iou_threshold, tp);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
