/* Plain-C restatement of the reference per-image NMS (test infrastructure, see oracle/__init__.py).
 *
 *   utils/utils.py:232-296  non_max_suppression  (filter, conf=obj*cls, argmax, class offset, cap 300)
 *   utils/utils.py:67-74    xywh2xyxy
 *   torchvision.ops.nms     greedy kernel (third-party; restated from its documented behaviour and
 *                           pinned against the installed torchvision 0.26.0 by the CPU tests):
 *                           stable descending sort, IoU = inter/(a+b-inter) in fp32 without +1,
 *                           suppress iff (double)iou > iou_threshold.
 *
 * Build with -ffp-contract=off: the fp32 products must not be fused into the following add/sub.
 */
#include <stdlib.h>
#include <string.h>

typedef struct { float score; int idx; } sitem;

static int cmp_desc_stable(const void *a, const void *b) {
    const sitem *x = (const sitem *)a, *y = (const sitem *)b;
    if (x->score > y->score) return -1;
    if (x->score < y->score) return 1;
    return (x->idx > y->idx) - (x->idx < y->idx);   /* ties: lower original index first */
}

/* x: [M, 5+C] row-major fp32.  out: [max_det,6], src_idx: [max_det].  max_wh: the class offset of utils.py:283 (the
 * reference's value is 4096).  Returns kept count. */
int oracle_nms_image(const float *x, int M, int C, float conf_thres, double iou_thres,
                     const int *classes, int n_classes, int max_det, float max_wh, float *out, int *src_idx) {
    const int D = 5 + C;
    float *box = (float *)malloc(sizeof(float) * 4 * (size_t)(M > 0 ? M : 1));
    float *obox = (float *)malloc(sizeof(float) * 4 * (size_t)(M > 0 ? M : 1));
    float *area = (float *)malloc(sizeof(float) * (size_t)(M > 0 ? M : 1));
    float *conf = (float *)malloc(sizeof(float) * (size_t)(M > 0 ? M : 1));
    int *cls = (int *)malloc(sizeof(int) * (size_t)(M > 0 ? M : 1));
    int *src = (int *)malloc(sizeof(int) * (size_t)(M > 0 ? M : 1));
    sitem *ord = (sitem *)malloc(sizeof(sitem) * (size_t)(M > 0 ? M : 1));
    unsigned char *dead = (unsigned char *)calloc((size_t)(M > 0 ? M : 1), 1);
    int n = 0, kept = 0;
    if (!box || !obox || !area || !conf || !cls || !src || !ord || !dead) { kept = -1; goto done; }

    for (int r = 0; r < M; ++r) {
        const float *row = x + (size_t)r * D;
        const float obj = row[4];
        if (!(obj > conf_thres)) continue;                    /* utils.py:254 */
        float best = row[5] * obj; int bj = 0;                /* utils.py:261,267 (first max) */
        for (int c = 1; c < C; ++c) {
            const float p = row[5 + c] * obj;
            if (p > best) { best = p; bj = c; }
        }
        if (!(best > conf_thres)) continue;                   /* utils.py:268 */
        if (classes) {                                        /* utils.py:271-272 */
            int ok = 0;
            for (int k = 0; k < n_classes; ++k) ok |= (classes[k] == bj);
            if (!ok) continue;
        }
        const float hw = row[2] / 2.0f, hh = row[3] / 2.0f;   /* utils.py:67-74 */
        box[4 * n + 0] = row[0] - hw; box[4 * n + 1] = row[1] - hh;
        box[4 * n + 2] = row[0] + hw; box[4 * n + 3] = row[1] + hh;
        conf[n] = best; cls[n] = bj; src[n] = r; ++n;
    }
    /* n > max_nms (30000) top-k branch (utils.py:278-280) cannot trigger for M <= 30000 */
    for (int i = 0; i < n; ++i) {
        const float off = (float)cls[i] * max_wh;             /* utils.py:283-285 */
        for (int k = 0; k < 4; ++k) obox[4 * i + k] = box[4 * i + k] + off;
        area[i] = (obox[4 * i + 2] - obox[4 * i + 0]) * (obox[4 * i + 3] - obox[4 * i + 1]);
        ord[i].score = conf[i]; ord[i].idx = i;
    }
    qsort(ord, (size_t)n, sizeof(sitem), cmp_desc_stable);
    for (int a = 0; a < n && kept < max_det; ++a) {           /* cap: i[:max_det], utils.py:287-288 */
        const int i = ord[a].idx;
        if (dead[i]) continue;
        memcpy(out + 6 * kept, box + 4 * i, 4 * sizeof(float));
        out[6 * kept + 4] = conf[i]; out[6 * kept + 5] = (float)cls[i];
        src_idx[kept] = src[i]; ++kept;
        const float ix1 = obox[4 * i], iy1 = obox[4 * i + 1], ix2 = obox[4 * i + 2], iy2 = obox[4 * i + 3];
        const float ia = area[i];
        for (int b = a + 1; b < n; ++b) {
            const int j = ord[b].idx;
            if (dead[j]) continue;
            const float xx1 = ix1 > obox[4 * j] ? ix1 : obox[4 * j];
            const float yy1 = iy1 > obox[4 * j + 1] ? iy1 : obox[4 * j + 1];
            const float xx2 = ix2 < obox[4 * j + 2] ? ix2 : obox[4 * j + 2];
            const float yy2 = iy2 < obox[4 * j + 3] ? iy2 : obox[4 * j + 3];
            float w = xx2 - xx1, h = yy2 - yy1;
            w = w > 0.0f ? w : 0.0f; h = h > 0.0f ? h : 0.0f;
            const float inter = w * h;
            const float ovr = inter / (ia + area[j] - inter);
            if ((double)ovr > iou_thres) dead[j] = 1;
        }
    }
done:
    free(box); free(obox); free(area); free(conf); free(cls); free(src); free(ord); free(dead);
    return kept;
}
