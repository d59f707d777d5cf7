/* Plain-C restatement of the reference's DEPLOY post-process (test infrastructure, see oracle/__init__.py):
 * the decode + per-class greedy NMS that the ncnn sample runs on the export_onnx head tensors.
 *
 *   sample/ncnn/src/yolo-fastestv2.cpp:113-131   getCategory   first strict maximum of cls*obj above 0
 *   sample/ncnn/src/yolo-fastestv2.cpp:134-183   predHandle    grid decode in double, boxes truncated to int
 *   sample/ncnn/src/yolo-fastestv2.cpp:58-76     intersection_area (int coordinates)
 *   sample/ncnn/src/yolo-fastestv2.cpp:78-110    nmsHandle     sort by score, greedy, suppress iff IoU > thr and same class
 *   sample/ncnn/src/include/yolo-fastestv2.h:9-25 TargetBox    int x1,y1,x2,y2; area() = float(x2-x1) * float(y2-y1)
 *
 * Pinned: tests/golden/ncnn_post.npz holds outputs of the reference's own C++ (compiled in place by `make ref`, stub ncnn /
 * OpenCV headers in oracle/ncnn_shim/) and tests/test_ncnn_post_cpu.py checks this restatement against them bit for bit.
 * One stated difference: the reference orders candidates with std::sort, whose order among EQUAL scores is unspecified; here
 * ties keep push order (level, row, column, anchor), which libstdc++'s sort also gives while at most 16 candidates pass.
 * Box corners go through yfv2_ncnn_corner (include/yfv2.h), the sample's `int = double` as compiled for x86-64 (INT_MIN for NaN
 * and out-of-range values), so this restatement gives the same corners on every host; int differences of corners wrap.
 *
 * Build with -ffp-contract=off -fwrapv.
 */
#include <math.h>
#include <stdlib.h>

#include "yfv2.h"

typedef struct { int x1, y1, x2, y2, cate; float score; int order; } tbox;

static float tb_area(const tbox *b) { return (float)(b->x2 - b->x1) * (float)(b->y2 - b->y1); }           /* .h:12-24 */

static float inter_area(const tbox *a, const tbox *b) {                                                     /* .cpp:58-71 */
    if (a->x1 > b->x2 || a->x2 < b->x1 || a->y1 > b->y2 || a->y2 < b->y1) return 0.f;
    float iw = (float)((a->x2 < b->x2 ? a->x2 : b->x2) - (a->x1 > b->x1 ? a->x1 : b->x1));
    float ih = (float)((a->y2 < b->y2 ? a->y2 : b->y2) - (a->y1 > b->y1 ? a->y1 : b->y1));
    return iw * ih;
}

static int cmp_score_desc(const void *pa, const void *pb) {
    const tbox *a = (const tbox *)pa, *b = (const tbox *)pb;
    if (a->score > b->score) return -1;
    if (a->score < b->score) return 1;
    return (a->order > b->order) - (a->order < b->order);
}

/* outs[lv]: [h][w][5A+C] fp32 (sigmoid reg | sigmoid obj | softmax cls: model/detector.py:33-44), lv 0 = stride 16 map.
 * anchors: 2*A*2 floats (w,h per anchor, level-major) as the sample's `bias` vector (:34-37).  scale_w/h = source image
 * size / network input size (:189-190).  Writes up to max_out boxes in descending score order; returns the TOTAL kept. */
int oracle_ncnn_post(const float *out2, int h2, int w2, const float *out3, int h3, int w3, int A, int C, int in_w, int in_h,
                     const float *anchors, float thresh, float nms_thresh, float scale_w, float scale_h, int max_out,
                     int *boxes, float *scores, int *cates) {
    const float *outs[2] = {out2, out3};
    const int hs[2] = {h2, h3}, ws[2] = {w2, w3};
    const int ch = 5 * A + C;
    const size_t cap = (size_t)A * ((size_t)h2 * w2 + (size_t)h3 * w3);
    tbox *tmp = (tbox *)malloc(sizeof(tbox) * (cap ? cap : 1));
    int *picked = (int *)malloc(sizeof(int) * (cap ? cap : 1));
    int n = 0, np = 0;
    (void)in_w;
    if (!tmp || !picked) { free(tmp); free(picked); return -1; }
    for (int i = 0; i < 2; ++i) {                                                                         /* :137-182 */
        const int outH = hs[i], outW = ws[i];
        const int stride = in_h / outH;                                                                    /* :147 */
        const float *values = outs[i];
        for (int h = 0; h < outH; ++h)
            for (int w = 0; w < outW; ++w) {
                for (int b = 0; b < A; ++b) {
                    int category = -1;                                                                     /* :156-157 */
                    float score = -1.f, best = 0.f;
                    const float obj = values[4 * A + b];                                                   /* :116 */
                    for (int k = 0; k < C; ++k) {                                                          /* :118-128 */
                        float cs = values[4 * A + A + k];
                        cs *= obj;
                        if (cs > best) { score = cs; category = k; best = cs; }
                    }
                    if (score > thresh) {                                                                  /* :161 */
                        float bcx = (float)(((double)values[b * 4 + 0] * 2. - 0.5 + (double)w) * (double)stride);
                        float bcy = (float)(((double)values[b * 4 + 1] * 2. - 0.5 + (double)h) * (double)stride);
                        const double tw = (double)values[b * 4 + 2] * 2., th = (double)values[b * 4 + 3] * 2.;
                        float bw = (float)((tw * tw) * (double)anchors[(i * A * 2) + b * 2 + 0]);          /* pow(x, 2) is exact here */
                        float bh = (float)((th * th) * (double)anchors[(i * A * 2) + b * 2 + 1]);
                        tbox t;
                        t.x1 = yfv2_ncnn_corner(((double)bcx - 0.5 * (double)bw) * (double)scale_w);       /* :170-173: double -> int */
                        t.y1 = yfv2_ncnn_corner(((double)bcy - 0.5 * (double)bh) * (double)scale_h);
                        t.x2 = yfv2_ncnn_corner(((double)bcx + 0.5 * (double)bw) * (double)scale_w);
                        t.y2 = yfv2_ncnn_corner(((double)bcy + 0.5 * (double)bh) * (double)scale_h);
                        t.score = score; t.cate = category; t.order = n;
                        tmp[n++] = t;
                    }
                }
                values += ch;                                                                              /* :179 */
            }
    }
    qsort(tmp, (size_t)n, sizeof(tbox), cmp_score_desc);                                                   /* :84 */
    for (int i = 0; i < n; ++i) {                                                                          /* :86-103 */
        int keep = 1;
        for (int j = 0; j < np; ++j) {
            const float ia = inter_area(&tmp[i], &tmp[picked[j]]);
            const float ua = tb_area(&tmp[i]) + tb_area(&tmp[picked[j]]) - ia;
            const float iou = ia / ua;
            if (iou > nms_thresh && tmp[i].cate == tmp[picked[j]].cate) { keep = 0; break; }
        }
        if (keep) picked[np++] = i;
    }
    for (int i = 0; i < np && i < max_out; ++i) {
        const tbox *t = &tmp[picked[i]];
        boxes[4 * i] = t->x1; boxes[4 * i + 1] = t->y1; boxes[4 * i + 2] = t->x2; boxes[4 * i + 3] = t->y2;
        scores[i] = t->score; cates[i] = t->cate;
    }
    free(tmp); free(picked);
    return np;
}
