/*
 * yfv2.h — C ABI of libyfv2.so, the H100 (sm_90a) implementation of the Yolo-FastestV2 hot path.
 *
 * The reference (dog-qiuqiu/Yolo-FastestV2 @ ac2a5e3) has no FFI of its own: its boundary is the
 * Python import surface (SURVEY.md 8b).  Each entry point below replaces one reference function; the
 * Python mirror modules under yolo-fastestv2_b200/{model,utils}/ call these through ctypes and give
 * the result the reference's return types.  INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes.  Every function returns 0 on success or a negative
 *     YFV2_E* code; yfv2_last_error() returns a thread-local message for the last failure.
 *   - All `float*` / `void*` tensor arguments are DEVICE pointers unless the name ends in `_host`.
 *   - The caller owns every buffer (inputs, outputs, packed weights, workspace).  The library never
 *     allocates or frees device memory; the only state is the opaque host-side yfv2_plan.
 *   - `stream` is a cudaStream_t passed as void* (Python: torch.cuda.current_stream().cuda_stream).
 *     All launches are asynchronous on it; nothing here synchronises the device, except the
 *     *_host convenience calls which say so.
 *   - No C++ exception crosses the ABI.  There is no CPU fallback: without a CUDA device every
 *     compute entry point returns YFV2_ECUDA.
 */
#ifndef YFV2_H_
#define YFV2_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YFV2_OK            0
#define YFV2_EINVAL       -1   /* bad argument (null pointer, unsupported shape) */
#define YFV2_ECUDA        -2   /* a CUDA runtime call or launch failed */
#define YFV2_EUNSUPPORTED -3   /* valid request this build does not implement */
#define YFV2_ENOMEM       -4   /* host allocation failed / workspace too small */

#define YFV2_ABI_VERSION   1

#if defined(__GNUC__)
#define YFV2_API __attribute__((visibility("default")))
#else
#define YFV2_API
#endif

/* Number of float tensors yfv2_pack_weights consumes, in reference state_dict order:
 * 225 parameters (Detector.parameters(), model/detector.py:8-19) and 73 BatchNorm layers. */
#define YFV2_NUM_PARAMS    225
#define YFV2_NUM_BN         73
#define YFV2_NUM_GRADS  243095  /* 80 classes, 3 anchors */

typedef struct yfv2_plan yfv2_plan;

YFV2_API int         yfv2_abi_version(void);
YFV2_API const char* yfv2_last_error(void);

/* ---- plan -----------------------------------------------------------------------------------------
 * One plan per (device, N, H, W, A, C, training).  H and W must be multiples of 32
 * (model/backbone/shufflenetv2.py strides; utils/loss.py:78).  Replaces Detector.__init__'s shape
 * bookkeeping (model/detector.py:8-19).  A <= 8, C <= 256 (else YFV2_EINVAL); A + C <= 192, i.e. up to 189 classes at 3
 * anchors (the heads' output convolution runs as one or two 96-column tiles; larger: YFV2_EUNSUPPORTED). */
YFV2_API int yfv2_plan_create(yfv2_plan** plan, int device, int N, int H, int W, int A, int C, int training);
YFV2_API int yfv2_plan_destroy(yfv2_plan* plan);
YFV2_API int yfv2_plan_workspace_bytes(const yfv2_plan* plan, size_t* bytes);
/* The workspace is caller-owned but DEDICATED to the plan while the plan is in use: activation planes live in it inside
 * zero frames (the padding of every 3x3 / 5x5 convolution) which the first forward on a given workspace pointer writes
 * once and later forwards rely on.  If the memory was used for anything else in between, or was freed and re-allocated
 * (a caching allocator may hand back the same address), call yfv2_plan_invalidate_workspace() before the next forward. */
YFV2_API int yfv2_plan_invalidate_workspace(yfv2_plan* plan);
YFV2_API int yfv2_plan_packed_bytes(const yfv2_plan* plan, size_t* bytes);
/* number of kernels one yfv2_forward / yfv2_detect launches (for bench.py's gpu_launches) */
YFV2_API int yfv2_plan_forward_launches(const yfv2_plan* plan, int* n);

/* ---- weights ----------------------------------------------------------------------------------------
 * params:     225 device pointers, Detector.parameters() order (== state_dict order without buffers).
 * bn_running: 146 device pointers, (running_mean, running_var) for each of the 73 BatchNorm2d in
 *             state_dict order.  Eval plans fold BN into per-channel scale/shift kept next to the
 *             transposed conv weights (eps = 1e-5, nn.BatchNorm2d default used by the reference). */
YFV2_API int yfv2_pack_weights(yfv2_plan* plan, const float* const* params, const float* const* bn_running,
                      void* packed, void* stream);

/* ---- Detector.forward (model/detector.py:21-31,46-47) ------------------------------------------------
 * x: [N,3,H,W] fp32 NCHW in [0,1] (BGR).  preds: six dense NCHW tensors
 * (reg_2 [N,4A,H/16,W/16], obj_2 [N,A,..], cls_2 [N,C,..], reg_3, obj_3, cls_3 at H/32) raw logits. */
YFV2_API int yfv2_forward(yfv2_plan* plan, const float* x, const void* packed, float* const preds[6],
                 void* workspace, void* stream);
/* Same, from uint8 [N,3,H,W]: fuses the `imgs.float() / 255.0` of utils/utils.py:368, test.py:38,
 * train.py:101 into the stem kernel's load. */
YFV2_API int yfv2_forward_u8(yfv2_plan* plan, const uint8_t* x, const void* packed, float* const preds[6],
                    void* workspace, void* stream);

/* ---- handel_preds (utils/utils.py:303-358) -----------------------------------------------------------
 * anchors_host: 2*A*2 doubles (level-major, cfg["anchors"]).  out: [N, (H/16*W/16 + H/32*W/32)*A, 5+C]
 * fp32, row (y*w+x)*A+a within a level, stride-16 level first.  img_h is cfg["height"] (the reference
 * derives ONE stride from it for both axes, utils/utils.py:332). */
YFV2_API int yfv2_decode(const float* const preds[6], int N, int H, int W, int A, int C,
                const double* anchors_host, float* out, void* stream);

/* ---- export_onnx head (model/detector.py:33-44): sigmoid(reg) | sigmoid(obj) | softmax(cls), channel-last --------------
 * out2: [N, H/16, W/16, 5A+C], out3: [N, H/32, W/32, 5A+C] (what Detector(..., export_onnx=True).forward returns). */
YFV2_API int yfv2_export_heads(const float* const preds[6], int N, int H, int W, int A, int C, float* out2, float* out3,
                               void* stream);

/* ---- deploy post-process: what yoloFastestv2::detection does after the forward (sample/ncnn/src/yolo-fastestv2.cpp) --------
 * predHandle (:134-183: cls*obj first strict maximum above 0, grid decode in double, corners (c -/+ w/2)*scale truncated to
 * int) + nmsHandle (:78-110: descending score, greedy, suppressed iff IoU > nms_thresh with a kept box of the SAME class;
 * IoU on the int corners, :58-71) on the two export_onnx tensors of yfv2_export_heads.  H, W: network input size (inputHeight /
 * inputWidth); anchors_host: 2*A*2 floats (the sample's `bias`, :34-37); scale_w/h: source image size / network input size
 * (:189-190).  Outputs per image, descending score: boxes [N,max_out,4] int32 (x1,y1,x2,y2), scores [N,max_out], cates
 * [N,max_out] int32, counts [N] = number kept (rows past min(count, max_out): zeros / cate -1; the sample has no cap, so pass
 * max_out = A*(H/16*W/16 + H/32*W/32) to never truncate).
 *   Categories: the first strict maximum of cls*obj above 0, so among equal products the smaller class wins and NaN products
 *   are skipped; a cell with none has score -1, cate -1 and is a candidate iff -1 > thresh (those suppress each other as a
 *   class of their own).
 *   Ties: equal scores keep push order (level, row, column, anchor).  The sample's std::sort leaves that order open; libstdc++'s
 *   gives push order too while at most 16 candidates pass (insertion sort, stable).
 *   Corners: each (c -/+ w/2)*scale in double becomes an int by yfv2_ncnn_corner below: truncation toward zero, and INT_MIN
 *   for NaN or a truncated value outside the int range (what the sample's `int = double` compiles to on x86-64, cvttsd2si).
 *   Box widths and intersections of such corners are int differences that wrap.
 *   Limits: A <= 8, 1 <= C <= 32767, H and W multiples of 32, max_out >= 1 (else YFV2_EINVAL); the M = A*(H/16*W/16 +
 *   H/32*W/32) candidate slots of one image are sorted and suppressed in one CTA's shared memory (about 20 bytes per slot
 *   plus 8 per slot of M rounded up to a power of two, at most 227 KiB: A=3 up to 672x672, A=1 up to 1184x1184, A=8 up to
 *   416x416), a larger M is YFV2_EUNSUPPORTED before anything is launched.  out3 must hold N*(H/32)*(W/32)*(5A+C) floats. */
#ifdef __CUDACC__
#define YFV2_HOST_DEVICE __host__ __device__
#else
#define YFV2_HOST_DEVICE
#endif
#include <limits.h>
static inline YFV2_HOST_DEVICE int yfv2_ncnn_corner(double v) {
    return (v > -2147483649.0 && v < 2147483648.0) ? (int)v : INT_MIN;
}
YFV2_API int yfv2_ncnn_post(const float* out2, const float* out3, int N, int H, int W, int A, int C, const float* anchors_host,
                            float thresh, float nms_thresh, float scale_w, float scale_h, int max_out, int* boxes, float* scores,
                            int* cates, int* counts, void* stream);

/* ---- non_max_suppression (utils/utils.py:232-296) + torchvision.ops.nms ------------------------------
 * dets: [N,M,5+C].  out: [N,max_det,6] rows (x1,y1,x2,y2,conf,cls) by descending conf; counts: [N];
 * kept_idx (optional, may be NULL): [N,max_det] row index into dets[n].  class_filter: n_filter device
 * ints or NULL.  Candidates per image are limited to YFV2_NMS_MAX_CAND (the reference's max_nms=30000
 * branch, utils/utils.py:278-280, cannot trigger below that); larger M returns YFV2_EUNSUPPORTED.
 * The reference's 1-second wall-clock abort (utils/utils.py:292-294) is not reproduced. */
#define YFV2_NMS_MAX_CAND 8192
YFV2_API int yfv2_nms_workspace_bytes(int N, int M, int C, size_t* bytes);
YFV2_API int yfv2_nms(const float* dets, int N, int M, int C, float conf_thres, double iou_thres,
             const int* class_filter, int n_filter, int max_det, float max_wh,
             float* out, int* counts, int* kept_idx, void* workspace, void* stream);

/* Fused decode + NMS straight from the six head tensors (no [N,M,5+C] round trip through HBM);
 * bit-identical to yfv2_decode followed by yfv2_nms. */
YFV2_API int yfv2_decode_nms(const float* const preds[6], int N, int H, int W, int A, int C,
                    const double* anchors_host, float conf_thres, double iou_thres,
                    const int* class_filter, int n_filter, int max_det, float max_wh,
                    float* out, int* counts, int* kept_idx, void* workspace, void* stream);

/* ---- detections of regions (tiles, zones) of frames -> one list per frame in frame pixels: a cross-region NMS --------------
 * No reference counterpart: the reference detects on whole images (test.py:34-68).  Region t is a crop (x0, y0, w, h) of frame
 * `frame`, stretched to the W x H network input; dets [T, max_det_in, 6] / counts [T] are its rows as yfv2_nms / yfv2_decode_nms
 * write them (x1, y1, x2, y2, conf, cls in network-input pixels; the first min(max(counts[t], 0), max_det_in) rows are read).
 * regions: T HOST descriptors, the regions of one frame contiguous and frame indices ascending (a frame may have none).
 * Per frame, bit-exact to tests/region_oracle.py:
 *   1. mapping: sx = (double)w / W, sy = (double)h / H, x' = x*sx + x0, y' = y*sy + y0, each a rounded fp64 product then a
 *      rounded fp64 sum (no FMA); conf and cls are copied.  With x0 = y0 = 0 this is the x * (w / W) of test.py:57-68.
 *   2. order: conf descending, ties by region t, then by row; rows whose conf is NaN are dropped.
 *   3. greedy: walking that order, row j is kept unless an already kept row i has t(i) != t(j) (rows of one region were already
 *      separated by its own NMS), the same cls, and overlap(i, j) > thr.
 *   4. overlap in fp64, no +1: inter = max(0, min(x2) - max(x1)) * max(0, min(y2) - max(y1)), area = (x2 - x1) * (y2 - y1),
 *      with min(a, b) = a < b ? a : b, max(a, b) = a > b ? a : b and a = the kept row's value; metric 0 (IoU):
 *      inter / (area_i + area_j - inter), metric 1 (IoS): inter / min(area_i, area_j).  A NaN overlap never suppresses.
 *   5. at most max_det rows per frame.
 * out: [F, max_det, 6] float64 in that order (rows past out_counts[f]: zeros); out_counts [F]; kept_src (optional, may be NULL):
 * [F, max_det] t * max_det_in + row of each kept row (-1 past the count).  Checked before any launch (YFV2_EINVAL, naming the bad
 * region or argument): non-null pointers, T, F, W, H >= 1, 1 <= max_det_in, max_det <= 4096, metric 0 or 1, thr not NaN,
 * T * max_det_in < 2^31; per region w, h >= 1, x0, y0 >= 0, frame in [0, F) and not decreasing; per frame its regions x
 * max_det_in <= YFV2_NMS_MAX_CAND and at most YFV2_MERGE_MAX_REGIONS regions.  No workspace. */
#define YFV2_MERGE_MAX_REGIONS 1024
typedef struct yfv2_region {
    int frame;             /* index of the frame the region belongs to */
    int x0, y0, w, h;      /* the crop, in pixels of that frame */
} yfv2_region;
YFV2_API int yfv2_merge_regions(const float* dets, const int* counts, const yfv2_region* regions, int T, int max_det_in, int F,
                                int H, int W, double thr, int metric, int max_det, double* out, int* out_counts, int* kept_src,
                                void* stream);

/* ---- multi-object tracking across video frames: ByteTrack's association and lifecycle, S streams in one device state ---------
 * No reference counterpart (the reference detects on single images).  The tracker keeps S streams (cameras) of at most K tracks
 * each in one caller-owned device buffer of yfv2_track_state_bytes(S, K) bytes; yfv2_track_reset clears chosen streams (no
 * tracks, frame 0, next id 1) and must run on every stream before its first update.  One yfv2_track_update call gives B distinct
 * streams one frame each, in ONE launch with one CTA per stream; it allocates nothing and never synchronises.  Class-agnostic: a
 * track takes the class of its latest detection.  Bit-exact to tests/track_oracle.py.
 *
 * Arithmetic: IEEE fp64, one rounding per operation (no FMA, no sqrt); min(a, b) = a < b ? a : b, max(a, b) = a > b ? a : b.
 * Detections: dets [B, M, 6] float64 rows (x1, y1, x2, y2, conf, cls) in frame pixels (what yfv2_merge_regions writes), counts [B]
 * (the first min(max(counts[b], 0), M) rows are read).  A row is used when all six values are finite, x2 > x1, y2 > y1 and
 * conf > low_thresh; it is "high" if conf > high_thresh, else "low".  Its measurement z = (cx, cy, a, h): w = x2 - x1,
 * h = y2 - y1, cx = x1 + w/2, cy = y1 + h/2, a = w / h.
 * Kalman filter, constant velocity on (cx, cy, a, h), DeepSORT's noise model in four decoupled 2x2 blocks: coordinate k keeps
 * position variance p, cross term x, velocity variance v; sp = 1/20, sv = 1/160; products left to right, squares as s * s.
 *   initiate: mean = (z, 0, 0, 0, 0); std_pos = ((2*sp)*h, (2*sp)*h, 1e-2, (2*sp)*h); std_vel = ((10*sv)*h, (10*sv)*h, 1e-5,
 *             (10*sv)*h); p = std_pos^2, x = 0, v = std_vel^2.
 *   predict (every live track; a lost one first sets mean[7] = 0): h = mean[3] before the step; q_pos = (sp*h, sp*h, 1e-2,
 *             sp*h)^2, q_vel = (sv*h, sv*h, 1e-5, sv*h)^2; mean[k] += mean[k+4]; t = x + v; p = ((p + x) + t) + q_pos; x = t;
 *             v = v + q_vel.
 *   update:  h = predicted mean[3]; r = (sp*h, sp*h, 1e-1, sp*h)^2; s = p + r; k0 = p / s; k1 = x / s; y = z[k] - mean[k];
 *             mean[k] += k0*y; mean[k+4] += k1*y; p = p - k0*p; x' = x - k0*x; v = v - k1*x (the old x).
 *   box:      h = mean[3]; w = mean[2]*h; x1 = mean[0] - w/2; y1 = mean[1] - h/2; x2 = x1 + w; y2 = y1 + h.
 *   IoU(a, b), no +1: inter = max(0, min(a.x2, b.x2) - max(a.x1, b.x1)) * max(0, min(a.y2, b.y2) - max(a.y1, b.y1));
 *             IoU = inter / ((area_a + area_b) - inter), area = (x2 - x1) * (y2 - y1); a is the track (the tracked one in
 *             step 9).
 * One association stage: rows = tracks in ascending id, columns = detections in row order, cost c = 1 - IoU or, "fused",
 * 1 - IoU*conf; a pair is allowed iff c < thr.  (1) Only tracks and detections with an allowed pair are kept, in order; the
 * smaller side plays the solver's rows (the tracks on equal sizes).  (2) C[i][j] = c - thr if allowed, else 0.  (3) Crouse's
 * shortest augmenting path (scipy's linear_sum_assignment), rows in order; per row: SR = SC = {}, i = row, minVal = 0, shortest
 * = +inf; until an unassigned column is reached: SR += i; for j not in SC: r = ((minVal + C[i][j]) - u[i]) - v[j], if r <
 * shortest[j]: shortest[j] = r, path[j] = i; j* = the lowest j not in SC with the least shortest[j]; minVal = shortest[j*];
 * SC += j*; i = row4col[j*].  Then u[row] += minVal; u[i] += minVal - shortest[col4row[i]] for the other i in SR; v[j] -= minVal
 * - shortest[j] for j in SC; augment along path.  (4) Assigned pairs that are not allowed stay unmatched.
 * One update of stream s: (1) frame += 1, predict every live track.  (2) stage 1, fused, thr = match_thresh: confirmed tracks
 * (tracked or lost) x high detections.  (3) stage 2, thr 0.5: confirmed tracked tracks unmatched by stage 1 x low detections.
 * (4) confirmed tracked tracks still unmatched become lost.  (5) stage 3, fused, thr 0.7: tentative tracks x high detections
 * still unmatched; unmatched tentative tracks are removed.  (6) matched tracks: Kalman update, state tracked, confirmed, score,
 * cls and det_row of the detection, end_frame = frame (a lost track found again keeps its id).  (7) births, in row order: every
 * unmatched high detection with conf >= new_thresh starts a track with id next_id++, start_frame = end_frame = frame, confirmed
 * iff frame == 1; with K live tracks it is not created, spends no id and counts in dropped[b].  (8) lost tracks with frame -
 * end_frame > max_age are removed.  (9) of every pair (p tracked, tentative or not; q lost) with IoU(box p, box q) > 0.85, judged
 * on the state before any of these removals, q is removed if age(p) > age(q), else p (age = frame - start_frame).  (10) out
 * [B, K, 8] float64: the confirmed tracked tracks in ascending id, (x1, y1, x2, y2, score, cls, id, det_row) with the box of the
 * updated mean; out_counts [B]; rows past the count are zeros.
 * Checked before any launch (YFV2_EINVAL, naming the argument): non-null pointers; 1 <= K <= YFV2_TRACK_MAX_CAPACITY;
 * 1 <= M <= YFV2_TRACK_MAX_ROWS; 1 <= B <= min(S, YFV2_TRACK_MAX_BATCH); streams_host[b] in [0, S), each at most once; thresholds finite with 0 <= low <
 * high <= new <= 1 and 0 < match <= 1; max_age >= 0. */
#define YFV2_TRACK_MAX_CAPACITY 1024
#define YFV2_TRACK_MAX_ROWS     2048
#define YFV2_TRACK_MAX_BATCH    4096   /* streams per call: their indices travel in the launch's parameters */
#define YFV2_TRACK_TRACKED 1
#define YFV2_TRACK_LOST    2
typedef struct yfv2_track_params {
    double high_thresh, low_thresh, new_thresh, match_thresh;   /* ByteTrack's 0.5, 0.1, 0.6, 0.8 */
    int max_age;                                                /* frames a lost track survives (30) */
} yfv2_track_params;
typedef struct yfv2_track {
    double mean[8];        /* cx, cy, a, h, then their velocities */
    double cov[12];        /* coordinate k (cx, cy, a, h): p, x, v at [3k], [3k+1], [3k+2] */
    double score, cls;     /* of the latest detection */
    int id, state;         /* YFV2_TRACK_TRACKED | YFV2_TRACK_LOST */
    int confirmed, start_frame, end_frame, det_row;
} yfv2_track;
YFV2_API int yfv2_track_state_bytes(int S, int K, size_t* bytes);
YFV2_API int yfv2_track_reset(void* state, int S, int K, const int* streams_host, int B, void* stream);
YFV2_API int yfv2_track_update(void* state, int S, int K, const int* streams_host, int B, const double* dets, const int* counts,
                               int M, const yfv2_track_params* params, double* out, int* out_counts, int* dropped, void* stream);
/* test hook: stream s's frame, next id and live tracks in ascending id (n_host of them, at most K) copied to the host; synchronises
 * `stream` */
YFV2_API int yfv2_track_debug_read(const void* state, int S, int K, int s, int* frame_host, int* next_id_host, yfv2_track* tracks_host,
                                   int* n_host, void* stream);

/* ---- get_batch_statistics (utils/utils.py:184-230): true-positive flags of NMS output rows ----------------
 * dets [N,max_det,6] / counts [N] as yfv2_nms writes them (a count above max_det is taken as max_det); targets [nt,6]
 * rows (image, class, x1, y1, x2, y2) in pixels (what evaluation() builds at utils/utils.py:372-375), in any order and
 * any number (an image claims at most max_det of its annotations, and that claim list is all the state kept per image).
 * max_det <= YFV2_EVAL_MAX_DET, else YFV2_EUNSUPPORTED before the launch.  tp [N,max_det] receives 1.0 for a true
 * positive, 0.0 otherwise (rows past counts[n] are 0).  Same greedy order and the same fp32 IoU (+1 convention) as the
 * reference, and its torch max(0) choice of annotation (first maximum; a NaN IoU counts as the maximum and then fails the
 * threshold): bit-identical flags. */
#define YFV2_EVAL_MAX_DET 8192
YFV2_API int yfv2_batch_statistics(const float* dets, const int* counts, int N, int max_det, const float* targets, int nt,
                                   float iou_threshold, float* tp, void* stream);

/* ---- contrast_and_brightness (utils/datasets.py:10-16; the augmentation img_aug applies, :63-68) on the device ----
 * out = cv2.addWeighted(img, alpha[n], zeros, 1 - alpha[n], beta[n]) for uint8 images: per byte
 * saturate_cast<uint8>(cvRound(fl32(fl32(x * alpha) + beta))).  img / out: N images of bytes_per_image bytes each (any
 * layout: the operation is elementwise; in place allowed); alpha / beta: device arrays [N] (the reference draws both from
 * random.uniform(0.25, 1.75) per image on the host).  Bit-identical to OpenCV 4.x. */
YFV2_API int yfv2_aug_contrast_brightness(const uint8_t* img, uint8_t* out, const float* alpha, const float* beta, int N,
                                          long long bytes_per_image, void* stream);

/* ---- img_aug with random_resize and augment_hsv (utils/datasets.py:63-68 with :66-67 enabled) on the device -------------
 * One pass over img [N,3,H,W] (planar B, G, R uint8, the training batch) into out, per image in img_aug's order:
 *   YFV2_AUG_CONTRAST  contrast_and_brightness (:10-16), the arithmetic of yfv2_aug_contrast_brightness, on every source byte;
 *   YFV2_AUG_RESIZE    random_resize (:54-61): cv2.resize(cv2.resize(img, (rw, rh)), (W, H)), both INTER_LINEAR with the
 *                      arithmetic of yfv2_resize_bgr_u8; the rw x rh image is recomputed where read, never stored;
 *   YFV2_AUG_HSV       augment_hsv (:39-51): cv2.cvtColor(COLOR_BGR2HSV), the image's three LUTs on H, S, V,
 *                      cv2.cvtColor(COLOR_HSV2BGR), both conversions bit-identical to OpenCV 4.13's 8-bit paths (x86,
 *                      with the HSV2BGR rounding of the last W mod 32 pixels of a row, see yfv2_debug_hsv2bgr).
 * params: HOST array [N]; alpha / beta are read with YFV2_AUG_CONTRAST, rw / rh (1 <= rw <= W, 1 <= rh <= H; the reference
 * draws int(W * uniform(0.8, 1)), then int(H * uniform(0.8, 1))) with YFV2_AUG_RESIZE.  luts: device [N][3][256] uint8 (hue,
 * saturation, value LUTs as datasets.py:44-47 build them from the image's gains), required with YFV2_AUG_HSV, else ignored.
 * In place (img == out) is allowed without YFV2_AUG_RESIZE; any other overlap is refused.  H, W <= 32768.  Every argument is
 * checked before anything is launched (YFV2_EINVAL). */
#define YFV2_AUG_CONTRAST 1
#define YFV2_AUG_RESIZE   2
#define YFV2_AUG_HSV      4
typedef struct yfv2_aug_params {
    float alpha, beta;     /* contrast_and_brightness */
    int rw, rh;            /* random_resize's intermediate size */
} yfv2_aug_params;
YFV2_API int yfv2_aug_batch(const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_params* params,
                            const uint8_t* luts, int flags, void* stream);
/* ---- img_aug with every line enabled: yfv2_aug_batch plus motion_blur (utils/datasets.py:18-37, img_aug's second step) ----
 * Takes yfv2_aug_batch's arguments and flags, plus YFV2_AUG_BLUR, and runs contrast -> motion_blur -> random_resize ->
 * augment_hsv per image.  blur: HOST array [N], one descriptor per image: ksize 0 is an image that drew no blur (the reference's
 * randint(1, 2) == 2); ksize 2 or 3 is the drawn degree, with taps[0 .. ksize^2 - 1] the fp32 kernel in row-major order as
 * cv2.filter2D receives it (cv2.warpAffine of diag(ones(degree)) by getRotationMatrix2D((degree/2, degree/2), angle, 1), over
 * degree, rounded to fp32; yfv2_engine.motion_blur_taps computes it).  A blurred image is
 *   cv2.filter2D(img, -1, taps): anchor (ksize/2, ksize/2), BORDER_REFLECT_101 per channel, per byte the fp32 fused multiply-add
 *     chain over the nonzero taps in row-major order from 0, rounded half to even and saturated;
 *   cv2.normalize(., 0, 255, NORM_MINMAX): min and max over all three channels, scale = 255 * (1 / (max - min)) (0 when the
 *     image is constant), shift = -min * scale in fp64, byte = rint(fmaf(x, (float)scale, (float)shift)) saturated.
 * workspace: device, at least yfv2_aug_blur_workspace_bytes(N, H, W) bytes, overlapping neither img nor out; required with
 * YFV2_AUG_BLUR (it holds each blurred image between the two passes), else ignored, as is blur.  Without YFV2_AUG_BLUR the
 * call is yfv2_aug_batch.  Every argument, ksize and tap is checked before anything is launched (YFV2_EINVAL). */
#define YFV2_AUG_BLUR     8
typedef struct yfv2_aug_blur {
    int ksize;             /* 0 (no blur), 2 or 3 */
    float taps[9];         /* [ksize][ksize] row-major */
} yfv2_aug_blur;
YFV2_API int yfv2_aug_blur_workspace_bytes(int N, int H, int W, size_t* bytes);
YFV2_API int yfv2_aug_batch_blur(const uint8_t* img, uint8_t* out, int N, int H, int W, const yfv2_aug_params* params,
                                 const uint8_t* luts, const yfv2_aug_blur* blur, int flags, void* workspace,
                                 size_t workspace_bytes, void* stream);
/* Test hooks: n packed 3-byte pixels through the device's cv2.cvtColor COLOR_BGR2HSV / COLOR_HSV2BGR (any input bytes).  cv2's
 * 8-bit HSV2BGR rounds the last (row_w mod 32) pixels of each row differently from the others (OpenCV 4.13 x86: vector code
 * truncates, the scalar tail rounds), so the pixels are taken as rows of row_w. */
YFV2_API int yfv2_debug_bgr2hsv(const uint8_t* in, uint8_t* out, long long n, void* stream);
YFV2_API int yfv2_debug_hsv2bgr(const uint8_t* in, uint8_t* out, long long n, int row_w, void* stream);

/* ---- raw frames -> network input: cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR) on the device ----------------
 * The resize the reference runs on the host before every forward (test.py:35; utils/datasets.py:107 for training and
 * validation), fused with the HWC -> CHW transpose of test.py:36-37.  frames: N HOST descriptors of packed HWC BGR uint8 frames
 * in device memory (what cv2.imread and video decoders produce); each frame has its own size, so one batch may mix sizes, and
 * `pitch` (bytes between rows, >= 3*w) lets a crop of a larger frame be passed in place.  dst: device uint8 [N,3,H,W], the input
 * of yfv2_forward_u8 / yfv2_detect_u8_host.  H, W: any size in 1..32768 (not only multiples of 32).  Bit-identical to OpenCV's
 * x86 8-bit INTER_LINEAR path (11-bit fixed-point weights; DESIGN.md §7).  The coefficients are computed in the kernel, so there
 * is no workspace; descriptors are checked before anything is launched. */
typedef struct yfv2_frame {
    const uint8_t* data;   /* device pointer to pixel (0,0): B, G, R bytes */
    int w, h;              /* size in pixels */
    long long pitch;       /* bytes from one row to the next */
} yfv2_frame;
YFV2_API int yfv2_resize_bgr_u8(const yfv2_frame* frames, int N, int H, int W, uint8_t* dst, void* stream);

/* ---- YUV 4:2:0 frames -> network input: cv2.cvtColor(COLOR_YUV2BGR_*) + cv2.resize INTER_LINEAR on the device ---------------
 * What a caller with decoded video or camera frames runs on the host before test.py:35-37: cv2.cvtColor(frame,
 * cv2.COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12) (BT.601 limited range, the only YUV 4:2:0 conversion cv2 has), then the resize
 * and transpose of yfv2_resize_bgr_u8.  Each source pixel is converted in the kernel, so it reads 1.5 bytes per pixel instead of
 * 3.  frames: N HOST descriptors of frames in device memory; one batch may mix sizes, pitches and layouts.  Every layout is one
 * luma plane (w x h bytes, rows y_pitch apart) and chroma of (w/2) x (h/2) samples, sample (i, j) of U at u + i*uv_pitch +
 * j*uv_step, of V likewise from v:
 *   NV12: u = the interleaved UV plane, v = u + 1, uv_step 2;   NV21: v = the VU plane, u = v + 1, uv_step 2;
 *   I420: u, v = the U and V planes, uv_step 1;                 YV12: the same with V stored before U.
 * Planes need not be adjacent (a decoder surface with padded rows and height is passed as it is).  w and h must be even (cv2
 * refuses odd sizes too); y_pitch >= w, uv_pitch >= w for uv_step 2 and >= w/2 for uv_step 1.  dst, H, W: as yfv2_resize_bgr_u8.
 * Bit-identical to cv2.resize(cv2.cvtColor(...)) of OpenCV 4.x on x86 (DESIGN.md §7); descriptors are checked before anything
 * is launched. */
typedef struct yfv2_yuv420_frame {
    const uint8_t* y;      /* device pointer to luma pixel (0,0) */
    long long y_pitch;     /* bytes from one luma row to the next */
    const uint8_t* u;      /* device pointer to the U sample of pixel (0,0) */
    const uint8_t* v;      /* device pointer to the V sample of pixel (0,0) */
    long long uv_pitch;    /* bytes from one chroma row (two pixel rows) to the next, for U and V alike */
    int uv_step;           /* bytes from one chroma sample to the next along a row: 2 interleaved (NV12 / NV21), 1 planar */
    int w, h;              /* size in pixels, both even */
} yfv2_yuv420_frame;
YFV2_API int yfv2_resize_yuv420_u8(const yfv2_yuv420_frame* frames, int N, int H, int W, uint8_t* dst, void* stream);

/* ---- RGB, BGRA / RGBA, grey and planar RGB frames -> network input: cv2.cvtColor(COLOR_*2BGR) + cv2.resize INTER_LINEAR -------
 * One descriptor for every 8-bit layout that is a channel move away from packed BGR: channel k of pixel (r, c) is the byte at
 * ch_k + r*pitch + c*step, with ch_k = b, g, r.  Every such move commutes with the resize, so the result is the bytes of
 * cv2.resize(cv2.cvtColor(frame, code), (W, H), INTER_LINEAR) for the code named below, with d the address of pixel (0,0):
 *   BGR  (cv2.imread, no conversion)       b, g, r = d, d+1, d+2;  step 3      (yfv2_resize_bgr_u8 is 2.5 % faster for it)
 *   RGB  (PIL, most PyTorch data code)     b, g, r = d+2, d+1, d;  step 3      COLOR_RGB2BGR
 *   BGRA / BGRx (GStreamer, capture APIs)  b, g, r = d, d+1, d+2;  step 4      COLOR_BGRA2BGR (alpha ignored, as cv2 ignores it)
 *   RGBA / RGBx                            b, g, r = d+2, d+1, d;  step 4      COLOR_RGBA2BGR
 *   grey (IR / mono cameras)               b, g, r = d, d, d;      step 1      COLOR_GRAY2BGR
 *   planar CHW RGB (GPU JPEG decoders)     b, g, r = d+2s, d+s, d; step 1      transpose + COLOR_RGB2BGR (s: the channel stride)
 * frames: N HOST descriptors of frames in device memory; one batch may mix sizes, pitches and layouts.  Needs b, g, r non-null,
 * w, h > 0, step >= 1, pitch >= step*w and step*w < 2^31.  dst, H, W: as yfv2_resize_bgr_u8.  Descriptors are checked before
 * anything is launched. */
typedef struct yfv2_strided_frame {
    const uint8_t* b;      /* device pointer to the B byte of pixel (0,0) */
    const uint8_t* g;      /* ... the G byte */
    const uint8_t* r;      /* ... the R byte */
    long long pitch;       /* bytes from one row to the next, for all three channels */
    int step;              /* bytes from one pixel to the next along a row */
    int w, h;              /* size in pixels */
} yfv2_strided_frame;
YFV2_API int yfv2_resize_strided_u8(const yfv2_strided_frame* frames, int N, int H, int W, uint8_t* dst, void* stream);

/* ---- packed YUV 4:2:2 frames -> network input: cv2.cvtColor(COLOR_YUV2BGR_YUYV / _UYVY / _YVYU) + cv2.resize INTER_LINEAR ---
 * What USB (V4L2 YUYV) webcams and HDMI / SDI capture cards (UYVY) deliver.  Two pixels share one 4-byte macropixel: the luma of
 * pixel (r, c) is at y + r*pitch + 2c, and the U and V of the pair (r, 2j), (r, 2j + 1) at u + r*pitch + 4j and v + r*pitch + 4j:
 *   YUYV (YUY2): y = d, u = d+1, v = d+3;   UYVY: u = d, y = d+1, v = d+2;   YVYU: y = d, v = d+1, u = d+3.
 * Each pixel is converted with the BT.601 limited-range fixed point of yfv2_resize_yuv420_u8 (chroma not interpolated), which is
 * what cv2.cvtColor does for these codes.  Needs y, u, v non-null, w even and > 0 (cv2 asserts an even width), h > 0 (odd allowed),
 * pitch >= 2*w.  frames, dst, H, W: as yfv2_resize_strided_u8. */
typedef struct yfv2_yuv422_frame {
    const uint8_t* y;      /* device pointer to the luma of pixel (0,0) */
    const uint8_t* u;      /* device pointer to the U of pixels (0,0), (0,1) */
    const uint8_t* v;      /* device pointer to the V of pixels (0,0), (0,1) */
    long long pitch;       /* bytes from one row to the next */
    int w, h;              /* size in pixels, w even */
} yfv2_yuv422_frame;
YFV2_API int yfv2_resize_yuv422_u8(const yfv2_yuv422_frame* frames, int N, int H, int W, uint8_t* dst, void* stream);

/* ---- JPEG files -> packed HWC BGR frames: cv2.imread(path) (test.py:34; utils/datasets.py:106) on the device -----------------
 * The bytes OpenCV 4.13 (libjpeg-turbo 3.1) returns for IMREAD_COLOR: ISLOW IDCT, fancy upsampling, jdcolor's YCbCr -> BGR, grey
 * replicated to B = G = R, and the EXIF orientation applied.  Supported: baseline sequential Huffman-coded DCT (SOF0, SOF1) with
 * 8-bit samples, 1 or 3 components, luma sampling 1x1, 2x1, 2x2, 1x2 or 4x1 with 1x1 chroma, restart intervals, one scan; with
 * flags YFV2_JPEG_PROGRESSIVE also progressive Huffman-coded DCT (SOF2) within the same limits, up to 128 scans, tables and restart
 * intervals redefined between scans.  Anything else (progressive without the flag, arithmetic, lossless, hierarchical, 12/16-bit,
 * 2 or 4 components, Adobe RGB, several scans of a baseline file, other sampling, not a JPEG) is refused per file by the parse,
 * with a reason.  A progressive file is also refused, its reason naming the scan, component or coefficient, when a scan breaks
 * libjpeg's progression rules (YFV2_EINVAL: a DC scan with Se != 0; an AC scan with Ss > Se, Se > 63 or several components; Ah != 0
 * with Al != Ah - 1; Al > 13: cv2 returns no image), when it goes against what earlier scans sent (YFV2_EUNSUPPORTED: AC before
 * the component's DC, or Ah other than the bits already known), when a coefficient is never sent or not refined to its last bit
 * (YFV2_EUNSUPPORTED: libjpeg smooths such blocks), when a scan lists its components out of frame order (YFV2_EUNSUPPORTED:
 * libjpeg decodes it, this decoder does not), or when it has more than 128 scans.  A progressive file that ends before its
 * EOI is accepted and flagged 1: cv2.imdecode returns no image for it.
 *
 * yfv2_jpeg_parse_ex (host only, no device needed): the N files lie in one host buffer, file i at files_host[offsets_host[i] ..
 * offsets_host[i+1]).  Fills info_host[N] (status 0 or a YFV2_E* code with its reason; size after orientation; frame_offset) and
 * the sizes the decode needs: meta_bytes (the blob), workspace_bytes, frames_bytes (the arena; frame i is [h][w][3] BGR at
 * frame_offset, rows 3*w apart, usable as a yfv2_frame as it is).  With meta_host NULL only the sizes are computed; otherwise the
 * blob (decode tables, geometry and the byte range of every entropy-coded segment) is written into meta_host[meta_cap].  Returns
 * the first refused file's code (yfv2_last_error names it), YFV2_ENOMEM when meta_cap is too small, YFV2_EINVAL for flag bits other
 * than YFV2_JPEG_PROGRESSIVE.  yfv2_jpeg_parse is yfv2_jpeg_parse_ex with flags 0.
 *
 * yfv2_jpeg_decode: files (device) is a copy of the same buffer, files_bytes long; meta_dev a device copy of the blob, meta_host the
 * blob itself (checked, with the buffer sizes, before anything is launched).  Writes every frame into `frames` and a per-image flag
 * word into errors[N] (device int32; 1: a segment ran out of data, the file ends inside the scan or a progressive file before its
 * EOI, 2: an invalid Huffman code or a progressive scan's run past its band,
 * 4: RSTn markers out of sequence; the frame is still written, from zero bits past a segment's end, but is not promised to equal
 * cv2's: a frame with no flag set is cv2's byte for byte).  phases: YFV2_JPEG_ALL, or the subset of the three launches to run in
 * this call (entropy decode into the workspace, IDCT into planes in the workspace, upsample + colour into frames), for timing them
 * separately.  YFV2_JPEG_ENTROPY includes the progressive images' scans: their coefficients are zeroed, then one launch per level of
 * scans that depend on each other.
 * Nothing is allocated and nothing synchronises. */
#define YFV2_JPEG_ENTROPY 1
#define YFV2_JPEG_IDCT    2
#define YFV2_JPEG_COLOR   4
#define YFV2_JPEG_ALL     7
#define YFV2_JPEG_PROGRESSIVE 1   /* yfv2_jpeg_parse_ex flags: accept progressive files */
typedef struct yfv2_jpeg_info {
    int status;            /* 0, or why the file is refused: YFV2_EUNSUPPORTED (out of scope) or YFV2_EINVAL (malformed) */
    int w, h;              /* the decoded frame's size, EXIF orientation applied */
    int components;        /* 1 (grey) or 3 (YCbCr) */
    int h_samp, v_samp;    /* luma sampling factors (1, 1 for grey) */
    int orientation;       /* EXIF orientation 1..8 (1 without EXIF) */
    int restart_interval;  /* MCUs per restart interval (of the first scan), 0: none */
    int segments;          /* entropy-coded segments of all scans, each decoded by one thread */
    int scans;             /* 1, or a progressive file's scans */
    long long frame_offset;/* byte offset of the frame in the arena */
    char reason[96];       /* status != 0: what is refused */
} yfv2_jpeg_info;
YFV2_API int yfv2_jpeg_parse(const uint8_t* files_host, const long long* offsets_host, int N, yfv2_jpeg_info* info_host,
                             void* meta_host, size_t meta_cap, size_t* meta_bytes, size_t* workspace_bytes, size_t* frames_bytes);
YFV2_API int yfv2_jpeg_parse_ex(const uint8_t* files_host, const long long* offsets_host, int N, int flags, yfv2_jpeg_info* info_host,
                                void* meta_host, size_t meta_cap, size_t* meta_bytes, size_t* workspace_bytes, size_t* frames_bytes);
YFV2_API int yfv2_jpeg_decode(const void* meta_host, const void* meta_dev, size_t meta_bytes, const uint8_t* files, size_t files_bytes,
                              uint8_t* frames, size_t frames_bytes, int* errors, void* workspace, size_t workspace_bytes, int phases,
                              void* stream);
/* yfv2_jpeg_decode_resize: JPEG files straight into the network input, cv2.resize(cv2.imread(f), (W, H), INTER_LINEAR) transposed
 * to CHW (utils/datasets.py:106-110).  The same blob, files and workspace as yfv2_jpeg_decode, checked the same way before anything
 * is launched, but no frame arena: the entropy and IDCT phases run as in yfv2_jpeg_decode, then one launch upsamples, converts,
 * orients and resizes every image into dst [N][3][H][W] uint8 (device), 1 <= H, W <= 32768.  Image i is byte for byte
 * yfv2_jpeg_decode's frame i followed by yfv2_resize_bgr_u8 at (W, H); errors[N] are yfv2_jpeg_decode's flags.  Nothing is
 * allocated and nothing synchronises. */
YFV2_API int yfv2_jpeg_decode_resize(const void* meta_host, const void* meta_dev, size_t meta_bytes, const uint8_t* files,
                                     size_t files_bytes, int H, int W, uint8_t* dst, int* errors, void* workspace,
                                     size_t workspace_bytes, void* stream);

/* ---- frames and regions -> JPEG files: cv2.imencode('.jpg', img, params) on the device ----------------------------------------
 * Output i is, byte for byte, cv2.imencode('.jpg', img_i, params_i)[1] of OpenCV 4.13 (libjpeg-turbo 3.1): baseline, the Annex K
 * Huffman tables, islow FDCT, jccolor's fixed-point RGB -> YCbCr, jcsample's downsampling, JFIF APP0.  img_i is the BGR image
 * cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR) gives the frame (yfv2_resize_*'s conversions), or for YFV2_JPEG_SRC_GRAY the grey
 * frame itself (a one-component JPEG, as cv2 writes a 2-D array), cropped to [y0, y0 + h) x [x0, x0 + w) AFTER the conversion.
 * params_i: cv2's (IMWRITE_*, value) pairs, nparams ints (host): IMWRITE_JPEG_QUALITY (1; default 95; clamped to 0..100 as cv2
 * does, 0 encodes as 1), IMWRITE_JPEG_RST_INTERVAL (4; MCUs per restart interval, clamped to 0..65535 as cv2 does),
 * IMWRITE_JPEG_SAMPLING_FACTOR (7; 0x221111 4:2:0 default, 0x211111 4:2:2, 0x111111 4:4:4; 0x121111 and 0x411111:
 * YFV2_EUNSUPPORTED; other values YFV2_EINVAL).  IMWRITE_JPEG_PROGRESSIVE (2) and _OPTIMIZE (3) other than 0 and
 * IMWRITE_JPEG_LUMA_QUALITY (5) / _CHROMA_QUALITY (6) >= 0 change cv2's output and are refused (YFV2_EUNSUPPORTED); ids of other
 * formats are ignored, as cv2 ignores them.  Regions larger than 32768 on a side: YFV2_EUNSUPPORTED.
 *
 * yfv2_jpeg_encode_plan (host only, no device needed; frame pointers are recorded, never read): checks every output and its frame
 * descriptor, names the first refused output (yfv2_last_error), and reports meta_bytes (the blob: headers, geometry, quantiser
 * tables), workspace_bytes and arena_bytes.  out_offsets[N + 1] (may be NULL) receives where each output starts in the arena.
 * Each output's arena slot is its worst case: headers + 2 * (blocks * 209 + segments) + 2 * segments + 2 bytes (every block at
 * the longest codes the tables have, every byte stuffed).  With meta_host NULL only the sizes are computed.
 * yfv2_jpeg_encode: meta_dev a device copy of the blob, meta_host the blob itself (checked before any launch).  Writes output i at
 * arena + out_offsets[i] and its length into lengths[i] (device int64).  phases: YFV2_JPEG_ENC_ALL, or the stages to run in this
 * call, in order, for timing them separately (transform: coefficients; scan: bit counts and offsets; pack: the bits of every
 * segment; stuff: byte stuffing, markers and the final bytes).  Nothing is allocated and nothing synchronises. */
#define YFV2_JPEG_SRC_BGR     0   /* f.bgr */
#define YFV2_JPEG_SRC_STRIDED 1   /* f.strided: RGB, BGRA / RGBA, planar RGB (and grey replicated to BGR) */
#define YFV2_JPEG_SRC_GRAY    2   /* f.strided, the byte at b: a one-component JPEG */
#define YFV2_JPEG_SRC_YUV420  3   /* f.yuv420 */
#define YFV2_JPEG_SRC_YUV422  4   /* f.yuv422 */
#define YFV2_JPEG_ENC_TRANSFORM 1
#define YFV2_JPEG_ENC_SCAN      2
#define YFV2_JPEG_ENC_PACK      4
#define YFV2_JPEG_ENC_STUFF     8
#define YFV2_JPEG_ENC_ALL      15
typedef struct yfv2_jpeg_enc_src {
    int kind;                /* YFV2_JPEG_SRC_* */
    int x0, y0, w, h;        /* the region of the converted frame, inside it, w, h >= 1 */
    union {
        yfv2_frame bgr;
        yfv2_strided_frame strided;
        yfv2_yuv420_frame yuv420;
        yfv2_yuv422_frame yuv422;
    } f;                     /* the frame, in device memory */
    const int* params;       /* host: nparams ints, cv2.imencode's (IMWRITE_*, value) pairs; may be NULL with nparams 0 */
    int nparams;
} yfv2_jpeg_enc_src;
YFV2_API int yfv2_jpeg_encode_plan(const yfv2_jpeg_enc_src* srcs, int N, void* meta_host, size_t meta_cap, size_t* meta_bytes,
                                   size_t* workspace_bytes, long long* out_offsets, size_t* arena_bytes);
YFV2_API int yfv2_jpeg_encode(const void* meta_host, const void* meta_dev, size_t meta_bytes, void* workspace, size_t workspace_bytes,
                              uint8_t* arena, size_t arena_bytes, long long* lengths, int phases, void* stream);

/* ---- anchor k-means (genanchors.py:17-102): R runs of the reference's kmeans over one box set, iteration by iteration ---------
 * boxes: device [N][2] fp64 (w, h) as genanchors reads them from the label files.  State of run r, all device and caller-owned:
 * centroids [R][k][2] fp64 (before the first step: the initial picks, boxes[init[r][j]]), assignments [R][N] int32 (before the
 * first step: all -1), iterations [R] (0), status [R] (YFV2_ANCHOR_ACTIVE), changed [R] (0; every step leaves it 0).
 * yfv2_anchor_kmeans_step runs one iteration t of every active run, bit-identical to the reference's:
 *   similarity  IOU's four branches in its order, each a chain of individually rounded fp64 operations (no FMA);
 *   assignment  the argmin of d = 1 - s (the first minimum, or the first NaN, as np.argmin);
 *   stop        no assignment changed: YFV2_ANCHOR_CONVERGED, and the centroids are those iteration t used (the reference's
 *               result after t `iter` lines); t == max_iter: YFV2_ANCHOR_NOT_CONVERGED with the centroids iteration t used;
 *               a cluster left without members: YFV2_ANCHOR_EMPTY_CLUSTER, with the centroids and assignments of iteration t
 *               (the reference divides 0 by 0 there and never stops);
 *   update      otherwise centroid j = (the fp64 sum of its members' w, h, added one after another in increasing box index from
 *               0.0) / (double)count.
 * iterations[r] becomes t for the runs it advanced; *active (device int) receives the number of runs still active, the one value
 * a driver reads back per iteration.  Runs that have stopped are not touched.  Nothing is allocated and nothing synchronises.
 * yfv2_anchor_avg_iou writes avg_IOU (genanchors.py:34-40) of each run's centroids into avg_iou [R] fp64: per box Python's max
 * over its k similarities (a first NaN stays, a later one is skipped), summed in box order from 0.0, over N.
 * Both: N >= 1, 1 <= R <= 65535, k >= 1 and non-null pointers, max_iter >= 1, else YFV2_EINVAL; k > YFV2_ANCHOR_MAX_K:
 * YFV2_EUNSUPPORTED; checked before anything is launched. */
#define YFV2_ANCHOR_MAX_K          16   /* two levels x anchor_num <= 8 */
#define YFV2_ANCHOR_ACTIVE          0
#define YFV2_ANCHOR_CONVERGED       1
#define YFV2_ANCHOR_EMPTY_CLUSTER   2
#define YFV2_ANCHOR_NOT_CONVERGED   3
YFV2_API int yfv2_anchor_kmeans_step(const double* boxes, int N, int k, int R, int max_iter, double* centroids, int* assignments,
                                     int* iterations, int* status, int* changed, int* active, void* stream);
YFV2_API int yfv2_anchor_avg_iou(const double* boxes, int N, int k, int R, const double* centroids, double* avg_iou, void* stream);

/* ---- whole inference step with HOST buffers (the evaluation() inner loop, utils/utils.py:367-383) ----
 * x_host: pinned uint8 [N,3,H,W]; out_host: pinned [N,max_det,6]; counts_host: pinned [N]; anchors_host: 4 * A doubles as
 * for yfv2_decode; workspace: at least yfv2_detect_workspace_bytes(plan, max_det) device bytes (more than
 * yfv2_plan_workspace_bytes: the input copy, the head tensors and the detections live behind the forward's workspace).
 * Copies in, runs forward_u8 + decode_nms, copies out, all on `stream`; returns without synchronising.  Every argument
 * yfv2_decode_nms would refuse (max_det outside 1..4096, more than YFV2_NMS_MAX_CAND candidates per image, NMS state over
 * the shared memory) is refused with its error before anything is enqueued.  Rows past counts_host[n] are unspecified. */
YFV2_API int yfv2_detect_u8_host(yfv2_plan* plan, const uint8_t* x_host, const void* packed,
                        const double* anchors_host, float conf_thres, double iou_thres, int max_det,
                        float* out_host, int* counts_host, void* workspace, void* stream);
YFV2_API size_t yfv2_detect_workspace_bytes(const yfv2_plan* plan, int max_det);

/* ---- compute_loss (utils/loss.py:130-208) with build_target (:53-124) and CIoU (:8-51) ---------------------------
 * preds: the six head tensors (as returned by yfv2_forward or by any other model), targets: device [nt,6] fp32 rows
 * (img_idx, cls, cx, cy, w, h) normalised; anchors_host as for yfv2_decode.  losses: device float[4] =
 * (lbox*3.2, lobj*64, lcls*32, sum) — the four values the reference returns.  dpreds (optional, may be NULL): six
 * tensors shaped like preds receiving d(loss)/d(preds) (what loss.backward() would put into the head tensors).
 * Asynchronous on `stream`; workspace from yfv2_loss_workspace_bytes. */
YFV2_API int yfv2_loss_workspace_bytes(int N, int H, int W, int A, int C, int nt, size_t* bytes);
YFV2_API int yfv2_compute_loss(const float* const preds[6], const float* targets, int nt, int N, int H, int W, int A, int C,
                               const double* anchors_host, float* losses, float* const dpreds[6], void* workspace,
                               void* stream);
/* test hook: copy out the matched rows of one pyramid level in the reference's order (offset type, anchor, target):
 * idx = device int32 [4][5*A*nt] rows (b, a, gj, gi), tbox device [.,4] fp32, anch device [.,2] fp64, tcls device int32.
 * Synchronises `stream` to return the row count. */
YFV2_API int yfv2_loss_read_targets(const void* workspace, int level, int N, int H, int W, int A, int nt, int* count_host,
                                    int* idx, float* tbox, double* anch, int* tcls, void* stream);

/* ---- training operators (train-mode forward with batch-statistics BatchNorm, and the backward of every op) --------
 * Dense NCHW fp32 device tensors; composed into the network by the Python mirror's autograd Functions
 * (yolo-fastestv2_b200/model/train_ops.py).  Reference: what autograd does for train.py:105-110.
 *   conv1x1:  y[n][m][p] = sum_k w[m][k] x[n][k][p] (+bias);  bwd outputs are optional (NULL to skip).
 *   dwconv:   depthwise ks x ks (3|5), stride 1|2, pad ks/2.   stem: dense 3x3 s2 p1 with 3 input channels.
 *   bn_train: batch statistics over (N, HW), running-stat update (momentum 0.1, unbiased var), optional fused ReLU;
 *             scratch = 2*C doubles; save_mean / save_invstd feed the backward.  bwd: dgamma / dbeta may be NULL (not written;
 *             the sums dx needs are still taken), as autograd skips the gradient of a BatchNorm affine with requires_grad=False.
 *   bn_eval:  a BatchNorm module in .eval() inside a train-mode network (F.batch_norm with training=False, eps 1e-5):
 *             y = [ReLU]((x - running_mean) * (running_var + eps)^-1/2 * gamma + beta); the running statistics are read, never
 *             updated.  fwd writes the mean / invstd it used to save_mean / save_invstd.  bwd: dx = g * gamma * invstd,
 *             dgamma = sum(g * xhat), dbeta = sum(g) (g = dy masked by y > 0 under ReLU; no batch-mean terms, the statistics
 *             are constants); each of dx, dgamma, dbeta may be NULL, not all three; scratch (2*C doubles) only with dgamma or dbeta.
 *   maxpool:  3x3 s2 p1 with argmax indices;  upsample2: nearest x2. */
YFV2_API int yfv2_op_conv1x1_fwd(const float* x, const float* w, const float* bias, float* y, int N, int K, int M, int HW, void* stream);
YFV2_API int yfv2_op_conv1x1_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, float* dbias, int N, int K, int M,
                                 int HW, void* stream);
YFV2_API int yfv2_op_dwconv_fwd(const float* x, const float* w, float* y, int N, int C, int H, int W, int ks, int stride, void* stream);
YFV2_API int yfv2_op_dwconv_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, int N, int C, int H, int W, int ks,
                                int stride, void* stream);
YFV2_API int yfv2_op_stem_fwd(const float* x, const float* w, float* y, int N, int M, int H, int W, void* stream);
YFV2_API int yfv2_op_stem_wgrad(const float* x, const float* dy, float* dw, int N, int M, int H, int W, void* stream);
YFV2_API int yfv2_op_bn_train_fwd(const float* x, const float* gamma, const float* beta, float* running_mean, float* running_var, float* y,
                                  float* save_mean, float* save_invstd, double* scratch, int N, int C, int HW, int relu, void* stream);
YFV2_API int yfv2_op_bn_train_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean,
                                  const float* save_invstd, float* dx, float* dgamma, float* dbeta, double* scratch, int N, int C, int HW,
                                  int relu, void* stream);
YFV2_API int yfv2_op_bn_eval_fwd(const float* x, const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                                 float* y, float* save_mean, float* save_invstd, int N, int C, int HW, int relu, void* stream);
YFV2_API int yfv2_op_bn_eval_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean,
                                 const float* save_invstd, float* dx, float* dgamma, float* dbeta, double* scratch, int N, int C, int HW,
                                 int relu, void* stream);
YFV2_API int yfv2_op_maxpool_fwd(const float* x, float* y, int* idx, int planes, int H, int W, void* stream);
YFV2_API int yfv2_op_maxpool_bwd(const float* dy, const int* idx, float* dx, int planes, int H, int W, void* stream);
YFV2_API int yfv2_op_upsample2_fwd(const float* x, float* y, int planes, int H, int W, void* stream);
YFV2_API int yfv2_op_upsample2_bwd(const float* dy, float* dx, int planes, int H, int W, void* stream);

/* ---- native training step: the train-mode forward and the backward of the WHOLE network as one call each ----------------
 * Replaces what nn.Module.train() + autograd do for the reference's train.py:105-110 over model/detector.py:21-31 (batch-statistics
 * BatchNorm incl. running-stat updates, ShuffleV2 shuffle / split / concat, FPN, heads, output convs).  Everything sits in a
 * caller-owned workspace laid out at create time (activations the backward needs, their gradients, scratch); no allocation per step.
 *   params[YFV2_NUM_PARAMS] / bn_running[2*YFV2_NUM_BN]: as yfv2_pack_weights (model.parameters() order; running_mean, running_var
 *     per BatchNorm layer — updated in place with momentum 0.1, num_batches_tracked is the caller's).
 *   x: fp32 [N,3,H,W].  preds[6]: the raw head tensors (written by forward; read again by backward).
 *   dpreds[6]: d(loss)/d(preds) (e.g. from yfv2_compute_loss).  grads_flat: ONE buffer of yfv2_trainer_grad_floats() floats holding
 *     every parameter's gradient at yfv2_trainer_param_offset(i) in parameter order (the bucket a data-parallel step all-reduces);
 *     accumulate != 0 adds to it (gradient accumulation over sub-batches, train.py:122-124), 0 overwrites.
 * yfv2_train_backward must follow the yfv2_train_forward of the same batch on the same workspace (and stream order).
 *
 * Fine-tuning mode (yfv2_trainer_set_mode; default: every parameter trainable, every BatchNorm layer in train mode):
 *   trainable[YFV2_NUM_PARAMS] (NULL: all 1): 0 for a parameter with requires_grad=False.  As autograd: it receives no gradient,
 *     and an op's backward runs only if its output depends on a trainable parameter (the image does not), writing d(input) only
 *     for an input that does; the backward below the lowest trainable layer is not run at all.
 *   bn_eval[YFV2_NUM_BN] (NULL: all 0): 1 for a BatchNorm module in .eval() (e.g. after model.backbone.eval()): it normalises with
 *     the running statistics and leaves them alone, as bn_eval above; its gamma / beta may still be trainable.
 *   The mode takes effect at the next yfv2_train_forward.  yfv2_train_backward refuses, before any launch, a mode changed since
 *   that forward and a mode with no trainable parameter (torch: "element 0 of tensors does not require grad").
 *   yfv2_trainer_grad_floats / yfv2_trainer_param_offset report the current mode's flat layout: the trainable parameters only,
 *   in parameter order (train_ddp.FlatGradBucket's layout); offset -1 for a frozen parameter. */
typedef struct yfv2_trainer yfv2_trainer;
YFV2_API int yfv2_trainer_create(yfv2_trainer** out, int device, int N, int H, int W, int A, int C);
YFV2_API void yfv2_trainer_destroy(yfv2_trainer* t);
YFV2_API int yfv2_trainer_workspace_bytes(const yfv2_trainer* t, size_t* bytes);
YFV2_API int yfv2_trainer_grad_floats(const yfv2_trainer* t, long long* n);
YFV2_API int yfv2_trainer_param_offset(const yfv2_trainer* t, int index, long long* offset, long long* numel);
YFV2_API int yfv2_trainer_set_mode(yfv2_trainer* t, const unsigned char* trainable, const unsigned char* bn_eval);
YFV2_API int yfv2_train_forward(yfv2_trainer* t, const float* x, const float* const* params, float* const* bn_running,
                                float* const preds[6], void* workspace, void* stream);
YFV2_API int yfv2_train_backward(yfv2_trainer* t, const float* x, const float* const* params, float* const preds[6],
                                 const float* const dpreds[6], float* grads_flat, int accumulate, void* workspace, void* stream);

/* ---- stage-granular forward (profiling / tests) ---------------------------------------------------------
 * A forward is a list of fused stages; yfv2_plan_stage_name(i) names them ("stem", "stage2.0", ...,
 * "stage4.1/pw1", "stage4.1/dwpw", "fpn.S3", "fpn.S2", "heads2.a", ...).  yfv2_forward_range runs stages
 * [first,last) (last < 0: to the end).  Consecutive stages with the same yfv2_plan_stage_group() value are ONE
 * kernel launch when the range covers them (chained stride-1 ShuffleV2 blocks, csrc/k_blk.cu); a range that cuts
 * a group runs the covered part as its own launch, so every block output can still be tapped.
 * yfv2_plan_forward_launches() counts the launches of a whole forward.  A block's output is only intact until a
 * later stage recycles its planes. */
YFV2_API const char* yfv2_plan_stage_name(const yfv2_plan* plan, int i);
YFV2_API int yfv2_plan_stage_group(const yfv2_plan* plan, int i);    /* index of the first stage of stage i's launch; -1: bad i */
YFV2_API int yfv2_forward_range(yfv2_plan* plan, const void* x, int is_u8, const void* packed, float* const preds[6],
                                void* workspace, int first, int last, void* stream);

/* ---- test hook: dense NCHW copy of an intermediate tensor of the last forward -------------------------
 * which: 0 stem output, 1..16 ShuffleV2 block outputs in network order (logical channel order, i.e. what
 * the reference's block returns), 17 S2, 18 S3, 19..22 mid-head scratch (cls2, reg2, cls3, reg3).
 * dims4 receives [N,C,h,w]; out may be NULL to query dims only. */
YFV2_API int yfv2_debug_gather(const yfv2_plan* plan, const void* workspace, int which, float* out, int* dims4,
                               void* stream);

/* ---- test hooks: the native trainer's program and where it keeps every tensor in the workspace -----------------------
 * Host only: nothing is launched and no device memory is read.  yfv2_trainer_debug_ops / _tensors write min(cap, count) records
 * and return the count in *n (cap 0 with a NULL array queries it).  An op reads tensors a (and b), writes tensor y:
 *   kind: 0 stem (3x3 s2 conv, weight pw), 1 BatchNorm train (+ReLU if relu; gamma pg, beta pb, layer bn; aux: workspace float
 *         offset of 2C doubles of fp64 sums, then mean[C] at aux + 4C and invstd[C] at aux + 5C), 2 max-pool 3x3 s2 p1 (aux: int32
 *         argmax per output element), 3 1x1 conv (M outputs, weight pw, bias pbias), 4 depthwise conv (ks, stride, weight pw),
 *         5 nearest 2x up-sampling, 6 odd channels of a, 7 [even channels of a | b], 8 [a | b] (channel concat).
 *   Parameter indices are model.parameters() positions, -1 where the op has none; aux is -1 for kinds without private storage.
 * A tensor's activation and gradient are dense NCHW [N, C, H, W] at workspace float offsets off / goff; ext >= 0 marks head tensor
 * `ext` (the caller's preds / dpreds, off = goff = -1) and ext = -2 the input image.
 * layout_host[8] receives, in floats: workspace size, then the offset of the fan-in gradient scratch, the offset and size of the
 * parameter-gradient scratch (a shared layer's second use), the offset and size of the flat gradient slot, the offset and size of
 * the per-block weight-gradient partials. */
typedef struct yfv2_trainer_op {
    int kind;
    int a, b, y;                 /* tensor ids (b = -1 for one-input ops) */
    int pw, pg, pb, pbias, bn;
    int relu, ks, stride, M;
    long long aux;
} yfv2_trainer_op;
typedef struct yfv2_trainer_tensor {
    long long off, goff;
    int C, H, W;
    int ext;
} yfv2_trainer_tensor;
YFV2_API int yfv2_trainer_debug_ops(const yfv2_trainer* t, yfv2_trainer_op* ops_host, int cap, int* n);
YFV2_API int yfv2_trainer_debug_tensors(const yfv2_trainer* t, yfv2_trainer_tensor* tens_host, int cap, int* n);
YFV2_API int yfv2_trainer_debug_layout(const yfv2_trainer* t, long long* layout_host);
/* Host only, for the current mode: the ops whose backward runs, in the order it runs them (op = index into yfv2_trainer_debug_ops),
 * and which outputs each writes: da / db the gradient of input a / b, dw, dbias, dgamma, dbeta the parameter gradients; bn_eval 1
 * for a BatchNorm run by the eval-mode kernels.  (A train-mode BatchNorm with da = 0 still computes a dx nobody reads, into its
 * input's own gradient slot.)  Writes min(cap, count) records, the count in *n. */
typedef struct yfv2_trainer_bwd_op {
    int op;
    int da, db, dw, dbias, dgamma, dbeta, bn_eval;
} yfv2_trainer_bwd_op;
YFV2_API int yfv2_trainer_debug_backward(const yfv2_trainer* t, yfv2_trainer_bwd_op* ops_host, int cap, int* n);

/* ---- test hook: the kernel launches of a whole forward, as the forward itself chooses them ----------------------------------
 * Host only: nothing is launched and workspace is not dereferenced; its address decides the kernels that need 16-byte-aligned
 * planes (NULL: a 16-byte-aligned workspace).  is_u8: a uint8 input; sms: the GPU's multiprocessors (0: this device's count, 132
 * without a device).  Writes min(cap, count) records and returns the count in *n (cap 0 with a NULL array queries it); an argument
 * the forward would refuse is refused here with the same code and message.
 *   kernel:   the demangled name after yfv2::(anonymous namespace)::, without spaces ("walk::blk_kernel<24,2>", "head2_kernel")
 *   grid:     fixed grid; persistent: grid[0] is the SM count, and the launch runs min(items, CTAs per SM by occupancy x grid[0])
 *             CTAs that walk the items
 *   R, bands: block launches: rows per band, bands per image (items = N x bands); G: the step of walk::blk_kernel<K,1>, 0 elsewhere
 *   window_stride: heads: channel stride (floats) of a staged 5x5 window slot; 0: the stencils read the planes */
typedef struct yfv2_launch {
    char kernel[32];
    int first, last;             /* fused stages [first, last) (yfv2_plan_stage_name) */
    long long smem;              /* dynamic shared memory, bytes */
    int grid[3];
    int persistent;
    int items;
    int R, bands, G;
    int window_stride;
} yfv2_launch;
YFV2_API int yfv2_plan_debug_launches(const yfv2_plan* plan, const void* workspace, int is_u8, int sms, yfv2_launch* out, int cap,
                                      int* n);

/* ---- test hook: one pointwise contraction on the tensor-core engine (3xTF32), out[n][p] = sum_k w[n][k]*x[k][p] ----
 * x: [K][P], w: [N][K], out: [N][P], pack_ws: unused (kept for ABI stability), may be NULL. */
YFV2_API int yfv2_debug_pw_tc(const float* x, const float* w, float* out, float* pack_ws, int K, int N, int P,
                              void* stream);

/* ---- profiling hook: yfv2_decode_nms runs an instrumented kernel while dev_buf != NULL and writes, per image, 16 int64:
 * clock64 ticks of [0] candidate generation, [1] sort, [2] staging of the first chunk, [3] chunk vs kept, [4] pairs inside the
 * chunk, [5] resolve + append, [6] unused, [7] tail; [8] chunks, [9] candidates, [10] kept.  dev_buf: N x 16 int64 on the device. */
YFV2_API int yfv2_debug_nms_profile(long long* dev_buf);

#ifdef __cplusplus
}
#endif
#endif /* YFV2_H_ */
