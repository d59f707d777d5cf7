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
 * max_out = A*(H/16*W/16 + H/32*W/32) to never truncate).  Equal scores keep push order (the sample's std::sort leaves it open). */
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

/* ---- get_batch_statistics (utils/utils.py:184-230): true-positive flags of NMS output rows ----------------
 * dets [N,max_det,6] / counts [N] as yfv2_nms writes them; targets [nt,6] rows (image, class, x1, y1, x2, y2) in
 * pixels (what evaluation() builds at utils/utils.py:372-375), nt <= 8192.  tp [N,max_det] receives 1.0 for a true
 * positive, 0.0 otherwise (rows past counts[n] are 0).  Same greedy order and the same fp32 IoU (+1 convention) as the
 * reference: bit-identical flags. */
YFV2_API int yfv2_batch_statistics(const float* dets, const int* counts, int N, int max_det, const float* targets, int nt,
                                   float iou_threshold, float* tp, void* stream);

/* ---- contrast_and_brightness (utils/datasets.py:10-16; the augmentation img_aug applies, :63-68) on the device ----
 * out = cv2.addWeighted(img, alpha[n], zeros, 1 - alpha[n], beta[n]) for uint8 images: per byte
 * saturate_cast<uint8>(cvRound(fl32(fl32(x * alpha) + beta))).  img / out: N images of bytes_per_image bytes each (any
 * layout: the operation is elementwise; in place allowed); alpha / beta: device arrays [N] (the reference draws both from
 * random.uniform(0.25, 1.75) per image on the host).  Bit-identical to OpenCV 4.x. */
YFV2_API int yfv2_aug_contrast_brightness(const uint8_t* img, uint8_t* out, const float* alpha, const float* beta, int N,
                                          long long bytes_per_image, void* stream);

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

/* ---- whole inference step with HOST buffers (the evaluation() inner loop, utils/utils.py:367-383) ----
 * x_host: pinned uint8 [N,3,H,W]; out_host: pinned [N,max_det,6]; counts_host: pinned [N].
 * Copies in, runs forward_u8 + decode_nms, copies out, all on `stream`; returns without synchronising. */
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
 *             scratch = 2*C doubles; save_mean / save_invstd feed the backward.
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
 * yfv2_train_backward must follow the yfv2_train_forward of the same batch on the same workspace (and stream order). */
typedef struct yfv2_trainer yfv2_trainer;
YFV2_API int yfv2_trainer_create(yfv2_trainer** out, int device, int N, int H, int W, int A, int C);
YFV2_API void yfv2_trainer_destroy(yfv2_trainer* t);
YFV2_API int yfv2_trainer_workspace_bytes(const yfv2_trainer* t, size_t* bytes);
YFV2_API int yfv2_trainer_grad_floats(const yfv2_trainer* t, long long* n);
YFV2_API int yfv2_trainer_param_offset(const yfv2_trainer* t, int index, long long* offset, long long* numel);
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

/* ---- test hook: how a head launch of a forward on `workspace` reads its 5x5 depthwise taps ------------------------------
 * which: 0 heads2.a, 1 heads2.b, 2 heads3.a, 3 heads3.b.  Returns 1 when the launch stages the input windows in shared memory,
 * 0 when it reads the planes, < 0 on a bad argument (workspace NULL included: the choice depends on the plane addresses).
 * Host only: workspace is not dereferenced. */
YFV2_API int yfv2_debug_heads_staged(const yfv2_plan* plan, const void* workspace, int which);

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
