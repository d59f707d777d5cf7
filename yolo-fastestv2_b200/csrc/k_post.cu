// K6 / K7 — anchor-grid decode and per-image NMS, plus the fused decode+NMS that never writes the
// [N, M, 5+C] candidate tensor.
//
//   decode  <- reference utils/utils.py:298-358  (make_grid + handel_preds)
//   nms     <- reference utils/utils.py:67-74,232-296 (xywh2xyxy + non_max_suppression) and the greedy
//              kernel of torchvision.ops.nms that it calls at :286.
//
// Bit-exactness contract (tests/test_post_gpu.py): given identical [N,M,5+C] inputs the kept rows and
// indices equal the reference's bit for bit.  That needs: fp32 products obj*cls with first-max argmax,
// strict '>' filters, box = xy -/+ wh/2, class offset cls*4096 added in fp32, IoU = inter/(a+b-inter)
// in fp32 compared as double against the threshold, stable descending order (ties by original row),
// and no FMA contraction anywhere in that arithmetic — every step uses the __f*_rn intrinsics.
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <new>

#include "common.cuh"
#include "nms.cuh"

namespace yfv2 {
namespace {

constexpr int kCPL = 8;              // classes per lane -> C <= 256
constexpr int kChunkCells = 32;
constexpr int kSStride = kChunkCells + 1;
constexpr int kNmsListMinDet = 513;    // per-class kept lists pay off only for long kept lists (see sort_and_suppress)
constexpr int kNmsListClasses = 256;   // per-class kept lists (heads + class histogram) for up to this many classes

struct PostGeom {
    int N, A, C, D, M;               // D = 5+C, M = rows per image
    int h[2], w[2], hw[2];
    float stride[2];
    double anc[2][kMaxA][2];
    const float* reg[2];
    const float* obj[2];
    const float* cls[2];
};

__device__ __forceinline__ float sigmoid_rn(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// (value, index) argmax, ties -> smaller index; every lane ends with the same pair
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
}

// Stage the 5A+C logits of `ncell` consecutive cells of one level into S[ch][kSStride] (coalesced reads).
__device__ __forceinline__ void stage_cells(float* __restrict__ S, const PostGeom& g, int n, int lv, int cell0, int ncell) {
    const int A = g.A, C = g.C, hw = g.hw[lv];
    const int nch = 5 * A + C;
    for (int i = threadIdx.x; i < nch * kChunkCells; i += NT) {
        const int ch = i >> 5, cl = i & 31;
        if (cl < ncell) {
            const float* src;
            if (ch < 4 * A) src = g.reg[lv] + ((long long)n * 4 * A + ch) * hw;
            else if (ch < 5 * A) src = g.obj[lv] + ((long long)n * A + (ch - 4 * A)) * hw;
            else src = g.cls[lv] + ((long long)n * C + (ch - 5 * A)) * hw;
            S[ch * kSStride + cl] = __ldg(src + cell0 + cl);
        }
    }
}

// Chunk blockIdx.x of image blockIdx.y, for grids of (chunks of level 0, then chunks of level 1; N): its cells staged into S.
struct Chunk {
    int n, lv, cell0, ncell;
};
__device__ __forceinline__ Chunk stage_chunk(float* __restrict__ S, const PostGeom& g, int chunks0) {
    Chunk k;
    k.n = blockIdx.y;
    k.lv = blockIdx.x < chunks0 ? 0 : 1;
    k.cell0 = (k.lv ? blockIdx.x - chunks0 : blockIdx.x) * kChunkCells;
    k.ncell = min(kChunkCells, g.hw[k.lv] - k.cell0);
    stage_cells(S, g, k.n, k.lv, k.cell0, k.ncell);
    __syncthreads();
    return k;
}

// Box of one (cell, anchor) from its four box logits, utils/utils.py:331-343: xy = (sigmoid*2 - 0.5 + grid) * stride, and
// (sigmoid*2)**2 in fp32, which the float64 anchor then promotes (utils/utils.py:305-306,337).  Returns (cx, cy, w, h).
__device__ __forceinline__ float4 decode_box(float lx, float ly, float lw, float lh, int x, int y, float st, double aw, double ah) {
    const float sx = sigmoid_rn(lx), sy = sigmoid_rn(ly), sw = sigmoid_rn(lw), sh = sigmoid_rn(lh);
    const float tw = __fmul_rn(sw, 2.0f), th = __fmul_rn(sh, 2.0f);
    return make_float4(__fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sx, 2.0f), 0.5f), (float)x), st),
                       __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sy, 2.0f), 0.5f), (float)y), st),
                       (float)__dmul_rn((double)__fmul_rn(tw, tw), aw), (float)__dmul_rn((double)__fmul_rn(th, th), ah));
}

// Softmax over the C class logits of staged cell cl (utils/utils.py:326, model/detector.py:40); lane l gets classes l, l+32, ...
// (0 past C).
__device__ __forceinline__ void warp_softmax(const float* __restrict__ S, int A, int C, int cl, int lane, float (&pr)[kCPL]) {
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < kCPL; ++j) {
        const int c = lane + 32 * j;
        pr[j] = (c < C) ? S[(5 * A + c) * kSStride + cl] : -INFINITY;
        m = fmaxf(m, pr[j]);
    }
    m = warp_max(m);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kCPL; ++j) {
        const int c = lane + 32 * j;
        pr[j] = (c < C) ? expf(__fsub_rn(pr[j], m)) : 0.f;
        sum = __fadd_rn(sum, pr[j]);
    }
    sum = warp_sum(sum);
#pragma unroll
    for (int j = 0; j < kCPL; ++j) pr[j] = __fdiv_rn(pr[j], sum);
}

// One warp decodes one staged cell.  Lane l keeps softmax probabilities of classes l, l+32, ...;
// lanes a < A additionally keep the box (cx, cy, w, h) and objectness of anchor a.
struct CellRegs {
    float p[kCPL];
    float4 box;
    float ob;
};
__device__ __forceinline__ void decode_cell(const float* __restrict__ S, const PostGeom& g, int lv, int cell, int cl,
                                            int lane, CellRegs& r) {
    const int A = g.A;
    warp_softmax(S, A, g.C, cl, lane, r.p);
    r.box = make_float4(0.f, 0.f, 0.f, 0.f);
    r.ob = 0.f;
    if (lane < A) {
        const int y = cell / g.w[lv], x = cell - y * g.w[lv];
        const float* s = S + (4 * lane) * kSStride + cl;
        r.box = decode_box(s[0], s[kSStride], s[2 * kSStride], s[3 * kSStride], x, y, g.stride[lv], g.anc[lv][lane][0],
                           g.anc[lv][lane][1]);
        r.ob = sigmoid_rn(S[(4 * A + lane) * kSStride + cl]);
    }
}

// ---------------------------------------------------------------------------------------------------
// decode kernel: grid (chunks per image, N)
__global__ void __launch_bounds__(NT)
decode_kernel(PostGeom g, float* __restrict__ out, int chunks0) {
    __shared__ float S[(5 * kMaxA + 32 * kCPL) * kSStride];
    const Chunk k = stage_chunk(S, g, chunks0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int A = g.A, C = g.C, D = g.D;
    const long long row_base = (long long)k.n * g.M + (k.lv ? (long long)g.hw[0] * A : 0);
    for (int cl = warp; cl < k.ncell; cl += NT / 32) {
        CellRegs r;
        decode_cell(S, g, k.lv, k.cell0 + cl, cl, lane, r);
        float* o = out + (row_base + (long long)(k.cell0 + cl) * A) * D;
        if (lane < A) {
            float* b = o + (long long)lane * D;
            b[0] = r.box.x; b[1] = r.box.y; b[2] = r.box.z; b[3] = r.box.w; b[4] = r.ob;
        }
        for (int a = 0; a < A; ++a)
#pragma unroll
            for (int j = 0; j < kCPL; ++j) {
                const int c = lane + 32 * j;
                if (c < C) o[(long long)a * D + 5 + c] = r.p[j];       // same cls row for every anchor (:326)
            }
    }
}

// ---------------------------------------------------------------------------------------------------
// export_onnx head (reference model/detector.py:33-44): sigmoid(reg) | sigmoid(obj) | softmax(cls) concatenated channel-last,
// one [N,h,w,5A+C] tensor per level — the wire format the ncnn sample consumes.  grid (chunks per image, N).
__global__ void __launch_bounds__(NT)
export_head_kernel(PostGeom g, float* __restrict__ out2, float* __restrict__ out3, int chunks0) {
    __shared__ float S[(5 * kMaxA + 32 * kCPL) * kSStride];
    const Chunk k = stage_chunk(S, g, chunks0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int A = g.A, C = g.C, D = 5 * A + C;
    float* out = k.lv ? out3 : out2;
    for (int cl = warp; cl < k.ncell; cl += NT / 32) {
        float* o = out + ((long long)k.n * g.hw[k.lv] + k.cell0 + cl) * D;
        for (int ch = lane; ch < 5 * A; ch += 32) o[ch] = sigmoid_rn(S[ch * kSStride + cl]);
        float pr[kCPL];
        warp_softmax(S, A, C, cl, lane, pr);
#pragma unroll
        for (int j = 0; j < kCPL; ++j) {
            const int c = lane + 32 * j;
            if (c < C) o[5 * A + c] = pr[j];
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// NMS
struct NmsParams {
    float conf_thres;
    double iou_thres;
    double iou_mid;    // fl32(q) > iou_thres  <=>  q > iou_mid (or >= when iou_tie_up), see iou_gt()
    float iou_mid_f;   // (float)iou_mid: a 1e-6-wide fp32 pre-test decides almost every pair without the fp64 product
    float iou_fast_mid;  // iou_fast(): iou_mid_f, or NaN when iou_mid <= 0 (every pair then takes the exact path)
    float iou_zero;      // iou_fast(): 0 (an empty intersection is below a positive threshold), or NaN when iou_mid <= 0
    int iou_tie_up;
    const int* class_filter;
    int n_filter;
    int max_det;
    float max_wh;
    float* out;        // [N,max_det,6]
    int* counts;       // [N]
    int* kept_idx;     // [N,max_det] or null
    int M;             // candidate rows per image
    int MCp;           // pow2 >= M
    int C;             // classes (per-class kept lists need C <= kNmsListClasses)
    long long* prof;   // yfv2_debug_nms_profile: per image 16 x int64 (clock64 ticks per phase), else null
};

struct NmsSmem {
    unsigned long long* keys;   // [MCp]
    float4* cbox;               // [M]  xyxy, not offset
    unsigned short* ccls;       // [M]
    float4* kbox;               // [max_det] offset boxes of kept
    float* karea;               // [max_det]
    float4* chbox;              // [2][64]  double buffered: chunk c in buffer c & 1
    float* charea;              // [2][64]
    unsigned int* cmask;        // [64][2]  kill rows of the chunk's candidates
    unsigned char* alist;       // [64]     chunk indices of the candidates alive after (a), in order
    // per-class kept lists: they live in the padding tail of `keys` (entries [M, MCp) are zeros once the sort is done) and in
    // `kbox` before the first box is kept, so they cost no shared memory (one more CTA per SM matters to the scoring pass)
    unsigned int* kcn;          // [max_det] low 16 bits: class of kept box, high 16: next kept box of that class (0xFFFF: end)
    unsigned short* khead;      // [kNmsListClasses] newest kept box per class
    unsigned short* chcls;      // [2][64] classes of the staged chunks (own storage: the padding tail of `keys` only has room for the lists)
    unsigned int* chist;        // [kNmsListClasses] candidates per class (aliases kbox; only used before the suppression loop)
    bool lists_fit;
    struct Misc {
        unsigned int count;         // candidates pushed
        unsigned int dead[2];       // chunk candidates suppressed by a kept box, phase (a)
        unsigned int kept[2];       // chunk candidates kept, phase (c)
        unsigned int outside;       // some box outside (-max_wh/2, max_wh/2)
        unsigned int majority;      // some class holds more than half of the candidates
        unsigned int unused;
    }* misc;
};

// The shared memory of one NMS CTA, laid out from `base` (16-byte aligned).  Returns the end of the layout.
__host__ __device__ __forceinline__ unsigned char* nms_layout(NmsSmem& s, unsigned char* base, int M, int MCp, int max_det) {
    s.keys = take<unsigned long long>(base, MCp);
    s.cbox = take<float4>(base, M);
    s.ccls = take<unsigned short>(base, M);
    s.kbox = take<float4>(base, max_det);
    s.karea = take<float>(base, max_det);
    s.chbox = take<float4>(base, 2 * kChunk);
    s.charea = take<float>(base, 2 * kChunk);
    s.cmask = take<unsigned int>(base, 2 * kChunk);
    s.alist = take<unsigned char>(base, kChunk);
    s.chcls = take<unsigned short>(base, 2 * kChunk);
    s.misc = take<NmsSmem::Misc>(base, 1);
    unsigned char* tail = reinterpret_cast<unsigned char*>(s.keys + M);
    s.kcn = reinterpret_cast<unsigned int*>(tail); tail += (size_t)max_det * 4;
    s.khead = reinterpret_cast<unsigned short*>(tail); tail += kNmsListClasses * 2;
    s.lists_fit = tail <= reinterpret_cast<unsigned char*>(s.keys + MCp) && (size_t)max_det * 16 >= kNmsListClasses * 4;
    s.chist = reinterpret_cast<unsigned int*>(s.kbox);
    return base;
}

inline size_t nms_smem_bytes(int M, int MCp, int max_det) {
    NmsSmem s;
    return reinterpret_cast<size_t>(nms_layout(s, nullptr, M, MCp, max_det));
}

__device__ __forceinline__ bool class_ok(const NmsParams& p, int cls) {
    if (!p.class_filter) return true;
    bool ok = false;
    for (int k = 0; k < p.n_filter; ++k) ok |= (p.class_filter[k] == cls);
    return ok;
}

// xywh -> xyxy (utils/utils.py:67-74) and store candidate `slot`; called by the lane that owns the candidate.
// Also records whether every box of the image lies inside (-max_wh/2, max_wh/2): then the class offsets of utils/utils.py:283 put
// the classes on disjoint intervals, boxes of different classes can never intersect (their fp32 intersection width is exactly 0,
// rounding is monotone) and the suppression phases may skip such pairs by comparing class ids — bit-identical to testing them.
__device__ __forceinline__ void write_candidate(const NmsSmem& s, unsigned int slot, float cx, float cy, float w, float h, float conf,
                                                int cls, int row, float max_wh) {
    const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);
    const float4 bb = make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
    const float lim = 0.5f * max_wh;
    if (!(fabsf(bb.x) < lim && fabsf(bb.y) < lim && fabsf(bb.z) < lim && fabsf(bb.w) < lim)) s.misc->outside = 1u;    // (NaN lands here too)
    s.cbox[slot] = bb;
    s.ccls[slot] = (unsigned short)cls;
    s.keys[slot] = ((unsigned long long)f2sortable(conf) << 32) |
                   ((unsigned long long)(0xFFFFu - (unsigned)row) << 16) | (unsigned long long)slot;
}
// Warp-aggregated slot allocation: one shared-memory atomic per warp call instead of one per candidate.  All 32 lanes call.
__device__ __forceinline__ unsigned int alloc_slots(unsigned int* count, bool want) {
    const unsigned int bal = __ballot_sync(0xffffffffu, want);
    unsigned int base = 0;
    if ((threadIdx.x & 31) == 0 && bal) base = atomicAdd(count, (unsigned int)__popc(bal));
    base = __shfl_sync(0xffffffffu, base, 0);
    return base + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u));
}

// torchvision: ovr = inter / (a_i + a_j - inter) in fp32, suppressed iff (double)ovr > thr.  The fp32 quotient exceeds thr
// iff the real quotient lies beyond the rounding boundary `mid` between the two floats that bracket thr, so for a positive
// finite denominator the test is inter > mid*u (>= when the tie rounds up) — both sides exact in fp64 (24-bit x 25-bit
// product) — and the IEEE division subroutine is only needed for degenerate denominators.  Bit-exact by construction.
__device__ __forceinline__ bool iou_gt(const float4& a, float aa, const float4& b, float ab, const NmsParams& p) {
    const float w = fmaxf(0.f, __fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)));
    const float h = fmaxf(0.f, __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)));
    const float inter = __fmul_rn(w, h);
    // disjoint boxes (nearly every pair: other classes sit max_wh apart): IoU is 0, -0 or NaN, never above a threshold whose
    // midpoint is positive -- same answer as the code below without its fp64 work
    if (inter == 0.f && p.iou_mid > 0.0) return false;
    const float u = __fsub_rn(__fadd_rn(aa, ab), inter);
    if (u > 0.f && u < 3.0e38f && inter < 3.0e38f) {
        // fp32 estimate of mid*u: off by at most 2^-23 relative (rounding of mid and of the product); outside a 1e-6 band around
        // it the exact comparison below cannot come out differently
        const float tq = __fmul_rn(p.iou_mid_f, u);
        if (tq > 1.0e-30f) {
            if (inter > __fmul_rn(tq, 1.000001f)) return true;
            if (inter < __fmul_rn(tq, 0.999999f)) return false;
        }
        const double lhs = (double)inter, rhs = __dmul_rn(p.iou_mid, (double)u);
        return p.iou_tie_up ? lhs >= rhs : lhs > rhs;
    }
    return (double)__fdiv_rn(inter, u) > p.iou_thres;
}

// Branch-free front of iou_gt for the two suppression passes (ncu, round 2: the five early-outs of iou_gt serialised the four
// "independent" tests of an unrolled trip: 35 issued instructions and 5 branch bubbles per test, 27 % of the kernel's stall
// samples were `wait` behind those branches).  `res` is iou_gt's answer whenever `amb` is false: the fp32 estimate of mid*u is
// off by at most 2^-23 relative, so outside a 1e-6 band around it the exact fp64 comparison cannot come out differently, and an
// exactly empty intersection never exceeds a positive threshold; everything else (the band, zero / huge / NaN operands, a
// non-positive threshold, for which the host sets iou_mid_f = NaN) is `amb` and goes through iou_gt itself.
__device__ __forceinline__ void iou_fast(const float4& a, float aa, const float4& b, float ab, const NmsParams& p, bool& res, bool& amb) {
    const float w = fmaxf(0.f, __fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)));
    const float h = fmaxf(0.f, __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)));
    const float inter = __fmul_rn(w, h);
    const float u = __fsub_rn(__fadd_rn(aa, ab), inter);
    const float tq = __fmul_rn(p.iou_fast_mid, u);
    const bool sane = (tq > 1.0e-30f) & (fmaxf(u, inter) < 3.0e38f);            // false for NaN operands too
    const bool above = inter > __fmul_rn(tq, 1.000001f), below = inter < __fmul_rn(tq, 0.999999f);
    res = above & sane;
    amb = !(((above | below) & sane) | (inter == p.iou_zero));                    // iou_zero: 0, or NaN when the threshold is not positive
}

// Sort the pushed candidates and run the blocked greedy suppression.  All threads of the CTA call this.
// PROF (debug builds of the kernels, yfv2_debug_nms_profile): thread 0 accumulates clock64 ticks per phase; `tstart` is the
// kernel's first timestamp.  Phases: 0 candidate generation, 1 class histogram + sort, 2 staging of the first chunk, 3 chunk vs
// kept, 4 ranking + pairs inside the chunk, 5 resolve + append (+ staging of the next chunk), 6 unused, 7 tail; [8] chunks,
// [9] candidates, [10] kept.
template <bool PROF>
__device__ void sort_and_suppress(const NmsSmem& s, const NmsParams& p, int n, long long tstart = 0) {
    long long acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tlast = tstart;
    int nchunks = 0;
    auto tick = [&](int k) {
        if (PROF && threadIdx.x == 0) { const long long tn = clock64(); acc[k] += tn - tlast; tlast = tn; }
    };
    __syncthreads();
    tick(0);
    const int cnt = (int)s.misc->count;
    // classes on disjoint intervals (see write_candidate) and a threshold whose rounding boundary is positive: pairs of different
    // classes have IoU exactly 0 and are skipped on their class ids
    // ... worth it only when the candidates are spread over classes: every kept box then sits in a per-class list (newest first)
    // and a candidate walks its own class's list instead of all kept boxes.  A single dominant class (randomly initialised
    // heads: every candidate has the same arg-max) keeps the dense 4-way unrolled scan.
    // (since the dense scan went branch-free it is the faster one while the kept list is short -- configs[4] sets, cap 300: 2.9 / 2.5 ms
    // per 10 000 images against 3.4 / 2.9 with the lists -- so the lists are only used for caps above kNmsListMinDet)
    bool by_class = s.lists_fit && s.misc->outside == 0u && p.iou_mid > 0.0 && p.max_wh > 0.f && p.C <= kNmsListClasses &&
                    p.max_det >= kNmsListMinDet;
    if (by_class) {
        for (int i = threadIdx.x; i < kNmsListClasses; i += NT) s.chist[i] = 0u;
        if (threadIdx.x == 0) s.misc->majority = 0u;
        __syncthreads();
        for (int i = threadIdx.x; i < cnt; i += NT) atomicAdd(&s.chist[s.ccls[i]], 1u);
        __syncthreads();
        for (int i = threadIdx.x; i < kNmsListClasses; i += NT) if (2u * s.chist[i] > (unsigned)cnt) s.misc->majority = 1u;
        __syncthreads();
        by_class = s.misc->majority == 0u;
    }
    const int n2 = pow2_at_least(cnt);
    for (int i = cnt + threadIdx.x; i < n2; i += NT) s.keys[i] = 0ull;
    __syncthreads();
    if (n2 == NT) bitonic_sort_desc_reg<1>(s.keys);
    else if (n2 == 2 * NT) bitonic_sort_desc_reg<2>(s.keys);
    else if (n2 == 4 * NT) bitonic_sort_desc_reg<4>(s.keys);
    else if (n2 == 8 * NT) bitonic_sort_desc_reg<8>(s.keys);
    else bitonic_sort_desc(s.keys, n2);
    if (by_class) {                                          // the padding tail of `keys` is free from here on
        for (int i = threadIdx.x; i < kNmsListClasses; i += NT) s.khead[i] = 0xFFFFu;
        __syncthreads();
    }
    tick(1);

    float* out = p.out + (long long)n * p.max_det * 6;
    int* kidx = p.kept_idx ? p.kept_idx + (long long)n * p.max_det : nullptr;
    int nk = 0;
    const int t = threadIdx.x;
    // Chunk c of 64 sorted candidates is staged (offset boxes, areas, classes) into buffer c & 1 while chunk c - 1 is being resolved.
    // Per chunk: (a) the chunk against everything kept so far -> dead bits; (b) pairs among the survivors -> kill rows; (c) greedy
    // resolve over the rows + (d) append.  Round-2 profile of the first version of this loop (a 64x64 pair matrix on all threads with
    // 16 branchy tests each, a one-thread resolve over 64-bit masks, separate load and append phases, five barriers), per image:
    // pair matrix 37 us, resolve 26 us, load + append 7 us of 146 -- most rows of the matrix belonged to candidates (a) had already
    // killed, and 255 threads waited on the resolve.  (Tried and dropped: resolving inside one warp with the IoU tests on the chain,
    // one or four picks per trip: 185 / 209 us per launch against 203 before.)
    auto stage = [&](int c0, int buf, int j) {               // candidate j of the chunk starting at sorted position c0
        if (c0 + j < cnt) {
            const unsigned int slot = (unsigned int)(s.keys[c0 + j] & 0xFFFFull);
            const float4 b = s.cbox[slot];
            const float off = __fmul_rn((float)s.ccls[slot], p.max_wh);            // utils/utils.py:283
            const float4 ob = make_float4(__fadd_rn(b.x, off), __fadd_rn(b.y, off), __fadd_rn(b.z, off), __fadd_rn(b.w, off));
            s.chbox[buf * kChunk + j] = ob;
            s.charea[buf * kChunk + j] = __fmul_rn(__fsub_rn(ob.z, ob.x), __fsub_rn(ob.w, ob.y));
            if (by_class) s.chcls[buf * kChunk + j] = s.ccls[slot];
        }
    };
    if (t < kChunk) stage(0, 0, t);
    if (t == 0) { s.misc->dead[0] = 0u; s.misc->dead[1] = 0u; }
    __syncthreads();
    tick(2);
    for (int c0 = 0, it = 0; c0 < cnt && nk < p.max_det; c0 += kChunk, ++it) {
        const int cn = min(kChunk, cnt - c0);
        const float4* chbox = s.chbox + (it & 1) * kChunk;
        const float* charea = s.charea + (it & 1) * kChunk;
        const unsigned short* chcls = s.chcls + (it & 1) * kChunk;
        ++nchunks;
        {   // (a) chunk candidates against everything kept so far
            const int j = t & (kChunk - 1), q = t / kChunk;
            if (j < cn && by_class) {
                // walk the kept boxes of this candidate's class; the candidate's four threads test every fourth node
                const float4 bj = chbox[j];
                const float aj = charea[j];
                bool dead = false;
                int k = 0;
                for (unsigned i = s.khead[chcls[j]]; i != 0xFFFFu && !dead; i = s.kcn[i] >> 16, ++k)
                    if ((k & (NT / kChunk - 1)) == q) dead = iou_gt(s.kbox[i], s.karea[i], bj, aj, p);
                if (dead) atomicOr(&s.misc->dead[j >> 5], 1u << (j & 31));
            } else if (j < cn) {
                const float4 bj = chbox[j];
                const float aj = charea[j];
                // four kept boxes per trip: the loads and IoU fronts are independent, only the exit test is shared
                bool dead = false;
                constexpr int STEP = NT / kChunk;
                int i = q;
                for (; i + 3 * STEP < nk && !dead; i += 4 * STEP) {
                    bool d[4], m[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) iou_fast(s.kbox[i + u * STEP], s.karea[i + u * STEP], bj, aj, p, d[u], m[u]);
                    if (m[0] | m[1] | m[2] | m[3]) {                           // rare: some pair sits in the 1e-6 band / is degenerate
#pragma unroll
                        for (int u = 0; u < 4; ++u)
                            d[u] = iou_gt(s.kbox[i + u * STEP], s.karea[i + u * STEP], bj, aj, p);
                    }
                    dead = d[0] | d[1] | d[2] | d[3];
                }
                for (; i < nk && !dead; i += STEP) dead = iou_gt(s.kbox[i], s.karea[i], bj, aj, p);
                if (dead) atomicOr(&s.misc->dead[j >> 5], 1u << (j & 31));
            }
        }
        __syncthreads();
        tick(3);
        // (b) pairs INSIDE the chunk, only among the candidates (a) left alive (typically ~20 of 64 in a crowded class): the live
        // candidates are ranked (alist), thread <-> ordered pair of ranks, one IoU test per thread and round, hits OR-ed into the
        // 64-bit kill row of the earlier candidate.  Threads 64..127 meanwhile stage the next chunk into the other buffer.
        unsigned long long alive = ~(((unsigned long long)s.misc->dead[1] << 32) | s.misc->dead[0]);
        if (cn < 64) alive &= (1ull << cn) - 1ull;
        const int na = __popcll(alive);
        if (t < kChunk) {
            s.cmask[2 * t] = 0u; s.cmask[2 * t + 1] = 0u;
            if ((alive >> t) & 1ull) s.alist[__popcll(alive & ((1ull << t) - 1ull))] = (unsigned char)t;
        } else if (t < 2 * kChunk) {
            stage(c0 + kChunk, (it + 1) & 1, t - kChunk);       // (nothing to do past the end)
        }
        __syncthreads();
        if (t == 0) { s.misc->dead[0] = 0u; s.misc->dead[1] = 0u; }  // every thread has read the dead bits
        if (na * na <= 4 * NT) {
            for (int pi = t; pi < na * na; pi += NT) {
                const int rx = pi / na, ry = pi - rx * na;
                if (ry > rx) {
                    const int x = s.alist[rx], y = s.alist[ry];       // x earlier (higher confidence) than y
                    if (!by_class || chcls[x] == chcls[y]) {
                        bool d, m;
                        iou_fast(chbox[x], charea[x], chbox[y], charea[y], p, d, m);
                        if (m) d = iou_gt(chbox[x], charea[x], chbox[y], charea[y], p);
                        if (d) atomicOr(&s.cmask[2 * x + (y >> 5)], 1u << (y & 31));
                    }
                }
            }
        } else {
            // most of the chunk survived (a) (candidates spread over many classes): ranking buys nothing, thread <-> candidate i and
            // 16 of the later candidates, dead rows / columns and pairs of different classes skipped
            const int i = t >> 2, jq = t & 3;
            if ((alive >> i) & 1ull) {
                const float4 bi = chbox[i];
                const float ai = charea[i];
                const unsigned short ci = by_class ? chcls[i] : (unsigned short)0;
                unsigned int bits = 0u;
#pragma unroll 4
                for (int e = 0; e < 16; ++e) {
                    const int j = jq * 16 + e;
                    if (j > i && ((alive >> j) & 1ull) && (!by_class || chcls[j] == ci)) {
                        bool d, m;
                        iou_fast(bi, ai, chbox[j], charea[j], p, d, m);
                        if (m) d = iou_gt(bi, ai, chbox[j], charea[j], p);
                        bits |= (unsigned)d << e;
                    }
                }
                if (bits) atomicOr(&s.cmask[2 * i + (jq >> 1)], bits << ((jq & 1) * 16));
            }
        }
        __syncthreads();
        tick(4);
        // (c) greedy resolve over the kill rows by warp 0: resolve_chunk written out (calling it here reorders two compares in the
        // SASS of every NMS kernel)
        if (t < 32) {
            unsigned int lo = (unsigned int)alive, hi = (unsigned int)(alive >> 32), klo = 0u, khi = 0u;
            int room = p.max_det - nk;
            while (lo && room > 0) {
                const int i = __ffs((int)lo) - 1;
                klo |= 1u << i;
                --room;
                lo &= ~(1u << i) & ~s.cmask[2 * i];
                hi &= ~s.cmask[2 * i + 1];
            }
            while (hi && room > 0) {
                const int i = __ffs((int)hi) - 1;
                khi |= 1u << i;
                --room;
                hi &= ~(1u << i) & ~s.cmask[2 * (i + 32) + 1];
            }
            if (t == 0) { s.misc->kept[0] = klo; s.misc->kept[1] = khi; }
        }
        __syncthreads();
        const unsigned long long kept = ((unsigned long long)s.misc->kept[1] << 32) | (unsigned long long)s.misc->kept[0];
        if (by_class && t == 0) {                                     // per-class lists of kept boxes, in kept order
            int pos = nk;
            for (unsigned long long r = kept; r; r &= r - 1ull, ++pos) {
                const unsigned c = chcls[__ffsll((long long)r) - 1];
                s.kcn[pos] = c | ((unsigned)s.khead[c] << 16);
                s.khead[c] = (unsigned short)pos;
            }
        }
        if (t < cn && ((kept >> t) & 1ull)) {   // (d) append
            const int pos = nk + __popcll(kept & ((1ull << t) - 1ull));
            s.kbox[pos] = chbox[t];
            s.karea[pos] = charea[t];
            const unsigned long long key = s.keys[c0 + t];
            const unsigned int slot = (unsigned int)(key & 0xFFFFull);
            const float4 b = s.cbox[slot];
            float* o = out + pos * 6;
            o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w;
            o[4] = sortable2f((unsigned int)(key >> 32));
            o[5] = (float)s.ccls[slot];
            if (kidx) kidx[pos] = 0xFFFF - (int)((key >> 16) & 0xFFFFull);
        }
        nk += __popcll(kept);
        __syncthreads();
        tick(5);
    }
    if (t == 0) p.counts[n] = nk;
    for (int i = nk * 6 + t; i < p.max_det * 6; i += NT) out[i] = 0.f;
    if (kidx) for (int i = nk + t; i < p.max_det; i += NT) kidx[i] = -1;
    if (PROF) {
        __syncthreads();
        tick(7);
        if (t == 0 && p.prof) {
            long long* q = p.prof + (long long)n * 16;
            for (int k = 0; k < 8; ++k) q[k] = acc[k];
            q[8] = nchunks; q[9] = cnt; q[10] = nk;
        }
    }
}

// NMS from an [N,M,5+C] tensor: one CTA per image, warp per row for the scoring pass.  Three CTAs per SM: the scoring pass is
// bound by the latency of its row loads (see below), and at two (above 85 registers) it is a third slower on the bench_nms sets.
__global__ void __launch_bounds__(NT, 3)
nms_kernel(const float* __restrict__ dets, int C, NmsParams p) {
    extern __shared__ __align__(16) unsigned char smraw[];
    NmsSmem s;
    nms_layout(s, smraw, p.M, p.MCp, p.max_det);
    const int n = blockIdx.x;
    if (threadIdx.x == 0) { s.misc->count = 0u; s.misc->outside = 0u; }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int D = 5 + C;
    const float* img = dets + (long long)n * p.M * D;
    // Four rows per warp and trip: a row is one dependent round trip to DRAM (objectness, then its class scores) and the pass is
    // bound by that latency (10 000 images: 6.2 GB in 7.8 ms = 0.8 TB/s with one row in flight per warp), so the loads of four
    // rows are issued together.  Row order only matters through the sort key (conf, row), not through the slot a row lands in.
    constexpr int RU = 4, NW = NT / 32;
    for (int r0 = warp; r0 < p.M; r0 += RU * NW) {
        const float* row[RU];
        float obj[RU], box[RU][4];
        bool pass[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u) {
            const int r = r0 + u * NW;
            row[u] = img + (long long)(r < p.M ? r : r0) * D;
            obj[u] = __ldg(row[u] + 4);
        }
#pragma unroll
        for (int u = 0; u < RU; ++u) pass[u] = (r0 + u * NW < p.M) && (obj[u] > p.conf_thres);    // utils/utils.py:254 (warp uniform)
        float best[RU];
        int bi[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u) { best[u] = -INFINITY; bi[u] = 0x7fffffff; }
        for (int c = lane; c < C; c += 32) {
            float v[RU];
#pragma unroll
            for (int u = 0; u < RU; ++u) v[u] = pass[u] ? __ldg(row[u] + 5 + c) : 0.f;
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                const float w = __fmul_rn(v[u], obj[u]);               // :261
                if (pass[u] && w > best[u]) { best[u] = w; bi[u] = c; }
            }
        }
#pragma unroll
        for (int u = 0; u < RU; ++u)
#pragma unroll
            for (int k = 0; k < 4; ++k) box[u][k] = (pass[u] && lane == 0) ? __ldg(row[u] + k) : 0.f;
#pragma unroll
        for (int u = 0; u < RU; ++u) {
            if (!pass[u]) continue;
            warp_argmax(best[u], bi[u]);                               // :267 first max
            if (lane == 0 && best[u] > p.conf_thres && class_ok(p, bi[u])) {    // :268, :271-272
                const unsigned int slot = atomicAdd(&s.misc->count, 1u);
                write_candidate(s, slot, box[u][0], box[u][1], box[u][2], box[u][3], best[u], bi[u], r0 + u * NW, p.max_wh);
            }
        }
    }
    sort_and_suppress<false>(s, p, n);
}

constexpr int kCT = 80;

// Softmax of one cell, one thread (thread_cell_candidates_80x3): e[kCT] holds the class logits on entry and the exponentials on
// return.  The expf arguments and the summation tree (32 partial sums of classes l, l+32, l+64, then the
// xor-butterfly levels 16, 8, 4, 2, 1) are warp_softmax's, so the sum is bit for bit the one decode_kernel divides by.
struct CellSoftmax {
    float sum, emax;
    int cstar;   // first arg-max of e
    int nnear;   // classes with e >= 0.99999 emax (cstar among them)
};
__device__ __forceinline__ CellSoftmax thread_softmax(float (&e)[kCT]) {
    CellSoftmax r;
    float m = -INFINITY;
#pragma unroll
    for (int c = 0; c < kCT; ++c) m = fmaxf(m, e[c]);
    r.emax = 0.f;
    r.cstar = 0;
#pragma unroll
    for (int c = 0; c < kCT; ++c) {
        e[c] = expf(__fsub_rn(e[c], m));
        if (e[c] > r.emax) { r.emax = e[c]; r.cstar = c; }
    }
    float ps[32];
#pragma unroll
    for (int l = 0; l < 32; ++l) {
        float t = e[l];                                           // (0 + e_l) is exact
        if (l + 32 < kCT) t = __fadd_rn(t, e[l + 32]);
        if (l + 64 < kCT) t = __fadd_rn(t, e[l + 64]);
        ps[l] = t;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1)
#pragma unroll
        for (int i = 0; i < o; ++i) ps[i] = __fadd_rn(ps[i], ps[i + o]);
    r.sum = ps[0];
    const float near = r.emax * 0.99999f;
    r.nnear = 0;
#pragma unroll
    for (int c = 0; c < kCT; ++c) r.nnear += (e[c] >= near) ? 1 : 0;
    return r;
}

// The reference's class for conf = fl(fl(emax/sum)*obj): the first class with the largest product.  conf_c = fl(fl(e_c/sum)*obj)
// is monotone in e_c, so that is the first arg-max of e unless an earlier class rounds to the same product, which needs e_c
// within 1e-5 of emax while the product is normal (24 bits).  A subnormal conf (tiny objectness, conf_thres = 0) has fewer
// bits, classes further below can round to it, and then every earlier class is re-checked.
__device__ __forceinline__ int first_max_class(const float (&e)[kCT], const CellSoftmax& sm, float obj, float conf) {
    const bool sub = conf < FLT_MIN;
    int cls = sm.cstar;
    if (sm.nnear > 1 || sub) {                                    // rare
        const float near = sub ? 0.f : sm.emax * 0.99999f;
        bool found = false;
#pragma unroll
        for (int c = 0; c < kCT; ++c)
            if (!found && c < sm.cstar && e[c] >= near && __fmul_rn(__fdiv_rn(e[c], sm.sum), obj) == conf) { cls = c; found = true; }
    }
    return cls;
}

// Fused: candidates come straight from the head logits.
//
// C <= 80: ONE THREAD PER CELL instead of one warp per cell.  A thread keeps the C exponentials of its cell in registers and
// computes the warp version's probabilities bit for bit (thread_softmax).  Per (cell, anchor) only the winning class needs the
// division and the product (first_max_class).  ~10x fewer warp instructions than warp-per-cell (the loads are coalesced
// across the 32 cells of a warp).
// This generic version writes the same softmax and re-check out inline (with the near-tie count per anchor): built from the two
// helpers, ptxas spills more of e[] in it (304 instead of 160 bytes of stack on sm_90a, nvcc 12.9).
__device__ __forceinline__ void thread_cell_candidates(const PostGeom& g, const NmsParams& p, const NmsSmem& s, int n, int lv, int cell,
                                                       bool in_range, int row0) {
    const int A = g.A, C = g.C, hw = g.hw[lv];
    float e[kCT];
    float sum = 1.f, emax = 0.f;
    int cstar = 0;
    if (in_range) {
        const float* cp = g.cls[lv] + (long long)n * C * hw + cell;
        float m = -INFINITY;
#pragma unroll
        for (int c = 0; c < kCT; ++c) { e[c] = (c < C) ? __ldg(cp + (long long)c * hw) : -INFINITY; m = fmaxf(m, e[c]); }
#pragma unroll
        for (int c = 0; c < kCT; ++c) {
            e[c] = (c < C) ? expf(__fsub_rn(e[c], m)) : 0.f;
            if (e[c] > emax) { emax = e[c]; cstar = c; }             // first arg-max
        }
        float ps[32];
#pragma unroll
        for (int l = 0; l < 32; ++l) {
            float t = e[l];                                           // (0 + e_l) is exact
            if (l + 32 < kCT) t = __fadd_rn(t, e[l + 32]);
            if (l + 64 < kCT) t = __fadd_rn(t, e[l + 64]);
            ps[l] = t;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1)
#pragma unroll
            for (int i = 0; i < o; ++i) ps[i] = __fadd_rn(ps[i], ps[i + o]);
        sum = ps[0];
    }
    const int y = cell / g.w[lv], x = cell - y * g.w[lv];
    for (int a = 0; a < A; ++a) {
        bool want = false;
        float conf = 0.f;
        float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
        int cls = 0;
        if (in_range) {
            const float obj = sigmoid_rn(__ldg(g.obj[lv] + ((long long)n * A + a) * hw + cell));
            if (obj > p.conf_thres) {
                conf = __fmul_rn(__fdiv_rn(emax, sum), obj);
                cls = cstar;
                const bool sub = conf < FLT_MIN;                      // subnormal product: any earlier class may round to it
                const float near = sub ? 0.f : emax * 0.99999f;
                int nnear = 0;
#pragma unroll
                for (int c = 0; c < kCT; ++c) nnear += (e[c] >= near) ? 1 : 0;
                if (nnear > 1) {                                      // rare: an earlier class may round to the same product
                    bool found = false;
#pragma unroll
                    for (int c = 0; c < kCT; ++c)
                        if (!found && c < cstar && e[c] >= near && __fmul_rn(__fdiv_rn(e[c], sum), obj) == conf) { cls = c; found = true; }
                }
                if (conf > p.conf_thres && class_ok(p, cls)) {
                    want = true;
                    const float* rp = g.reg[lv] + ((long long)n * 4 * A + 4 * a) * hw + cell;
                    box = decode_box(__ldg(rp), __ldg(rp + hw), __ldg(rp + 2 * (long long)hw), __ldg(rp + 3 * (long long)hw), x, y,
                                     g.stride[lv], g.anc[lv][a][0], g.anc[lv][a][1]);
                }
            }
        }
        const unsigned int slot = alloc_slots(&s.misc->count, want);
        if (want) write_candidate(s, slot, box.x, box.y, box.z, box.w, conf, cls, row0 + cell * A + a, p.max_wh);
    }
}

// The common shape (80 classes, 3 anchors) with everything static.  ncu on the generic version above (round 2, batch 256): the
// candidate phase was 26 % of the kernel (59 us of 227 per image) and 5500 issued instructions per thread and pass, 70 % of them
// predicated 64-bit address arithmetic for `(c < C) ? __ldg(cp + (long long)c * hw)`, with seven dependent global round trips per
// pass (classes, then objectness and box logits anchor by anchor).  Here the class count is a constant, offsets are 32-bit, the
// three objectness logits travel with the class logits and the box logits of all wanted anchors in one more batch.  Same
// arithmetic, same results bit for bit.
__device__ __forceinline__ void thread_cell_candidates_80x3(const PostGeom& g, const NmsParams& p, const NmsSmem& s, int n, int lv, int cell,
                                                            bool in_range, int row0) {
    constexpr int A = 3, C = kCT;
    const int hw = g.hw[lv];
    float e[C];
    CellSoftmax sm = {1.f, 0.f, 0, 0};
    float ol[A] = {0.f, 0.f, 0.f};
    if (in_range) {
        const float* cp = g.cls[lv] + (long long)n * C * hw + cell;
        const float* op = g.obj[lv] + (long long)n * A * hw + cell;
#pragma unroll
        for (int c = 0; c < C; ++c) e[c] = __ldg(cp + c * hw);
#pragma unroll
        for (int a = 0; a < A; ++a) ol[a] = __ldg(op + a * hw);
        sm = thread_softmax(e);
    }
    bool want[A];
    float conf[A];
    int cls[A];
#pragma unroll
    for (int a = 0; a < A; ++a) {
        want[a] = false; conf[a] = 0.f; cls[a] = sm.cstar;
        if (in_range) {
            const float obj = sigmoid_rn(ol[a]);
            if (obj > p.conf_thres) {
                conf[a] = __fmul_rn(__fdiv_rn(sm.emax, sm.sum), obj);
                cls[a] = first_max_class(e, sm, obj, conf[a]);
                want[a] = conf[a] > p.conf_thres && class_ok(p, cls[a]);
            }
        }
    }
    const int y = cell / g.w[lv], x = cell - y * g.w[lv];
    float r[A][4];
    {
        const float* rp = g.reg[lv] + (long long)n * 4 * A * hw + cell;
#pragma unroll
        for (int a = 0; a < A; ++a)
#pragma unroll
            for (int k = 0; k < 4; ++k) r[a][k] = want[a] ? __ldg(rp + (4 * a + k) * hw) : 0.f;
    }
#pragma unroll
    for (int a = 0; a < A; ++a) {
        float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
        if (want[a]) box = decode_box(r[a][0], r[a][1], r[a][2], r[a][3], x, y, g.stride[lv], g.anc[lv][a][0], g.anc[lv][a][1]);
        const unsigned int slot = alloc_slots(&s.misc->count, want[a]);
        if (want[a]) write_candidate(s, slot, box.x, box.y, box.z, box.w, conf[a], cls[a], row0 + cell * A + a, p.max_wh);
    }
}

// FAST selects the candidate generation at compile time (one path per kernel: the register allocation and the instruction footprint
// of one path no longer pay for the others): 2 = thread per cell with 80 classes x 3 anchors static, 1 = thread per cell, any
// other C <= 80, 0 = warp per cell (any C; the path above 80 classes).
template <bool PROF, int FAST>
__global__ void __launch_bounds__(NT, 2)
decode_nms_kernel(PostGeom g, NmsParams p) {
    pdl_wait();
    const long long tstart = PROF ? clock64() : 0ll;
    extern __shared__ __align__(16) unsigned char smraw[];
    NmsSmem s;
    float* const S = reinterpret_cast<float*>(nms_layout(s, smraw, p.M, p.MCp, p.max_det));   // warp per cell: its staged cells
    const int n = blockIdx.x;
    if (threadIdx.x == 0) { s.misc->count = 0u; s.misc->outside = 0u; }
    const int A = g.A, C = g.C;
    if (FAST) {
        __syncthreads();
#pragma unroll 1
        for (int lv = 0; lv < 2; ++lv) {
            const int row0 = lv ? g.hw[0] * A : 0;
#pragma unroll 1
            for (int c0 = 0; c0 < g.hw[lv]; c0 += NT) {
                const int cell = c0 + threadIdx.x;
                const bool in_range = cell < g.hw[lv];
                if (FAST == 2) thread_cell_candidates_80x3(g, p, s, n, lv, in_range ? cell : 0, in_range, row0);
                else thread_cell_candidates(g, p, s, n, lv, in_range ? cell : 0, in_range, row0);
            }
        }
    } else {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int lv = 0; lv < 2; ++lv) {
            const int row0 = lv ? g.hw[0] * A : 0;
            for (int cell0 = 0; cell0 < g.hw[lv]; cell0 += kChunkCells) {
                const int ncell = min(kChunkCells, g.hw[lv] - cell0);
                __syncthreads();
                stage_cells(S, g, n, lv, cell0, ncell);
                __syncthreads();
                for (int cl = warp; cl < ncell; cl += NT / 32) {
                    CellRegs r;
                    decode_cell(S, g, lv, cell0 + cl, cl, lane, r);
                    float my_conf = 0.f;
                    int my_cls = 0;
                    bool my_want = false;
                    for (int a = 0; a < A; ++a) {
                        const float obj = __shfl_sync(0xffffffffu, r.ob, a);
                        if (!(obj > p.conf_thres)) continue;
                        float best = -INFINITY;
                        int bi = 0x7fffffff;
#pragma unroll
                        for (int j = 0; j < kCPL; ++j) {
                            const int c = lane + 32 * j;
                            if (c < C) {
                                const float v = __fmul_rn(r.p[j], obj);
                                if (v > best) { best = v; bi = c; }
                            }
                        }
                        warp_argmax(best, bi);
                        if (lane == a && best > p.conf_thres && class_ok(p, bi)) { my_want = true; my_conf = best; my_cls = bi; }
                    }
                    const unsigned int slot = alloc_slots(&s.misc->count, my_want);
                    if (my_want)
                        write_candidate(s, slot, r.box.x, r.box.y, r.box.z, r.box.w, my_conf, my_cls, row0 + (cell0 + cl) * A + lane, p.max_wh);
                }
            }
        }
    }
    sort_and_suppress<PROF>(s, p, n, tstart);
}

// ---------------------------------------------------------------------------------------------------
// Cross-region merge (yfv2_merge_regions): the NMS rows of T region images -> one list per frame in frame pixels.  One CTA per
// frame.  The region descriptors of a launch's frames travel in the kernel parameters; the rows are read from global memory and
// mapped to frame pixels on the fly, and only the kept boxes are held in shared memory (fp64).
constexpr int kMergeFrames = 128;              // frames per launch

struct MergeArgs {
    const float* dets;           // [T, max_det_in, 6]
    const int* counts;           // [T]
    double* out;                 // [F, max_det, 6]
    int* out_counts;             // [F]
    int* kept_src;               // [F, max_det] or null
    double thr;
    int W, H, max_det_in, max_det, metric;
    int f0;                      // first frame of the launch
    int t0;                      // global index of the launch's first region
    int MCp;                     // key buffer: pow2 >= max(64, the largest frame's candidate slots)
    int KC;                      // kept-box capacity: min(max_det, the largest frame's candidate slots)
    int rbeg[kMergeFrames + 1];  // regions of frame f0 + i: [rbeg[i], rbeg[i + 1]) of reg[]
    int4 reg[YFV2_MERGE_MAX_REGIONS];   // x0, y0, w, h
};

struct MergeSmem {
    unsigned long long* keys;   // [MCp]  (sortable conf << 32) | ~(t_local * max_det_in + row)
    double4* kbox;              // [KC]   kept boxes, frame pixels
    float* kcls;                // [KC]
    unsigned short* kt;         // [KC]   region of each kept box, relative to the frame's first
    double4* chbox;             // [64]   the chunk's candidates
    float* chcls;               // [64]
    unsigned short* cht;        // [64]
    unsigned int* cmask;        // [64][2] kill rows inside the chunk
    unsigned int* misc;         // [0] candidates pushed, [1..2] dead bits of the chunk, [3..4] kept bits of the chunk
};

__host__ __device__ __forceinline__ unsigned char* merge_layout(MergeSmem& s, unsigned char* base, int MCp, int KC) {
    s.keys = take<unsigned long long>(base, MCp);
    s.kbox = take<double4>(base, KC);
    s.chbox = take<double4>(base, kChunk);
    s.kcls = take<float>(base, KC);
    s.chcls = take<float>(base, kChunk);
    s.cmask = take<unsigned int>(base, 2 * kChunk);
    s.misc = take<unsigned int>(base, 8);
    s.kt = take<unsigned short>(base, KC);
    s.cht = take<unsigned short>(base, kChunk);
    return base;
}

inline size_t merge_smem_bytes(int MCp, int KC) {
    MergeSmem s;
    return reinterpret_cast<size_t>(merge_layout(s, nullptr, MCp, KC));
}

// min / max as the contract defines them (region_oracle.py uses the same comparisons, so NaN coordinates agree)
__device__ __forceinline__ double dmin(double a, double b) { return a < b ? a : b; }
__device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }

// fp64 overlap of box a (kept, or earlier in the order) and box b, strictly above thr.  metric 0: IoU = inter / (a_a + a_b - inter);
// 1: IoS = inter / min(a_a, a_b).  No +1 in the widths (torchvision's convention); every operation rounded on its own; a NaN
// quotient compares false.  Unlike iou_gt (fp32, class offsets) the class test is the caller's.
__device__ __forceinline__ bool overlap_gt(const double4& a, const double4& b, double thr, int metric) {
    const double iw = dmax(0.0, __dsub_rn(dmin(a.z, b.z), dmax(a.x, b.x)));
    const double ih = dmax(0.0, __dsub_rn(dmin(a.w, b.w), dmax(a.y, b.y)));
    const double inter = __dmul_rn(iw, ih);
    const double aa = __dmul_rn(__dsub_rn(a.z, a.x), __dsub_rn(a.w, a.y));
    const double ab = __dmul_rn(__dsub_rn(b.z, b.x), __dsub_rn(b.w, b.y));
    const double den = metric ? dmin(aa, ab) : __dsub_rn(__dadd_rn(aa, ab), inter);
    return __ddiv_rn(inter, den) > thr;
}

// Row `slot` (t_local * max_det_in + row) of the frame whose first region is tg0 (rb in a.reg): its box mapped to frame pixels
// (contract step 1), its region relative to the frame's first (tl) and its row in dets (r: r[4] conf, r[5] cls).
__device__ __forceinline__ double4 map_row(const MergeArgs& a, long long tg0, int rb, unsigned int slot, int& tl, const float*& r) {
    const int mdi = a.max_det_in;
    tl = (int)slot / mdi;
    const int row = (int)slot - tl * mdi;
    r = a.dets + ((tg0 + tl) * mdi + row) * 6;
    const int4 g = a.reg[rb + tl];
    const double sx = __ddiv_rn((double)g.z, (double)a.W), sy = __ddiv_rn((double)g.w, (double)a.H);
    const double x0 = (double)g.x, y0 = (double)g.y;
    return make_double4(__dadd_rn(__dmul_rn((double)__ldg(r), sx), x0), __dadd_rn(__dmul_rn((double)__ldg(r + 1), sy), y0),
                        __dadd_rn(__dmul_rn((double)__ldg(r + 2), sx), x0), __dadd_rn(__dmul_rn((double)__ldg(r + 3), sy), y0));
}

// The merge's side of greedy_pass: candidates staged from the rows in global memory, mapped to frame pixels; a box suppresses
// only boxes of other regions and the same class.
struct MergePass {
    const MergeArgs& a;
    const MergeSmem& s;
    double* out;
    int* ksrc;
    long long tg0;                                               // global index of the frame's first region
    int rb;                                                      // the frame's first region in a.reg

    __device__ __forceinline__ void stage(int j, unsigned long long key) const {
        const unsigned int slot = 0xFFFFFFFFu - (unsigned int)(key & 0xFFFFFFFFull);
        int tl;
        const float* r;
        s.chbox[j] = map_row(a, tg0, rb, slot, tl, r);
        s.chcls[j] = __ldg(r + 5);
        s.cht[j] = (unsigned short)tl;
    }
    struct Cand {
        double4 box;
        float cls;
        unsigned short t;
    };
    __device__ __forceinline__ Cand cand(int j) const { return {s.chbox[j], s.chcls[j], s.cht[j]}; }
    __device__ __forceinline__ bool kept_other_source(int i, const Cand& c) const { return s.kt[i] != c.t; }
    __device__ __forceinline__ bool kept_same_class(int i, const Cand& c) const { return s.kcls[i] == c.cls; }
    __device__ __forceinline__ bool kept_kills(int i, const Cand& c) const { return overlap_gt(s.kbox[i], c.box, a.thr, a.metric); }
    __device__ __forceinline__ bool other_source(const Cand& c, int j) const { return s.cht[j] != c.t; }
    __device__ __forceinline__ bool same_class(const Cand& c, int j) const { return s.chcls[j] == c.cls; }
    __device__ __forceinline__ bool kills(const Cand& c, int j) const { return overlap_gt(c.box, s.chbox[j], a.thr, a.metric); }
    __device__ __forceinline__ void append(int pos, int j, const unsigned long long& key) const {
        const double4 b = s.chbox[j];
        s.kbox[pos] = b;
        s.kcls[pos] = s.chcls[j];
        s.kt[pos] = s.cht[j];
        const unsigned int slot = 0xFFFFFFFFu - (unsigned int)(key & 0xFFFFFFFFull);
        double* o = out + pos * 6;
        o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w;
        o[4] = (double)__ldg(a.dets + (tg0 * a.max_det_in + slot) * 6 + 4);     // (the key holds conf + 0)
        o[5] = (double)s.chcls[j];
        if (ksrc) ksrc[pos] = (int)(tg0 * a.max_det_in + slot);
    }
};

// Candidates of frame block fl into s.keys, sorted descending (contract step 2); returns their number.  All threads call this.
// (merge_regions_kernel spells the same steps out inline: calling this helper there reschedules its SASS.)
__device__ __forceinline__ int merge_candidates(const MergeArgs& a, const MergeSmem& s, int fl) {
    const int t = threadIdx.x;
    const int rb = a.rbeg[fl], nreg = a.rbeg[fl + 1] - rb;
    const int mdi = a.max_det_in;
    const long long tg0 = (long long)a.t0 + rb;
    if (t == 0) s.misc[0] = 0u;
    __syncthreads();
    // candidates: rows below each region's count whose conf is not NaN, keyed by (conf, then lower t, then lower row first)
    const int nslots = nreg * mdi;
    for (int base = 0; base < nslots; base += NT) {
        const int slot = base + t;
        bool want = false;
        unsigned long long key = 0ull;
        if (slot < nslots) {
            const int tl = slot / mdi, row = slot - tl * mdi;
            const int cnt = min(max(__ldg(a.counts + tg0 + tl), 0), mdi);
            if (row < cnt) {
                const float conf = __ldg(a.dets + ((tg0 + tl) * mdi + row) * 6 + 4);
                if (!isnan(conf)) {
                    want = true;
                    // + 0 turns -0 into +0, so that the two zeros tie like any equal confidences
                    key = ((unsigned long long)f2sortable(__fadd_rn(conf, 0.0f)) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)slot);
                }
            }
        }
        const unsigned int pos = alloc_slots(&s.misc[0], want);
        if (want) s.keys[pos] = key;
    }
    __syncthreads();
    const int cnt = (int)s.misc[0];
    sort_keys_desc(s.keys, cnt);
    return cnt;
}

__global__ void __launch_bounds__(NT)
merge_regions_kernel(const __grid_constant__ MergeArgs a) {
    extern __shared__ __align__(32) unsigned char smraw[];
    MergeSmem s;
    merge_layout(s, smraw, a.MCp, a.KC);
    const int t = threadIdx.x, fl = blockIdx.x, f = a.f0 + fl;
    const int rb = a.rbeg[fl], nreg = a.rbeg[fl + 1] - rb;
    const int mdi = a.max_det_in;
    const long long tg0 = (long long)a.t0 + rb;                  // global index of the frame's first region
    if (t == 0) s.misc[0] = 0u;
    __syncthreads();
    // candidates: rows below each region's count whose conf is not NaN, keyed by (conf, then lower t, then lower row first)
    const int nslots = nreg * mdi;
    for (int base = 0; base < nslots; base += NT) {
        const int slot = base + t;
        bool want = false;
        unsigned long long key = 0ull;
        if (slot < nslots) {
            const int tl = slot / mdi, row = slot - tl * mdi;
            const int cnt = min(max(__ldg(a.counts + tg0 + tl), 0), mdi);
            if (row < cnt) {
                const float conf = __ldg(a.dets + ((tg0 + tl) * mdi + row) * 6 + 4);
                if (!isnan(conf)) {
                    want = true;
                    // + 0 turns -0 into +0, so that the two zeros tie like any equal confidences
                    key = ((unsigned long long)f2sortable(__fadd_rn(conf, 0.0f)) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)slot);
                }
            }
        }
        const unsigned int pos = alloc_slots(&s.misc[0], want);
        if (want) s.keys[pos] = key;
    }
    __syncthreads();
    const int cnt = (int)s.misc[0];
    sort_keys_desc(s.keys, cnt);

    double* out = a.out + (long long)f * a.max_det * 6;
    int* ksrc = a.kept_src ? a.kept_src + (long long)f * a.max_det : nullptr;
    const int nk = greedy_pass(s.keys, cnt, a.max_det, s.cmask, s.misc + 1, MergePass{a, s, out, ksrc, tg0, rb});
    if (t == 0) a.out_counts[f] = nk;
    for (int i = nk * 6 + t; i < a.max_det * 6; i += NT) out[i] = 0.0;
    if (ksrc) for (int i = nk + t; i < a.max_det; i += NT) ksrc[i] = -1;
}

// Greedy non-maximum merging (yfv2_merge_regions_nmm): merge_regions_kernel's pass, which also marks the output rows by slot in
// `kept` (one bit per candidate slot), then
//   absorb: every other sorted row, after the cap too, scans the kept boxes in order and stops at the first one that would
//           suppress it (step 3's test).  The first matching kept row comes before the row: a kept row before it that matches
//           suppressed it, and a row after the last kept one comes after all of them.  Each absorbed row becomes the grouping key
//           (0xFFFF - absorber) << 32 | (0xFFFF - sorted position) << 16 | slot, compacted to the front of the key buffer (a
//           tile's writes land below the next tile's reads) and sorted descending: absorbers ascending, each group in order.
//   fold:   the thread holding a group's first key grows the absorber's box B through the group, re-testing each row against B.
// All sizes fit 16 bits: absorber < 4096, sorted position and slot < YFV2_NMS_MAX_CAND.  The bitmap is the only shared memory
// added to merge_regions_kernel's (MCp / 8 bytes, 1 KB at the limit).
struct MergeNmmPass : MergePass {
    unsigned int* kept;
    __device__ __forceinline__ void append(int pos, int j, const unsigned long long& key) const {
        MergePass::append(pos, j, key);
        const unsigned int slot = 0xFFFFFFFFu - (unsigned int)(key & 0xFFFFFFFFull);
        atomicOr(&kept[slot >> 5], 1u << (slot & 31));
    }
};

inline size_t merge_nmm_smem_bytes(int MCp, int KC) { return merge_smem_bytes(MCp, KC) + (size_t)MCp / 8; }

__global__ void __launch_bounds__(NT)
merge_regions_nmm_kernel(const __grid_constant__ MergeArgs a, int* merged) {
    extern __shared__ __align__(32) unsigned char smraw[];
    MergeSmem s;
    unsigned char* tail = merge_layout(s, smraw, a.MCp, a.KC);
    unsigned int* kept = take<unsigned int>(tail, a.MCp / 32);
    const int t = threadIdx.x, fl = blockIdx.x, f = a.f0 + fl;
    const int rb = a.rbeg[fl];
    const long long tg0 = (long long)a.t0 + rb;
    double* out = a.out + (long long)f * a.max_det * 6;
    int* ksrc = a.kept_src ? a.kept_src + (long long)f * a.max_det : nullptr;
    for (int i = t; i < a.MCp / 32; i += NT) kept[i] = 0u;
    const int cnt = merge_candidates(a, s, fl);
    const int nk = greedy_pass(s.keys, cnt, a.max_det, s.cmask, s.misc + 1, MergeNmmPass{{a, s, out, ksrc, tg0, rb}, kept});
    if (t == 0) a.out_counts[f] = nk;
    for (int i = nk * 6 + t; i < a.max_det * 6; i += NT) out[i] = 0.0;
    if (ksrc) for (int i = nk + t; i < a.max_det; i += NT) ksrc[i] = -1;
    int* mrg = merged ? merged + (long long)f * a.max_det : nullptr;
    if (mrg) for (int i = t; i < a.max_det; i += NT) mrg[i] = 0;   // ordered before the fold's writes by the barriers between

    // absorb
    if (t == 0) s.misc[0] = 0u;
    __syncthreads();
    for (int base = 0; base < cnt; base += NT) {
        const int p = base + t;
        bool want = false;
        unsigned long long g = 0ull;
        if (p < cnt) {
            const unsigned int slot = 0xFFFFFFFFu - (unsigned int)(s.keys[p] & 0xFFFFFFFFull);
            if (!((kept[slot >> 5] >> (slot & 31)) & 1u)) {
                int tl;
                const float* r;
                const double4 box = map_row(a, tg0, rb, slot, tl, r);
                const float cls = __ldg(r + 5);
                for (int i = 0; i < nk; ++i) {
                    if (s.kt[i] != tl && s.kcls[i] == cls && overlap_gt(s.kbox[i], box, a.thr, a.metric)) {
                        want = true;
                        g = ((unsigned long long)(0xFFFFu - (unsigned)i) << 32) | ((unsigned long long)(0xFFFFu - (unsigned)p) << 16) | slot;
                        break;
                    }
                }
            }
        }
        __syncthreads();                                         // the tile's keys are read
        const unsigned int pos = alloc_slots(&s.misc[0], want);
        if (want) s.keys[pos] = g;
    }
    __syncthreads();
    const int ng = (int)s.misc[0];
    sort_keys_desc(s.keys, ng);

    // fold
    for (int k = t; k < ng; k += NT) {
        const unsigned int gi = (unsigned int)(s.keys[k] >> 32);
        if (k > 0 && (unsigned int)(s.keys[k - 1] >> 32) == gi) continue;
        const int i = (int)(0xFFFFu - gi);
        double4 B = s.kbox[i];
        int m = 0;
        for (int q = k; q < ng; ++q) {
            const unsigned long long key = s.keys[q];
            if ((unsigned int)(key >> 32) != gi) break;
            int tl;
            const float* r;
            const double4 b = map_row(a, tg0, rb, (unsigned int)(key & 0xFFFFu), tl, r);
            if (overlap_gt(B, b, a.thr, a.metric)) {
                B = make_double4(dmin(B.x, b.x), dmin(B.y, b.y), dmax(B.z, b.z), dmax(B.w, b.w));
                ++m;
            }
        }
        double* o = out + i * 6;
        o[0] = B.x; o[1] = B.y; o[2] = B.z; o[3] = B.w;
        if (mrg) mrg[i] = m;
    }
}

long long* g_nms_prof = nullptr;       // yfv2_debug_nms_profile

int fill_geom(PostGeom& g, const float* const preds[6], int N, int H, int W, int A, int C, const double* anchors_host) {
    if (!preds || !anchors_host || N <= 0 || A <= 0 || A > kMaxA || C <= 0 || C > 32 * kCPL || H % 32 || W % 32 || H <= 0 || W <= 0) {
        set_error("decode: bad arguments (N=%d H=%d W=%d A=%d C=%d; need A<=%d, C<=%d, H,W multiples of 32)", N, H, W, A, C,
                  kMaxA, 32 * kCPL);
        return YFV2_EINVAL;
    }
    g.N = N; g.A = A; g.C = C; g.D = 5 + C;
    for (int lv = 0; lv < 2; ++lv) {
        const int s = lv ? 32 : 16;
        g.h[lv] = H / s; g.w[lv] = W / s; g.hw[lv] = g.h[lv] * g.w[lv];
        g.stride[lv] = (float)((double)H / (double)g.h[lv]);      // cfg["height"] / h, one stride for both axes (:332)
        for (int a = 0; a < A; ++a) {
            g.anc[lv][a][0] = anchors_host[(lv * A + a) * 2];
            g.anc[lv][a][1] = anchors_host[(lv * A + a) * 2 + 1];
        }
        g.reg[lv] = preds[3 * lv]; g.obj[lv] = preds[3 * lv + 1]; g.cls[lv] = preds[3 * lv + 2];
        if (!g.reg[lv] || !g.obj[lv] || !g.cls[lv]) { set_error("decode: null head tensor"); return YFV2_EINVAL; }
    }
    g.M = (g.hw[0] + g.hw[1]) * A;
    return YFV2_OK;
}

int fill_nms(NmsParams& p, int M, float conf_thres, double iou_thres, const int* class_filter, int n_filter, int max_det,
             float max_wh, float* out, int* counts, int* kept_idx) {
    if (!out || !counts || max_det <= 0 || max_det > 4096 || M <= 0) { set_error("nms: bad arguments"); return YFV2_EINVAL; }
    if (M > YFV2_NMS_MAX_CAND) { set_error("nms: M=%d candidates per image exceeds %d", M, YFV2_NMS_MAX_CAND); return YFV2_EUNSUPPORTED; }
    p.conf_thres = conf_thres; p.iou_thres = iou_thres;
    {   // rounding boundary of the fp32 quotient around the (double) threshold
        float f0 = (float)iou_thres;                       // nearest float
        if ((double)f0 > iou_thres) f0 = nextafterf(f0, -INFINITY);
        const float f1 = nextafterf(f0, INFINITY);          // smallest float > thr
        p.iou_mid = ((double)f0 + (double)f1) * 0.5;
        p.iou_mid_f = (float)p.iou_mid;
        p.iou_fast_mid = p.iou_mid > 0.0 ? p.iou_mid_f : nanf("");
        p.iou_zero = p.iou_mid > 0.0 ? 0.f : nanf("");
        unsigned int bits; memcpy(&bits, &f1, 4);
        p.iou_tie_up = (bits & 1u) == 0u;                   // ties-to-even: the midpoint rounds to f1 iff f1 is even
    }
    p.class_filter = n_filter > 0 ? class_filter : nullptr; p.n_filter = n_filter;
    p.max_det = max_det; p.max_wh = max_wh; p.out = out; p.counts = counts; p.kept_idx = kept_idx; p.M = M;
    p.MCp = pow2_at_least(M);
    p.C = 1 << 30;                                           // callers that know the class count set it
    p.prof = nullptr;
    return YFV2_OK;
}

// The fused decode+NMS launch: kernel variant and dynamic shared memory, from checked geometry and parameters
struct DecodeNmsLaunch {
    PostGeom g;
    NmsParams p;
    void (*kern)(PostGeom, NmsParams);
    size_t bytes;
};

int decode_nms_prepare(DecodeNmsLaunch& d, const float* const preds[6], int N, int H, int W, int A, int C, const double* anchors_host,
                       float conf_thres, double iou_thres, const int* class_filter, int n_filter, int max_det, float max_wh, float* out,
                       int* counts, int* kept_idx) {
    int rc = fill_geom(d.g, preds, N, H, W, A, C, anchors_host);
    if (rc) return rc;
    rc = fill_nms(d.p, d.g.M, conf_thres, iou_thres, class_filter, n_filter, max_det, max_wh, out, counts, kept_idx);
    if (rc) return rc;
    d.p.C = C;
    d.p.prof = g_nms_prof;
    const int fast = C > kCT ? 0 : (C == kCT && A == 3) ? 2 : 1;
    static void (*const kernels[2][3])(PostGeom, NmsParams) = {
        {decode_nms_kernel<false, 0>, decode_nms_kernel<false, 1>, decode_nms_kernel<false, 2>},
        {decode_nms_kernel<true, 0>, decode_nms_kernel<true, 1>, decode_nms_kernel<true, 2>}};
    d.kern = kernels[d.p.prof != nullptr][fast];
    // the warp-per-cell path stages 5A+C logits of 32 cells behind the NMS state
    d.bytes = nms_smem_bytes(d.p.M, d.p.MCp, d.p.max_det) + (fast ? 0 : (size_t)(5 * A + C) * kSStride * sizeof(float));
    if (d.bytes > kSmemCap) { set_error("decode_nms: %zu bytes of shared memory needed", d.bytes); return YFV2_EUNSUPPORTED; }
    return YFV2_OK;
}
}  // namespace

int decode_nms_check(const float* const preds[6], int N, int H, int W, int A, int C, const double* anchors_host, float conf_thres,
                     double iou_thres, const int* class_filter, int n_filter, int max_det, float max_wh, float* out, int* counts,
                     int* kept_idx) {
    DecodeNmsLaunch d;
    return decode_nms_prepare(d, preds, N, H, W, A, C, anchors_host, conf_thres, iou_thres, class_filter, n_filter, max_det, max_wh,
                              out, counts, kept_idx);
}
}  // namespace yfv2

using namespace yfv2;

extern "C" int yfv2_decode(const float* const preds[6], int N, int H, int W, int A, int C, const double* anchors_host,
                           float* out, void* stream) {
    PostGeom g;
    int rc = fill_geom(g, preds, N, H, W, A, C, anchors_host);
    if (rc) return rc;
    if (!out) { set_error("decode: null output"); return YFV2_EINVAL; }
    const int chunks0 = (g.hw[0] + kChunkCells - 1) / kChunkCells, chunks1 = (g.hw[1] + kChunkCells - 1) / kChunkCells;
    decode_kernel<<<dim3(chunks0 + chunks1, N), NT, 0, (cudaStream_t)stream>>>(g, out, chunks0);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_export_heads(const float* const preds[6], int N, int H, int W, int A, int C, float* out2, float* out3, void* stream) {
    PostGeom g;
    const double dummy[4 * kMaxA] = {0};
    int rc = fill_geom(g, preds, N, H, W, A, C, dummy);
    if (rc) return rc;
    if (!out2 || !out3) { set_error("export_heads: null output"); return YFV2_EINVAL; }
    const int chunks0 = (g.hw[0] + kChunkCells - 1) / kChunkCells, chunks1 = (g.hw[1] + kChunkCells - 1) / kChunkCells;
    export_head_kernel<<<dim3(chunks0 + chunks1, N), NT, 0, (cudaStream_t)stream>>>(g, out2, out3, chunks0);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_nms_workspace_bytes(int N, int M, int C, size_t* bytes) {
    (void)N; (void)M; (void)C;
    if (!bytes) return YFV2_EINVAL;
    *bytes = 0;       // the blocked greedy pass keeps all of its state in shared memory
    return YFV2_OK;
}

extern "C" int yfv2_nms(const float* dets, int N, int M, int C, float conf_thres, double iou_thres, const int* class_filter,
                        int n_filter, int max_det, float max_wh, float* out, int* counts, int* kept_idx, void* workspace,
                        void* stream) {
    (void)workspace;
    if (!dets || N <= 0 || C <= 0) { set_error("nms: bad arguments"); return YFV2_EINVAL; }
    NmsParams p;
    int rc = fill_nms(p, M, conf_thres, iou_thres, class_filter, n_filter, max_det, max_wh, out, counts, kept_idx);
    if (rc) return rc;
    p.C = C;
    const size_t bytes = nms_smem_bytes(p.M, p.MCp, p.max_det);
    if (bytes > kSmemCap) { set_error("nms: %zu bytes of shared memory needed", bytes); return YFV2_EUNSUPPORTED; }
    YFV2_CUDA(cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    nms_kernel<<<N, NT, bytes, (cudaStream_t)stream>>>(dets, C, p);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_decode_nms(const float* const preds[6], int N, int H, int W, int A, int C, const double* anchors_host,
                               float conf_thres, double iou_thres, const int* class_filter, int n_filter, int max_det,
                               float max_wh, float* out, int* counts, int* kept_idx, void* workspace, void* stream) {
    (void)workspace;
    DecodeNmsLaunch d;
    const int rc = decode_nms_prepare(d, preds, N, H, W, A, C, anchors_host, conf_thres, iou_thres, class_filter, n_filter, max_det,
                                      max_wh, out, counts, kept_idx);
    if (rc) return rc;
    YFV2_CUDA(cudaFuncSetAttribute(d.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d.bytes));
    {   // nothing is read before pdl_wait(), so overlapping the predecessor's tail is always safe
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)N); cfg.blockDim = dim3(NT); cfg.dynamicSmemBytes = d.bytes; cfg.stream = (cudaStream_t)stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = pdl_allowed() ? 1 : 0;
        YFV2_CUDA(cudaLaunchKernelEx(&cfg, d.kern, d.g, d.p));
    }
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

/* test / profiling hook: per-image clock64 ticks of the phases of decode_nms_kernel (see sort_and_suppress).  `dev_buf`: N x 16
 * int64 on the device, or NULL to switch the instrumented kernel off again.  Process-wide; not for concurrent use. */
extern "C" int yfv2_debug_nms_profile(long long* dev_buf) {
    g_nms_prof = dev_buf;
    return YFV2_OK;
}

namespace yfv2 {
namespace {
// yfv2_merge_regions (nmm false) and yfv2_merge_regions_nmm: the same checks, launches and layout; `who` names the call in errors.
int merge_regions_run(const char* who, bool nmm, const float* dets, const int* counts, const yfv2_region* regions, int T,
                      int max_det_in, int F, int H, int W, double thr, int metric, int max_det, double* out, int* out_counts,
                      int* kept_src, int* merged, void* stream) {
    if (!dets || !counts || !regions || !out || !out_counts) { set_error("%s: null dets / counts / regions / out / out_counts", who); return YFV2_EINVAL; }
    if (T < 1 || F < 1 || W < 1 || H < 1) { set_error("%s: need T, F, W, H >= 1 (T=%d F=%d W=%d H=%d)", who, T, F, W, H); return YFV2_EINVAL; }
    if (max_det_in < 1 || max_det_in > 4096 || max_det < 1 || max_det > 4096) {
        set_error("%s: max_det_in=%d and max_det=%d must be in 1..4096", who, max_det_in, max_det);
        return YFV2_EINVAL;
    }
    if (metric != 0 && metric != 1) { set_error("%s: metric=%d (0: IoU, 1: IoS)", who, metric); return YFV2_EINVAL; }
    if (thr != thr) { set_error("%s: thr is NaN", who); return YFV2_EINVAL; }
    if ((long long)T * max_det_in > INT_MAX) { set_error("%s: T * max_det_in = %lld rows exceeds 2^31 - 1", who, (long long)T * max_det_in); return YFV2_EINVAL; }
    int run = 0;                                                   // regions of the current frame
    for (int t = 0; t < T; ++t) {
        const yfv2_region& r = regions[t];
        const char* why = nullptr;
        if (r.w < 1 || r.h < 1) why = "w and h must be >= 1";
        else if (r.x0 < 0 || r.y0 < 0) why = "x0 and y0 must be >= 0";
        else if (r.frame < 0 || r.frame >= F) why = "frame outside [0, F)";
        else if (t && r.frame < regions[t - 1].frame) why = "frame index decreases (regions of a frame must be contiguous, frames ascending)";
        if (why) {
            set_error("%s: region %d: %s (frame %d of F=%d, x0 %d, y0 %d, %dx%d)", who, t, why, r.frame, F, r.x0, r.y0, r.w, r.h);
            return YFV2_EINVAL;
        }
        run = (t && r.frame == regions[t - 1].frame) ? run + 1 : 1;
        if (run > YFV2_MERGE_MAX_REGIONS || (long long)run * max_det_in > YFV2_NMS_MAX_CAND) {
            set_error("%s: region %d: frame %d has %d regions x max_det_in %d: more than %d regions or %d candidates", who, t,
                      r.frame, run, max_det_in, YFV2_MERGE_MAX_REGIONS, YFV2_NMS_MAX_CAND);
            return YFV2_EINVAL;
        }
    }
    // launches of whole frames: at most kMergeFrames frames and YFV2_MERGE_MAX_REGIONS regions each
    std::unique_ptr<MergeArgs> ap(new (std::nothrow) MergeArgs);  // 17 KB of kernel parameters: on the heap, not the stack
    if (!ap) { set_error("%s: host allocation failed", who); return YFV2_ENOMEM; }
    MergeArgs& a = *ap;
    a.dets = dets; a.counts = counts; a.out = out; a.out_counts = out_counts; a.kept_src = kept_src;
    a.thr = thr; a.W = W; a.H = H; a.max_det_in = max_det_in; a.max_det = max_det; a.metric = metric;
    int t = 0;
    for (int f0 = 0; f0 < F;) {
        int nf = 0, nr = 0, most = 0;
        const int t0 = t;
        while (f0 + nf < F && nf < kMergeFrames) {
            int e = t;
            while (e < T && regions[e].frame == f0 + nf) ++e;
            if (nr + (e - t) > YFV2_MERGE_MAX_REGIONS) break;
            a.rbeg[nf] = nr;
            for (int k = t; k < e; ++k) a.reg[nr + k - t] = make_int4(regions[k].x0, regions[k].y0, regions[k].w, regions[k].h);
            nr += e - t;
            most = std::max(most, e - t);
            t = e;
            ++nf;
        }
        a.rbeg[nf] = nr;
        a.f0 = f0; a.t0 = t0;
        const int slots = most * max_det_in;
        a.MCp = pow2_at_least(slots);
        a.KC = std::max(1, std::min(max_det, slots));
        const size_t bytes = nmm ? merge_nmm_smem_bytes(a.MCp, a.KC) : merge_smem_bytes(a.MCp, a.KC);
        if (bytes > kSmemCap) { set_error("%s: %zu bytes of shared memory needed", who, bytes); return YFV2_EUNSUPPORTED; }
        if (nmm) {
            YFV2_CUDA(cudaFuncSetAttribute(merge_regions_nmm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
            merge_regions_nmm_kernel<<<nf, NT, bytes, (cudaStream_t)stream>>>(a, merged);
        } else {
            YFV2_CUDA(cudaFuncSetAttribute(merge_regions_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
            merge_regions_kernel<<<nf, NT, bytes, (cudaStream_t)stream>>>(a);
        }
        YFV2_LAUNCH_CHECK();
        f0 += nf;
    }
    return YFV2_OK;
}
}  // namespace
}  // namespace yfv2

extern "C" int yfv2_merge_regions(const float* dets, const int* counts, const yfv2_region* regions, int T, int max_det_in, int F,
                                  int H, int W, double thr, int metric, int max_det, double* out, int* out_counts, int* kept_src,
                                  void* stream) {
    return yfv2::merge_regions_run("merge_regions", false, dets, counts, regions, T, max_det_in, F, H, W, thr, metric, max_det, out,
                                   out_counts, kept_src, nullptr, stream);
}

extern "C" int yfv2_merge_regions_nmm(const float* dets, const int* counts, const yfv2_region* regions, int T, int max_det_in,
                                      int F, int H, int W, double thr, int metric, int max_det, double* out, int* out_counts,
                                      int* kept_src, int* merged, void* stream) {
    return yfv2::merge_regions_run("merge_regions_nmm", true, dets, counts, regions, T, max_det_in, F, H, W, thr, metric, max_det,
                                   out, out_counts, kept_src, merged, stream);
}
