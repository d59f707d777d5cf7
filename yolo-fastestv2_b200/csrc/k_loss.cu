// K8 / K9 — training loss of Yolo-FastestV2 on the device: target matching, CIoU / BCE / CE, and d(loss)/d(preds).
//
//   build_target  <- reference utils/loss.py:53-124   (YOLOv5-style anchor matching with 4-neighbour offsets)
//   ciou          <- reference utils/loss.py:8-51     (x1y1x2y2=False, CIoU=True; runs in fp64 because the anchors are
//                                                      float64, loss.py:59-60,160-161)
//   compute_loss  <- reference utils/loss.py:130-208  (balance [1.0, 0.4]; gains 3.2 / 64 / 32; obj target is the constant 1)
//
// The reference does this with ~60 small host-launched tensor ops plus autograd; here it is five launches:
//   1. build_target_kernel   one CTA per pyramid level: flags for all (offset, anchor, target) candidates, ORDERED
//                            compaction (so rows come out in the reference's order: offset-major, anchor, target)
//   2. mark_obj_kernel       scatter the obj targets into a byte map
//   3. loss_rows_kernel      per matched row: CIoU term and softmax-CE term (+ their gradients, atomics into dpreds)
//   4. obj_loss_kernel       dense BCE-with-logits over every obj logit (+ gradient), per-block partial sums in fp64
//   5. finalize_kernel       fixed-order fp64 reductions -> (lbox, lobj, lcls, loss)
// dtype flow follows the reference: grid coordinates / tbox in fp32, anchor ratio test and the CIoU in fp64, except the terms of
// the fp32 target box alone (its corners, area, centre and atan(w/h)), which are fp32 there too.
#include "common.cuh"

namespace yfv2 {
namespace {

constexpr int kLossThreads = 256;
constexpr int kMaxA = 8;
constexpr double kPi = 3.14159265358979323846;

struct LossGeom {
    int N, A, C, nt;
    int h[2], w[2];
    double anc[2][kMaxA][2];        // anchors / stride (fp64), loss.py:84
    const float* reg[2]; const float* obj[2]; const float* cls[2];
    float* dreg[2]; float* dobj[2]; float* dcls[2];     // may be null (no gradients wanted)
};

struct Rows {                         // one level's matched rows, capacity 5*A*nt
    int* b; int* a; int* gj; int* gi; int* cls;
    float* tbox;                      // [cap,4]
    double* anch;                     // [cap,2]
    double* t_box;                    // per-row (1 - ciou)
    double* t_cls;                    // per-row cross entropy
};

struct LossWs {
    Rows rows[2];
    int* counts;                      // [2]
    unsigned char* tobj[2];           // [N,A,h,w] byte maps
    double* obj_partials;             // [2][nblocks]
    int obj_blocks;
};

// ---- 1. build_target ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool candidate(const LossGeom& g, int lv, const float* __restrict__ targets, int o, int a, int t,
                                          float& gx, float& gy, float& gw, float& gh) {
    const float wf = (float)g.w[lv], hf = (float)g.h[lv];
    const float* tr = targets + (size_t)t * 6;
    gx = __fmul_rn(tr[2], wf); gy = __fmul_rn(tr[3], hf);          // gt = targets * gain, fp32 (loss.py:87-89)
    gw = __fmul_rn(tr[4], wf); gh = __fmul_rn(tr[5], hf);
    const double rw = (double)gw / g.anc[lv][a][0], rh = (double)gh / g.anc[lv][a][1];     // fp64 ratio (loss.py:93)
    const double m = fmax(fmax(rw, 1.0 / rw), fmax(rh, 1.0 / rh));
    if (!(m < 2.0)) return false;                                     // loss.py:94
    if (o == 0) return true;
    const float gxi = __fsub_rn(wf, gx), gyi = __fsub_rn(hf, gy);    // gain[[2,3]] - gxy (loss.py:100)
    switch (o) {                                                      // loss.py:101-102
        case 1: return fmodf(gx, 1.0f) < 0.5f && gx > 1.0f;
        case 2: return fmodf(gy, 1.0f) < 0.5f && gy > 1.0f;
        case 3: return fmodf(gxi, 1.0f) < 0.5f && gxi > 1.0f;
        default: return fmodf(gyi, 1.0f) < 0.5f && gyi > 1.0f;
    }
}

__global__ void __launch_bounds__(1024)
build_target_kernel(LossGeom g, const float* __restrict__ targets, LossWs ws) {
    const int lv = blockIdx.x;
    const Rows R = ws.rows[lv];
    const int total = 5 * g.A * g.nt;
    __shared__ int warp_cnt[32];
    __shared__ int base_s;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c0 = 0; c0 < total; c0 += 1024) {
        const int idx = c0 + threadIdx.x;
        bool flag = false;
        int o = 0, a = 0, t = 0;
        float gx = 0, gy = 0, gw = 0, gh = 0;
        if (idx < total) {
            o = idx / (g.A * g.nt);
            const int r = idx - o * (g.A * g.nt);
            a = r / g.nt; t = r - a * g.nt;
            flag = candidate(g, lv, targets, o, a, t, gx, gy, gw, gh);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        int before = base_s;
        for (int wI = 0; wI < warp; ++wI) before += warp_cnt[wI];
        if (flag) {
            const int row = before + __popc(bal & ((1u << lane) - 1u));
            const float offx = o == 1 ? 0.5f : (o == 3 ? -0.5f : 0.f);
            const float offy = o == 2 ? 0.5f : (o == 4 ? -0.5f : 0.f);
            int gi = (int)__fsub_rn(gx, offx), gj = (int)__fsub_rn(gy, offy);          // .long(): truncation (loss.py:114)
            gi = min(max(gi, 0), g.w[lv] - 1); gj = min(max(gj, 0), g.h[lv] - 1);      // clamp_ BEFORE tbox (loss.py:119-120)
            const float* tr = targets + (size_t)t * 6;
            R.b[row] = (int)tr[0]; R.cls[row] = (int)tr[1];
            R.a[row] = a; R.gj[row] = gj; R.gi[row] = gi;
            R.tbox[4 * row + 0] = __fsub_rn(gx, (float)gi); R.tbox[4 * row + 1] = __fsub_rn(gy, (float)gj);
            R.tbox[4 * row + 2] = gw; R.tbox[4 * row + 3] = gh;
            R.anch[2 * row + 0] = g.anc[lv][a][0]; R.anch[2 * row + 1] = g.anc[lv][a][1];
        }
        __syncthreads();
        if (threadIdx.x == 0) { int s = 0; for (int wI = 0; wI < 32; ++wI) s += warp_cnt[wI]; base_s += s; }
        __syncthreads();
    }
    if (threadIdx.x == 0) ws.counts[lv] = base_s;
}

// ---- 2. obj target map -------------------------------------------------------------------------------------------------
__global__ void mark_obj_kernel(LossGeom g, LossWs ws) {
    const int lv = blockIdx.y;
    const Rows R = ws.rows[lv];
    const int m = ws.counts[lv];
    const int hw = g.h[lv] * g.w[lv];
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x)
        ws.tobj[lv][((size_t)R.b[r] * g.A + R.a[r]) * hw + R.gj[r] * g.w[lv] + R.gi[r]] = 1;       // tobj[b,a,gj,gi] = 1.0 (loss.py:177)
}

// ---- 3. matched rows: CIoU + CE ---------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// acc += t * d min(a, b)/da  and  acc += t * d max(a, b)/da, with torch.min / torch.max's derivative: a tie gives each argument
// half (loss.py:23,33).  Off ties the arithmetic is that of a plain `if (a < b) acc += t`.
__device__ __forceinline__ void add_dmin(double& acc, double a, double b, double t) { if (a < b) acc += t; else if (a == b) acc += 0.5 * t; }
__device__ __forceinline__ void add_dmax(double& acc, double a, double b, double t) { if (a > b) acc += t; else if (a == b) acc += 0.5 * t; }

__global__ void __launch_bounds__(kLossThreads)
loss_rows_kernel(LossGeom g, LossWs ws) {
    const int lv = blockIdx.y;
    const Rows R = ws.rows[lv];
    const int m = ws.counts[lv];
    const int h = g.h[lv], w = g.w[lv], hw = h * w, A = g.A, C = g.C;
    const double gbox = m > 0 ? -3.2 / (double)m : 0.0;            // d(lbox*3.2)/d(ciou_r): lbox += mean(1 - ciou) (loss.py:163,203)
    const float gcls = m > 0 ? 32.0f / ((float)m * (float)C) : 0.f; // d(lcls*32)/d(CE_r): lcls += mean(CE)/classes (loss.py:198,205)
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
        const int b = R.b[r], a = R.a[r], gj = R.gj[r], gi = R.gi[r];
        const size_t cell = (size_t)gj * w + gi;
        // ---- box ----
        const float* rp = g.reg[lv] + ((size_t)b * 4 * A + 4 * a) * hw + cell;
        const float sx = sigmoidf_(rp[0]), sy = sigmoidf_(rp[hw]), sw = sigmoidf_(rp[2 * (size_t)hw]), sh = sigmoidf_(rp[3 * (size_t)hw]);
        const double px = (double)(sx * 2.0f - 0.5f), py = (double)(sy * 2.0f - 0.5f);            // fp32 then promoted (loss.py:159)
        const double aw = R.anch[2 * r], ah = R.anch[2 * r + 1];
        const float tw2 = sw * 2.0f, th2 = sh * 2.0f;
        const double pw = (double)(tw2 * tw2) * aw, ph = (double)(th2 * th2) * ah;                // loss.py:160
        const double b1x1 = px - pw / 2, b1x2 = px + pw / 2, b1y1 = py - ph / 2, b1y2 = py + ph / 2;
        // tbox is fp32 in the reference, so what it computes from the target box alone is fp32 and promoted where it meets the
        // fp64 predicted box: the corners, w2 * h2, the centre sums and atan(w2 / h2) (loss.py:19-20,28-29,42,46).  An fp64 atan
        // would make D exactly 0 for a prediction with the target's aspect, and 0/0 in alpha where the prediction IS the target.
        const float tx = R.tbox[4 * r], ty = R.tbox[4 * r + 1], tw = R.tbox[4 * r + 2], th = R.tbox[4 * r + 3];
        const float b2x1f = __fsub_rn(tx, __fmul_rn(tw, 0.5f)), b2x2f = __fadd_rn(tx, __fmul_rn(tw, 0.5f));
        const float b2y1f = __fsub_rn(ty, __fmul_rn(th, 0.5f)), b2y2f = __fadd_rn(ty, __fmul_rn(th, 0.5f));
        const float w2f = __fsub_rn(b2x2f, b2x1f), h2f = __fsub_rn(b2y2f, b2y1f);
        const double b2x1 = b2x1f, b2x2 = b2x2f, b2y1 = b2y1f, b2y2 = b2y2f;
        const double iw_raw = fmin(b1x2, b2x2) - fmax(b1x1, b2x1), ih_raw = fmin(b1y2, b2y2) - fmax(b1y1, b2y1);
        const double iw = fmax(iw_raw, 0.0), ih = fmax(ih_raw, 0.0);
        const double inter = iw * ih;
        const double w1 = b1x2 - b1x1, h1 = b1y2 - b1y1;
        const double uni = (w1 * h1 + 1e-16) + (double)__fmul_rn(w2f, h2f) - inter;
        const double iou = inter / uni;
        const double cw = fmax(b1x2, b2x2) - fmin(b1x1, b2x1), chh = fmax(b1y2, b2y2) - fmin(b1y1, b2y1);
        const double c2 = cw * cw + chh * chh + 1e-16;
        const double Sx = (double)__fadd_rn(b2x1f, b2x2f) - (b1x1 + b1x2), Sy = (double)__fadd_rn(b2y1f, b2y2f) - (b1y1 + b1y2);
        const double rho2 = Sx * Sx / 4 + Sy * Sy / 4;
        const double D = (double)atanf(__fdiv_rn(w2f, h2f)) - atan(w1 / h1);
        const double v = (4.0 / (kPi * kPi)) * D * D;
        const double alpha = v / (1.0 - iou + v);                     // no_grad (loss.py:47-48)
        const double ciou = iou - (rho2 / c2 + v * alpha);
        R.t_box[r] = 1.0 - ciou;
        if (g.dreg[lv]) {
            // reverse mode by hand; G* = d(ciou)/d(.)
            const double Ginter = 1.0 / uni + inter / (uni * uni);    // through iou = inter / (U0 - inter)
            const double GU0 = -inter / (uni * uni);
            const double Gc2 = rho2 / (c2 * c2);
            const double Grho = -1.0 / c2;
            const double Gv = -alpha;
            double gx1 = 0, gx2 = 0, gy1 = 0, gy2 = 0;                // d(ciou)/d(b1 corners)
            // intersection
            // (the clamp's derivative at iw_raw == 0 is 1, as torch's clamp(0) has it)
            if (iw_raw >= 0.0) { const double t = Ginter * ih; add_dmin(gx2, b1x2, b2x2, t); add_dmax(gx1, b1x1, b2x1, -t); }
            if (ih_raw >= 0.0) { const double t = Ginter * iw; add_dmin(gy2, b1y2, b2y2, t); add_dmax(gy1, b1y1, b2y1, -t); }
            // U0 = w1*h1 + ...
            gx2 += GU0 * h1; gx1 -= GU0 * h1; gy2 += GU0 * w1; gy1 -= GU0 * w1;
            // enclosing box
            { const double t = Gc2 * 2 * cw; add_dmax(gx2, b1x2, b2x2, t); add_dmin(gx1, b1x1, b2x1, -t); }
            { const double t = Gc2 * 2 * chh; add_dmax(gy2, b1y2, b2y2, t); add_dmin(gy1, b1y1, b2y1, -t); }
            // centre distance
            gx1 += Grho * (-Sx / 2); gx2 += Grho * (-Sx / 2); gy1 += Grho * (-Sy / 2); gy2 += Grho * (-Sy / 2);
            // aspect term v = c * (atan(w2/h2) - atan(w1/h1))^2, through atan' = 1 / (1 + x*x) and d(w1/h1) = (1/h1, -(w1/h1)/h1)
            // as autograd takes it.  Where h1 is 0 in fp64 (a predicted height below the rounding of py) that is 0 * inf = NaN in the
            // reference, and so here; the closed form D*w1 / (w1^2 + h1^2) would be finite.
            const double x1 = w1 / h1;
            const double Gat = -Gv * (8.0 / (kPi * kPi)) * D / (1.0 + x1 * x1);    // d(ciou)/d(w1/h1)
            const double Gw1 = Gat / h1, Gh1 = -Gat * (x1 / h1);
            gx2 += Gw1; gx1 -= Gw1; gy2 += Gh1; gy1 -= Gh1;
            // corners -> (px, py, pw, ph)
            const double gpx = gx1 + gx2, gpy = gy1 + gy2, gpw = (gx2 - gx1) / 2, gph = (gy2 - gy1) / 2;
            // -> logits; the xy branch is fp32 in the reference graph, the wh branch fp64 until the sigmoid
            float* dp = g.dreg[lv] + ((size_t)b * 4 * A + 4 * a) * hw + cell;
            const float dsx = (float)(gbox * gpx) * 2.0f * sx * (1.0f - sx);
            const float dsy = (float)(gbox * gpy) * 2.0f * sy * (1.0f - sy);
            const float dsw = (float)(gbox * gpw * aw * 2.0 * (double)tw2) * 2.0f * sw * (1.0f - sw);
            const float dsh = (float)(gbox * gph * ah * 2.0 * (double)th2) * 2.0f * sh * (1.0f - sh);
            atomicAdd(dp, dsx); atomicAdd(dp + hw, dsy); atomicAdd(dp + 2 * (size_t)hw, dsw); atomicAdd(dp + 3 * (size_t)hw, dsh);
        }
        // ---- class: softmax cross entropy over C logits at (b, :, gj, gi) (loss.py:194-198) ----
        if (C > 1) {
            const float* cp = g.cls[lv] + (size_t)b * C * hw + cell;
            float mx = -INFINITY;
            for (int c = 0; c < C; ++c) mx = fmaxf(mx, cp[(size_t)c * hw]);
            float sum = 0.f;
            for (int c = 0; c < C; ++c) sum += expf(cp[(size_t)c * hw] - mx);
            const float lse = mx + logf(sum);
            const int tc = R.cls[r];
            R.t_cls[r] = (double)(lse - cp[(size_t)tc * hw]);
            if (g.dcls[lv]) {
                float* dc = g.dcls[lv] + (size_t)b * C * hw + cell;
                for (int c = 0; c < C; ++c) {
                    const float pr = expf(cp[(size_t)c * hw] - lse);
                    atomicAdd(dc + (size_t)c * hw, gcls * (pr - (c == tc ? 1.f : 0.f)));
                }
            }
        } else {
            R.t_cls[r] = 0.0;
        }
    }
}

// ---- 4. dense objectness BCE ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLossThreads)
obj_loss_kernel(LossGeom g, LossWs ws) {
    const int lv = blockIdx.y;
    const size_t total = (size_t)g.N * g.A * g.h[lv] * g.w[lv];
    const float balance = lv == 0 ? 1.0f : 0.4f;                     // loss.py:131
    const float gscale = 64.0f * balance / (float)total;             // d(lobj*64)/d(element): BCE mean * balance (loss.py:181,204)
    double acc = 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const float x = g.obj[lv][i];
        const float t = ws.tobj[lv][i] ? 1.0f : 0.0f;
        // BCEWithLogits, pos_weight 1: (1-t)*x + log1p(exp(-|x|)) + max(-x, 0)
        acc += (double)((1.0f - t) * x + log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.0f));
        if (g.dobj[lv]) g.dobj[lv][i] = gscale * (sigmoidf_(x) - t);
    }
    __shared__ double red[kLossThreads];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = kLossThreads / 2; s > 0; s >>= 1) { if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s]; __syncthreads(); }
    if (threadIdx.x == 0) ws.obj_partials[(size_t)lv * ws.obj_blocks + blockIdx.x] = red[0];
}

// ---- 5. finalize ---------------------------------------------------------------------------------------------------------
__device__ double block_sum(const double* v, int n, double* red) {
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += kLossThreads) acc += v[i];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = kLossThreads / 2; s > 0; s >>= 1) { if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s]; __syncthreads(); }
    const double r = red[0];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kLossThreads)
finalize_kernel(LossGeom g, LossWs ws, float* __restrict__ losses) {
    __shared__ double red[kLossThreads];
    float lbox = 0.f, lobj = 0.f, lcls = 0.f;
    for (int lv = 0; lv < 2; ++lv) {
        const int m = ws.counts[lv];
        const double sb = block_sum(ws.rows[lv].t_box, m, red);
        const double sc = block_sum(ws.rows[lv].t_cls, m, red);
        const double so = block_sum(ws.obj_partials + (size_t)lv * ws.obj_blocks, ws.obj_blocks, red);
        const double total = (double)g.N * g.A * g.h[lv] * g.w[lv];
        if (m > 0) {
            lbox += (float)(sb / m);                                    // lbox += (1 - ciou).mean()  (fp64 mean added into fp32)
            if (g.C > 1) lcls += (float)(sc / m) / (float)g.C;          // lcls += CE.mean() / classes
        }
        lobj += (float)(so / total) * (lv == 0 ? 1.0f : 0.4f);
    }
    if (threadIdx.x == 0) {
        lbox *= 3.2f; lobj *= 64.f; lcls *= 32.f;                      // loss.py:203-205
        losses[0] = lbox; losses[1] = lobj; losses[2] = lcls; losses[3] = lbox + lobj + lcls;
    }
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

int carve(LossWs& ws, unsigned char* base, size_t* total, int N, int A, const int h[2], const int w[2], int nt) {
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
    const size_t cap = (size_t)5 * A * (nt > 0 ? nt : 1);
    for (int lv = 0; lv < 2; ++lv) {
        Rows& R = ws.rows[lv];
        R.b = (int*)take(cap * 4); R.a = (int*)take(cap * 4); R.gj = (int*)take(cap * 4); R.gi = (int*)take(cap * 4); R.cls = (int*)take(cap * 4);
        R.tbox = (float*)take(cap * 16); R.anch = (double*)take(cap * 16);
        R.t_box = (double*)take(cap * 8); R.t_cls = (double*)take(cap * 8);
    }
    ws.counts = (int*)take(2 * sizeof(int));
    for (int lv = 0; lv < 2; ++lv) ws.tobj[lv] = take((size_t)N * A * h[lv] * w[lv]);
    ws.obj_blocks = 256;
    ws.obj_partials = (double*)take((size_t)2 * ws.obj_blocks * sizeof(double));
    *total = off;
    return 0;
}

int fill(LossGeom& g, const float* const preds[6], float* const dpreds[6], int N, int H, int W, int A, int C, int nt,
         const double* anchors_host) {
    if (!preds || !anchors_host || N <= 0 || A <= 0 || A > kMaxA || C <= 0 || H % 32 || W % 32 || H <= 0 || W <= 0 || nt < 0) {
        set_error("loss: bad arguments (N=%d H=%d W=%d A=%d C=%d nt=%d)", N, H, W, A, C, nt);
        return YFV2_EINVAL;
    }
    g.N = N; g.A = A; g.C = C; g.nt = nt;
    for (int lv = 0; lv < 2; ++lv) {
        const int s = lv ? 32 : 16;
        g.h[lv] = H / s; g.w[lv] = W / s;
        const double stride = (double)W / (double)g.w[lv];           // cfg["width"]/w (loss.py:81)
        for (int a = 0; a < A; ++a) {
            g.anc[lv][a][0] = anchors_host[(lv * A + a) * 2] / stride;
            g.anc[lv][a][1] = anchors_host[(lv * A + a) * 2 + 1] / stride;
        }
        g.reg[lv] = preds[3 * lv]; g.obj[lv] = preds[3 * lv + 1]; g.cls[lv] = preds[3 * lv + 2];
        if (!g.reg[lv] || !g.obj[lv] || !g.cls[lv]) { set_error("loss: null head tensor"); return YFV2_EINVAL; }
        g.dreg[lv] = dpreds ? dpreds[3 * lv] : nullptr; g.dobj[lv] = dpreds ? dpreds[3 * lv + 1] : nullptr; g.dcls[lv] = dpreds ? dpreds[3 * lv + 2] : nullptr;
    }
    return YFV2_OK;
}
}  // namespace
}  // namespace yfv2

using namespace yfv2;

extern "C" int yfv2_loss_workspace_bytes(int N, int H, int W, int A, int C, int nt, size_t* bytes) {
    (void)C;
    if (!bytes || N <= 0 || H <= 0 || W <= 0 || H % 32 || W % 32 || A <= 0 || nt < 0) { set_error("loss_workspace_bytes: bad arguments"); return YFV2_EINVAL; }
    LossWs ws;
    const int h[2] = {H / 16, H / 32}, w[2] = {W / 16, W / 32};
    carve(ws, nullptr, bytes, N, A, h, w, nt);
    return YFV2_OK;
}

extern "C" int yfv2_compute_loss(const float* const preds[6], const float* targets, int nt, int N, int H, int W, int A, int C,
                                 const double* anchors_host, float* losses, float* const dpreds[6], void* workspace, void* stream) {
    LossGeom g;
    int rc = fill(g, preds, dpreds, N, H, W, A, C, nt, anchors_host);
    if (rc) return rc;
    if (!losses || !workspace || (nt > 0 && !targets)) { set_error("compute_loss: null argument"); return YFV2_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    LossWs ws;
    size_t total = 0;
    carve(ws, (unsigned char*)workspace, &total, N, A, g.h, g.w, nt);
    YFV2_CUDA(cudaMemsetAsync(ws.counts, 0, 2 * sizeof(int), s));
    for (int lv = 0; lv < 2; ++lv) {
        const size_t hw = (size_t)g.h[lv] * g.w[lv];
        YFV2_CUDA(cudaMemsetAsync(ws.tobj[lv], 0, (size_t)N * A * hw, s));
        if (g.dreg[lv]) YFV2_CUDA(cudaMemsetAsync(g.dreg[lv], 0, (size_t)N * 4 * A * hw * sizeof(float), s));
        if (g.dcls[lv]) YFV2_CUDA(cudaMemsetAsync(g.dcls[lv], 0, (size_t)N * C * hw * sizeof(float), s));
    }
    if (nt > 0) {
        build_target_kernel<<<2, 1024, 0, s>>>(g, targets, ws);
        YFV2_LAUNCH_CHECK();
        const int rb = (5 * A * nt + kLossThreads - 1) / kLossThreads;
        mark_obj_kernel<<<dim3(rb < 512 ? rb : 512, 2), kLossThreads, 0, s>>>(g, ws);
        YFV2_LAUNCH_CHECK();
        loss_rows_kernel<<<dim3(rb < 1024 ? rb : 1024, 2), kLossThreads, 0, s>>>(g, ws);
        YFV2_LAUNCH_CHECK();
    }
    obj_loss_kernel<<<dim3(ws.obj_blocks, 2), kLossThreads, 0, s>>>(g, ws);
    YFV2_LAUNCH_CHECK();
    finalize_kernel<<<1, kLossThreads, 0, s>>>(g, ws, losses);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// Copies one level's matched rows out (tests): idx [4,cap] int32 rows (b,a,gj,gi), tbox [cap,4], anch [cap,2] fp64, tcls [cap].
extern "C" int yfv2_loss_read_targets(const void* workspace, int level, int N, int H, int W, int A, int nt, int* count_host,
                                      int* idx, float* tbox, double* anch, int* tcls, void* stream) {
    if (!workspace || level < 0 || level > 1 || !count_host) { set_error("loss_read_targets: bad arguments"); return YFV2_EINVAL; }
    LossWs ws;
    size_t total = 0;
    const int h[2] = {H / 16, H / 32}, w[2] = {W / 16, W / 32};
    carve(ws, (unsigned char*)workspace, &total, N, A, h, w, nt);
    cudaStream_t s = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemcpyAsync(count_host, ws.counts + level, sizeof(int), cudaMemcpyDeviceToHost, s));
    YFV2_CUDA(cudaStreamSynchronize(s));
    const size_t m = (size_t)*count_host, cap = (size_t)5 * A * (nt > 0 ? nt : 1);
    if (m > cap) { set_error("loss_read_targets: corrupt count"); return YFV2_EINVAL; }
    const Rows& R = ws.rows[level];
    if (idx) {
        YFV2_CUDA(cudaMemcpyAsync(idx, R.b, m * 4, cudaMemcpyDeviceToDevice, s));
        YFV2_CUDA(cudaMemcpyAsync(idx + cap, R.a, m * 4, cudaMemcpyDeviceToDevice, s));
        YFV2_CUDA(cudaMemcpyAsync(idx + 2 * cap, R.gj, m * 4, cudaMemcpyDeviceToDevice, s));
        YFV2_CUDA(cudaMemcpyAsync(idx + 3 * cap, R.gi, m * 4, cudaMemcpyDeviceToDevice, s));
    }
    if (tbox) YFV2_CUDA(cudaMemcpyAsync(tbox, R.tbox, m * 16, cudaMemcpyDeviceToDevice, s));
    if (anch) YFV2_CUDA(cudaMemcpyAsync(anch, R.anch, m * 16, cudaMemcpyDeviceToDevice, s));
    if (tcls) YFV2_CUDA(cudaMemcpyAsync(tcls, R.cls, m * 4, cudaMemcpyDeviceToDevice, s));
    return YFV2_OK;
}
