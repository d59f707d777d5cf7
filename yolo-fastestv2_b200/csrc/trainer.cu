// Native training step (SURVEY 8 rows a13 / 8b): the train-mode forward and the backward of the whole network as ONE C-ABI
// call each, instead of ~250 torch.autograd.Function nodes composed op by op from Python (model/train_ops.py) with eager
// torch kernels for channel shuffle / split / concat in between.
//
// Reference: what nn.Module.train() + autograd do for train.py:105-110 over model/detector.py:21-31, backbone/shufflenetv2.py:19-63,
// 97-109 and fpn.py:5-64.  The network is laid out once, at yfv2_trainer_create, as a static program over an activation arena:
//   * parameters are indexed in `model.parameters()` order (module definition order: in a stride-2 block branch_main comes before
//     branch_proj, the FPN registers conv1x1_2, conv1x1_3, cls_head_2, reg_head_2, reg_head_3, cls_head_3), BatchNorm layers in
//     the same order as yfv2_pack_weights takes their running statistics;
//   * every op's output and its gradient own a slice of the caller's workspace, so the forward keeps exactly what the backward
//     needs and nothing is allocated per step;
//   * channel_shuffle + split + concat of a stride-1 block are two strided channel copies (K_ODD: the odd channels feed
//     branch_main; K_CATE: [even channels | branch_main output]); their backward writes disjoint halves of the input gradient;
//   * a tensor with several consumers (the input of a stride-2 block, C2, C3, S2, S3, the head features feeding obj and cls) gets
//     the gradient of the consumer that runs first in the backward by assignment and the others by accumulation through a
//     scratch tensor; the shared output convolutions (used at both pyramid levels) accumulate their weight gradients the same way.
// The arithmetic is the training operators of k_train.cu: the step is the list of their describe_* records.  Gradients of all 225
// parameters leave in ONE flat buffer in parameter order (the bucket train_ddp.py all-reduces), either assigned or accumulated.
//
// Fine-tuning mode (yfv2_trainer_set_mode): what autograd does for parameters with requires_grad=False and BatchNorm modules in
// .eval() inside a train-mode model.  The static program stays; the mode only selects, per op, the kernels and outputs:
//   * rg(tensor): the tensor depends on a trainable parameter.  rg(image) = false, rg(y) = rg(a) | rg(b) | (the op owns a trainable
//     parameter).  An op's backward runs iff rg(y); it writes d(a) iff rg(a) and a parameter gradient iff that parameter is trainable.
//     Every consumer of an rg tensor has an rg output, so the first-consumer-assigns rule above holds unchanged;
//   * an eval-mode BatchNorm normalises with the running statistics, leaves them alone and has no batch-mean terms in its backward;
//   * the flat buffer holds the trainable parameters only, in parameter order (train_ddp.FlatGradBucket's layout).
#include <algorithm>
#include <cstdlib>
#include <new>
#include <vector>

#include "common.cuh"

namespace yfv2 {
namespace {

enum Kind { K_STEM, K_BN, K_POOL, K_PW, K_DW, K_UP, K_ODD, K_CATE, K_CAT2 };

struct Ten {
    long long off, goff;     // activation / gradient offsets (floats) in the workspace; -1 for external tensors
    int C, H, W;
    int ext;                 // >= 0: head tensor `ext` (caller's preds / dpreds); -2: the input image
    int last_use;            // index of the last op that reads it (that op's backward runs first: it assigns the gradient)
    bool partial;            // consumed by a K_ODD / K_CATE pair writing disjoint halves of the gradient
};

struct Op {
    int kind;
    int a, b, y;             // tensor ids: inputs a [, b], output y
    int pw, pg, pb, pbias;   // parameter indices: weight, BN gamma, BN beta, conv bias (-1: none)
    int bn;                  // BatchNorm layer index (running statistics)
    int relu, ks, stride, M;
    long long aux;           // workspace offset of op-private storage (BN: mean | invstd | fp64 scratch; pool: argmax indices)
};

struct CB { int w, g, b, bn; };      // conv weight + its BatchNorm (gamma, beta, layer index)

// what one op's backward does under the current mode (yfv2_trainer_debug_backward)
struct BwdOp { bool run, da, db, dw, dbias, dgamma, dbeta, bn_eval; };

}  // namespace
}  // namespace yfv2

struct yfv2_trainer {
    int device, N, H, W, A, C;
    std::vector<yfv2::Ten> tens;
    std::vector<yfv2::Op> ops;
    std::vector<long long> poff;         // offset of every parameter's gradient in the flat buffer
    std::vector<long long> pnumel;
    long long ptotal = 0;
    long long ws_floats = 0;
    long long gflat_off = 0, scratch_off = 0, pscratch_off = 0, wscratch_off = 0, pscratch_floats = 0;
    int x_ten = -1;
    int out_ten[6];
    // fine-tuning mode: the current one, and the one the last forward ran under (a backward must see the same)
    std::vector<unsigned char> trainable, bn_eval, fwd_trainable, fwd_bn_eval;
    std::vector<yfv2::BwdOp> bwd;        // per op, from the current mode
    std::vector<long long> coff;         // offset of every parameter's gradient in the caller's flat buffer; -1: frozen
    long long ctotal = 0;
    unsigned long long mode_hash = 0;
    // CUDA-graph replay of the two static programs (~1000 launches per step otherwise: the step is host-bound at 8 GPUs): a
    // program is captured on a private stream the first time a set of pointers is seen and replayed while they stay the same
    struct GraphSlot { cudaGraphExec_t exec = nullptr; unsigned long long key = 0; };
    GraphSlot g_fwd, g_bwd[2];
    cudaStream_t cap_stream = nullptr;
};

namespace yfv2 {
namespace {

struct Builder {
    yfv2_trainer& t;
    int nbn = 0;
    explicit Builder(yfv2_trainer& tr) : t(tr) {}
    long long alloc(long long floats) { const long long o = t.ws_floats; t.ws_floats += (floats + 63) & ~63LL; return o; }
    int param(long long numel) { t.poff.push_back(t.ptotal); t.pnumel.push_back(numel); t.ptotal += numel; return (int)t.poff.size() - 1; }
    CB conv_bn(long long wnumel, int C) { CB c; c.w = param(wnumel); c.g = param(C); c.b = param(C); c.bn = nbn++; return c; }
    int ten(int C, int H, int W, int ext = -1) {
        Ten x{};
        x.C = C; x.H = H; x.W = W; x.ext = ext; x.last_use = -1; x.partial = false;
        if (ext == -1) { x.off = alloc((long long)t.N * C * H * W); x.goff = alloc((long long)t.N * C * H * W); }
        else { x.off = -1; x.goff = -1; }
        t.tens.push_back(x);
        return (int)t.tens.size() - 1;
    }
    int push(Op o) {
        const int id = (int)t.ops.size();
        if (o.a >= 0) t.tens[o.a].last_use = id;
        if (o.b >= 0) t.tens[o.b].last_use = id;
        t.ops.push_back(o);
        return o.y;
    }
    static Op blank(int kind) { Op o{}; o.kind = kind; o.a = o.b = o.y = -1; o.pw = o.pg = o.pb = o.pbias = -1; o.bn = -1; return o; }

    int bn(int x, const CB& c, bool relu) {
        const Ten& X = t.tens[x];
        Op o = blank(K_BN);
        o.a = x; o.y = ten(X.C, X.H, X.W); o.pg = c.g; o.pb = c.b; o.bn = c.bn; o.relu = relu ? 1 : 0;
        o.aux = alloc(6LL * X.C);                         // 2C doubles (fp64 partial sums) | mean[C] | invstd[C]
        return push(o);
    }
    int pw(int x, int w, int M, int bias = -1, int ext = -1) {
        const Ten& X = t.tens[x];
        Op o = blank(K_PW);
        o.a = x; o.y = ten(M, X.H, X.W, ext); o.pw = w; o.pbias = bias; o.M = M;
        return push(o);
    }
    int dw(int x, int w, int ks, int stride) {
        const Ten& X = t.tens[x];
        const int Ho = (X.H + 2 * (ks / 2) - ks) / stride + 1, Wo = (X.W + 2 * (ks / 2) - ks) / stride + 1;
        Op o = blank(K_DW);
        o.a = x; o.y = ten(X.C, Ho, Wo); o.pw = w; o.ks = ks; o.stride = stride;
        return push(o);
    }
    int pw_bn(int x, const CB& c, int M, bool relu) { return bn(pw(x, c.w, M), c, relu); }
    int dw_bn(int x, const CB& c, int ks, int stride, bool relu) { return bn(dw(x, c.w, ks, stride), c, relu); }
};

constexpr long long kWScratchFloats = 4LL << 20;      // per-block partial weight gradients of one layer (16 MB)
constexpr int kStageRepeats[3] = {4, 8, 4};
constexpr int kStageOut[3] = {48, 96, 192};

void build(yfv2_trainer& t) {
    Builder b(t);
    // ---- parameter layout, module definition order -----------------------------------------------------------------
    const CB first = b.conv_bn(24 * 27, 24);
    struct Blk { CB pw1, dw, pw2, pdw, ppw; int K, stride; } blk[16];
    {
        int bi = 0, cin = 24;
        for (int st = 0; st < 3; ++st) {
            const int K = kStageOut[st] / 2;
            for (int r = 0; r < kStageRepeats[st]; ++r, ++bi) {
                Blk& q = blk[bi];
                q.K = K; q.stride = r == 0 ? 2 : 1;
                const int kin = q.stride == 2 ? cin : K;                  // branch_main's first 1x1 reads the whole input when stride 2
                q.pw1 = b.conv_bn((long long)K * kin, K);
                q.dw = b.conv_bn((long long)K * 9, K);
                q.pw2 = b.conv_bn((long long)K * K, K);
                if (q.stride == 2) { q.pdw = b.conv_bn((long long)cin * 9, cin); q.ppw = b.conv_bn((long long)K * cin, K); }
            }
            cin = kStageOut[st];
        }
    }
    const CB c2 = b.conv_bn(72LL * 288, 72), c3 = b.conv_bn(72LL * 192, 72);
    struct Head { CB dw1, pw1, dw2, pw2; } head[4];          // definition order: cls_head_2, reg_head_2, reg_head_3, cls_head_3
    for (int h = 0; h < 4; ++h) {
        head[h].dw1 = b.conv_bn(72 * 25, 72); head[h].pw1 = b.conv_bn(72 * 72, 72);
        head[h].dw2 = b.conv_bn(72 * 25, 72); head[h].pw2 = b.conv_bn(72 * 72, 72);
    }
    const int w_reg = b.param(4LL * t.A * 72), b_reg = b.param(4 * t.A);
    const int w_obj = b.param((long long)t.A * 72), b_obj = b.param(t.A);
    const int w_cls = b.param((long long)t.C * 72), b_cls = b.param(t.C);

    // ---- the program, forward order (model/detector.py:21-31) --------------------------------------------------------
    t.x_ten = b.ten(3, t.H, t.W, -2);
    int x;
    {
        Op o = Builder::blank(K_STEM);
        o.a = t.x_ten; o.y = b.ten(24, t.H / 2, t.W / 2); o.pw = first.w;
        x = b.push(o);
    }
    x = b.bn(x, first, true);
    {
        const Ten X = t.tens[x];
        Op o = Builder::blank(K_POOL);
        o.a = x; o.y = b.ten(24, (X.H - 1) / 2 + 1, (X.W - 1) / 2 + 1);
        o.aux = b.alloc((long long)t.N * 24 * t.tens[o.y].H * t.tens[o.y].W);
        x = b.push(o);
    }
    int feat[3];
    {
        int bi = 0;
        for (int st = 0; st < 3; ++st) {
            for (int r = 0; r < kStageRepeats[st]; ++r, ++bi) {
                const Blk& q = blk[bi];
                const int K = q.K;
                if (q.stride == 2) {
                    const int proj = b.pw_bn(b.dw_bn(x, q.pdw, 3, 2, false), q.ppw, K, true);
                    int m = b.pw_bn(x, q.pw1, K, true);
                    m = b.dw_bn(m, q.dw, 3, 2, false);
                    m = b.pw_bn(m, q.pw2, K, true);
                    Op o = Builder::blank(K_CAT2);
                    o.a = proj; o.b = m; o.y = b.ten(2 * K, t.tens[m].H, t.tens[m].W);
                    x = b.push(o);
                } else {
                    t.tens[x].partial = true;
                    Op od = Builder::blank(K_ODD);
                    od.a = x; od.y = b.ten(K, t.tens[x].H, t.tens[x].W);
                    int m = b.push(od);
                    m = b.pw_bn(m, q.pw1, K, true);
                    m = b.dw_bn(m, q.dw, 3, 1, false);
                    m = b.pw_bn(m, q.pw2, K, true);
                    Op o = Builder::blank(K_CATE);
                    o.a = x; o.b = m; o.y = b.ten(2 * K, t.tens[m].H, t.tens[m].W);
                    x = b.push(o);
                }
            }
            feat[st] = x;
        }
    }
    const int C2 = feat[1], C3 = feat[2];
    const int S3 = b.pw_bn(C3, c3, 72, true);
    auto run_head = [&](const Head& h, int s) {
        int y = b.dw_bn(s, h.dw1, 5, 1, true);
        y = b.pw_bn(y, h.pw1, 72, false);
        y = b.dw_bn(y, h.dw2, 5, 1, true);
        return b.pw_bn(y, h.pw2, 72, false);
    };
    const int cls3 = run_head(head[3], S3), reg3 = run_head(head[2], S3);
    int up;
    {
        Op o = Builder::blank(K_UP);
        o.a = C3; o.y = b.ten(192, 2 * t.tens[C3].H, 2 * t.tens[C3].W);
        up = b.push(o);
    }
    int P2;
    {
        Op o = Builder::blank(K_CAT2);
        o.a = up; o.b = C2; o.y = b.ten(288, t.tens[C2].H, t.tens[C2].W);
        P2 = b.push(o);
    }
    const int S2 = b.pw_bn(P2, c2, 72, true);
    const int cls2 = run_head(head[0], S2), reg2 = run_head(head[1], S2);
    const int lv_cls[2] = {cls2, cls3}, lv_reg[2] = {reg2, reg3};
    for (int lv = 0; lv < 2; ++lv) {
        t.out_ten[3 * lv + 0] = b.pw(lv_reg[lv], w_reg, 4 * t.A, b_reg, 3 * lv + 0);
        t.out_ten[3 * lv + 1] = b.pw(lv_cls[lv], w_obj, t.A, b_obj, 3 * lv + 1);
        t.out_ten[3 * lv + 2] = b.pw(lv_cls[lv], w_cls, t.C, b_cls, 3 * lv + 2);
    }
    // ---- shared storage ------------------------------------------------------------------------------------------------
    long long biggest = 0, pbig = 0;
    for (const Ten& x_ : t.tens) if (x_.ext == -1) biggest = std::max(biggest, (long long)t.N * x_.C * x_.H * x_.W);
    for (long long n : t.pnumel) pbig = std::max(pbig, n);
    // the second use of a shared output convolution puts its bias gradient right behind the weight's (describe_backward)
    for (int w : {w_reg, w_obj, w_cls}) pbig = std::max(pbig, t.pnumel[w] + t.pnumel[w + 1]);
    t.scratch_off = b.alloc(biggest);
    t.pscratch_off = b.alloc(pbig);
    t.pscratch_floats = pbig;
    t.gflat_off = b.alloc(t.ptotal);
    t.wscratch_off = b.alloc(kWScratchFloats);
}

// The per-op backward plan and the flat layout of the current mode (host only)
void apply_mode(yfv2_trainer& t) {
    std::vector<char> rg(t.tens.size(), 0);
    t.bwd.assign(t.ops.size(), BwdOp{});
    auto tr = [&](int p) { return p >= 0 && t.trainable[p] != 0; };
    for (size_t i = 0; i < t.ops.size(); ++i) {
        const Op& o = t.ops[i];
        BwdOp& b = t.bwd[i];
        const bool ra = rg[o.a] != 0, rb = o.b >= 0 && rg[o.b] != 0;
        b.dw = tr(o.pw); b.dbias = tr(o.pbias); b.dgamma = tr(o.pg); b.dbeta = tr(o.pb);
        b.run = ra || rb || b.dw || b.dbias || b.dgamma || b.dbeta;
        b.da = b.run && ra; b.db = b.run && rb;
        b.bn_eval = o.kind == K_BN && t.bn_eval[o.bn] != 0;
        rg[o.y] = b.run ? 1 : 0;
    }
    t.coff.assign(t.poff.size(), -1);
    t.ctotal = 0;
    for (size_t i = 0; i < t.poff.size(); ++i)
        if (t.trainable[i]) { t.coff[i] = t.ctotal; t.ctotal += t.pnumel[i]; }
    unsigned long long h = 1469598103934665603ull;                  // FNV-1a over both masks
    for (unsigned char v : t.trainable) h = (h ^ v) * 1099511628211ull;
    for (unsigned char v : t.bn_eval) h = (h ^ (unsigned)(v + 2)) * 1099511628211ull;
    t.mode_hash = h;
}

#define TRYT(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)

}  // namespace
}  // namespace yfv2

using namespace yfv2;

extern "C" int yfv2_trainer_create(yfv2_trainer** out, int device, int N, int H, int W, int A, int C) {
    if (!out || N <= 0 || H <= 0 || W <= 0 || H % 32 || W % 32 || A <= 0 || C <= 0) {
        set_error("trainer_create: bad arguments (N=%d H=%d W=%d A=%d C=%d; H, W multiples of 32)", N, H, W, A, C);
        return YFV2_EINVAL;
    }
    if ((long long)N * (H / 32) * (W / 32) == 1) {      // every stride-32 BatchNorm would normalise one value (F.batch_norm refuses)
        set_error("trainer_create: expected more than 1 value per channel when training (N=%d, %dx%d: one value at stride 32)", N, H, W);
        return YFV2_EINVAL;
    }
    yfv2_trainer* t = new (std::nothrow) yfv2_trainer();
    if (!t) { set_error("trainer_create: out of host memory"); return YFV2_ENOMEM; }
    t->device = device; t->N = N; t->H = H; t->W = W; t->A = A; t->C = C;
    build(*t);
    if ((int)t->poff.size() != YFV2_NUM_PARAMS) {
        set_error("trainer_create: internal layout has %d parameters, expected %d", (int)t->poff.size(), YFV2_NUM_PARAMS);
        delete t;
        return YFV2_EINVAL;
    }
    t->trainable.assign(YFV2_NUM_PARAMS, 1);
    t->bn_eval.assign(YFV2_NUM_BN, 0);
    t->fwd_trainable = t->trainable; t->fwd_bn_eval = t->bn_eval;
    apply_mode(*t);
    *out = t;
    return YFV2_OK;
}
extern "C" void yfv2_trainer_destroy(yfv2_trainer* t) {
    if (!t) return;
    if (t->g_fwd.exec) cudaGraphExecDestroy(t->g_fwd.exec);
    for (auto& g : t->g_bwd) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (t->cap_stream) cudaStreamDestroy(t->cap_stream);
    delete t;
}
extern "C" int yfv2_trainer_workspace_bytes(const yfv2_trainer* t, size_t* bytes) {
    if (!t || !bytes) { set_error("trainer_workspace_bytes: null argument"); return YFV2_EINVAL; }
    *bytes = (size_t)t->ws_floats * sizeof(float);
    return YFV2_OK;
}
extern "C" int yfv2_trainer_grad_floats(const yfv2_trainer* t, long long* n) {
    if (!t || !n) { set_error("trainer_grad_floats: null argument"); return YFV2_EINVAL; }
    *n = t->ctotal;
    return YFV2_OK;
}
extern "C" int yfv2_trainer_param_offset(const yfv2_trainer* t, int index, long long* offset, long long* numel) {
    if (!t || index < 0 || index >= (int)t->poff.size() || !offset || !numel) { set_error("trainer_param_offset: bad argument"); return YFV2_EINVAL; }
    *offset = t->coff[index]; *numel = t->pnumel[index];
    return YFV2_OK;
}
extern "C" int yfv2_trainer_set_mode(yfv2_trainer* t, const unsigned char* trainable, const unsigned char* bn_eval) {
    if (!t) { set_error("trainer_set_mode: null trainer"); return YFV2_EINVAL; }
    for (int i = 0; trainable && i < YFV2_NUM_PARAMS; ++i)
        if (trainable[i] > 1) { set_error("trainer_set_mode: trainable[%d] = %d is not 0 or 1", i, trainable[i]); return YFV2_EINVAL; }
    for (int i = 0; bn_eval && i < YFV2_NUM_BN; ++i)
        if (bn_eval[i] > 1) { set_error("trainer_set_mode: bn_eval[%d] = %d is not 0 or 1", i, bn_eval[i]); return YFV2_EINVAL; }
    for (int i = 0; i < YFV2_NUM_PARAMS; ++i) t->trainable[i] = trainable ? trainable[i] : 1;
    for (int i = 0; i < YFV2_NUM_BN; ++i) t->bn_eval[i] = bn_eval ? bn_eval[i] : 0;
    apply_mode(*t);
    return YFV2_OK;
}
extern "C" int yfv2_trainer_debug_backward(const yfv2_trainer* t, yfv2_trainer_bwd_op* ops_host, int cap, int* n) {
    if (!t || !n || cap < 0 || (cap > 0 && !ops_host)) { set_error("trainer_debug_backward: bad argument"); return YFV2_EINVAL; }
    int k = 0;
    for (int oi = (int)t->ops.size() - 1; oi >= 0; --oi) {      // backward order
        const BwdOp& b = t->bwd[oi];
        if (!b.run) continue;
        if (k < cap) {
            yfv2_trainer_bwd_op& d = ops_host[k];
            d.op = oi; d.da = b.da; d.db = b.db; d.dw = b.dw; d.dbias = b.dbias; d.dgamma = b.dgamma; d.dbeta = b.dbeta; d.bn_eval = b.bn_eval;
        }
        ++k;
    }
    *n = k;
    return YFV2_OK;
}

extern "C" int yfv2_trainer_debug_ops(const yfv2_trainer* t, yfv2_trainer_op* ops_host, int cap, int* n) {
    if (!t || !n || cap < 0 || (cap > 0 && !ops_host)) { set_error("trainer_debug_ops: bad argument"); return YFV2_EINVAL; }
    *n = (int)t->ops.size();
    for (int i = 0; i < cap && i < *n; ++i) {
        const Op& o = t->ops[i];
        yfv2_trainer_op& d = ops_host[i];
        d.kind = o.kind; d.a = o.a; d.b = o.b; d.y = o.y;
        d.pw = o.pw; d.pg = o.pg; d.pb = o.pb; d.pbias = o.pbias; d.bn = o.bn;
        d.relu = o.relu; d.ks = o.ks; d.stride = o.stride; d.M = o.M;
        d.aux = o.kind == K_BN || o.kind == K_POOL ? o.aux : -1;
    }
    return YFV2_OK;
}
extern "C" int yfv2_trainer_debug_tensors(const yfv2_trainer* t, yfv2_trainer_tensor* tens_host, int cap, int* n) {
    if (!t || !n || cap < 0 || (cap > 0 && !tens_host)) { set_error("trainer_debug_tensors: bad argument"); return YFV2_EINVAL; }
    *n = (int)t->tens.size();
    for (int i = 0; i < cap && i < *n; ++i) {
        const Ten& x = t->tens[i];
        yfv2_trainer_tensor& d = tens_host[i];
        d.off = x.off; d.goff = x.goff; d.C = x.C; d.H = x.H; d.W = x.W; d.ext = x.ext;
    }
    return YFV2_OK;
}
extern "C" int yfv2_trainer_debug_layout(const yfv2_trainer* t, long long* layout_host) {
    if (!t || !layout_host) { set_error("trainer_debug_layout: bad argument"); return YFV2_EINVAL; }
    const long long v[8] = {t->ws_floats, t->scratch_off, t->pscratch_off, t->pscratch_floats, t->gflat_off, t->ptotal,
                            t->wscratch_off, kWScratchFloats};
    for (int i = 0; i < 8; ++i) layout_host[i] = v[i];
    return YFV2_OK;
}

namespace {
struct Ptrs {
    float* ws; const float* x; float* const* preds; const float* const* dpreds;
    const float* act(const yfv2_trainer& t, int id) const {
        const Ten& q = t.tens[id];
        return q.ext == -2 ? x : (q.ext >= 0 ? preds[q.ext] : ws + q.off);
    }
    float* actw(const yfv2_trainer& t, int id) const { const Ten& q = t.tens[id]; return q.ext >= 0 ? preds[q.ext] : ws + q.off; }
    const float* grad(const yfv2_trainer& t, int id) const { const Ten& q = t.tens[id]; return q.ext >= 0 ? dpreds[q.ext] : ws + q.goff; }
    float* gradw(const yfv2_trainer& t, int id) const { return ws + t.tens[id].goff; }
};
}  // namespace

// The records of the train-mode forward, in launch order: what yfv2_train_forward captures and yfv2_trainer_debug_launches returns
static int describe_forward(const yfv2_trainer* t, const float* x, const float* const* params, float* const* bn_running,
                            float* const preds[6], void* workspace, int sms, TrainLaunches& L) {
    Ptrs P{(float*)workspace, x, preds, nullptr};
    const int N = t->N;
    for (int oi = 0; oi < (int)t->ops.size(); ++oi) {
        const Op& o = t->ops[oi];
        const size_t first = L.size();
        const Ten& A = t->tens[o.a];
        const Ten& Y = t->tens[o.y];
        const float* a = P.act(*t, o.a);
        float* y = P.actw(*t, o.y);
        switch (o.kind) {
        case K_STEM: TRYT(describe_stem_fwd(a, params[o.pw], y, N, Y.C, A.H, A.W, L)); break;
        case K_BN: {
            double* scr = reinterpret_cast<double*>(P.ws + o.aux);
            float* mean = P.ws + o.aux + 4LL * A.C;
            if (t->bn_eval[o.bn])
                TRYT(describe_bn_eval_fwd(a, params[o.pg], params[o.pb], bn_running[2 * o.bn], bn_running[2 * o.bn + 1], y, mean, mean + A.C,
                                          N, A.C, A.H * A.W, o.relu, L));
            else
                TRYT(describe_bn_train_fwd(a, params[o.pg], params[o.pb], bn_running[2 * o.bn], bn_running[2 * o.bn + 1], y, mean, mean + A.C,
                                           scr, N, A.C, A.H * A.W, o.relu, L));
        } break;
        case K_POOL: TRYT(describe_maxpool_fwd(a, y, reinterpret_cast<int*>(P.ws + o.aux), N * A.C, A.H, A.W, L)); break;
        case K_PW: TRYT(describe_conv1x1_fwd(a, params[o.pw], o.pbias >= 0 ? params[o.pbias] : nullptr, y, N, A.C, o.M, A.H * A.W, L)); break;
        case K_DW: TRYT(describe_dwconv_fwd(a, params[o.pw], y, N, A.C, A.H, A.W, o.ks, o.stride, L)); break;
        case K_UP: TRYT(describe_upsample2_fwd(a, y, N * A.C, A.H, A.W, L)); break;
        case K_ODD: describe_chan_copy(a, A.C, 1, 2, y, Y.C, 0, 1, Y.C, N, A.H * A.W, 0, sms, L); break;
        case K_CATE: {
            const Ten& B = t->tens[o.b];
            describe_chan_copy(a, A.C, 0, 2, y, Y.C, 0, 1, A.C / 2, N, A.H * A.W, 0, sms, L);
            describe_chan_copy(P.act(*t, o.b), B.C, 0, 1, y, Y.C, A.C / 2, 1, B.C, N, A.H * A.W, 0, sms, L);
        } break;
        case K_CAT2: {
            const Ten& B = t->tens[o.b];
            describe_chan_copy(a, A.C, 0, 1, y, Y.C, 0, 1, A.C, N, Y.H * Y.W, 0, sms, L);
            describe_chan_copy(P.act(*t, o.b), B.C, 0, 1, y, Y.C, A.C, 1, B.C, N, Y.H * Y.W, 0, sms, L);
        } break;
        default: set_error("train_forward: unknown op"); return YFV2_EINVAL;
        }
        for (size_t j = first; j < L.size(); ++j) L[j].op = oi;
    }
    return YFV2_OK;
}

// The records of the backward under the current mode, in launch order: what yfv2_train_backward captures
static int describe_backward(const yfv2_trainer* t, const float* x, const float* const* params, float* const preds[6],
                             const float* const dpreds[6], float* grads_flat, int accumulate, void* workspace, int sms, TrainLaunches& L) {
    Ptrs P{(float*)workspace, x, preds, dpreds};
    const int N = t->N;
    float* G = P.ws + t->gflat_off;                 // parameter gradients of this step, assigned
    float* scratch = P.ws + t->scratch_off;
    float* pscratch = P.ws + t->pscratch_off;
    std::vector<char> pwritten(t->poff.size(), 0);
    // parameter gradient target: the flat slot on first use, the parameter scratch (then added) for a shared layer's second use
    auto ptarget = [&](int idx, bool* via) { *via = pwritten[idx] != 0; return *via ? pscratch : G + t->poff[idx]; };
    auto pcommit = [&](int idx, bool via) {
        pwritten[idx] = 1;
        if (via) describe_axpy(pscratch, G + t->poff[idx], t->pnumel[idx], 1, sms, L);
    };
    for (int oi = (int)t->ops.size() - 1; oi >= 0; --oi) {
        const Op& o = t->ops[oi];
        const BwdOp& bo = t->bwd[oi];
        if (!bo.run) continue;                      // no trainable parameter upstream of its output
        const size_t first = L.size();
        const Ten& A = t->tens[o.a];
        const Ten& Y = t->tens[o.y];
        const float* a = P.act(*t, o.a);
        const float* dy = P.grad(*t, o.y);
        // gradient of input a: assigned by the consumer that runs first in the backward (the last one in the forward), accumulated
        // through the scratch tensor by the others; inputs that need no gradient (the image, frozen bottoms of the network) get none
        const bool need_da = bo.da;
        const bool acc_a = need_da && !A.partial && A.last_use != oi;
        float* da = !need_da ? nullptr : (acc_a ? scratch : P.gradw(*t, o.a));
        const long long an = (long long)N * A.C * A.H * A.W;
        switch (o.kind) {
        case K_STEM: {                              // runs only for a trainable stem weight (the image needs no gradient)
            bool via; float* dw = ptarget(o.pw, &via);
            TRYT(describe_stem_wgrad(a, dy, dw, N, Y.C, A.H, A.W, L));
            pcommit(o.pw, via);
        } break;
        case K_BN: {
            double* scr = reinterpret_cast<double*>(P.ws + o.aux);
            const float* mean = P.ws + o.aux + 4LL * A.C;
            // gamma and beta of one layer are never shared, so both go straight to their slots
            float* dg = bo.dgamma ? G + t->poff[o.pg] : nullptr;
            float* db = bo.dbeta ? G + t->poff[o.pb] : nullptr;
            if (bo.bn_eval) {
                TRYT(describe_bn_eval_bwd(a, P.act(*t, o.y), dy, params[o.pg], mean, mean + A.C, da, dg, db, scr, N, A.C, A.H * A.W, o.relu, L));
            } else {
                // the batch-statistics backward needs the sums for its gamma / beta anyway; without rg(a) its dx goes to a's own
                // gradient slot, which nothing reads (a's producer does not run)
                TRYT(describe_bn_train_bwd(a, P.act(*t, o.y), dy, params[o.pg], mean, mean + A.C, da ? da : P.gradw(*t, o.a), dg, db, scr,
                                           N, A.C, A.H * A.W, o.relu, L));
            }
            if (dg) pwritten[o.pg] = 1;
            if (db) pwritten[o.pb] = 1;
        } break;
        case K_POOL: TRYT(describe_maxpool_bwd(dy, reinterpret_cast<const int*>(P.ws + o.aux), da, N * A.C, A.H, A.W, L)); break;
        case K_PW: {
            bool vw = false, vb = false;
            float* dw = bo.dw ? ptarget(o.pw, &vw) : nullptr;
            float* db = nullptr;
            if (bo.dbias) { vb = pwritten[o.pbias] != 0; db = vb ? pscratch + t->pnumel[o.pw] : G + t->poff[o.pbias]; }  // bias rides behind the weight in the scratch
            TRYT(describe_conv1x1_bwd(a, params[o.pw], dy, da, dw, db, N, A.C, o.M, A.H * A.W, P.ws + t->wscratch_off, (size_t)kWScratchFloats,
                                      sms, L));
            if (vb) describe_axpy(pscratch + t->pnumel[o.pw], G + t->poff[o.pbias], t->pnumel[o.pbias], 1, sms, L);
            if (dw) pcommit(o.pw, vw);
            if (db) pwritten[o.pbias] = 1;
        } break;
        case K_DW: {
            bool vw = false; float* dw = bo.dw ? ptarget(o.pw, &vw) : nullptr;
            TRYT(describe_dwconv_bwd(a, params[o.pw], dy, da, dw, N, A.C, A.H, A.W, o.ks, o.stride, L));
            if (dw) pcommit(o.pw, vw);
        } break;
        case K_UP: TRYT(describe_upsample2_bwd(dy, da, N * A.C, A.H, A.W, L)); break;
        case K_ODD: describe_chan_copy(dy, Y.C, 0, 1, P.gradw(*t, o.a), A.C, 1, 2, Y.C, N, A.H * A.W, 0, sms, L); break;          // odd half of d(a)
        case K_CATE: {
            const Ten& B = t->tens[o.b];
            if (bo.da) describe_chan_copy(dy, Y.C, 0, 1, P.gradw(*t, o.a), A.C, 0, 2, A.C / 2, N, A.H * A.W, 0, sms, L);              // even half of d(a)
            if (bo.db) describe_chan_copy(dy, Y.C, A.C / 2, 1, P.gradw(*t, o.b), B.C, 0, 1, B.C, N, A.H * A.W, 0, sms, L);
        } break;
        case K_CAT2: {
            const Ten& B = t->tens[o.b];
            const bool acc_b = B.last_use != oi;
            if (bo.da) describe_chan_copy(dy, Y.C, 0, 1, P.gradw(*t, o.a), A.C, 0, 1, A.C, N, Y.H * Y.W, acc_a ? 1 : 0, sms, L);
            if (bo.db) describe_chan_copy(dy, Y.C, A.C, 1, P.gradw(*t, o.b), B.C, 0, 1, B.C, N, Y.H * Y.W, acc_b ? 1 : 0, sms, L);
        } break;
        default: set_error("train_backward: unknown op"); return YFV2_EINVAL;
        }
        if (acc_a && o.kind != K_CAT2 && o.kind != K_ODD && o.kind != K_CATE) describe_axpy(scratch, P.gradw(*t, o.a), an, 1, sms, L);
        for (size_t j = first; j < L.size(); ++j) { L[j].op = oi; L[j].bwd = true; }
    }
    for (size_t i = 0; i < pwritten.size(); ++i)
        if ((pwritten[i] != 0) != (t->trainable[i] != 0)) {
            set_error("train_backward: parameter %d %s a gradient (internal)", (int)i, pwritten[i] ? "frozen but received" : "received no");
            return YFV2_EINVAL;
        }
    // the trainable parameters' slots, packed in parameter order: one copy per run of consecutive trainable parameters (all
    // trainable: one copy of the whole slot)
    for (size_t i = 0; i < t->poff.size();) {
        if (!t->trainable[i]) { ++i; continue; }
        size_t j = i;
        long long n = 0;
        while (j < t->poff.size() && t->trainable[j]) n += t->pnumel[j++];
        describe_axpy(G + t->poff[i], grads_flat + t->coff[i], n, accumulate ? 1 : 0, sms, L);
        L.back().bwd = true;
        i = j;
    }
    return YFV2_OK;
}

namespace {
// yfv2_train_backward's refusal of a mode with no trainable parameter (torch: nothing requires grad), shared with its test hook
int check_trainable(const yfv2_trainer* t) {
    if (t->ctotal == 0) { set_error("train_backward: no parameter is trainable (element 0 of tensors does not require grad)"); return YFV2_EINVAL; }
    return YFV2_OK;
}
unsigned long long mix(unsigned long long h, unsigned long long v) {
    h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    return h;
}
unsigned long long mix(unsigned long long h, const void* p) { return mix(h, (unsigned long long)reinterpret_cast<uintptr_t>(p)); }
// the SM count and persistent-CTA cap the launches were described for (yfv2_debug_set_dispatch changes both): a graph captured
// under another dispatch is not replayed
unsigned long long dispatch_key(unsigned long long h) { return mix(mix(h, (unsigned long long)sm_count()), (unsigned long long)persistent_cta_cap()); }
// Replays `slot` if it was captured for `key`; otherwise captures body() on the trainer's private stream, instantiates and replays.
template <class Body>
int replay_or_capture(yfv2_trainer* t, yfv2_trainer::GraphSlot& slot, unsigned long long key, cudaStream_t s, Body&& body) {
    if (!slot.exec || slot.key != key) {
        if (slot.exec) { cudaGraphExecDestroy(slot.exec); slot.exec = nullptr; }
        if (!t->cap_stream) YFV2_CUDA(cudaStreamCreateWithFlags(&t->cap_stream, cudaStreamNonBlocking));
        YFV2_CUDA(cudaStreamBeginCapture(t->cap_stream, cudaStreamCaptureModeThreadLocal));
        const int rc = body(t->cap_stream);
        cudaGraph_t graph = nullptr;
        const cudaError_t e = cudaStreamEndCapture(t->cap_stream, &graph);
        if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (e != cudaSuccess || !graph) { set_error("trainer: stream capture failed: %s", cudaGetErrorString(e)); return YFV2_ECUDA; }
        const cudaError_t ei = cudaGraphInstantiate(&slot.exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ei != cudaSuccess) { slot.exec = nullptr; set_error("trainer: graph instantiation failed: %s", cudaGetErrorString(ei)); return YFV2_ECUDA; }
        slot.key = key;
    }
    YFV2_CUDA(cudaGraphLaunch(slot.exec, s));
    return YFV2_OK;
}
}  // namespace

extern "C" int yfv2_train_forward(yfv2_trainer* t, const float* x, const float* const* params, float* const* bn_running,
                                  float* const preds[6], void* workspace, void* stream) {
    if (!t || !x || !params || !bn_running || !preds || !workspace) { set_error("train_forward: null argument"); return YFV2_EINVAL; }
    for (int i = 0; i < 6; ++i) if (!preds[i]) { set_error("train_forward: null output %d", i); return YFV2_EINVAL; }
    for (int i = 0; i < YFV2_NUM_PARAMS; ++i) if (!params[i]) { set_error("train_forward: null parameter %d", i); return YFV2_EINVAL; }
    for (int i = 0; i < 2 * YFV2_NUM_BN; ++i) if (!bn_running[i]) { set_error("train_forward: null BN buffer %d", i); return YFV2_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long key = mix(mix(mix(dispatch_key(0x1234ull), t->mode_hash), x), workspace);
    for (int i = 0; i < YFV2_NUM_PARAMS; ++i) key = mix(key, params[i]);
    for (int i = 0; i < 2 * YFV2_NUM_BN; ++i) key = mix(key, bn_running[i]);
    for (int i = 0; i < 6; ++i) key = mix(key, preds[i]);
    const int rc = replay_or_capture(t, t->g_fwd, key, s, [&](cudaStream_t cs) {
        TrainLaunches L;
        TRYT(describe_forward(t, x, params, bn_running, preds, workspace, sm_count(), L));
        return launch_all(L, cs);
    });
    if (rc == YFV2_OK) { t->fwd_trainable = t->trainable; t->fwd_bn_eval = t->bn_eval; }
    return rc;
}

extern "C" int yfv2_train_backward(yfv2_trainer* t, const float* x, const float* const* params, float* const preds[6],
                                   const float* const dpreds[6], float* grads_flat, int accumulate, void* workspace, void* stream) {
    if (!t || !x || !params || !preds || !dpreds || !grads_flat || !workspace) { set_error("train_backward: null argument"); return YFV2_EINVAL; }
    for (int i = 0; i < 6; ++i) if (!preds[i] || !dpreds[i]) { set_error("train_backward: null head tensor %d", i); return YFV2_EINVAL; }
    for (int i = 0; i < YFV2_NUM_PARAMS; ++i) if (!params[i]) { set_error("train_backward: null parameter %d", i); return YFV2_EINVAL; }
    TRYT(check_trainable(t));
    if (t->trainable != t->fwd_trainable || t->bn_eval != t->fwd_bn_eval) {
        set_error("train_backward: the mode changed after the forward (yfv2_trainer_set_mode applies from the next yfv2_train_forward)");
        return YFV2_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long key = mix(mix(mix(mix(dispatch_key(0x4321ull), t->mode_hash), x), workspace), grads_flat);
    for (int i = 0; i < YFV2_NUM_PARAMS; ++i) key = mix(key, params[i]);
    for (int i = 0; i < 6; ++i) key = mix(mix(key, preds[i]), dpreds[i]);
    return replay_or_capture(t, t->g_bwd[accumulate ? 1 : 0], key, s, [&](cudaStream_t cs) {
        TrainLaunches L;
        TRYT(describe_backward(t, x, params, preds, dpreds, grads_flat, accumulate, workspace, sm_count(), L));
        return launch_all(L, cs);
    });
}

// ---- test hook: the records of one training step ------------------------------------------------------------------------------
extern "C" int yfv2_trainer_debug_launches(const yfv2_trainer* t, const void* workspace, int sms, yfv2_train_launch* out, int cap, int* n) {
    if (!t || !n || sms < 0 || cap < 0 || (cap > 0 && !out)) { set_error("trainer_debug_launches: bad argument"); return YFV2_EINVAL; }
    TRYT(check_trainable(t));
    // the caller's tensors: any 16-byte-aligned addresses (never dereferenced); NULL workspace: a 16-byte-aligned one
    float* const fake = reinterpret_cast<float*>((uintptr_t)256);
    void* ws = workspace ? const_cast<void*>(workspace) : fake;
    const std::vector<const float*> params(YFV2_NUM_PARAMS, fake);
    const std::vector<float*> bn_running(2 * YFV2_NUM_BN, fake);
    float* const preds[6] = {fake, fake, fake, fake, fake, fake};
    const float* const dpreds[6] = {fake, fake, fake, fake, fake, fake};
    if (!sms) sms = sm_count();
    TrainLaunches L;
    TRYT(describe_forward(t, fake, params.data(), bn_running.data(), preds, ws, sms, L));
    TRYT(describe_backward(t, fake, params.data(), preds, dpreds, fake, 0, ws, sms, L));
    return debug_records(L, out, cap, n);
}
