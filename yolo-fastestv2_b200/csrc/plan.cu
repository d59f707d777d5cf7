// Host side of libyfv2.so: plan construction (shape bookkeeping, channel-plane tables, packed-weight and
// workspace layouts), weight packing, and the C ABI declared in include/yfv2.h.
//
// Mirrors the wiring of the reference model (model/detector.py:8-47, model/fpn.py:31-64,
// model/backbone/shufflenetv2.py:65-109) without any of its module objects: the plan is a flat list of
// fused-kernel launches over plane pools.
#include <stdarg.h>
#include <string.h>

#include <atomic>
#include <new>
#include <vector>

#include <stdlib.h>

#include "common.cuh"

namespace yfv2 {

bool blk_s1_chainable(int K, int H, int W);      // k_net.cu

enum class StageKind { stem, block_s1, block_s2, fpn, heads };
constexpr int kMaxStages = 64;

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static thread_local bool g_pdl_next = false;
static thread_local bool g_pdl_call = true;      // false inside yfv2_detect_u8_host: with copies and a second stream in flight the
                                                 // early-resident dependents cost more than the hidden prologues save (measured)
bool pdl_take() { const bool r = g_pdl_next && g_pdl_call; g_pdl_next = true; return r; }
void pdl_reset() { g_pdl_next = false; }
bool pdl_allowed() { return g_pdl_call; }

// yfv2_debug_set_dispatch: the SM count the dispatch assumes (0: the device's) and the CTAs of a persistent launch (0: sized by
// occupancy).  Process-wide, not per thread: the autograd engine runs the trainer's backward on a thread of its own.
static std::atomic<int> g_sim_sms{0}, g_sim_ctas{0};
int persistent_cta_cap() { return g_sim_ctas.load(); }

int sm_count() {
    if (const int s = g_sim_sms.load()) return s;
    static thread_local int n = 0;
    if (!n) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

// pack sizes of the per-layer weight layouts (common.cuh)
size_t shuffle_pack_floats(int K, int stride) {
    const size_t pwn = pw_pack_floats(K, K), dwn = dw3_pack_floats(K);
    return stride == 1 ? 2 * pwn + dwn : 3 * pwn + 2 * dwn;
}
size_t head_pack_floats() { return 2 * ((size_t)dw5_pack_floats(72) + pw_pack_floats(72, 72)); }

namespace {

constexpr int kStageRepeats[3] = {4, 8, 4};          // shufflenetv2.py:69
constexpr int kStageWidth[3] = {24, 48, 96};         // branch width = out_channels / 2 (detector.py:11)
constexpr int kNumBlocks = 16;
constexpr int kFpnDepth = 72;                        // detector.py:10
constexpr int kHeadTile = 96;                        // output columns per tile of the heads' second half (k_net.cu)

// ---- pack kernels ---------------------------------------------------------------------------------------
// w: [Nout][K] row-major conv weight.  Writes Wt[k][n_off+n], scale/shift[n_off+n] with row length Np.
// BN folded as PyTorch's eval path does: alpha = invstd*gamma, beta' = beta - mean*alpha.
__global__ void pack_pw_kernel(const float* __restrict__ w, int Nout, int K, const float* gamma, const float* beta,
                               const float* mean, const float* var, const float* bias, float* Wt, int Np, int n_off,
                               float* scale, float* shift) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < Nout * K) {
        const int n = i / K, k = i - n * K;
        Wt[(size_t)k * Np + n_off + n] = w[i];
    }
    if (i < Nout) {
        float sc = 1.0f, sh = 0.0f;
        if (gamma) {
            const float invstd = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var[i], kBnEps)));
            sc = __fmul_rn(invstd, gamma[i]);
            sh = __fsub_rn(beta[i], __fmul_rn(mean[i], sc));
        } else if (bias) {
            sh = bias[i];
        }
        scale[n_off + i] = sc;
        shift[n_off + i] = sh;
    }
}

// w: [C][KK] depthwise weight -> per channel [KK taps][scale][shift][pad] with row length R
__global__ void pack_dw_kernel(const float* __restrict__ w, int Cn, int KK, int R, const float* gamma, const float* beta,
                               const float* mean, const float* var, float* dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < Cn * KK) {
        const int c = i / KK, t = i - c * KK;
        dst[(size_t)c * R + t] = w[i];
    }
    if (i < Cn) {
        const float invstd = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var[i], kBnEps)));
        const float sc = __fmul_rn(invstd, gamma[i]);
        dst[(size_t)i * R + KK] = sc;
        dst[(size_t)i * R + KK + 1] = __fsub_rn(beta[i], __fmul_rn(mean[i], sc));
    }
}

// Heads, second half (reference fpn.py DWConvblock tail + detector.py:17-19,35-41): pw(72->72), its BN and the shared output
// conv are consecutive affine maps with no activation between them, so they are ONE matrix at inference time:
//   F = Wout . diag(sc) . Wpw,   f = Wout . sh + bias          (products accumulated in fp64, rounded once to fp32)
// rows [n_off, n_off+Mo) of the folded [NPt x K] matrix Fw (NPt = 96 or 192) and of the bias Fb.
__global__ void fold_head_kernel(const float* __restrict__ wout, const float* __restrict__ bout, int Mo, const float* __restrict__ wpw,
                                 const float* gamma, const float* beta, const float* mean, const float* var, int K, int n_off,
                                 float* __restrict__ Fw, float* __restrict__ Fb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < Mo * K) {
        const int m = i / K, k = i - m * K;
        double acc = 0.0;
        for (int j = 0; j < K; ++j) {
            const float invstd = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var[j], kBnEps)));
            const float sc = __fmul_rn(invstd, gamma[j]);
            acc += (double)wout[m * K + j] * (double)sc * (double)wpw[j * K + k];
        }
        Fw[(size_t)(n_off + m) * K + k] = (float)acc;
    }
    if (i < Mo) {
        double acc = (double)bout[i];
        for (int j = 0; j < K; ++j) {
            const float invstd = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var[j], kBnEps)));
            const float sc = __fmul_rn(invstd, gamma[j]);
            const float sh = __fsub_rn(beta[j], __fmul_rn(mean[j], sc));
            acc += (double)wout[i * K + j] * (double)sh;
        }
        Fb[n_off + i] = (float)acc;
    }
}
// dense NCHW copy of a logical tensor (tests / debugging only)
__global__ void gather_kernel(Planes P, ChanTab tab, int Cn, float* __restrict__ out, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int HW = P.H * P.W;
    const int p = (int)(i % HW);
    const int c = (int)((i / HW) % Cn);
    const int n = (int)(i / ((long long)HW * Cn));
    const int y = p / P.W, x = p - y * P.W;
    out[i] = plane_ptr(P, n, tab.c[c])[P.org + y * P.Ws + x];
}

struct Cursor {           // walks parameters / BN layers in state_dict order
    const float* const* params;
    const float* const* bn;
    int p = 0, b = 0;
};

}  // namespace
}  // namespace yfv2

using namespace yfv2;

struct yfv2_plan {
    int device, N, H, W, A, C, training;
    int h[4], w[4];                    // strides 4, 8, 16, 32
    size_t plane[4];                   // pool plane stride (floats) per resolution, zero frame of 1 included
    size_t plane2[4];                  // same with a frame of 2 (inputs of the 5x5 depthwise heads)
    int ws1[4], ws2[4];                // row strides for the two frame widths
    const void* ws_zeroed;             // workspace whose frames have been zeroed
    int pool_planes[4];                // 24, 72, 144, 288
    size_t off_pool[4];
    size_t off_s2, off_s3, off_t[4];   // t: cls2, reg2, cls3, reg3 mid-block scratch
    size_t ws_floats;
    size_t pk_stem, pk_block[kNumBlocks], pk_fpn3, pk_fpn2, pk_head[4], pk_out_reg, pk_out_oc, pk_floats;
    int blk_K[kNumBlocks], blk_stride[kNumBlocks], blk_res[kNumBlocks];   // res = index of OUTPUT resolution
    ChanTab tin[kNumBlocks], tout[kNumBlocks];
    ChanTab c2, c3;
    ChanTab logical[kNumBlocks];       // logical channel order of each block's output (debug gather)
    int launches;
    size_t pk_foldw[4];                // heads' second pointwise + BN + output conv folded into one matrix [NPt][72] | bias[NPt]
    int fold_rows[4];                  // NPt: 96 or 192 output columns (one or two tiles of the head kernel)
    int n_stages;
    // group: the first stage of the launch this stage shares
    struct Stage { StageKind kind; int a, b; char name[24]; int group; } stages[kMaxStages];
};

namespace {

Planes pool_planes(const yfv2_plan* p, float* ws, int r) {
    Planes P;
    P.base = ws + p->off_pool[r];
    P.sC = (long long)p->plane[r];
    P.sN = (long long)p->plane[r] * p->pool_planes[r];
    P.H = p->h[r]; P.W = p->w[r];
    P.Ws = p->ws1[r]; P.pad = 1; P.org = P.Ws + 1;
    return P;
}
Planes flat_planes(const yfv2_plan* p, float* ws, size_t off, int r) {
    Planes P;
    P.base = ws + off;
    P.sC = (long long)p->plane2[r];
    P.sN = (long long)p->plane2[r] * kFpnDepth;
    P.H = p->h[r]; P.W = p->w[r];
    P.Ws = p->ws2[r]; P.pad = 2; P.org = 2 * P.Ws + 2;
    return P;
}

void build_tables(yfv2_plan* p) {
    std::vector<int> L(24);
    for (int i = 0; i < 24; ++i) L[i] = i;
    int bi = 0;
    for (int st = 0; st < 3; ++st) {
        const int K = kStageWidth[st];
        std::vector<int> freep;
        for (int rep = 0; rep < kStageRepeats[st]; ++rep, ++bi) {
            p->blk_K[bi] = K;
            p->blk_res[bi] = st + 1;
            if (rep == 0) {
                // stride 2: read every logical channel of the previous stage, write 2K fresh planes 0..2K-1
                p->blk_stride[bi] = 2;
                for (int i = 0; i < K; ++i) p->tin[bi].c[i] = (unsigned short)L[i];
                L.resize(2 * K);
                for (int i = 0; i < 2 * K; ++i) { L[i] = i; p->tout[bi].c[i] = (unsigned short)i; }
                freep.clear();
                for (int i = 2 * K; i < 3 * K; ++i) freep.push_back(i);
            } else {
                // stride 1: channel_shuffle (shufflenetv2.py:57-63): even logical channels pass through,
                // odd ones feed branch_main; output = cat(pass, main)
                p->blk_stride[bi] = 1;
                std::vector<int> pass, mainin;
                for (int i = 0; i < 2 * K; ++i) (i % 2 ? mainin : pass).push_back(L[i]);
                for (int i = 0; i < K; ++i) {
                    p->tin[bi].c[i] = (unsigned short)mainin[i];
                    p->tout[bi].c[i] = (unsigned short)freep[i];
                }
                L = pass;
                L.insert(L.end(), freep.begin(), freep.end());
                freep = mainin;
            }
            for (size_t i = 0; i < L.size(); ++i) p->logical[bi].c[i] = (unsigned short)L[i];
        }
        if (st == 1) for (int i = 0; i < 96; ++i) p->c2.c[i] = (unsigned short)L[i];
        if (st == 2) for (int i = 0; i < 192; ++i) p->c3.c[i] = (unsigned short)L[i];
    }
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

extern "C" int yfv2_abi_version(void) { return YFV2_ABI_VERSION; }
extern "C" const char* yfv2_last_error(void) { return g_err; }

extern "C" int yfv2_debug_set_dispatch(int sms, int persistent_ctas) {
    if (sms < 0 || persistent_ctas < 0) {
        set_error("debug_set_dispatch: negative setting (sms=%d persistent_ctas=%d); 0 turns a setting off", sms, persistent_ctas);
        return YFV2_EINVAL;
    }
    g_sim_sms = sms;
    g_sim_ctas = persistent_ctas;
    return YFV2_OK;
}

extern "C" int yfv2_plan_create(yfv2_plan** out, int device, int N, int H, int W, int A, int C, int training) {
    if (!out || N <= 0 || H <= 0 || W <= 0 || H % 32 || W % 32 || A <= 0 || A > 8 || C <= 0 || C > 256) {
        set_error("plan_create: bad arguments (N=%d H=%d W=%d A=%d C=%d); H and W must be multiples of 32, A<=8, C<=256",
                  N, H, W, A, C);
        return YFV2_EINVAL;
    }
    if (training) {
        set_error("plan_create: training plans (batch-statistics BN + backward) are not implemented in this build");
        return YFV2_EUNSUPPORTED;
    }
    yfv2_plan* p = new (std::nothrow) yfv2_plan();
    if (!p) { set_error("plan_create: out of host memory"); return YFV2_ENOMEM; }
    memset(p, 0, sizeof(*p));
    p->device = device; p->N = N; p->H = H; p->W = W; p->A = A; p->C = C; p->training = training;
    const int pools[4] = {24, 72, 144, 288};
    size_t off = 0;
    for (int r = 0; r < 4; ++r) {
        p->h[r] = H >> (r + 2); p->w[r] = W >> (r + 2);
        p->ws1[r] = (int)align_up(p->w[r] + 2, 4); p->ws2[r] = (int)align_up(p->w[r] + 4, 4);
        p->plane[r] = (size_t)(p->h[r] + 2) * p->ws1[r];
        p->plane2[r] = (size_t)(p->h[r] + 4) * p->ws2[r];
        p->pool_planes[r] = pools[r];
        p->off_pool[r] = off;
        off += align_up(p->plane[r] * pools[r] * (size_t)N, 64);
    }
    p->off_s2 = off; off += align_up(p->plane2[2] * kFpnDepth * (size_t)N, 64);
    p->off_s3 = off; off += align_up(p->plane2[3] * kFpnDepth * (size_t)N, 64);
    for (int i = 0; i < 4; ++i) {
        p->off_t[i] = off;
        off += align_up(p->plane2[i < 2 ? 2 : 3] * kFpnDepth * (size_t)N, 64);
    }
    p->ws_floats = off;
    build_tables(p);
    size_t pk = 0;
    p->pk_stem = pk; pk += align_up(kStemPackFloats, 4);
    for (int b = 0; b < kNumBlocks; ++b) { p->pk_block[b] = pk; pk += align_up(shuffle_pack_floats(p->blk_K[b], p->blk_stride[b]), 4); }
    p->pk_fpn3 = pk; pk += pw_pack_floats(192, kFpnDepth);
    p->pk_fpn2 = pk; pk += pw_pack_floats(288, kFpnDepth);
    for (int i = 0; i < 4; ++i) { p->pk_head[i] = pk; pk += align_up(head_pack_floats(), 4); }
    p->pk_out_reg = pk; pk += pw_pack_floats(kFpnDepth, 4 * A);
    p->pk_out_oc = pk; pk += pw_pack_floats(kFpnDepth, A + C);
    if (A + C > 2 * kHeadTile || 4 * A > kHeadTile) {
        set_error("plan_create: anchors+classes = %d exceeds the two 96-wide output-conv tiles of this build (at most 192)", A + C);
        delete p;
        return YFV2_EUNSUPPORTED;
    }
    for (int i = 0; i < 4; ++i) {      // i: 0 cls2, 1 reg2, 2 cls3, 3 reg3
        const int cols = i & 1 ? 4 * A : A + C;
        p->fold_rows[i] = cols <= kHeadTile ? kHeadTile : 2 * kHeadTile;
        p->pk_foldw[i] = pk; pk += align_up((size_t)p->fold_rows[i] * kFpnDepth + p->fold_rows[i], 4);
    }
    p->pk_floats = pk;

    auto add = [&](StageKind kind, int a, int b, const char* fmt, int x, int y) {
        yfv2_plan::Stage& st = p->stages[p->n_stages++];
        st.kind = kind; st.a = a; st.b = b;
        snprintf(st.name, sizeof(st.name), fmt, x, y);
    };
    add(StageKind::stem, 0, 0, "stem", 0, 0);
    for (int b = 0, st = 0, rep = 0; b < kNumBlocks; ++b) {
        add(p->blk_stride[b] == 2 ? StageKind::block_s2 : StageKind::block_s1, b, 0, "stage%d.%d", st + 2, rep);
        if (++rep == kStageRepeats[st]) { rep = 0; ++st; }
    }
    add(StageKind::fpn, 1, 0, "fpn.S3", 0, 0); add(StageKind::fpn, 2, 0, "fpn.S2", 0, 0);
    for (int lv = 0; lv < 2; ++lv) {
        add(StageKind::heads, lv, 0, "heads%d.a", lv + 2, 0);
        add(StageKind::heads, lv, 1, "heads%d.b", lv + 2, 0);
    }
    // launch groups: consecutive stride-1 blocks of a stage run as one chained launch when an image fits (k_net.cu)
    p->launches = 0;
    for (int i = 0; i < p->n_stages; ++i) {
        yfv2_plan::Stage& st = p->stages[i];
        st.group = i;
        if (i > 0 && st.kind == StageKind::block_s1 && p->stages[i - 1].kind == StageKind::block_s1 &&
            p->blk_K[st.a] == p->blk_K[p->stages[i - 1].a] && i - p->stages[i - 1].group < 7 && blk_s1_chainable(p->blk_K[st.a], p->h[p->blk_res[st.a]], p->w[p->blk_res[st.a]]))
            st.group = p->stages[i - 1].group;
        if (st.group == i) ++p->launches;
    }
    *out = p;
    return YFV2_OK;
}

extern "C" int yfv2_plan_destroy(yfv2_plan* p) {
    delete p;
    return YFV2_OK;
}

extern "C" int yfv2_plan_workspace_bytes(const yfv2_plan* p, size_t* bytes) {
    if (!p || !bytes) { set_error("workspace_bytes: null argument"); return YFV2_EINVAL; }
    *bytes = p->ws_floats * sizeof(float);
    return YFV2_OK;
}

extern "C" int yfv2_plan_packed_bytes(const yfv2_plan* p, size_t* bytes) {
    if (!p || !bytes) { set_error("packed_bytes: null argument"); return YFV2_EINVAL; }
    *bytes = p->pk_floats * sizeof(float);
    return YFV2_OK;
}

extern "C" const char* yfv2_plan_stage_name(const yfv2_plan* p, int i) {
    if (!p || i < 0 || i >= p->n_stages) return nullptr;
    return p->stages[i].name;
}

extern "C" int yfv2_plan_invalidate_workspace(yfv2_plan* p) {
    if (!p) { set_error("invalidate_workspace: null plan"); return YFV2_EINVAL; }
    p->ws_zeroed = nullptr;          // the next forward re-zeroes the frames around every activation plane
    return YFV2_OK;
}

extern "C" int yfv2_plan_stage_group(const yfv2_plan* p, int i) {
    if (!p || i < 0 || i >= p->n_stages) return -1;
    return p->stages[i].group;
}

extern "C" int yfv2_plan_forward_launches(const yfv2_plan* p, int* n) {
    if (!p || !n) { set_error("forward_launches: null argument"); return YFV2_EINVAL; }
    *n = p->launches;
    return YFV2_OK;
}

namespace {

int pack_pw(Cursor& cur, bool bn, bool bias, int Nout, int K, float* pack, int Np, int n_off, cudaStream_t s) {
    const float* w = cur.params[cur.p];
    const float *g = nullptr, *b = nullptr, *m = nullptr, *v = nullptr, *bi = nullptr;
    if (bn) { g = cur.params[cur.p + 1]; b = cur.params[cur.p + 2]; m = cur.bn[2 * cur.b]; v = cur.bn[2 * cur.b + 1]; cur.p += 3; cur.b += 1; }
    else if (bias) { bi = cur.params[cur.p + 1]; cur.p += 2; }
    else cur.p += 1;
    if (!w || (bn && (!g || !b || !m || !v)) || (bias && !bi)) { set_error("pack_weights: null tensor pointer near param %d", cur.p); return YFV2_EINVAL; }
    const int total = Nout * K;
    pack_pw_kernel<<<(total + 255) / 256, 256, 0, s>>>(w, Nout, K, g, b, m, v, bi, pack, Np, n_off, pack + (size_t)K * Np,
                                                        pack + (size_t)K * Np + Np);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

int pack_dw(Cursor& cur, int Cn, int ksz, float* pack, cudaStream_t s) {
    const float* w = cur.params[cur.p];
    const float *g = cur.params[cur.p + 1], *b = cur.params[cur.p + 2], *m = cur.bn[2 * cur.b], *v = cur.bn[2 * cur.b + 1];
    cur.p += 3; cur.b += 1;
    if (!w || !g || !b || !m || !v) { set_error("pack_weights: null tensor pointer near param %d", cur.p); return YFV2_EINVAL; }
    const int KK = ksz * ksz, R = ksz == 3 ? 12 : 28;
    pack_dw_kernel<<<(Cn * KK + 255) / 256, 256, 0, s>>>(w, Cn, KK, R, g, b, m, v, pack);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

#define TRY(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)

}  // namespace

extern "C" int yfv2_pack_weights(yfv2_plan* p, const float* const* params, const float* const* bn_running, void* packed,
                                 void* stream) {
    if (!p || !params || !bn_running || !packed) { set_error("pack_weights: null argument"); return YFV2_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    float* pk = (float*)packed;
    YFV2_CUDA(cudaMemsetAsync(pk, 0, p->pk_floats * sizeof(float), s));
    Cursor cur{params, bn_running};
    // backbone.first_conv (shufflenetv2.py:74-78)
    TRY(pack_pw(cur, true, false, 24, 27, pk + p->pk_stem, 24, 0, s));
    for (int b = 0; b < kNumBlocks; ++b) {
        const int K = p->blk_K[b];
        float* d = pk + p->pk_block[b];
        const int pwn = pw_pack_floats(K, K), dwn = dw3_pack_floats(K);
        if (p->blk_stride[b] == 2) {
            // state_dict order: branch_main (pw1, dw, pw2) then branch_proj (dw, pw); pack order DWp|PWp|PW1|DW|PW2
            TRY(pack_pw(cur, true, false, K, K, d + dwn + pwn, K, 0, s));
            TRY(pack_dw(cur, K, 3, d + dwn + 2 * pwn, s));
            TRY(pack_pw(cur, true, false, K, K, d + 2 * dwn + 2 * pwn, K, 0, s));
            TRY(pack_dw(cur, K, 3, d, s));
            TRY(pack_pw(cur, true, false, K, K, d + dwn, K, 0, s));
        } else {
            TRY(pack_pw(cur, true, false, K, K, d, K, 0, s));
            TRY(pack_dw(cur, K, 3, d + pwn, s));
            TRY(pack_pw(cur, true, false, K, K, d + pwn + dwn, K, 0, s));
        }
    }
    // fpn: conv1x1_2, conv1x1_3, cls_head_2, reg_head_2, reg_head_3, cls_head_3 (fpn.py:35-49 registration order)
    TRY(pack_pw(cur, true, false, kFpnDepth, 288, pk + p->pk_fpn2, kFpnDepth, 0, s));
    TRY(pack_pw(cur, true, false, kFpnDepth, 192, pk + p->pk_fpn3, kFpnDepth, 0, s));
    const int head_order[4] = {0, 1, 3, 2};     // pk_head index: 0 cls2, 1 reg2, 2 cls3, 3 reg3
    struct Pw2 { const float *w, *g, *b, *m, *v; } pw2[4];
    for (int i = 0; i < 4; ++i) {
        float* d = pk + p->pk_head[head_order[i]];
        const int dwn = dw5_pack_floats(kFpnDepth), pwn = pw_pack_floats(kFpnDepth, kFpnDepth);
        const int hi_ = head_order[i];
        TRY(pack_dw(cur, kFpnDepth, 5, d, s));
        TRY(pack_pw(cur, true, false, kFpnDepth, kFpnDepth, d + dwn, kFpnDepth, 0, s));
        TRY(pack_dw(cur, kFpnDepth, 5, d + dwn + pwn, s));
        pw2[hi_] = Pw2{cur.params[cur.p], cur.params[cur.p + 1], cur.params[cur.p + 2], cur.bn[2 * cur.b], cur.bn[2 * cur.b + 1]};
        TRY(pack_pw(cur, true, false, kFpnDepth, kFpnDepth, d + 2 * dwn + pwn, kFpnDepth, 0, s));
    }
    // output_reg_layers, output_obj_layers, output_cls_layers (detector.py:17-19); obj and cls share one pack
    const float* wo[3] = {cur.params[cur.p], cur.params[cur.p + 2], cur.params[cur.p + 4]};       // reg, obj, cls weights
    const float* bo[3] = {cur.params[cur.p + 1], cur.params[cur.p + 3], cur.params[cur.p + 5]};   // and biases
    TRY(pack_pw(cur, false, true, 4 * p->A, kFpnDepth, pk + p->pk_out_reg, round4(4 * p->A), 0, s));
    const int Moc = round4(p->A + p->C);
    TRY(pack_pw(cur, false, true, p->A, kFpnDepth, pk + p->pk_out_oc, Moc, 0, s));
    TRY(pack_pw(cur, false, true, p->C, kFpnDepth, pk + p->pk_out_oc, Moc, p->A, s));
    // folded second halves of the four heads (cls heads feed obj|cls, reg heads feed reg)
    for (int h = 0; h < 4; ++h) {
        const Pw2& q = pw2[h];
        float* Fw = pk + p->pk_foldw[h];
        float* Fb = Fw + (size_t)p->fold_rows[h] * kFpnDepth;
        const int K = kFpnDepth;
        auto fold = [&](int which, int Mo, int n_off) -> int {
            if (!wo[which] || !bo[which]) { set_error("pack_weights: null output-layer tensor"); return YFV2_EINVAL; }
            fold_head_kernel<<<(Mo * K + 255) / 256, 256, 0, s>>>(wo[which], bo[which], Mo, q.w, q.g, q.b, q.m, q.v, K, n_off, Fw, Fb);
            YFV2_LAUNCH_CHECK();
            return YFV2_OK;
        };
        if (h & 1) { TRY(fold(0, 4 * p->A, 0)); }
        else { TRY(fold(1, p->A, 0)); TRY(fold(2, p->C, p->A)); }
    }
    if (cur.p != YFV2_NUM_PARAMS || cur.b != YFV2_NUM_BN) {
        set_error("pack_weights: internal walk consumed %d params / %d BN layers", cur.p, cur.b);
        return YFV2_EINVAL;
    }
    return YFV2_OK;
}

namespace {
// the input of head level lv (S2 or S3) and its mid-head scratch of the cls and reg branches
void head_planes(const yfv2_plan* p, float* ws, int lv, Planes& sIn, Planes& t_cls, Planes& t_reg) {
    sIn = flat_planes(p, ws, lv ? p->off_s3 : p->off_s2, 2 + lv);
    t_cls = flat_planes(p, ws, p->off_t[2 * lv], 2 + lv);
    t_reg = flat_planes(p, ws, p->off_t[2 * lv + 1], 2 + lv);
}

// The launches of fused stages [first, last) of a forward on workspace ws over sms SMs, in order: each stage is one launch, except
// that consecutive stride-1 blocks of one launch group inside the range run as one chained launch.  ws decides the kernels that
// need 16-byte-aligned planes (the band walks, the heads' staged windows); it is not dereferenced.  Host only.
int plan_launches(const yfv2_plan* p, float* ws, int is_u8, int sms, int first, int last, Launch* out, int* n) {
    *n = 0;
    for (int si = first; si < last; ++si) {
        const yfv2_plan::Stage& st = p->stages[si];
        Launch& L = out[(*n)++] = Launch{};
        L.first = si;
        const int b = st.a;
        switch (st.kind) {
        case StageKind::stem: TRY(describe_stem(p->N, p->H, p->W, is_u8, sms, L)); break;
        case StageKind::block_s1: {
            int nb = 1;
            while (si + nb < last && p->stages[si + nb].group == st.group) ++nb;
            TRY(describe_blk_s1(p->blk_K[b], pool_planes(p, ws, p->blk_res[b]), nb, p->N, sms, L));
            si += nb - 1;
        } break;
        case StageKind::block_s2:
            TRY(describe_blk_s2(p->blk_K[b], pool_planes(p, ws, p->blk_res[b] - 1), pool_planes(p, ws, p->blk_res[b]), p->N, sms, L));
            break;
        case StageKind::fpn: {
            const int r = st.a == 1 ? 3 : 2;
            TRY(describe_fpn(st.a, p->h[r], p->w[r], p->N, sms, L));
        } break;
        case StageKind::heads: {
            Planes sIn, t_cls, t_reg;
            head_planes(p, ws, st.a, sIn, t_cls, t_reg);
            TRY(describe_heads(st.b, sIn, t_cls, t_reg, p->A, p->C, p->N, sms, L));
        } break;
        }
        L.last = si + 1;
    }
    return YFV2_OK;
}

// Runs fused stages [first, last) of the forward: the launches plan_launches describes, each with its arguments.
int forward_impl(yfv2_plan* p, const void* x, int is_u8, const void* packed, float* const preds[6], void* workspace,
                 int first, int last, cudaStream_t s) {
    if (!p || !x || !packed || !preds || !workspace) { set_error("forward: null argument"); return YFV2_EINVAL; }
    for (int i = 0; i < 6; ++i) if (!preds[i]) { set_error("forward: null output %d", i); return YFV2_EINVAL; }
    if (last < 0) last = p->n_stages;
    if (first < 0 || last > p->n_stages || first > last) { set_error("forward: bad stage range [%d,%d)", first, last); return YFV2_EINVAL; }
    float* ws = (float*)workspace;
    const float* pk = (const float*)packed;
    Launch launches[kMaxStages];
    int n = 0;
    TRY(plan_launches(p, ws, is_u8, sm_count(), first, last, launches, &n));
    pdl_reset();                                            // the first kernel of this call is serialized normally
    if (p->ws_zeroed != workspace) {
        // the zero frames around every plane are never written afterwards (kernels store interior pixels only)
        YFV2_CUDA(cudaMemsetAsync(workspace, 0, p->ws_floats * sizeof(float), s));
        p->ws_zeroed = workspace;
    }
    for (int i = 0; i < n; ++i) {
        const Launch& L = launches[i];
        const yfv2_plan::Stage& st = p->stages[L.first];
        const int b = st.a;
        switch (st.kind) {
        case StageKind::stem: {
            StemArgs a{L, x, is_u8, p->N, p->H, p->W, pool_planes(p, ws, 0), pk + p->pk_stem};
            TRY(launch_stem(a, s));
        } break;
        case StageKind::heads: {
            const int lv = st.a, half = st.b;
            Planes sIn, t_cls, t_reg;
            head_planes(p, ws, lv, sIn, t_cls, t_reg);
            const float* w_cls = pk + p->pk_head[2 * lv];
            const float* w_reg = pk + p->pk_head[2 * lv + 1];
            // each half of a head pack is DW5 | PW
            const size_t dwn = dw5_pack_floats(kFpnDepth), half_off = (size_t)half * (dwn + pw_pack_floats(kFpnDepth, kFpnDepth));
            const float* wdw[2] = {w_cls + half_off, w_reg + half_off};
            const float* wpw[2] = {half ? pk + p->pk_foldw[2 * lv] : w_cls + dwn, half ? pk + p->pk_foldw[2 * lv + 1] : w_reg + dwn};
            TRY(heads_launch(L, half, sIn, t_cls, t_reg, wdw, wpw, preds[3 * lv], preds[3 * lv + 1], preds[3 * lv + 2], p->A, p->C,
                             p->N, s));
        } break;
        case StageKind::block_s1: {   // fused stride-1 blocks [L.first, L.last)
            const int K = p->blk_K[b];
            const float *w1[7], *w2[7], *wd[7];
            for (int j = 0; j < L.last - L.first; ++j) {
                const float* d = pk + p->pk_block[b + j];
                const int pwn = pw_pack_floats(K, K);
                w1[j] = d; wd[j] = d + pwn; w2[j] = d + pwn + dw3_pack_floats(K);
            }
            TRY(blk_launch_s1(L, K, pool_planes(p, ws, p->blk_res[b]), &p->tin[b], &p->tout[b], w1, wd, w2, s));
        } break;
        case StageKind::block_s2: {   // fused stride-2 block; pack order DWp | PWp | PW1 | DW | PW2
            const int K = p->blk_K[b];
            const float* d = pk + p->pk_block[b];
            const int dwn = dw3_pack_floats(K), pwn = pw_pack_floats(K, K);
            TRY(blk_launch_s2(L, K, pool_planes(p, ws, p->blk_res[b] - 1), pool_planes(p, ws, p->blk_res[b]), p->tin[b], p->tout[b],
                              d, d + dwn, d + dwn + pwn, d + dwn + 2 * pwn, d + 2 * dwn + 2 * pwn, s));
        } break;
        case StageKind::fpn: {        // FPN reducers: S3 from C3, S2 from cat(up2(C3), C2)
            const Planes c3 = pool_planes(p, ws, 3), c2 = pool_planes(p, ws, 2);
            const Planes out = st.a == 1 ? flat_planes(p, ws, p->off_s3, 3) : flat_planes(p, ws, p->off_s2, 2);
            TRY(fpn_launch(L, c3, p->c3, c2, p->c2, out, pk + (st.a == 1 ? p->pk_fpn3 : p->pk_fpn2), p->N, s));
        } break;
        }
    }
    return YFV2_OK;
}
}  // namespace

extern "C" int yfv2_forward_range(yfv2_plan* p, const void* x, int is_u8, const void* packed, float* const preds[6],
                                  void* workspace, int first, int last, void* stream) {
    return forward_impl(p, x, is_u8, packed, preds, workspace, first, last, (cudaStream_t)stream);
}

extern "C" int yfv2_forward(yfv2_plan* p, const float* x, const void* packed, float* const preds[6], void* workspace,
                            void* stream) {
    return forward_impl(p, x, 0, packed, preds, workspace, 0, -1, (cudaStream_t)stream);
}

extern "C" int yfv2_forward_u8(yfv2_plan* p, const uint8_t* x, const void* packed, float* const preds[6], void* workspace,
                               void* stream) {
    return forward_impl(p, x, 1, packed, preds, workspace, 0, -1, (cudaStream_t)stream);
}

// ---- whole step with host buffers ---------------------------------------------------------------------------
namespace {
struct DetectLayout {
    size_t off_x, off_pred[6], off_out, off_counts, total;
};
DetectLayout detect_layout(const yfv2_plan* p, int max_det) {
    DetectLayout L;
    size_t off = align_up(p->ws_floats * sizeof(float), 256);
    L.off_x = off; off += align_up((size_t)p->N * 3 * p->H * p->W, 256);
    for (int lv = 0; lv < 2; ++lv) {
        const size_t hw = (size_t)p->h[2 + lv] * p->w[2 + lv];
        const int ch[3] = {4 * p->A, p->A, p->C};
        for (int k = 0; k < 3; ++k) { L.off_pred[3 * lv + k] = off; off += align_up((size_t)p->N * ch[k] * hw * sizeof(float), 256); }
    }
    L.off_out = off; off += align_up((size_t)p->N * max_det * 6 * sizeof(float), 256);
    L.off_counts = off; off += align_up((size_t)p->N * sizeof(int), 256);
    L.total = off;
    return L;
}
}  // namespace

extern "C" size_t yfv2_detect_workspace_bytes(const yfv2_plan* p, int max_det) {
    if (!p || max_det <= 0) return 0;
    return detect_layout(p, max_det).total;
}

extern "C" int yfv2_detect_u8_host(yfv2_plan* p, const uint8_t* x_host, const void* packed, const double* anchors_host,
                                   float conf_thres, double iou_thres, int max_det, float* out_host, int* counts_host,
                                   void* workspace, void* stream) {
    if (!p || !x_host || !packed || !anchors_host || !out_host || !counts_host || !workspace || max_det <= 0) {
        set_error("detect_u8_host: null argument");
        return YFV2_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const DetectLayout L = detect_layout(p, max_det);
    unsigned char* ws = (unsigned char*)workspace;
    uint8_t* x_dev = ws + L.off_x;
    float* preds[6];
    for (int i = 0; i < 6; ++i) preds[i] = (float*)(ws + L.off_pred[i]);
    float* out_dev = (float*)(ws + L.off_out);
    int* counts_dev = (int*)(ws + L.off_counts);
    // a request the fused decode+NMS refuses is refused here, before the copy and the forward are enqueued
    TRY(decode_nms_check(preds, p->N, p->H, p->W, p->A, p->C, anchors_host, conf_thres, iou_thres, nullptr, 0, max_det, 4096.0f,
                         out_dev, counts_dev, nullptr));
    YFV2_CUDA(cudaMemcpyAsync(x_dev, x_host, (size_t)p->N * 3 * p->H * p->W, cudaMemcpyHostToDevice, s));
    struct PdlOff { PdlOff() { g_pdl_call = false; } ~PdlOff() { g_pdl_call = true; } } pdl_off_guard;
    TRY(forward_impl(p, x_dev, 1, packed, preds, ws, 0, -1, s));
    TRY(yfv2_decode_nms(preds, p->N, p->H, p->W, p->A, p->C, anchors_host, conf_thres, iou_thres, nullptr, 0, max_det,
                        4096.0f, out_dev, counts_dev, nullptr, nullptr, stream));
    YFV2_CUDA(cudaMemcpyAsync(out_host, out_dev, (size_t)p->N * max_det * 6 * sizeof(float), cudaMemcpyDeviceToHost, s));
    YFV2_CUDA(cudaMemcpyAsync(counts_host, counts_dev, (size_t)p->N * sizeof(int), cudaMemcpyDeviceToHost, s));
    return YFV2_OK;
}

// ---- debug: dense NCHW copy of an intermediate tensor ------------------------------------------------------
extern "C" int yfv2_debug_gather(const yfv2_plan* p, const void* workspace, int which, float* out, int* dims4, void* stream) {
    if (!p || !workspace || !dims4) { set_error("debug_gather: null argument"); return YFV2_EINVAL; }
    float* ws = (float*)workspace;
    Planes P; ChanTab tab; int Cn;
    for (int i = 0; i < kMaxCh; ++i) tab.c[i] = (unsigned short)i;
    if (which == 0) { P = pool_planes(p, ws, 0); Cn = 24; }
    else if (which >= 1 && which <= kNumBlocks) { const int b = which - 1; P = pool_planes(p, ws, p->blk_res[b]); Cn = 2 * p->blk_K[b]; tab = p->logical[b]; }
    else if (which == 17) { P = flat_planes(p, ws, p->off_s2, 2); Cn = kFpnDepth; }
    else if (which == 18) { P = flat_planes(p, ws, p->off_s3, 3); Cn = kFpnDepth; }
    else if (which >= 19 && which <= 22) { const int i = which - 19; P = flat_planes(p, ws, p->off_t[i], i < 2 ? 2 : 3); Cn = kFpnDepth; }
    else { set_error("debug_gather: unknown tensor id %d", which); return YFV2_EINVAL; }
    dims4[0] = p->N; dims4[1] = Cn; dims4[2] = P.H; dims4[3] = P.W;
    if (!out) return YFV2_OK;
    const long long total = (long long)p->N * Cn * P.H * P.W;
    gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(P, tab, Cn, out, total);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// ---- test hook: the launch records of a whole forward ---------------------------------------------------------------------
extern "C" int yfv2_plan_debug_launches(const yfv2_plan* p, const void* workspace, int is_u8, int sms, yfv2_launch* out, int cap,
                                        int* n) {
    if (!p || !n || sms < 0 || cap < 0 || (cap > 0 && !out)) { set_error("plan_debug_launches: bad argument"); return YFV2_EINVAL; }
    // NULL: any 16-byte-aligned workspace (its address is only tested for alignment)
    float* ws = workspace ? (float*)workspace : reinterpret_cast<float*>((uintptr_t)256);
    Launch launches[kMaxStages];
    TRY(plan_launches(p, ws, is_u8, sms ? sms : sm_count(), 0, p->n_stages, launches, n));
    for (int i = 0; i < cap && i < *n; ++i) {
        const Launch& L = launches[i];
        yfv2_launch& d = out[i];
        snprintf(d.kernel, sizeof(d.kernel), "%s", kernel_ref(L.kernel).name);
        d.first = L.first; d.last = L.last;
        d.smem = (long long)L.smem;
        d.grid[0] = (int)L.grid.x; d.grid[1] = (int)L.grid.y; d.grid[2] = (int)L.grid.z;
        d.persistent = L.persistent; d.items = L.items;
        d.R = L.R; d.bands = L.bands; d.G = L.G; d.window_stride = L.CS;
    }
    return YFV2_OK;
}
