// Shared declarations for libyfv2.so (sm_90a, H100).
//
// Activation storage ("plane pools"): every intermediate tensor of the network lives as separate
// channel planes, plane(n, c) = base + n*sN + c*sC.  A plane is an H x W fp32 image inside a ZERO FRAME:
// rows of Ws floats (Ws = W + 2*pad rounded up to 4), `pad` zero rows above and below, pixel (y,x) at
// org + y*Ws + x.  Kernels only ever write interior pixels, so the frame (zeroed once per workspace) is
// the zero padding of every 3x3 / 5x5 convolution: kernels read a band of rows *with its halo* without any
// bounds test.  A logical
// tensor is a list of physical plane ids (ChanTab).  ShuffleNetV2's channel_shuffle / split / concat
// (reference model/backbone/shufflenetv2.py:48-63) therefore cost nothing: they are edits of the id
// list done on the host when the plan is built, and the "passthrough" half of a stride-1 block is
// never read or written at all.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/yfv2.h"

namespace yfv2 {

constexpr int kMaxCh = 288;       // widest logical tensor: cat(up(C3), C2), fpn.py:58
constexpr float kBnEps = 1e-5f;   // nn.BatchNorm2d default

struct Planes {
    float* base;
    long long sN;   // floats between consecutive images
    long long sC;   // floats between consecutive planes
    int H, W;       // image size
    int Ws;         // row stride (floats), multiple of 4
    int pad;        // zero frame width (rows and columns)
    int org;        // offset of pixel (0,0) inside a plane = pad*Ws + pad
};

struct ChanTab {
    unsigned short c[kMaxCh];
};

__device__ __forceinline__ float* plane_ptr(const Planes& P, int n, int c) {
    return P.base + (long long)n * P.sN + (long long)c * P.sC;
}

// ---- error plumbing (host) ---------------------------------------------------------------------
void set_error(const char* fmt, ...);

#define YFV2_CUDA(call)                                                                       \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            yfv2::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return YFV2_ECUDA;                                                                \
        }                                                                                     \
    } while (0)

#define YFV2_LAUNCH_CHECK()                                                                   \
    do {                                                                                      \
        cudaError_t e__ = cudaGetLastError();                                                 \
        if (e__ != cudaSuccess) {                                                             \
            yfv2::set_error("%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
            return YFV2_ECUDA;                                                                \
        }                                                                                     \
    } while (0)

// ---- packed weight layouts (floats) ----------------------------------------------------------------
// PW  (1x1 conv K->N [+BN]):  Wt[K][Np] (Np = N rounded up to 4, zero padded), scale[Np], shift[Np]
// DW3 (3x3 depthwise + BN):   per channel 12 floats: w[9], scale, shift, 0
// DW5 (5x5 depthwise + BN):   per channel 28 floats: w[25], scale, shift, 0
// STEM (3x3 s2 3->24 + BN):   Wt[27][24] (k = c*9+ky*3+kx), scale[24], shift[24]
__host__ __device__ constexpr int round4(int x) { return (x + 3) & ~3; }
__host__ __device__ constexpr int pw_pack_floats(int K, int N) { return K * round4(N) + 2 * round4(N); }
__host__ __device__ constexpr int dw3_pack_floats(int C) { return C * 12; }
__host__ __device__ constexpr int dw5_pack_floats(int C) { return C * 28; }
constexpr int kStemPackFloats = 27 * 24 + 48;

// ---- device helpers --------------------------------------------------------------------------------
// cooperative copy global -> shared, count floats (both 4-byte aligned only)
__device__ __forceinline__ void copy_to_smem(float* dst, const float* __restrict__ src, int count) {
    for (int i = threadIdx.x; i < count; i += blockDim.x) dst[i] = __ldg(src + i);
}

// acc[i][n] += Wt[k][n] * x[i]  for one k; Wt row is N floats in shared memory, read as float4 broadcasts
template <int N, int PPT>
__device__ __forceinline__ void fma_row(const float* __restrict__ wrow, const float (&x)[PPT], float (&acc)[PPT][N]) {
#pragma unroll
    for (int n4 = 0; n4 < N / 4; ++n4) {
        const float4 w = *reinterpret_cast<const float4*>(wrow + 4 * n4);
#pragma unroll
        for (int i = 0; i < PPT; ++i) {
            acc[i][4 * n4 + 0] = fmaf(w.x, x[i], acc[i][4 * n4 + 0]);
            acc[i][4 * n4 + 1] = fmaf(w.y, x[i], acc[i][4 * n4 + 1]);
            acc[i][4 * n4 + 2] = fmaf(w.z, x[i], acc[i][4 * n4 + 2]);
            acc[i][4 * n4 + 3] = fmaf(w.w, x[i], acc[i][4 * n4 + 3]);
        }
    }
}

// ---- cp.async (LDGSTS) helpers: fire-and-forget global->shared copies, no register staging ----------------
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gsrc) : "memory");
}
// 16 bytes (both addresses 16-byte aligned), bypassing L1; src_bytes == 0 reads nothing and zero-fills the 16 bytes
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gsrc, uint32_t src_bytes) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
}

int sm_count();                  // the device's SM count, or the one yfv2_debug_set_dispatch set
int persistent_cta_cap();        // yfv2_debug_set_dispatch: CTAs of a persistent launch (at most one per item), 0: by occupancy
constexpr size_t kSmemCap = 227 * 1024;

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------
// Every stage of a forward is its own kernel with a fixed prologue (weights -> shared memory, barrier
// init: 5-15 us when ~300 CTAs pull the same weight pack out of L2).  None of that depends on the previous stage, so the
// stage kernels are launched with programmatic stream serialization: a kernel may become resident while its predecessor
// drains, runs its prologue, and executes pdl_wait() (griddepcontrol.wait: predecessor complete and its memory visible)
// before it touches any activation.  pdl_trigger() at the top of every kernel lets the successor be scheduled as soon as
// SM resources free up.  Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// The first kernel of a forward call is launched normally (its prologue may read weights an earlier pack kernel wrote).
bool pdl_take();                 // true if the next launch may overlap its predecessor; arms the flag
void pdl_reset();                // next launch is a plain one
bool pdl_allowed();              // PDL enabled for the current API call
// kern: a __global__ function taking one argument struct, arg: that struct
inline cudaError_t launch_k(const void* kern, dim3 grid, int block, size_t smem, cudaStream_t s, bool pdl, const void* arg) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = dim3((unsigned)block); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    void* args[1] = {const_cast<void*>(arg)};
    return cudaLaunchKernelExC(&cfg, kern, args);
}

// ---- the forward's launches: described on the host (plan.cu plan_launches), then launched --------------------
// Every kernel a forward can launch.  kernel_ref() maps an id to the __global__ function and its name, both from one
// YFV2_KERNEL_REF expression: the name is the demangled symbol after yfv2::(anonymous namespace)::, without spaces.
enum class KernelId {
    stem_f32, stem_u8, chain96, s2_image96, fpn192, fpn288, head0, head1, head2,
    blk24_s1, blk24_s2, blk48_s1, blk48_s2, blk96_s1, blk96_s2,     // blk_kernel<K, STRIDE>
    walk24_s1, walk48_s1, walk24_s2, walk48_s2,                     // walk::blk_kernel<K, STRIDE>
};
struct KernelRef { const void* fn; const char* name; };
#define YFV2_KERNEL_REF(...) yfv2::KernelRef{reinterpret_cast<const void*>(&__VA_ARGS__), #__VA_ARGS__}
KernelRef kernel_ref(KernelId k);           // k_net.cu
KernelRef stem_kernel_ref(bool u8);         // k_stem.cu

constexpr int kThreads = 256;               // threads per CTA of every forward kernel

// One kernel launch of a forward: what it runs over which fused stages, with which grid and shared memory.
struct Launch {
    KernelId kernel;
    int first, last;            // fused stages [first, last) of the plan
    size_t smem;                // dynamic shared memory, bytes
    dim3 grid;                  // fixed grid; persistent: grid.x is the SM count, and the launch takes
    bool persistent;            //   min(items, CTAs per SM by occupancy x grid.x) CTAs that walk the items
    int items;                  // work items the grid walks
    int R, bands, G;            // block launches: rows per band, bands per image, walk step (walk::blk_kernel<K, 1>)
    int CS;                     // heads: channel stride of a staged window slot (floats); 0: the stencils read the planes
    struct { int TRo, TWo, S, tilesX, tilesY; bool vec; } stem;    // stem tiling; vec: staged asynchronously if x is aligned
};

// Records of single launches (k_net.cu, k_stem.cu); an argument error is set_error + its code
int describe_stem(int N, int H, int W, int is_u8, int sms, Launch& L);
int describe_blk_s1(int K, const Planes& P, int nblk, int N, int sms, Launch& L);
int describe_blk_s2(int K, const Planes& in, const Planes& out, int N, int sms, Launch& L);
int describe_fpn(int which, int H, int W, int N, int sms, Launch& L);
int describe_heads(int half, const Planes& sIn, const Planes& tcls, const Planes& treg, int A, int C, int N, int sms, Launch& L);

// The one launch path: shared-memory attribute, the occupancy-sized grid of a persistent launch, the launch, its check
int launch(const Launch& L, const void* args, cudaStream_t s);

// Argument structs of the launches, filled from the record (k_net.cu, k_stem.cu)
struct StemArgs {
    const Launch& launch;    // describe_stem's record
    const void* x;       // [N,3,H,W] fp32 or uint8
    int is_u8;
    int N, H, W;         // input dims
    Planes out;          // 24 planes at H/4 x W/4, ids 0..23
    const float* wpack;  // STEM layout
};
int launch_stem(const StemArgs& a, cudaStream_t s);
int blk_launch_s1(const Launch& L, int K, const Planes& P, const ChanTab* tin, const ChanTab* tout, const float* const* w1,
                  const float* const* wdw, const float* const* w2, cudaStream_t s);
int blk_launch_s2(const Launch& L, int K, const Planes& in, const Planes& out, const ChanTab& tin, const ChanTab& tout, const float* wdwp,
                  const float* wp, const float* w1, const float* wdwm, const float* w2, cudaStream_t s);
int fpn_launch(const Launch& L, const Planes& c3, const ChanTab& t3, const Planes& c2, const ChanTab& t2, const Planes& out,
               const float* pw, int N, cudaStream_t s);
int heads_launch(const Launch& L, int half, const Planes& sIn, const Planes& tcls, const Planes& treg, const float* const wdw[2],
                 const float* const wpw[2], float* reg, float* obj, float* cls, int A, int C, int N, cudaStream_t s);

// Every host-side check of yfv2_decode_nms (k_post.cu): geometry, NMS arguments and the kernel's shared memory; set_error + its
// code on a refusal.  Callers that enqueue work before the fused decode+NMS (yfv2_detect_u8_host) run it first.
int decode_nms_check(const float* const preds[6], int N, int H, int W, int A, int C, const double* anchors_host, float conf_thres,
                     double iou_thres, const int* class_filter, int n_filter, int max_det, float max_wh, float* out, int* counts,
                     int* kept_idx);

// ---- the training operators' launches: described on the host (k_train.cu describe_*), then launched ----------------------------
// Every kernel a yfv2_op_* call or the native trainer launches, and the memsets they make.
enum class TrainKernel {
    memset, gemm2_32, gemm2_64, wgrad_rows, wgrad_tiled32, wgrad_tiled64, wgrad_reduce, bias_grad,
    dw_fwd3, dw_fwd5, dw_dgrad3, dw_dgrad5, dw_wgrad3, dw_wgrad5, stem_fwd24, stem_fwd_generic, stem_wgrad,
    bn_stats, bn_finalize, bn_apply, bn_bwd_reduce, bn_bwd_apply, bn_eval_stats, bn_eval_bwd_apply, bn_affine_grads,
    maxpool_fwd, maxpool_bwd, upsample2_fwd, upsample2_bwd, chan_copy, axpy,
};

constexpr size_t kTrainLaunchPtrs = 10, kTrainLaunchInts = 10;      // most pointer / integer arguments of a training kernel

// One kernel launch (or memset) of a training operator: the kernel and its geometry, the facts its variant was chosen by, and its
// arguments in the kernel's signature order, pointers in p and integers in n (a memset: p[0] and bytes).
struct TrainLaunch {
    TrainKernel kernel = TrainKernel::memset;
    dim3 grid;
    int block = 256;
    size_t smem = 0;                         // dynamic shared memory, bytes
    int op = -1;                             // native trainer: the op of its program the launch belongs to (-1: none)
    bool bwd = false;                        //   and whether it runs in the backward
    int bm = 0;                              // gemm2: tile height
    bool vec_b = false, vec_c = false;       // gemm2: float4 access of B / C
    bool vec = false;                        // bn_stats / bn_apply / bn_eval_bwd_apply: float4 access
    int pchunk = 0, chunks = 0;              // wgrad: pixels per block slice, slices per image
    bool partial = false;                    // wgrad: per-block partial sums summed by wgrad_reduce_kernel, else atomics into zeroed dw
    int slices = 0;                          // BatchNorm per-channel reductions: image slices (grid.y)
    int accumulate = 0;                      // chan_copy / axpy: add to the destination
    size_t bytes = 0;                        // memset
    const void* p[kTrainLaunchPtrs] = {};
    long long n[kTrainLaunchInts] = {};
    double d = 0.0;
    float f = 0.f;
};
using TrainLaunches = std::vector<TrainLaunch>;

// One describe function per operator (k_train.cu): appends the records of one call; the addresses are never dereferenced, they only
// decide alignment.  An argument the operator refuses is set_error + its code, with nothing appended.
int describe_conv1x1_fwd(const float* x, const float* w, const float* bias, float* y, int N, int K, int M, int HW, TrainLaunches& L);
int describe_conv1x1_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, float* dbias, int N, int K, int M, int HW,
                         float* wscratch, size_t wscratch_floats, int sms, TrainLaunches& L);
int describe_dwconv_fwd(const float* x, const float* w, float* y, int N, int C, int H, int W, int ks, int stride, TrainLaunches& L);
int describe_dwconv_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, int N, int C, int H, int W, int ks, int stride,
                        TrainLaunches& L);
int describe_stem_fwd(const float* x, const float* w, float* y, int N, int M, int H, int W, TrainLaunches& L);
int describe_stem_wgrad(const float* x, const float* dy, float* dw, int N, int M, int H, int W, TrainLaunches& L);
int describe_bn_train_fwd(const float* x, const float* gamma, const float* beta, float* running_mean, float* running_var, float* y,
                          float* save_mean, float* save_invstd, double* scratch, int N, int C, int HW, int relu, TrainLaunches& L);
int describe_bn_train_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean, const float* save_invstd,
                          float* dx, float* dgamma, float* dbeta, double* scratch, int N, int C, int HW, int relu, TrainLaunches& L);
int describe_bn_eval_fwd(const float* x, const float* gamma, const float* beta, const float* running_mean, const float* running_var, float* y,
                         float* save_mean, float* save_invstd, int N, int C, int HW, int relu, TrainLaunches& L);
int describe_bn_eval_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean, const float* save_invstd,
                         float* dx, float* dgamma, float* dbeta, double* scratch, int N, int C, int HW, int relu, TrainLaunches& L);
int describe_maxpool_fwd(const float* x, float* y, int* idx, int planes, int H, int W, TrainLaunches& L);
int describe_maxpool_bwd(const float* dy, const int* idx, float* dx, int planes, int H, int W, TrainLaunches& L);
int describe_upsample2_fwd(const float* x, float* y, int planes, int H, int W, TrainLaunches& L);
int describe_upsample2_bwd(const float* dy, float* dx, int planes, int H, int W, TrainLaunches& L);
// the native trainer's channel copies and gradient sums: dst[n][doff + c*dstep][p] (+)= src[n][soff + c*sstep][p], dst[i] (+)= src[i]
void describe_chan_copy(const float* src, int Cs, int soff, int sstep, float* dst, int Cd, int doff, int dstep, int count, int N, int HW,
                        int accumulate, int sms, TrainLaunches& L);
void describe_axpy(const float* src, float* dst, long long n, int accumulate, int sms, TrainLaunches& L);

// The one launch path of the training operators: the record's kernel or memset, then its check
int launch(const TrainLaunch& L, cudaStream_t s);
int launch_all(const TrainLaunches& L, cudaStream_t s);
// The records as the test hooks return them: min(cap, count) written, the count in *n
int debug_records(const TrainLaunches& L, yfv2_train_launch* out, int cap, int* n);

}  // namespace yfv2
