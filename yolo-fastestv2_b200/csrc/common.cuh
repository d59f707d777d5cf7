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

int sm_count();
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
template <class Arg, class Kern>
cudaError_t launch_k(Kern kern, int grid, int block, size_t smem, cudaStream_t s, bool pdl, const Arg& arg) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3((unsigned)block); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, arg);
}

// ---- kernel launchers (defined in the k_*.cu files) ---------------------------------------------------
struct StemArgs {
    const void* x;       // [N,3,H,W] fp32 or uint8
    int is_u8;
    int N, H, W;         // input dims
    Planes out;          // 24 planes at H/4 x W/4, ids 0..23
    const float* wpack;  // STEM layout
};
int launch_stem(const StemArgs& a, cudaStream_t s);

// conv1x1 backward with an optional scratch for per-block partial weight gradients (k_train.cu; the C-ABI operator passes none)
int conv1x1_bwd_impl(const float* x, const float* w, const float* dy, float* dx, float* dw, float* dbias, int N, int K, int M, int HW,
                     float* wscratch, size_t wscratch_floats, cudaStream_t s);

}  // namespace yfv2
