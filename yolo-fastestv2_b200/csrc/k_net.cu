// The network after the stem on Hopper tensor cores: ShuffleNetV2 blocks, the LightFPN reducers and the detection heads.
// Every 1x1 convolution is a 3xTF32 mma.sync contraction (tc.cuh) whose A operand is produced in registers straight from
// its source, so no intermediate of a block or a head ever goes through global memory:
//
//   stride-1 block (shufflenetv2.py:21-30):  pw1+BN+ReLU over the band's rows plus a one-row halo -> shared memory T;
//                                            then per output pixel dw3x3+BN from T (A operand) -> pw2+BN+ReLU -> planes
//   stride-2 block:                           the same with a stride-2 depthwise, plus the projection branch
//                                            dw3x3/2+BN read from the input planes (A operand) -> pw+BN+ReLU -> planes
//   FPN reducers (fpn.py:35-43,51-58):        1x1+BN+ReLU over C3, or over cat(nearest-up(C3), C2) without building it
//   heads (fpn.py:5-24, detector.py:17-19):   dw5x5+BN+ReLU (A operand) -> pw+BN into the flat planes; then
//                                            dw5x5+BN+ReLU -> the folded [pw, BN, output conv] matrix -> NCHW head tensors
//
// A work item of a block kernel is one image band: its pw1 output (with halo) is recomputed by the neighbouring band instead
// of being exchanged.  When a whole image fits in one band, consecutive stride-1 blocks of a stage run as one launch: the CTA
// owns the image for the whole chain, so block j+1 reads what block j wrote after a CTA barrier (plain loads, no .nc path).
#include "common.cuh"
#include "tc.cuh"

namespace yfv2 {

namespace {
using namespace tc;

constexpr int kThreads = 256;                 // 8 warps, one 16-pixel row tile each at a time
constexpr int kWarps = kThreads / 32;
constexpr int kMaxChain = 7;
constexpr size_t kChainBudget = 110 * 1024;   // whole-image bands below this keep two CTAs per SM
constexpr size_t kBandBudget = 110 * 1024;

// weights of one pointwise layer in shared memory: W[K][S] | scale[NP] | shift[NP]
__host__ __device__ constexpr int pw_smem_floats(int K, int NP) { return K * w_stride(NP) + 2 * NP; }

// from the CUDA-core pack layout (Wt[K][round4(N)] | scale | shift), N real columns, zero padded to NP
__device__ void load_pw(float* dst, const float* __restrict__ src, int K, int N, int NP) {
    const int S = w_stride(NP), Np = round4(N);
    for (int i = threadIdx.x; i < K * NP; i += blockDim.x) {
        const int k = i / NP, n = i - k * NP;
        dst[k * S + n] = n < N ? __ldg(src + k * Np + n) : 0.f;
    }
    for (int n = threadIdx.x; n < NP; n += blockDim.x) {
        dst[K * S + n] = n < N ? __ldg(src + K * Np + n) : 0.f;
        dst[K * S + NP + n] = n < N ? __ldg(src + K * Np + Np + n) : 0.f;
    }
}
__device__ void load_floats(float* dst, const float* __restrict__ src, int count) {
    for (int i = threadIdx.x; i < count; i += blockDim.x) dst[i] = __ldg(src + i);
}

// The same for a square K x K layer (K % 4 == 0: the pack rows are K contiguous floats) and count % 4 == 0, by 16-byte cp.async
// when the pack is 16-byte aligned, so that every thread has all its copies in flight at once (element-wise, they cost a
// whole-image CTA tens of microseconds per block).  The caller commits the group and waits for it before its barrier.
__device__ void cp16(float* dst, const float* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ void load_pw_async(float* dst, const float* __restrict__ src, int K) {
    if ((uintptr_t)src & 15) { load_pw(dst, src, K, K, K); return; }
    const int S = w_stride(K), R4 = K / 4;
    for (int i = threadIdx.x; i < (K + 2) * R4; i += blockDim.x) {      // rows 0..K-1: W, row K: scale, row K+1: shift
        const int k = i / R4, c = 4 * (i - k * R4);
        cp16(dst + (k < K ? k * S : K * S + (k - K) * K) + c, src + k * K + c);
    }
}
__device__ void load_floats_async(float* dst, const float* __restrict__ src, int count) {
    if ((uintptr_t)src & 15) { load_floats(dst, src, count); return; }
    for (int i = 4 * threadIdx.x; i < count; i += 4 * blockDim.x) cp16(dst + i, src + i);
}

// dw3x3 + BN of one pixel, the A-operand value of a pointwise contraction of the whole-image block kernels: tp = the top-left
// tap, ld = the row stride of the plane, w = the channel's DW3 pack row.  The same operations in the same order as the stencils
// of blk_kernel (written out there, so that its code stays as measured); tests/test_stage4_gpu.py pins the two bit for bit.
__device__ __forceinline__ float dw3_bn(const float* tp, int ld, const float* w) {
    float v = 0.f;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) v = fmaf(tp[dy * ld + dx], w[dy * 3 + dx], v);
    return fmaf(v, w[9], w[10]);
}

// ---- ShuffleNetV2 blocks ------------------------------------------------------------------------------------------------
struct BlkArgs {
    Planes in, out;
    int Hi, Wi, Ho, Wo;
    int R, bands, items, nblk;
    const float* pw1[kMaxChain];
    const float* dw[kMaxChain];
    const float* pw2[kMaxChain];
    const float *dwp, *pwp;                    // stride 2: projection branch
    unsigned short tin[kMaxChain][96];
    unsigned short tout[kMaxChain][96];        // stride 2: projection branch output (channels 0..K-1 of the block)
    unsigned short tmain[96];                  // stride 2: main branch output (channels K..2K-1)
    int G;                                     // walk::blk_kernel<K, 1>: output rows per step
};

__host__ __device__ constexpr int blk_rin(int stride, int R) { return stride * (R - 1) + 3; }
__host__ constexpr size_t blk_smem_bytes(int K, int stride, int R, int Wi) {
    return ((size_t)2 * pw_smem_floats(K, K) + 12 * K + (size_t)K * blk_rin(stride, R) * (Wi + 2)) * sizeof(float);
}

template <int K, int STRIDE>
__global__ void __launch_bounds__(kThreads)
blk_kernel(const __grid_constant__ BlkArgs p) {
    pdl_trigger();
    constexpr int KS = K / 8, NT = K / 8, S = w_stride(K);
    extern __shared__ __align__(16) float smem[];
    float* sW1 = smem;
    float* sW2 = sW1 + pw_smem_floats(K, K);
    float* sD = sW2 + pw_smem_floats(K, K);               // [K][12]: w[9] | scale | shift | 0
    float* T = sD + 12 * K;                               // [K][Rin][Wt] pw1 output, zero columns 0 and Wt-1
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int Wt = p.Wi + 2;
    const Planes in = p.in, out = p.out;

    // A stride-1 block loads its weights once and the CTA walks (image, band) items; a chain owns one whole image and reloads
    // each block's weights in turn; a stride-2 block reloads its main-branch weights per item, because the projection branch
    // takes over their buffers at the end of the item.
    for (int i = threadIdx.x; i < K * blk_rin(STRIDE, p.R); i += kThreads) { T[i * Wt] = 0.f; T[i * Wt + Wt - 1] = 0.f; }
    const bool resident = STRIDE == 1 && p.nblk == 1;
    if (resident) {
        load_pw(sW1, p.pw1[0], K, K, K);
        load_pw(sW2, p.pw2[0], K, K, K);
        load_floats(sD, p.dw[0], 12 * K);
    }
    pdl_wait();
    for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
    const int n = item / p.bands, band = item - n * p.bands;
    const int y0 = band * p.R, rows = min(p.R, p.Ho - y0);
    const int Rin = blk_rin(STRIDE, rows), plT = Rin * Wt;
    const int M1 = Rin * p.Wi, M2 = rows * p.Wo;
    for (int j = 0; j < p.nblk; ++j) {
        if (!resident) {
            load_pw(sW1, p.pw1[j], K, K, K);
            load_pw(sW2, p.pw2[j], K, K, K);
            load_floats(sD, p.dw[j], 12 * K);
        }
        __syncthreads();
        // pw1 + BN + ReLU over the band's input rows (halo included); rows outside the map are the depthwise zero padding
        const unsigned short* tin = p.tin[j];
        for (int m0 = warp * 16; m0 < M1; m0 += kWarps * 16) {
            int off[2]; bool ok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi, iy = STRIDE * y0 - 1 + r;
                ok[h] = m < M1 && iy >= 0 && iy < p.Hi;
                off[h] = in.org + iy * in.Ws + c;
            }
            const float* ib = in.base + (long long)n * in.sN;
            float acc[NT][4];
            warp_gemm<KS, NT>(acc, sW1, S, [&](int ks, float (&a)[4]) {
                const long long c0 = (long long)tin[8 * ks + t] * in.sC, c1 = (long long)tin[8 * ks + t + 4] * in.sC;
                a[0] = ok[0] ? ib[c0 + off[0]] : 0.f;
                a[1] = ok[1] ? ib[c0 + off[1]] : 0.f;
                a[2] = ok[0] ? ib[c1 + off[0]] : 0.f;
                a[3] = ok[1] ? ib[c1 + off[1]] : 0.f;
            });
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h;
                if (m >= M1) continue;
                const int r = m / p.Wi, c = m - r * p.Wi;
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * nt + 2 * t + e;
                        const float v = fmaxf(fmaf(acc[nt][2 * h + e], sW1[K * S + col], sW1[K * S + K + col]), 0.f);
                        T[col * plT + r * Wt + c + 1] = ok[h] ? v : 0.f;
                    }
            }
        }
        __syncthreads();
        // dw3x3 (stride STRIDE) + BN from T as the A operand -> pw2 + BN + ReLU -> output planes
        const unsigned short* tdst = STRIDE == 2 ? p.tmain : p.tout[j];
        for (int m0 = warp * 16; m0 < M2; m0 += kWarps * 16) {
            int base[2]; bool ok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h, r = m / p.Wo, c = m - r * p.Wo;
                ok[h] = m < M2;
                base[h] = ok[h] ? STRIDE * r * Wt + STRIDE * c : 0;
            }
            float acc[NT][4];
            warp_gemm<KS, NT>(acc, sW2, S, [&](int ks, float (&a)[4]) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int k = 8 * ks + t + 4 * q;
                    const float* w = sD + 12 * k;
                    const float* tk = T + k * plT;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float* tp = tk + base[h];
                        float v = 0.f;
#pragma unroll
                        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                            for (int dx = 0; dx < 3; ++dx) v = fmaf(tp[dy * Wt + dx], w[dy * 3 + dx], v);
                        a[2 * q + h] = ok[h] ? fmaf(v, w[9], w[10]) : 0.f;
                    }
                }
            });
            float* ob = out.base + (long long)n * out.sN;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h;
                if (!ok[h]) continue;
                const int r = m / p.Wo, c = m - r * p.Wo;
                const int o = out.org + (y0 + r) * out.Ws + c;
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * nt + 2 * t + e;
                        ob[(long long)tdst[col] * out.sC + o] = fmaxf(fmaf(acc[nt][2 * h + e], sW2[K * S + col], sW2[K * S + K + col]), 0.f);
                    }
            }
        }
        __syncthreads();          // T, the weights and (in a chain) this block's output planes are consumed next
    }
    if constexpr (STRIDE == 2) {
        // projection branch: dw3x3/2 + BN straight from the input planes -> pw + BN + ReLU
        load_pw(sW1, p.pwp, K, K, K);
        load_floats(sD, p.dwp, 12 * K);
        __syncthreads();
        const unsigned short* tin = p.tin[0];
        const float* ib = in.base + (long long)n * in.sN;
        for (int m0 = warp * 16; m0 < M2; m0 += kWarps * 16) {
            int off[2]; bool ok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h, r = m / p.Wo, c = m - r * p.Wo;
                ok[h] = m < M2;
                off[h] = ok[h] ? in.org + (2 * (y0 + r) - 1) * in.Ws + 2 * c - 1 : in.org;
            }
            float acc[NT][4];
            warp_gemm<KS, NT>(acc, sW1, S, [&](int ks, float (&a)[4]) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int k = 8 * ks + t + 4 * q;
                    const float* w = sD + 12 * k;
                    const float* pk = ib + (long long)tin[k] * in.sC;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float* tp = pk + off[h];
                        float v = 0.f;
#pragma unroll
                        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                            for (int dx = 0; dx < 3; ++dx) v = fmaf(tp[dy * in.Ws + dx], w[dy * 3 + dx], v);
                        a[2 * q + h] = ok[h] ? fmaf(v, w[9], w[10]) : 0.f;
                    }
                }
            });
            float* ob = out.base + (long long)n * out.sN;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h;
                if (!ok[h]) continue;
                const int r = m / p.Wo, c = m - r * p.Wo;
                const int o = out.org + (y0 + r) * out.Ws + c;
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * nt + 2 * t + e;
                        ob[(long long)p.tout[0][col] * out.sC + o] = fmaxf(fmaf(acc[nt][2 * h + e], sW1[K * S + col], sW1[K * S + K + col]), 0.f);
                    }
            }
        }
    }
    __syncthreads();          // the next item refills T
    }
}

// ---- stride-2 block: a band walked in steps of rows ------------------------------------------------------------------------
// The K = 24 / 48 stride-2 blocks (stage2.0, stage3.0) keep the bands of blk_rows and one CTA per band, but the CTA walks its
// band G output rows at a time instead of running pw1 over the whole band first:
//   * All five weight packs are loaded at once by 16-byte cp.async, with the band's first input rows, and stay resident: the
//     projection branch does not take over the main branch's buffers.
//   * Input rows are staged whole (frame columns included) by 16-byte cp.async into a ring X of 4G + 1 rows per channel; the
//     copies of step s + 1 are issued before step s computes.  pw1 and the projection branch's dw3x3/2 both read X, not the
//     global planes.
//   * T holds the 2G + 1 pw1 rows of a step; its bottom row is carried into the next step as that step's top row.
//   * The pw2 and projection tiles of a step run in one phase over all warps.
// As in blk_kernel, the band's first step computes the pw1 row above the band, and outside the map the T row is zero.  Every
// value is computed with the same operations in the same order as blk_kernel<K, 2> (an mma.sync output row depends only on its
// own A row), so the outputs are bit-identical to it.
//
// The kernel keeps the name blk_kernel<K, 2> (in namespace walk) and the grid of one CTA per band: profiler traces and launch
// models that know the banded kernel describe it unchanged.
namespace walk {
constexpr int G = 1;              // output rows per step

__host__ __device__ constexpr int ring_rows(int G) { return 4 * G + 1; }
// channel stride of X (n floats, n % 4 == 0): the four t lanes of an A-fragment read fall on distinct banks
__host__ __device__ constexpr int ring_stride(int n) { return n % 32 == 8 || n % 32 == 24 ? n : ring_stride(n + 4); }
__host__ constexpr size_t smem_bytes(int K, int Wi, int Ws) {
    return ((size_t)3 * pw_smem_floats(K, K) + 24 * K + (size_t)K * ring_stride(ring_rows(G) * Ws) + (size_t)K * (2 * G + 1) * (Wi + 2))
           * sizeof(float);
}

// dw3x3 + BN with the three rows of the stencil at p + row[0..2]: the operations of blk_kernel's stencils, in their order
__device__ __forceinline__ float dw3_bn_rows(const float* p, const int (&row)[3], const float* w) {
    float v = 0.f;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) v = fmaf(p[row[dy] + dx], w[dy * 3 + dx], v);
    return fmaf(v, w[9], w[10]);
}

template <int K, int STRIDE>
__global__ void __launch_bounds__(kThreads, 2)
blk_kernel(const __grid_constant__ BlkArgs p) {
    static_assert(STRIDE == 2, "blk_kernel<K, 1> is specialised below");
    pdl_trigger();
    constexpr int KS = K / 8, NT = K / 8, S = w_stride(K), RX = ring_rows(G), RT = 2 * G + 1;
    extern __shared__ __align__(16) float smem[];
    float* sW1 = smem;
    float* sW2 = sW1 + pw_smem_floats(K, K);
    float* sWp = sW2 + pw_smem_floats(K, K);
    float* sD = sWp + pw_smem_floats(K, K);               // main branch dw3x3/2: [K][12]
    float* sDp = sD + 12 * K;                             // projection branch dw3x3/2
    const Planes in = p.in, out = p.out;
    const int Ws = in.Ws, CS = ring_stride(RX * Ws);
    float* X = sDp + 12 * K;                              // [K][CS]: input row iy (-1 .. Hi, frame included) at X row (iy + 1) % RX
    const int Wt = p.Wi + 2, plT = RT * Wt;
    float* T = X + K * CS;                                // [K][RT][Wt]: pw1 row of input row iy at T row (iy + 1) % RT
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const unsigned short* tin = p.tin[0];

    for (int i = threadIdx.x; i < K * RT; i += kThreads) { T[i * Wt] = 0.f; T[i * Wt + Wt - 1] = 0.f; }
    load_pw_async(sW1, p.pw1[0], K);
    load_pw_async(sW2, p.pw2[0], K);
    load_pw_async(sWp, p.pwp, K);
    load_floats_async(sD, p.dw[0], 12 * K);
    load_floats_async(sDp, p.dwp, 12 * K);
    cp_async_commit();
    pdl_wait();

    // input rows [iy0, iy0 + cnt) of image n -> X (plane row iy starts at (iy + 1) Ws: the frame is one pixel wide)
    const int C4 = Ws / 4;
    auto stage_rows = [&](int n, int iy0, int cnt) {
        const float* ib = in.base + (long long)n * in.sN + (long long)(iy0 + 1) * Ws;
        for (int i = threadIdx.x; i < K * cnt * C4; i += kThreads) {
            const int kr = i / C4, c = 4 * (i - kr * C4), k = kr / cnt, r = kr - k * cnt;
            cp16(X + k * CS + (iy0 + 1 + r) % RX * Ws + c, ib + (long long)tin[k] * in.sC + r * Ws + c);
        }
        cp_async_commit();
    };

    {
        // this CTA's band: output rows [ys, ye) of image n
        const int n = blockIdx.x / p.bands, ys = (blockIdx.x - n * p.bands) * p.R, ye = min(p.Ho, ys + p.R);
        float* ob = out.base + (long long)n * out.sN;
        stage_rows(n, 2 * ys - 1, 2 * min(G, ye - ys) + 1);
        for (int y = ys; y < ye; y += G) {
            const int rows = min(G, ye - y);
            cp_async_wait<0>();
            __syncthreads();      // this step's input rows have landed; the previous step is done with X and T
            if (y + G < ye) stage_rows(n, 2 * (y + G), 2 * min(G, ye - y - G));
            // pw1 + BN + ReLU -> T over the step's new input rows (the top halo row too in the band's first step); rows outside
            // the map are the depthwise zero padding
            const int r0 = y == ys ? 2 * y - 1 : 2 * y, M1 = (2 * y + 2 * rows - r0) * p.Wi;
            for (int m0 = warp * 16; m0 < M1; m0 += kWarps * 16) {
                int xo[2], to[2]; bool ok[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi, iy = r0 + r;
                    ok[h] = m < M1 && iy >= 0 && iy < p.Hi;
                    xo[h] = (iy + 1) % RX * Ws + c + 1;
                    to[h] = (iy + 1) % RT * Wt + c + 1;
                }
                float acc[NT][4];
                warp_gemm<KS, NT>(acc, sW1, S, [&](int ks, float (&a)[4]) {
                    const float* x0 = X + (8 * ks + t) * CS;
                    const float* x1 = x0 + 4 * CS;
                    a[0] = ok[0] ? x0[xo[0]] : 0.f;
                    a[1] = ok[1] ? x0[xo[1]] : 0.f;
                    a[2] = ok[0] ? x1[xo[0]] : 0.f;
                    a[3] = ok[1] ? x1[xo[1]] : 0.f;
                });
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (m0 + g + 8 * h >= M1) continue;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            const float v = fmaxf(fmaf(acc[nt][2 * h + e], sW1[K * S + col], sW1[K * S + K + col]), 0.f);
                            T[col * plT + to[h]] = ok[h] ? v : 0.f;
                        }
                }
            }
            __syncthreads();
            // even tiles: dw3x3/2 + BN from T -> pw2 + BN + ReLU -> planes K..2K-1 of the block;
            // odd tiles: dw3x3/2 + BN from X -> pw + BN + ReLU -> planes 0..K-1
            const int M2 = rows * p.Wo, tiles = (M2 + 15) / 16;
            for (int tile = warp; tile < 2 * tiles; tile += kWarps) {
                const bool proj = tile & 1;
                const int m0 = (tile >> 1) * 16;
                int row[2][3], oo[2]; bool ok[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wo, c = m - r * p.Wo, iy = 2 * (y + r) - 1;
                    ok[h] = m < M2;
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy)
                        row[h][dy] = ok[h] ? (proj ? (iy + 1 + dy) % RX * Ws : (iy + 1 + dy) % RT * Wt) + 2 * c : 0;
                    oo[h] = out.org + (y + r) * out.Ws + c;
                }
                const float* src = proj ? X : T;
                const int ld = proj ? CS : plT;
                const float* sw = proj ? sWp : sW2;
                const float* sd = proj ? sDp : sD;
                float acc[NT][4];
                warp_gemm<KS, NT>(acc, sw, S, [&](int ks, float (&a)[4]) {
#pragma unroll
                    for (int q = 0; q < 2; ++q) {
                        const int k = 8 * ks + t + 4 * q;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float v = dw3_bn_rows(src + k * ld, row[h], sd + 12 * k);
                            a[2 * q + h] = ok[h] ? v : 0.f;
                        }
                    }
                });
                const unsigned short* tdst = proj ? p.tout[0] : p.tmain;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!ok[h]) continue;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            ob[(long long)tdst[col] * out.sC + oo[h]] = fmaxf(fmaf(acc[nt][2 * h + e], sw[K * S + col], sw[K * S + K + col]), 0.f);
                        }
                }
            }
        }
    }
}

// ---- stride-1 block: bands walked in steps of rows by a persistent grid -----------------------------------------------------
// A single K = 24 / 48 stride-1 block (stage2.1-3, stage3.1-7) keeps the bands of blk_rows and the persistent grid of
// blk_kernel<K, 1>, and walks each band G output rows at a time (G = BlkArgs::G, chosen by the host from the map width):
//   * pw1, pw2 and the dw pack are loaded once per CTA by 16-byte cp.async, issued before pdl_wait and resident for the launch.
//   * Input rows are staged whole (frame columns included) by 16-byte cp.async into a ring X of 2G + 2 rows per channel, in the
//     order the CTA consumes them (X row j of the CTA's sequence at slot j % (2G + 2)).  The copies of step s + 1 are issued
//     before step s computes; in an item's last step they are the first rows of the CTA's next item, when both fit in the ring.
//   * A step runs pw1 + BN + ReLU over its new input rows into a ring T of G + 2 pw1 rows (the band's first step also over the
//     row above and the row below the step), a barrier, then dw3x3 + BN from T as the A operand of pw2 + BN + ReLU -> planes.
//   * Pass k of the persistent loop takes item k gridDim + blockIdx.x for even k and k gridDim + gridDim - 1 - blockIdx.x for odd
//     k, so a CTA that takes a band of an image's tall head in one pass takes a short tail band in the next.
// Every value is computed with the operations of blk_kernel<K, 1> in their order, so the outputs are bit-identical to it.
__host__ __device__ constexpr int s1_ring_rows(int G) { return 2 * G + 2; }
__host__ constexpr size_t s1_smem_bytes(int K, int G, int Wi, int Ws) {
    return ((size_t)2 * pw_smem_floats(K, K) + 12 * K + (size_t)K * ring_stride(s1_ring_rows(G) * Ws) + (size_t)K * (G + 2) * (Wi + 2))
           * sizeof(float);
}

template <int K>
__device__ __forceinline__ void blk_s1_walk(const BlkArgs& p) {
    pdl_trigger();
    constexpr int KS = K / 8, NT = K / 8, S = w_stride(K);
    extern __shared__ __align__(16) float smem[];
    float* sW1 = smem;
    float* sW2 = sW1 + pw_smem_floats(K, K);
    float* sD = sW2 + pw_smem_floats(K, K);               // [K][12]: w[9] | scale | shift | 0
    const Planes in = p.in, out = p.out;
    const int Gs = p.G, RX = s1_ring_rows(Gs), RT = Gs + 2, Ws = in.Ws, CS = ring_stride(RX * Ws);
    float* X = sD + 12 * K;                               // [K][CS]: X row j of the CTA's sequence at row j % RX
    const int Wt = p.Wi + 2, plT = RT * Wt;
    float* T = X + K * CS;                                // [K][RT][Wt]: pw1 row of input row iy at T row (iy + 1) % RT
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const unsigned short* tin = p.tin[0];
    const unsigned short* tout = p.tout[0];

    for (int i = threadIdx.x; i < K * RT; i += kThreads) { T[i * Wt] = 0.f; T[i * Wt + Wt - 1] = 0.f; }
    load_pw_async(sW1, p.pw1[0], K);
    load_pw_async(sW2, p.pw2[0], K);
    load_floats_async(sD, p.dw[0], 12 * K);
    cp_async_commit();
    pdl_wait();

    // input rows [iy0, iy0 + cnt) of image n -> X rows seq0 .. seq0 + cnt - 1 of the sequence; rows outside the map are not
    // copied (pw1 writes zeros for them).  Plane row iy starts at (iy + 1) Ws: the frame is one pixel wide.
    const int C4 = Ws / 4;
    auto stage_rows = [&](int n, int iy0, int cnt, int seq0) {
        const float* ib = in.base + (long long)n * in.sN + (long long)(iy0 + 1) * Ws;
        for (int i = threadIdx.x; i < K * cnt * C4; i += kThreads) {
            const int kr = i / C4, c = 4 * (i - kr * C4), k = kr / cnt, r = kr - k * cnt;
            if (iy0 + r >= 0 && iy0 + r < p.Hi) cp16(X + k * CS + (seq0 + r) % RX * Ws + c, ib + (long long)tin[k] * in.sC + r * Ws + c);
        }
        cp_async_commit();
    };
    auto item_of = [&](int pass) { return pass * (int)gridDim.x + (pass & 1 ? gridDim.x - 1 - blockIdx.x : blockIdx.x); };
    // the first step of band `item` reads its input rows [ys - 1, ys + rows + 1)
    auto first_rows = [&](int item, int& n, int& ys, int& ye) {
        n = item / p.bands; ys = (item - n * p.bands) * p.R; ye = min(p.Ho, ys + p.R);
        return min(Gs, ye - ys) + 2;
    };

    int sb = 0, na = 0;         // sequence index of the current step's first X row; X rows in flight for the next step (0: none)
    for (int pass = 0, item = item_of(0); item < p.items; item = item_of(++pass)) {
        int n, ys, ye;
        const int a0 = first_rows(item, n, ys, ye);
        if (na == 0) { na = a0; stage_rows(n, ys - 1, a0, sb); }      // not issued by the previous item's last step
        float* ob = out.base + (long long)n * out.sN;
        for (int y = ys; y < ye; y += Gs) {
            const int rows = min(Gs, ye - y), r0 = y == ys ? y - 1 : y + 1, a = na;    // X rows sb .. sb + a - 1: input rows r0 ..
            cp_async_wait<0>();
            __syncthreads();      // this step's input rows have landed; the previous step is done with X and T
            na = 0;
            if (y + Gs < ye) {
                na = min(Gs, ye - y - Gs);
                stage_rows(n, y + Gs + 1, na, sb + a);
            } else if (item_of(pass + 1) < p.items) {
                int n2, ys2, ye2;
                const int a2 = first_rows(item_of(pass + 1), n2, ys2, ye2);
                if (a + a2 <= RX) { na = a2; stage_rows(n2, ys2 - 1, a2, sb + a); }
            }
            // pw1 + BN + ReLU -> T over the step's input rows; rows outside the map are the depthwise zero padding
            const int M1 = a * p.Wi;
            for (int m0 = warp * 16; m0 < M1; m0 += kWarps * 16) {
                int xo[2], to[2]; bool ok[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi, iy = r0 + r;
                    ok[h] = m < M1 && iy >= 0 && iy < p.Hi;
                    xo[h] = (sb + r) % RX * Ws + c + 1;
                    to[h] = (iy + 1) % RT * Wt + c + 1;
                }
                float acc[NT][4];
                warp_gemm<KS, NT>(acc, sW1, S, [&](int ks, float (&a)[4]) {
                    const float* x0 = X + (8 * ks + t) * CS;
                    const float* x1 = x0 + 4 * CS;
                    a[0] = ok[0] ? x0[xo[0]] : 0.f;
                    a[1] = ok[1] ? x0[xo[1]] : 0.f;
                    a[2] = ok[0] ? x1[xo[0]] : 0.f;
                    a[3] = ok[1] ? x1[xo[1]] : 0.f;
                });
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (m0 + g + 8 * h >= M1) continue;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            const float v = fmaxf(fmaf(acc[nt][2 * h + e], sW1[K * S + col], sW1[K * S + K + col]), 0.f);
                            T[col * plT + to[h]] = ok[h] ? v : 0.f;
                        }
                }
            }
            __syncthreads();
            // dw3x3 + BN from T as the A operand -> pw2 + BN + ReLU -> output planes
            const int M2 = rows * p.Wo;
            for (int m0 = warp * 16; m0 < M2; m0 += kWarps * 16) {
                int row[2][3], oo[2]; bool ok[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wo, c = m - r * p.Wo;
                    ok[h] = m < M2;
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy) row[h][dy] = ok[h] ? (y + r + dy) % RT * Wt + c : 0;
                    oo[h] = out.org + (y + r) * out.Ws + c;
                }
                float acc[NT][4];
                warp_gemm<KS, NT>(acc, sW2, S, [&](int ks, float (&a)[4]) {
#pragma unroll
                    for (int q = 0; q < 2; ++q) {
                        const int k = 8 * ks + t + 4 * q;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float v = dw3_bn_rows(T + k * plT, row[h], sD + 12 * k);
                            a[2 * q + h] = ok[h] ? v : 0.f;
                        }
                    }
                });
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!ok[h]) continue;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            ob[(long long)tout[col] * out.sC + oo[h]] = fmaxf(fmaf(acc[nt][2 * h + e], sW2[K * S + col], sW2[K * S + K + col]), 0.f);
                        }
                }
            }
            sb += a;
        }
    }
}

template <>
__global__ void __launch_bounds__(kThreads, 2) blk_kernel<24, 1>(const __grid_constant__ BlkArgs p) { blk_s1_walk<24>(p); }
template <>
__global__ void __launch_bounds__(kThreads, 2) blk_kernel<48, 1>(const __grid_constant__ BlkArgs p) { blk_s1_walk<48>(p); }
}  // namespace walk

// ---- stride-2 block on whole images -------------------------------------------------------------------------------------
// When a CTA's 8 warps cover the output map with one 16-pixel tile each, the block runs per image instead of per band: all
// five weight packs stay resident across the CTA's images (persistent grid), and T holds kS2Chunk pw1 channels at a time.
// For each chunk, pw1 runs over the whole input map (no halo recompute), then the chunk's dw3x3/2 feeds the matching k-steps
// of pw2, accumulated in registers across chunks.  The k-steps run in ascending order and every value is computed as in
// blk_kernel<K, 2>, so the outputs are bit-identical to the banded kernel.
constexpr int kS2Chunk = 32;

__host__ constexpr size_t blk_s2_image_smem_bytes(int K, int Ho, int Wi) {
    return ((size_t)3 * pw_smem_floats(K, K) + 24 * K + (size_t)kS2Chunk * (2 * Ho + 1) * (Wi + 2)) * sizeof(float);
}
bool blk_s2_whole_image(int K, int Ho, int Wo, int Wi) {
    return K == 96 && Ho * Wo <= 16 * kWarps && blk_s2_image_smem_bytes(K, Ho, Wi) <= kSmemCap;
}

template <int K>
__global__ void __launch_bounds__(kThreads, 1)
blk_s2_image_kernel(const __grid_constant__ BlkArgs p) {
    pdl_trigger();
    static_assert(K % kS2Chunk == 0, "pw1 channel chunks must tile K");
    constexpr int KS = K / 8, NT = K / 8, S = w_stride(K), CT = kS2Chunk / 8;
    extern __shared__ __align__(16) float smem[];
    float* sW1 = smem;
    float* sW2 = sW1 + pw_smem_floats(K, K);
    float* sWp = sW2 + pw_smem_floats(K, K);
    float* sD = sWp + pw_smem_floats(K, K);               // main branch dw3x3/2: [K][12]
    float* sDp = sD + 12 * K;                             // projection branch dw3x3/2
    float* T = sDp + 12 * K;                              // [kS2Chunk][2 Ho + 1][Wi + 2]: T row r is input row r - 1
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int Wt = p.Wi + 2, plT = (2 * p.Ho + 1) * Wt;
    const int M1 = p.Hi * p.Wi, M2 = p.Ho * p.Wo;
    const Planes in = p.in, out = p.out;
    const unsigned short* tin = p.tin[0];

    // pw1 writes the interior of T only: row 0, rows past the input and the side columns stay zero
    for (int i = threadIdx.x; i < kS2Chunk * plT; i += kThreads) T[i] = 0.f;
    load_pw_async(sW1, p.pw1[0], K);
    load_pw_async(sW2, p.pw2[0], K);
    load_pw_async(sWp, p.pwp, K);
    load_floats_async(sD, p.dw[0], 12 * K);
    load_floats_async(sDp, p.dwp, 12 * K);
    cp_async_commit();
    cp_async_wait<0>();
    pdl_wait();
    __syncthreads();

    // this warp's output tile
    const int mo = warp * 16;
    int base[2], offp[2], oo[2]; bool ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = mo + g + 8 * h, r = m / p.Wo, c = m - r * p.Wo;
        ok[h] = m < M2;
        base[h] = ok[h] ? 2 * r * Wt + 2 * c : 0;
        offp[h] = ok[h] ? in.org + (2 * r - 1) * in.Ws + 2 * c - 1 : in.org;
        oo[h] = out.org + r * out.Ws + c;
    }
    for (int n = blockIdx.x; n < p.items; n += gridDim.x) {
        const float* ib = in.base + (long long)n * in.sN;
        float* ob = out.base + (long long)n * out.sN;
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
        for (int c0 = 0; c0 < K; c0 += kS2Chunk) {
            // pw1 + BN + ReLU, output channels [c0, c0 + kS2Chunk), over the whole input map; all A fragments of a tile are
            // loaded before its MMAs
            for (int m0 = warp * 16; m0 < M1; m0 += kWarps * 16) {
                int off[2]; bool okin[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi;
                    okin[h] = m < M1;
                    off[h] = in.org + r * in.Ws + c;
                }
                float af[KS][4];
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) {
                    const long long k0 = (long long)tin[8 * ks + t] * in.sC, k1 = (long long)tin[8 * ks + t + 4] * in.sC;
                    af[ks][0] = okin[0] ? ib[k0 + off[0]] : 0.f;
                    af[ks][1] = okin[1] ? ib[k0 + off[1]] : 0.f;
                    af[ks][2] = okin[0] ? ib[k1 + off[0]] : 0.f;
                    af[ks][3] = okin[1] ? ib[k1 + off[1]] : 0.f;
                }
                float a1[CT][4];
                warp_gemm_regs<KS, CT>(a1, sW1 + c0, S, af);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!okin[h]) continue;
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi;
#pragma unroll
                    for (int nt = 0; nt < CT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            T[col * plT + (r + 1) * Wt + c + 1] =
                                fmaxf(fmaf(a1[nt][2 * h + e], sW1[K * S + c0 + col], sW1[K * S + K + c0 + col]), 0.f);
                        }
                }
            }
            __syncthreads();
            // dw3x3/2 + BN of the chunk from T: k-steps [c0 / 8, c0 / 8 + CT) of pw2
            if (mo < M2)
                warp_gemm_acc<CT, NT>(acc, sW2 + c0 * S, S, [&](int ks, float (&a)[4]) {
#pragma unroll
                    for (int q = 0; q < 2; ++q) {
                        const int k = 8 * ks + t + 4 * q;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float v = dw3_bn(T + k * plT + base[h], Wt, sD + 12 * (c0 + k));
                            a[2 * q + h] = ok[h] ? v : 0.f;
                        }
                    }
                });
            __syncthreads();      // the next chunk overwrites T
        }
        if (mo >= M2) continue;
        auto store = [&](const float* sc, const unsigned short* tdst) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!ok[h]) continue;
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * nt + 2 * t + e;
                        ob[(long long)tdst[col] * out.sC + oo[h]] = fmaxf(fmaf(acc[nt][2 * h + e], sc[col], sc[K + col]), 0.f);
                    }
            }
        };
        // main branch: pw2 + BN + ReLU -> planes K..2K-1 of the block
        store(sW2 + K * S, p.tmain);
        // projection branch: dw3x3/2 + BN straight from the input planes -> pw + BN + ReLU -> planes 0..K-1
        warp_gemm<KS, NT>(acc, sWp, S, [&](int ks, float (&a)[4]) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int k = 8 * ks + t + 4 * q;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float v = dw3_bn(ib + (long long)tin[k] * in.sC + offp[h], in.Ws, sDp + 12 * k);
                    a[2 * q + h] = ok[h] ? v : 0.f;
                }
            }
        });
        store(sWp + K * S, p.tout[0]);
    }
}

// ---- stride-1 chains on whole images, one CTA per SM ----------------------------------------------------------------------
// A chain whose whole image fits in one SM's shared memory but not in kChainBudget (K = 96: stage4.1-3 at 352x352, 151 KB) runs
// a persistent grid of one CTA per SM.  The CTA takes all its images through block j before block j+1, so each block's weights
// are loaded once per CTA, and the loads overlap the compute: block j+1's pw1 matrix is copied into sW1 while block j runs its
// last pw2, its pw2 matrix and dw pack into sW2 / sD while block j+1 runs its first pw1.  T keeps its zero frame for the whole
// launch, so pw1 runs over the H x W pixels of the image only, not over the two halo rows outside it.  Every value is computed
// as in blk_kernel<K, 1>, so the outputs are bit-identical to running the blocks one launch each.
template <int K>
__global__ void __launch_bounds__(kThreads, 1)
blk_chain_kernel(const __grid_constant__ BlkArgs p) {
    pdl_trigger();
    constexpr int KS = K / 8, NT = K / 8, S = w_stride(K);
    extern __shared__ __align__(16) float smem[];
    float* sW1 = smem;
    float* sW2 = sW1 + pw_smem_floats(K, K);
    float* sD = sW2 + pw_smem_floats(K, K);
    float* T = sD + 12 * K;                               // [K][H + 2][W + 2]: T row r is image row r - 1
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int Wt = p.Wi + 2, plT = (p.Hi + 2) * Wt, M = p.Hi * p.Wi;
    const Planes P = p.in;

    for (int i = threadIdx.x; i < K * plT; i += kThreads) T[i] = 0.f;
    load_pw_async(sW1, p.pw1[0], K);
    cp_async_commit();
    load_pw_async(sW2, p.pw2[0], K);
    load_floats_async(sD, p.dw[0], 12 * K);
    cp_async_commit();
    pdl_wait();
    const int last = blockIdx.x + (p.items - 1 - blockIdx.x) / gridDim.x * gridDim.x;      // this CTA's last image
    for (int j = 0; j < p.nblk; ++j) {
        const unsigned short* tin = p.tin[j];
        const unsigned short* tout = p.tout[j];
        for (int n = blockIdx.x; n < p.items; n += gridDim.x) {
            float* ib = P.base + (long long)n * P.sN;
            cp_async_wait<1>();       // sW1 of block j; its sW2 / sD may still be in flight
            __syncthreads();
            // pw1 + BN + ReLU over the image's pixels
            for (int m0 = warp * 16; m0 < M; m0 += kWarps * 16) {
                int off[2]; bool ok[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi;
                    ok[h] = m < M;
                    off[h] = P.org + r * P.Ws + c;
                }
                float acc[NT][4];
                warp_gemm<KS, NT>(acc, sW1, S, [&](int ks, float (&a)[4]) {
                    const long long c0 = (long long)tin[8 * ks + t] * P.sC, c1 = (long long)tin[8 * ks + t + 4] * P.sC;
                    a[0] = ok[0] ? ib[c0 + off[0]] : 0.f;
                    a[1] = ok[1] ? ib[c0 + off[1]] : 0.f;
                    a[2] = ok[0] ? ib[c1 + off[0]] : 0.f;
                    a[3] = ok[1] ? ib[c1 + off[1]] : 0.f;
                });
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!ok[h]) continue;
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            T[col * plT + (r + 1) * Wt + c + 1] = fmaxf(fmaf(acc[nt][2 * h + e], sW1[K * S + col], sW1[K * S + K + col]), 0.f);
                        }
                }
            }
            cp_async_wait<0>();       // sW2 / sD of block j
            __syncthreads();
            if (n == last && j + 1 < p.nblk) { load_pw_async(sW1, p.pw1[j + 1], K); cp_async_commit(); }
            // dw3x3 + BN from T as the A operand -> pw2 + BN + ReLU -> the block's output planes
            for (int m0 = warp * 16; m0 < M; m0 += kWarps * 16) {
                int base[2]; bool ok[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi;
                    ok[h] = m < M;
                    base[h] = ok[h] ? r * Wt + c : 0;
                }
                float acc[NT][4];
                warp_gemm<KS, NT>(acc, sW2, S, [&](int ks, float (&a)[4]) {
#pragma unroll
                    for (int q = 0; q < 2; ++q) {
                        const int k = 8 * ks + t + 4 * q;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float v = dw3_bn(T + k * plT + base[h], Wt, sD + 12 * k);
                            a[2 * q + h] = ok[h] ? v : 0.f;
                        }
                    }
                });
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!ok[h]) continue;
                    const int m = m0 + g + 8 * h, r = m / p.Wi, c = m - r * p.Wi;
                    const int o = P.org + r * P.Ws + c;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * nt + 2 * t + e;
                            ib[(long long)tout[col] * P.sC + o] = fmaxf(fmaf(acc[nt][2 * h + e], sW2[K * S + col], sW2[K * S + K + col]), 0.f);
                        }
                }
            }
            __syncthreads();          // T, sW2 / sD and this block's output planes are consumed next
            if (n == last && j + 1 < p.nblk) {
                load_pw_async(sW2, p.pw2[j + 1], K);
                load_floats_async(sD, p.dw[j + 1], 12 * K);
                cp_async_commit();
            }
        }
    }
}

int persistent_grid(long long items, int per_sm) {
    const long long cap = (long long)per_sm * sm_count();
    return (int)(items < cap ? items : cap);
}

template <class Kern>
int smem_attr(Kern kern, size_t bytes) {
    YFV2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return YFV2_OK;
}

// rows per band: the largest band within the budget, shrunk while the grid would leave SMs idle
int blk_rows(int K, int stride, int Ho, int Wi, int N) {
    int R = Ho;
    while (R > 1 && blk_smem_bytes(K, stride, R, Wi) > kBandBudget) --R;
    while (R > 1 && (size_t)N * ((Ho + R - 1) / R) < (size_t)2 * sm_count()) R = (R + 1) / 2;
    return R;
}

template <int K, int STRIDE>
int run_blk(BlkArgs& a, int N, cudaStream_t s) {
    a.bands = (a.Ho + a.R - 1) / a.R;
    a.items = N * a.bands;
    const size_t bytes = blk_smem_bytes(K, STRIDE, a.R, a.Wi);
    if (bytes > kSmemCap) { set_error("block: a %d-row band of %d columns does not fit in shared memory", a.R, a.Wi); return YFV2_EUNSUPPORTED; }
    if (int rc = smem_attr(blk_kernel<K, STRIDE>, bytes)) return rc;
    int grid = a.items;
    // A stride-1 block keeps its weights resident in a persistent grid (K=96 at 352x352: 182 -> 120 us on an H100).  The
    // stride-2 blocks were measured slower that way (stage4.0 610 -> 760 us, stage2.0 463 -> 488 us) and take one CTA per item;
    // K = 24 and 48 run on walk::blk_kernel wherever it fits.
    if (STRIDE == 1 && a.nblk == 1) {
        int per_sm = 0;
        YFV2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, blk_kernel<K, STRIDE>, kThreads, bytes));
        grid = persistent_grid(a.items, per_sm > 0 ? per_sm : 1);
    }
    YFV2_CUDA(launch_k(blk_kernel<K, STRIDE>, grid, kThreads, bytes, s, pdl_take(), a));
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// The band walk stages whole plane rows by 16-byte copies from planes with a one-pixel frame; the plan's pool planes are such
// planes, 16-byte aligned.  Wider maps, whose ring and T rows do not fit next to the weights, keep blk_kernel<K, 2>.
bool blk_s2_walk_fits(int K, const Planes& in) {
    return (K == 24 || K == 48) && in.pad == 1 && ((uintptr_t)in.base & 15) == 0 && in.Ws % 4 == 0 && in.sC % 4 == 0 &&
           in.sN % 4 == 0 && walk::smem_bytes(K, in.W, in.Ws) <= kSmemCap;
}

// The stride-1 walk takes the largest step of at most s1_step_max(K) rows whose rings fit next to the weights within
// kS1WalkBudget (two CTAs per SM), on the same planes as the stride-2 walk; 0 where no step fits (past 158 columns at K = 24, 62
// at K = 48) and for K = 96, which keep blk_kernel<K, 1>.  The caps are the fastest steps measured at 352x352 (DESIGN.md §5):
// 4 rows at K = 24 (44 columns), 3 at K = 48 (22 columns).
constexpr size_t kS1WalkBudget = 113 * 1024;
constexpr int s1_step_max(int K) { return K == 24 ? 4 : 3; }
int blk_s1_walk_step(int K, const Planes& P) {
    if (!((K == 24 || K == 48) && P.pad == 1 && ((uintptr_t)P.base & 15) == 0 && P.Ws % 4 == 0 && P.sC % 4 == 0 && P.sN % 4 == 0))
        return 0;
    for (int G = s1_step_max(K); G >= 1; --G)
        if (walk::s1_smem_bytes(K, G, P.W, P.Ws) <= kS1WalkBudget) return G;
    return 0;
}

template <int K, int STRIDE>
int run_blk_walk(BlkArgs& a, int N, cudaStream_t s) {
    a.bands = (a.Ho + a.R - 1) / a.R;
    a.items = N * a.bands;
    auto kern = walk::blk_kernel<K, STRIDE>;
    const size_t bytes = STRIDE == 2 ? walk::smem_bytes(K, a.Wi, a.in.Ws) : walk::s1_smem_bytes(K, a.G, a.Wi, a.in.Ws);
    if (int rc = smem_attr(kern, bytes)) return rc;
    int grid = a.items;       // stride 2: one CTA per band; stride 1: the persistent grid of blk_kernel<K, 1>
    if (STRIDE == 1) {
        int per_sm = 0;
        YFV2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, bytes));
        grid = persistent_grid(a.items, per_sm > 0 ? per_sm : 1);
    }
    YFV2_CUDA(launch_k(kern, grid, kThreads, bytes, s, pdl_take(), a));
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

template <int K>
int dispatch_blk(int stride, BlkArgs& a, int N, cudaStream_t s) {
    return stride == 1 ? run_blk<K, 1>(a, N, s) : run_blk<K, 2>(a, N, s);
}

// whole-image kernels: one CTA per SM, a persistent grid over the N images
template <class Kern>
int run_whole_image(Kern kern, size_t bytes, BlkArgs& a, int N, cudaStream_t s) {
    a.R = a.Ho; a.bands = 1; a.items = N;
    if (int rc = smem_attr(kern, bytes)) return rc;
    int per_sm = 0;
    YFV2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, bytes));
    YFV2_CUDA(launch_k(kern, persistent_grid(N, per_sm > 0 ? per_sm : 1), kThreads, bytes, s, pdl_take(), a));
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// ---- FPN reducers -------------------------------------------------------------------------------------------------------
struct FpnArgs {
    Planes c3, c2, out;
    unsigned short t3[192], t2[96];
    const float* pw;
    int N, H, W, chunks;       // output map; chunks of 16 * kWarps pixels per image
};

// S3 = conv1x1_3(C3) (KIN = 192), S2 = conv1x1_2(cat(up2(C3), C2)) (KIN = 288); 72 output channels, BN + ReLU
template <int KIN>
__global__ void __launch_bounds__(kThreads)
fpn_kernel(const __grid_constant__ FpnArgs p) {
    pdl_trigger();
    constexpr int NT = 9, S = w_stride(72);
    extern __shared__ __align__(16) float smem[];
    load_pw(smem, p.pw, KIN, 72, 72);
    pdl_wait();
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int HW = p.H * p.W;
    for (int item = blockIdx.x; item < p.N * p.chunks; item += gridDim.x) {
        const int n = item / p.chunks, m0 = (item - n * p.chunks) * 16 * kWarps + 16 * warp;
        if (m0 >= HW) continue;
        int o3[2], o2[2], oo[2]; bool ok[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + g + 8 * h, y = m / p.W, x = m - y * p.W;
            ok[h] = m < HW;
            const int yy = ok[h] ? y : 0, xx = ok[h] ? x : 0;
            o3[h] = KIN == 192 ? p.c3.org + yy * p.c3.Ws + xx : p.c3.org + (yy >> 1) * p.c3.Ws + (xx >> 1);
            o2[h] = p.c2.org + yy * p.c2.Ws + xx;
            oo[h] = p.out.org + yy * p.out.Ws + xx;
        }
        const float* b3 = p.c3.base + (long long)n * p.c3.sN;
        const float* b2 = p.c2.base + (long long)n * p.c2.sN;
        float acc[NT][4];
        warp_gemm<KIN / 8, NT>(acc, smem, S, [&](int ks, float (&a)[4]) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int k = 8 * ks + t + 4 * q;
                const float* pl = k < 192 ? b3 + (long long)p.t3[k] * p.c3.sC : b2 + (long long)p.t2[k - 192] * p.c2.sC;
#pragma unroll
                for (int h = 0; h < 2; ++h) a[2 * q + h] = pl[k < 192 ? o3[h] : o2[h]];
            }
        });
        float* ob = p.out.base + (long long)n * p.out.sN;
        const float* sc = smem + KIN * S;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (!ok[h]) continue;
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * nt + 2 * t + e;
                    ob[(long long)col * p.out.sC + oo[h]] = fmaxf(fmaf(acc[nt][2 * h + e], sc[col], sc[72 + col]), 0.f);
                }
        }
    }
}

// ---- heads ----------------------------------------------------------------------------------------------------------------
struct HeadArgs {
    Planes in[2], out[2];          // branch 0 = cls head, 1 = reg head (flat planes, zero frame of 2)
    const float* dw[2];            // DW5 packs
    const float* pw[2];            // half 0: PW pack 72 -> 72; half 1: folded [NPt][72] matrix | bias[NPt], NPt = 96 or 192
    float* dst[2][2];              // half 1: branch 0 -> obj rows [0, A), cls rows [A, A + C); branch 1 -> reg rows [0, 4A)
    int split[2], rowsA[2], rowsB[2];
    int N, H, W, chunks;
    int CS;                        // staged path: channel stride of a window slot (floats); 0: the stencils read the planes
};

constexpr int kHeadTile = 96;      // output columns of one contraction of the second head half (12 n-tiles of 8)
constexpr int kHeadSlots = 3;      // window slots of 8 channels (one k-step) in flight
constexpr size_t kHeadBudget = 113 * 1024;     // two CTAs per SM (the cls and reg CTA of one blockIdx.x)

// The staged path copies, per (item, k-step), the input rows [y0 - 2, y1 + 2] of the item's pixel rows [y0, y1] for 8 channels:
// at most win rows of Ws floats per channel.  A run of 16 kWarps consecutive pixels spans at most this many map rows.
__host__ __device__ constexpr int head_win_rows(int H, int W) {
    return ((W - 1 + 16 * kWarps - 1) / W + 1 < H ? (W - 1 + 16 * kWarps - 1) / W + 1 : H) + 4;
}
__host__ constexpr size_t head_weight_bytes(int NP) { return ((size_t)pw_smem_floats(72, NP) + 72 * 28) * sizeof(float); }

// half 0: dw5x5 + BN + ReLU -> pw + BN -> flat planes.  half 1: dw5x5 + BN + ReLU -> folded matrix + bias -> head tensors.
// HALF 2 (head2_kernel) is half 1 for A + C > 96: the cls branch contracts the same A fragments, kept in registers, against two
// 96-column tiles of a [192][72] folded matrix; the reg branch (4A <= 32 columns) keeps one tile.  It contracts 48 columns at a
// time, so that the A fragments (36 registers) and one pass of accumulators (24) leave room for two CTAs per SM.
//
// The dw5x5 taps come from a window staged in shared memory where it fits (p.CS > 0, heads_launch): per k-step, the item's rows
// with their 2-row halo for the k-step's 8 channels, whole framed rows by 16-byte cp.async into a ring of kHeadSlots slots.  The
// copies of k-step j + 2 of the CTA's sequence (which runs on into its next item) are issued after the barrier of k-step j, when
// every warp is done with the slot they overwrite; so every warp takes part in every k-step, pixels or not.  A slot keeps the
// plane's row stride, and its channel stride is 8 or 24 modulo 32 words: the 4 t x 8 g lanes of a tap read hit 32 banks when the
// fragment row's 8 pixels lie in one map row.  Where they straddle two map rows the offsets of the g lanes jump by Ws - W + 1
// and t lanes can share a bank (1.25 wavefronts per tap read on average at 22x22, 1.56 at 11x11, 1.0 at 40x40).
// Elsewhere the taps are read from the planes.  Both compute every value with the same operations in the same order.
__device__ __forceinline__ float dw5_bn_relu(const float* tp, int ld, const float* w) {
    float v = 0.f;
#pragma unroll
    for (int dy = 0; dy < 5; ++dy)
#pragma unroll
        for (int dx = 0; dx < 5; ++dx) v = fmaf(tp[dy * ld + dx], w[dy * 5 + dx], v);
    return fmaxf(fmaf(v, w[25], w[26]), 0.f);
}

template <int HALF>
__device__ __forceinline__ void head_body(const HeadArgs& p) {
    pdl_trigger();
    constexpr int NP = HALF == 0 ? 72 : HALF == 1 ? kHeadTile : 2 * kHeadTile;   // weight columns in shared memory
    constexpr int NT = HALF == 0 ? 9 : HALF == 1 ? kHeadTile / 8 : kHeadTile / 16, S = w_stride(NP);   // n-tiles of one pass
    extern __shared__ __align__(16) float smem[];
    float* sW = smem;
    float* sD = sW + pw_smem_floats(72, NP);      // [72][28]: w[25] | scale | shift | 0
    float* X = sD + 72 * 28;                      // staged path: [kHeadSlots][8][CS]
    const int br = blockIdx.y;
    const int tiles = HALF == 2 && br == 0 ? 2 : 1;
    if (HALF == 0) {
        load_pw(sW, p.pw[br], 72, 72, 72);
    } else {
        const float* F = p.pw[br];
        const int NF = HALF == 2 ? kHeadTile * tiles : NP;   // rows of this branch's folded matrix; columns past NF stay unread
        for (int i = threadIdx.x; i < 72 * NF; i += kThreads) {
            const int k = i / NF, nn = i - k * NF;
            sW[k * S + nn] = __ldg(F + nn * 72 + k);
        }
        for (int nn = threadIdx.x; nn < NF; nn += kThreads) { sW[72 * S + nn] = 1.f; sW[72 * S + NP + nn] = __ldg(F + NF * 72 + nn); }
    }
    load_floats(sD, p.dw[br], 72 * 28);
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int HW = p.H * p.W, items = p.N * p.chunks, CS = p.CS;
    const Planes& in = p.in[br];
    // first pixel row of an item's chunk, and the floats per channel of its window
    auto chunk_rows = [&](int chunk, int& y0, int& len) {
        const int m = chunk * 16 * kWarps;
        y0 = m / p.W;
        len = ((min(HW, m + 16 * kWarps) - 1) / p.W - y0 + 5) * in.Ws;
    };
    // k-step j of this CTA's sequence (k-step j % 9 of its item j / 9) -> slot j % kHeadSlots; warp c copies channel c
    auto stage = [&](int j) {
        const int item = blockIdx.x + j / 9 * gridDim.x;
        if (item < items) {
            const int n = item / p.chunks;
            int y0, len;
            chunk_rows(item - n * p.chunks, y0, len);
            const float* src = in.base + (long long)n * in.sN + (long long)(8 * (j % 9) + warp) * in.sC + (long long)y0 * in.Ws;
            float* dst = X + (j % kHeadSlots * 8 + warp) * CS;
            for (int o = 4 * lane; o < len; o += 128) cp16(dst + o, src + o);
        }
        cp_async_commit();
    };
    if (CS) {
        for (int j = 0; j < kHeadSlots - 1; ++j) stage(j);
    }
    __syncthreads();
    for (int item = blockIdx.x, j0 = 0; item < items; item += gridDim.x, j0 += 9) {
        const int n = item / p.chunks, chunk = item - n * p.chunks, m0 = chunk * 16 * kWarps + 16 * warp;
        if (!CS && m0 >= HW) continue;
        int y0, len;
        chunk_rows(chunk, y0, len);
        int off[2]; bool ok[2];           // top-left tap in the window (staged) or in the plane
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + g + 8 * h, y = m / p.W, x = m - y * p.W;
            ok[h] = m < HW;
            off[h] = CS ? (ok[h] ? (y - y0) * in.Ws + x : 0) : ok[h] ? in.org + (y - 2) * in.Ws + x - 2 : in.org;
        }
        auto load_staged = [&](int ks, float (&a)[4]) {
            cp_async_wait<kHeadSlots - 2>();
            __syncthreads();          // k-step j0 + ks has landed; every warp is done with the slot k-step j0 + ks + 2 fills
            stage(j0 + ks + kHeadSlots - 1);
            const float* slot = X + (j0 + ks) % kHeadSlots * 8 * CS;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const float* w = sD + 28 * (8 * ks + t + 4 * q);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float v = dw5_bn_relu(slot + (t + 4 * q) * CS + off[h], in.Ws, w);
                    a[2 * q + h] = ok[h] ? v : 0.f;
                }
            }
        };
        const float* ib = in.base + (long long)n * in.sN;
        auto load_planes = [&](int ks, float (&a)[4]) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int k = 8 * ks + t + 4 * q;
                const float* w = sD + 28 * k;
                const float* pk = ib + (long long)k * in.sC;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float v = dw5_bn_relu(pk + off[h], in.Ws, w);
                    a[2 * q + h] = ok[h] ? v : 0.f;
                }
            }
        };
        // columns [c0, c0 + 8 NT) of the scaled result -> flat planes (half 0) or head tensors (half 1)
        auto store = [&](const float (&acc)[NT][4], int c0) {
            const float* sc = sW + 72 * S;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!ok[h]) continue;
                const int m = m0 + g + 8 * h;
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = c0 + 8 * nt + 2 * t + e;
                        const float v = fmaf(acc[nt][2 * h + e], sc[col], sc[NP + col]);
                        if (HALF == 0) {
                            const Planes& o = p.out[br];
                            const int y = m / p.W, x = m - y * p.W;
                            o.base[(long long)n * o.sN + (long long)col * o.sC + o.org + y * o.Ws + x] = v;
                        } else if (col < p.split[br]) {
                            p.dst[br][0][((long long)n * p.rowsA[br] + col) * HW + m] = v;
                        } else if (col < p.split[br] + p.rowsB[br]) {
                            p.dst[br][1][((long long)n * p.rowsB[br] + col - p.split[br]) * HW + m] = v;
                        }
                    }
            }
        };
        // one contraction per path, so that each keeps only its own operands in registers
        auto contract = [&](auto&& load_a) {
            if constexpr (HALF < 2) {
                float acc[NT][4];
                warp_gemm<9, NT>(acc, sW, S, load_a);
                store(acc, 0);
            } else {
                // The dw5x5 stencil (1800 FMAs per pixel) is computed once; each 96-column tile costs 324 MMAs per warp on it.
                float af[9][4];
#pragma unroll
                for (int ks = 0; ks < 9; ++ks) load_a(ks, af[ks]);
#pragma unroll 1
                for (int c0 = 0; c0 < kHeadTile * tiles; c0 += 8 * NT) {
                    float acc[NT][4];
                    warp_gemm_regs<9, NT>(acc, sW + c0, S, af);
                    store(acc, c0);
                }
            }
        };
        if (CS) contract(load_staged);
        else contract(load_planes);
    }
}

// Two CTAs per SM: 128 registers (half 1: 8 bytes of spill).  Left unbounded, ptxas gives the staged-window build 142 and 146.
template <int HALF>
__global__ void __launch_bounds__(kThreads, 2)
head_kernel(const __grid_constant__ HeadArgs p) { head_body<HALF>(p); }

// Two CTAs per SM: 128 registers with 16 bytes of spill.  Left unbounded (before the staged window), ptxas gave it 144 registers
// and one CTA per SM, which measured slower on an H100 (150 classes, batch 256 @352x352: heads2.b 430 us against 363-379 us).
__global__ void __launch_bounds__(kThreads, 2)
head2_kernel(const __grid_constant__ HeadArgs p) { head_body<2>(p); }

// ---- test hook: out[n][p] = sum_k w[n][k] x[k][p] -------------------------------------------------------------------------
template <int K, int NP>
__global__ void __launch_bounds__(kThreads)
pw_test_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ out, int N, int P) {
    constexpr int S = w_stride(NP);
    extern __shared__ __align__(16) float smem[];
    for (int i = threadIdx.x; i < K * NP; i += kThreads) {
        const int k = i / NP, nn = i - k * NP;
        smem[k * S + nn] = nn < N ? w[nn * K + k] : 0.f;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int m0 = (blockIdx.x * kWarps + warp) * 16;
    if (m0 >= P) return;
    float acc[NP / 8][4];
    warp_gemm<K / 8, NP / 8>(acc, smem, S, [&](int ks, float (&a)[4]) {
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + g + 8 * h;
                a[2 * q + h] = m < P ? x[(size_t)(8 * ks + t + 4 * q) * P + m] : 0.f;
            }
    });
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + g + 8 * h;
        if (m >= P) continue;
#pragma unroll
        for (int nt = 0; nt < NP / 8; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = 8 * nt + 2 * t + e;
                if (col < N) out[(size_t)col * P + m] = acc[nt][2 * h + e];
            }
    }
}

template <int K, int NP>
int run_pw_test(const float* x, const float* w, float* out, int N, int P, cudaStream_t s) {
    const size_t bytes = (size_t)K * w_stride(NP) * sizeof(float);
    if (int rc = smem_attr(pw_test_kernel<K, NP>, bytes)) return rc;
    pw_test_kernel<K, NP><<<(P + 16 * kWarps - 1) / (16 * kWarps), kThreads, bytes, s>>>(x, w, out, N, P);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

}  // namespace

// A chain needs a whole image per CTA: within kChainBudget (two CTAs per SM) blk_kernel runs it; K = 96 chains up to one SM's
// shared memory run on blk_chain_kernel (stage4.1-3 at 352x352, where three launches of 2-row bands recompute most of pw1 as halo).
bool blk_s1_chainable(int K, int H, int W) {
    const size_t bytes = blk_smem_bytes(K, 1, H, W);
    return bytes <= kChainBudget || (K == 96 && bytes <= kSmemCap);
}

int blk_launch_s1(int K, const Planes& P, int nblk, const ChanTab* tin, const ChanTab* tout, const float* const* w1,
                  const float* const* wdw, const float* const* w2, int N, cudaStream_t s) {
    if (nblk < 1 || nblk > kMaxChain || (nblk > 1 && !blk_s1_chainable(K, P.H, P.W))) {
        set_error("block: a chain of %d stride-1 blocks needs a whole %dx%d image per CTA", nblk, P.H, P.W);
        return YFV2_EINVAL;
    }
    BlkArgs a{};
    a.in = P; a.out = P;
    a.Hi = a.Ho = P.H; a.Wi = a.Wo = P.W;
    a.nblk = nblk;
    a.R = nblk > 1 ? P.H : blk_rows(K, 1, P.H, P.W, N);
    for (int j = 0; j < nblk; ++j) {
        a.pw1[j] = w1[j]; a.dw[j] = wdw[j]; a.pw2[j] = w2[j];
        for (int i = 0; i < K; ++i) { a.tin[j][i] = tin[j].c[i]; a.tout[j][i] = tout[j].c[i]; }
    }
    const size_t bytes = blk_smem_bytes(K, 1, P.H, P.W);
    if (nblk > 1 && bytes > kChainBudget) return run_whole_image(blk_chain_kernel<96>, bytes, a, N, s);   // K = 96 (chainable)
    if (nblk == 1 && (a.G = blk_s1_walk_step(K, P)) > 0) return K == 24 ? run_blk_walk<24, 1>(a, N, s) : run_blk_walk<48, 1>(a, N, s);
    switch (K) {
    case 24: return dispatch_blk<24>(1, a, N, s);
    case 48: return dispatch_blk<48>(1, a, N, s);
    case 96: return dispatch_blk<96>(1, a, N, s);
    }
    set_error("block: unsupported width %d", K);
    return YFV2_EUNSUPPORTED;
}

int blk_launch_s2(int K, const Planes& in, const Planes& out, const ChanTab& tin, const ChanTab& tout, const float* wdwp, const float* wp,
                  const float* w1, const float* wdwm, const float* w2, int N, cudaStream_t s) {
    BlkArgs a{};
    a.in = in; a.out = out;
    a.Hi = in.H; a.Wi = in.W; a.Ho = out.H; a.Wo = out.W;
    a.nblk = 1;
    a.pw1[0] = w1; a.dw[0] = wdwm; a.pw2[0] = w2; a.dwp = wdwp; a.pwp = wp;
    for (int i = 0; i < K; ++i) { a.tin[0][i] = tin.c[i]; a.tout[0][i] = tout.c[i]; a.tmain[i] = tout.c[K + i]; }
    if (blk_s2_whole_image(K, out.H, out.W, in.W))      // K = 96
        return run_whole_image(blk_s2_image_kernel<96>, blk_s2_image_smem_bytes(K, out.H, in.W), a, N, s);
    a.R = blk_rows(K, 2, out.H, in.W, N);
    if (blk_s2_walk_fits(K, in)) return K == 24 ? run_blk_walk<24, 2>(a, N, s) : run_blk_walk<48, 2>(a, N, s);
    switch (K) {
    case 24: return dispatch_blk<24>(2, a, N, s);
    case 48: return dispatch_blk<48>(2, a, N, s);
    case 96: return dispatch_blk<96>(2, a, N, s);
    }
    set_error("block: unsupported width %d", K);
    return YFV2_EUNSUPPORTED;
}

// which = 1: S3 from C3; which = 2: S2 from cat(up2(C3), C2)
int fpn_launch(int which, const Planes& c3, const ChanTab& t3, const Planes& c2, const ChanTab& t2, const Planes& out, const float* pw,
               int N, cudaStream_t s) {
    FpnArgs a{};
    a.c3 = c3; a.c2 = c2; a.out = out; a.pw = pw;
    for (int i = 0; i < 192; ++i) a.t3[i] = t3.c[i];
    for (int i = 0; i < 96; ++i) a.t2[i] = t2.c[i];
    a.N = N; a.H = out.H; a.W = out.W;
    a.chunks = (out.H * out.W + 16 * kWarps - 1) / (16 * kWarps);
    auto run = [&](auto kern, int kin) -> int {
        const size_t bytes = (size_t)pw_smem_floats(kin, 72) * sizeof(float);
        if (int rc = smem_attr(kern, bytes)) return rc;
        YFV2_CUDA(launch_k(kern, persistent_grid((long long)N * a.chunks, 2), kThreads, bytes, s, pdl_take(), a));
        YFV2_LAUNCH_CHECK();
        return YFV2_OK;
    };
    return which == 1 ? run(fpn_kernel<192>, 192) : run(fpn_kernel<288>, 288);
}

// weight columns of the kernel that runs head half `half`: 72 (head_kernel<0>), 96 (head_kernel<1>), 192 (head2_kernel); 0: none
int head_columns(int half, int A, int C) {
    if (half == 0) return 72;
    if (A + C <= kHeadTile) return kHeadTile;
    if (A + C <= 2 * kHeadTile && 4 * A <= kHeadTile) return 2 * kHeadTile;
    return 0;
}

// The channel stride of a window slot where the staged window fits, else 0 (the stencils read the planes).  It fits when the planes
// of both branches allow 16-byte copies of whole rows and kHeadSlots slots fit next to the weights within kHeadBudget.  Tall maps
// of one or two columns (a chunk spans up to 16 kWarps rows) and very wide maps (one slot of 6 rows exceeds the budget) do not.
int heads_window_stride(int half, const Planes& sIn, const Planes& tcls, const Planes& treg, int A, int C) {
    const int np = head_columns(half, A, C);
    const Planes* in[2] = {half ? &tcls : &sIn, half ? &treg : &sIn};
    for (const Planes* q : in)
        if (q->pad != 2 || ((uintptr_t)q->base & 15) || q->Ws % 4 || q->sC % 4 || q->sN % 4 || q->Ws != in[0]->Ws) return 0;
    const int cs = walk::ring_stride(head_win_rows(in[0]->H, in[0]->W) * in[0]->Ws);
    return np && head_weight_bytes(np) + (size_t)kHeadSlots * 8 * cs * sizeof(float) <= kHeadBudget ? cs : 0;
}

int heads_launch(int half, const Planes& sIn, const Planes& tcls, const Planes& treg, const float* const wdw[2], const float* const wpw[2],
                 float* reg, float* obj, float* cls, int A, int C, int N, cudaStream_t s) {
    HeadArgs a{};
    a.CS = heads_window_stride(half, sIn, tcls, treg, A, C);
    for (int b = 0; b < 2; ++b) { a.dw[b] = wdw[b]; a.pw[b] = wpw[b]; }
    a.out[0] = tcls; a.out[1] = treg;
    if (half == 0) { a.in[0] = sIn; a.in[1] = sIn; }
    else { a.in[0] = tcls; a.in[1] = treg; }
    a.dst[0][0] = obj; a.dst[0][1] = cls; a.split[0] = A; a.rowsA[0] = A; a.rowsB[0] = C;
    a.dst[1][0] = reg; a.dst[1][1] = reg; a.split[1] = 4 * A; a.rowsA[1] = 4 * A; a.rowsB[1] = 0;
    a.N = N; a.H = sIn.H; a.W = sIn.W;
    a.chunks = (sIn.H * sIn.W + 16 * kWarps - 1) / (16 * kWarps);
    auto run = [&](auto kern, int np) -> int {
        const size_t bytes = head_weight_bytes(np) + (size_t)kHeadSlots * 8 * a.CS * sizeof(float);
        if (int rc = smem_attr(kern, bytes)) return rc;
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)persistent_grid((long long)N * a.chunks, 1), 2);
        cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = bytes; cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = pdl_take() ? 1 : 0;
        YFV2_CUDA(cudaLaunchKernelEx(&cfg, kern, a));
        YFV2_LAUNCH_CHECK();
        return YFV2_OK;
    };
    switch (head_columns(half, A, C)) {
    case 72: return run(head_kernel<0>, 72);
    case kHeadTile: return run(head_kernel<1>, kHeadTile);
    case 2 * kHeadTile: return run(head2_kernel, 2 * kHeadTile);
    }
    set_error("heads: anchors+classes = %d exceeds two %d-column output tiles", A + C, kHeadTile);
    return YFV2_EUNSUPPORTED;
}
static_assert(head_weight_bytes(2 * kHeadTile) <= kSmemCap, "two head tiles must fit in shared memory");

}  // namespace yfv2

using namespace yfv2;

extern "C" int yfv2_debug_pw_tc(const float* x, const float* w, float* out, float* pack_ws, int K, int N, int P, void* stream) {
    (void)pack_ws;
    if (!x || !w || !out || P <= 0) { set_error("debug_pw_tc: bad argument"); return YFV2_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    if (K == 24 && N == 24) return run_pw_test<24, 24>(x, w, out, N, P, s);
    if (K == 48 && N == 48) return run_pw_test<48, 48>(x, w, out, N, P, s);
    if (K == 96 && N == 96) return run_pw_test<96, 96>(x, w, out, N, P, s);
    if (K == 72 && N == 72) return run_pw_test<72, 72>(x, w, out, N, P, s);
    if (K == 72 && N == 83) return run_pw_test<72, 88>(x, w, out, N, P, s);
    set_error("debug_pw_tc: unsupported K=%d N=%d", K, N);
    return YFV2_EUNSUPPORTED;
}
