// Training-side operators (SURVEY 8 row a13): train-mode forward (batch-statistics BatchNorm) and the backward of every
// op of the network, as plain dense-NCHW fp32 kernels behind the C ABI.  The Python mirror composes them with
// torch.autograd.Function objects (yolo-fastestv2_b200/model/train_ops.py), so autograd's graph does the bookkeeping and
// the arithmetic is ours.  Round-1 goal here is correctness against the reference's autograd (tests/test_train_gpu.py);
// these are straightforward FFMA kernels, not yet the fused tensor-core path of the inference engine.
//
//   conv1x1   fwd / dgrad / wgrad (+bias)      one generic strided batched GEMM (64x64x16 tiles, 4x4 micro-tiles)
//   dwconv    fwd / dgrad / wgrad              3x3 or 5x5, stride 1 or 2, pad k/2      (shufflenetv2.py:25,36; fpn.py:12,19)
//   stem conv fwd / wgrad                      dense 3x3 s2 p1, 3->24                   (shufflenetv2.py:75)
//   batchnorm train fwd / bwd (+ReLU)          batch statistics, running-stat update    (nn.BatchNorm2d, momentum .1, eps 1e-5)
//   maxpool 3x3 s2 p1 fwd / bwd, nearest 2x upsample fwd / bwd                           (shufflenetv2.py:80; fpn.py:57)
#include <cstdlib>

#include "common.cuh"

namespace yfv2 {
namespace {

// ---------------------------------------------------------------------------------------------------------------------
// Generic batched GEMM with arbitrary strides:  C[b](i,j) (+)= sum_k A[b](i,k) * B[b](k,j)
// ---------------------------------------------------------------------------------------------------------------------
struct GemmArgs {
    const float* A; const float* B; float* C;
    int M, N, K, batch;
    long long sAi, sAk, sAb, sBk, sBj, sBb, sCi, sCj, sCb;
    const float* bias;      // per-row (i) bias added once (only when !atomic), may be null
    int atomic;             // atomicAdd into C (reduction over the batch dimension with sCb == 0)
};

__global__ void __launch_bounds__(256)
gemm_kernel(GemmArgs g) {
    __shared__ float As[16][64 + 4];
    __shared__ float Bs[16][64 + 4];
    const int b = blockIdx.z;
    const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
    const float* A = g.A + b * g.sAb;
    const float* B = g.B + b * g.sBb;
    float* C = g.C + b * g.sCb;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    for (int k0 = 0; k0 < g.K; k0 += 16) {
        for (int t = threadIdx.x; t < 16 * 64; t += 256) {
            const int kk = t >> 6, ii = t & 63;
            const int k = k0 + kk;
            As[kk][ii] = (k < g.K && i0 + ii < g.M) ? A[(long long)(i0 + ii) * g.sAi + (long long)k * g.sAk] : 0.f;
            Bs[kk][ii] = (k < g.K && j0 + ii < g.N) ? B[(long long)k * g.sBk + (long long)(j0 + ii) * g.sBj] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) {
            float a[4], bb[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) { a[q] = As[kk][ty * 4 + q]; bb[q] = Bs[kk][tx * 4 + q]; }
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[q][r] = fmaf(a[q], bb[r], acc[q][r]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int i = i0 + ty * 4 + q;
        if (i >= g.M) continue;
        const float bv = (g.bias && !g.atomic) ? g.bias[i] : 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int j = j0 + tx * 4 + r;
            if (j >= g.N) continue;
            float* dst = C + (long long)i * g.sCi + (long long)j * g.sCj;
            if (g.atomic) atomicAdd(dst, acc[q][r]);
            else *dst = acc[q][r] + bv;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// conv1x1 forward / dgrad: C[b](i, j) = sum_k A(i, k) B[b](k, j) with j = pixel (contiguous in B and C), A the weight matrix
// (shared by the batch; k- or i-contiguous).  torch.profiler on the round-1 generic kernel above: 153 launches, 7.8 ms of a
// 22.6 ms batch-64 step (4.5 TFLOP/s): scalar loads with 64-bit index math per element, 4x4 micro-tiles, and a 64-row tile
// for 24-row outputs.  Here: BM x 128 tiles (BM = 32 for the 24-channel layers, 64 otherwise), 16-deep k slabs, float4 loads of the
// pixel-contiguous operand, TM x 4 micro-tiles (TM = BM / 8), next slab prefetched into registers while the current one is
// multiplied.
// ---------------------------------------------------------------------------------------------------------------------
struct Gemm2Args {
    const float* A; const float* B; float* C;
    int M, N, K, batch;
    long long sAi, sAk;              // A(i, k) = A[i * sAi + k * sAk]
    long long sBk, sBb, sCi, sCb;    // B[b](k, j) = B[b * sBb + k * sBk + j];  C[b](i, j) = C[b * sCb + i * sCi + j]
    const float* bias;               // per-row bias or null
};

template <int BM>
__global__ void __launch_bounds__(256)
gemm2_kernel(Gemm2Args g) {
    constexpr int BN = 128, BK = 16, TM = BM / 8;
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int b = blockIdx.z;
    const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
    const float* B = g.B + (long long)b * g.sBb;
    float* C = g.C + (long long)b * g.sCb;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // thread -> rows [ty*TM, +TM), cols [tx*4, +4)
    const bool vecB = ((g.N & 3) == 0) && ((g.sBk & 3) == 0) && ((g.sBb & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.B) & 15) == 0);
    const bool vecC = ((g.N & 3) == 0) && ((g.sCi & 3) == 0) && ((g.sCb & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.C) & 15) == 0);
    // loader roles: A slab = BM x 16 floats (BM*16/256 per thread), B slab = 16 x 128 floats (8 per thread: two float4)
    constexpr int APT = BM * BK / 256;
    float ra[APT];
    float4 rb[2];
    auto load_slab = [&](int k0) {
#pragma unroll
        for (int q = 0; q < APT; ++q) {
            const int e = threadIdx.x + q * 256;
            const int ii = e % BM, kk = e / BM;                      // consecutive threads: consecutive i
            const int i = i0 + ii, k = k0 + kk;
            ra[q] = (i < g.M && k < g.K) ? __ldg(g.A + (long long)i * g.sAi + (long long)k * g.sAk) : 0.f;
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int kk = (threadIdx.x >> 5) + 8 * q, j = j0 + tx * 4;
            const int k = k0 + kk;
            const float* src = B + (long long)k * g.sBk + j;
            if (k < g.K && vecB && j + 3 < g.N) rb[q] = __ldg(reinterpret_cast<const float4*>(src));
            else {
                rb[q].x = (k < g.K && j + 0 < g.N) ? __ldg(src + 0) : 0.f;
                rb[q].y = (k < g.K && j + 1 < g.N) ? __ldg(src + 1) : 0.f;
                rb[q].z = (k < g.K && j + 2 < g.N) ? __ldg(src + 2) : 0.f;
                rb[q].w = (k < g.K && j + 3 < g.N) ? __ldg(src + 3) : 0.f;
            }
        }
    };
    auto store_slab = [&]() {
#pragma unroll
        for (int q = 0; q < APT; ++q) {
            const int e = threadIdx.x + q * 256;
            As[e / BM][e % BM] = ra[q];
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) *reinterpret_cast<float4*>(&Bs[(threadIdx.x >> 5) + 8 * q][tx * 4]) = rb[q];
    };
    float acc[TM][4];
#pragma unroll
    for (int a = 0; a < TM; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    load_slab(0);
    for (int k0 = 0; k0 < g.K; k0 += BK) {
        store_slab();
        __syncthreads();
        if (k0 + BK < g.K) load_slab(k0 + BK);                        // in flight during the multiply
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[TM];
#pragma unroll
            for (int q = 0; q < TM; q += 4) {
                const float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + q]);
                a[q] = v.x; a[q + 1] = v.y; a[q + 2] = v.z; a[q + 3] = v.w;
            }
            const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
#pragma unroll
            for (int q = 0; q < TM; ++q) {
                acc[q][0] = fmaf(a[q], bv.x, acc[q][0]); acc[q][1] = fmaf(a[q], bv.y, acc[q][1]);
                acc[q][2] = fmaf(a[q], bv.z, acc[q][2]); acc[q][3] = fmaf(a[q], bv.w, acc[q][3]);
            }
        }
        __syncthreads();
    }
    const int j = j0 + tx * 4;
#pragma unroll
    for (int q = 0; q < TM; ++q) {
        const int i = i0 + ty * TM + q;
        if (i >= g.M) continue;
        const float bv = g.bias ? __ldg(g.bias + i) : 0.f;
        float* dst = C + (long long)i * g.sCi + j;
        if (vecC && j + 3 < g.N) *reinterpret_cast<float4*>(dst) = make_float4(acc[q][0] + bv, acc[q][1] + bv, acc[q][2] + bv, acc[q][3] + bv);
        else {
#pragma unroll
            for (int r = 0; r < 4; ++r) if (j + r < g.N) dst[r] = acc[q][r] + bv;
        }
    }
}

int run_gemm2(const Gemm2Args& g, cudaStream_t s) {
    if (g.M <= 32) {
        dim3 grid((g.N + 127) / 128, (g.M + 31) / 32, g.batch);
        gemm2_kernel<32><<<grid, 256, 0, s>>>(g);
    } else {
        dim3 grid((g.N + 127) / 128, (g.M + 63) / 64, g.batch);
        gemm2_kernel<64><<<grid, 256, 0, s>>>(g);
    }
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// conv1x1 wgrad: dW[m][k] = sum_{n,p} dY[n][m][p] X[n][k][p].  Output at most a few hundred x a few hundred, contraction over all
// N*HW pixels: a block owns a (64 x 64) output tile and one slice of the pixels (both operands pixel-contiguous: float4 loads,
// transposed into shared memory), 4 x 4 micro-tiles, and adds its partial tile with atomics (dW is zeroed first).
// ---------------------------------------------------------------------------------------------------------------------
// BT = 64: 16 x 16 threads, every thread all 32 pixels of a slab.  BT = 32 (the 24-channel layers): 8 x 8 threads per pixel
// quarter, four quarters of the slab side by side (a 64-wide tile would idle 6/7 of its FMAs on a 24 x 24 output).
template <int BT>
__global__ void __launch_bounds__(256)
wgrad1x1_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dw, int N, int M, int K, int HW, int pchunk,
                float* __restrict__ partial) {
    constexpr int BK = 32, TPT = BT / 4, SUBS = 256 / (TPT * TPT), KPS = BK / SUBS;      // threads per tile side, pixel sub-groups
    __shared__ float As[BK][BT + 1];
    __shared__ float Bs[BK][BT + 1];
    const int m0 = blockIdx.y * BT, k0 = blockIdx.x * BT;
    const int chunks_per_img = (HW + pchunk - 1) / pchunk;
    const int n = blockIdx.z / chunks_per_img, p_begin = (blockIdx.z % chunks_per_img) * pchunk;
    const int p_end = min(HW, p_begin + pchunk);
    const float* A = dy + (long long)n * M * HW;
    const float* B = x + (long long)n * K * HW;
    const int sub = threadIdx.x / (TPT * TPT), tt = threadIdx.x % (TPT * TPT);
    const int tx = tt % TPT, ty = tt / TPT;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    constexpr int EPT = BT * BK / 256;                      // elements of each operand per thread and slab
    for (int p0 = p_begin; p0 < p_end; p0 += BK) {
        {
            const int r = threadIdx.x / (BK / EPT), pp = (threadIdx.x % (BK / EPT)) * EPT;      // row, first of EPT consecutive pixels
#pragma unroll
            for (int q = 0; q < EPT; ++q) {
                const int p = p0 + pp + q;
                As[pp + q][r] = (m0 + r < M && p < p_end) ? __ldg(A + (long long)(m0 + r) * HW + p) : 0.f;
                Bs[pp + q][r] = (k0 + r < K && p < p_end) ? __ldg(B + (long long)(k0 + r) * HW + p) : 0.f;
            }
        }
        __syncthreads();
#pragma unroll
        for (int kq = 0; kq < KPS; ++kq) {
            const int kk = sub * KPS + kq;
            float a[4], bb[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) { a[q] = As[kk][ty * 4 + q]; bb[q] = Bs[kk][tx * 4 + q]; }
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[q][r] = fmaf(a[q], bb[r], acc[q][r]);
        }
        __syncthreads();
    }
    // partial != null: this block's tile goes to its own slice partial[blockIdx.z][M][K] with plain stores (wgrad_reduce_kernel sums
    // the slices: no atomics, deterministic); otherwise atomicAdd into the zeroed dw
    float* dst = partial ? partial + (long long)blockIdx.z * M * K : dw;
    if (SUBS > 1) {                                          // fold the pixel sub-groups inside the block first
        __shared__ float red[SUBS > 1 ? SUBS - 1 : 1][BT][BT + 1];
        if (sub > 0) {
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int r = 0; r < 4; ++r) red[sub - 1][ty * 4 + q][tx * 4 + r] = acc[q][r];
        }
        __syncthreads();
        if (sub > 0) return;
#pragma unroll
        for (int u = 0; u < SUBS - 1; ++u)
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[q][r] += red[u][ty * 4 + q][tx * 4 + r];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int m = m0 + ty * 4 + q;
        if (m >= M) continue;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int k = k0 + tx * 4 + r;
            if (k < K) { if (partial) dst[(long long)m * K + k] = acc[q][r]; else atomicAdd(dst + (long long)m * K + k, acc[q][r]); }
        }
    }
}

// dw[i] = sum over the nb block slices of partial[b][i]
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ partial, int nb, int MK, float* __restrict__ dw) {
    __shared__ float red[4][64];
    const int i = blockIdx.x * 64 + (threadIdx.x & 63), q = threadIdx.x >> 6;
    float v = 0.f;
    if (i < MK) for (int b = q; b < nb; b += 4) v += partial[(long long)b * MK + i];
    red[q][threadIdx.x & 63] = v;
    __syncthreads();
    if (q == 0 && i < MK) dw[i] = (red[0][threadIdx.x] + red[1][threadIdx.x]) + (red[2][threadIdx.x] + red[3][threadIdx.x]);
}

// conv1x1 wgrad for the narrowest layers (K = 24 input channels, M a multiple of 24): no shared memory, no barriers.
// lane = pixel, a warp owns three output rows (channels m0..m0+2) and keeps 3 x KK partial sums per lane: per pixel 3 + KK
// coalesced loads feed 3 KK FMAs; one butterfly reduction and 3 KK atomics per warp at the end of the block's pixel slice.
// (torch.profiler: the tiled kernel above spent 170 us per 24x24 layer at 352x352 / batch 64 -- two barriers per 32 pixels for a
// 24 x 24 output; the operands are 95 MB, 15 us of HBM time.)
template <int KK, int RPW>
__global__ void __launch_bounds__(24 / RPW * 32)
wgrad_rows_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dw, int N, int M, int HW, int pchunk,
                  float* __restrict__ partial) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * 24 + warp * RPW;             // 24 rows per block (24 / RPW warps), blockIdx.y walks the 24-row groups
    const int chunks_per_img = (HW + pchunk - 1) / pchunk;
    const int n = blockIdx.x / chunks_per_img, p_begin = (blockIdx.x % chunks_per_img) * pchunk;
    const int p_end = min(HW, p_begin + pchunk);
    const float* dyp = dy + ((long long)n * M + m0) * HW;
    const float* xp = x + (long long)n * KK * HW;
    float acc[RPW][KK];
#pragma unroll
    for (int q = 0; q < RPW; ++q)
#pragma unroll
        for (int k = 0; k < KK; ++k) acc[q][k] = 0.f;
    for (int p = p_begin + lane; p < p_end; p += 32) {
        float d[RPW];
#pragma unroll
        for (int q = 0; q < RPW; ++q) d[q] = __ldg(dyp + (long long)q * HW + p);
#pragma unroll
        for (int k = 0; k < KK; ++k) {
            const float v = __ldg(xp + (long long)k * HW + p);
#pragma unroll
            for (int q = 0; q < RPW; ++q) acc[q][k] = fmaf(d[q], v, acc[q][k]);
        }
    }
    float* dst = partial ? partial + (long long)blockIdx.x * M * KK : dw;
#pragma unroll
    for (int q = 0; q < RPW; ++q)
#pragma unroll
        for (int k = 0; k < KK; ++k) {
            float v = acc[q][k];
#pragma unroll
            for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == ((q * KK + k) & 31)) {               // spread the writers over the lanes
                if (partial) dst[(long long)(m0 + q) * KK + k] = v; else atomicAdd(dst + (long long)(m0 + q) * KK + k, v);
            }
        }
}

int run_gemm(const GemmArgs& g, cudaStream_t s) {
    dim3 grid((g.N + 63) / 64, (g.M + 63) / 64, g.batch);
    gemm_kernel<<<grid, 256, 0, s>>>(g);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// per-row sums of dy [N,M,HW] -> dbias[M]
__global__ void bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ db, int N, int M, int HW) {
    const int m = blockIdx.x;
    double acc = 0.0;
    for (long long t = threadIdx.x; t < (long long)N * HW; t += blockDim.x) {
        const int n = (int)(t / HW), p = (int)(t - (long long)n * HW);
        acc += dy[((long long)n * M + m) * HW + p];
    }
    __shared__ double red[256];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) { if (threadIdx.x < st) red[threadIdx.x] += red[threadIdx.x + st]; __syncthreads(); }
    if (threadIdx.x == 0) db[m] = (float)red[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// depthwise conv, kernel KS (3/5), stride S, pad KS/2, dense NCHW
// ---------------------------------------------------------------------------------------------------------------------
template <int KS>
__global__ void dw_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int N, int C, int H, int W,
                              int Ho, int Wo, int S) {
    const long long total = (long long)N * C * Ho * Wo;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), c = (int)((i / ((long long)Wo * Ho)) % C);
        const long long n = i / ((long long)Wo * Ho * C);
        const float* xp = x + (n * C + c) * (long long)H * W;
        const float* wp = w + c * KS * KS;
        float acc = 0.f;
#pragma unroll
        for (int ky = 0; ky < KS; ++ky) {
            const int iy = oy * S - KS / 2 + ky;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int kx = 0; kx < KS; ++kx) {
                const int ix = ox * S - KS / 2 + kx;
                if (ix >= 0 && ix < W) acc = fmaf(wp[ky * KS + kx], xp[iy * W + ix], acc);
            }
        }
        y[i] = acc;
    }
}

template <int KS>
__global__ void dw_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, int N, int C, int H, int W,
                                int Ho, int Wo, int S) {
    const long long total = (long long)N * C * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), c = (int)((i / ((long long)W * H)) % C);
        const long long n = i / ((long long)W * H * C);
        const float* dp = dy + (n * C + c) * (long long)Ho * Wo;
        const float* wp = w + c * KS * KS;
        float acc = 0.f;
#pragma unroll
        for (int ky = 0; ky < KS; ++ky) {
            const int t = iy + KS / 2 - ky;            // oy*S = t
            if (t < 0 || t % S) continue;
            const int oy = t / S;
            if (oy >= Ho) continue;
#pragma unroll
            for (int kx = 0; kx < KS; ++kx) {
                const int u = ix + KS / 2 - kx;
                if (u < 0 || u % S) continue;
                const int ox = u / S;
                if (ox < Wo) acc = fmaf(wp[ky * KS + kx], dp[oy * Wo + ox], acc);
            }
        }
        dx[i] = acc;
    }
}

// one CTA per (channel, slice of the batch): KS*KS partial sums per thread, block reduce, atomicAdd into dw
template <int KS>
__global__ void __launch_bounds__(256)
dw_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw, int N, int C, int H, int W, int Ho, int Wo,
                int S) {
    const int c = blockIdx.x;
    float acc[KS * KS];
#pragma unroll
    for (int t = 0; t < KS * KS; ++t) acc[t] = 0.f;
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const float* xp = x + ((long long)n * C + c) * H * W;
        const float* dp = dy + ((long long)n * C + c) * Ho * Wo;
        for (int p = threadIdx.x; p < Ho * Wo; p += 256) {
            const int oy = p / Wo, ox = p - oy * Wo;
            const float d = dp[p];
#pragma unroll
            for (int ky = 0; ky < KS; ++ky) {
                const int iy = oy * S - KS / 2 + ky;
                if (iy < 0 || iy >= H) continue;
#pragma unroll
                for (int kx = 0; kx < KS; ++kx) {
                    const int ix = ox * S - KS / 2 + kx;
                    if (ix >= 0 && ix < W) acc[ky * KS + kx] = fmaf(d, xp[iy * W + ix], acc[ky * KS + kx]);
                }
            }
        }
    }
    __shared__ float red[8][KS * KS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int t = 0; t < KS * KS; ++t) {
        float v = acc[t];
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < KS * KS) {
        float v = 0.f;
        for (int wi = 0; wi < 8; ++wi) v += red[wi][threadIdx.x];
        atomicAdd(dw + c * KS * KS + threadIdx.x, v);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// stem: dense conv 3x3 s2 p1, Cin=3 -> M
// ---------------------------------------------------------------------------------------------------------------------
// thread = one output position, all M (<= 24) channels: the 27 input values are loaded once and reused M times, the weights come
// from shared memory as warp-uniform float4 reads (the round-1 kernel ran one thread per output ELEMENT: 27 loads per FMA chain,
// 0.94 ms per batch-64 launch)
template <int MM>
__global__ void __launch_bounds__(256)
stem_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int N, int H, int W) {
    __shared__ __align__(16) float sw[27][MM];                 // [tap = (c, ky, kx)][m]
    for (int i = threadIdx.x; i < 27 * MM; i += 256) { const int m = i / 27, t = i - m * 27; sw[t][m] = __ldg(w + i); }
    __syncthreads();
    const int Ho = H / 2, Wo = W / 2;
    const long long total = (long long)N * Ho * Wo;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho);
        const long long n = i / ((long long)Wo * Ho);
        float acc[MM];
#pragma unroll
        for (int m = 0; m < MM; ++m) acc[m] = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = 2 * oy - 1 + ky;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = 2 * ox - 1 + kx;
                    const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
                    const float v = ok ? __ldg(x + ((n * 3 + c) * H + (ok ? iy : 0)) * W + (ok ? ix : 0)) : 0.f;
                    const float* wr = sw[(c * 3 + ky) * 3 + kx];
#pragma unroll
                    for (int m = 0; m < MM; m += 4) {
                        const float4 w4 = *reinterpret_cast<const float4*>(wr + m);
                        acc[m] = fmaf(w4.x, v, acc[m]); acc[m + 1] = fmaf(w4.y, v, acc[m + 1]);
                        acc[m + 2] = fmaf(w4.z, v, acc[m + 2]); acc[m + 3] = fmaf(w4.w, v, acc[m + 3]);
                    }
                }
            }
        float* yp = y + (n * MM) * (long long)Ho * Wo + (long long)oy * Wo + ox;
#pragma unroll
        for (int m = 0; m < MM; ++m) yp[(long long)m * Ho * Wo] = acc[m];
    }
}
// generic fallback (any M): one thread per output element
__global__ void stem_fwd_generic_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int N, int M, int H, int W) {
    const int Ho = H / 2, Wo = W / 2;
    const long long total = (long long)N * M * Ho * Wo;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), m = (int)((i / ((long long)Wo * Ho)) % M);
        const long long n = i / ((long long)Wo * Ho * M);
        float acc = 0.f;
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = 2 * oy - 1 + ky;
                if (iy < 0 || iy >= H) continue;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = 2 * ox - 1 + kx;
                    if (ix >= 0 && ix < W) acc = fmaf(w[((m * 3 + c) * 3 + ky) * 3 + kx], x[((n * 3 + c) * H + iy) * W + ix], acc);
                }
            }
        y[i] = acc;
    }
}

// grid (M / 4 channel groups, slices): a thread keeps 4 x 27 partial sums over its positions (the 27 input values of a position are
// loaded once per group of four channels instead of once per channel), block reduce, atomicAdd
__global__ void __launch_bounds__(256)
stem_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw, int N, int M, int H, int W) {
    const int Ho = H / 2, Wo = W / 2;
    const int m0 = blockIdx.x * 4;
    float acc[4][27];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int t = 0; t < 27; ++t) acc[q][t] = 0.f;
    const long long total = (long long)N * Ho * Wo;
    for (long long qi = (long long)blockIdx.y * 256 + threadIdx.x; qi < total; qi += (long long)gridDim.y * 256) {
        const int ox = (int)(qi % Wo), oy = (int)((qi / Wo) % Ho);
        const long long n = qi / ((long long)Wo * Ho);
        float d[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) d[q] = m0 + q < M ? __ldg(dy + ((n * M + m0 + q) * Ho + oy) * Wo + ox) : 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = 2 * oy - 1 + ky;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = 2 * ox - 1 + kx;
                    const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
                    const float v = ok ? __ldg(x + ((n * 3 + c) * H + (ok ? iy : 0)) * W + (ok ? ix : 0)) : 0.f;
#pragma unroll
                    for (int q = 0; q < 4; ++q) acc[q][(c * 3 + ky) * 3 + kx] = fmaf(d[q], v, acc[q][(c * 3 + ky) * 3 + kx]);
                }
            }
    }
    __shared__ float red[8][4 * 27];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int t = 0; t < 27; ++t) {
            float v = acc[q][t];
#pragma unroll
            for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) red[warp][q * 27 + t] = v;
        }
    __syncthreads();
    if (threadIdx.x < 4 * 27) {
        float v = 0.f;
        for (int wi = 0; wi < 8; ++wi) v += red[wi][threadIdx.x];
        const int q = threadIdx.x / 27, t = threadIdx.x - q * 27;
        if (m0 + q < M) atomicAdd(dw + (m0 + q) * 27 + t, v);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// BatchNorm (training mode)
// ---------------------------------------------------------------------------------------------------------------------
// stats[c] = (sum, sumsq) in fp64; grid (C, slices): a block walks whole (n, c) planes (no per-element index division), images
// n = blockIdx.y, blockIdx.y + gridDim.y, ...
__global__ void __launch_bounds__(256)
bn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int N, int C, int HW) {
    const int c = blockIdx.x;
    double s1 = 0.0, s2 = 0.0;
    const bool vec = (HW & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const float* xp = x + ((long long)n * C + c) * HW;
        if (vec) {
            for (int p = threadIdx.x * 4; p < HW; p += 1024) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(xp + p));
                s1 += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
                s2 += ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w);
            }
        } else {
            for (int p = threadIdx.x; p < HW; p += 256) { const float v = __ldg(xp + p); s1 += v; s2 += (double)v * v; }
        }
    }
    __shared__ double r1[256], r2[256];
    r1[threadIdx.x] = s1; r2[threadIdx.x] = s2;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if (threadIdx.x < st) { r1[threadIdx.x] += r1[threadIdx.x + st]; r2[threadIdx.x] += r2[threadIdx.x + st]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { atomicAdd(stats + 2 * c, r1[0]); atomicAdd(stats + 2 * c + 1, r2[0]); }
}

// mean / invstd from the sums; running-stat update as nn.BatchNorm2d: momentum 0.1, unbiased variance
__global__ void bn_finalize_kernel(const double* __restrict__ stats, float* __restrict__ mean, float* __restrict__ invstd,
                                   float* __restrict__ running_mean, float* __restrict__ running_var, int C, double count, float momentum) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const double m = stats[2 * c] / count;
    double var = stats[2 * c + 1] / count - m * m;
    if (var < 0.0) var = 0.0;
    mean[c] = (float)m;
    invstd[c] = (float)(1.0 / sqrt(var + (double)kBnEps));
    if (running_mean) {
        const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
    }
}

// grid (N*C planes, chunks of 1024 pixels): the channel is a block constant, four pixels per thread
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ invstd,
                const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y, int C, int HW, int relu) {
    const long long pl = blockIdx.x;
    const int c = (int)(pl % C);
    const float a = __ldg(invstd + c) * __ldg(gamma + c), mu = __ldg(mean + c), be = __ldg(beta + c), is = __ldg(invstd + c), ga = __ldg(gamma + c);
    (void)a;
    const float* xp = x + pl * HW;
    float* yp = y + pl * HW;
    const int p0 = blockIdx.y * 1024 + threadIdx.x * 4;
    // ReLU as torch's threshold (r <= 0 ? 0 : r): a NaN passes through, where fmaxf(NaN, 0) would return 0
    auto f = [&](float v) { float r = (v - mu) * is * ga + be; return relu ? (r <= 0.f ? 0.f : r) : r; };      // same association as before
    if ((HW & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
        if (p0 < HW) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(xp + p0));
            *reinterpret_cast<float4*>(yp + p0) = make_float4(f(v.x), f(v.y), f(v.z), f(v.w));
        }
    } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) if (p0 + q < HW) yp[p0 + q] = f(__ldg(xp + p0 + q));
    }
}

// sums[c] = (sum dy, sum dy*xhat) with the ReLU mask applied (dy zeroed where y <= 0, as threshold_backward: a NaN y passes dy);
// grid (C, slices), whole planes per block
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy, const float* __restrict__ mean,
                     const float* __restrict__ invstd, double* __restrict__ sums, int N, int C, int HW, int relu) {
    const int c = blockIdx.x;
    double s1 = 0.0, s2 = 0.0;
    const float mu = mean[c], is = invstd[c];
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const long long base = ((long long)n * C + c) * HW;
        for (int p = threadIdx.x; p < HW; p += 256) {
            float d = __ldg(dy + base + p);
            if (relu && __ldg(y + base + p) <= 0.f) d = 0.f;
            s1 += d; s2 += (double)d * ((__ldg(x + base + p) - mu) * is);
        }
    }
    __shared__ double r1[256], r2[256];
    r1[threadIdx.x] = s1; r2[threadIdx.x] = s2;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if (threadIdx.x < st) { r1[threadIdx.x] += r1[threadIdx.x + st]; r2[threadIdx.x] += r2[threadIdx.x + st]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { atomicAdd(sums + 2 * c, r1[0]); atomicAdd(sums + 2 * c + 1, r2[0]); }
}

// dx = gamma*invstd/m * (m*dy - sum(dy) - xhat*sum(dy*xhat));  dgamma = sum(dy*xhat), dbeta = sum(dy).  grid (N*C planes, chunks)
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                    const double* __restrict__ sums, float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                    int C, int HW, double count, int relu) {
    const long long pl = blockIdx.x;
    const int c = (int)(pl % C);
    const float mu = __ldg(mean + c), is = __ldg(invstd + c), ga = __ldg(gamma + c);
    const float sd = (float)(sums[2 * c] / count), sdx = (float)(sums[2 * c + 1] / count);
    const long long base = pl * HW;
    const int p0 = blockIdx.y * 1024 + threadIdx.x * 4;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int p = p0 + q;
        if (p < HW) {
            float d = __ldg(dy + base + p);
            if (relu && __ldg(y + base + p) <= 0.f) d = 0.f;
            const float xh = (__ldg(x + base + p) - mu) * is;
            dx[base + p] = ga * is * (d - sd - xh * sdx);
        }
    }
    if (pl < C && blockIdx.y == 0 && threadIdx.x == 0) {      // planes 0..C-1 are image 0's channels: one writer per channel
        dgamma[c] = (float)sums[2 * c + 1];
        dbeta[c] = (float)sums[2 * c];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// maxpool 3x3 s2 p1 (with argmax) and nearest 2x upsample
// ---------------------------------------------------------------------------------------------------------------------
__global__ void maxpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int* __restrict__ idx, long long planes, int H, int W) {
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long total = planes * Ho * Wo;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho);
        const long long pl = i / ((long long)Wo * Ho);
        const float* xp = x + pl * H * W;
        float best = -INFINITY; int bi = -1;
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = 2 * oy - 1 + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = 2 * ox - 1 + kx;
                if (ix < 0 || ix >= W) continue;
                const float v = xp[iy * W + ix];
                // ATen's max_pool2d rule: the first maximum, but a NaN always wins (so the last NaN of the window is kept)
                if (v > best || isnan(v) || bi < 0) { best = v; bi = iy * W + ix; }
            }
        }
        y[i] = best; idx[i] = bi;
    }
}
__global__ void maxpool_bwd_kernel(const float* __restrict__ dy, const int* __restrict__ idx, float* __restrict__ dx, long long planes, int H, int W) {
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long total = planes * Ho * Wo;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long pl = i / ((long long)Wo * Ho);
        atomicAdd(dx + pl * H * W + idx[i], dy[i]);
    }
}
__global__ void upsample2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long planes, int H, int W) {
    const long long total = planes * 4 * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(i % (2 * W)), oy = (int)((i / (2 * W)) % (2 * H));
        const long long pl = i / ((long long)4 * H * W);
        y[i] = x[pl * H * W + (oy >> 1) * W + (ox >> 1)];
    }
}
__global__ void upsample2_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, long long planes, int H, int W) {
    const long long total = planes * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x0 = (int)(i % W), y0 = (int)((i / W) % H);
        const long long pl = i / ((long long)H * W);
        const float* d = dy + pl * 4 * H * W + (2 * y0) * (2 * W) + 2 * x0;
        dx[i] = (d[0] + d[1]) + (d[2 * W] + d[2 * W + 1]);
    }
}

int grid_for(long long total) { long long b = (total + 255) / 256; return (int)(b < 1 ? 1 : (b > 148 * 32 ? 148 * 32 : b)); }

}  // namespace
}  // namespace yfv2

using namespace yfv2;

#define ARGCHK(cond, msg) do { if (!(cond)) { set_error("%s", msg); return YFV2_EINVAL; } } while (0)

// y[n][m][p] = sum_k w[m][k] x[n][k][p] (+ bias[m])
extern "C" YFV2_API int yfv2_op_conv1x1_fwd(const float* x, const float* w, const float* bias, float* y, int N, int K, int M, int HW, void* stream) {
    ARGCHK(x && w && y && N > 0 && K > 0 && M > 0 && HW > 0, "conv1x1_fwd: bad arguments");
    static const bool old_gemm = getenv("YFV2_TRAIN_GEMM_OLD") != nullptr;      // round-1 generic kernel, kept for A/B runs
    if (old_gemm) {
        GemmArgs g{w, x, y, M, HW, K, N, K, 1, 0, HW, 1, (long long)K * HW, HW, 1, (long long)M * HW, bias, 0};
        return run_gemm(g, (cudaStream_t)stream);
    }
    Gemm2Args g{w, x, y, M, HW, K, N, K, 1, HW, (long long)K * HW, HW, (long long)M * HW, bias};
    return run_gemm2(g, (cudaStream_t)stream);
}
// dx[n][k][p] = sum_m w[m][k] dy[n][m][p];  dw[m][k] = sum_{n,p} dy[n][m][p] x[n][k][p];  dbias[m] = sum dy
// wscratch (optional, wscratch_floats long): per-block partial weight gradients, summed by a second kernel instead of fp32 atomics
// into dw (torch.profiler: ~150 k same-address-line atomics per 24x24 layer cost 160 us where the arithmetic needs 20).
namespace yfv2 {
int conv1x1_bwd_impl(const float* x, const float* w, const float* dy, float* dx, float* dw, float* dbias, int N, int K, int M, int HW,
                     float* wscratch, size_t wscratch_floats, cudaStream_t s) {
    if (!(x && w && dy && N > 0 && K > 0 && M > 0 && HW > 0)) { set_error("conv1x1_bwd: bad arguments"); return YFV2_EINVAL; }
    static const bool old_gemm = getenv("YFV2_TRAIN_GEMM_OLD") != nullptr;
    static const bool tiled_only = getenv("YFV2_TRAIN_WGRAD_TILED") != nullptr;
    if (dx) {
        int rc;
        if (old_gemm) {
            GemmArgs g{w, dy, dx, K, HW, M, N, 1, K, 0, HW, 1, (long long)M * HW, HW, 1, (long long)K * HW, nullptr, 0};
            rc = run_gemm(g, s);
        } else {
            Gemm2Args g{w, dy, dx, K, HW, M, N, 1, K, HW, (long long)M * HW, HW, (long long)K * HW, nullptr};      // A(i=k, kk=m) = w[m][k]
            rc = run_gemm2(g, s);
        }
        if (rc) return rc;
    }
    if (dw) {
        if (old_gemm) {
            YFV2_CUDA(cudaMemsetAsync(dw, 0, (size_t)M * K * sizeof(float), s));
            GemmArgs g{dy, x, dw, M, K, HW, N, HW, 1, (long long)M * HW, 1, HW, (long long)K * HW, K, 1, 0, nullptr, 1};
            int rc = run_gemm(g, s);
            if (rc) return rc;
        } else if (K == 24 && M % 24 == 0 && !tiled_only) {      // (K = 48: 50 loads per 96 FMAs per lane measured 250 us per layer; the tiled kernel wins)
            // pixel slices sized so that the grid has about two waves whatever the map size
            int pchunk = 2048;
            while (pchunk > 256 && (long long)N * (M / 24) * ((HW + pchunk - 1) / pchunk) < 2LL * sm_count()) pchunk >>= 1;
            const int chunks = (HW + pchunk - 1) / pchunk;
            const dim3 grid((unsigned)(N * chunks), (unsigned)(M / 24));
            float* part = (wscratch && (size_t)N * chunks * M * K <= wscratch_floats) ? wscratch : nullptr;
            if (!part) YFV2_CUDA(cudaMemsetAsync(dw, 0, (size_t)M * K * sizeof(float), s));
            wgrad_rows_kernel<24, 3><<<grid, 256, 0, s>>>(dy, x, dw, N, M, HW, pchunk, part);
            YFV2_LAUNCH_CHECK();
            if (part) { wgrad_reduce_kernel<<<(M * K + 63) / 64, 256, 0, s>>>(part, N * chunks, M * K, dw); YFV2_LAUNCH_CHECK(); }
        } else {
            const int BT = (M <= 32 && K <= 32) ? 32 : 64;
            const int tiles = ((M + BT - 1) / BT) * ((K + BT - 1) / BT);
            int pchunk = 1024;
            while (pchunk > 64 && (long long)tiles * N * ((HW + pchunk - 1) / pchunk) < 4LL * sm_count()) pchunk >>= 1;
            const int chunks = (HW + pchunk - 1) / pchunk;
            const dim3 grid((K + BT - 1) / BT, (M + BT - 1) / BT, N * chunks);
            float* part = (wscratch && (size_t)N * chunks * M * K <= wscratch_floats) ? wscratch : nullptr;
            if (!part) YFV2_CUDA(cudaMemsetAsync(dw, 0, (size_t)M * K * sizeof(float), s));
            if (BT == 32) wgrad1x1_kernel<32><<<grid, 256, 0, s>>>(dy, x, dw, N, M, K, HW, pchunk, part);
            else wgrad1x1_kernel<64><<<grid, 256, 0, s>>>(dy, x, dw, N, M, K, HW, pchunk, part);
            YFV2_LAUNCH_CHECK();
            if (part) { wgrad_reduce_kernel<<<(M * K + 63) / 64, 256, 0, s>>>(part, N * chunks, M * K, dw); YFV2_LAUNCH_CHECK(); }
        }
    }
    if (dbias) {
        bias_grad_kernel<<<M, 256, 0, s>>>(dy, dbias, N, M, HW);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}
}  // namespace yfv2
extern "C" YFV2_API int yfv2_op_conv1x1_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, float* dbias, int N, int K, int M,
                                            int HW, void* stream) {
    return yfv2::conv1x1_bwd_impl(x, w, dy, dx, dw, dbias, N, K, M, HW, nullptr, 0, (cudaStream_t)stream);
}

extern "C" YFV2_API int yfv2_op_dwconv_fwd(const float* x, const float* w, float* y, int N, int C, int H, int W, int ks, int stride, void* stream) {
    ARGCHK(x && w && y && (ks == 3 || ks == 5) && (stride == 1 || stride == 2), "dwconv_fwd: bad arguments");
    const int Ho = (H + 2 * (ks / 2) - ks) / stride + 1, Wo = (W + 2 * (ks / 2) - ks) / stride + 1;
    const long long total = (long long)N * C * Ho * Wo;
    if (ks == 3) dw_fwd_kernel<3><<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(x, w, y, N, C, H, W, Ho, Wo, stride);
    else dw_fwd_kernel<5><<<grid_for(total), 256, 0, (cudaStream_t)stream>>>(x, w, y, N, C, H, W, Ho, Wo, stride);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
extern "C" YFV2_API int yfv2_op_dwconv_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, int N, int C, int H, int W, int ks,
                                           int stride, void* stream) {
    ARGCHK(x && w && dy && (ks == 3 || ks == 5) && (stride == 1 || stride == 2), "dwconv_bwd: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const int Ho = (H + 2 * (ks / 2) - ks) / stride + 1, Wo = (W + 2 * (ks / 2) - ks) / stride + 1;
    if (dx) {
        const long long total = (long long)N * C * H * W;
        if (ks == 3) dw_dgrad_kernel<3><<<grid_for(total), 256, 0, s>>>(dy, w, dx, N, C, H, W, Ho, Wo, stride);
        else dw_dgrad_kernel<5><<<grid_for(total), 256, 0, s>>>(dy, w, dx, N, C, H, W, Ho, Wo, stride);
        YFV2_LAUNCH_CHECK();
    }
    if (dw) {
        YFV2_CUDA(cudaMemsetAsync(dw, 0, (size_t)C * ks * ks * sizeof(float), s));
        dim3 grid(C, N < 16 ? N : 16);
        if (ks == 3) dw_wgrad_kernel<3><<<grid, 256, 0, s>>>(x, dy, dw, N, C, H, W, Ho, Wo, stride);
        else dw_wgrad_kernel<5><<<grid, 256, 0, s>>>(x, dy, dw, N, C, H, W, Ho, Wo, stride);
        YFV2_LAUNCH_CHECK();
    }
    return YFV2_OK;
}

extern "C" YFV2_API int yfv2_op_stem_fwd(const float* x, const float* w, float* y, int N, int M, int H, int W, void* stream) {
    ARGCHK(x && w && y && H % 2 == 0 && W % 2 == 0, "stem_fwd: bad arguments");
    if (M == 24) stem_fwd_kernel<24><<<grid_for((long long)N * (H / 2) * (W / 2)), 256, 0, (cudaStream_t)stream>>>(x, w, y, N, H, W);
    else stem_fwd_generic_kernel<<<grid_for((long long)N * M * (H / 2) * (W / 2)), 256, 0, (cudaStream_t)stream>>>(x, w, y, N, M, H, W);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
extern "C" YFV2_API int yfv2_op_stem_wgrad(const float* x, const float* dy, float* dw, int N, int M, int H, int W, void* stream) {
    ARGCHK(x && dy && dw, "stem_wgrad: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemsetAsync(dw, 0, (size_t)M * 27 * sizeof(float), s));
    stem_wgrad_kernel<<<dim3((M + 3) / 4, 128), 256, 0, s>>>(x, dy, dw, N, M, H, W);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

// scratch: 2*C doubles.  save_mean / save_invstd: [C] each.  running_* may be null (no update).
extern "C" YFV2_API int yfv2_op_bn_train_fwd(const float* x, const float* gamma, const float* beta, float* running_mean, float* running_var, float* y,
                                             float* save_mean, float* save_invstd, double* scratch, int N, int C, int HW, int relu, void* stream) {
    ARGCHK(x && gamma && beta && y && save_mean && save_invstd && scratch && N > 0 && C > 0 && HW > 0, "bn_train_fwd: bad arguments");
    // F.batch_norm in training mode refuses one value per channel (its variance is undefined)
    ARGCHK((long long)N * HW > 1, "bn_train_fwd: expected more than 1 value per channel when training");
    cudaStream_t s = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemsetAsync(scratch, 0, (size_t)2 * C * sizeof(double), s));
    const long long per = (long long)N * HW;
    int slices = (int)((per + 256 * 16 - 1) / (256 * 16));
    slices = slices < 1 ? 1 : (slices > 64 ? 64 : slices);
    if (slices > N) slices = N;
    bn_stats_kernel<<<dim3(C, slices), 256, 0, s>>>(x, scratch, N, C, HW);
    YFV2_LAUNCH_CHECK();
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, s>>>(scratch, save_mean, save_invstd, running_mean, running_var, C, (double)per, 0.1f);
    YFV2_LAUNCH_CHECK();
    bn_apply_kernel<<<dim3((unsigned)(N * C), (unsigned)((HW + 1023) / 1024)), 256, 0, s>>>(x, save_mean, save_invstd, gamma, beta, y, C, HW, relu);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
extern "C" YFV2_API int yfv2_op_bn_train_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean,
                                             const float* save_invstd, float* dx, float* dgamma, float* dbeta, double* scratch, int N, int C, int HW,
                                             int relu, void* stream) {
    ARGCHK(x && y && dy && gamma && save_mean && save_invstd && dx && dgamma && dbeta && scratch, "bn_train_bwd: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemsetAsync(scratch, 0, (size_t)2 * C * sizeof(double), s));
    const long long per = (long long)N * HW;
    int slices = (int)((per + 256 * 16 - 1) / (256 * 16));
    slices = slices < 1 ? 1 : (slices > 64 ? 64 : slices);
    if (slices > N) slices = N;
    bn_bwd_reduce_kernel<<<dim3(C, slices), 256, 0, s>>>(x, y, dy, save_mean, save_invstd, scratch, N, C, HW, relu);
    YFV2_LAUNCH_CHECK();
    bn_bwd_apply_kernel<<<dim3((unsigned)(N * C), (unsigned)((HW + 1023) / 1024)), 256, 0, s>>>(x, y, dy, save_mean, save_invstd, gamma, scratch, dx,
                                                                                               dgamma, dbeta, C, HW, (double)per, relu);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" YFV2_API int yfv2_op_maxpool_fwd(const float* x, float* y, int* idx, int planes, int H, int W, void* stream) {
    ARGCHK(x && y && idx, "maxpool_fwd: bad arguments");
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    maxpool_fwd_kernel<<<grid_for((long long)planes * Ho * Wo), 256, 0, (cudaStream_t)stream>>>(x, y, idx, planes, H, W);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
extern "C" YFV2_API int yfv2_op_maxpool_bwd(const float* dy, const int* idx, float* dx, int planes, int H, int W, void* stream) {
    ARGCHK(dy && idx && dx, "maxpool_bwd: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemsetAsync(dx, 0, (size_t)planes * H * W * sizeof(float), s));
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    maxpool_bwd_kernel<<<grid_for((long long)planes * Ho * Wo), 256, 0, s>>>(dy, idx, dx, planes, H, W);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
extern "C" YFV2_API int yfv2_op_upsample2_fwd(const float* x, float* y, int planes, int H, int W, void* stream) {
    ARGCHK(x && y, "upsample2_fwd: bad arguments");
    upsample2_fwd_kernel<<<grid_for((long long)planes * 4 * H * W), 256, 0, (cudaStream_t)stream>>>(x, y, planes, H, W);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
extern "C" YFV2_API int yfv2_op_upsample2_bwd(const float* dy, float* dx, int planes, int H, int W, void* stream) {
    ARGCHK(dy && dx, "upsample2_bwd: bad arguments");
    upsample2_bwd_kernel<<<grid_for((long long)planes * H * W), 256, 0, (cudaStream_t)stream>>>(dy, dx, planes, H, W);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
