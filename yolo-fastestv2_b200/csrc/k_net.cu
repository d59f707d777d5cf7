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
    // stride-2 blocks were measured slower that way (stage4.0 610 -> 760 us, stage2.0 463 -> 488 us) and take one CTA per item.
    if (STRIDE == 1 && a.nblk == 1) {
        int per_sm = 0;
        YFV2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, blk_kernel<K, STRIDE>, kThreads, bytes));
        grid = persistent_grid(a.items, per_sm > 0 ? per_sm : 1);
    }
    YFV2_CUDA(launch_k(blk_kernel<K, STRIDE>, grid, kThreads, bytes, s, pdl_take(), a));
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

template <int K>
int dispatch_blk(int stride, BlkArgs& a, int N, cudaStream_t s) {
    return stride == 1 ? run_blk<K, 1>(a, N, s) : run_blk<K, 2>(a, N, s);
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
};

constexpr int kHeadTile = 96;      // output columns of one contraction of the second head half (12 n-tiles of 8)

// half 0: dw5x5 + BN + ReLU -> pw + BN -> flat planes.  half 1: dw5x5 + BN + ReLU -> folded matrix + bias -> head tensors.
// HALF 2 (head2_kernel) is half 1 for A + C > 96: the cls branch contracts the same A fragments, kept in registers, against two
// 96-column tiles of a [192][72] folded matrix; the reg branch (4A <= 32 columns) keeps one tile.  It contracts 48 columns at a
// time, so that the A fragments (36 registers) and one pass of accumulators (24) leave room for two CTAs per SM.
template <int HALF>
__device__ __forceinline__ void head_body(const HeadArgs& p) {
    pdl_trigger();
    constexpr int NP = HALF == 0 ? 72 : HALF == 1 ? kHeadTile : 2 * kHeadTile;   // weight columns in shared memory
    constexpr int NT = HALF == 0 ? 9 : HALF == 1 ? kHeadTile / 8 : kHeadTile / 16, S = w_stride(NP);   // n-tiles of one pass
    extern __shared__ __align__(16) float smem[];
    float* sW = smem;
    float* sD = sW + pw_smem_floats(72, NP);      // [72][28]: w[25] | scale | shift | 0
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
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int HW = p.H * p.W;
    const Planes in = p.in[br];
    for (int item = blockIdx.x; item < p.N * p.chunks; item += gridDim.x) {
        const int n = item / p.chunks, m0 = (item - n * p.chunks) * 16 * kWarps + 16 * warp;
        if (m0 >= HW) continue;
        int off[2]; bool ok[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + g + 8 * h, y = m / p.W, x = m - y * p.W;
            ok[h] = m < HW;
            off[h] = ok[h] ? in.org + (y - 2) * in.Ws + x - 2 : in.org;
        }
        const float* ib = in.base + (long long)n * in.sN;
        auto load_a = [&](int ks, float (&a)[4]) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int k = 8 * ks + t + 4 * q;
                const float* w = sD + 28 * k;
                const float* pk = ib + (long long)k * in.sC;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float* tp = pk + off[h];
                    float v = 0.f;
#pragma unroll
                    for (int dy = 0; dy < 5; ++dy)
#pragma unroll
                        for (int dx = 0; dx < 5; ++dx) v = fmaf(tp[dy * in.Ws + dx], w[dy * 5 + dx], v);
                    a[2 * q + h] = ok[h] ? fmaxf(fmaf(v, w[25], w[26]), 0.f) : 0.f;
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
    }
}

template <int HALF>
__global__ void __launch_bounds__(kThreads)
head_kernel(const __grid_constant__ HeadArgs p) { head_body<HALF>(p); }

// Two CTAs per SM, as half 1 gets on its own: 128 registers with 180 bytes of spill.  Left unbounded, ptxas gives it 144 registers
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

bool blk_s1_chainable(int K, int H, int W) { return blk_smem_bytes(K, 1, H, W) <= kChainBudget; }

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
    a.R = blk_rows(K, 2, out.H, in.W, N);
    a.pw1[0] = w1; a.dw[0] = wdwm; a.pw2[0] = w2; a.dwp = wdwp; a.pwp = wp;
    for (int i = 0; i < K; ++i) { a.tin[0][i] = tin.c[i]; a.tout[0][i] = tout.c[i]; a.tmain[i] = tout.c[K + i]; }
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

int heads_launch(int half, const Planes& sIn, const Planes& tcls, const Planes& treg, const float* const wdw[2], const float* const wpw[2],
                 float* reg, float* obj, float* cls, int A, int C, int N, cudaStream_t s) {
    HeadArgs a{};
    for (int b = 0; b < 2; ++b) { a.dw[b] = wdw[b]; a.pw[b] = wpw[b]; }
    a.out[0] = tcls; a.out[1] = treg;
    if (half == 0) { a.in[0] = sIn; a.in[1] = sIn; }
    else { a.in[0] = tcls; a.in[1] = treg; }
    a.dst[0][0] = obj; a.dst[0][1] = cls; a.split[0] = A; a.rowsA[0] = A; a.rowsB[0] = C;
    a.dst[1][0] = reg; a.dst[1][1] = reg; a.split[1] = 4 * A; a.rowsA[1] = 4 * A; a.rowsB[1] = 0;
    a.N = N; a.H = sIn.H; a.W = sIn.W;
    a.chunks = (sIn.H * sIn.W + 16 * kWarps - 1) / (16 * kWarps);
    auto run = [&](auto kern, int np) -> int {
        const size_t bytes = ((size_t)pw_smem_floats(72, np) + 72 * 28) * sizeof(float);
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
    if (half == 0) return run(head_kernel<0>, 72);
    if (A + C <= kHeadTile) return run(head_kernel<1>, kHeadTile);
    if (A + C <= 2 * kHeadTile && 4 * A <= kHeadTile) return run(head2_kernel, 2 * kHeadTile);
    set_error("heads: anchors+classes = %d exceeds two %d-column output tiles", A + C, kHeadTile);
    return YFV2_EUNSUPPORTED;
}
static_assert((pw_smem_floats(72, 2 * kHeadTile) + 72 * 28) * sizeof(float) <= kSmemCap, "two head tiles must fit in shared memory");

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
