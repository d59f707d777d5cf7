// K0 — stem: conv3x3 s2 p1 (3->24, no bias) + BN + ReLU + maxpool3x3 s2 p1, one pass.
// Reference: model/backbone/shufflenetv2.py:74-80,103-104.  Input NCHW fp32 (or uint8 with the `/255.0` of
// utils/utils.py:368 fused into the load), output 24 framed planes at H/4 x W/4.
//
// Why CUDA cores and not the tensor core: the contraction per conv position is only K = 27 taps x N = 24 channels, and the
// stem's time goes into staging the input patch and pooling, not into the products.  An implicit-GEMM stem on the mma.sync
// contraction of tc.cuh (patch in shared memory, 16 conv positions per warp, uint8 pixels as exact TF32 operands with the
// 1/255 in the weights, pooling from a conv tile in shared memory) measured 1400 us against 772 us for this kernel per
// batch-256 352x352 step on an H100 80GB HBM3 at 700 W (two alternating runs each).  This kernel is a register-tiled direct
// convolution that pools in registers: one thread = 4 adjacent conv positions of one conv row x all 24 channels
// (96 accumulators), inputs come from three aligned LDS.128 per (channel, kernel row), weights from warp-uniform
// LDS.128, i.e. 2592 FFMA against ~190 shared-memory instructions (93 % FFMA in the main loop).
//
// A work item is (image, band of TRo pooled rows, tile of TWo <= 44 pooled columns):
//   0. fp32: the input patch arrives by one TMA bulk copy per (channel, row), issued after the previous item's conv, while it
//      pools.  uint8: the raw bytes of the next item arrive by 16-byte cp.async (zero-filled outside the image) in the half of
//      Hs that is free during the conv, issued before the conv; after it they are converted into Xin through a 256-entry
//      table of v / 255.0f (one correctly rounded division per byte value, so no per-pixel division).  A base that is not
//      16-byte aligned (or, for uint8, W not a multiple of 16): scalar loads after the conv;
//   1. conv + BN (scale folded into the weights, shift = accumulator init) for the CR = 2 TRo + 1 conv rows the pool
//      windows touch; positions outside the conv output become -inf (PyTorch pads max_pool2d with -inf);
//   2. horizontal 3-max in registers (the one column a thread lacks comes from its right neighbour through shared
//      memory), vertical 3-max + ReLU from shared memory -> framed output planes.  ReLU commutes with max, so it runs
//      once per pooled value instead of once per conv value.
#include "common.cuh"
#include "tc.cuh"

namespace yfv2 {

namespace {
using namespace tc;

constexpr int ST_THREADS = 256;
constexpr int kStemW = 27 * 24 + 24;              // folded weights [27][24] | shift[24]

struct StemFArgs {
    const void* x;
    Planes out;
    const float* wpack;     // [27][24] | scale[24] | shift[24]
    int N, H, W;
    int TRo, TWo, tilesX, tilesY, S;
    int vec;                // fp32: base 16-byte aligned -> bulk copies; uint8: base and W multiples of 16 -> cp.async
};

// bytes per staged uint8 row: the Wst = 4 TWo + 12 columns from ic0, plus up to 12 before them from ic0 & ~15, rounded to 16
__host__ __device__ __forceinline__ int stem_byte_row(int TWo) { return (4 * TWo + 24 + 15) & ~15; }

__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <bool U8>
__global__ void __launch_bounds__(ST_THREADS, 2)
stem_kernel(const __grid_constant__ StemFArgs p) {
    pdl_trigger();                                     // the first stride-2 block may start its prologue now
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t xbar;
    const int TRo = p.TRo, TWo = p.TWo, S = p.S;
    const int CR = 2 * TRo + 1, IR = 4 * TRo + 3, Wst = 4 * TWo + 12;     // staged column 0 <-> input column 4*ox0 - 4
    const int HSW = 2 * S;
    float* sW = smem;                                  // folded weights + shift
    float* lut = sW + kStemW;                          // [256] byte v -> v / 255.0f
    float* Xin = lut + 256;                            // [3][IR][Wst]
    float* Hs = Xin + 3 * IR * Wst;                    // [24][CR][HSW] horizontal maxima; its head doubles as
    float* E = Hs;                                     // [24][CR][S]   first conv column of every strip
    // [3][IR][Wb] raw uint8 patch of the next item, in the half of Hs that is free from B0 until B2 (E is the other half)
    const int Wb = stem_byte_row(TWo);
    uint8_t* Xb = reinterpret_cast<uint8_t*>(Hs + 24 * CR * S);
    const int tid = threadIdx.x;
    {   // BN scale folded into the weights (one rounding per weight), shift kept as the accumulator's start value
        const float* scale = p.wpack + 27 * 24;
        for (int i = tid; i < 27 * 24; i += ST_THREADS) sW[i] = __fmul_rn(__ldg(p.wpack + i), __ldg(scale + (i % 24)));
        if (tid < 24) sW[27 * 24 + tid] = __ldg(scale + 24 + tid);
        // the `/255.0` of utils/utils.py:368 as a table: the same correctly rounded quotient without a division per pixel
        if (U8)
            for (int v = tid; v < 256; v += ST_THREADS) lut[v] = __fdiv_rn((float)v, 255.0f);
    }
    if (tid == 0) { mbar_init(&xbar, 1); fence_mbar_init(); }
    __syncthreads();
    pdl_wait();
    const int H = p.H, W = p.W, HC = H / 2, WC = W / 2, HO = H / 4, WO = W / 4;
    const int items = p.N * p.tilesX * p.tilesY;

    auto stage = [&](int item) {
        const int n = item / (p.tilesX * p.tilesY);
        const int rem = item - n * (p.tilesX * p.tilesY);
        const int ty = rem / p.tilesX, tx = rem - ty * p.tilesX;
        const int iy0 = 4 * (ty * TRo) - 3, ic0 = 4 * (tx * TWo) - 4;
        const int c_lo = max(ic0, 0), c_hi = min(ic0 + Wst, W);
        if (!p.vec) {
            for (int i = tid; i < 3 * IR * Wst; i += ST_THREADS) {
                const int cr = i / Wst, j = i - cr * Wst;
                const int c = cr / IR, r = cr - c * IR;
                const int iy = iy0 + r, ix = ic0 + j;
                float v = 0.f;
                if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
                    const size_t idx = (((size_t)n * 3 + c) * H + iy) * W + ix;
                    v = U8 ? lut[__ldg(reinterpret_cast<const uint8_t*>(p.x) + idx)] : __ldg(reinterpret_cast<const float*>(p.x) + idx);
                }
                Xin[i] = v;
            }
        } else if (!U8) {
            const int r_lo = max(iy0, 0), r_hi = min(iy0 + IR, H);
            if (tid == 0) mbar_expect_tx(&xbar, (uint32_t)(3 * (r_hi - r_lo) * (c_hi - c_lo) * sizeof(float)));
            for (int i = tid; i < 3 * IR; i += ST_THREADS) {
                const int c = i / IR, r = i - c * IR;
                const int iy = iy0 + r;
                float* dst = Xin + (c * IR + r) * Wst;
                if (iy >= 0 && iy < H) {
                    bulk_g2s(dst + (c_lo - ic0), reinterpret_cast<const float*>(p.x) + (((size_t)n * 3 + c) * H + iy) * W + c_lo,
                             (uint32_t)((c_hi - c_lo) * sizeof(float)), &xbar);
                    for (int j = 0; j < c_lo - ic0; ++j) dst[j] = 0.f;
                    for (int j = c_hi - ic0; j < Wst; ++j) dst[j] = 0.f;
                } else {
                    for (int j = 0; j < Wst; ++j) dst[j] = 0.f;
                }
            }
        } else {
            // raw bytes -> Xb rows of Wb bytes that start at input column ic0 & ~15, 16 per cp.async: every copy in flight at
            // once.  The base and W are multiples of 16, so a chunk lies wholly inside or wholly outside the image; outside
            // ones are zero-filled (byte 0 converts to 0.f)
            const uint8_t* x8 = reinterpret_cast<const uint8_t*>(p.x);
            const int a0 = ic0 & ~15, q16 = Wb / 16;
            for (int i = tid; i < 3 * IR * q16; i += ST_THREADS) {
                const int cr = i / q16, j = i - cr * q16;
                const int c = cr / IR, r = cr - c * IR;
                const int iy = iy0 + r, ix = a0 + 16 * j;
                const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
                cp_async16_zfill(Xb + 16 * i, in ? x8 + (((size_t)n * 3 + c) * H + iy) * W + ix : x8, in ? 16u : 0u);
            }
        }
    };
    // uint8 with aligned base: Xb (complete, after a barrier) -> Xin, 4 pixels per step
    auto convert = [&](int item) {
        const int tx = item % p.tilesX;
        const int off = (4 * (tx * TWo) - 4) & 15;           // ic0 - (ic0 & ~15)
        const int q4 = Wst / 4;
        for (int i = tid; i < 3 * IR * q4; i += ST_THREADS) {
            const int cr = i / q4, j4 = i - cr * q4;
            const uint32_t b = *reinterpret_cast<const uint32_t*>(Xb + cr * Wb + off + 4 * j4);
            *reinterpret_cast<float4*>(Xin + 4 * i) = make_float4(lut[b & 255u], lut[(b >> 8) & 255u], lut[(b >> 16) & 255u], lut[b >> 24]);
        }
    };
    const bool async_u8 = U8 && p.vec;

    const int r = tid / S, s = tid - r * S;                  // conv row of the band / strip of 4 conv columns
    const int p_oyl = tid / TWo, p_pc = tid - p_oyl * TWo;   // pooled pixel this thread writes in step 3
    uint32_t xpar = 0;
    if (blockIdx.x < items) {
        stage(blockIdx.x);
        if (async_u8) {
            cp_async_wait_all();
            __syncthreads();
            convert(blockIdx.x);
        }
    }
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int n = item / (p.tilesX * p.tilesY);
        const int rem = item - n * (p.tilesX * p.tilesY);
        const int ty = rem / p.tilesX, tx = rem - ty * p.tilesX;
        const int oy0 = ty * TRo, ox0 = tx * TWo;
        const int rows = min(TRo, HO - oy0), cols = min(TWo, WO - ox0);
        const bool active = r < 2 * rows + 1;
        if (!U8 && p.vec) { mbar_wait(&xbar, xpar); xpar ^= 1u; }
        __syncthreads();                                      // B0: edge zero-fill / converted uint8 visible; Hs free again
        const bool more = item + gridDim.x < items;
        if (async_u8 && more) stage(item + gridDim.x);        // the next item's bytes arrive while this one convolves

        // ---- 1. conv: acc[j][ch], j = position 4s+j of conv row r (tile-local) ----------------------------------------
        float h0[24], h1[24];
        if (active) {
            // accumulators as channel pairs, read from shared memory as float4 / float2 weight vectors
            float2 acc2[4][12];
#pragma unroll
            for (int m = 0; m < 12; ++m) {
                const float2 sh = *reinterpret_cast<const float2*>(sW + 27 * 24 + 2 * m);
#pragma unroll
                for (int j = 0; j < 4; ++j) acc2[j][m] = sh;
            }
            const float* xb = Xin + (2 * r) * Wst + 8 * s;   // staged col of (position j, tap kx) = 8s + 2j + kx + 1
#pragma unroll
            for (int c = 0; c < 3; ++c) {
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    float x[12];
                    const float4* xr = reinterpret_cast<const float4*>(xb + (c * IR + ky) * Wst);
#pragma unroll
                    for (int t = 0; t < 3; ++t) { const float4 v = xr[t]; x[4 * t] = v.x; x[4 * t + 1] = v.y; x[4 * t + 2] = v.z; x[4 * t + 3] = v.w; }
                    float2 xx[9];
#pragma unroll
                    for (int t = 0; t < 9; ++t) xx[t] = make_float2(x[t + 1], x[t + 1]);
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float4* wr = reinterpret_cast<const float4*>(sW + ((c * 3 + ky) * 3 + kx) * 24);
#pragma unroll
                        for (int q = 0; q < 6; ++q) {
                            const float4 w = wr[q];
                            const float2 w01 = make_float2(w.x, w.y), w23 = make_float2(w.z, w.w);
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                acc2[j][2 * q] = ffma2(xx[2 * j + kx], w01, acc2[j][2 * q]);
                                acc2[j][2 * q + 1] = ffma2(xx[2 * j + kx], w23, acc2[j][2 * q + 1]);
                            }
                        }
                    }
                }
            }
            float acc[4][24];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int m = 0; m < 12; ++m) { acc[j][2 * m] = acc2[j][m].x; acc[j][2 * m + 1] = acc2[j][m].y; }
            // conv positions outside the conv output never win a pool window
            const int cy = 2 * oy0 - 1 + r, cx = 2 * ox0 - 1 + 4 * s;
            const bool rowok = cy >= 0 && cy < HC;
            if (!rowok || cx < 0 || cx + 3 >= WC) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const bool ok = rowok && cx + j >= 0 && cx + j < WC;
                    if (!ok) {
#pragma unroll
                        for (int ch = 0; ch < 24; ++ch) acc[j][ch] = -INFINITY;
                    }
                }
            }
            // horizontal 3-max, part 1: pooled column 2s <- positions 0,1,2; 2s+1 <- positions 2,3 (+ the neighbour's 0 below)
#pragma unroll
            for (int ch = 0; ch < 24; ++ch) {
                E[(ch * CR + r) * S + s] = acc[0][ch];
                h0[ch] = max3(acc[0][ch], acc[1][ch], acc[2][ch]);
                h1[ch] = fmaxf(acc[2][ch], acc[3][ch]);
            }
        }
        if (async_u8 && more) cp_async_wait_all();          // this thread's bytes of the next item have landed
        __syncthreads();                                      // B1: every read of Xin is done, E and Xb are visible
        if (async_u8 && more) {
            convert(item + gridDim.x);
        } else if (more) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of Xin before the async-proxy refill
            stage(item + gridDim.x);                          // overlaps the pooling below
        }
        if (active && s + 1 < S) {
#pragma unroll
            for (int ch = 0; ch < 24; ++ch) h1[ch] = fmaxf(h1[ch], E[(ch * CR + r) * S + s + 1]);
        }
        __syncthreads();                                      // B2: E has been read, Hs may overwrite it
        if (active) {
#pragma unroll
            for (int ch = 0; ch < 24; ++ch)
                *reinterpret_cast<float2*>(Hs + (ch * CR + r) * HSW + 2 * s) = make_float2(h0[ch], h1[ch]);
        }
        __syncthreads();                                      // B3
        // ---- 3. vertical 3-max + ReLU -> output planes: thread <-> pooled pixel of the tile, loop over the channels --------
        if (p_oyl < rows && p_pc < cols) {
            const float* hb = Hs + (2 * p_oyl) * HSW + p_pc;
            float* op = plane_ptr(p.out, n, 0) + p.out.org + (oy0 + p_oyl) * p.out.Ws + ox0 + p_pc;
            const int hstep = CR * HSW;
            const size_t ostep = (size_t)p.out.sC;
#pragma unroll 4
            for (int ch = 0; ch < 24; ++ch) {
                *op = fmaxf(max3(hb[0], hb[HSW], hb[2 * HSW]), 0.f);
                hb += hstep;
                op += ostep;
            }
        }
    }
}

__host__ size_t stem_smem_bytes(int TRo, int TWo, int S) {
    const int CR = 2 * TRo + 1, IR = 4 * TRo + 3, Wst = 4 * TWo + 12;
    return (size_t)(kStemW + 256 + 3 * IR * Wst + 24 * CR * 2 * S + 4) * sizeof(float);
}
// the uint8 patch fits the half of Hs that E leaves free
__host__ bool stem_bytes_fit(int TRo, int TWo, int S) {
    return 3 * (4 * TRo + 3) * stem_byte_row(TWo) <= 24 * (2 * TRo + 1) * S * (int)sizeof(float);
}
}  // namespace

int launch_stem(const StemArgs& a, cudaStream_t s) {
    const auto& t = a.launch.stem;
    const StemFArgs k{a.x, a.out, a.wpack, a.N, a.H, a.W, t.TRo, t.TWo, t.tilesX, t.tilesY, t.S, ((uintptr_t)a.x & 15) == 0 && t.vec};
    return launch(a.launch, &k, s);
}

static_assert(ST_THREADS == kThreads, "launch() runs every forward kernel with kThreads threads");

KernelRef stem_kernel_ref(bool u8) { return u8 ? YFV2_KERNEL_REF(stem_kernel<true>) : YFV2_KERNEL_REF(stem_kernel<false>); }

int describe_stem(int N, int H, int W, int is_u8, int sms, Launch& L) {
    if (H % 4 || W % 4 || H < 4 || W < 4) { set_error("stem: input %dx%d must be a multiple of 4", H, W); return YFV2_EINVAL; }
    auto& k = L.stem;
    const int HO = H / 4, WO = W / 4;
    // tiles of at most 44 pooled columns, as equal as possible; S strips of 4 conv columns cover the 2 TWo + 1 conv columns
    k.tilesX = (WO + 43) / 44;
    k.TWo = (WO + k.tilesX - 1) / k.tilesX;
    k.S = (2 * k.TWo + 1 + 3) / 4;
    // as many conv rows as the 256 threads cover, within ~half an SM's shared memory (two CTAs per SM)
    k.TRo = (ST_THREADS / k.S - 1) / 2;
    if (k.TRo > HO) k.TRo = HO;
    while (k.TRo > 1 && stem_smem_bytes(k.TRo, k.TWo, k.S) > 112 * 1024) --k.TRo;
    if (k.TRo < 1) k.TRo = 1;
    const size_t bytes = stem_smem_bytes(k.TRo, k.TWo, k.S);
    if ((2 * k.TRo + 1) * k.S > ST_THREADS || k.TRo * k.TWo > ST_THREADS || bytes > kSmemCap - 1024) { set_error("stem: unsupported geometry %dx%d", H, W); return YFV2_EUNSUPPORTED; }
    // asynchronous staging needs 16-byte aligned rows (uint8: and room for the bytes); other inputs take the scalar loads
    k.vec = !is_u8 || (W % 16 == 0 && stem_bytes_fit(k.TRo, k.TWo, k.S));
    k.tilesY = (HO + k.TRo - 1) / k.TRo;
    L.kernel = is_u8 ? KernelId::stem_u8 : KernelId::stem_f32;
    L.smem = bytes;
    L.items = N * k.tilesX * k.tilesY;
    L.grid = dim3((unsigned)(L.items < 2 * sms ? L.items : 2 * sms));
    return YFV2_OK;
}

}  // namespace yfv2
