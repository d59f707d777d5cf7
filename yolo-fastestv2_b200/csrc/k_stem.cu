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
//   0. fp32: the input patch arrives in Xin by one TMA bulk copy per (channel, row), issued after the previous item's conv.
//      uint8: the raw bytes arrive by 16-byte cp.async (zero-filled outside the image) in one of two byte patches, issued
//      while the previous item convolves from the other; each conv thread converts the bytes it reads through a 256-entry
//      table of v / 255.0f (one correctly rounded division per byte value, so no per-pixel division).  A base that is not
//      16-byte aligned (or, for uint8, W not a multiple of 16): scalar loads at the same points;
//   1. conv + BN (scale folded into the weights, shift = accumulator init) for the CR = 2 TRo + 1 conv rows the pool
//      windows touch; positions outside the conv output become -inf (PyTorch pads max_pool2d with -inf);
//   2. horizontal 3-max in registers (the one column a thread lacks comes from the next lane by a shuffle, or from the next
//      warp through shared memory) -> Hs;
//   3. vertical 3-max + ReLU from Hs -> framed output planes, while the next item convolves.  ReLU commutes with max, so it
//      runs once per pooled value instead of once per conv value.
// Two barriers per item: B0 (patch staged, Hs complete) and B1 (patch and Hs read, Eb written).
#include "common.cuh"
#include "tc.cuh"

namespace yfv2 {

namespace {
using namespace tc;

constexpr int ST_THREADS = 256;
constexpr int kStemW = 27 * 24 + 24;              // folded weights [27][24] | shift[24]
constexpr int kStemE = (ST_THREADS / 32) * 24;    // one conv column per warp, passed to the warp before
// copies of the byte -> float table: lane l reads copy l % 16, so two lanes of a warp share a bank only when they are 16 apart
// and their bytes differ with the same parity (at most 2 wavefronts per table read, 1.5 on random bytes)
constexpr int kLutCopies = 16;

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
    const int HSW = 2 * S, Wb = stem_byte_row(TWo);
    float* sW = smem;                                  // folded weights + shift
    float* Eb = sW + kStemW;                           // [8 warps][24] first conv column of each warp's lane 0
    float* Hs = Eb + kStemE;                           // [24][CR][HSW] horizontal maxima of the last convolved item
    float* Xin = Hs + 24 * CR * HSW;                   // fp32: [3][IR][Wst] input patch
    float* lut = Xin;                                  // uint8: [256][kLutCopies] byte v -> v / 255.0f, one copy per bank pair
    uint8_t* Xb = reinterpret_cast<uint8_t*>(lut + 256 * kLutCopies);   // uint8: two [3][IR][Wb] raw patches
    const int xbytes = 3 * IR * Wb;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {   // BN scale folded into the weights (one rounding per weight), shift kept as the accumulator's start value
        const float* scale = p.wpack + 27 * 24;
        for (int i = tid; i < 27 * 24; i += ST_THREADS) sW[i] = __fmul_rn(__ldg(p.wpack + i), __ldg(scale + (i % 24)));
        if (tid < 24) sW[27 * 24 + tid] = __ldg(scale + 24 + tid);
        // the `/255.0` of utils/utils.py:368 as a table: the same correctly rounded quotient without a division per pixel
        if (U8)
            for (int i = tid; i < 256 * kLutCopies; i += ST_THREADS) lut[i] = __fdiv_rn((float)(i / kLutCopies), 255.0f);
    }
    if (tid == 0) { mbar_init(&xbar, 1); fence_mbar_init(); }
    __syncthreads();
    pdl_wait();
    const int H = p.H, W = p.W, HC = H / 2, WC = W / 2, HO = H / 4, WO = W / 4;
    const int items = p.N * p.tilesX * p.tilesY;

    // the input patch of `item`: uint8 into the raw patch xb, fp32 into Xin
    auto stage = [&](int item, uint8_t* xb) {
        const int n = item / (p.tilesX * p.tilesY);
        const int rem = item - n * (p.tilesX * p.tilesY);
        const int ty = rem / p.tilesX, tx = rem - ty * p.tilesX;
        const int iy0 = 4 * (ty * TRo) - 3, ic0 = 4 * (tx * TWo) - 4;
        if (U8) {
            // rows of Wb bytes that start at input column a0 = ic0 & ~15, so staged column j is byte (ic0 - a0) + j of its row
            const uint8_t* x8 = reinterpret_cast<const uint8_t*>(p.x);
            const int a0 = ic0 & ~15;
            if (p.vec) {
                // 16 bytes per cp.async, a row per 16 threads, every copy in flight at once.  The base and W are multiples of
                // 16, so a chunk lies wholly inside or wholly outside the image; outside ones are zero-filled (byte 0 -> 0.f)
                const int j = tid & 15;
                if (j < Wb / 16) {
                    int c = 0, r = tid >> 4;
                    for (int cr = r; cr < 3 * IR; cr += ST_THREADS / 16, r += ST_THREADS / 16) {
                        while (r >= IR) { r -= IR; ++c; }
                        const int iy = iy0 + r, ix = a0 + 16 * j;
                        const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
                        cp_async16_zfill(xb + cr * Wb + 16 * j, in ? x8 + (((size_t)n * 3 + c) * H + iy) * W + ix : x8, in ? 16u : 0u);
                    }
                }
            } else {
                for (int i = tid; i < 3 * IR * Wst; i += ST_THREADS) {
                    const int cr = i / Wst, j = i - cr * Wst;
                    const int c = cr / IR, r = cr - c * IR;
                    const int iy = iy0 + r, ix = ic0 + j;
                    uint8_t v = 0;
                    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(x8 + (((size_t)n * 3 + c) * H + iy) * W + ix);
                    xb[cr * Wb + (ic0 - a0) + j] = v;
                }
            }
        } else if (!p.vec) {
            for (int i = tid; i < 3 * IR * Wst; i += ST_THREADS) {
                const int cr = i / Wst, j = i - cr * Wst;
                const int c = cr / IR, r = cr - c * IR;
                const int iy = iy0 + r, ix = ic0 + j;
                float v = 0.f;
                if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(reinterpret_cast<const float*>(p.x) + (((size_t)n * 3 + c) * H + iy) * W + ix);
                Xin[i] = v;
            }
        } else {
            const int c_lo = max(ic0, 0), c_hi = min(ic0 + Wst, W);
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
        }
    };

    const int r = tid / S, s = tid - r * S;                  // conv row of the band / strip of 4 conv columns
    const int p_oyl = tid / TWo, p_pc = tid - p_oyl * TWo;   // pooled pixel this thread writes in step 3
    // ---- 3. vertical 3-max + ReLU of `item` from Hs -> output planes: thread <-> pooled pixel, loop over the channels ------
    auto pool = [&](int item) {
        const int n = item / (p.tilesX * p.tilesY);
        const int rem = item - n * (p.tilesX * p.tilesY);
        const int ty = rem / p.tilesX, tx = rem - ty * p.tilesX;
        const int oy0 = ty * TRo, ox0 = tx * TWo;
        if (p_oyl < min(TRo, HO - oy0) && p_pc < min(TWo, WO - ox0)) {
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
    };
    const float* lt = lut + (lane & (kLutCopies - 1));       // this lane's copy of the table
    uint32_t xpar = 0;
    if (blockIdx.x < items) stage(blockIdx.x, Xb);
    int buf = 0;
    for (int item = blockIdx.x; item < items; item += gridDim.x, buf ^= 1) {
        const int n = item / (p.tilesX * p.tilesY);
        const int rem = item - n * (p.tilesX * p.tilesY);
        const int ty = rem / p.tilesX, tx = rem - ty * p.tilesX;
        const int oy0 = ty * TRo, ox0 = tx * TWo;
        const int rows = min(TRo, HO - oy0);
        const bool active = r < 2 * rows + 1;
        if (U8 && p.vec) cp_async_wait_all();                // this thread's bytes of the item have landed
        __syncthreads();                                      // B0: the item's patch is staged; Hs holds the previous item
        const bool more = item + gridDim.x < items;
        if (U8 && more) stage(item + gridDim.x, Xb + (buf ^ 1) * xbytes);   // arrives while this item convolves
        if (item != blockIdx.x) pool(item - gridDim.x);
        if (!U8 && p.vec) { mbar_wait(&xbar, xpar); xpar ^= 1u; }

        // ---- 1. conv: acc[j][ch], j = position 4s+j of conv row r (tile-local) ----------------------------------------
        float h0[24], h1[24], e0[24];
        if (active) {
            // accumulators as channel pairs, read from shared memory as float4 / float2 weight vectors
            float2 acc2[4][12];
#pragma unroll
            for (int m = 0; m < 12; ++m) {
                const float2 sh = *reinterpret_cast<const float2*>(sW + 27 * 24 + 2 * m);
#pragma unroll
                for (int j = 0; j < 4; ++j) acc2[j][m] = sh;
            }
            // staged col of (position j, tap kx) = 8s + 2j + kx + 1
            const float* xf = Xin + (2 * r) * Wst + 8 * s;
            const uint8_t* x8 = Xb + buf * xbytes + (2 * r) * Wb + ((4 * ox0 - 4) & 15) + 8 * s;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    float x[9];                               // staged cols 8s + 1 .. 8s + 9
                    if constexpr (U8) {
                        // bytes 1 .. 9 of three aligned words, each converted by the lane's copy of the table
                        const uint32_t* xw = reinterpret_cast<const uint32_t*>(x8 + (c * IR + ky) * Wb);
                        const uint32_t b0 = xw[0], b1 = xw[1], b2 = xw[2];
                        x[0] = lt[((b0 >> 8) & 255u) * kLutCopies];
                        x[1] = lt[((b0 >> 16) & 255u) * kLutCopies];
                        x[2] = lt[(b0 >> 24) * kLutCopies];
                        x[3] = lt[(b1 & 255u) * kLutCopies];
                        x[4] = lt[((b1 >> 8) & 255u) * kLutCopies];
                        x[5] = lt[((b1 >> 16) & 255u) * kLutCopies];
                        x[6] = lt[(b1 >> 24) * kLutCopies];
                        x[7] = lt[(b2 & 255u) * kLutCopies];
                        x[8] = lt[((b2 >> 8) & 255u) * kLutCopies];
                    } else {
                        const float4* xr = reinterpret_cast<const float4*>(xf + (c * IR + ky) * Wst);
                        const float4 v0 = xr[0], v1 = xr[1], v2 = xr[2];
                        x[0] = v0.y; x[1] = v0.z; x[2] = v0.w; x[3] = v1.x; x[4] = v1.y; x[5] = v1.z; x[6] = v1.w; x[7] = v2.x; x[8] = v2.y;
                    }
                    float2 xx[9];
#pragma unroll
                    for (int t = 0; t < 9; ++t) xx[t] = make_float2(x[t], x[t]);
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
                e0[ch] = acc[0][ch];
                h0[ch] = max3(acc[0][ch], acc[1][ch], acc[2][ch]);
                h1[ch] = fmaxf(acc[2][ch], acc[3][ch]);
            }
        }
        // ---- 2. part 2: strip s + 1 (thread tid + 1) is the next lane, or lane 0 of the next warp through Eb ----------------
        const bool right = active && s + 1 < S;
#pragma unroll
        for (int ch = 0; ch < 24; ++ch) {
            const float nb = __shfl_down_sync(0xffffffffu, e0[ch], 1);
            if (right && lane != 31) h1[ch] = fmaxf(h1[ch], nb);
        }
        if (active && lane == 0) {
#pragma unroll
            for (int ch = 0; ch < 24; ++ch) Eb[warp * 24 + ch] = e0[ch];
        }
        __syncthreads();                                      // B1: every read of the patch and of Hs is done, Eb is visible
        if (!U8 && more) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of Xin before the async-proxy refill
            stage(item + gridDim.x, nullptr);                 // lands while this item's maxima are written and pooled
        }
        if (right && lane == 31) {
#pragma unroll
            for (int ch = 0; ch < 24; ++ch) h1[ch] = fmaxf(h1[ch], Eb[(warp + 1) * 24 + ch]);
        }
        if (active) {
#pragma unroll
            for (int ch = 0; ch < 24; ++ch)
                *reinterpret_cast<float2*>(Hs + (ch * CR + r) * HSW + 2 * s) = make_float2(h0[ch], h1[ch]);
        }
    }
    if (blockIdx.x < items) {                                 // the CTA's last item
        __syncthreads();
        pool(blockIdx.x + (items - 1 - (int)blockIdx.x) / (int)gridDim.x * gridDim.x);
    }
}

__host__ size_t stem_smem_bytes(int TRo, int TWo, int S, bool u8) {
    const int CR = 2 * TRo + 1, IR = 4 * TRo + 3, Wst = 4 * TWo + 12;
    const size_t head = (size_t)(kStemW + kStemE + 24 * CR * 2 * S) * sizeof(float);
    return head + (u8 ? 256 * kLutCopies * sizeof(float) + 2 * (size_t)(3 * IR * stem_byte_row(TWo)) : 3 * (size_t)(IR * Wst) * sizeof(float));
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
    while (k.TRo > 1 && stem_smem_bytes(k.TRo, k.TWo, k.S, is_u8) > 112 * 1024) --k.TRo;
    if (k.TRo < 1) k.TRo = 1;
    const size_t bytes = stem_smem_bytes(k.TRo, k.TWo, k.S, is_u8);
    if ((2 * k.TRo + 1) * k.S > ST_THREADS || k.TRo * k.TWo > ST_THREADS || bytes > kSmemCap - 1024) { set_error("stem: unsupported geometry %dx%d", H, W); return YFV2_EUNSUPPORTED; }
    // asynchronous staging needs 16-byte aligned rows; other inputs take the scalar loads
    k.vec = !is_u8 || W % 16 == 0;
    k.tilesY = (HO + k.TRo - 1) / k.TRo;
    L.kernel = is_u8 ? KernelId::stem_u8 : KernelId::stem_f32;
    L.smem = bytes;
    L.items = N * k.tilesX * k.tilesY;
    L.grid = dim3((unsigned)(L.items < 2 * sms ? L.items : 2 * sms));
    return YFV2_OK;
}

}  // namespace yfv2
