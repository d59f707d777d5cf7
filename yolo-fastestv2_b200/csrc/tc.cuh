// Hopper (sm_90a) building blocks: mbarrier / TMA bulk copies, and the warp-level 3xTF32 tensor-core contraction every 1x1
// "pointwise" convolution of the network runs on.
//
// Scheme: error-compensated TF32 ("3xTF32").  An fp32 operand a is split as a = hi + lo with hi = a with the low 13 mantissa
// bits cleared (exactly a tf32 value) and lo = a - hi (exact in fp32, |lo| < 2^-10 |a|); the product A*B is accumulated as
// Alo*Bhi + Ahi*Blo + Ahi*Bhi in fp32 (the dropped Alo*Blo term is ~2^-20 relative).  Single-pass TF32 misses the 1e-4
// parity bar of the network by orders of magnitude, the 3-pass split meets it.
//
// One warp owns a 16-pixel row tile of the output (mma.sync m16n8k8): the A fragment is produced by a caller functor straight
// from wherever the operand lives (activation planes, a depthwise convolution computed on the fly), the weights are a
// [K][S] fp32 matrix in shared memory (S = row stride chosen so the B-fragment reads are bank-conflict free).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace yfv2 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// Bounded spin: a protocol bug must surface as a trapped kernel, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
#pragma unroll 1        // (left to itself nvcc unrolls this spin 64x at every call site: ~2 KB of SASS each)
    for (uint32_t it = 0; it < (1u << 26); ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return;
    }
    __trap();
}

// ---- TMA bulk copy: contiguous global -> shared, completion counted in bytes on an mbarrier ---------------------------
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- 3xTF32 warp contraction -----------------------------------------------------------------------------------
// Row stride (floats) of a [K][N] weight matrix in shared memory: the B fragment of a warp reads rows t, t+4 (t = lane % 4)
// at columns g (g = lane / 4), conflict free when the stride is 8 or 24 modulo 32.
__host__ __device__ constexpr int w_stride(int N) { return (N % 16 == 0) ? N + 8 : N; }
__host__ __device__ constexpr int round_up(int x, int m) { return (x + m - 1) / m * m; }

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x) & 0xFFFFE000u;
    lo = __float_as_uint(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[nt] = A(16 x 8 KS) * W(8 KS x 8 NT) for the calling warp's 16-row tile.
// load_a(ks, a) fills this lane's A fragment of k-step ks: a[0] = (row g, k 8ks+t), a[1] = (g+8, 8ks+t), a[2] = (g, 8ks+t+4),
// a[3] = (g+8, 8ks+t+4).  Result: acc[nt][0..1] = (row g, columns 8nt+2t, 8nt+2t+1), acc[nt][2..3] = the same for row g+8.
template <int KS, int NT, class LoadA>
__device__ __forceinline__ void warp_gemm(float (&acc)[NT][4], const float* __restrict__ sW, int S, LoadA&& load_a) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll 2
    for (int ks = 0; ks < KS; ++ks) {
        float a[4];
        load_a(ks, a);
        uint32_t ah[4], al[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_tf32(a[i], ah[i], al[i]);
        const float* w0 = sW + (8 * ks + t) * S + g;
        const float* w1 = w0 + 4 * S;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            uint32_t bh0, bl0, bh1, bl1;
            split_tf32(w0[8 * nt], bh0, bl0);
            split_tf32(w1[8 * nt], bh1, bl1);
            mma_tf32(acc[nt], al, bh0, bh1);      // small terms first
            mma_tf32(acc[nt], ah, bl0, bl1);
            mma_tf32(acc[nt], ah, bh0, bh1);
        }
    }
}

// The same contraction with the KS A fragments already in registers (a[ks] as load_a would fill it), so that one A operand can
// be contracted against several column tiles of W.  Fully unrolled: a[] must stay in registers.  Per accumulator the MMAs run in
// the order warp_gemm issues them, so the result is bit-identical to warp_gemm on the same operands.
template <int KS, int NT>
__device__ __forceinline__ void warp_gemm_regs(float (&acc)[NT][4], const float* __restrict__ sW, int S, const float (&a)[KS][4]) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        uint32_t ah[4], al[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_tf32(a[ks][i], ah[i], al[i]);
        const float* w0 = sW + (8 * ks + t) * S + g;
        const float* w1 = w0 + 4 * S;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            uint32_t bh0, bl0, bh1, bl1;
            split_tf32(w0[8 * nt], bh0, bl0);
            split_tf32(w1[8 * nt], bh1, bl1);
            mma_tf32(acc[nt], al, bh0, bh1);
            mma_tf32(acc[nt], ah, bl0, bl1);
            mma_tf32(acc[nt], ah, bh0, bh1);
        }
    }
}

}  // namespace tc
}  // namespace yfv2
