// Pieces shared by the post-processing kernels of k_post.cu (the NMS, the fused decode+NMS, the cross-region merge) and k_ncnn.cu
// (the deploy post-process): the CTA and chunk sizes, the shared-memory layout helper, sortable float keys, the bitonic sorting
// networks and the blocked greedy suppression pass.
#pragma once

#include "common.cuh"

namespace yfv2 {
namespace {

constexpr int NT = 256;                // threads of a post-processing CTA
constexpr int kChunk = 64;             // sorted candidates per step of the blocked greedy pass
constexpr int kMaxA = 8;               // anchors per level

// n elements of T at `at`; the next buffer starts 16-byte aligned
template <class T>
__host__ __device__ __forceinline__ T* take(unsigned char*& at, size_t n) {
    T* r = reinterpret_cast<T*>(at);
    at += (n * sizeof(T) + 15) & ~(size_t)15;
    return r;
}

// Size of a key buffer: the power of two >= max(m, 64), the smallest sort the networks below run.
__host__ __device__ __forceinline__ int pow2_at_least(int m) {
    int p = 64;
    while (p < m) p <<= 1;
    return p;
}

// fp32 <-> unsigned keys whose unsigned order is the float order
__device__ __forceinline__ unsigned int f2sortable(float f) {
    const unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float sortable2f(unsigned int s) {
    return __uint_as_float((s & 0x80000000u) ? (s & 0x7fffffffu) : ~s);
}

__device__ void bitonic_sort_desc(unsigned long long* keys, int n2) {
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += NT) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], b = keys[ixj];
                    const bool desc = (i & k) == 0;
                    if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// Same network with E = n2 / NT keys per thread held in registers (thread t owns elements [E t, E t + E)): strides below E
// are compare-exchanges inside the thread, strides below 32 E are 64-bit warp shuffles, and only the log2(NT/32) largest
// strides of the last merges (6 of the 66 steps for 2048 keys) go through shared memory and barriers.  The keys are
// unique (or equal padding zeros), so every correct sorting network yields the same order as bitonic_sort_desc.
// The stage loops are unrolled for E <= 4 and rolled for E = 8: unrolled, the 2048-key network is ~4000 SASS instructions that
// every warp runs exactly once, and ncu found 58 % of the stall samples inside it on instruction fetch (decode + NMS 178.8 us
// per launch unrolled, 161.1 rolled, on the bench workload).  Rolled, k and j are run-time values and the strides below E
// dispatch to three instantiated bodies of sort_intra.
template <int E, int J>
__device__ __forceinline__ void sort_intra(unsigned long long (&v)[E], int k, int t) {
#pragma unroll
    for (int m = 0; m < E; ++m) {
        if ((m & J) == 0) {
            const int i = E * t + m;
            const unsigned long long a = v[m], b = v[m | J];
            const bool desc = (i & k) == 0;
            if (desc ? (a < b) : (a > b)) { v[m] = b; v[m | J] = a; }
        }
    }
}
template <int E>
__device__ void bitonic_sort_desc_reg(unsigned long long* keys) {
    constexpr int n2 = NT * E;
    const int t = threadIdx.x;
    unsigned long long v[E];
#pragma unroll
    for (int m = 0; m < E; ++m) v[m] = keys[E * t + m];
#pragma unroll (E == 8 ? 1 : 16)
    for (int k = 2; k <= n2; k <<= 1) {
#pragma unroll (E == 8 ? 1 : 16)
        for (int j = k >> 1; j > 0; j >>= 1) {
            if (j >= E) {
                unsigned long long o[E];
                const int pj = j / E;                            // partner thread t ^ pj
                if (j >= 32 * E) {
                    __syncthreads();                             // every earlier read of `keys` is done
#pragma unroll
                    for (int m = 0; m < E; ++m) keys[m * NT + t] = v[m];          // transposed: conflict-free both ways
                    __syncthreads();
#pragma unroll
                    for (int m = 0; m < E; ++m) o[m] = keys[m * NT + (t ^ pj)];
                } else {
#pragma unroll
                    for (int m = 0; m < E; ++m) o[m] = __shfl_xor_sync(0xffffffffu, v[m], pj);
                }
                // element i = E t + m: bits of j and k at or above E only depend on t, so the direction is the same for all m
                const int i0 = E * t;
                const bool keep_max = ((i0 & k) == 0) == ((i0 & j) == 0);
#pragma unroll
                for (int m = 0; m < E; ++m) {
                    const unsigned long long a = v[m], b = o[m];
                    v[m] = keep_max ? (a > b ? a : b) : (a < b ? a : b);
                }
            } else {
                if (E > 4 && j == 4) sort_intra<E, (E > 4 ? 4 : 1)>(v, k, t);
                else if (E > 2 && j == 2) sort_intra<E, (E > 2 ? 2 : 1)>(v, k, t);
                else sort_intra<E, 1>(v, k, t);
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int m = 0; m < E; ++m) keys[E * t + m] = v[m];
    __syncthreads();
}

// Sorts the first `cnt` keys descending: pads them with zeros to n2 = pow2_at_least(cnt) (the buffer must hold n2) and runs the
// register network for 256..2048 keys, the shared-memory one otherwise.  All threads of the CTA call this.
// (sort_and_suppress spells the same dispatch out inline: calling this helper there changes its register allocation.)
__device__ __forceinline__ void sort_keys_desc(unsigned long long* keys, int cnt) {
    const int n2 = pow2_at_least(cnt);
    for (int i = cnt + threadIdx.x; i < n2; i += NT) keys[i] = 0ull;
    __syncthreads();
    if (n2 == NT) bitonic_sort_desc_reg<1>(keys);
    else if (n2 == 2 * NT) bitonic_sort_desc_reg<2>(keys);
    else if (n2 == 4 * NT) bitonic_sort_desc_reg<4>(keys);
    else if (n2 == 8 * NT) bitonic_sort_desc_reg<8>(keys);
    else bitonic_sort_desc(keys, n2);
}

// Greedy resolve of one chunk over its kill rows (cmask[2 i], cmask[2 i + 1]: the later candidates i suppresses), run by the 32
// lanes of one warp, which all return the kept mask: the lowest live candidate is kept and its row cleared from the live set, until
// `room` are kept.  Two 32-bit halves keep the dependent chain short (find-first-set, one shared load, one logic op per kept
// candidate); a row's upper half is applied to the upper live bits off the chain.
__device__ __forceinline__ unsigned long long resolve_chunk(unsigned long long alive, const unsigned int* cmask, int room) {
    unsigned int lo = (unsigned int)alive, hi = (unsigned int)(alive >> 32), klo = 0u, khi = 0u;
    while (lo && room > 0) {
        const int i = __ffs((int)lo) - 1;
        klo |= 1u << i;
        --room;
        lo &= ~(1u << i) & ~cmask[2 * i];
        hi &= ~cmask[2 * i + 1];
    }
    while (hi && room > 0) {
        const int i = __ffs((int)hi) - 1;
        khi |= 1u << i;
        --room;
        hi &= ~(1u << i) & ~cmask[2 * (i + 32) + 1];
    }
    return ((unsigned long long)khi << 32) | klo;
}

// Blocked greedy suppression over `cnt` keys sorted descending, keeping at most `cap`; returns the number kept.  Chunk by chunk of
// kChunk sorted candidates: (a) the chunk against every box kept so far, four threads per candidate, each testing every fourth
// kept box -> dead bits; (b) pairs inside the chunk among the survivors of (a), a thread per earlier candidate and 16 later ones
// -> kill rows; (c) resolve_chunk by warp 0; (d) append.  The policy `p` holds what differs between callers:
//   p.stage(j, key)        candidate j of the chunk (its sort key: `key`) into the chunk arrays
//   p.cand(j)              what the pair tests need of chunk candidate j, loaded into registers once before its pairs
//   p.kept_other_source(i, c), p.kept_same_class(i, c), p.kept_kills(i, c)
//                          kept box i suppresses chunk candidate c (as p.cand returned it) iff all three hold
//   p.other_source(c, j), p.same_class(c, j), p.kills(c, j)
//                          chunk candidate c suppresses the later chunk candidate j iff all three hold
//   p.append(pos, j, key)  chunk candidate j is kept box `pos`
// Each test is one comparison, so that the && chain is the branch condition itself: a && inside one method leaves a bool that is
// rebuilt and tested again in the pair loops (nvcc 12.9), which made the merge 1 % slower.
// `cmask`: 2 kChunk words of shared memory, `flags`: 4 (dead bits, then kept bits).  All threads of the CTA call this; it ends
// on a barrier.  (The NMS, sort_and_suppress, runs its own tuned version of these phases.)
template <class P>
__device__ __forceinline__ int greedy_pass(const unsigned long long* keys, int cnt, int cap, unsigned int* cmask, unsigned int* flags,
                                           const P& p) {
    const int t = threadIdx.x;
    int nk = 0;
    for (int c0 = 0; c0 < cnt && nk < cap; c0 += kChunk) {
        const int cn = min(kChunk, cnt - c0);
        if (t < cn) p.stage(t, keys[c0 + t]);
        if (t < 2 * kChunk) cmask[t] = 0u;
        if (t == 0) { flags[0] = 0u; flags[1] = 0u; }
        __syncthreads();
        {   // (a)
            const int j = t & (kChunk - 1), q = t / kChunk;
            if (j < cn) {
                const auto c = p.cand(j);
                bool dead = false;
                for (int i = q; i < nk && !dead; i += NT / kChunk) dead = p.kept_other_source(i, c) && p.kept_same_class(i, c) && p.kept_kills(i, c);
                if (dead) atomicOr(&flags[j >> 5], 1u << (j & 31));
            }
        }
        __syncthreads();
        unsigned long long alive = ~(((unsigned long long)flags[1] << 32) | flags[0]);
        if (cn < kChunk) alive &= (1ull << cn) - 1ull;
        {   // (b)
            const int i = t >> 2, jq = t & 3;
            if ((alive >> i) & 1ull) {
                const auto c = p.cand(i);
                unsigned int bits = 0u;
                // two pairs per trip: fully unrolled, the merge kernel takes 122 registers instead of 64 (the deploy post-process 103);
                // rolled, the merge is 2 % slower
#pragma unroll 2
                for (int e = 0; e < 16; ++e) {
                    const int j = jq * 16 + e;
                    if (j > i && ((alive >> j) & 1ull) && p.other_source(c, j) && p.same_class(c, j) && p.kills(c, j))
                        bits |= 1u << e;
                }
                if (bits) atomicOr(&cmask[2 * i + (jq >> 1)], bits << ((jq & 1) * 16));
            }
        }
        __syncthreads();
        if (t < 32) {   // (c)
            const unsigned long long kept = resolve_chunk(alive, cmask, cap - nk);
            if (t == 0) { flags[2] = (unsigned int)kept; flags[3] = (unsigned int)(kept >> 32); }
        }
        __syncthreads();
        const unsigned long long kept = ((unsigned long long)flags[3] << 32) | flags[2];
        if (t < cn && ((kept >> t) & 1ull)) p.append(nk + __popcll(kept & ((1ull << t) - 1ull)), t, keys[c0 + t]);   // (d)
        nk += __popcll(kept);
        __syncthreads();
    }
    return nk;
}

}  // namespace
}  // namespace yfv2
