// Anchor k-means on the device: the reference's genanchors.py (kmeans, IOU, avg_IOU; :17-102), bit-identical iteration by
// iteration, for R runs at once (seeded restarts).  One yfv2_anchor_kmeans_step advances every active run by one iteration with
// two launches:
//   assign  one thread per (box, run): the argmin of 1 - IOU over the run's centroids (anchors.cuh), written over the previous
//           iteration's assignment; a block that changed any raises the run's flag.
//   update  one CTA per run, one warp per cluster: the fp64 sums of the members' w and h in increasing box index, added one
//           after another (centroid_sums[a[i]] += X[i]), and the member count.  Per step the warp reads 128 assignments,
//           stages the members' boxes in shared memory in box order (ballot + prefix count), loads the next step's
//           assignments, and lane 0 adds the staged values: the sum is one dependent chain, as the reference's loop is, and
//           only the fp64 adds are on it.  A reordered or tree sum would change a centroid's last bits and, through ties,
//           later assignments.  Thread 0 then ends the run (converged: no assignment changed; NOT_CONVERGED:
//           max_iter reached; EMPTY_CLUSTER: a cluster without members, where the reference divides 0 by 0 and never stops)
//           or commits sum / count as the next iteration's centroids.
// The chains are serial by nature: one iteration costs about the longest cluster's member count of dependent adds, and R runs
// cost about the same as one while their R x k warps fit on the SMs.
#include "common.cuh"
#include "anchors.cuh"

namespace yfv2 {
namespace {

using anchors::kMaxK;
constexpr int kAssignThreads = 256;
constexpr int kUpdateGroups = 4;    // 32-box groups a cluster's warp stages per step
constexpr int kAvgThreads = 256;    // boxes of avg_IOU per chunk

__global__ void __launch_bounds__(kAssignThreads)
anchor_assign_kernel(const double* __restrict__ boxes, int N, int k, const double* __restrict__ centroids, int* __restrict__ assignments,
                     const int* __restrict__ status, int* __restrict__ changed) {
    const int r = blockIdx.y;
    if (status[r] != YFV2_ANCHOR_ACTIVE) return;
    __shared__ double c[2 * kMaxK];
    if (threadIdx.x < 2 * k) c[threadIdx.x] = centroids[(size_t)r * 2 * k + threadIdx.x];
    __syncthreads();
    const long long i = (long long)blockIdx.x * kAssignThreads + threadIdx.x;
    bool diff = false;
    if (i < N) {
        const int a = anchors::assign(boxes[2 * i], boxes[2 * i + 1], c, k);
        int* p = assignments + (size_t)r * N + i;
        diff = *p != a;
        if (diff) *p = a;
    }
    if (__syncthreads_or(diff) && threadIdx.x == 0) changed[r] = 1;
}

__global__ void __launch_bounds__(32 * kMaxK)
anchor_update_kernel(const double* __restrict__ boxes, int N, int k, int max_iter, double* __restrict__ centroids,
                     const int* __restrict__ assignments, int* __restrict__ iterations, int* __restrict__ status, int* __restrict__ changed,
                     int* __restrict__ active) {
    const int r = blockIdx.x;
    if (status[r] != YFV2_ANCHOR_ACTIVE) return;
    __shared__ double next[2 * kMaxK];
    __shared__ int count[kMaxK];
    __shared__ double stage[kMaxK][2][32 * kUpdateGroups];
    __shared__ int commit;
    const bool moved = changed[r] != 0;
    const int j = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (moved) {
        const int* a_run = assignments + (size_t)r * N;
        double* sw_buf = stage[j][0];
        double* sh_buf = stage[j][1];
        double sw = 0.0, sh = 0.0;
        int cnt = 0, a[kUpdateGroups];
#pragma unroll
        for (int u = 0; u < kUpdateGroups; ++u) a[u] = 32 * u + lane < N ? a_run[32 * u + lane] : -1;
        for (long long base = 0; base < N; base += 32 * kUpdateGroups) {
            int n = 0;                                               // members of this step, staged in box order
#pragma unroll
            for (int u = 0; u < kUpdateGroups; ++u) {
                const unsigned m = __ballot_sync(0xffffffffu, a[u] == j);
                if (a[u] == j) {
                    const long long i = base + 32 * u + lane;
                    const int q = n + __popc(m & ((1u << lane) - 1u));
                    sw_buf[q] = boxes[2 * i];
                    sh_buf[q] = boxes[2 * i + 1];
                }
                n += __popc(m);
            }
            const long long ahead = base + 32 * kUpdateGroups;       // the next step's assignments load during the adds
#pragma unroll
            for (int u = 0; u < kUpdateGroups; ++u) a[u] = ahead + 32 * u + lane < N ? a_run[ahead + 32 * u + lane] : -1;
            __syncwarp();
            if (lane == 0)
                for (int q = 0; q < n; ++q) {
                    sw = anchors::add(sw, sw_buf[q]);
                    sh = anchors::add(sh, sh_buf[q]);
                }
            cnt += n;
            __syncwarp();
        }
        if (lane == 0) {
            next[2 * j] = anchors::div(sw, (double)cnt);
            next[2 * j + 1] = anchors::div(sh, (double)cnt);
            count[j] = cnt;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int t = iterations[r] + 1;
        int st = YFV2_ANCHOR_ACTIVE;
        if (!moved) st = YFV2_ANCHOR_CONVERGED;
        else if (t >= max_iter) st = YFV2_ANCHOR_NOT_CONVERGED;
        else
            for (int q = 0; q < k; ++q)
                if (count[q] == 0) st = YFV2_ANCHOR_EMPTY_CLUSTER;
        iterations[r] = t;
        status[r] = st;
        changed[r] = 0;
        commit = st == YFV2_ANCHOR_ACTIVE;
        if (commit) atomicAdd(active, 1);
    }
    __syncthreads();
    if (commit && threadIdx.x < 2 * k) centroids[(size_t)r * 2 * k + threadIdx.x] = next[threadIdx.x];
}

// avg_IOU (genanchors.py:34-40): per box the builtin max of its similarities, summed in box order from 0.0 by one chain, over N.
// One CTA per run: every thread computes one box's maximum of a 256-box chunk into one of two buffers while thread 0 adds the
// previous chunk; one barrier per chunk keeps a buffer from being rewritten before thread 0 has added it.
__global__ void __launch_bounds__(kAvgThreads)
anchor_avg_iou_kernel(const double* __restrict__ boxes, int N, int k, const double* __restrict__ centroids, double* __restrict__ out) {
    const int r = blockIdx.x;
    __shared__ double c[2 * kMaxK];
    __shared__ double stage[2][kAvgThreads];
    if (threadIdx.x < 2 * k) c[threadIdx.x] = centroids[(size_t)r * 2 * k + threadIdx.x];
    __syncthreads();
    double acc = 0.0;
    int buf = 0;
    for (long long base = 0; base < N; base += kAvgThreads, buf ^= 1) {
        const long long i = base + threadIdx.x;
        if (i < N) stage[buf][threadIdx.x] = anchors::best_similarity(boxes[2 * i], boxes[2 * i + 1], c, k);
        __syncthreads();
        if (threadIdx.x == 0) {
            const int n = (int)min((long long)kAvgThreads, N - base);
            for (int q = 0; q < n; ++q) acc = anchors::add(acc, stage[buf][q]);
        }
    }
    if (threadIdx.x == 0) out[r] = anchors::div(acc, (double)N);
}

int check_args(const char* what, const void* boxes, int N, int k, int R, const void* centroids) {
    if (!boxes || !centroids || N <= 0 || R <= 0 || k <= 0) {
        set_error("%s: bad argument (boxes %p, centroids %p, N %d, k %d, R %d)", what, boxes, centroids, N, k, R);
        return YFV2_EINVAL;
    }
    if (R > 65535) { set_error("%s: R = %d runs in one batch (limit 65535)", what, R); return YFV2_EINVAL; }
    if (k > kMaxK) { set_error("%s: k = %d clusters (limit %d)", what, k, kMaxK); return YFV2_EUNSUPPORTED; }
    return YFV2_OK;
}

}  // namespace
}  // namespace yfv2

extern "C" int yfv2_anchor_kmeans_step(const double* boxes, int N, int k, int R, int max_iter, double* centroids, int* assignments,
                                       int* iterations, int* status, int* changed, int* active, void* stream) {
    using namespace yfv2;
    if (int rc = check_args("anchor_kmeans_step", boxes, N, k, R, centroids)) return rc;
    if (!assignments || !iterations || !status || !changed || !active || max_iter < 1) {
        set_error("anchor_kmeans_step: bad argument (a null state array, or max_iter %d < 1)", max_iter);
        return YFV2_EINVAL;
    }
    const cudaStream_t s = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemsetAsync(active, 0, sizeof(int), s));
    const dim3 grid((unsigned)((N + kAssignThreads - 1) / kAssignThreads), (unsigned)R);
    anchor_assign_kernel<<<grid, kAssignThreads, 0, s>>>(boxes, N, k, centroids, assignments, status, changed);
    YFV2_LAUNCH_CHECK();
    anchor_update_kernel<<<R, 32 * k, 0, s>>>(boxes, N, k, max_iter, centroids, assignments, iterations, status, changed, active);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_anchor_avg_iou(const double* boxes, int N, int k, int R, const double* centroids, double* avg_iou, void* stream) {
    using namespace yfv2;
    if (int rc = check_args("anchor_avg_iou", boxes, N, k, R, centroids)) return rc;
    if (!avg_iou) { set_error("anchor_avg_iou: bad argument (avg_iou is null)"); return YFV2_EINVAL; }
    anchor_avg_iou_kernel<<<R, kAvgThreads, 0, (cudaStream_t)stream>>>(boxes, N, k, centroids, avg_iou);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}
