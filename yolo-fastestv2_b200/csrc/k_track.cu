// Multi-object tracking across video frames (yfv2_track_*): ByteTrack's three-stage association and track lifecycle with a
// constant-velocity Kalman filter, for S streams kept in one caller-owned device buffer.  One update call runs ONE launch with
// one CTA per stream of the call; the contract is stated in include/yfv2.h and restated by tests/track_oracle.py.
//
// Every fp64 operation is an explicit __d*_rn intrinsic: nvcc would otherwise contract a*b + c into DFMA, and the oracle rounds
// each product and sum on its own.
//
// Memory: a stream's state is a header (frame, next id, live count), the slots of its live tracks in ascending id (`ord`) and K
// yfv2_track slots, all in global memory.  A CTA keeps in shared memory what its loops touch many times: the boxes of its tracks
// and detections, the confidences, the solver's per-row / per-column arrays and the index lists of each stage; the Kalman state
// of a track is read and written in global memory by the one thread that owns the track.
//
// Counting (yfv2_count_*) lives here too, because it reads this layout: one CTA per stream walks the tracker's `ord` and counts
// line crossings and zone entries, exits and occupancy of the tracks' anchors (tests/count_oracle.py restates it).
#include <float.h>
#include <limits.h>
#include <math.h>

#include <algorithm>
#include <memory>
#include <new>
#include <vector>

#include "common.cuh"

namespace yfv2 {
namespace {

constexpr int NT = 128;                         // threads per CTA
constexpr int NW = NT / 32;
constexpr int kTrackLaunch = YFV2_TRACK_MAX_BATCH;
constexpr double kSigP = 1.0 / 20, kSigV = 1.0 / 160;
constexpr double k2SigP = 2 * kSigP, k10SigV = 10 * kSigV;
constexpr double kStage2Thr = 0.5, kStage3Thr = 0.7, kDupIou = 0.85;

// ---- state layout: per stream, at s * stride ---------------------------------------------------------------------------------
//   int hdr[4] = {frame, next_id, n, 0};  int ord[K] (16-byte rounded);  yfv2_track tracks[K]
__host__ __device__ inline size_t tracks_offset(int K) { return 16 + (((size_t)K * 4 + 15) & ~(size_t)15); }
__host__ __device__ inline size_t stream_stride(int K) {
    return (tracks_offset(K) + (size_t)K * sizeof(yfv2_track) + 255) & ~(size_t)255;
}

struct TrackArgs {
    unsigned char* state;
    size_t stride;
    int K, M;
    const double* dets;          // [B, M, 6]
    const int* counts;           // [B]
    double* out;                 // [B, K, 8]
    int* out_counts;             // [B]
    int* dropped;                // [B]
    yfv2_track_params p;
    int streams[kTrackLaunch];   // stream of CTA b
};

struct ResetArgs {
    unsigned char* state;
    size_t stride;
    int streams[kTrackLaunch];
};

// ---- shared memory of one CTA, sized from K and M -------------------------------------------------------------------------------
struct TrackSmem {
    double4* tbox;       // [K]  box of each track, by rank (position in ord)
    double4* dbox;       // [M]  detection boxes, by input row
    double* dconf;       // [M]
    double* shortest;    // [L]  solver, per column (L = max(K, M))
    double* v;           // [L]
    double* u;           // [R]  solver, per row (R = min(K, M))
    short* path;         // [L]
    short* row4col;      // [L]
    short* col4row;      // [R]
    short* sr;           // [R]  rows visited by the current augmenting path
    short* rt;           // [K]  tracks (ranks) of the reduced problem
    short* rd;           // [M]  detections (rows) of the reduced problem
    short* ord;          // [K]  slot of each rank
    short* ord2;         // [K]
    short* tm;           // [K]  detection row matched to each rank, -1
    short* rows;         // [K]  a stage's tracks (ranks)
    short* lst;          // [K]  lost tracks for the duplicate rule
    short* freel;        // [K]  free slots
    short* hi;           // [M]  high detections (rows)
    short* lo;           // [M]  low detections
    short* dm;           // [M]  rank matched to each detection row, -1
    short* cols;         // [M]  a stage's detections; the births
    unsigned char* sc;   // [L]  column visited by the current path
    unsigned char* tkind;   // [K]  0 tentative, 1 confirmed tracked, 2 lost
    unsigned char* tflag;   // [K]
    unsigned char* gone;    // [K]
    unsigned char* dup;     // [K]
    unsigned char* used;    // [K]  by slot
    unsigned char* dkind;   // [M]  0 unused, 1 high, 2 low
    unsigned char* dflag;   // [M]
    double* redv;        // [2 * NW]
    int* redj;           // [2 * NW]
    int* scratch;        // [NW]
};

template <class T>
__host__ __device__ __forceinline__ T* take(unsigned char*& at, size_t n) {
    T* r = reinterpret_cast<T*>(at);
    at += (n * sizeof(T) + 15) & ~(size_t)15;
    return r;
}

__host__ __device__ inline unsigned char* track_layout(TrackSmem& s, unsigned char* base, int K, int M) {
    const int L = K > M ? K : M, R = K < M ? K : M;
    s.tbox = take<double4>(base, K);
    s.dbox = take<double4>(base, M);
    s.dconf = take<double>(base, M);
    s.shortest = take<double>(base, L);
    s.v = take<double>(base, L);
    s.u = take<double>(base, R);
    s.redv = take<double>(base, 2 * NW);
    s.redj = take<int>(base, 2 * NW);
    s.scratch = take<int>(base, NW);
    s.path = take<short>(base, L);
    s.row4col = take<short>(base, L);
    s.col4row = take<short>(base, R);
    s.sr = take<short>(base, R);
    s.rt = take<short>(base, K);
    s.rd = take<short>(base, M);
    s.ord = take<short>(base, K);
    s.ord2 = take<short>(base, K);
    s.tm = take<short>(base, K);
    s.rows = take<short>(base, K);
    s.lst = take<short>(base, K);
    s.freel = take<short>(base, K);
    s.hi = take<short>(base, M);
    s.lo = take<short>(base, M);
    s.dm = take<short>(base, M);
    s.cols = take<short>(base, M);
    s.sc = take<unsigned char>(base, L);
    s.tkind = take<unsigned char>(base, K);
    s.tflag = take<unsigned char>(base, K);
    s.gone = take<unsigned char>(base, K);
    s.dup = take<unsigned char>(base, K);
    s.used = take<unsigned char>(base, K);
    s.dkind = take<unsigned char>(base, M);
    s.dflag = take<unsigned char>(base, M);
    return base;
}

inline size_t track_smem_bytes(int K, int M) {
    TrackSmem s;
    return reinterpret_cast<size_t>(track_layout(s, nullptr, K, M));
}

// ---- arithmetic of the contract --------------------------------------------------------------------------------------------------
__device__ __forceinline__ double dmin(double a, double b) { return a < b ? a : b; }
__device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }
__device__ __forceinline__ double sq(double a) { return __dmul_rn(a, a); }

__device__ __forceinline__ double iou(const double4& a, const double4& b) {
    const double iw = dmax(0.0, __dsub_rn(dmin(a.z, b.z), dmax(a.x, b.x)));
    const double ih = dmax(0.0, __dsub_rn(dmin(a.w, b.w), dmax(a.y, b.y)));
    const double inter = __dmul_rn(iw, ih);
    const double aa = __dmul_rn(__dsub_rn(a.z, a.x), __dsub_rn(a.w, a.y));
    const double ab = __dmul_rn(__dsub_rn(b.z, b.x), __dsub_rn(b.w, b.y));
    return __ddiv_rn(inter, __dsub_rn(__dadd_rn(aa, ab), inter));
}

__device__ __forceinline__ double4 track_box(const double* m) {
    const double h = m[3], w = __dmul_rn(m[2], h);
    const double x1 = __dsub_rn(m[0], __ddiv_rn(w, 2.0)), y1 = __dsub_rn(m[1], __ddiv_rn(h, 2.0));
    return make_double4(x1, y1, __dadd_rn(x1, w), __dadd_rn(y1, h));
}

__device__ __forceinline__ void measure(const double4& d, double z[4]) {
    const double w = __dsub_rn(d.z, d.x), h = __dsub_rn(d.w, d.y);
    z[0] = __dadd_rn(d.x, __ddiv_rn(w, 2.0));
    z[1] = __dadd_rn(d.y, __ddiv_rn(h, 2.0));
    z[2] = __ddiv_rn(w, h);
    z[3] = h;
}

__device__ void kf_initiate(yfv2_track* tr, const double z[4]) {
    const double sp = __dmul_rn(k2SigP, z[3]), sv = __dmul_rn(k10SigV, z[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        tr->mean[k] = z[k];
        tr->mean[k + 4] = 0.0;
        tr->cov[3 * k] = sq(k == 2 ? 1e-2 : sp);
        tr->cov[3 * k + 1] = 0.0;
        tr->cov[3 * k + 2] = sq(k == 2 ? 1e-5 : sv);
    }
}

__device__ void kf_predict(yfv2_track* tr) {
    if (tr->state == YFV2_TRACK_LOST) tr->mean[7] = 0.0;
    const double h = tr->mean[3];
    const double qp = sq(__dmul_rn(kSigP, h)), qv = sq(__dmul_rn(kSigV, h));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        tr->mean[k] = __dadd_rn(tr->mean[k], tr->mean[k + 4]);
        const double p = tr->cov[3 * k], x = tr->cov[3 * k + 1], v = tr->cov[3 * k + 2];
        const double t = __dadd_rn(x, v);
        tr->cov[3 * k] = __dadd_rn(__dadd_rn(__dadd_rn(p, x), t), k == 2 ? sq(1e-2) : qp);
        tr->cov[3 * k + 1] = t;
        tr->cov[3 * k + 2] = __dadd_rn(v, k == 2 ? sq(1e-5) : qv);
    }
}

__device__ void kf_update(yfv2_track* tr, const double z[4]) {
    const double rp = sq(__dmul_rn(kSigP, tr->mean[3]));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double p = tr->cov[3 * k], x = tr->cov[3 * k + 1], v = tr->cov[3 * k + 2];
        const double s = __dadd_rn(p, k == 2 ? sq(1e-1) : rp);
        const double k0 = __ddiv_rn(p, s), k1 = __ddiv_rn(x, s);
        const double y = __dsub_rn(z[k], tr->mean[k]);
        tr->mean[k] = __dadd_rn(tr->mean[k], __dmul_rn(k0, y));
        tr->mean[k + 4] = __dadd_rn(tr->mean[k + 4], __dmul_rn(k1, y));
        tr->cov[3 * k] = __dsub_rn(p, __dmul_rn(k0, p));
        tr->cov[3 * k + 1] = __dsub_rn(x, __dmul_rn(k0, x));
        tr->cov[3 * k + 2] = __dsub_rn(v, __dmul_rn(k1, x));
    }
}

// ---- block helpers -------------------------------------------------------------------------------------------------------------
// The i in [0, n) with pred(i), in ascending order: emit(position, i).  Every thread calls it and gets the count.
template <class Pred, class Emit>
__device__ int block_select(int n, int* scratch, Pred pred, Emit emit) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int total = 0;
    for (int base = 0; base < n; base += NT) {
        const int i = base + t;
        const bool p = i < n && pred(i);
        const unsigned int bal = __ballot_sync(0xffffffffu, p);
        if (lane == 0) scratch[warp] = __popc(bal);
        __syncthreads();
        int off = total, chunk = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
            const int c = scratch[w];
            off += w < warp ? c : 0;
            chunk += c;
        }
        if (p) emit(off + __popc(bal & ((1u << lane) - 1u)), i);
        total += chunk;
        __syncthreads();
    }
    return total;
}

__device__ __forceinline__ bool lex_less(double a, int ja, double b, int jb) { return a < b || (a == b && ja < jb); }

// c of track rank tk and detection row dj: 1 - IoU, or 1 - IoU * conf when fused
__device__ __forceinline__ double pair_cost(const TrackSmem& s, int tk, int dj, bool fused) {
    const double i = iou(s.tbox[tk], s.dbox[dj]);
    return __dsub_rn(1.0, fused ? __dmul_rn(i, s.dconf[dj]) : i);
}

// One association stage: tracks rows[0, nt) (ranks, ascending id) against detections cols[0, nd) (rows, ascending).  Matches are
// recorded in s.tm (by rank) and s.dm (by detection row).  Columns of the solver are owned by thread j % NT: shortest, path, sc
// and v of a column are touched only by its owner while a path grows, so each step of a path costs one barrier (the argmin).
//
// The argmin starts from (+inf, INT_MAX) and takes only a strictly smaller shortest[j], so it needs a column below +inf at every
// step.  There always is one, whatever the duals do: when row cur starts, u[cur] is 0 (only rows already processed change their
// u) and so is v[j] of every unassigned column (only columns in SC change their v, and they all end assigned), so the first
// sweep sets shortest[j] = C(cur, j) for each of the ncol - cur >= 1 unassigned columns; C is c - thr < 0 or 0, never +inf
// (c = -inf, from a confidence near DBL_MAX, gives -inf); and no unassigned column enters SC before the one that ends the path.
// shortest[j] is never NaN (NaN < x is false).  So with huge confidences the duals may reach +-inf or NaN and change which
// optimum is found, but bj is always a real column and the rule of yfv2.h fixes it; tests/track_oracle.py raises if a step ever
// found none.
__device__ void associate(TrackSmem& s, const short* rows, int nt, const short* cols, int nd, bool fused, double thr) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (nt == 0 || nd == 0) return;
    for (int k = t; k < nt; k += NT) s.tflag[k] = 0;
    for (int q = t; q < nd; q += NT) s.dflag[q] = 0;
    __syncthreads();
    for (int pq = t; pq < nt * nd; pq += NT) {
        const int k = pq / nd, q = pq - k * nd;
        if (pair_cost(s, rows[k], cols[q], fused) < thr) { s.tflag[k] = 1; s.dflag[q] = 1; }
    }
    __syncthreads();
    const int ntr = block_select(nt, s.scratch, [&](int k) { return s.tflag[k] != 0; }, [&](int pos, int k) { s.rt[pos] = rows[k]; });
    const int ndr = block_select(nd, s.scratch, [&](int q) { return s.dflag[q] != 0; }, [&](int pos, int q) { s.rd[pos] = cols[q]; });
    if (ntr == 0) return;
    const bool tr = ntr > ndr;                       // the detections play the rows
    const int nrow = tr ? ndr : ntr, ncol = tr ? ntr : ndr;
    const short* rowl = tr ? s.rd : s.rt;
    const short* coll = tr ? s.rt : s.rd;
    auto C = [&](int i, int j) {
        const int tk = tr ? coll[j] : rowl[i], dj = tr ? rowl[i] : coll[j];
        const double c = pair_cost(s, tk, dj, fused);
        return c < thr ? __dsub_rn(c, thr) : 0.0;
    };
    for (int i = t; i < nrow; i += NT) { s.u[i] = 0.0; s.col4row[i] = -1; }
    for (int j = t; j < ncol; j += NT) { s.v[j] = 0.0; s.row4col[j] = -1; }
    __syncthreads();
    int par = 0;
    for (int cur = 0; cur < nrow; ++cur) {
        for (int j = t; j < ncol; j += NT) { s.shortest[j] = __longlong_as_double(0x7ff0000000000000ll); s.path[j] = -1; s.sc[j] = 0; }
        int i = cur, sink = -1, nsr = 0;
        double minVal = 0.0;
        while (sink < 0) {
            if (t == 0) s.sr[nsr] = (short)i;
            ++nsr;
            const double ui = s.u[i];
            double bv = __longlong_as_double(0x7ff0000000000000ll);
            int bj = INT_MAX;
            for (int j = t; j < ncol; j += NT) {
                if (s.sc[j]) continue;
                const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, C(i, j)), ui), s.v[j]);
                double sh = s.shortest[j];
                if (r < sh) { sh = r; s.shortest[j] = r; s.path[j] = (short)i; }
                if (sh < bv) { bv = sh; bj = j; }
            }
#pragma unroll
            for (int off = 16; off; off >>= 1) {
                const double ov = __shfl_down_sync(0xffffffffu, bv, off);
                const int oj = __shfl_down_sync(0xffffffffu, bj, off);
                if (lex_less(ov, oj, bv, bj)) { bv = ov; bj = oj; }
            }
            if (lane == 0) { s.redv[par * NW + warp] = bv; s.redj[par * NW + warp] = bj; }
            __syncthreads();
            bv = s.redv[par * NW];
            bj = s.redj[par * NW];
#pragma unroll
            for (int w = 1; w < NW; ++w)
                if (lex_less(s.redv[par * NW + w], s.redj[par * NW + w], bv, bj)) { bv = s.redv[par * NW + w]; bj = s.redj[par * NW + w]; }
            par ^= 1;
            minVal = bv;
            if (bj % NT == t) s.sc[bj] = 1;
            const int r4c = s.row4col[bj];
            if (r4c < 0) sink = bj; else i = r4c;
        }
        __syncthreads();
        if (t == 0) s.u[cur] = __dadd_rn(s.u[cur], minVal);
        for (int k = t; k < nsr; k += NT) {
            const int ii = s.sr[k];
            if (ii != cur) s.u[ii] = __dadd_rn(s.u[ii], __dsub_rn(minVal, s.shortest[s.col4row[ii]]));
        }
        for (int j = t; j < ncol; j += NT)
            if (s.sc[j]) s.v[j] = __dsub_rn(s.v[j], __dsub_rn(minVal, s.shortest[j]));
        __syncthreads();
        if (t == 0) {
            int j = sink;
            for (;;) {
                const int ii = s.path[j];
                s.row4col[j] = (short)ii;
                const int tmp = s.col4row[ii];
                s.col4row[ii] = (short)j;
                j = tmp;
                if (ii == cur) break;
            }
        }
        __syncthreads();
    }
    for (int i = t; i < nrow; i += NT) {
        const int j = s.col4row[i];
        const int tk = tr ? coll[j] : rowl[i], dj = tr ? rowl[i] : coll[j];
        if (pair_cost(s, tk, dj, fused) < thr) { s.tm[tk] = (short)dj; s.dm[dj] = (short)tk; }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(NT)
track_update_kernel(const __grid_constant__ TrackArgs a) {
    extern __shared__ __align__(16) unsigned char smraw[];
    TrackSmem s;
    track_layout(s, smraw, a.K, a.M);
    const int t = threadIdx.x, b = blockIdx.x, K = a.K, M = a.M;
    unsigned char* base = a.state + (size_t)a.streams[b] * a.stride;
    int* hdr = reinterpret_cast<int*>(base);
    int* gord = hdr + 4;
    yfv2_track* tracks = reinterpret_cast<yfv2_track*>(base + tracks_offset(K));
    const int frame = hdr[0] + 1, next_id = hdr[1], n = hdr[2];
    const yfv2_track_params& P = a.p;

    // detections: validity and group, boxes and confidences in shared memory
    const int cnt = min(max(a.counts[b], 0), M);
    const double* drow = a.dets + (size_t)b * M * 6;
    for (int j = t; j < cnt; j += NT) {
        const double* r = drow + (size_t)j * 6;
        const double x1 = r[0], y1 = r[1], x2 = r[2], y2 = r[3], conf = r[4], cls = r[5];
        const bool ok = isfinite(x1) && isfinite(y1) && isfinite(x2) && isfinite(y2) && isfinite(conf) && isfinite(cls) && x2 > x1 &&
                        y2 > y1 && conf > P.low_thresh;
        s.dkind[j] = ok ? (conf > P.high_thresh ? 1 : 2) : 0;
        s.dbox[j] = make_double4(x1, y1, x2, y2);
        s.dconf[j] = conf;
        s.dm[j] = -1;
    }
    // predict every live track
    for (int k = t; k < n; k += NT) {
        const int slot = gord[k];
        s.ord[k] = (short)slot;
        yfv2_track* tr = tracks + slot;
        kf_predict(tr);
        s.tbox[k] = track_box(tr->mean);
        s.tm[k] = -1;
        s.tkind[k] = tr->state == YFV2_TRACK_LOST ? 2 : (tr->confirmed ? 1 : 0);
    }
    __syncthreads();
    const int nh = block_select(cnt, s.scratch, [&](int j) { return s.dkind[j] == 1; }, [&](int pos, int j) { s.hi[pos] = (short)j; });
    const int nl = block_select(cnt, s.scratch, [&](int j) { return s.dkind[j] == 2; }, [&](int pos, int j) { s.lo[pos] = (short)j; });

    // stage 1: confirmed tracks (tracked or lost) x high detections
    int nr = block_select(n, s.scratch, [&](int k) { return s.tkind[k] != 0; }, [&](int pos, int k) { s.rows[pos] = (short)k; });
    associate(s, s.rows, nr, s.hi, nh, true, P.match_thresh);
    // stage 2: confirmed tracked tracks left unmatched x low detections
    nr = block_select(n, s.scratch, [&](int k) { return s.tkind[k] == 1 && s.tm[k] < 0; }, [&](int pos, int k) { s.rows[pos] = (short)k; });
    associate(s, s.rows, nr, s.lo, nl, false, kStage2Thr);
    // stage 3: tentative tracks x high detections still unmatched
    nr = block_select(n, s.scratch, [&](int k) { return s.tkind[k] == 0; }, [&](int pos, int k) { s.rows[pos] = (short)k; });
    const int nc = block_select(nh, s.scratch, [&](int q) { return s.dm[s.hi[q]] < 0; }, [&](int pos, int q) { s.cols[pos] = s.hi[q]; });
    associate(s, s.rows, nr, s.cols, nc, true, kStage3Thr);

    // matched tracks take their detection; unmatched confirmed tracked ones are lost; unmatched tentative ones go
    for (int k = t; k < n; k += NT) {
        yfv2_track* tr = tracks + s.ord[k];
        const int j = s.tm[k];
        s.gone[k] = 0;
        if (j >= 0) {
            double z[4];
            measure(s.dbox[j], z);
            kf_update(tr, z);
            tr->state = YFV2_TRACK_TRACKED;
            tr->confirmed = 1;
            tr->score = s.dconf[j];
            tr->cls = drow[(size_t)j * 6 + 5];
            tr->end_frame = frame;
            tr->det_row = j;
        } else if (s.tkind[k] == 1) {
            tr->state = YFV2_TRACK_LOST;
        } else if (s.tkind[k] == 0) {
            s.gone[k] = 1;
        }
    }
    for (int q = t; q < K; q += NT) s.used[q] = 0;
    __syncthreads();
    const int n1 = block_select(n, s.scratch, [&](int k) { return !s.gone[k]; }, [&](int pos, int k) { s.ord2[pos] = s.ord[k]; });
    for (int k = t; k < n1; k += NT) s.used[s.ord2[k]] = 1;
    __syncthreads();

    // births, in row order, into the lowest free slots
    block_select(K, s.scratch, [&](int q) { return !s.used[q]; }, [&](int pos, int q) { s.freel[pos] = (short)q; });
    const int nb = block_select(nh, s.scratch, [&](int q) { const int j = s.hi[q]; return s.dm[j] < 0 && s.dconf[j] >= P.new_thresh; },
                                [&](int pos, int q) { s.cols[pos] = s.hi[q]; });
    const int born = min(nb, K - n1);
    for (int q = t; q < born; q += NT) {
        const int j = s.cols[q], slot = s.freel[q];
        yfv2_track* tr = tracks + slot;
        double z[4];
        measure(s.dbox[j], z);
        kf_initiate(tr, z);
        tr->score = s.dconf[j];
        tr->cls = drow[(size_t)j * 6 + 5];
        tr->id = next_id + q;
        tr->state = YFV2_TRACK_TRACKED;
        tr->confirmed = frame == 1;
        tr->start_frame = frame;
        tr->end_frame = frame;
        tr->det_row = j;
        s.ord2[n1 + q] = (short)slot;
    }
    const int n2 = n1 + born;
    __syncthreads();

    // lost tracks past max_age go; then the duplicate rule, judged on the boxes of the updated means
    for (int k = t; k < n2; k += NT) {
        const yfv2_track* tr = tracks + s.ord2[k];
        s.tbox[k] = track_box(tr->mean);
        const bool lost = tr->state == YFV2_TRACK_LOST;
        s.tkind[k] = lost ? 2 : 1;
        s.gone[k] = lost && frame - tr->end_frame > P.max_age;
        s.dup[k] = 0;
    }
    __syncthreads();
    const int ntk = block_select(n2, s.scratch, [&](int k) { return s.tkind[k] == 1; }, [&](int pos, int k) { s.rows[pos] = (short)k; });
    const int nlo = block_select(n2, s.scratch, [&](int k) { return s.tkind[k] == 2 && !s.gone[k]; }, [&](int pos, int k) { s.lst[pos] = (short)k; });
    for (int pq = t; pq < ntk * nlo; pq += NT) {
        const int p = s.rows[pq / nlo], q = s.lst[pq % nlo];
        if (iou(s.tbox[p], s.tbox[q]) > kDupIou) {
            const int ap = frame - tracks[s.ord2[p]].start_frame, aq = frame - tracks[s.ord2[q]].start_frame;
            if (ap > aq) s.dup[q] = 1; else s.dup[p] = 1;
        }
    }
    __syncthreads();
    const int n3 = block_select(n2, s.scratch, [&](int k) { return !s.gone[k] && !s.dup[k]; }, [&](int pos, int k) { s.ord[pos] = s.ord2[k]; });

    // output: confirmed tracked tracks in ascending id
    double* out = a.out + (size_t)b * K * 8;
    const int no = block_select(n3, s.scratch, [&](int k) { const yfv2_track* tr = tracks + s.ord[k]; return tr->state == YFV2_TRACK_TRACKED && tr->confirmed; },
                                [&](int pos, int k) {
                                    const yfv2_track* tr = tracks + s.ord[k];
                                    const double4 bx = track_box(tr->mean);
                                    double* o = out + (size_t)pos * 8;
                                    o[0] = bx.x; o[1] = bx.y; o[2] = bx.z; o[3] = bx.w;
                                    o[4] = tr->score; o[5] = tr->cls; o[6] = (double)tr->id; o[7] = (double)tr->det_row;
                                });
    for (int e = no * 8 + t; e < K * 8; e += NT) out[e] = 0.0;
    for (int k = t; k < n3; k += NT) gord[k] = s.ord[k];
    if (t == 0) {
        hdr[0] = frame;
        hdr[1] = next_id + born;
        hdr[2] = n3;
        a.out_counts[b] = no;
        a.dropped[b] = nb - born;
    }
}

__global__ void track_reset_kernel(const __grid_constant__ ResetArgs a) {
    int* hdr = reinterpret_cast<int*>(a.state + (size_t)a.streams[blockIdx.x] * a.stride);
    if (threadIdx.x == 0) { hdr[0] = 0; hdr[1] = 1; hdr[2] = 0; hdr[3] = 0; }
}

int check_streams(const char* what, int S, int K, const int* streams, int B, std::vector<unsigned char>& seen) {
    if (S < 1 || K < 1 || K > YFV2_TRACK_MAX_CAPACITY) {
        set_error("%s: need S >= 1 and capacity K in 1..%d (S=%d K=%d)", what, YFV2_TRACK_MAX_CAPACITY, S, K);
        return YFV2_EINVAL;
    }
    if (B < 1 || B > S || B > kTrackLaunch) {
        set_error("%s: B=%d streams in the call: need 1 <= B <= min(S=%d, %d)", what, B, S, kTrackLaunch);
        return YFV2_EINVAL;
    }
    seen.assign((size_t)S, 0);
    for (int b = 0; b < B; ++b) {
        const int s = streams[b];
        if (s < 0 || s >= S) { set_error("%s: streams[%d]=%d outside [0, S=%d)", what, b, s, S); return YFV2_EINVAL; }
        if (seen[s]) { set_error("%s: streams[%d]=%d appears twice in the call", what, b, s); return YFV2_EINVAL; }
        seen[s] = 1;
    }
    return YFV2_OK;
}

// ---- line and zone counting (yfv2_count_*): reads the tracker state above, one CTA per stream ---------------------------------
// Counter state, per stream at s * stride:  int hdr[4] = {nl, nz, 0, 0};  long long totals[2L + 2Z];  double4 lines[L];
// int nverts[Z];  float2 verts[Z][P];  then the records of the K slots: int id[K];  unsigned inside[K];  double2 anchor[K];
// signed char side[K][L].
constexpr int kMaxLines = YFV2_COUNT_MAX_LINES, kMaxZones = YFV2_COUNT_MAX_ZONES, kMaxVerts = YFV2_COUNT_MAX_VERTICES;

struct CountLayout {
    size_t totals, lines, nverts, verts, rid, rin, rpos, rside, stride;
};

__host__ __device__ inline size_t up16(size_t v) { return (v + 15) & ~(size_t)15; }

inline CountLayout count_layout(int K, int L, int Z, int P) {
    CountLayout c;
    c.totals = 16;
    c.lines = c.totals + up16((size_t)(2 * L + 2 * Z) * sizeof(long long));
    c.nverts = c.lines + (size_t)L * sizeof(double4);
    c.verts = c.nverts + up16((size_t)Z * sizeof(int));
    c.rid = c.verts + up16((size_t)Z * P * sizeof(float2));
    c.rin = c.rid + up16((size_t)K * sizeof(int));
    c.rpos = c.rin + up16((size_t)K * sizeof(unsigned));
    c.rside = c.rpos + (size_t)K * sizeof(double2);
    c.stride = (c.rside + (size_t)K * L + 255) & ~(size_t)255;
    return c;
}

struct CountArgs {
    const unsigned char* track;
    unsigned char* count;
    size_t track_stride;
    CountLayout lay;
    int K, L, Z, P, E;
    double* events;              // [B, E, 8]
    int* event_counts;           // [B]
    int* occupancy;              // [B, Z]
    int streams[kTrackLaunch];
};

struct CountResetArgs {
    unsigned char* count;
    CountLayout lay;
    int K, L, Z;
    int streams[kTrackLaunch];
};

struct CountSmem {
    double4 lines[kMaxLines];
    float2 verts[kMaxZones * kMaxVerts];   // zone z's vertices from z * P on
    int nverts[kMaxZones];
    int occ[kMaxZones];
    int tot[2 * kMaxLines + 2 * kMaxZones];   // this call's events: per line dir +1, dir -1; per zone entries, exits
    int scratch[NW];
};

__device__ __forceinline__ double orient(double ax, double ay, double bx, double by, double px, double py) {
    return __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(py, ay)), __dmul_rn(__dsub_rn(by, ay), __dsub_rn(px, ax)));
}

__device__ __forceinline__ int sgn(double v) { return (v > 0.0) - (v < 0.0); }

// cv2.pointPolygonTest(contour, (x, y), false) >= 0 for a float32 contour of n vertices: the differences in float32, the products
// and their difference in fp64, as cv2 computes them
__device__ bool in_polygon(const float2* v, int n, float x, float y) {
    float2 b = v[n - 1];
    int crossings = 0;
    bool edge = false;
    for (int i = 0; i < n; ++i) {
        const float2 a = b;
        b = v[i];
        if ((a.y <= y && b.y <= y) || (a.y > y && b.y > y) || (a.x < x && b.x < x)) {
            if (y == b.y && (x == b.x || (y == a.y && ((a.x <= x && x <= b.x) || (b.x <= x && x <= a.x))))) edge = true;
            continue;
        }
        double dist = __dsub_rn(__dmul_rn((double)__fsub_rn(y, a.y), (double)__fsub_rn(b.x, a.x)),
                                __dmul_rn((double)__fsub_rn(x, a.x), (double)__fsub_rn(b.y, a.y)));
        if (dist == 0.0) edge = true;
        if (b.y < a.y) dist = -dist;
        crossings += dist > 0.0;
    }
    return edge || (crossings & 1);
}

// Exclusive prefix sum of v over the CTA; every thread calls it and gets the CTA's total.
__device__ int block_scan(int v, int* scratch, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, off);
        if (lane >= off) x += y;
    }
    if (lane == 31) scratch[warp] = x;
    __syncthreads();
    int before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
        const int c = scratch[w];
        before += w < warp ? c : 0;
        total += c;
    }
    __syncthreads();
    return before + x - v;
}

// One appearance of a track at anchor (qx, qy), in zones `qin`, against its record (fresh: none yet).  Without `write` the
// events are only counted; with it they are written to ev from position pos on (those below E), and this call's totals and the
// record's sides are updated.
__device__ int appear(CountSmem& s, int nl, int nz, bool fresh, double px, double py, double qx, double qy, signed char* side,
                      unsigned pin, unsigned qin, bool write, double* ev, int pos, int E, double id, double cls, double frame) {
    int cnt = 0;
    auto emit = [&](int kind, int index, int dir) {
        if (write && pos + cnt < E) {
            double* o = ev + (size_t)(pos + cnt) * 8;
            o[0] = kind; o[1] = index; o[2] = dir; o[3] = id; o[4] = cls; o[5] = qx; o[6] = qy; o[7] = frame;
        }
        ++cnt;
    };
    for (int l = 0; l < nl; ++l) {
        const double4 g = s.lines[l];
        const int sq = sgn(orient(g.x, g.y, g.z, g.w, qx, qy));
        const int stored = fresh ? 0 : side[l];
        if (stored != 0 && sq == -stored && sgn(orient(g.x, g.y, g.z, g.w, px, py)) * sq <= 0 &&
            sgn(orient(px, py, qx, qy, g.x, g.y)) * sgn(orient(px, py, qx, qy, g.z, g.w)) <= 0) {
            if (write) atomicAdd(&s.tot[2 * l + (sq > 0 ? 0 : 1)], 1);
            emit(YFV2_COUNT_LINE, l, sq);
        }
        if (write && (sq != 0 || fresh)) side[l] = (signed char)sq;
    }
    for (int z = 0; z < nz; ++z) {
        const unsigned bit = 1u << z;
        if (fresh || ((pin ^ qin) & bit) == 0) continue;
        const bool entry = (qin & bit) != 0;
        if (write) atomicAdd(&s.tot[2 * kMaxLines + 2 * z + (entry ? 0 : 1)], 1);
        emit(entry ? YFV2_COUNT_ENTRY : YFV2_COUNT_EXIT, z, entry ? 1 : -1);
    }
    return cnt;
}

__global__ void __launch_bounds__(NT)
count_update_kernel(const __grid_constant__ CountArgs a) {
    __shared__ CountSmem s;
    const int t = threadIdx.x, b = blockIdx.x, K = a.K, L = a.L, Z = a.Z, P = a.P, E = a.E;
    const CountLayout& c = a.lay;
    const unsigned char* tb = a.track + (size_t)a.streams[b] * a.track_stride;
    const int* thdr = reinterpret_cast<const int*>(tb);
    const int* gord = thdr + 4;
    const yfv2_track* tracks = reinterpret_cast<const yfv2_track*>(tb + tracks_offset(K));
    unsigned char* cb = a.count + (size_t)a.streams[b] * c.stride;
    const int* chdr = reinterpret_cast<const int*>(cb);
    long long* totals = reinterpret_cast<long long*>(cb + c.totals);
    int* rid = reinterpret_cast<int*>(cb + c.rid);
    unsigned* rin = reinterpret_cast<unsigned*>(cb + c.rin);
    double2* rpos = reinterpret_cast<double2*>(cb + c.rpos);
    signed char* rside = reinterpret_cast<signed char*>(cb + c.rside);
    const int frame = thdr[0], n = thdr[2], nl = chdr[0], nz = chdr[1];

    const double4* glines = reinterpret_cast<const double4*>(cb + c.lines);
    const int* gnv = reinterpret_cast<const int*>(cb + c.nverts);
    const float2* gverts = reinterpret_cast<const float2*>(cb + c.verts);
    for (int l = t; l < nl; l += NT) s.lines[l] = glines[l];
    for (int q = t; q < nz * P; q += NT) s.verts[q] = gverts[q];
    for (int z = t; z < kMaxZones; z += NT) { s.nverts[z] = z < nz ? gnv[z] : 0; s.occ[z] = 0; }
    for (int q = t; q < 2 * kMaxLines + 2 * kMaxZones; q += NT) s.tot[q] = 0;
    __syncthreads();

    // ranks of ord are in ascending id: one chunk of NT tracks at a time, the events of a chunk placed by a prefix sum
    double* ev = a.events + (size_t)b * E * 8;
    int base = 0;
    for (int k0 = 0; k0 < n; k0 += NT) {
        const int k = k0 + t;
        const int slot = k < n ? gord[k] : 0;
        const yfv2_track* tr = tracks + slot;
        const bool app = k < n && tr->state == YFV2_TRACK_TRACKED && tr->confirmed;
        int cnt = 0, pos = 0, chunk = 0;
        bool fresh = true;
        double qx = 0.0, qy = 0.0, px = 0.0, py = 0.0, id = 0.0, cls = 0.0;
        unsigned pin = 0, qin = 0;
        if (app) {
            const double4 bx = track_box(tr->mean);
            qx = __ddiv_rn(__dadd_rn(bx.x, bx.z), 2.0);
            qy = bx.w;
            const float fx = __double2float_rn(qx), fy = __double2float_rn(qy);
            for (int z = 0; z < nz; ++z)
                if (in_polygon(s.verts + z * P, s.nverts[z], fx, fy)) { qin |= 1u << z; atomicAdd(&s.occ[z], 1); }
            fresh = rid[slot] != tr->id;
            if (!fresh) { const double2 p = rpos[slot]; px = p.x; py = p.y; pin = rin[slot]; }
            id = (double)tr->id;
            cls = tr->cls;
            cnt = appear(s, nl, nz, fresh, px, py, qx, qy, rside + (size_t)slot * L, pin, qin, false, ev, 0, E, id, cls, frame);
        }
        pos = base + block_scan(cnt, s.scratch, chunk);
        if (app) {
            appear(s, nl, nz, fresh, px, py, qx, qy, rside + (size_t)slot * L, pin, qin, true, ev, pos, E, id, cls, frame);
            rid[slot] = tr->id;
            rin[slot] = qin;
            rpos[slot] = make_double2(qx, qy);
        }
        base += chunk;
    }
    __syncthreads();
    for (int e = min(base, E) * 8 + t; e < E * 8; e += NT) ev[e] = 0.0;
    for (int z = t; z < Z; z += NT) a.occupancy[(size_t)b * Z + z] = s.occ[z];
    for (int l = t; l < nl; l += NT) { totals[2 * l] += s.tot[2 * l]; totals[2 * l + 1] += s.tot[2 * l + 1]; }
    for (int z = t; z < nz; z += NT) {
        totals[2 * L + 2 * z] += s.tot[2 * kMaxLines + 2 * z];
        totals[2 * L + 2 * z + 1] += s.tot[2 * kMaxLines + 2 * z + 1];
    }
    if (t == 0) a.event_counts[b] = base;
}

__global__ void count_reset_kernel(const __grid_constant__ CountResetArgs a) {
    unsigned char* cb = a.count + (size_t)a.streams[blockIdx.x] * a.lay.stride;
    long long* totals = reinterpret_cast<long long*>(cb + a.lay.totals);
    int* rid = reinterpret_cast<int*>(cb + a.lay.rid);
    for (int q = threadIdx.x; q < 2 * a.L + 2 * a.Z; q += blockDim.x) totals[q] = 0;
    for (int k = threadIdx.x; k < a.K; k += blockDim.x) rid[k] = 0;
}

int check_count_dims(const char* what, int S, int K, int L, int Z, int P) {
    if (S < 1 || K < 1 || K > YFV2_TRACK_MAX_CAPACITY) {
        set_error("%s: need S >= 1 and capacity K in 1..%d, as the tracker's (S=%d K=%d)", what, YFV2_TRACK_MAX_CAPACITY, S, K);
        return YFV2_EINVAL;
    }
    if (L < 0 || L > kMaxLines || Z < 0 || Z > kMaxZones || P < 3 || P > kMaxVerts) {
        set_error("%s: need L in 0..%d lines, Z in 0..%d zones and P in 3..%d vertices (L=%d Z=%d P=%d)", what, kMaxLines, kMaxZones,
                  kMaxVerts, L, Z, P);
        return YFV2_EINVAL;
    }
    return YFV2_OK;
}

}  // namespace
}  // namespace yfv2

using namespace yfv2;

extern "C" int yfv2_track_state_bytes(int S, int K, size_t* bytes) {
    if (!bytes) { set_error("track_state_bytes: null bytes"); return YFV2_EINVAL; }
    if (S < 1 || K < 1 || K > YFV2_TRACK_MAX_CAPACITY) {
        set_error("track_state_bytes: need S >= 1 and capacity K in 1..%d (S=%d K=%d)", YFV2_TRACK_MAX_CAPACITY, S, K);
        return YFV2_EINVAL;
    }
    *bytes = (size_t)S * stream_stride(K);
    return YFV2_OK;
}

extern "C" int yfv2_track_reset(void* state, int S, int K, const int* streams_host, int B, void* stream) {
    if (!state || !streams_host) { set_error("track_reset: null state / streams_host"); return YFV2_EINVAL; }
    std::vector<unsigned char> seen;
    if (int rc = check_streams("track_reset", S, K, streams_host, B, seen)) return rc;
    ResetArgs a;
    a.state = static_cast<unsigned char*>(state);
    a.stride = stream_stride(K);
    std::copy(streams_host, streams_host + B, a.streams);
    track_reset_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(a);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_track_update(void* state, int S, int K, const int* streams_host, int B, const double* dets, const int* counts,
                                 int M, const yfv2_track_params* params, double* out, int* out_counts, int* dropped, void* stream) {
    if (!state || !streams_host || !dets || !counts || !params || !out || !out_counts || !dropped) {
        set_error("track_update: null state / streams_host / dets / counts / params / out / out_counts / dropped");
        return YFV2_EINVAL;
    }
    std::vector<unsigned char> seen;
    if (int rc = check_streams("track_update", S, K, streams_host, B, seen)) return rc;
    if (M < 1 || M > YFV2_TRACK_MAX_ROWS) { set_error("track_update: M=%d rows per stream: need 1..%d", M, YFV2_TRACK_MAX_ROWS); return YFV2_EINVAL; }
    const yfv2_track_params& p = *params;
    if (!isfinite(p.high_thresh) || !isfinite(p.low_thresh) || !isfinite(p.new_thresh) || !isfinite(p.match_thresh)) {
        set_error("track_update: thresholds must be finite (high %g, low %g, new %g, match %g)", p.high_thresh, p.low_thresh, p.new_thresh,
                  p.match_thresh);
        return YFV2_EINVAL;
    }
    if (!(0.0 <= p.low_thresh && p.low_thresh < p.high_thresh && p.high_thresh <= p.new_thresh && p.new_thresh <= 1.0)) {
        set_error("track_update: need 0 <= low_thresh < high_thresh <= new_thresh <= 1 (low %g, high %g, new %g)", p.low_thresh,
                  p.high_thresh, p.new_thresh);
        return YFV2_EINVAL;
    }
    if (!(0.0 < p.match_thresh && p.match_thresh <= 1.0)) { set_error("track_update: need 0 < match_thresh <= 1 (%g)", p.match_thresh); return YFV2_EINVAL; }
    if (p.max_age < 0) { set_error("track_update: max_age=%d must be >= 0", p.max_age); return YFV2_EINVAL; }
    std::unique_ptr<TrackArgs> ap(new (std::nothrow) TrackArgs);   // 16 KB of kernel parameters: on the heap, not the stack
    if (!ap) { set_error("track_update: host allocation failed"); return YFV2_ENOMEM; }
    TrackArgs& a = *ap;
    a.state = static_cast<unsigned char*>(state);
    a.stride = stream_stride(K);
    a.K = K; a.M = M;
    a.dets = dets; a.counts = counts; a.out = out; a.out_counts = out_counts; a.dropped = dropped;
    a.p = p;
    std::copy(streams_host, streams_host + B, a.streams);
    const size_t bytes = track_smem_bytes(K, M);
    if (bytes > kSmemCap) { set_error("track_update: %zu bytes of shared memory needed", bytes); return YFV2_EUNSUPPORTED; }
    YFV2_CUDA(cudaFuncSetAttribute(track_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    track_update_kernel<<<B, NT, bytes, (cudaStream_t)stream>>>(a);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_track_debug_read(const void* state, int S, int K, int s, int* frame_host, int* next_id_host, yfv2_track* tracks_host,
                                     int* n_host, void* stream) {
    if (!state || !frame_host || !next_id_host || !tracks_host || !n_host) { set_error("track_debug_read: null pointer"); return YFV2_EINVAL; }
    if (S < 1 || K < 1 || K > YFV2_TRACK_MAX_CAPACITY || s < 0 || s >= S) {
        set_error("track_debug_read: need S >= 1, K in 1..%d and s in [0, S) (S=%d K=%d s=%d)", YFV2_TRACK_MAX_CAPACITY, S, K, s);
        return YFV2_EINVAL;
    }
    const unsigned char* base = static_cast<const unsigned char*>(state) + (size_t)s * stream_stride(K);
    std::vector<int> head(4 + (size_t)K);
    std::vector<yfv2_track> all((size_t)K);
    cudaStream_t st = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemcpyAsync(head.data(), base, head.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    YFV2_CUDA(cudaMemcpyAsync(all.data(), base + tracks_offset(K), all.size() * sizeof(yfv2_track), cudaMemcpyDeviceToHost, st));
    YFV2_CUDA(cudaStreamSynchronize(st));
    const int n = head[2];
    if (n < 0 || n > K) { set_error("track_debug_read: stream %d holds %d tracks (capacity %d): state not reset?", s, n, K); return YFV2_EINVAL; }
    *frame_host = head[0];
    *next_id_host = head[1];
    *n_host = n;
    for (int k = 0; k < n; ++k) tracks_host[k] = all[(size_t)head[4 + k]];
    return YFV2_OK;
}

extern "C" int yfv2_count_state_bytes(int S, int K, int L, int Z, int P, size_t* bytes) {
    if (!bytes) { set_error("count_state_bytes: null bytes"); return YFV2_EINVAL; }
    if (int rc = check_count_dims("count_state_bytes", S, K, L, Z, P)) return rc;
    *bytes = (size_t)S * count_layout(K, L, Z, P).stride;
    return YFV2_OK;
}

extern "C" int yfv2_count_reset(void* count_state, int S, int K, int L, int Z, int P, const int* streams_host, int B, void* stream) {
    if (!count_state || !streams_host) { set_error("count_reset: null count_state / streams_host"); return YFV2_EINVAL; }
    if (int rc = check_count_dims("count_reset", S, K, L, Z, P)) return rc;
    std::vector<unsigned char> seen;
    if (int rc = check_streams("count_reset", S, K, streams_host, B, seen)) return rc;
    std::unique_ptr<CountResetArgs> ap(new (std::nothrow) CountResetArgs);
    if (!ap) { set_error("count_reset: host allocation failed"); return YFV2_ENOMEM; }
    CountResetArgs& a = *ap;
    a.count = static_cast<unsigned char*>(count_state);
    a.lay = count_layout(K, L, Z, P);
    a.K = K; a.L = L; a.Z = Z;
    std::copy(streams_host, streams_host + B, a.streams);
    count_reset_kernel<<<B, NT, 0, (cudaStream_t)stream>>>(a);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_count_set_geometry(void* count_state, int S, int K, int L, int Z, int P, int s, const double* lines_host, int nl,
                                       const float* zones_host, const int* nverts_host, int nz, void* stream) {
    if (!count_state) { set_error("count_set_geometry: null count_state"); return YFV2_EINVAL; }
    if (int rc = check_count_dims("count_set_geometry", S, K, L, Z, P)) return rc;
    if (s < 0 || s >= S) { set_error("count_set_geometry: stream %d outside [0, S=%d)", s, S); return YFV2_EINVAL; }
    if (nl < 0 || nl > L) { set_error("count_set_geometry: %d lines: need 0..L=%d", nl, L); return YFV2_EINVAL; }
    if (nz < 0 || nz > Z) { set_error("count_set_geometry: %d zones: need 0..Z=%d", nz, Z); return YFV2_EINVAL; }
    if ((nl > 0 && !lines_host) || (nz > 0 && (!zones_host || !nverts_host))) {
        set_error("count_set_geometry: null lines_host / zones_host / nverts_host");
        return YFV2_EINVAL;
    }
    for (int l = 0; l < nl; ++l) {
        const double* g = lines_host + 4 * (size_t)l;
        if (!isfinite(g[0]) || !isfinite(g[1]) || !isfinite(g[2]) || !isfinite(g[3])) {
            set_error("count_set_geometry: lines[%d] has a non-finite coordinate", l);
            return YFV2_EINVAL;
        }
        if (g[0] == g[2] && g[1] == g[3]) { set_error("count_set_geometry: lines[%d] has A = B = (%g, %g)", l, g[0], g[1]); return YFV2_EINVAL; }
    }
    for (int z = 0; z < nz; ++z) {
        const int nv = nverts_host[z];
        if (nv < 3 || nv > P) { set_error("count_set_geometry: zones[%d] has %d vertices: need 3..P=%d", z, nv, P); return YFV2_EINVAL; }
        for (int i = 0; i < 2 * nv; ++i)
            if (!isfinite(zones_host[(size_t)z * P * 2 + i])) {
                set_error("count_set_geometry: zones[%d] vertex %d has a non-finite coordinate", z, i / 2);
                return YFV2_EINVAL;
            }
    }
    // header, zeroed totals, lines and zones in one copy from the host; then the records cleared
    const CountLayout c = count_layout(K, L, Z, P);
    std::vector<unsigned char> head(c.rid, 0);
    int* hdr = reinterpret_cast<int*>(head.data());
    hdr[0] = nl;
    hdr[1] = nz;
    if (nl) std::copy(lines_host, lines_host + 4 * (size_t)nl, reinterpret_cast<double*>(head.data() + c.lines));
    if (nz) {
        std::copy(nverts_host, nverts_host + nz, reinterpret_cast<int*>(head.data() + c.nverts));
        std::copy(zones_host, zones_host + (size_t)nz * P * 2, reinterpret_cast<float*>(head.data() + c.verts));
    }
    unsigned char* base = static_cast<unsigned char*>(count_state) + (size_t)s * c.stride;
    cudaStream_t st = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemcpyAsync(base, head.data(), head.size(), cudaMemcpyHostToDevice, st));
    YFV2_CUDA(cudaMemsetAsync(base + c.rid, 0, (size_t)K * sizeof(int), st));
    return YFV2_OK;
}

extern "C" int yfv2_count_update(const void* track_state, void* count_state, int S, int K, int L, int Z, int P, const int* streams_host,
                                 int B, int E, double* events, int* event_counts, int* occupancy, void* stream) {
    if (!track_state || !count_state || !streams_host || !event_counts || (Z > 0 && !occupancy) || (E > 0 && !events)) {
        set_error("count_update: null track_state / count_state / streams_host / events / event_counts / occupancy");
        return YFV2_EINVAL;
    }
    if (int rc = check_count_dims("count_update", S, K, L, Z, P)) return rc;
    std::vector<unsigned char> seen;
    if (int rc = check_streams("count_update", S, K, streams_host, B, seen)) return rc;
    if (E < 0) { set_error("count_update: E=%d events per stream: need E >= 0", E); return YFV2_EINVAL; }
    std::unique_ptr<CountArgs> ap(new (std::nothrow) CountArgs);   // 16 KB of kernel parameters: on the heap, not the stack
    if (!ap) { set_error("count_update: host allocation failed"); return YFV2_ENOMEM; }
    CountArgs& a = *ap;
    a.track = static_cast<const unsigned char*>(track_state);
    a.count = static_cast<unsigned char*>(count_state);
    a.track_stride = stream_stride(K);
    a.lay = count_layout(K, L, Z, P);
    a.K = K; a.L = L; a.Z = Z; a.P = P; a.E = E;
    a.events = events; a.event_counts = event_counts; a.occupancy = occupancy;
    std::copy(streams_host, streams_host + B, a.streams);
    count_update_kernel<<<B, NT, 0, (cudaStream_t)stream>>>(a);
    YFV2_LAUNCH_CHECK();
    return YFV2_OK;
}

extern "C" int yfv2_count_debug_read(const void* count_state, int S, int K, int L, int Z, int P, int s, int* geom_host,
                                     long long* totals_host, int* ids_host, double* anchors_host, signed char* sides_host,
                                     unsigned int* inside_host, void* stream) {
    if (!count_state || !geom_host || !totals_host || !ids_host || !anchors_host || (L > 0 && !sides_host) || !inside_host) {
        set_error("count_debug_read: null pointer");
        return YFV2_EINVAL;
    }
    if (int rc = check_count_dims("count_debug_read", S, K, L, Z, P)) return rc;
    if (s < 0 || s >= S) { set_error("count_debug_read: stream %d outside [0, S=%d)", s, S); return YFV2_EINVAL; }
    const CountLayout c = count_layout(K, L, Z, P);
    std::vector<unsigned char> blk(c.stride);
    cudaStream_t st = (cudaStream_t)stream;
    YFV2_CUDA(cudaMemcpyAsync(blk.data(), static_cast<const unsigned char*>(count_state) + (size_t)s * c.stride, c.stride,
                              cudaMemcpyDeviceToHost, st));
    YFV2_CUDA(cudaStreamSynchronize(st));
    const unsigned char* p = blk.data();
    std::copy(p, p + 2 * sizeof(int), reinterpret_cast<unsigned char*>(geom_host));
    std::copy(p + c.totals, p + c.totals + (size_t)(2 * L + 2 * Z) * sizeof(long long), reinterpret_cast<unsigned char*>(totals_host));
    std::copy(p + c.rid, p + c.rid + (size_t)K * sizeof(int), reinterpret_cast<unsigned char*>(ids_host));
    std::copy(p + c.rin, p + c.rin + (size_t)K * sizeof(unsigned), reinterpret_cast<unsigned char*>(inside_host));
    std::copy(p + c.rpos, p + c.rpos + (size_t)K * 2 * sizeof(double), reinterpret_cast<unsigned char*>(anchors_host));
    if (L > 0) std::copy(p + c.rside, p + c.rside + (size_t)K * L, reinterpret_cast<unsigned char*>(sides_host));
    return YFV2_OK;
}
