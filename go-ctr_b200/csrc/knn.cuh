// knn.cuh — top-k cosine search over the ITEM_EMB table: search.Searcher (feature/embedding/search/search.go:66-134,
// searchutil.go:17-26, embutil.go:21-27).  SURVEY.md §2 feature/embedding, DESIGN.md §1a row f5.
//
// Arithmetic (bit-identical to search.go on the table values widened to float64):
//   Norm(v)  = sqrt(sum_d v_d*v_d), sequential over d, correctly rounded sqrt
//   Cosine   = 0 if either norm is 0, else dot / nq / nv: sequential float64 dot, two IEEE divisions in that order.
// A product of two widened float32 values is exact, so row norms and row-query dots may use DFMA.  Float64 vector
// queries use unfused __dmul_rn / __dadd_rn (Go on amd64 never fuses).
// Selection: the first k items under (similarity descending, row ascending), similarity strictly > 0.  NaN scores
// compare false and never qualify.  The order is total, so the result does not depend on slicing or tiling.
//
// k_knn_scan: grid (query tile, row slice).  The query tile sits in shared memory as float64; each thread scores
// kRows rows of a step against every query of the tile, row norms computed once per step for the whole tile.  A step's
// rows are staged through shared memory kChunk columns at a time, so HBM is read with coalesced 128-bit loads.  Per
// query the CTA keeps a sorted top-k list and a candidate buffer in shared memory; a candidate enters the buffer only
// if it beats the list's current k-th entry, and after every step one warp per query inserts the buffered candidates.
// k_knn_merge: one CTA per query streams the slices' lists through the same list/buffer and writes the final top-k.
//
// Row-sharded ITEM_EMB (world > 1): the scan walks this rank's shard, whose local row l is global row l·world + rank;
// exclusion and the tie order use the global row, so every rank's lists hold global rows and merging the ranks' lists
// with k_knn_merge gives what one scan of the whole table gives.
//
// The list/buffer machinery is shared with the recommendation top-k (rec.cuh): a Key type names the score type and the
// rule a score must meet to enter a list.
#pragma once
#include "common.cuh"
#include <climits>

namespace ctr {
namespace knn {

constexpr int kThreads = 128;
constexpr int kRows = 2;                      // rows per thread and step
constexpr int kStep = kThreads * kRows;       // rows per step == candidate buffer capacity per query
constexpr int kMaxK = 1024;
constexpr int kEmptyRow = INT_MAX;            // list entries start as (Key::empty(), kEmptyRow): every qualifying score beats them
constexpr int kChunk = 32;                    // columns of a step's rows staged in shared memory at a time
constexpr int kTileLd = kChunk + 4;           // padded row pitch: the per-thread float4 reads are conflict-free
constexpr size_t kTileBytes = (size_t)kStep * kTileLd * 4;

// list order: score descending, then row ascending (a total order: NaN never enters a list)
template <typename T>
__device__ __forceinline__ bool better(T s1, int r1, T s2, int r2) { return s1 > s2 || (s1 == s2 && r1 < r2); }

// search.Searcher: cosine similarities, only those > 0 qualify (search.go)
struct SimKey {
    using T = double;
    __device__ static double empty() { return 0.0; }
    __device__ static bool qualifies(double s) { return s > 0.0; }
};
// recommendation (rec.cuh): pre-sigmoid logits, any that is not NaN qualifies; (-inf, kEmptyRow) loses to (-inf, row)
struct LogitKey {
    using T = float;
    __device__ static float empty() { return -__int_as_float(0x7f800000); }
    __device__ static bool qualifies(float s) { return s == s; }
};
// the float64 MLP's recommendation (ctr_mlp_recommend_topk): float64 output-layer logits, LogitKey's rule
struct Logit64Key {
    using T = double;
    __device__ static double empty() { return -__longlong_as_double(0x7ff0000000000000ll); }
    __device__ static bool qualifies(double s) { return s == s; }
};

// shared-memory layout of QT queries' top-k state
template <class K>
struct Smem {
    using T = typename K::T;
    double* q;      // [QT][Dp] query tile (search scan only)
    double* qn;     // [QT] query norms
    T* ls;          // [QT][k] list scores, sorted best first
    T* bs;          // [QT][kStep] candidate buffer
    int* lr;        // [QT][k] list rows
    int* br;        // [QT][kStep]
    int* bn;        // [QT] buffered candidates
    int* ex;        // [QT] excluded row (-1: none)
};
template <class K>
__host__ __device__ inline size_t smem_bytes(int QT, int Dp, int k) {
    return (size_t)QT * ((size_t)Dp * 8 + ((size_t)k + kStep) * (sizeof(typename K::T) + 4) + 16);
}
template <class K>
__device__ inline Smem<K> carve(char* p, int QT, int Dp, int k) {
    using T = typename K::T;
    Smem<K> s;
    s.q = (double*)p;   p += (size_t)QT * Dp * 8;
    s.qn = (double*)p;  p += (size_t)QT * 8;
    s.ls = (T*)p;       p += (size_t)QT * k * sizeof(T);
    s.bs = (T*)p;       p += (size_t)QT * kStep * sizeof(T);
    s.lr = (int*)p;     p += (size_t)QT * k * 4;
    s.br = (int*)p;     p += (size_t)QT * kStep * 4;
    s.bn = (int*)p;     p += (size_t)QT * 4;
    s.ex = (int*)p;
    return s;
}

// one warp inserts n buffered candidates into a sorted list of k entries (insertion order does not matter: the order
// is total).  Candidates that no longer beat the k-th entry are dropped.
template <typename T>
__device__ void warp_insert(T* ls, int* lr, int k, const T* bs, const int* br, int n, int lane) {
    for (int c = 0; c < n; c++) {
        const T s = bs[c]; const int r = br[c];
        if (!better(s, r, ls[k - 1], lr[k - 1])) continue;          // uniform: every lane reads the same entries
        int cnt = 0;
        for (int i = lane; i < k; i += 32) cnt += better(ls[i], lr[i], s, r) ? 1 : 0;
        const int pos = __reduce_add_sync(0xffffffffu, cnt);       // entries better than the candidate: a prefix
        for (int top = k - 2; top >= pos; top -= 32) {              // shift [pos, k-1) up by one, top chunk first
            const int i = top - lane;
            T vs = 0; int vr = 0;
            if (i >= pos) { vs = ls[i]; vr = lr[i]; }
            __syncwarp();
            if (i >= pos) { ls[i + 1] = vs; lr[i + 1] = vr; }
            __syncwarp();
        }
        if (lane == 0) { ls[pos] = s; lr[pos] = r; }
        __syncwarp();
    }
}

// after a step: warp w inserts the buffers of queries w, w + nwarps, ...  Call between two __syncthreads().
template <int QT, class K>
__device__ __forceinline__ void flush(const Smem<K>& sm, int k) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int q = warp; q < QT; q += kThreads / 32) {
        const int n = sm.bn[q];
        if (n == 0) continue;
        warp_insert(sm.ls + (size_t)q * k, sm.lr + (size_t)q * k, k, sm.bs + (size_t)q * kStep, sm.br + (size_t)q * kStep, n, lane);
        if (lane == 0) sm.bn[q] = 0;
    }
}

template <class K>
__device__ __forceinline__ void offer(const Smem<K>& sm, int q, int k, typename K::T s, int row) {
    if (K::qualifies(s) && better(s, row, sm.ls[(size_t)q * k + k - 1], sm.lr[(size_t)q * k + k - 1])) {
        const int i = atomicAdd(&sm.bn[q], 1);
        sm.bs[(size_t)q * kStep + i] = s; sm.br[(size_t)q * kStep + i] = row;
    }
}

// ROWQ: query i is table row qrow[i] (excluded from its own result); else the float64 vector qvec[i] (excl may name a
// row to exclude, -1 = none).  tab holds nrows local rows; local row l is global row l·world + rank.  ROWQ reads the
// query rows from tab and so needs world == 1.  Out: per (query, slice) the sorted top-k list, [nq][slices][k].
template <int QT, bool ROWQ>
__global__ void __launch_bounds__(kThreads) k_knn_scan(const float* __restrict__ tab, long ld, long nrows, int world, int rank, int D,
                                                        const double* __restrict__ qvec, const int* __restrict__ qrow,
                                                        const int* __restrict__ excl, int nq, int k, long rows_per_slice,
                                                        double* __restrict__ out_sim, int* __restrict__ out_row) {
    extern __shared__ __align__(16) char smem_raw[];
    const int Dp = (D + 3) & ~3;
    float* tile = (float*)smem_raw;           // [kStep][kTileLd]: the step's rows, kChunk columns at a time
    const Smem<SimKey> sm = carve<SimKey>(smem_raw + kTileBytes, QT, Dp, k);
    const int q0 = blockIdx.x * QT;
    const int slice = blockIdx.y, slices = gridDim.y;

    for (int i = threadIdx.x; i < QT * Dp; i += kThreads) {
        const int qi = i / Dp, d = i - qi * Dp, g = q0 + qi;
        double v = 0.0;
        if (g < nq && d < D) v = ROWQ ? (double)tab[(size_t)qrow[g] * ld + d] : qvec[(size_t)g * D + d];
        sm.q[i] = v;
    }
    for (int i = threadIdx.x; i < QT * k; i += kThreads) { sm.ls[i] = SimKey::empty(); sm.lr[i] = kEmptyRow; }
    if (threadIdx.x < QT) {
        const int g = q0 + threadIdx.x;
        sm.bn[threadIdx.x] = 0;
        sm.ex[threadIdx.x] = g < nq ? (ROWQ ? qrow[g] : (excl ? excl[g] : -1)) : -1;
    }
    __syncthreads();
    if (threadIdx.x < QT) {                   // embutil.Norm: sequential float64 sum of squares
        const double* qv = sm.q + (size_t)threadIdx.x * Dp;
        double n = 0.0;
        for (int d = 0; d < D; d++) n = ROWQ ? __fma_rn(qv[d], qv[d], n) : __dadd_rn(n, __dmul_rn(qv[d], qv[d]));
        sm.qn[threadIdx.x] = __dsqrt_rn(n);
    }
    __syncthreads();

    const long r0 = (long)slice * rows_per_slice, r1 = min(nrows, r0 + rows_per_slice);
    for (long base = r0; base < r1; base += kStep) {
        long row[kRows]; bool ok[kRows];
        double acc[QT][kRows], nv[kRows];
#pragma unroll
        for (int r = 0; r < kRows; r++) {
            row[r] = base + threadIdx.x + r * kThreads; ok[r] = row[r] < r1; nv[r] = 0.0;
#pragma unroll
            for (int q = 0; q < QT; q++) acc[q][r] = 0.0;
        }
        // the rows are read from HBM coalesced (consecutive threads, consecutive float4 of a row) into shared memory;
        // each thread then walks its own rows there, in order over d, as the sequential sums require
        for (int c0 = 0; c0 < Dp; c0 += kChunk) {
            const int cw4 = min(kChunk, Dp - c0) >> 2;
            __syncthreads();                                  // the previous chunk has been read
#pragma unroll 4
            for (int i = threadIdx.x; i < kStep * cw4; i += kThreads) {
                const int rr = i / cw4, c4 = i - rr * cw4;
                const long gr = base + rr;
                const float4 v = gr < r1 ? __ldg(reinterpret_cast<const float4*>(tab + gr * ld + c0) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
                *reinterpret_cast<float4*>(tile + rr * kTileLd + c4 * 4) = v;
            }
            __syncthreads();
#pragma unroll 2
            for (int d0 = 0; d0 < cw4 * 4; d0 += 4) {
                float4 v[kRows];
#pragma unroll
                for (int r = 0; r < kRows; r++) v[r] = *reinterpret_cast<const float4*>(tile + (threadIdx.x + r * kThreads) * kTileLd + d0);
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int d = c0 + d0 + j;
                    if (d >= D) break;
#pragma unroll
                    for (int r = 0; r < kRows; r++) {
                        const float f = j == 0 ? v[r].x : j == 1 ? v[r].y : j == 2 ? v[r].z : v[r].w;
                        const double x = (double)f;
                        nv[r] = __fma_rn(x, x, nv[r]);                                    // exact product
#pragma unroll
                        for (int q = 0; q < QT; q++) {
                            const double qd = sm.q[(size_t)q * Dp + d];
                            acc[q][r] = ROWQ ? __fma_rn(qd, x, acc[q][r]) : __dadd_rn(acc[q][r], __dmul_rn(qd, x));
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < kRows; r++) {
            if (!ok[r]) continue;
            const double n2 = __dsqrt_rn(nv[r]);
            const int grow = (int)row[r] * world + rank;          // global rows fit int32 (checked by the host)
#pragma unroll
            for (int q = 0; q < QT; q++) {
                const double n1 = sm.qn[q];
                const double s = (n1 == 0.0 || n2 == 0.0) ? 0.0 : __ddiv_rn(__ddiv_rn(acc[q][r], n1), n2);
                if (grow != sm.ex[q]) offer(sm, q, k, s, grow);
            }
        }
        __syncthreads();
        flush<QT>(sm, k);
        __syncthreads();
    }

    for (int i = threadIdx.x; i < QT * k; i += kThreads) {
        const int qi = i / k, j = i - qi * k, g = q0 + qi;
        if (g >= nq) break;
        const size_t o = ((size_t)g * slices + slice) * k + j;
        out_sim[o] = sm.ls[i]; out_row[o] = sm.lr[i];
    }
}

// one CTA per query: the top-k of `slices` lists of k entries; list s of query g starts at element g·qstride + s·sstride
// ([n][slices][k]: qstride = slices·k, sstride = k; the ranks' gathered [world][n][k]: qstride = k, sstride = n·k).
// Positions past the count hold row -1 and score 0.
// out_count == nullptr: the list is written as it stands, empty entries included, to be merged again; it may then
// overwrite the first input list (every input is read before the first write).
template <class K>
__global__ void __launch_bounds__(kThreads) k_knn_merge(const typename K::T* in_sim, const int* in_row, int slices, int k, long qstride,
                                                         long sstride, int32_t* out_row, typename K::T* out_sim, int32_t* __restrict__ out_count) {
    using T = typename K::T;
    extern __shared__ __align__(16) char smem_raw[];
    const Smem<K> sm = carve<K>(smem_raw, 1, 0, k);
    const int g = blockIdx.x;
    for (int i = threadIdx.x; i < k; i += kThreads) { sm.ls[i] = K::empty(); sm.lr[i] = kEmptyRow; }
    if (threadIdx.x == 0) sm.bn[0] = 0;
    __syncthreads();
    const long n = (long)slices * k;
    const T* is = in_sim + (size_t)g * qstride;
    const int* ir = in_row + (size_t)g * qstride;
    for (long base = 0; base < n; base += kStep) {
#pragma unroll
        for (int r = 0; r < kRows; r++) {
            const long i = base + threadIdx.x + r * kThreads;
            if (i >= n) continue;
            long o = i;                                   // contiguous lists: no division
            if (sstride != k) { const long s = i / k; o = s * sstride + (i - s * k); }
            offer(sm, 0, k, is[o], ir[o]);
        }
        __syncthreads();
        flush<1>(sm, k);
        __syncthreads();
    }
    if (!out_count) {
        for (int i = threadIdx.x; i < k; i += kThreads) { out_row[(size_t)g * k + i] = sm.lr[i]; out_sim[(size_t)g * k + i] = sm.ls[i]; }
        return;
    }
    int cnt = 0;
    for (int i = threadIdx.x; i < k; i += kThreads) {
        const bool v = sm.lr[i] != kEmptyRow;
        out_row[(size_t)g * k + i] = v ? sm.lr[i] : -1;
        out_sim[(size_t)g * k + i] = v ? sm.ls[i] : T(0);
        cnt += v ? 1 : 0;
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    __shared__ int wsum[kThreads / 32];
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kThreads / 32; w++) t += wsum[w];
        out_count[g] = t;
    }
}

}  // namespace knn
}  // namespace ctr
