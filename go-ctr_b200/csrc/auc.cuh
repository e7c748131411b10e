// auc.cuh — utils.RocAuc32 on the device (util.go:131-148 → nn/metrics/ranking.go:13-150):
// labels binarised at 0.5, scores sorted descending, equal scores form one threshold group
// (ranking.go:27-35), cumulative tp/fp, trapezoid over the normalised curve (ranking.go:106-118).
// SURVEY.md §8(f) row f4 (on-device eval).  CUB does the sort/scans; the curve logic is below.
// The grouped AUC of ctr_group_auc (GAUC, the DIN paper's metric) reuses the score key and label of ctr_roc_auc.
#pragma once
#include "common.cuh"
#include "owner.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <cmath>
#include <utility>
#include <vector>

namespace ctr {

// the sort key of a score: equal keys are one threshold group, ascending keys are descending scores
__device__ __forceinline__ unsigned auc_score_key(float p) {
    if (p == 0.0f) p = 0.0f;                           // -0 == +0 compare equal in the reference
    unsigned u = __float_as_uint(p);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);    // ascending-order-preserving
    return ~u;                                         // ascending sort of ~u == descending scores
}
__device__ __forceinline__ int auc_positive(float y) { return y > 0.5f ? 1 : 0; }   // util.go:134-138

__global__ void k_auc_keys(const float* __restrict__ pred, const float* __restrict__ y, long n,
                           unsigned* __restrict__ keys, int* __restrict__ pos_flag) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        keys[i] = auc_score_key(pred[i]);
        pos_flag[i] = auc_positive(y[i]);
    }
}
__global__ void k_auc_heads(const unsigned* __restrict__ keys, long n, int* __restrict__ head) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        head[i] = (i == 0 || keys[i] != keys[i - 1]) ? (int)i : 0;
}
struct MaxOp { __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; } };

__global__ void k_auc_area(const unsigned* __restrict__ keys, const int* __restrict__ tp, const int* __restrict__ start,
                           long n, double* __restrict__ area) {
    double local = 0.0;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        if (i + 1 < n && keys[i + 1] == keys[i]) continue;      // not the end of a threshold group
        long s = start[i];
        double tpi = tp[i], fpi = (double)(i + 1) - tpi;
        double tpp = s > 0 ? (double)tp[s - 1] : 0.0, fpp = s > 0 ? (double)s - tpp : 0.0;
        local += (fpi - fpp) * (tpi + tpp) * 0.5;
    }
    local = warp_sum_d(local);
    if ((threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(area, local);
}

// pred_h / y_h are host pointers; returns cudaSuccess and *auc (NaN when one class is absent)
inline cudaError_t auc_run(cudaStream_t st, const float* pred_h, const float* y_h, long n, double* auc) {
    DevBuf<float> d_pred, d_y; DevBuf<unsigned> k0, k1; DevBuf<int> f0, f1, tp, head;
    DevBuf<double> d_area; DevBuf<unsigned char> tmp;
#define AUC_TRY(x) do { const cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)
    AUC_TRY(d_pred.alloc(n)); AUC_TRY(d_y.alloc(n));
    AUC_TRY(k0.alloc(n)); AUC_TRY(k1.alloc(n));
    AUC_TRY(f0.alloc(n)); AUC_TRY(f1.alloc(n));
    AUC_TRY(tp.alloc(n)); AUC_TRY(head.alloc(n));
    AUC_TRY(d_area.alloc(1));
    AUC_TRY(cudaMemcpyAsync(d_pred, pred_h, n * sizeof(float), cudaMemcpyHostToDevice, st));
    AUC_TRY(cudaMemcpyAsync(d_y, y_h, n * sizeof(float), cudaMemcpyHostToDevice, st));
    AUC_TRY(cudaMemsetAsync(d_area, 0, sizeof(double), st));
    size_t b0 = 0, b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b0, k0.get(), k1.get(), f0.get(), f1.get(), (int)n, 0, 32, st);
    cub::DeviceScan::InclusiveSum(nullptr, b1, f1.get(), tp.get(), (int)n, st);
    cub::DeviceScan::InclusiveScan(nullptr, b2, head.get(), head.get(), MaxOp(), (int)n, st);
    size_t bytes = b0 > b1 ? b0 : b1; bytes = bytes > b2 ? bytes : b2;
    AUC_TRY(tmp.alloc(bytes ? bytes : 1));
    int grid = (int)((n + 255) / 256); if (grid > 132 * 8) grid = 132 * 8;
    k_auc_keys<<<grid, 256, 0, st>>>(d_pred, d_y, n, k0, f0);
    AUC_TRY(cub::DeviceRadixSort::SortPairs(tmp, bytes, k0.get(), k1.get(), f0.get(), f1.get(), (int)n, 0, 32, st));
    AUC_TRY(cub::DeviceScan::InclusiveSum(tmp, bytes, f1.get(), tp.get(), (int)n, st));
    k_auc_heads<<<grid, 256, 0, st>>>(k1, n, head);
    AUC_TRY(cub::DeviceScan::InclusiveScan(tmp, bytes, head.get(), head.get(), MaxOp(), (int)n, st));
    k_auc_area<<<grid, 256, 0, st>>>(k1, tp, head, n, d_area);
    double area = 0; int P = 0;
    AUC_TRY(cudaMemcpyAsync(&area, d_area, sizeof(double), cudaMemcpyDeviceToHost, st));
    AUC_TRY(cudaMemcpyAsync(&P, tp + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
    AUC_TRY(cudaStreamSynchronize(st));
    AUC_TRY(cudaGetLastError());
#undef AUC_TRY
    double N = (double)n - (double)P;
    *auc = (P > 0 && N > 0) ? area / ((double)P * N) : nan("");
    return cudaSuccess;
}

// ---- grouped AUC (ctr_group_auc): RocAuc32 within each group, the groups' AUCs weighted by impressions -------------
// Samples are ordered by (group ascending, score key ascending) with two stable radix passes; then one scan gives every
// element the positives before it, the start of its group and the start of its threshold group, and one reduce-by-key
// over the sorted group keys sums each group's count, positives and integer trapezoid area.  No step's cost depends on
// how the samples are spread over the groups.

// signed int64 order as unsigned order
__device__ __forceinline__ unsigned long long gauc_group_key(long long g) { return (unsigned long long)g ^ 0x8000000000000000ull; }

struct GaucScan { int tp, gs, ts; };        // inclusive: positives up to here, start of the group, start of the threshold group
struct GaucScanOp {
    __device__ __forceinline__ GaucScan operator()(const GaucScan& a, const GaucScan& b) const {
        return {a.tp + b.tp, a.gs > b.gs ? a.gs : b.gs, a.ts > b.ts ? a.ts : b.ts};
    }
};
struct GaucAgg { long long area2; int n, pos; };   // area2 = sum (fp_i - fp_{i-1}) (tp_i + tp_{i-1}) over threshold-group ends
struct GaucAggOp {
    __device__ __forceinline__ GaucAgg operator()(const GaucAgg& a, const GaucAgg& b) const {
        return {a.area2 + b.area2, a.n + b.n, a.pos + b.pos};
    }
};
struct GaucPart { double hi, lo; long long w, used; };   // sum of n_g AUC_g as a double-double, sum of n_g, used groups
struct GaucResult { double gauc; long long groups, used; };

__global__ void k_gauc_keys(const float* __restrict__ pred, long n, unsigned* __restrict__ keys, int* __restrict__ idx) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        keys[i] = auc_score_key(pred[i]);
        idx[i] = (int)i;
    }
}
// after the score pass: the group key to sort by next, and the score key with the label flag in bit 0 to carry along
__global__ void k_gauc_gather(const unsigned* __restrict__ keys, const int* __restrict__ idx, const long long* __restrict__ group,
                              const float* __restrict__ y, long n, unsigned long long* __restrict__ gkey,
                              unsigned long long* __restrict__ packed) {
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < n; j += (long)gridDim.x * blockDim.x) {
        const int i = idx[j];
        gkey[j] = gauc_group_key(group[i]);
        packed[j] = (unsigned long long)keys[j] << 32 | (unsigned)auc_positive(y[i]);
    }
}
__global__ void k_gauc_heads(const unsigned long long* __restrict__ gkey, const unsigned long long* __restrict__ packed, long n,
                             GaucScan* __restrict__ s) {
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < n; j += (long)gridDim.x * blockDim.x) {
        const unsigned long long v = packed[j];
        const bool gh = j == 0 || gkey[j] != gkey[j - 1];
        const bool th = gh || (v >> 32) != (packed[j - 1] >> 32);
        s[j] = {(int)(v & 1), gh ? (int)j : 0, th ? (int)j : 0};
    }
}
// each threshold-group end adds its trapezoid, counted from its group's start
__global__ void k_gauc_terms(const unsigned long long* __restrict__ gkey, const unsigned long long* __restrict__ packed,
                             const GaucScan* __restrict__ s, long n, GaucAgg* __restrict__ val) {
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < n; j += (long)gridDim.x * blockDim.x) {
        const unsigned long long v = packed[j];
        long long term = 0;
        if (j + 1 == n || gkey[j + 1] != gkey[j] || (packed[j + 1] >> 32) != (v >> 32)) {
            const GaucScan e = s[j];
            const int base = e.gs > 0 ? s[e.gs - 1].tp : 0;
            const long long tpi = e.tp - base, fpi = (long long)(j - e.gs + 1) - tpi;
            long long tpp = 0, fpp = 0;
            if (e.ts > e.gs) { tpp = s[e.ts - 1].tp - base; fpp = (long long)(e.ts - e.gs) - tpp; }
            term = (fpi - fpp) * (tpi + tpp);
        }
        val[j] = {term, 1, (int)(v & 1)};
    }
}

// hi + lo += b_hi + b_lo (Knuth's two-sum of the high parts, the low parts added to its error)
__device__ __forceinline__ void dd_add(double& hi, double& lo, double b_hi, double b_lo) {
    const double s = hi + b_hi, bb = s - hi;
    const double l = lo + b_lo + ((hi - (s - bb)) + (b_hi - bb));
    hi = s + l;
    lo = l - (hi - s);
}
__device__ __forceinline__ GaucPart gauc_part_add(GaucPart a, const GaucPart& b) {
    dd_add(a.hi, a.lo, b.hi, b.lo);
    a.w += b.w; a.used += b.used;
    return a;
}
// the block's sum in thread 0, in a fixed order (lanes, then warps), so equal inputs give equal bits
__device__ GaucPart gauc_block_sum(GaucPart p) {
    __shared__ GaucPart sh[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const GaucPart q{__shfl_down_sync(0xffffffffu, p.hi, o), __shfl_down_sync(0xffffffffu, p.lo, o),
                         __shfl_down_sync(0xffffffffu, p.w, o), __shfl_down_sync(0xffffffffu, p.used, o)};
        p = gauc_part_add(p, q);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) sh[warp] = p;
    __syncthreads();
    if (warp == 0) {
        p = lane < nw ? sh[lane] : GaucPart{0.0, 0.0, 0, 0};
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const GaucPart q{__shfl_down_sync(0xffffffffu, p.hi, o), __shfl_down_sync(0xffffffffu, p.lo, o),
                             __shfl_down_sync(0xffffffffu, p.w, o), __shfl_down_sync(0xffffffffu, p.used, o)};
            p = gauc_part_add(p, q);
        }
    }
    return p;
}

// per group: AUC_g = area2 / (2 P N) (NaN when a class is absent) and the per-group outputs the caller asked for (null
// pointers are skipped); per block: its part of the impression-weighted sum over the used groups
__global__ void k_gauc_groups(const unsigned long long* __restrict__ uniq, const GaucAgg* __restrict__ agg, const int* __restrict__ runs,
                              long long* __restrict__ out_group, int* __restrict__ out_n, int* __restrict__ out_pos,
                              double* __restrict__ out_auc, GaucPart* __restrict__ part) {
    const long R = *runs;
    GaucPart p{0.0, 0.0, 0, 0};
    for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < R; g += (long)gridDim.x * blockDim.x) {
        const GaucAgg a = agg[g];
        const int P = a.pos, N = a.n - a.pos;
        const bool used = P > 0 && N > 0;
        const double auc = used ? (double)a.area2 / (2.0 * (double)P * (double)N) : __longlong_as_double(0x7ff8000000000000ll);
        if (out_group) out_group[g] = (long long)(uniq[g] ^ 0x8000000000000000ull);
        if (out_n) out_n[g] = a.n;
        if (out_pos) out_pos[g] = P;
        if (out_auc) out_auc[g] = auc;
        if (used) { dd_add(p.hi, p.lo, __dmul_rn((double)a.n, auc), 0.0); p.w += a.n; p.used++; }
    }
    p = gauc_block_sum(p);
    if (threadIdx.x == 0) part[blockIdx.x] = p;
}
__global__ void k_gauc_final(const GaucPart* __restrict__ part, int nparts, const int* __restrict__ runs, GaucResult* __restrict__ res) {
    GaucPart p{0.0, 0.0, 0, 0};
    for (int b = threadIdx.x; b < nparts; b += blockDim.x) p = gauc_part_add(p, part[b]);
    p = gauc_block_sum(p);
    if (threadIdx.x == 0)
        *res = {p.used > 0 ? (p.hi + p.lo) / (double)p.w : __longlong_as_double(0x7ff8000000000000ll), (long long)*runs, p.used};
}

// The fold's shape is fixed (kGaucParts blocks of 256 threads, not a multiple of the device's SM count), so the weighted
// mean depends on the sequence of groups alone: ctr_group_auc and ctr_group_auc_dist fold the same groups to the same bits.
constexpr int kGaucParts = 264;

// The grouped driver's launches, shared by ctr_group_auc and ctr_group_auc_dist (and the kernel probe).  launch(name, f)
// runs f, a lambda that enqueues work on st, and returns 0 or an error code; the engine's launch() profiles it under name.
// From samples sorted by (group key, score key) in gkey / packed: the groups' keys in uniq, their (area2, n, positives)
// in agg and their number in *d_runs.  n >= 1.
template <class Launch>
int gauc_group_terms(Launch&& launch, const unsigned long long* gkey, const unsigned long long* packed, long n, GaucScan* scan,
                     GaucAgg* val, unsigned long long* uniq, GaucAgg* agg, int* d_runs, void* tmp, size_t bytes, int grid, cudaStream_t st) {
    int rc;
    if ((rc = launch("gauc_heads", [&] { k_gauc_heads<<<grid, 256, 0, st>>>(gkey, packed, n, scan); }))) return rc;
    if ((rc = launch("gauc_scan", [&] {
             cub::DeviceScan::InclusiveScan(tmp, bytes, scan, scan, GaucScanOp(), (int)n, st); }))) return rc;
    if ((rc = launch("gauc_terms", [&] { k_gauc_terms<<<grid, 256, 0, st>>>(gkey, packed, scan, n, val); }))) return rc;
    return launch("gauc_reduce", [&] {
        cub::DeviceReduce::ReduceByKey(tmp, bytes, gkey, uniq, val, agg, d_runs, GaucAggOp(), (int)n, st); });
}
// the per-group AUCs (the out_* arrays may be null) and the impression-weighted mean of the *d_runs groups in res
template <class Launch>
int gauc_fold_groups(Launch&& launch, const unsigned long long* uniq, const GaucAgg* agg, const int* d_runs, long long* out_group,
                     int* out_n, int* out_pos, double* out_auc, GaucPart* part, GaucResult* res, cudaStream_t st) {
    int rc;
    if ((rc = launch("gauc_groups", [&] { k_gauc_groups<<<kGaucParts, 256, 0, st>>>(uniq, agg, d_runs, out_group, out_n, out_pos, out_auc, part); })))
        return rc;
    return launch("gauc_final", [&] { k_gauc_final<<<1, 256, 0, st>>>(part, kGaucParts, d_runs, res); });
}

// ---- ROC AUC and GAUC over every rank's samples (ctr_roc_auc_dist, ctr_group_auc_dist) ---------------------------------
// Both calls range-partition their data by key so that everything one key decides meets on one rank: a tie group of
// scores (ROC AUC) or a group of samples (GAUC).  Ranks own ascending key ranges in rank order.  The steps below are
// per rank and take no handle, so the kernel probe runs them on shards of one device; the exchanges are in engine.cu.
//
// ROC AUC: a run is (score key, positives << 32 | negatives).  Each rank sorts its keys, sums the counts of equal keys
// (auc_dist_rle), sends the runs of each key range to its owner, and sums equal keys again over what it received (the
// same auc_dist_rle).  Counts packed this way add without carries while the total is below 2^32.  The area is the
// integer sum over the owner's runs j of neg_j (2 tp_{j-1} + pos_j), where tp_{j-1} counts every positive of a lower key,
// on this rank or on a lower rank.

constexpr int kDistSamples = 31;   // regular samples of each rank's sorted keys; with the key count one gather slot of 32

__global__ void k_auc_dist_keys(const float* __restrict__ pred, const float* __restrict__ y, long n, unsigned* __restrict__ keys,
                                unsigned long long* __restrict__ cnt) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        keys[i] = auc_score_key(pred[i]);
        cnt[i] = auc_positive(y[i]) ? 1ull << 32 : 1ull;
    }
}
struct SumU64 { __device__ __forceinline__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; } };

// out[0] = the number of keys *d_u, out[1 + i] = key (i * u) / kDistSamples of the sorted keys (0 when u = 0)
template <typename K>
__global__ void k_dist_samples(const K* __restrict__ keys, const int* __restrict__ d_u, long long* __restrict__ out) {
    const long u = *d_u;
    const int t = threadIdx.x;
    if (t == 0) out[0] = u;
    if (t < kDistSamples) out[1 + t] = u > 0 ? (long long)keys[(long)t * u / kDistSamples] : 0;
}
// off[d] = the first sorted key that belongs to rank d or later: off[0] = 0, off[d] = #keys <= spl[d - 1], off[W] = u
template <typename K>
__global__ void k_dist_part(const K* __restrict__ keys, const int* __restrict__ d_u, const unsigned long long* __restrict__ spl, int W,
                            long long* __restrict__ off) {
    const long u = *d_u;
    const int d = threadIdx.x;
    if (d > W) return;
    if (d == 0 || d == W) { off[d] = d == 0 ? 0 : u; return; }
    const unsigned long long s = spl[d - 1];
    long lo = 0, hi = u;
    while (lo < hi) { const long mid = (lo + hi) >> 1; if ((unsigned long long)keys[mid] <= s) lo = mid + 1; else hi = mid; }
    off[d] = lo;
}
// this rank's share of 2 x the area: neg_j (2 tp_{j-1} + pos_j) over its merged runs, inc the inclusive sum of cnt and
// base the positives of every lower rank; the sum is exact (2 P N < 2^64), so the order of the atomics does not matter
__global__ void k_auc_dist_area(const unsigned long long* __restrict__ cnt, const unsigned long long* __restrict__ inc, long m,
                                unsigned long long base, unsigned long long* __restrict__ acc) {
    unsigned long long local = 0;
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < m; j += (long)gridDim.x * blockDim.x) {
        const unsigned long long c = cnt[j], pos = c >> 32, neg = c & 0xffffffffull;
        const unsigned long long before = base + (inc[j] >> 32) - pos;
        local += neg * (2 * before + pos);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(acc, local);
}
// GAUC's record of a sample: the group key to partition and sort by, and the score key with the label in bit 0
__global__ void k_gauc_dist_rec(const float* __restrict__ pred, const float* __restrict__ y, const long long* __restrict__ group, long n,
                                unsigned long long* __restrict__ gkey, unsigned long long* __restrict__ packed) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        gkey[i] = gauc_group_key(group[i]);
        packed[i] = (unsigned long long)auc_score_key(pred[i]) << 32 | (unsigned)auc_positive(y[i]);
    }
}

inline int dist_grid(long n) { long g = (n + 255) / 256; if (g > 132 * 8) g = 132 * 8; return (int)(g > 0 ? g : 1); }

// CUB scratch of auc_dist_rle over n entries
inline size_t auc_dist_rle_bytes(long n, cudaStream_t st) {
    size_t a = 0, b = 0, c = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned long long*)nullptr,
                                    (unsigned long long*)nullptr, (int)n, 0, 32, st);
    cub::DeviceReduce::ReduceByKey(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned long long*)nullptr,
                                   (unsigned long long*)nullptr, (int*)nullptr, SumU64(), (int)n, st);
    cub::DeviceScan::InclusiveSum(nullptr, c, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n, st);
    return std::max(std::max(a, b), std::max(c, (size_t)1));
}
// runs of (key, count) pairs: sorted by key into ks / cs, equal keys summed into ukey / ucnt, their number in *d_u
inline cudaError_t auc_dist_rle(const unsigned* k, const unsigned long long* c, long n, unsigned* ks, unsigned long long* cs,
                                unsigned* ukey, unsigned long long* ucnt, int* d_u, void* tmp, size_t bytes, cudaStream_t st) {
    if (n == 0) return cudaMemsetAsync(d_u, 0, sizeof(int), st);
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, bytes, k, ks, c, cs, (int)n, 0, 32, st);
    if (e == cudaSuccess) e = cub::DeviceReduce::ReduceByKey(tmp, bytes, ks, ukey, cs, ucnt, d_u, SumU64(), (int)n, st);
    return e;
}
// one rank's runs of its own samples (device pred / y; k0 / c0 / ks / cs scratch of n entries)
inline cudaError_t auc_dist_local(const float* pred, const float* y, long n, unsigned* k0, unsigned long long* c0, unsigned* ks,
                                  unsigned long long* cs, unsigned* ukey, unsigned long long* ucnt, int* d_u, void* tmp, size_t bytes,
                                  cudaStream_t st) {
    if (n > 0) k_auc_dist_keys<<<dist_grid(n), 256, 0, st>>>(pred, y, n, k0, c0);
    const cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : auc_dist_rle(k0, c0, n, ks, cs, ukey, ucnt, d_u, tmp, bytes, st);
}
// the regular samples of u sorted keys into smp[kDistSamples + 1] (device)
template <typename K>
inline cudaError_t dist_samples(const K* keys, const int* d_u, long long* smp, cudaStream_t st) {
    k_dist_samples<K><<<1, 32, 0, st>>>(keys, d_u, smp);
    return cudaGetLastError();
}
// The W - 1 splitters from every rank's samples (all[r (kDistSamples + 1)] = u_r, then its samples as in
// k_dist_samples).  Every sample of rank r weighs u_r; splitter d is the smallest sample key at which the cumulative
// weight in ascending key order reaches d / W of the total.  Rank d then owns the keys in (spl[d - 1], spl[d]].
inline void dist_splitters(const int64_t* all, int W, unsigned long long* spl) {
    std::vector<std::pair<unsigned long long, unsigned long long>> s;
    unsigned long long total = 0;
    for (int r = 0; r < W; r++) {
        const int64_t* a = all + (size_t)r * (kDistSamples + 1);
        if (a[0] <= 0) continue;
        for (int i = 0; i < kDistSamples; i++) s.push_back({(unsigned long long)a[1 + i], (unsigned long long)a[0]});
        total += (unsigned long long)a[0] * kDistSamples;
    }
    std::sort(s.begin(), s.end());
    size_t i = 0;
    unsigned long long cum = 0;
    for (int d = 1; d < W; d++) {
        while (i < s.size() && cum * (unsigned long long)W < (unsigned long long)d * total) cum += s[i++].second;
        spl[d - 1] = i > 0 ? s[i - 1].first : 0ull;
    }
}
// the send offsets off[0 .. W] of u sorted keys (device spl [W - 1], off [W + 1])
template <typename K>
inline cudaError_t dist_part(const K* keys, const int* d_u, const unsigned long long* spl, int W, long long* off, cudaStream_t st) {
    k_dist_part<K><<<1, 32, 0, st>>>(keys, d_u, spl, W, off);
    return cudaGetLastError();
}
// this rank's 2 x area into acc[0] (zeroed here) from its m merged runs; inc is scratch of m entries.  The positives and
// negatives of the runs come back in *pos / *neg (host; synchronises st).
inline cudaError_t auc_dist_totals(const unsigned long long* cnt, long m, unsigned long long* inc, void* tmp, size_t bytes,
                                   unsigned long long* pos, unsigned long long* neg, cudaStream_t st) {
    *pos = *neg = 0;
    if (m == 0) return cudaSuccess;
    cudaError_t e = cub::DeviceScan::InclusiveSum(tmp, bytes, cnt, inc, (int)m, st);
    unsigned long long t = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&t, inc + (m - 1), sizeof t, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    *pos = t >> 32; *neg = t & 0xffffffffull;
    return e;
}
inline cudaError_t auc_dist_area(const unsigned long long* cnt, const unsigned long long* inc, long m, unsigned long long base,
                                 unsigned long long* acc, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(acc, 0, sizeof(unsigned long long), st);
    if (e == cudaSuccess && m > 0) { k_auc_dist_area<<<dist_grid(m), 256, 0, st>>>(cnt, inc, m, base, acc); e = cudaGetLastError(); }
    return e;
}
// ROC AUC from the integer totals, rounded once as auc_run rounds it
inline double auc_dist_value(unsigned long long area2, unsigned long long P, unsigned long long N) {
    return (P > 0 && N > 0) ? ((double)area2 * 0.5) / ((double)P * (double)N) : nan("");
}

// GAUC: records (group key, score key << 32 | label) sorted by group key on the sender, range-partitioned by group key,
// then ordered by (group, score) on the owner with two stable radix passes and reduced by gauc_group_terms.
inline size_t gauc_dist_bytes(long n, cudaStream_t st) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n, 0, 64, st);
    cub::DeviceScan::InclusiveScan(nullptr, b, (GaucScan*)nullptr, (GaucScan*)nullptr, GaucScanOp(), (int)n, st);
    size_t c = 0;
    cub::DeviceReduce::ReduceByKey(nullptr, c, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const GaucAgg*)nullptr,
                                   (GaucAgg*)nullptr, (int*)nullptr, GaucAggOp(), (int)n, st);
    return std::max(std::max(a, b), std::max(c, (size_t)1));
}
// one rank's records sorted by group key into g1 / v1 (g0 / v0 scratch); n >= 1
inline cudaError_t gauc_dist_sort(const float* pred, const float* y, const long long* group, long n, unsigned long long* g0,
                                  unsigned long long* v0, unsigned long long* g1, unsigned long long* v1, void* tmp, size_t bytes,
                                  cudaStream_t st) {
    k_gauc_dist_rec<<<dist_grid(n), 256, 0, st>>>(pred, y, group, n, g0, v0);
    const cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : cub::DeviceRadixSort::SortPairs(tmp, bytes, g0, g1, v0, v1, (int)n, 0, 64, st);
}
// the m received records (rg / rv) in (group, score) order in g1 / v1 (g0 / v0 scratch); m >= 1
inline cudaError_t gauc_dist_order(const unsigned long long* rg, const unsigned long long* rv, long m, unsigned long long* g0,
                                   unsigned long long* v0, unsigned long long* g1, unsigned long long* v1, void* tmp, size_t bytes,
                                   cudaStream_t st) {
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, bytes, rv, v0, rg, g0, (int)m, 32, 64, st);
    return e != cudaSuccess ? e : cub::DeviceRadixSort::SortPairs(tmp, bytes, g0, g1, v0, v1, (int)m, 0, 64, st);
}

// ---- curves and average precision (ctr_roc_curve, ctr_pr_curve, ctr_average_precision): binaryClfCurve --------------
// (ranking.go:13-57) on ctr_roc_auc's key sort and positive-count scan.  The ends of the threshold groups are compacted
// into points (tp_j, fp_j, key_j), one per group from the highest score down; small kernels turn the points into the
// ROC arrays (ranking.go:71-103), the PR arrays (:183-209) or the AP terms (:212-222).  Every NaN these kernels make
// is the quiet NaN 0x7ff8000000000000.

__device__ __forceinline__ double clf_nan() { return __longlong_as_double(0x7ff8000000000000ll); }

// float32 bits widened to float64 exactly, without float arithmetic (no flush of subnormals); NaNs keep sign and payload
__device__ __forceinline__ double clf_widen(unsigned u) {
    const unsigned long long s = (unsigned long long)(u >> 31) << 63, m = u & 0x7fffffu;
    const unsigned e = (u >> 23) & 0xffu;
    if (e == 0xffu) return __longlong_as_double((long long)(s | 0x7ff0000000000000ull | m << 29));
    if (e == 0u) { const double d = __dmul_rn((double)m, 0x1p-149); return s ? -d : d; }
    return __longlong_as_double((long long)(s | (unsigned long long)(e + 896u) << 52 | m << 29));
}
// the threshold of a threshold group: the inverse of auc_score_key, widened (the ±0 group has key(+0), so +0.0)
__device__ __forceinline__ double clf_threshold(unsigned key) {
    const unsigned v = ~key;
    return clf_widen((v & 0x80000000u) ? (v & 0x7fffffffu) : ~v);
}

struct ClfPoint { int tp, fp; unsigned key; };
// m points; tp / fp of the first and last point; last_ind = the first j with tp_j >= tp_last (sort.SearchFloat64s);
// other = 1 when some label is neither the lowest nor the highest label (typeOfTarget is not "binary"), or NaN
struct ClfSummary { int m, tp0, fp0, tp_last, fp_last, last_ind; unsigned lo, hi; int other; };

// an order-preserving key of a non-NaN label (-0 read as +0), for the label range; clf_label_of inverts it
__device__ __forceinline__ unsigned clf_label_key(float v) {
    if (v == 0.0f) v = 0.0f;
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float clf_label_of(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// lowest and highest non-NaN label (typeOfTarget's lo / hi); sum->lo / sum->hi start at 0xffffffff / 0
__global__ void k_clf_label_range(const float* __restrict__ y, long n, ClfSummary* __restrict__ sum) {
    unsigned lo = 0xffffffffu, hi = 0u;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float v = y[i];
        if (v != v) continue;
        const unsigned k = clf_label_key(v);
        lo = k < lo ? k : lo; hi = k > hi ? k : hi;
    }
    lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi);
    if ((threadIdx.x & 31) == 0) { atomicMin(&sum->lo, lo); atomicMax(&sum->hi, hi); }
}
// typeOfTarget's second loop: a label equal to neither lo nor hi (a NaN among them) makes the target not binary.
// With rewrite, y[i] becomes 1 where y[i] == 1 and 0 elsewhere, so that auc_positive reads pos_label = 1.
__global__ void k_clf_label_check(float* __restrict__ y, long n, ClfSummary* __restrict__ sum, int rewrite) {
    const float lo = clf_label_of(sum->lo), hi = clf_label_of(sum->hi);
    unsigned other = 0;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float v = y[i];
        other |= (v != lo && v != hi) ? 1u : 0u;
        if (rewrite) y[i] = v == 1.0f ? 1.0f : 0.0f;
    }
    other = __reduce_or_sync(0xffffffffu, other);
    if ((threadIdx.x & 31) == 0 && other) atomicOr(&sum->other, 1);
}

__global__ void k_clf_keys(const float* __restrict__ pred, const float* __restrict__ y, long n, double pos_label,
                           unsigned* __restrict__ keys, int* __restrict__ pos_flag) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        keys[i] = auc_score_key(pred[i]);
        pos_flag[i] = (double)y[i] == pos_label ? 1 : 0;                  // ranking.go:41
    }
}
// selects the last element of each threshold group in the sorted keys
struct ClfIsEnd {
    const unsigned* keys; long n;
    __device__ __forceinline__ bool operator()(const int& i) const { return i + 1 == n || keys[i + 1] != keys[i]; }
};
__global__ void k_clf_points(const unsigned* __restrict__ keys, const int* __restrict__ tp, const int* __restrict__ ends,
                             const int* __restrict__ d_m, long n, ClfPoint* __restrict__ pts, ClfSummary* __restrict__ sum) {
    const int m = *d_m, tp_last = tp[n - 1];
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < m; j += (long)gridDim.x * blockDim.x) {
        const int i = ends[j], t = tp[i];
        const ClfPoint p{t, i + 1 - t, keys[i]};
        pts[j] = p;
        if (j == 0) { sum->m = m; sum->tp0 = p.tp; sum->fp0 = p.fp; }
        if (j == m - 1) { sum->tp_last = p.tp; sum->fp_last = p.fp; }
        if (t >= tp_last && (j == 0 || tp[ends[j - 1]] < tp_last)) sum->last_ind = (int)j;
    }
}

// ROCCurve: the point (0, 0) prepended when fp_0 != 0 with threshold thresholds[0] + 1 (a NaN threshold kept as it is),
// fpr = fps * (1 / fpmax) and tpr = tps * (1 / tpmax) as floats.Scale does, all NaN when fpmax / tpmax is 0
__global__ void k_clf_roc(const ClfPoint* __restrict__ pts, const ClfSummary* __restrict__ sum, double* __restrict__ fpr,
                          double* __restrict__ tpr, double* __restrict__ thr) {
    const ClfSummary s = *sum;
    const int pre = s.fp0 != 0 ? 1 : 0;
    const double rf = 1.0 / (double)s.fp_last, rt = 1.0 / (double)s.tp_last;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o < (long)s.m + pre; o += (long)gridDim.x * blockDim.x) {
        double fp = 0.0, tp = 0.0, t;
        if (o < pre) {
            const double t0 = clf_threshold(pts[0].key);
            t = t0 != t0 ? t0 : __dadd_rn(t0, 1.0);
        } else {
            const ClfPoint p = pts[o - pre];
            fp = (double)p.fp; tp = (double)p.tp; t = clf_threshold(p.key);
        }
        fpr[o] = s.fp_last > 0 ? __dmul_rn(fp, rf) : clf_nan();
        tpr[o] = s.tp_last > 0 ? __dmul_rn(tp, rt) : clf_nan();
        thr[o] = t;
    }
}
// PrecisionRecallCurve: the points 0 … last_ind reversed, precision tp / (tp + fp), recall tp / tp_last (NaN when
// tp_last is 0), then (precision 1, recall 0) without a threshold
__global__ void k_clf_pr(const ClfPoint* __restrict__ pts, const ClfSummary* __restrict__ sum, double* __restrict__ prec,
                         double* __restrict__ rec, double* __restrict__ thr) {
    const ClfSummary s = *sum;
    for (long o = blockIdx.x * (long)blockDim.x + threadIdx.x; o <= (long)s.last_ind + 1; o += (long)gridDim.x * blockDim.x) {
        if (o > s.last_ind) { prec[o] = 1.0; rec[o] = 0.0; continue; }
        const ClfPoint p = pts[s.last_ind - o];
        prec[o] = __ddiv_rn((double)p.tp, (double)(p.tp + p.fp));
        rec[o] = s.tp_last > 0 ? __ddiv_rn((double)p.tp, (double)s.tp_last) : clf_nan();
        thr[o] = clf_threshold(p.key);
    }
}

// one AP term of ranking.go:218: (recall_j - recall_{j-1}) * precision_j with recall_{-1} = 0, from the counts of point
// j, the positives of point j - 1 (tpp) and the positives P of the whole curve
__device__ __forceinline__ double ap_term(int tp, int fp, int tpp, bool first, int P) {
    const double r = __ddiv_rn((double)tp, (double)P), rp = first ? 0.0 : __ddiv_rn((double)tpp, (double)P);
    return __dmul_rn(__dsub_rn(r, rp), __ddiv_rn((double)tp, (double)(tp + fp)));
}
// the AP terms of points 0 … last_ind as per-block double-double sums, each thread's terms in index order; with
// gauc_block_sum and a fixed grid the sum is the same bits on every call.  w counts the terms.
__global__ void k_ap_terms(const ClfPoint* __restrict__ pts, const ClfSummary* __restrict__ sum, GaucPart* __restrict__ part) {
    const ClfSummary s = *sum;
    GaucPart p{0.0, 0.0, 0, 0};
    if (s.tp_last > 0)
        for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j <= s.last_ind; j += (long)gridDim.x * blockDim.x) {
            const ClfPoint c = pts[j];
            dd_add(p.hi, p.lo, ap_term(c.tp, c.fp, j > 0 ? pts[j - 1].tp : 0, j == 0, s.tp_last), 0.0);
            p.w++;
        }
    p = gauc_block_sum(p);
    if (threadIdx.x == 0) part[blockIdx.x] = p;
}
// AP = the parts summed in block order; NaN with no positives (every recall is 0 / 0 in the reference)
__global__ void k_ap_final(const GaucPart* __restrict__ part, int nparts, const ClfSummary* __restrict__ sum, double* __restrict__ ap) {
    GaucPart p{0.0, 0.0, 0, 0};
    for (int b = threadIdx.x; b < nparts; b += blockDim.x) p = gauc_part_add(p, part[b]);
    p = gauc_block_sum(p);
    if (threadIdx.x == 0) *ap = sum->tp_last > 0 ? p.hi + p.lo : clf_nan();
}

// ---- grouped AP (ctr_group_average_precision): GAUC's (group, score) order and scan, AP terms per group -------------
struct GapAgg { double hi, lo; int n, pos; };
struct GapAggOp {
    __device__ __forceinline__ GapAgg operator()(GapAgg a, const GapAgg& b) const {
        dd_add(a.hi, a.lo, b.hi, b.lo);
        a.n += b.n; a.pos += b.pos;
        return a;
    }
};
// each group's positives P_g, stored at the group's first element (the terms need them before the reduction)
__global__ void k_gap_pos(const unsigned long long* __restrict__ gkey, const GaucScan* __restrict__ s, long n, int* __restrict__ gpos) {
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < n; j += (long)gridDim.x * blockDim.x) {
        if (j + 1 < n && gkey[j + 1] == gkey[j]) continue;
        const GaucScan e = s[j];
        gpos[e.gs] = e.tp - (e.gs > 0 ? s[e.gs - 1].tp : 0);
    }
}
// each threshold-group end adds its AP term, counted from its group's start (nothing in a group without positives).
// The terms after the group's last_ind are (1 - 1) * precision = 0 exactly, so they need no cut.
__global__ void k_gap_terms(const unsigned long long* __restrict__ gkey, const unsigned long long* __restrict__ packed,
                            const GaucScan* __restrict__ s, const int* __restrict__ gpos, long n, GapAgg* __restrict__ val) {
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < n; j += (long)gridDim.x * blockDim.x) {
        const unsigned long long v = packed[j];
        double term = 0.0;
        if (j + 1 == n || gkey[j + 1] != gkey[j] || (packed[j + 1] >> 32) != (v >> 32)) {
            const GaucScan e = s[j];
            const int P = gpos[e.gs];
            if (P > 0) {
                const int base = e.gs > 0 ? s[e.gs - 1].tp : 0;
                const int tp = e.tp - base, fp = (int)(j - e.gs + 1) - tp;
                const bool first = e.ts == e.gs;
                term = ap_term(tp, fp, first ? 0 : s[e.ts - 1].tp - base, first, P);
            }
        }
        val[j] = {term, 0.0, 1, (int)(v & 1)};
    }
}
// per group: AP_g (NaN when P_g = 0) and the per-group outputs the caller asked for; per block: its part of the sum of
// AP_g over the used groups, with w = used so that k_gauc_final's (hi + lo) / w is the unweighted mean
__global__ void k_gap_groups(const unsigned long long* __restrict__ uniq, const GapAgg* __restrict__ agg, const int* __restrict__ runs,
                             long long* __restrict__ out_group, int* __restrict__ out_n, int* __restrict__ out_pos,
                             double* __restrict__ out_ap, GaucPart* __restrict__ part) {
    const long R = *runs;
    GaucPart p{0.0, 0.0, 0, 0};
    for (long g = blockIdx.x * (long)blockDim.x + threadIdx.x; g < R; g += (long)gridDim.x * blockDim.x) {
        const GapAgg a = agg[g];
        const double ap = a.pos > 0 ? a.hi + a.lo : clf_nan();
        if (out_group) out_group[g] = (long long)(uniq[g] ^ 0x8000000000000000ull);
        if (out_n) out_n[g] = a.n;
        if (out_pos) out_pos[g] = a.pos;
        if (out_ap) out_ap[g] = ap;
        if (a.pos > 0) { dd_add(p.hi, p.lo, ap, 0.0); p.w++; p.used++; }
    }
    p = gauc_block_sum(p);
    if (threadIdx.x == 0) part[blockIdx.x] = p;
}

}  // namespace ctr
