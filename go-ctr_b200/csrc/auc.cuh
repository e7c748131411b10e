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

}  // namespace ctr
