// auc.cuh — utils.RocAuc32 on the device (util.go:131-148 → nn/metrics/ranking.go:13-150):
// labels binarised at 0.5, scores sorted descending, equal scores form one threshold group
// (ranking.go:27-35), cumulative tp/fp, trapezoid over the normalised curve (ranking.go:106-118).
// SURVEY.md §8(f) row f4 (on-device eval).  CUB does the sort/scans; the curve logic is below.
#pragma once
#include "common.cuh"
#include "owner.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace ctr {

__global__ void k_auc_keys(const float* __restrict__ pred, const float* __restrict__ y, long n,
                           unsigned* __restrict__ keys, int* __restrict__ pos_flag) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float p = pred[i];
        if (p == 0.0f) p = 0.0f;                       // -0 == +0 compare equal in the reference
        unsigned u = __float_as_uint(p);
        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u); // ascending-order-preserving
        keys[i] = ~u;                                   // ascending sort of ~u == descending scores
        pos_flag[i] = y[i] > 0.5f ? 1 : 0;              // util.go:134-138
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

}  // namespace ctr
