// metrics.cuh — nn/metrics/classification.go and regression.go on the device: AccuracyScore, ConfusionMatrix and
// PrecisionRecallFScoreSupport (with LabelEncoder, feature/preprocessing/label.go:273-340), and the column sums behind
// R2Score / MeanSquaredError / MeanAbsoluteError (mlp64.cuh's k_mlp64_r2_part / k_mlp64_r2_fold, generalised).
// Determinism: unweighted counts are 64-bit integers (atomics on integers are exact in any order); every weighted or
// floating-point sum is a double-double over fixed partitions, combined in a fixed order.  No float atomics.
#pragma once
#include "common.cuh"
#include "auc.cuh"
#include "mlp64.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>

namespace ctr {

// ---- class discovery (LabelEncoder.Fit :288-321, LabelBinarizer64.Fit basemlp64.go:1294-1313) -----------------------
// The keys are the labels with −0 made +0 (both encoders compare with ==, so ±0 are one class).  A stable radix sort of
// (key, position), then UniqueByKey: k0 receives the distinct keys ascending, p0 the first position of each in sample
// order, *count their number.  With tmp == nullptr only *bytes is set, to the scratch both steps need.
template <class T>
cudaError_t class_sort_unique(void* tmp, size_t* bytes, T* k0, T* k1, long* p0, long* p1, long* count, long n, cudaStream_t st) {
    cudaError_t e;
    if (!tmp) {
        size_t a = 0, b = 0;
        if ((e = cub::DeviceRadixSort::SortPairs(nullptr, a, (const T*)nullptr, (T*)nullptr, (const long*)nullptr, (long*)nullptr, n, 0, (int)sizeof(T) * 8, st)) != cudaSuccess) return e;
        if ((e = cub::DeviceSelect::UniqueByKey(nullptr, b, (const T*)nullptr, (const long*)nullptr, (T*)nullptr, (long*)nullptr, (long*)nullptr, n, st)) != cudaSuccess) return e;
        *bytes = std::max<size_t>(std::max(a, b), 1);
        return cudaSuccess;
    }
    if ((e = cub::DeviceRadixSort::SortPairs(tmp, *bytes, k0, k1, p0, p1, n, 0, (int)sizeof(T) * 8, st)) != cudaSuccess) return e;
    return cub::DeviceSelect::UniqueByKey(tmp, *bytes, k1, p1, k0, p0, count, n, st);
}
// after class_sort_unique: value[c] = Y[first[c]] for c < min(*count, cap), so each class keeps the sign of its first
// occurrence (LabelEncoder inserts the first value it meets; the binarizer's map keeps the first key)
template <class T>
__global__ void __launch_bounds__(256)
k_class_values(const T* __restrict__ Y, const long* __restrict__ first, const long* __restrict__ count, long cap, double* __restrict__ value) {
    const long c_n = *count < cap ? *count : cap;
    for (long c = blockIdx.x * (long)blockDim.x + threadIdx.x; c < c_n; c += (long)gridDim.x * blockDim.x) value[c] = (double)Y[first[c]];
}
// class_lower_bound (mlp64.cuh) is sort.SearchFloat64s, the encoding of both.

// ---- AccuracyScore (classification.go:12-34) ----------------------------------------------------------------------
// kMetParts contiguous row ranges, one block each; the block's sum in a fixed order (gauc_block_sum), the parts folded in
// order by one block.  A row is correct when every column compares equal with ==.
constexpr int kMetParts = 512;
struct MetAccPart { GaucPart num, den; int bad; };   // num.w = correct rows (unweighted); bad: a weight is not finite

__global__ void __launch_bounds__(256)
k_met_acc_part(const double* __restrict__ yt, const double* __restrict__ yp, const double* __restrict__ w, long n, int no,
               MetAccPart* __restrict__ part) {
    const long per = (n + kMetParts - 1) / kMetParts, r0 = blockIdx.x * per, r1 = min(n, r0 + per);
    GaucPart num{0.0, 0.0, 0, 0}, den{0.0, 0.0, 0, 0};
    int bad = 0;
    for (long r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
        const long o = r * (long)no;
        bool eq = true;
        for (int j = 0; j < no && eq; j++) eq = yt[o + j] == yp[o + j];
        if (!w) { num.w += eq; continue; }
        const double wi = w[r];
        bad |= !isfinite(wi);
        if (eq) dd_add(num.hi, num.lo, wi, 0.0);
        dd_add(den.hi, den.lo, wi, 0.0);
    }
    num = gauc_block_sum(num);
    __syncthreads();
    den = gauc_block_sum(den);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) part[blockIdx.x] = MetAccPart{num, den, bad};
}
// out[0] = N / D (normalize) or N, out[1] = 1 when some weight is not finite.  One block.
__global__ void __launch_bounds__(256)
k_met_acc_final(const MetAccPart* __restrict__ part, long n, bool weighted, int normalize, double* __restrict__ out) {
    GaucPart num{0.0, 0.0, 0, 0}, den{0.0, 0.0, 0, 0};
    int bad = 0;
    for (int p = threadIdx.x; p < kMetParts; p += blockDim.x) {
        num = gauc_part_add(num, part[p].num); den = gauc_part_add(den, part[p].den); bad |= part[p].bad;
    }
    num = gauc_block_sum(num);
    __syncthreads();
    den = gauc_block_sum(den);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) {
        const double N = weighted ? num.hi : (double)num.w, D = weighted ? den.hi : (double)n;
        out[0] = normalize ? N / D : N;
        out[1] = bad;
    }
}

// ---- ConfusionMatrix / PrecisionRecallFScoreSupport (classification.go:74-178) -----------------------------------
// First positions of the refusals, UINT64_MAX when absent
struct MetFlags { unsigned long long nan_true, nan_pred, bad_weight, above; };

// the class keys of y_true (−0 → +0) and their positions; the refusal flags of the inputs
__global__ void __launch_bounds__(256)
k_met_keys(const double* __restrict__ yt, const double* __restrict__ yp, const double* __restrict__ w, long n,
           double* __restrict__ key, long* __restrict__ pos, MetFlags* __restrict__ fl) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const double t = yt[i];
        if (t != t) atomicMin(&fl->nan_true, (unsigned long long)i);
        if (yp[i] != yp[i]) atomicMin(&fl->nan_pred, (unsigned long long)i);
        if (w && !isfinite(w[i])) atomicMin(&fl->bad_weight, (unsigned long long)i);
        key[i] = t == 0.0 ? 0.0 : t;
        pos[i] = i;
    }
}

// Shared-memory histograms hold at most this many 64-bit counters (32 KB)
constexpr int kMetSmemCounts = 4096;
// Classes kept in shared memory for the binary search when C is at most this (16 KB; with the counters, 48 KB at most)
constexpr int kMetSmemClasses = 2048;

// LabelEncoder.Transform (:324-339) of y_true and y_pred, and the unweighted counts.  cell[i] = t·C + p (t, p the class
// indices); pcls[i] = p.  cm (may be null) counts each cell, cls[0, C) the diagonal, cls[C, 2C) the rows (true class),
// cls[2C, 3C) the columns (predicted class).  A prediction above the largest class is flagged (the call refuses) and
// counted nowhere.  kShared: the classes and the counters in shared memory (C ≤ kMetSmemClasses for the classes;
// (cm ? C² : 0) + 3C ≤ kMetSmemCounts for the counters, else the counters are global atomics).
template <bool kSharedClasses, bool kSharedCounts>
__global__ void __launch_bounds__(256)
k_met_encode(const double* __restrict__ yt, const double* __restrict__ yp, long n, const double* __restrict__ classes, int C,
             unsigned long long* __restrict__ cell, unsigned long long* __restrict__ pcls, unsigned long long* __restrict__ cm,
             unsigned long long* __restrict__ cls, MetFlags* __restrict__ fl) {
    extern __shared__ double met_smem[];
    double* s_cls = met_smem;
    unsigned long long* s_cnt = (unsigned long long*)(met_smem + (kSharedClasses ? C : 0));
    const long cmc = cm ? (long)C * C : 0, ncnt = cmc + 3L * C;
    if (kSharedClasses) for (int c = threadIdx.x; c < C; c += blockDim.x) s_cls[c] = classes[c];
    if (kSharedCounts) for (long c = threadIdx.x; c < ncnt; c += blockDim.x) s_cnt[c] = 0;
    if (kSharedClasses || kSharedCounts) __syncthreads();
    const double* cl = kSharedClasses ? s_cls : classes;
    unsigned long long* cnt_cm = kSharedCounts ? s_cnt : cm;
    unsigned long long* cnt_cls = kSharedCounts ? s_cnt + cmc : cls;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const int t = class_lower_bound(cl, C, yt[i]);
        int p = class_lower_bound(cl, C, yp[i]);
        if (p >= C) { atomicMin(&fl->above, (unsigned long long)i); cell[i] = 0; pcls[i] = 0; continue; }
        cell[i] = (unsigned long long)t * C + p;
        pcls[i] = p;
        if (cm) atomicAdd(cnt_cm + (long)t * C + p, 1ull);
        if (t == p) atomicAdd(cnt_cls + t, 1ull);
        atomicAdd(cnt_cls + C + t, 1ull);
        atomicAdd(cnt_cls + 2L * C + p, 1ull);
    }
    if (!kSharedCounts) return;
    __syncthreads();
    for (long c = threadIdx.x; c < ncnt; c += blockDim.x) {
        const unsigned long long v = s_cnt[c];
        if (v) atomicAdd(c < cmc ? cm + c : cls + (c - cmc), v);
    }
}

// Weighted sums, after a stable sort of (key, weight) pairs: segment = a run of equal key / div.  Pass 1 cuts the
// array into tiles of kMetTile; the first element of every tile and of every segment within it starts a piece, summed
// as a double-double in array order up to the segment's or the tile's end.  Pass 2 adds each segment's pieces in tile
// order.  The order depends only on the sorted keys, so the same inputs give the same bits.
constexpr int kMetTile = 2048;
__global__ void __launch_bounds__(256)
k_met_seg_piece(const unsigned long long* __restrict__ key, unsigned long long div, const double* __restrict__ w, long n,
                double2* __restrict__ piece) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const unsigned long long k = key[i] / div;
        if (i % kMetTile != 0 && key[i - 1] / div == k) continue;
        const long end = min(n, (i / kMetTile + 1) * kMetTile);
        double hi = 0.0, lo = 0.0;
        for (long j = i; j < end && key[j] / div == k; j++) dd_add(hi, lo, w[j], 0.0);
        piece[i] = make_double2(hi, lo);
    }
}
struct MetSegHead {
    const unsigned long long* key; unsigned long long div;
    __device__ __forceinline__ bool operator()(const long& i) const { return i == 0 || key[i] / div != key[i - 1] / div; }
};
// pass 2 over the R segment heads: the segment's sum goes to out[key / div] (the dense matrix or a per-class array),
// and, when diag is non-null, a cell t·C + p with t == p also to diag[t]
__global__ void __launch_bounds__(256)
k_met_seg_total(const unsigned long long* __restrict__ key, unsigned long long div, const long* __restrict__ heads,
                const int* __restrict__ nheads, long n, const double2* __restrict__ piece, int C, double* __restrict__ out,
                double* __restrict__ diag) {
    const long R = *nheads;
    for (long r = blockIdx.x * (long)blockDim.x + threadIdx.x; r < R; r += (long)gridDim.x * blockDim.x) {
        const long s = heads[r], e = r + 1 < R ? heads[r + 1] : n;
        double hi = piece[s].x, lo = piece[s].y;
        for (long t = (s / kMetTile + 1) * kMetTile; t < e; t += kMetTile) dd_add(hi, lo, piece[t].x, piece[t].y);
        const unsigned long long k = key[s] / div;
        if (out) out[k] = hi;
        if (diag && k / C == k % C) diag[k / C] = hi;
    }
}

// prfs of PrecisionRecallFScoreSupport (:83-101), every operation rounded on its own as the reference's Go
__device__ __forceinline__ void met_prfs(double tp, double truesum, double predsum, double beta, double& p, double& r, double& f) {
    p = predsum > 0.0 ? __ddiv_rn(tp, predsum) : 0.0;
    r = truesum > 0.0 ? __ddiv_rn(tp, truesum) : 0.0;
    const double b2 = __dmul_rn(beta, beta), den = __dadd_rn(__dmul_rn(b2, p), r);
    f = den > 0.0 ? __ddiv_rn(__dmul_rn(__dmul_rn(__dadd_rn(1.0, b2), p), r), den) : 0.0;
}
enum { kMetMacro = 0, kMetMicro = 1, kMetWeighted = 2 };   // CTR_AVERAGE_*
// One block.  Per class c: tp, truesum, predsum (weighted: the double arrays; else the counts of k_met_encode), p, r,
// f and the unweighted support, into per_class [C, 4] when non-null.  out[0..3] = the class pos_label's (p, r, f,
// support), or with pos_label < 0 the average: macro / weighted = the mean of the classes' p, r, f (stat.Mean with no
// weights, :116-131), micro = prfs of the summed tp, truesum and predsum; support 0.  Sums are double-doubles in a fixed
// order.
__global__ void __launch_bounds__(256)
k_met_prf(const unsigned long long* __restrict__ cls, const double* __restrict__ tpw, const double* __restrict__ truew,
          const double* __restrict__ predw, int C, double beta, int pos_label, int average, double* __restrict__ per_class,
          double* __restrict__ out) {
    const bool weighted = tpw != nullptr;
    GaucPart a{0.0, 0.0, 0, 0}, b{0.0, 0.0, 0, 0}, c3{0.0, 0.0, 0, 0};
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const double tp = weighted ? tpw[c] : (double)cls[c];
        const double ts = weighted ? truew[c] : (double)cls[C + c];
        const double ps = weighted ? predw[c] : (double)cls[2L * C + c];
        double p, r, f;
        met_prfs(tp, ts, ps, beta, p, r, f);
        const double s = (double)cls[C + c];
        if (per_class) { double* o = per_class + 4L * c; o[0] = p; o[1] = r; o[2] = f; o[3] = s; }
        if (c == pos_label) { out[0] = p; out[1] = r; out[2] = f; out[3] = s; }
        if (average == kMetMicro) { dd_add(a.hi, a.lo, tp, 0.0); dd_add(b.hi, b.lo, ts, 0.0); dd_add(c3.hi, c3.lo, ps, 0.0); }
        else { dd_add(a.hi, a.lo, p, 0.0); dd_add(b.hi, b.lo, r, 0.0); dd_add(c3.hi, c3.lo, f, 0.0); }
    }
    if (pos_label >= 0) return;
    a = gauc_block_sum(a); __syncthreads();
    b = gauc_block_sum(b); __syncthreads();
    c3 = gauc_block_sum(c3);
    if (threadIdx.x != 0) return;
    if (average == kMetMicro) {
        double p, r, f;
        met_prfs(a.hi, b.hi, c3.hi, beta, p, r, f);
        out[0] = p; out[1] = r; out[2] = f;
    } else {
        out[0] = a.hi / (double)C; out[1] = b.hi / (double)C; out[2] = c3.hi / (double)C;
    }
    out[3] = 0.0;
}
// the counted matrix as doubles (the unweighted ConfusionMatrix)
__global__ void __launch_bounds__(256)
k_met_cm_f64(const unsigned long long* __restrict__ cm, long cells, double* __restrict__ out) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < cells; i += (long)gridDim.x * blockDim.x) out[i] = (double)cm[i];
}

// ---- MLPClassifier.Score (multilayer_perceptron.go:127-133 → AccuracyScore64, basemlp64.go:1143-1155) --------------
// rows of the output layer h [rows, no] against the labels Y [rows]: without classes the float64 probability itself
// must equal the label; with classes the predicted class (MaxIdx64, as k_mlp64_predict_label) must.  *hits += the
// block's count (an integer atomic: any order gives the same count).
__global__ void __launch_bounds__(256)
k_mlp64_acc_count(const double* __restrict__ h, int rows, int no, const double* __restrict__ classes, const float* __restrict__ Y,
                  unsigned long long* __restrict__ hits) {
    GaucPart c{0.0, 0.0, 0, 0};
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        const double* z = h + (long)r * no;
        double pred = z[0];
        if (classes) {
            int mi = 0;
            for (int j = 1; j < no; j++) if (z[j] > z[mi]) mi = j;
            pred = classes[mi];
        }
        c.w += pred == (double)Y[r];
    }
    c = gauc_block_sum(c);
    if (threadIdx.x == 0 && c.w) atomicAdd(hits, (unsigned long long)c.w);
}

}  // namespace ctr
