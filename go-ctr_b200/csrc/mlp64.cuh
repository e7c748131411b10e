// mlp64.cuh — model/mlp on the device (SURVEY.md §8a row a11, BASELINE configs[0]): the float64 scikit-learn-style
// MLP classifier the reference's default path trains (main.go:42-52 → model/mlp/mlp.go:45-65 →
// nn/neural_network/basemlp64.go `BaseMultilayerPerceptron64`: fit :484, fitStochastic :729, backprop :340,
// forwardPass :259, AdamOptimizer64.updateParams :1075), and the regressor over the same network (MLPRegressor,
// multilayer_perceptron.go:9-71: identity output on square_loss, dense multi-column targets, R²; see "the regressor").
//
// One hidden layer or more, biases, relu / logistic / identity / tanh hidden activation, logistic output + binary_log_loss with the
// probabilities clipped to (nextafter(0,1), nextafter(1,0)) (:180-195) — or, for labels that are not all 0 or 1, a
// softmax output + log_loss over the label classes (see "labels that are not all 0 or 1" below) — L2 term alpha/(2n)·Σw² in the loss (:361) and
// alpha/n·w in the coefficient gradients (:327), Adam whose beta powers advance once per parameter ELEMENT
// (:1082-1090 — the bias correction is gone within the first call) or SGD with momentum / Nesterov (:1024-1039),
// weight decay of the whole packed vector before every minibatch (:342-346), minibatches of 200 visited through a per-epoch
// shuffle (:788), tol / n_iter_no_change stopping (:826-840,886-890).
//
// All arithmetic is float64 (the reference's: gonum Dgemm).  A step is ~17 MFLOP — launch-latency, not throughput,
// bound: four kernels per minibatch, each thread owns one output element and walks its reduction in the oracle's
// order (k ascending), so the only differences against the CPU restatement are FMA contraction and libm ulps.
// Parameter layout = the reference's packed vector (:459-463): per layer [intercepts(fo) | coefs(fi x fo row-major)].
#pragma once
#include "common.cuh"

namespace ctr {

constexpr int kMlpMaxLayers = 8;
enum { MLP_ACT_RELU = 0, MLP_ACT_LOGISTIC = 1, MLP_ACT_IDENTITY = 2, MLP_ACT_TANH = 3 };

struct Mlp64Dims {
    int n_layers;                    // len(layerUnits) = hidden layers + 2
    int units[kMlpMaxLayers];        // [nFeatures, hidden..., nOutputs]
    long off[kMlpMaxLayers];         // offset of layer l's [intercepts | coefs] in the packed vector
    int hidden_act;
    // OutActivation (:418-430): MLP_ACT_LOGISTIC, or MLP_ACT_IDENTITY for the regressor's identity output and for a
    // softmax output, whose pre-activations k_mlp64_softmax then normalises
    int out_act;
};

__device__ __forceinline__ double mlp64_logistic(double z) { return 1.0 / (1.0 + exp(-z)); }   // :82-88
// the activation of layer l+1 on its pre-activation z: the hidden activation, or the output layer's (last)
__device__ __forceinline__ double mlp64_act(double z, const Mlp64Dims& d, bool last) {
    const int act = last ? d.out_act : d.hidden_act;
    if (act == MLP_ACT_LOGISTIC) z = mlp64_logistic(z);
    else if (act == MLP_ACT_RELU) z = z < 0.0 ? 0.0 : z;                     // :96-104
    else if (act == MLP_ACT_TANH) z = tanh(-z);                              // :88-94 — the argument is negated
    return z;
}

// hidden / output layer l -> l+1 for the m rows of the minibatch: out[r, j] = act(b[j] + sum_k in[r, k] * W[k, j]).
// in == nullptr: layer 0 reads the dataset rows X[idx[r]] (the shuffled visiting order, basemlp64.go:788-808).
// kLogit: the output layer writes its pre-activation z, the logit (ctr_mlp_recommend_topk ranks by it).
template <bool kLogit = false>
__global__ void __launch_bounds__(256)
k_mlp64_layer(const double* __restrict__ params, Mlp64Dims d, int l, const double* __restrict__ X, long ldx, const long* __restrict__ idx,
              const double* __restrict__ in, double* __restrict__ out, int m) {
    const int fi = d.units[l], fo = d.units[l + 1];
    const double* b = params + d.off[l];
    const double* W = b + fo;
    const bool last = (l + 1 == d.n_layers - 1);
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < (long)m * fo; t += (long)gridDim.x * blockDim.x) {
        const int r = (int)(t / fo), j = (int)(t % fo);
        const double* a = in ? in + (long)r * fi : X + (idx ? idx[r] : (long)r) * ldx;
        double z = 0.0;
        for (int k = 0; k < fi; k++) z += a[k] * W[(long)k * fo + j];
        z += b[j];                                                              // addIntercepts64 :205
        if (!(kLogit && last)) z = mlp64_act(z, d, last);
        out[t] = z;
    }
}

// ---- ctr_mlp_recommend_topk: one user against every item row ------------------------------------------------------
// Layer 0's input is [user_feat (uP) | S window rows (S·D) | item emb (D) | item feat (cF)]; only the last D + cF columns
// depend on the item.  k_mlp64_layer's chain for output j is z = 0; z += a[k]·W0[k, j] for k ascending (one DFMA each);
// z += b[j].  So the user's partial sum over the first pcols = uP + S·D columns is computed once (k_mlp64_prefix) and each
// item continues the same chain from it over its own columns (k_mlp64_rec_layer0): the same DFMAs in the same order, so
// the same bits as the predict route.  No DMMA: its accumulation order differs.

// pre[j] = sum_{k < pcols} x[k]·W0[k, j], x = [USER_FEAT row urow | ITEM_EMB rows hist[0, S)], widened from float32 as
// k_gather_rows<double> widens them.  A missing row (urow == nullptr, a history row outside [0, r.n_emb)) is zeros, and
// its columns are walked like any other: 0·inf stays NaN, as on the predict route.  The ITEM_EMB rows are r.emb's;
// PEER (a row-sharded ITEM_EMB) reads them through emb_src<true> as k_attn_fwd_user<PEER> stages the DIN history: the
// hot rows from this rank's replica, the rest from their owners.  The DFMA chain is the same in both forms.
template <bool PEER>
__global__ void __launch_bounds__(128)
k_mlp64_prefix(const double* __restrict__ params, Mlp64Dims d, const float* __restrict__ urow, int uP,
               RowSrc r, const int* __restrict__ hist, int S, int D, double* __restrict__ pre) {
    const int fo = d.units[1];
    const double* W = params + d.off[0] + fo;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < fo; j += gridDim.x * blockDim.x) {
        double z = 0.0;
        long k = 0;
        for (int c = 0; c < uP; c++, k++) z += (urow ? (double)__ldg(urow + c) : 0.0) * W[k * fo + j];
        for (int s = 0; s < S; s++) {
            const int row = __ldg(hist + s);
            const float* e = row_ok(row, r.n_emb) ? (PEER ? emb_src<true>(r, row) : r.emb + (long)row * r.lde) : nullptr;
            for (int c = 0; c < D; c++, k++) z += (e ? (double)__ldg(e + c) : 0.0) * W[k * fo + j];
        }
        pre[j] = z;
    }
}

constexpr int kRecTile = 128;    // items per tile: lane l of a warp owns items l, l + 32, l + 64, l + 96 of it
constexpr int kRecJ = 4;         // hidden units a warp carries at a time
// pitch (floats) of the tile's item columns in shared memory: odd, so the lanes' strided reads hit 32 distinct banks
__host__ __device__ inline int rec_tile_pitch(int T) { return T | 1; }
__host__ __device__ inline int rec_units_pad(int H) { return (H + kRecJ - 1) / kRecJ * kRecJ; }
// dynamic shared memory: [T][Hp] float64 slice of W0 (SMEM_W only), then [kRecTile][pitch] float32 item columns
__host__ inline size_t rec_layer0_smem(int T, int H, bool smem_w) {
    return (smem_w ? (size_t)T * rec_units_pad(H) * 8 : 0) + (size_t)kRecTile * rec_tile_pitch(T) * 4;
}

// out[b, j] = act(pre[j] + sum_{c < T} x_b[c]·W0[pcols + c, j] + b[j]) for items b = row0 .. row0 + n - 1, T = D + cF,
// x_b = [ITEM_EMB row | ITEM_FEAT row (zeros past n_ifeat)].  The output layer (a network without hidden layers) writes
// the logit.  A CTA stages the W0 rows of the item columns once (SMEM_W; else they are read through L1), then walks
// tiles of kRecTile items: the tile's columns are read from HBM once, coalesced, and each warp takes kRecJ units at a
// time for all the tile's items, so a W0 value in shared memory is a broadcast and an item value a conflict-free read.
// emb holds the rows this GPU scores: the whole table, or on a row-sharded ITEM_EMB this rank's shard (local row l is
// global row l·world + rank).  Item row l's ITEM_FEAT row is l·fworld + frank: fworld = world, frank = rank for a
// replicated ITEM_FEAT beside a sharded ITEM_EMB (n_ifeat its global rows); 1 and 0 for a sharded ITEM_FEAT (n_ifeat
// its local rows) and on one GPU.
template <bool SMEM_W>
__global__ void __launch_bounds__(256)
k_mlp64_rec_layer0(const double* __restrict__ params, Mlp64Dims d, const double* __restrict__ pre, int pcols,
                   const float* __restrict__ emb, long lde, const float* __restrict__ ifeat, long ldi, long n_ifeat, int fworld, int frank,
                   int D, int cF, long row0, int n, double* __restrict__ out) {
    extern __shared__ __align__(16) char smem_raw[];
    const int H = d.units[1], Hp = rec_units_pad(H), T = D + cF, Tp = rec_tile_pitch(T);
    const bool last = d.n_layers == 2;
    const double* b = params + d.off[0];
    const double* W = b + H + (long)pcols * H;                 // W0 rows pcols .. pcols + T - 1
    double* ws = reinterpret_cast<double*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + (SMEM_W ? (size_t)T * Hp * 8 : 0));
    if (SMEM_W)
        for (int i = threadIdx.x; i < T * Hp; i += blockDim.x) {
            const int k = i / Hp, j = i - k * Hp;
            ws[i] = j < H ? W[(long)k * H + j] : 0.0;
        }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int ntiles = (n + kRecTile - 1) / kRecTile;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int b0 = t * kRecTile, nb = min(kRecTile, n - b0);
        __syncthreads();                                        // the previous tile has been read
        for (int i = threadIdx.x; i < kRecTile * T; i += blockDim.x) {
            const int r = i / T, c = i - r * T;
            float v = 0.0f;
            if (r < nb) {
                const long row = row0 + b0 + r, frow = row * fworld + frank;
                if (c < D) v = __ldg(emb + row * lde + c);
                else if (frow < n_ifeat) v = __ldg(ifeat + frow * ldi + (c - D));
            }
            xs[r * Tp + c] = v;
        }
        __syncthreads();
        for (int j0 = warp * kRecJ; j0 < H; j0 += nw * kRecJ) {
            double acc[4][kRecJ];
#pragma unroll
            for (int jj = 0; jj < kRecJ; jj++) {
                const double p = j0 + jj < H ? pre[j0 + jj] : 0.0;
#pragma unroll
                for (int r = 0; r < 4; r++) acc[r][jj] = p;
            }
#pragma unroll 2
            for (int k = 0; k < T; k++) {
                double w[kRecJ];
                if (SMEM_W) {
                    const double2 w01 = *reinterpret_cast<const double2*>(ws + (size_t)k * Hp + j0);
                    const double2 w23 = *reinterpret_cast<const double2*>(ws + (size_t)k * Hp + j0 + 2);
                    w[0] = w01.x; w[1] = w01.y; w[2] = w23.x; w[3] = w23.y;
                } else {
#pragma unroll
                    for (int jj = 0; jj < kRecJ; jj++) w[jj] = j0 + jj < H ? __ldg(W + (long)k * H + j0 + jj) : 0.0;
                }
#pragma unroll
                for (int r = 0; r < 4; r++) {
                    const double x = (double)xs[(lane + 32 * r) * Tp + k];
#pragma unroll
                    for (int jj = 0; jj < kRecJ; jj++) acc[r][jj] = fma(x, w[jj], acc[r][jj]);
                }
            }
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const int i = lane + 32 * r;
                if (i >= nb) continue;
#pragma unroll
                for (int jj = 0; jj < kRecJ; jj++) {
                    const int j = j0 + jj;
                    if (j >= H) continue;
                    const double z = acc[r][jj] + b[j];
                    out[(long)(b0 + i) * H + j] = last ? z : mlp64_act(z, d, false);
                }
            }
        }
    }
}

// the tail every loss kernel shares: ll is the data term; adds the L2 term (:361) over sumCoefSquares (:311-319) and
// writes the minibatch loss and the epoch accumulator acc += loss * m (:805).  red is the block's [256] scratch.
__device__ __forceinline__ void mlp64_loss_finish(const double* __restrict__ params, const Mlp64Dims& d, double* red, double ll, int m,
                                                  double alpha, double* __restrict__ loss_out, double* __restrict__ epoch_acc) {
    __syncthreads();
    double sq = 0.0;
    for (int l = 0; l + 1 < d.n_layers; l++) {
        const double* W = params + d.off[l] + d.units[l + 1];
        const long cnt = (long)d.units[l] * d.units[l + 1];
        for (long i = threadIdx.x; i < cnt; i += 256) sq += W[i] * W[i];
    }
    red[threadIdx.x] = sq; __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) {
        const double loss = ll + (0.5 * alpha) * red[0] / (double)m;
        *loss_out = loss;
        if (epoch_acc) *epoch_acc += loss * (double)m;
    }
}

// loss of the minibatch (binary_log_loss :180-195 + L2 :361), delta of the output layer (h - y, :373-381), and the
// epoch accumulator acc += loss * m (:805).  One block; fixed-order reductions.
__global__ void __launch_bounds__(256)
k_mlp64_loss(const double* __restrict__ params, Mlp64Dims d, const double* __restrict__ h, const float* __restrict__ Y, const long* __restrict__ idx,
             int m, double alpha, double* __restrict__ delta, double* __restrict__ loss_out, double* __restrict__ epoch_acc) {
    __shared__ double red[256];
    const int no = d.units[d.n_layers - 1];
    const double hmin = 4.9406564584124654e-324, hmax = 0.99999999999999989;     // nextafter(0,1), nextafter(1,0)
    double s = 0.0;
    for (int i = threadIdx.x; i < m * no; i += 256) {
        const int r = i / no, j = i % no;
        const double y = (double)Y[(idx ? idx[r] : (long)r) * no + j];
        double hv = h[i];
        delta[i] = hv - y;
        hv = hv < hmin ? hmin : (hv > hmax ? hmax : hv);
        s += -y * log(hv) - (1.0 - y) * log1p(-hv);
    }
    red[threadIdx.x] = s; __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    mlp64_loss_finish(params, d, red, red[0] / (double)m, m, alpha, loss_out, epoch_acc);
}

// ---- labels that are not all 0 or 1 (BaseMultilayerPerceptron64.Fit :578-598) -----------------------------------
// LabelBinarizer64(0, 1) (:1294-1351): the classes are the distinct label values in ascending order, the target of a
// sample is the one-hot row of its class, and C >= 2 classes make a softmax output trained on log_loss (:504-511).
// The targets are never materialised: each sample carries its class index (int32), found by a binary search.
constexpr int kMlpMaxClasses = 1024;
// what class discovery hands the host in one copy
struct Mlp64Classes {
    double value[kMlpMaxClasses];    // the first min(count, kMlpMaxClasses) classes, ascending
    long count;                      // the number of distinct labels (written by cub::DeviceSelect::UniqueByKey)
    int nan;                         // a NaN label was seen
};

// discovery pass 1: sort keys and positions.  −0 becomes +0, so ±0 fall into one run (the reference's map compares with
// ==); a NaN label is flagged and the host refuses the fit.
__global__ void __launch_bounds__(256)
k_mlp64_label_keys(const float* __restrict__ Y, long n, float* __restrict__ key, long* __restrict__ pos, Mlp64Classes* __restrict__ res) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float y = Y[i];
        if (y != y) res->nan = 1;
        key[i] = y == 0.0f ? 0.0f : y;
        pos[i] = i;
    }
}
// discovery pass 2 is class_sort_unique and pass 3 k_class_values (metrics.cuh), shared with ctr_confusion_matrix.
// sort.SearchFloat64s (label.go:330): the first class >= y, C when y is above every class (or NaN)
__device__ __forceinline__ int class_lower_bound(const double* __restrict__ classes, int C, double y) {
    int lo = 0, hi = C;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (classes[mid] < y) lo = mid + 1; else hi = mid; }
    return lo;
}
// cls[i] = the index of label i in classes[0, C) (ascending, every label present; ±0 compare equal)
__global__ void __launch_bounds__(256)
k_mlp64_class_index(const float* __restrict__ Y, long n, const double* __restrict__ classes, int C, int* __restrict__ cls) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) cls[i] = class_lower_bound(classes, C, (double)Y[i]);
}

// softmax of each row of the output layer's pre-activations, in place (:104-117): exp of every column, their sum in
// column order, then one division per column.  No max subtraction: an overflow gives inf / inf = NaN, as in the reference.
__global__ void __launch_bounds__(256)
k_mlp64_softmax(double* __restrict__ h, int rows, int C) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        double* z = h + (long)r * C;
        double sum = 0.0;
        for (int j = 0; j < C; j++) { const double e = exp(z[j]); z[j] = e; sum += e; }
        for (int j = 0; j < C; j++) z[j] /= sum;
    }
}

// k_mlp64_loss for targets given as class indices cls[idx[r]]: log_loss (:162-178) — −y·log(clip(h)) summed only where
// y != 0, the clip of binary_log_loss, divided by the rows — or, with one output column (a single class v ∉ {0, 1}: an
// all-ones target), binary_log_loss, which on y = 1 is the same term.  Delta h − y, L2 and the accumulator as k_mlp64_loss.
__global__ void __launch_bounds__(256)
k_mlp64_loss_cls(const double* __restrict__ params, Mlp64Dims d, const double* __restrict__ h, const int* __restrict__ cls, const long* __restrict__ idx,
                 int m, double alpha, double* __restrict__ delta, double* __restrict__ loss_out, double* __restrict__ epoch_acc) {
    __shared__ double red[256];
    const int no = d.units[d.n_layers - 1];
    const double hmin = 4.9406564584124654e-324, hmax = 0.99999999999999989;     // nextafter(0,1), nextafter(1,0)
    double s = 0.0;
    for (int i = threadIdx.x; i < m * no; i += 256) {
        const int r = i / no, j = i % no;
        const double y = cls[idx ? idx[r] : (long)r] == j ? 1.0 : 0.0;
        double hv = h[i];
        delta[i] = hv - y;
        hv = hv < hmin ? hmin : (hv > hmax ? hmax : hv);
        if (y != 0.0) s += -y * log(hv);
    }
    red[threadIdx.x] = s; __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    mlp64_loss_finish(params, d, red, red[0] / (double)m, m, alpha, loss_out, epoch_acc);
}

// Predict with classes (:917-931): out[r] = float32(classes[MaxIdx64(h[r, 0:C))]) — the first strict maximum
// (mathCompat.go:93-101), so a NaN in column 0 wins and a NaN elsewhere never does.  One column: classes[0].
__global__ void __launch_bounds__(256)
k_mlp64_predict_label(const double* __restrict__ h, int rows, int C, const double* __restrict__ classes, float* __restrict__ out) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        const double* z = h + (long)r * C;
        int mi = 0;
        for (int j = 1; j < C; j++) if (z[j] > z[mi]) mi = j;
        out[r] = (float)classes[mi];
    }
}

// ---- the regressor (MLPRegressor, multilayer_perceptron.go:9-71): dense [n, no] targets -----------------------------
// The cold initialise decides the output from every target (:502-511): some target not 0 or 1 → identity output and
// square_loss; else one column → logistic and binary_log_loss (k_mlp64_loss, the binary classifier); else softmax and
// log_loss over the dense 0/1 rows, which need not be one-hot.

// flags[0] = some target is neither 0 nor 1; flags[1] = some target is NaN or ±inf (refused, DESIGN.md §2)
__global__ void __launch_bounds__(256)
k_mlp64_target_flags(const float* __restrict__ Y, long n, int* __restrict__ flags) {
    int not01 = 0, bad = 0;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float y = Y[i];
        not01 |= y != 0.0f && y != 1.0f;
        bad |= !isfinite(y);
    }
    if (__syncthreads_or(not01) && threadIdx.x == 0) flags[0] = 1;
    if (__syncthreads_or(bad) && threadIdx.x == 0) flags[1] = 1;
}

// k_mlp64_loss for dense targets Y[idx[r], 0:no): square_loss (:152-161) — Σ (h − y)², then / 2 / rows — or, with
// square == false, log_loss (:162-178) — −y·log(clip(h)) summed where y != 0, / rows.  Delta h − y, L2 and the
// accumulator as k_mlp64_loss.
__global__ void __launch_bounds__(256)
k_mlp64_loss_dense(const double* __restrict__ params, Mlp64Dims d, const double* __restrict__ h, const float* __restrict__ Y, const long* __restrict__ idx,
                   int m, double alpha, bool square, double* __restrict__ delta, double* __restrict__ loss_out, double* __restrict__ epoch_acc) {
    __shared__ double red[256];
    const int no = d.units[d.n_layers - 1];
    const double hmin = 4.9406564584124654e-324, hmax = 0.99999999999999989;     // nextafter(0,1), nextafter(1,0)
    double s = 0.0;
    for (int i = threadIdx.x; i < m * no; i += 256) {
        const int r = i / no, j = i % no;
        const double y = (double)Y[(idx ? idx[r] : (long)r) * no + j];
        double hv = h[i];
        const double e = hv - y;
        delta[i] = e;
        if (square) s += e * e;
        else {
            hv = hv < hmin ? hmin : (hv > hmax ? hmax : hv);
            if (y != 0.0) s += -y * log(hv);
        }
    }
    red[threadIdx.x] = s; __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    mlp64_loss_finish(params, d, red, square ? red[0] / 2.0 / (double)m : red[0] / (double)m, m, alpha, loss_out, epoch_acc);
}

// r2Score64 (basemlp64.go:1116-1141) over pred [n, no] and Y [n, no] in two passes, each a fixed partition of the rows
// into kR2Parts contiguous ranges per column (block (p, c)), a fixed tree inside the block, and the parts folded in
// order by one thread per column: the same bits on every run.  The same column sums serve R2Score, MeanSquaredError
// and MeanAbsoluteError (nn/metrics/regression.go, ctr_r2_score / ctr_mean_error): optional sample weights w [n]
// (null: every weight 1, and the sums are those of the unweighted form bit for bit), float or double targets.
constexpr int kR2Parts = 256;
enum : int {
    kR2Mean = 0,      // part[c][p] = {Σ w·y, Σ w}
    kR2Sums = 1,      // part[c][p] = {Σ w·(pred − y)², Σ w·(y − mean[c])²}
    kErrSquared = 2,  // part[c][p] = {Σ (pred − y)², rows}
    kErrAbsolute = 3  // part[c][p] = {Σ |pred − y|, rows}
};
template <class TY>
__global__ void __launch_bounds__(256)
k_mlp64_r2_part(const double* __restrict__ pred, const TY* __restrict__ Y, const double* __restrict__ w, long n, int no, int kind,
                const double* __restrict__ mean, double2* __restrict__ part) {
    __shared__ double2 red[256];
    const int p = blockIdx.x, c = blockIdx.y;
    const long per = (n + kR2Parts - 1) / kR2Parts, r0 = p * per, r1 = min(n, r0 + per);
    double a = 0.0, b = 0.0;
    for (long r = r0 + threadIdx.x; r < r1; r += 256) {
        const double y = (double)Y[r * no + c];
        if (kind == kR2Mean) {
            if (!w) { a += y; b += 1.0; } else { a += w[r] * y; b += w[r]; }
            continue;
        }
        const double t = pred[r * no + c] - y;
        if (kind == kErrSquared) { a += t * t; b += 1.0; continue; }
        if (kind == kErrAbsolute) { a += fabs(t); b += 1.0; continue; }
        const double u = y - mean[c];
        if (!w) { a += t * t; b += u * u; }
        else { a += w[r] * (t * t); b += w[r] * (u * u); }
    }
    red[threadIdx.x] = make_double2(a, b); __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { red[threadIdx.x].x += red[threadIdx.x + o].x; red[threadIdx.x].y += red[threadIdx.x + o].y; }
        __syncthreads();
    }
    if (threadIdx.x == 0) part[(long)c * kR2Parts + p] = red[0];
}
// Pass 1 (r2 == nullptr; kR2Mean or an error kind): mean[c] = a / b, the weighted column mean or the mean error, and
// when out is non-null out[0] = the mean of the columns' values in column order.  Pass 2 (kR2Sums): r2[c] = 1 − num /
// max(den, floor) (floor 0 for r2Score64, 1e-20 for R2Score, regression.go:112; a NaN den stays NaN, as Go's math.Max)
// and r2[no + c] = den; out[0] = the mean of the columns' r2 in column order, out[1] = the first column whose den is 0
// (r2Score64 panics there), or −1, out[2] = Σ den·r2 · (1 / Σ den) (R2Score's variance_weighted, :118-123).  One block.
__global__ void __launch_bounds__(256)
k_mlp64_r2_fold(const double2* __restrict__ part, int no, double floor, double* __restrict__ mean, double* __restrict__ r2, double* __restrict__ out) {
    for (int c = threadIdx.x; c < no; c += blockDim.x) {
        double a = 0.0, b = 0.0;
        for (int p = 0; p < kR2Parts; p++) { a += part[(long)c * kR2Parts + p].x; b += part[(long)c * kR2Parts + p].y; }
        if (!r2) mean[c] = a / b;
        else { r2[c] = 1.0 - a / (b < floor ? floor : b); r2[no + c] = b; }
    }
    if (!out) return;
    __syncthreads();
    if (threadIdx.x == 0) {
        if (!r2) {
            double acc = 0.0;
            for (int c = 0; c < no; c++) acc += mean[c];
            out[0] = acc / (double)no;
            return;
        }
        double acc = 0.0, bad = -1.0, dot = 0.0, sden = 0.0;
        for (int c = 0; c < no; c++) {
            if (bad < 0.0 && r2[no + c] == 0.0) bad = (double)c;
            acc += r2[c];
            dot += r2[no + c] * r2[c];
            sden += r2[no + c];
        }
        out[0] = acc / (double)no;
        out[1] = bad;
        out[2] = dot * (1.0 / sden);
    }
}

// gradients of layer l (computeLossGrad :322-331): coefGrads = actᵀ·delta / m + alpha/m · coefs, interceptGrads =
// column means of delta; thread (k, j) walks the m rows in order.  k == fi addresses the intercept row.
__global__ void __launch_bounds__(256)
k_mlp64_grads(const double* __restrict__ params, double* __restrict__ grads, Mlp64Dims d, int l, const double* __restrict__ X, long ldx,
              const long* __restrict__ idx, const double* __restrict__ act, const double* __restrict__ delta, int m, double alpha) {
    const int fi = d.units[l], fo = d.units[l + 1];
    const double* W = params + d.off[l] + fo;
    double* gb = grads + d.off[l];
    double* gW = gb + fo;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < (long)(fi + 1) * fo; t += (long)gridDim.x * blockDim.x) {
        const int k = (int)(t / fo), j = (int)(t % fo);
        double s = 0.0;
        if (k == fi) {
            for (int r = 0; r < m; r++) s += delta[(long)r * fo + j];                  // matRowMean64 :213-226
            gb[j] = s / (double)m;
        } else {
            for (int r = 0; r < m; r++) {
                const double a = act ? act[(long)r * fi + k] : X[(idx ? idx[r] : (long)r) * ldx + k];
                s += a * delta[(long)r * fo + j];
            }
            gW[(long)k * fo + j] = s / (double)m + alpha / (double)m * W[(long)k * fo + j];
        }
    }
}

// delta of hidden layer l from delta of layer l+1 (:388-396): (delta_{l+1} · Wᵀ) ⊙ act'(z).  For tanh the factor is
// 1 − a² (:131-138), the derivative of tanh(z) although the forward pass computed tanh(−z): every layer below an odd
// number of tanh layers receives the negated data gradient, as in the reference.
__global__ void __launch_bounds__(256)
k_mlp64_delta(const double* __restrict__ params, Mlp64Dims d, int l, const double* __restrict__ act, const double* __restrict__ dnext,
              double* __restrict__ dcur, int m) {
    const int fi = d.units[l], fo = d.units[l + 1];
    const double* W = params + d.off[l] + fo;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < (long)m * fi; t += (long)gridDim.x * blockDim.x) {
        const int r = (int)(t / fi), k = (int)(t % fi);
        double s = 0.0;
        for (int j = 0; j < fo; j++) s += dnext[(long)r * fo + j] * W[(long)k * fo + j];
        const double z = act[t];
        if (d.hidden_act == MLP_ACT_RELU) { if (z == 0.0) s = 0.0; }                   // :140-148
        else if (d.hidden_act == MLP_ACT_LOGISTIC) s *= z * (1.0 - z);                 // :124-131
        else if (d.hidden_act == MLP_ACT_TANH) s *= 1.0 - z * z;                       // :131-138
        dcur[t] = s;
    }
}

// AdamOptimizer64.updateParams (:1075-1091).  The reference multiplies beta1t / beta2t once per ELEMENT, in packed
// order, across calls: element i of call t (1-based) sees beta^((t-1)*np + i + 1).  Evaluated here in closed form.
__global__ void __launch_bounds__(256)
k_mlp64_adam(double* __restrict__ params, const double* __restrict__ grads, double* __restrict__ ms, double* __restrict__ vs, long np,
             double calls_before, double lr_init, double b1, double b2, double eps) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < np; i += (long)gridDim.x * blockDim.x) {
        const double g = grads[i];
        const double m = b1 * ms[i] + (1.0 - b1) * g;
        const double v = b2 * vs[i] + (1.0 - b2) * g * g;
        ms[i] = m; vs[i] = v;
        const double e = calls_before * (double)np + (double)(i + 1);
        const double b1t = pow(b1, e), b2t = pow(b2, e);
        const double lr = lr_init * sqrt(1.0 - b2t) / (1.0 - b1t);
        params[i] += -lr * m / (sqrt(v) + eps);
    }
}

// SGDOptimizer64.updateParams (:1024-1039): u = momentum·v − lr·g, v = u; p += momentum·v − lr·g (Nesterov) or u.
// vel is zero at the start of every fit (the optimizer is rebuilt per fit, :731-752).
__global__ void __launch_bounds__(256)
k_mlp64_sgd(double* __restrict__ params, const double* __restrict__ grads, double* __restrict__ vel, long np,
            double lr, double momentum, int nesterov) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < np; i += (long)gridDim.x * blockDim.x) {
        const double g = grads[i];
        const double u = momentum * vel[i] - lr * g;
        vel[i] = u;
        params[i] += nesterov ? momentum * u - lr * g : u;
    }
}

// weight decay at the top of backprop (:342-346): every packed element, intercepts included, times (1 − weight_decay),
// before the forward pass of the minibatch; keep = 1 − weight_decay is rounded once on the host as in the reference
__global__ void __launch_bounds__(256)
k_mlp64_decay(double* __restrict__ params, long np, double keep) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < np; i += (long)gridDim.x * blockDim.x) params[i] *= keep;
}

__global__ void __launch_bounds__(256)
k_f32_to_f64(const float* __restrict__ a, double* __restrict__ b, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) b[i] = (double)a[i];
}
__global__ void __launch_bounds__(256)
k_f64_to_f32(const double* __restrict__ a, float* __restrict__ b, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) b[i] = (float)a[i];
}

}  // namespace ctr
