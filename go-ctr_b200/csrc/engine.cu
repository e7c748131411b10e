// engine.cu — libctr_b200.so: handle, host-side mirror of model.Train / model.Predict
// (model/model.go:27-353 of auxten/go-ctr) and the C ABI of include/ctr_b200.h.
// sm_90a (Hopper) only; no CPU fallback: every compute entry point launches CUDA kernels or fails.
#include "../../include/ctr_b200.h"
#include "attn.cuh"
#include "mlp.cuh"
#include "umma_gemm.cuh"
#include "auc.cuh"
#include "ubcache.cuh"
#include "idmap.cuh"
#include "item2vec.cuh"
#include "mlp64.cuh"
#include "knn.cuh"
#include "rec.cuh"
#include "metrics.cuh"
#include "comm.cuh"

#include <nvtx3/nvToolsExt.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <condition_variable>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

using namespace ctr;

namespace {

std::string g_create_error;

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct Prof { double ms = 0; long n = 0; };

// Caller buffers are pageable (Go slices, numpy arrays): a cudaMemcpyAsync straight from them is staged
// synchronously by the driver and kills the copy/compute overlap.  The epoch entry points therefore copy each batch
// into a pinned ring first — with a few worker threads, since one memcpy stream is far slower than the DMA — and DMA from
// there.  The library never keeps a caller pointer past the call (cgo rule).
class CopyPool {
public:
    explicit CopyPool(int n) { for (int i = 0; i < n; i++) th_.emplace_back([this] { run(); }); }
    ~CopyPool() { { std::lock_guard<std::mutex> l(m_); stop_ = true; } cv_.notify_all(); for (auto& t : th_) t.join(); }
    // copies n bytes, split over the workers and the calling thread; returns when done
    void copy(void* dst, const void* src, size_t n) {
        const size_t kMin = (size_t)512 << 10;
        const int parts = (int)std::min<size_t>(th_.size() + 1, std::max<size_t>(1, n / kMin));
        if (parts <= 1) { memcpy(dst, src, n); return; }
        const size_t chunk = (n / parts + 63) & ~(size_t)63;
        { std::lock_guard<std::mutex> l(m_);
          for (int i = 1; i < parts; i++) {
              const size_t off = (size_t)i * chunk; if (off >= n) break;
              jobs_.push_back({(char*)dst + off, (const char*)src + off, std::min(chunk, n - off)}); pending_++;
          } }
        cv_.notify_all();
        memcpy(dst, src, std::min(chunk, n));
        std::unique_lock<std::mutex> l(m_);
        done_.wait(l, [this] { return pending_ == 0; });
    }
private:
    struct Job { char* d; const char* s; size_t n; };
    void run() {
        for (;;) {
            Job j;
            { std::unique_lock<std::mutex> l(m_);
              cv_.wait(l, [this] { return stop_ || !jobs_.empty(); });
              if (stop_ && jobs_.empty()) return;
              j = jobs_.back(); jobs_.pop_back(); }
            memcpy(j.d, j.s, j.n);
            { std::lock_guard<std::mutex> l(m_); if (--pending_ == 0) done_.notify_all(); }
        }
    }
    std::vector<std::thread> th_; std::vector<Job> jobs_;
    std::mutex m_; std::condition_variable cv_, done_; int pending_ = 0; bool stop_ = false;
};

}  // namespace

struct ctr_handle {
    ctr_config cfg{};
    int dev = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    mutable std::string err;
    std::mutex mu;                        // Predict may be hit concurrently (gin handlers, api.go:106-131)

    int in = 0, Kp = 0, H0p = 0, H1p = 0, Sp = 0, lddx = 0, Bmax = 0;
    int num_sms = 132;

    // tables (HBM resident)
    float* tab[3] = {nullptr, nullptr, nullptr};
    long tab_ld[3] = {0, 0, 0};
    int64_t tab_rows[3] = {0, 0, 0};      // logical (global) rows
    int64_t tab_local_rows[3] = {0, 0, 0};
    int tab_width[3] = {0, 0, 0};
    bool tab_sharded[3] = {false, false, false};   // world > 1: rows r % world == rank live here, the rest on the peers
    VmmBuf tab_vmm[3];                    // a sharded table lives in shareable (VMM) memory; tab[] points into it
    GrowBuf<float> tab_mem[3];            // any other table lives in growable memory (ctr_table_write_rows); tab[] points into it
    uint64_t tab_gen = 1;                 // bumped whenever an ITEM_* table is (re)allocated: peers must re-map it
    std::vector<int64_t> emb_vocab;       // ctr_item_emb_train's vocabulary when the caller's vocab_ids could not take it all

    // learnables, padded storage: W0 [Kp,H0p] W1 [H0p,H1p] W2 [H1p] att [Sp]; grads / Adam moments alike
    DevBuf<float> W[4], Mo[4], Vo[4];
    float* G[4] = {};                     // views into Gflat
    DevBuf<float> Gflat; size_t Gflat_n = 0;       // the four gradient tensors live in one buffer (one all-reduce, one memset)
    size_t wsize[4] = {};
    uint32_t step = 0;                    // optimiser steps taken (Adam t = step+1; dropout stream = step*4+layer)

    // activations
    DevBuf<float> X0, H0d, H1d, P, Z;
    DevBuf<float> dZ1, dZ0, dX;
    DevBuf<float> dUb, dIt;               // row-gradient buffers (deterministic / debug)
    DevBuf<unsigned> keys, keys2, pos, pos2;
    DevBuf<unsigned char> sort_tmp;
    DevBuf<double> d_cost;
    DevBuf<float> hot_acc; int hot_rows = 0, hot_reps = 0;
    GrowBuf<float> emb_m, emb_v;          // CTR_TABLE_ADAM: first / second moments of ITEM_EMB, same layout as the table (grown with it)
    // staging for host-pointer entry points
    DevBuf<int> s_user, s_item, s_hist; DevBuf<float> s_label;
    // epoch entry points (ctr_train_idx / ctr_train_keys): pinned host ring (filled by the copy pool from the caller's
    // pageable buffers) → device slots on a copy stream, overlapping the compute of the previous batch
    static constexpr int kPin = 3;
    PinnedBuf<unsigned char> feed_pin[kPin]; DevBuf<unsigned char> feed_dev[2]; size_t feed_bytes = 0;
    Event pin_free[kPin];
    std::unique_ptr<CopyPool> pool;
    Stream copy_stream;
    Event ev_copied[2], ev_consumed[2];
    DevBuf<double> d_costs;
    // ctr_train_keys: resolved + compacted samples resident in HBM
    DevBuf<int> kt_user, kt_item; DevBuf<long long> kt_ts; DevBuf<float> kt_label;
    DevBuf<int> kt_flag, kt_pos; DevBuf<unsigned char> kt_scan_tmp;
    DevBuf<unsigned long long> kt_count;
    static constexpr int kCnt = 8;                       // pinned ring of survivor counts read back chunk by chunk
    PinnedBuf<unsigned long long> kt_count_host; Event kt_counted[kCnt];
    // history windows of batch b+1 are cut on their own stream while batch b trains (two buffers); kt_queued marks the
    // engine stream's work queued before a ctr_train_keys call, which the call's first windows wait for
    Stream win_stream; DevBuf<int> kt_hist[2]; Event kt_win[2], kt_used[2], kt_queued;
    // ctr_mlp_fit_keys: the history window of every survivor [survivors, S], cut once per fit
    DevBuf<int> kt_hist_all;
    // dense-X residency
    DevBuf<float> dXd, dYd;

    int64_t launches = 0;
    bool profiling = false;
    std::map<std::string, Prof> prof;
    Event ev0, ev1;

    // wgmma GEMM engine (umma_gemm.cuh): pre-split K-major weight operands + TMA descriptors
    struct Umma {
        bool ready = false;
        bool dirty = true;                 // weights changed since the last split
        int nch_h0 = 0, nch_h1 = 0, nch_dx = 0;                            // 32-column chunks of the H0p / H1p / dX-wide tiles
        int stages_h0 = 0, stages_h1 = 0, stages_dx = 0;
        int bn_dx = 0;
        DevBuf<float> Wt0[2], Wt1[2], W1s[2], W0s[2];                       // [hi, lo]
        CUtensorMap mA_X0, mA_H0d, mA_dZ1, mA_dZ0;
        CUtensorMap mB_Wt0[2], mB_Wt1[2], mB_W1s[2], mB_W0s[2];
        CUtensorMap mK_X0, mK_H0d, mK_dZ0, mK_dZ1;      // {width, 32 samples} boxes over [batch, width] for the weight-gradient GEMMs
        int dw_stages0 = 0, dw_stages1 = 0;
    } um;

    // device-side ubcache (ubcache.cuh)
    DevBuf<long long> ub_off, ub_ts; DevBuf<int> ub_items; int64_t ub_users = 0, ub_n = 0;
    // the spare CSR an append / set writes before the two are swapped
    DevBuf<long long> ubx_off, ubx_ts; DevBuf<int> ubx_items;

    // device id maps (idmap.cuh): [CTR_IDMAP_USER, CTR_IDMAP_ITEM]
    DevBuf<unsigned long long> idm_keys[2]; DevBuf<int> idm_vals[2];
    int64_t idm_n[2] = {0, 0};              // the tables hold idm_keys[i].size() slots (a power of two)
    DevBuf<long long> k_keys; PinnedBuf<unsigned char> k_host; DevBuf<int> k_flags;   // staging for ctr_batch_predict_keys (device, pinned host)

    // grow-only device scratch of the host-buffer entry points (gather / window / id lookup; slot 3: ctr_knn_search;
    // slot 4: ctr_recommend_topk; slot 5: ubcache append / set; slot 6: ctr_mlp_recommend_topk): no cudaMalloc on the
    // serving path
    static constexpr int kScratch = 7;
    DevBuf<unsigned char> scratch[kScratch];

    Comm comm;
};

namespace {

int set_err(const ctr_handle* h, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

#define CU(h, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    return set_err(h, e_ == cudaErrorMemoryAllocation ? CTR_ENOMEM : CTR_ECUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

#define RET(x) do { int r_ = (x); if (r_ != CTR_OK) return r_; } while (0)

// every kernel launch goes through here: counts it and, when profiling, brackets it with events
// CTR_NVTX=1: every launch sits in an NVTX range named like the profile key (nsys / ncu --nvtx timelines)
const bool g_nvtx = getenv("CTR_NVTX") != nullptr;

template <typename F>
int launch(ctr_handle* h, const char* name, F&& f) {
    if (h->profiling) cudaEventRecord(h->ev0, h->stream);
    if (g_nvtx) nvtxRangePushA(name);
    f();
    if (g_nvtx) nvtxRangePop();
    h->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(h, CTR_ECUDA, "launch %s: %s", name, cudaGetErrorString(e));
    if (h->profiling) {
        cudaEventRecord(h->ev1, h->stream);
        cudaEventSynchronize(h->ev1);
        float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
        Prof& p = h->prof[name]; p.ms += ms; p.n++;
    }
    return CTR_OK;
}

// (re)allocates b for n elements (at least one), freeing its old allocation first; zeroed on the engine stream
template <typename T>
int dalloc(ctr_handle* h, DevBuf<T>& b, size_t n, bool zero = true) {
    CU(h, b.alloc(std::max<size_t>(n, 1)));
    if (zero) CU(h, cudaMemsetAsync(b, 0, b.size() * sizeof(T), h->stream));
    return CTR_OK;
}
// grow-only: reallocates b (old allocation freed first) only when it holds fewer than n elements
template <typename T>
int reserve(ctr_handle* h, DevBuf<T>& b, size_t n, bool zero = true) {
    return b.size() >= n ? CTR_OK : dalloc(h, b, n, zero);
}

// device scratch slot `i` with at least `bytes` (contents undefined); grows to exactly the request, freed with the handle
int scratch_get(ctr_handle* h, int i, size_t bytes, void** out) {
    if (h->scratch[i] && h->scratch[i].size() < bytes) cudaStreamSynchronize(h->stream);   // queued work may still read it
    RET(reserve(h, h->scratch[i], bytes, false));
    *out = h->scratch[i];
    return CTR_OK;
}

Dims dims_of(const ctr_handle* h) { return Dims{h->cfg.uP, h->cfg.S, h->cfg.D, h->cfg.cF, h->in}; }

int grid_for_warps(const ctr_handle* h, int B) {
    int blocks = (B + 7) / 8;
    return std::max(1, std::min(blocks, h->num_sms * 8));
}

// Attention kernel families (attn.cuh), in the order attn_path prefers them.  _peer is the _idx kernels' PEER
// instantiation for row-sharded tables.
enum AttnFamily { ATTN_PEER, ATTN_IDX, ATTN_VEC, ATTN_GEN };
const char* const kAttnKey[2][4] = {       // profile / NVTX keys: [backward][family]
    {"attn_fwd_peer", "attn_fwd_idx", "attn_fwd_vec", "attn_fwd_gen"},
    {"attn_bwd_peer", "attn_bwd_idx", "attn_bwd_vec", "attn_bwd_gen"}};
struct AttnPath { AttnFamily fwd, bwd; };

// the lane maps of the _vec / _idx kernels (kLanes) cover D in {16, 32, 64, 128}
bool attn_lanes_ok(int D) { return D == 16 || D == 32 || D == 64 || D == 128; }
// The _idx kernels also need S <= 64 (two history ids per lane), and the _idx forward uP % 4 == 0 and (Kp - 2D)/4 <= 32
// (one 16-byte feature chunk per lane).  Row-sharded tables run only on the _idx kernels: comm_check rejects other shapes.
bool attn_idx_shape_ok(const ctr_handle* h, bool fwd) {
    const ctr_config& c = h->cfg;
    return attn_lanes_ok(c.D) && c.S <= 64 && (!fwd || (c.uP % 4 == 0 && (h->Kp - 2 * c.D) / 4 <= 32));
}
AttnPath attn_path(const ctr_handle* h, const RowSrc& r) {
    if (r.world > 1) return {ATTN_PEER, ATTN_PEER};        // comm_check vetted the dims
    const bool aligned = r.dense ? (r.ldx % 4 == 0) && (r.ub0 % 4 == 0) && (r.it0 % 4 == 0) && (((uintptr_t)r.X) % 16 == 0)
                                 : r.lde % 4 == 0;
    if (!attn_lanes_ok(h->cfg.D) || !aligned) return {ATTN_GEN, ATTN_GEN};
    if (r.dense || !attn_idx_shape_ok(h, false)) return {ATTN_VEC, ATTN_VEC};
    // the forward also moves the dense features in 16-byte chunks
    const bool idx_fwd = attn_idx_shape_ok(h, true) && r.ldu % 4 == 0 && r.ldi % 4 == 0 && r.ufeat && r.ifeat;
    return {idx_fwd ? ATTN_IDX : ATTN_VEC, ATTN_IDX};
}

// the lane maps (kLanes, with_lanes), with_model and the grid rule live in attn.cuh
static_assert(CTR_MODEL_YOUTUBE == MODEL_YOUTUBE && CTR_MODEL_DIN_COS == MODEL_DIN_COS && CTR_MODEL_DIN_EUC == MODEL_DIN_EUC,
              "with_model takes the API's model ids");
int grid_attn(const ctr_handle* h, int B) { return attn_grid(h->num_sms, B); }

int attn_forward(ctr_handle* h, const RowSrc& r, int B) {
    const AttnFamily f = attn_path(h, r).fwd;
    return launch(h, kAttnKey[0][f], [&] {
        const Dims d = dims_of(h);
        const int g = grid_attn(h, B);
        if (f == ATTN_GEN) {
            k_attn_fwd_gen<<<grid_for_warps(h, B), 256, 0, h->stream>>>(r, d, h->cfg.model, h->W[3], h->X0, h->Kp, h->Kp, B);
            return;
        }
        with_model(h->cfg.model, [&](auto m) {
            constexpr int M = decltype(m)::value;
            auto idx = [&](auto peer) {
                constexpr bool P = decltype(peer)::value;
                with_lanes<false, P>(h->cfg.D, [&](auto l) {
                    using L = decltype(l);
                    k_attn_fwd_idx<L::LPR, L::VPL, M, P><<<g, kAttnThreads, 0, h->stream>>>(r, d, h->W[3], h->X0, h->Kp, h->Kp, B);
                });
            };
            if (f == ATTN_PEER) idx(std::true_type{});
            else if (f == ATTN_IDX) idx(std::false_type{});
            else with_lanes<false, false>(h->cfg.D, [&](auto l) {
                using L = decltype(l);
                const size_t smem = (size_t)(kAttnThreads / 32) * h->Kp * sizeof(float);
                k_attn_fwd_vec<L::LPR, L::VPL, M><<<g, kAttnThreads, smem, h->stream>>>(r, d, h->W[3], h->X0, h->Kp, h->Kp, B);
            });
        });
    });
}

// k_attn_fwd_user (ctr_recommend_topk) runs where the _vec / _idx lane maps cover D, the ITEM_EMB rows are 16-byte
// aligned and the user's history rows fit the opt-in shared memory; other shapes fill index buffers for attn_forward.
size_t attn_user_smem(const ctr_handle* h) { return user_smem_floats(h->cfg.S, h->cfg.D, h->Kp) * sizeof(float); }
bool attn_user_ok(const ctr_handle* h, size_t smem_optin) {
    return attn_lanes_ok(h->cfg.D) && h->tab_ld[CTR_TABLE_ITEM_EMB] % 4 == 0 && attn_user_smem(h) <= smem_optin;
}
// f(kernel) for the handle's model and D; peer: the row-sharded instantiation (same lane map: the same arithmetic)
template <typename F>
void with_user_kernel(const ctr_handle* h, bool peer, F&& f) {
    with_model(h->cfg.model, [&](auto m) {
        constexpr int M = decltype(m)::value;
        with_lanes<false, false>(h->cfg.D, [&](auto l) {
            using L = decltype(l);
            if (peer) f(k_attn_fwd_user<L::LPR, L::VPL, M, true>); else f(k_attn_fwd_user<L::LPR, L::VPL, M, false>);
        });
    });
}
// sets the kernel's dynamic shared-memory limit; returns its resident CTAs per SM
int attn_user_prepare(const ctr_handle* h, bool peer) {
    int occ = 1;
    const size_t smem = attn_user_smem(h);
    with_user_kernel(h, peer, [&](auto kern) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kAttnThreads, smem);
    });
    return std::max(occ, 1);
}
// X0 rows of the samples (user, item i0 + b, d_hist) for b < B (r.world > 1: local rows of this rank's shard); grid:
// one wave of resident CTAs, so that each stages the history once
int attn_forward_user(ctr_handle* h, const RowSrc& r, int user, const int* d_hist, int i0, int B, int grid) {
    return launch(h, "attn_fwd_user", [&] {
        const Dims d = dims_of(h);
        const size_t smem = attn_user_smem(h);
        with_user_kernel(h, r.world > 1, [&](auto kern) {
            kern<<<std::min(grid, grid_attn(h, B)), kAttnThreads, smem, h->stream>>>(r, d, h->W[3], user, d_hist, i0, h->comm.rank, h->X0, h->Kp, h->Kp, B);
        });
    });
}

int attn_backward(ctr_handle* h, const RowSrc& r, const BwdOut& o, int B) {
    const AttnFamily f = attn_path(h, r).bwd;
    return launch(h, kAttnKey[1][f], [&] {
        const Dims d = dims_of(h);
        const int g = grid_attn(h, B);
        const size_t datt_smem = (size_t)std::max(h->cfg.S, 1) * sizeof(float);
        if (f == ATTN_GEN) {
            k_attn_bwd_gen<<<grid_for_warps(h, B), 256, datt_smem, h->stream>>>(r, d, h->cfg.model, h->W[3], h->dX, h->lddx, o, B);
            return;
        }
        with_model(h->cfg.model, [&](auto m) {
            constexpr int M = decltype(m)::value;
            auto idx = [&](auto peer) {
                constexpr bool P = decltype(peer)::value;
                with_lanes<true, P>(h->cfg.D, [&](auto l) {
                    using L = decltype(l);
                    if (o.sgd) k_attn_bwd_idx<L::LPR, L::VPL, M, true, P><<<g, kAttnThreads, 0, h->stream>>>(r, d, h->W[3], h->dX, h->lddx, o, B);
                    else       k_attn_bwd_idx<L::LPR, L::VPL, M, false, P><<<g, kAttnThreads, 0, h->stream>>>(r, d, h->W[3], h->dX, h->lddx, o, B);
                });
            };
            if (f == ATTN_PEER) idx(std::true_type{});
            else if (f == ATTN_IDX) idx(std::false_type{});
            else with_lanes<true, false>(h->cfg.D, [&](auto l) {
                using L = decltype(l);
                k_attn_bwd_vec<L::LPR, L::VPL, M><<<g, kAttnThreads, datt_smem, h->stream>>>(r, d, h->W[3], h->dX, h->lddx, o, B);
            });
        });
    });
}

// ---- fp32 GEMM launchers ---------------------------------------------------------------------------
template <bool TA, bool TB, int EPI>
int gemm_big(ctr_handle* h, const char* name, GemmArgs g) {     // M = batch: 128x64 tiles
    constexpr int BM = 128, BN = 64;
    dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, 1);
    return launch(h, name, [&] { k_sgemm<BM, BN, 16, 8, 4, TA, TB, EPI><<<grid, 256, 0, h->stream>>>(g); });
}
int gemm_dw(ctr_handle* h, const char* name, GemmArgs g) {      // K = batch: 64x64 tiles, split-K atomics
    constexpr int BM = 64, BN = 64;
    int tiles = ((g.N + BN - 1) / BN) * ((g.M + BM - 1) / BM);
    int want_z = std::max(1, (h->num_sms * 4) / std::max(tiles, 1));
    int kchunk = round_up(std::max(16, (g.K + want_z - 1) / want_z), 16);
    g.kchunk = kchunk;
    dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, (g.K + kchunk - 1) / kchunk);
    return launch(h, name, [&] { k_sgemm<BM, BN, 16, 4, 4, true, false, EPI_ATOMIC><<<grid, 256, 0, h->stream>>>(g); });
}


// ---- wgmma GEMM launchers ----------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D map over a row-major [rows, cols] fp32 matrix with {box_k, box_rows} boxes; boxes reaching past the matrix
// are zero-filled, which pads K and the weight tiles to whole k-blocks and 32-column chunks
int make_map(ctr_handle* h, CUtensorMap* m, const float* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
             CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B, uint32_t box_k = umma::kKB) {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        cudaDriverEntryPointQueryResult q;
        void* p = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
            return set_err(h, CTR_ECUDA, "cuTensorMapEncodeTiled entry point not available");
        fn = (PFN_encodeTiled)p;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstr[1] = {ld * sizeof(float)};
    cuuint32_t box[2] = {box_k, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_err(h, CTR_ECUDA, "cuTensorMapEncodeTiled failed: %d", (int)r);
    return CTR_OK;
}

constexpr size_t kSmemMax = (size_t)227 * 1024;
constexpr size_t kSmemSlack = 1024 + 256;           // 1024-byte alignment of the ring + barriers
size_t umma_stage_bytes(int nch) { return ((size_t)umma::kBlockM + 2 * 32 * (size_t)nch) * umma::kKB * 4; }     // A + B_hi + B_lo
int umma_stages(int nch) { return (int)std::min<size_t>(6, (kSmemMax - kSmemSlack) / umma_stage_bytes(nch)); }
size_t umma_smem(int nch, int stages) { return (size_t)stages * umma_stage_bytes(nch) + kSmemSlack; }
// weight-gradient GEMM: two buffers of two Bᵀ copies (hi, lo) of 32*nch rows x 128 bytes, then the ring of raw [A | B] k-blocks
size_t dw_fixed_bytes(int nch) { return (size_t)2 * 2 * 32 * nch * 128; }
size_t dw_stage_bytes(int nch) { return (size_t)32 * (umma::kDwAPitch + 32 * nch) * 4; }
int dw_stages(int nch) { return (int)std::min<size_t>(6, (kSmemMax - kSmemSlack - dw_fixed_bytes(nch)) / dw_stage_bytes(nch)); }

bool umma_supported(const ctr_handle* h) {
    return h->H0p <= 256 && h->H1p <= 256 && round_up(2 * h->cfg.D, 16) <= 256 && h->H0p % 16 == 0 && h->H1p % 16 == 0;
}

// the kernels are instantiated per tile width (32-column chunks, 1..8); the launchers pick the instantiation
#define UMMA_NCH_SWITCH(nch, F) switch (nch) { \
    case 1: F(1); break; case 2: F(2); break; case 3: F(3); break; case 4: F(4); break; \
    case 5: F(5); break; case 6: F(6); break; case 7: F(7); break; default: F(8); break; }

template <class K>
cudaError_t allow_smem(K kernel) {
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
}

// the attribute belongs to the current device: set once per handle (umma_init) for the instantiations it launches
template <int EPI>
cudaError_t allow_smem_gemm(int nch) {
    cudaError_t e = cudaSuccess;
#define UMMA_ALLOW(N) e = allow_smem(umma::k_umma_gemm<EPI, N>)
    UMMA_NCH_SWITCH(nch, UMMA_ALLOW)
#undef UMMA_ALLOW
    return e;
}
cudaError_t allow_smem_dw(int nch) {
    cudaError_t e = cudaSuccess;
#define UMMA_ALLOW(N) e = allow_smem(umma::k_umma_dw<N>)
    UMMA_NCH_SWITCH(nch, UMMA_ALLOW)
#undef UMMA_ALLOW
    return e;
}

int umma_init(ctr_handle* h) {
    if (h->um.ready) return CTR_OK;
    const ctr_config& c = h->cfg;
    auto& u = h->um;
    u.bn_dx = round_up(2 * c.D, 16);
    u.nch_h0 = (h->H0p + 31) / 32; u.nch_h1 = (h->H1p + 31) / 32; u.nch_dx = (u.bn_dx + 31) / 32;
    u.stages_h0 = umma_stages(u.nch_h0); u.stages_h1 = umma_stages(u.nch_h1); u.stages_dx = umma_stages(u.nch_dx);
    u.dw_stages0 = dw_stages(u.nch_h0); u.dw_stages1 = dw_stages(u.nch_h1);
    // k_umma_dw frees a raw slot as soon as it is transposed, so its producer refills even a single slot while the
    // wgmmas run; k_umma_gemm holds a slot until its wgmma group retires and needs two
    if (std::min({u.stages_h0, u.stages_h1, u.stages_dx}) < 2 || std::min(u.dw_stages0, u.dw_stages1) < 1)
        return set_err(h, CTR_EINVAL, "wgmma GEMM: tile does not fit shared memory");
    for (int i = 0; i < 2; i++) {
        // allocated once per handle (the maps hold their addresses): a retry after a failed init keeps the live copies
        if (!u.Wt0[i]) RET(dalloc(h, u.Wt0[i], (size_t)h->H0p * h->Kp));
        if (!u.Wt1[i]) RET(dalloc(h, u.Wt1[i], (size_t)h->H1p * h->H0p));
        if (!u.W1s[i]) RET(dalloc(h, u.W1s[i], (size_t)h->H0p * h->H1p));
        if (!u.W0s[i]) RET(dalloc(h, u.W0s[i], (size_t)u.bn_dx * h->H0p));
        RET(make_map(h, &u.mB_Wt0[i], u.Wt0[i], h->H0p, h->Kp, h->Kp, 32 * u.nch_h0));
        RET(make_map(h, &u.mB_Wt1[i], u.Wt1[i], h->H1p, h->H0p, h->H0p, 32 * u.nch_h1));
        RET(make_map(h, &u.mB_W1s[i], u.W1s[i], h->H0p, h->H1p, h->H1p, 32 * u.nch_h0));
        RET(make_map(h, &u.mB_W0s[i], u.W0s[i], u.bn_dx, h->H0p, h->H0p, 32 * u.nch_dx));
    }
    RET(make_map(h, &u.mA_X0, h->X0, h->Bmax, h->Kp, h->Kp, umma::kBlockM));
    RET(make_map(h, &u.mA_H0d, h->H0d, h->Bmax, h->H0p, h->H0p, umma::kBlockM));
    RET(make_map(h, &u.mA_dZ1, h->dZ1, h->Bmax, h->H1p, h->H1p, umma::kBlockM));
    RET(make_map(h, &u.mA_dZ0, h->dZ0, h->Bmax, h->H0p, h->H0p, umma::kBlockM));
    // weight-gradient operands: rows limited to the training batch so that TMA zero-fills the K tail; unswizzled
    // {width, 32 samples} boxes (the A operand: kDwAPitch columns starting at the CTA's row block of C)
    RET(make_map(h, &u.mK_X0, h->X0, c.batch, h->Kp, h->Kp, 32, CU_TENSOR_MAP_SWIZZLE_NONE, umma::kDwAPitch));
    RET(make_map(h, &u.mK_H0d, h->H0d, c.batch, h->H0p, h->H0p, 32, CU_TENSOR_MAP_SWIZZLE_NONE, umma::kDwAPitch));
    RET(make_map(h, &u.mK_dZ0, h->dZ0, c.batch, h->H0p, h->H0p, 32, CU_TENSOR_MAP_SWIZZLE_NONE, 32 * u.nch_h0));
    RET(make_map(h, &u.mK_dZ1, h->dZ1, c.batch, h->H1p, h->H1p, 32, CU_TENSOR_MAP_SWIZZLE_NONE, 32 * u.nch_h1));
    CU(h, allow_smem_gemm<umma::UEPI_SIGMOID_DROP>(u.nch_h0)); CU(h, allow_smem_gemm<umma::UEPI_SIGMOID_DROP>(u.nch_h1));
    CU(h, allow_smem_gemm<umma::UEPI_DSIGMOID>(u.nch_h0)); CU(h, allow_smem_gemm<umma::UEPI_STORE>(u.nch_dx));
    CU(h, allow_smem_dw(u.nch_h0)); CU(h, allow_smem_dw(u.nch_h1));
    u.ready = true; u.dirty = true;
    return CTR_OK;
}

int umma_split_weights(ctr_handle* h) {
    auto& u = h->um;
    if (!u.dirty) return CTR_OK;
    const ctr_config& c = h->cfg;
    umma::SplitJobs jobs;
    jobs.j[0] = {h->W[0], h->H0p, h->in, c.H0, 1, u.Wt0[0], u.Wt0[1], h->Kp};                                      // W0ᵀ [H0, in]
    jobs.j[1] = {h->W[1], h->H1p, c.H0, c.H1, 1, u.Wt1[0], u.Wt1[1], h->H0p};                                     // W1ᵀ [H1, H0]
    jobs.j[2] = {h->W[1], h->H1p, c.H0, c.H1, 0, u.W1s[0], u.W1s[1], h->H1p};                                     // W1  [H0, H1]
    jobs.j[3] = {h->W[0] + (long)c.uP * h->H0p, h->H0p, 2 * c.D, c.H0, 0, u.W0s[0], u.W0s[1], h->H0p};            // W0[uP:uP+2D, :]
    RET(launch(h, "split_weights_tf32", [&] { umma::k_split_weights<<<dim3(48, 4), 256, 0, h->stream>>>(jobs); }));
    u.dirty = false;
    return CTR_OK;
}

template <int EPI>
int umma_gemm(ctr_handle* h, const char* name, int nch, const CUtensorMap& mA, const CUtensorMap* mB, umma::Args a) {
    const int tiles = (a.M + umma::kBlockM - 1) / umma::kBlockM;
    const int grid = std::min(tiles, h->num_sms);
    const size_t smem = umma_smem(nch, a.stages);
#define UMMA_GEMM_LAUNCH(N) umma::k_umma_gemm<EPI, N><<<grid, umma::kThreads, smem, h->stream>>>(mA, mB[0], mB[1], a)
    int rc = launch(h, name, [&] { UMMA_NCH_SWITCH(nch, UMMA_GEMM_LAUNCH) });
#undef UMMA_GEMM_LAUNCH
    return rc;
}

int umma_dw(ctr_handle* h, const char* name, int nch, const CUtensorMap& mA, const CUtensorMap& mB, umma::DwArgs a) {
    const int total_kb = (a.K + 31) / 32;
    const int mblocks = (a.M + umma::kBlockM - 1) / umma::kBlockM;
    const int slices = std::max(1, std::min(total_kb, h->num_sms / mblocks));
    a.kb_per = (total_kb + slices - 1) / slices;
    const dim3 grid(mblocks, (total_kb + a.kb_per - 1) / a.kb_per);
    const size_t smem = dw_fixed_bytes(nch) + (size_t)a.stages * dw_stage_bytes(nch) + kSmemSlack;
#define UMMA_DW_LAUNCH(N) umma::k_umma_dw<N><<<grid, umma::kThreads, smem, h->stream>>>(mA, mB, a)
    int rc = launch(h, name, [&] { UMMA_NCH_SWITCH(nch, UMMA_DW_LAUNCH) });
#undef UMMA_DW_LAUNCH
    return rc;
}

// the weight-gradient GEMMs run on the tensor cores when the padded widths fit 8 column chunks and the batch
// is the configured training batch (the TMA maps zero-fill rows beyond it)
bool use_umma_dw(const ctr_handle* h, int B) {
    return B == h->cfg.batch && h->Kp <= 256 && h->H0p <= 256 && h->H1p <= 256;
}

bool use_umma(const ctr_handle* h) {
    return h->cfg.gemm != CTR_GEMM_FP32 && umma_supported(h);     // AUTO → wgmma when the shape qualifies
}

// One pass of the hot path over one batch (model.go:107-196 inner loop body).
//   training: dropout on, backward + optimiser step (update) or gradients only (!update)
struct StepOpts {
    bool training = false, update = false;
    bool want_rows = false;              // fill h->dUb / h->dIt
    bool x0_ready = false;               // h->X0 already holds the MLP input rows (ctr_recommend_topk): no attention forward
    const float* d_label = nullptr;
    // sharded-table step (comm_impl.cuh): rows live in a per-lookup buffer, gradients are scaled to the
    // global mean and the dense gradients are all-reduced before Adam
    bool comm = false; float grad_scale = 1.0f; int adam_batch = 0;
    bool peer = false;                   // rows come from / go to the owners' shards over NVLink (RowSrc.world > 1)
    // replicated-table step: row gradients are summed into table_grad (layout of the table), all-reduced with the
    // dense gradients and applied on every rank
    float* table_grad = nullptr; size_t table_grad_n = 0;
};

int ensure_rowgrad_buffers(ctr_handle* h, int B) {
    RET(reserve(h, h->dUb, (size_t)B * h->cfg.S * h->cfg.D));
    return reserve(h, h->dIt, (size_t)B * h->cfg.D);
}

// Replica accumulators for the popular rows of ITEM_EMB (rows [0, hot_rows), see k_attn_bwd_vec).
// cfg.reserved[0]: 0 = auto (all rows of a small table / the first 32768 of a large one — keep rows
// ordered by popularity, as word2vec-style vocabularies are), >0 = that many rows, <0 = off.
int ensure_hot(ctr_handle* h) {
    const int64_t rows = h->tab_local_rows[CTR_TABLE_ITEM_EMB];
    int want = h->cfg.reserved[0];
    if (want == 0) want = (int)std::min<int64_t>(rows, 32768);
    if (want < 0) want = 0;
    want = (int)std::min<int64_t>(want, rows);
    if (h->hot_acc && h->hot_rows == want) return CTR_OK;
    h->hot_acc.reset();
    h->hot_rows = want; h->hot_reps = 0;
    if (want == 0) return CTR_OK;
    const size_t row_bytes = (size_t)h->cfg.D * sizeof(float);
    int reps = (int)std::min<size_t>(32, std::max<size_t>(1, ((size_t)64 << 20) / ((size_t)want * row_bytes)));
    h->hot_reps = reps;
    return dalloc(h, h->hot_acc, (size_t)reps * want * h->cfg.D);
}

// maps at least n elements of b (growable memory); the new part is not initialised
int grow_buf(ctr_handle* h, GrowBuf<float>& b, size_t n) {
    std::string err;
    if (!b.grow(std::max<size_t>(n, 1), h->dev, h->stream, &err)) return set_err(h, CTR_ENOMEM, "device memory (%zu bytes): %s", n * sizeof(float), err.c_str());
    return CTR_OK;
}

// CTR_TABLE_ADAM: moments of the embedding rows (zero-initialised, like the solver's, model.go:88)
int ensure_moments(ctr_handle* h) {
    if (h->emb_m) return CTR_OK;
    const size_t n = (size_t)std::max<int64_t>(h->tab_local_rows[CTR_TABLE_ITEM_EMB], 1) * h->tab_ld[CTR_TABLE_ITEM_EMB];
    GrowBuf<float> m, v;                 // both or neither
    RET(grow_buf(h, m, n)); RET(grow_buf(h, v, n));
    CU(h, cudaMemsetAsync(m, 0, n * sizeof(float), h->stream)); CU(h, cudaMemsetAsync(v, 0, n * sizeof(float), h->stream));
    h->emb_m = std::move(m); h->emb_v = std::move(v);
    return CTR_OK;
}
// the row-Adam constants of this step (the dense solver's step counter t = step + 1, gradient divided by adam_batch)
RowAdam row_adam_of(const ctr_handle* h, int adam_batch) {
    const ctr_config& c = h->cfg;
    const int t = (int)h->step + 1;
    return RowAdam{c.table_lr, c.beta1, c.beta2, c.eps, (float)(1.0 - std::pow((double)c.beta1, (double)t)), (float)(1.0 - std::pow((double)c.beta2, (double)t)),
                   adam_batch > 1 ? 1.0f / (float)adam_batch : 1.0f};
}

int deterministic_table_update(ctr_handle* h, const RowSrc& r, int B, int adam_batch) {
    const int S = h->cfg.S, D = h->cfg.D;
    size_t n = (size_t)B * (S + 1);
    if (!h->sort_tmp || h->keys.size() < n) {           // sort_tmp is allocated last: it exists only with the other four
        h->sort_tmp.reset();
        RET(dalloc(h, h->keys, n, false)); RET(dalloc(h, h->keys2, n, false));
        RET(dalloc(h, h->pos, n, false)); RET(dalloc(h, h->pos2, n, false));
        size_t bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, bytes, h->keys.get(), h->keys2.get(), h->pos.get(), h->pos2.get(), (int)n, 0, 32, h->stream);
        RET(dalloc(h, h->sort_tmp, bytes, false));
    }
    size_t bytes = h->sort_tmp.size();
    RET(launch(h, "scatter_keys", [&] {
        k_scatter_keys<<<std::min<int>((int)((n + 255) / 256), h->num_sms * 8), 256, 0, h->stream>>>(r.hist, r.item_row, S, B, r.nvalid, r.n_emb, h->keys, h->pos);
    }));
    RET(launch(h, "cub_radix_sort_pairs", [&] {
        cub::DeviceRadixSort::SortPairs(h->sort_tmp, bytes, h->keys.get(), h->keys2.get(), h->pos.get(), h->pos2.get(), (int)n, 0, 32, h->stream);
    }));
    if (h->cfg.table_opt == CTR_TABLE_ADAM) {
        RET(ensure_moments(h));
        const ctr_config& c = h->cfg;
        const int t = (int)h->step + 1;                    // the dense solver's step counter (k_adam runs after this)
        RowAdam ra{c.table_lr, c.beta1, c.beta2, c.eps, (float)(1.0 - std::pow((double)c.beta1, (double)t)), (float)(1.0 - std::pow((double)c.beta2, (double)t)),
                   adam_batch > 1 ? 1.0f / (float)adam_batch : 1.0f};
        return launch(h, "segment_adam", [&] {
            k_segment_adam<<<std::min<int>((int)((n * 32 + 255) / 256), h->num_sms * 16), 256, 0, h->stream>>>(
                h->keys2, h->pos2, (long)n, h->dUb, h->dIt, S, D, h->tab[CTR_TABLE_ITEM_EMB], h->emb_m, h->emb_v, h->tab_ld[CTR_TABLE_ITEM_EMB], ra);
        });
    }
    RET(launch(h, "segment_sgd", [&] {
        k_segment_sgd<<<std::min<int>((int)((n * 32 + 255) / 256), h->num_sms * 16), 256, 0, h->stream>>>(
            h->keys2, h->pos2, (long)n, h->dUb, h->dIt, S, D, h->tab[CTR_TABLE_ITEM_EMB], h->tab_ld[CTR_TABLE_ITEM_EMB], h->cfg.table_lr);
    }));
    return CTR_OK;
}

int step_core(ctr_handle* h, const RowSrc& r, int B, const StepOpts& o) {
    const ctr_config& c = h->cfg;
    if (B <= 0 || B > h->Bmax) return set_err(h, CTR_EINVAL, "batch %d outside (0, %d]", B, h->Bmax);
    const float d0 = o.training ? c.dropout0 : 0.0f, d1 = o.training ? c.dropout1 : 0.0f;

    if (!o.x0_ready) RET(attn_forward(h, r, B));
    const bool um = use_umma(h);
    if (um) {
        RET(umma_init(h));
        RET(umma_split_weights(h));
        umma::Args a{}; a.M = B; a.N = c.H0; a.Nz = h->H0p; a.K = h->Kp; a.C = h->H0d; a.ldc = h->H0p;
        a.drop_p = d0; a.seed = c.seed; a.stream = h->step * 4u + 0u; a.stages = h->um.stages_h0;
        RET(umma_gemm<umma::UEPI_SIGMOID_DROP>(h, "umma_fwd0_sigmoid", h->um.nch_h0, h->um.mA_X0, h->um.mB_Wt0, a));
        umma::Args b{}; b.M = B; b.N = c.H1; b.Nz = h->H1p; b.K = h->H0p; b.C = h->H1d; b.ldc = h->H1p;
        b.drop_p = d1; b.seed = c.seed; b.stream = h->step * 4u + 1u; b.stages = h->um.stages_h1;
        RET(umma_gemm<umma::UEPI_SIGMOID_DROP>(h, "umma_fwd1_sigmoid", h->um.nch_h1, h->um.mA_H0d, h->um.mB_Wt1, b));
    } else {
    {   // h0 = dropout(sigmoid(x·W0))   din.go:307-308
        GemmArgs g{}; g.A = h->X0; g.lda = h->Kp; g.B = h->W[0]; g.ldb = h->H0p; g.C = h->H0d; g.ldc = h->H0p;
        g.M = B; g.N = c.H0; g.K = h->in; g.Nz = h->H0p; g.drop_p = d0; g.seed = c.seed; g.stream = h->step * 4u + 0u;
        RET((gemm_big<false, false, EPI_SIGMOID_DROP>(h, "sgemm_fwd0_sigmoid", g)));
    }
    {   // h1 = dropout(sigmoid(h0·W1))  din.go:311-312
        GemmArgs g{}; g.A = h->H0d; g.lda = h->H0p; g.B = h->W[1]; g.ldb = h->H1p; g.C = h->H1d; g.ldc = h->H1p;
        g.M = B; g.N = c.H1; g.K = c.H0; g.Nz = h->H1p; g.drop_p = d1; g.seed = c.seed; g.stream = h->step * 4u + 1u;
        RET((gemm_big<false, false, EPI_SIGMOID_DROP>(h, "sgemm_fwd1_sigmoid", g)));
    }
    }
    const bool bwd = o.training;
    if (bwd) CU(h, cudaMemsetAsync(h->d_cost, 0, sizeof(double), h->stream));
    {
        HeadArgs a{}; a.H1d = h->H1d; a.ldh = h->H1p; a.H1 = c.H1; a.H1p = h->H1p; a.w2 = h->W[2];
        a.y = bwd ? o.d_label : nullptr; a.B = B; a.nvalid = r.nvalid; a.drop_p = d1;
        a.p = h->P; a.logit = h->Z; a.dZ1 = bwd ? h->dZ1.get() : nullptr; a.lddz = h->H1p; a.dW2 = h->G[2]; a.cost_sum = h->d_cost;
        // few, long-lived blocks: every block ends with H1 same-address atomics (dW2) and one on the cost — with one block per
        // 64 rows those serialised in L2 (~27 cycles each per address) and cost more than the 50 MB the kernel streams
        const int hgrid = std::max(1, std::min((B + 63) / 64, h->num_sms * 2));
        RET(launch(h, bwd ? "head_fwd_bwd" : "head_fwd", [&] { k_head<<<hgrid, 256, 0, h->stream>>>(a); }));
    }
    if (!bwd) return CTR_OK;

    const bool umdw = um && use_umma_dw(h, B);
    if (umdw) {   // dW1 += h0dᵀ · dZ1   (wgmma, MN-major operands, split-K over the grid)
        umma::DwArgs a{}; a.K = B; a.M = c.H0; a.N = h->H1p; a.C = h->G[1]; a.ldc = h->H1p; a.stages = h->um.dw_stages1;
        RET(umma_dw(h, "umma_dW1_splitk", h->um.nch_h1, h->um.mK_H0d, h->um.mK_dZ1, a));
    } else {   // dW1 += h0dᵀ · dZ1
        GemmArgs g{}; g.A = h->H0d; g.lda = h->H0p; g.B = h->dZ1; g.ldb = h->H1p; g.C = h->G[1]; g.ldc = h->H1p;
        g.M = c.H0; g.N = c.H1; g.K = B;
        RET(gemm_dw(h, "sgemm_dW1_splitk", g));
    }
    if (um) {
        umma::Args a{}; a.M = B; a.N = c.H0; a.Nz = h->H0p; a.K = h->H1p; a.C = h->dZ0; a.ldc = h->H0p;
        a.H = h->H0d; a.ldh = h->H0p; a.drop_p = d0; a.stages = h->um.stages_h0;
        RET(umma_gemm<umma::UEPI_DSIGMOID>(h, "umma_dZ0_dsigmoid", h->um.nch_h0, h->um.mA_dZ1, h->um.mB_W1s, a));
    } else {   // dZ0 = (dZ1 · W1ᵀ) ⊙ dsigmoid(h0d)
        GemmArgs g{}; g.A = h->dZ1; g.lda = h->H1p; g.B = h->W[1]; g.ldb = h->H1p; g.C = h->dZ0; g.ldc = h->H0p;
        g.M = B; g.N = c.H0; g.K = c.H1; g.Nz = h->H0p; g.H = h->H0d; g.ldh = h->H0p; g.drop_p = d0;
        RET((gemm_big<false, true, EPI_DSIGMOID>(h, "sgemm_dZ0_dsigmoid", g)));
    }
    if (umdw) {   // dW0 += x0ᵀ · dZ0
        umma::DwArgs a{}; a.K = B; a.M = h->in; a.N = h->H0p; a.C = h->G[0]; a.ldc = h->H0p; a.stages = h->um.dw_stages0;
        RET(umma_dw(h, "umma_dW0_splitk", h->um.nch_h0, h->um.mK_X0, h->um.mK_dZ0, a));
    } else {   // dW0 += x0ᵀ · dZ0
        GemmArgs g{}; g.A = h->X0; g.lda = h->Kp; g.B = h->dZ0; g.ldb = h->H0p; g.C = h->G[0]; g.ldc = h->H0p;
        g.M = h->in; g.N = c.H0; g.K = B;
        RET(gemm_dw(h, "sgemm_dW0_splitk", g));
    }
    const bool learn_rows = o.update && c.table_opt != CTR_TABLE_FROZEN && !r.dense;
    const bool need_attn_bwd = c.model != CTR_MODEL_YOUTUBE || learn_rows || o.want_rows;
    if (need_attn_bwd) {
        if (um) {
            umma::Args a{}; a.M = B; a.N = 2 * c.D; a.Nz = h->lddx; a.K = h->H0p; a.C = h->dX; a.ldc = h->lddx; a.stages = h->um.stages_dx;
            RET(umma_gemm<umma::UEPI_STORE>(h, "umma_dX", h->um.nch_dx, h->um.mA_dZ0, h->um.mB_W0s, a));
        } else {   // d concat[:, uP:uP+2D] = dZ0 · W0[uP:uP+2D, :]ᵀ
            GemmArgs g{}; g.A = h->dZ0; g.lda = h->H0p; g.B = h->W[0] + (long)c.uP * h->H0p; g.ldb = h->H0p;
            g.C = h->dX; g.ldc = h->lddx; g.M = B; g.N = 2 * c.D; g.K = c.H0; g.Nz = h->lddx;
            RET((gemm_big<false, true, EPI_STORE>(h, "sgemm_dX", g)));
        }
        const bool fused_only = o.comm || o.table_grad;        // multi-GPU steps always scatter with red.add
        const bool sorted_rows = c.table_opt == CTR_TABLE_SGD_DETERMINISTIC || c.table_opt == CTR_TABLE_ADAM;   // per-unique-row update from sorted keys
        const bool adam_rows = learn_rows && c.table_opt == CTR_TABLE_ADAM;
        const bool shard_adam = adam_rows && o.peer;           // owner-side gradient shards + touched lists (comm_impl.cuh)
        const bool buffers = o.want_rows || (learn_rows && sorted_rows && !fused_only);
        if (buffers) RET(ensure_rowgrad_buffers(h, B));
        BwdOut bo{}; bo.datt = h->G[3]; bo.dUb = buffers ? h->dUb.get() : nullptr; bo.dIt = buffers ? h->dIt.get() : nullptr;
        bo.sgd = (learn_rows && (c.table_opt == CTR_TABLE_SGD || fused_only)) ? 1 : 0;
        // what leaves the kernel: -lr/world * gradient (SGD: added straight into rows), or 1/world * gradient (Adam on a
        // replicated table: the all-reduced sum is the global-batch gradient the row solver consumes)
        bo.neg_lr = (adam_rows ? 1.0f : -c.table_lr) * o.grad_scale;
        bo.scatter_base = o.table_grad ? o.table_grad : h->tab[CTR_TABLE_ITEM_EMB];
        const bool hot = bo.sgd && attn_path(h, r).bwd != ATTN_GEN && !o.comm;
        if (hot) { RET(ensure_hot(h)); bo.hot_acc = h->hot_acc; bo.hot_rows = h->hot_rows; bo.hot_reps = h->hot_reps; }
        const bool peer_hot = o.peer && bo.sgd && h->comm.hot_k > 0;
        if (peer_hot) { bo.hot_acc = h->comm.hot_acc; bo.hot_rows = h->comm.hot_k; bo.hot_reps = h->comm.hot_reps; }
        if (shard_adam) {
            for (int j = 0; j < h->comm.world; j++) bo.peer_adam[j] = h->comm.peer_adam[j];
            bo.adam = h->comm.adam_lay;
            if (peer_hot) bo.hot_touch = h->comm.hot_sum.get() + (size_t)h->comm.hot_k * c.D;
        }
        // sharded tables: nobody's red.add may land in a row before every rank's forward has read it (row Adam adds
        // into the gradient shards, which nobody reads before the owner's update)
        if (o.peer && bo.sgd && !shard_adam) RET(comm_barrier(h));
        RET(attn_backward(h, r, bo, B));
        if (peer_hot)      // replica accumulators of the replicated hot rows → this rank's gradient sum (all-reduced below)
            RET(launch(h, "hot_rows_fold", [&] {
                k_hot_apply<<<h->num_sms * 4, 256, 0, h->stream>>>(h->comm.hot_sum, c.D, h->comm.hot_acc, h->comm.hot_k, h->comm.hot_reps, c.D, 1.0f);
            }));
        if (shard_adam) {  // every rank's red.adds into this rank's gradient shard have landed (and every forward has read
                           // the rows): the owner updates the rows its list holds
            RET(comm_barrier(h));
            RET(ensure_moments(h));
            const RowAdam ra = row_adam_of(h, o.adam_batch > 0 ? o.adam_batch : B);
            RET(launch(h, "shard_row_adam", [&] {
                k_shard_adam<<<h->num_sms * 8, 256, 0, h->stream>>>(h->comm.peer_adam[h->comm.rank], h->comm.adam_lay, h->tab[CTR_TABLE_ITEM_EMB],
                                                                   h->emb_m, h->emb_v, h->tab_ld[CTR_TABLE_ITEM_EMB], c.D, ra);
            }));
        }
        if (hot && h->hot_rows > 0)
            RET(launch(h, "hot_rows_apply", [&] {
                k_hot_apply<<<h->num_sms * 4, 256, 0, h->stream>>>(bo.scatter_base, h->tab_ld[CTR_TABLE_ITEM_EMB], h->hot_acc,
                                                                h->hot_rows, h->hot_reps, c.D, 1.0f);
            }));
        if (learn_rows && sorted_rows && !fused_only) RET(deterministic_table_update(h, r, B, o.adam_batch > 0 ? o.adam_batch : B));
    }
    if (o.update) {
        const bool tg = o.table_grad && c.table_opt != CTR_TABLE_FROZEN;
        const bool ph = o.peer && c.table_opt != CTR_TABLE_FROZEN && h->comm.hot_k > 0;
        const bool ph_adam = ph && c.table_opt == CTR_TABLE_ADAM;      // the hot rows' touch marks travel with their sums
        const size_t ph_n = (size_t)h->comm.hot_k * (c.D + (ph_adam ? 1 : 0));
        if (o.comm || o.table_grad) RET(comm_allreduce_grads(h, tg ? o.table_grad : ph ? h->comm.hot_sum.get() : nullptr, tg ? o.table_grad_n : ph ? ph_n : 0));
        if (ph_adam) {
            const RowAdam ra = row_adam_of(h, o.adam_batch > 0 ? o.adam_batch : B);
            RET(launch(h, "hot_rows_adam", [&] {
                k_hot_adam<<<h->num_sms * 8, 256, 0, h->stream>>>(h->comm.hot_tab, h->comm.hot_sum, h->comm.hot_sum.get() + (size_t)h->comm.hot_k * c.D,
                                                                 h->comm.hot_m, h->comm.hot_v, h->comm.hot_k, c.D, ra);
            }));
        } else if (ph)
            RET(launch(h, "hot_rows_apply", [&] {
                k_apply_table_grad<<<h->num_sms * 8, 256, 0, h->stream>>>(h->comm.hot_tab, h->comm.hot_sum, (long)h->comm.hot_k * c.D / 4);
            }));
        if (tg && c.table_opt == CTR_TABLE_ADAM) {
            RET(ensure_moments(h));
            const int t = (int)h->step + 1; const int ab = o.adam_batch > 0 ? o.adam_batch : B;
            RowAdam ra{c.table_lr, c.beta1, c.beta2, c.eps, (float)(1.0 - std::pow((double)c.beta1, (double)t)), (float)(1.0 - std::pow((double)c.beta2, (double)t)),
                       ab > 1 ? 1.0f / (float)ab : 1.0f};
            RET(launch(h, "apply_table_adam", [&] {
                k_apply_table_adam<<<h->num_sms * 8, 256, 0, h->stream>>>(h->tab[CTR_TABLE_ITEM_EMB], o.table_grad, h->emb_m, h->emb_v,
                                                                         (long)h->tab_rows[CTR_TABLE_ITEM_EMB], (int)h->tab_ld[CTR_TABLE_ITEM_EMB], ra);
            }));
        } else if (tg)
            RET(launch(h, "apply_table_grad", [&] {
                k_apply_table_grad<<<h->num_sms * 8, 256, 0, h->stream>>>(h->tab[CTR_TABLE_ITEM_EMB], o.table_grad, (long)(o.table_grad_n / 4));
            }));
        AdamArgs a{};
        const int in = h->in;
        a.t[0] = AdamTensor{h->W[0], h->G[0], h->Mo[0], h->Vo[0], in, c.H0, h->H0p};
        a.t[1] = AdamTensor{h->W[1], h->G[1], h->Mo[1], h->Vo[1], c.H0, c.H1, h->H1p};
        a.t[2] = AdamTensor{h->W[2], h->G[2], h->Mo[2], h->Vo[2], 1, c.H1, h->H1p};
        a.t[3] = AdamTensor{h->W[3], h->G[3], h->Mo[3], h->Vo[3], 1, c.S, h->Sp};
        a.nt = c.model == CTR_MODEL_YOUTUBE ? 3 : 4;       // Learnable(): dnn.go:153 vs din.go:161-169
        const int t = (int)h->step + 1;
        const int ab = o.adam_batch > 0 ? o.adam_batch : B;
        a.gscale = o.grad_scale;
        a.lr = c.lr; a.l2 = c.l2; a.inv_batch = ab > 1 ? 1.0f / (float)ab : 1.0f; a.b1 = c.beta1; a.b2 = c.beta2; a.eps = c.eps;
        a.c1 = (float)(1.0 - std::pow((double)c.beta1, (double)t));
        a.c2 = (float)(1.0 - std::pow((double)c.beta2, (double)t));
        const bool split_in_adam = um && h->um.ready;
        if (split_in_adam) {     // the next step's K-major TF32 operand copies come straight out of the optimiser (same layouts as umma_split_weights)
            auto& u = h->um;
            a.sp[0][0] = SplitOut{u.Wt0[0], u.Wt0[1], (long)h->Kp, 1, 0, in};                     // W0ᵀ [H0, in]
            a.sp[0][1] = SplitOut{u.W0s[0], u.W0s[1], (long)h->H0p, 0, c.uP, 2 * c.D};            // W0[uP:uP+2D, :]
            a.sp[1][0] = SplitOut{u.Wt1[0], u.Wt1[1], (long)h->H0p, 1, 0, c.H0};                  // W1ᵀ [H1, H0]
            a.sp[1][1] = SplitOut{u.W1s[0], u.W1s[1], (long)h->H1p, 0, 0, c.H0};                  // W1  [H0, H1]
            a.nsp[0] = a.nsp[1] = 2;
        }
        RET(launch(h, "adam_dense", [&] { k_adam<<<h->num_sms * 2, 256, 0, h->stream>>>(a); }));
        h->um.dirty = !split_in_adam;
        h->step++;
    }
    return CTR_OK;
}

int zero_grads(ctr_handle* h) {
    CU(h, cudaMemsetAsync(h->Gflat, 0, h->Gflat_n * sizeof(float), h->stream));
    return CTR_OK;
}

// Placement of the ITEM_* tables under world > 1: sharded by row % world (large tables), or replicated on every
// rank.  cfg.reserved[1]: 0 = by size (> 32 MB shards), 1 = always shard, 2 = always replicate.  USER_FEAT is
// always replicated.
bool table_sharded(const ctr_handle* h, int which, int64_t nrows, int32_t width) {
    if (h->comm.world <= 1 || which == CTR_TABLE_USER_FEAT) return false;
    const int pol = h->cfg.reserved[1];
    if (pol == 1) return true;
    if (pol == 2) return false;
    return (size_t)nrows * round_up(width, 4) * sizeof(float) > kReplicateBytes;
}

// (re)allocates table `which` for nrows logical rows; decides the placement; leaves the rows zeroed
void table_free(ctr_handle* h, int which) {
    if (h->tab_vmm[which].live) { cudaStreamSynchronize(h->stream); vmm_free(&h->tab_vmm[which]); }
    else h->tab_mem[which].reset();
    h->tab[which] = nullptr;
}
// device memory of a table: shareable VMM memory when the table is sharded (peers map it), growable memory otherwise
int table_mem(ctr_handle* h, int which, bool shard, size_t bytes) {
    table_free(h, which);
    if (shard) {
        std::string err;
        if (!vmm_alloc(bytes, h->dev, &h->tab_vmm[which], &err)) return set_err(h, CTR_ENOMEM, "table %d (%zu bytes): %s", which, bytes, err.c_str());
        h->tab[which] = (float*)h->tab_vmm[which].ptr;
    } else {
        RET(grow_buf(h, h->tab_mem[which], bytes / sizeof(float)));
        h->tab[which] = h->tab_mem[which].get();
    }
    CU(h, cudaMemsetAsync(h->tab[which], 0, bytes, h->stream));
    return CTR_OK;
}
// what new contents of a table reset, whether it was reallocated (table_alloc) or rewritten in place (ctr_item_emb_train)
void table_new_state(ctr_handle* h, int which) {
    if (which == CTR_TABLE_ITEM_EMB) {
        h->comm.replicate = h->comm.world > 1 && !h->tab_sharded[which];
        if (h->hot_acc) { h->hot_acc.reset(); h->hot_rows = 0; }
        h->emb_m.reset(); h->emb_v.reset();                       // a new table starts a new solver state
    }
    if (which != CTR_TABLE_USER_FEAT) h->tab_gen++;           // peers hold mappings of the old allocation
}
int table_alloc(ctr_handle* h, int which, int64_t nrows, int32_t width) {
    const long ld = round_up(width, 4);                       // 16-byte aligned rows for 128-bit loads
    const bool shard = table_sharded(h, which, nrows, width);
    const int64_t local = shard ? (nrows - h->comm.rank + h->comm.world - 1) / h->comm.world : nrows;
    const size_t bytes = (size_t)std::max<int64_t>(local, 1) * ld * sizeof(float);
    RET(table_mem(h, which, shard, bytes));
    h->tab_ld[which] = ld; h->tab_rows[which] = nrows; h->tab_local_rows[which] = local; h->tab_width[which] = width;
    h->tab_sharded[which] = shard;
    table_new_state(h, which);
    return CTR_OK;
}

RowSrc idx_src(const ctr_handle* h, const int* d_user, const int* d_item, const int* d_hist, int B) {
    RowSrc r{};
    r.emb = h->tab[CTR_TABLE_ITEM_EMB]; r.lde = h->tab_ld[CTR_TABLE_ITEM_EMB];
    r.ufeat = h->tab[CTR_TABLE_USER_FEAT]; r.ldu = h->tab_ld[CTR_TABLE_USER_FEAT];
    r.ifeat = h->tab[CTR_TABLE_ITEM_FEAT]; r.ldi = h->tab_ld[CTR_TABLE_ITEM_FEAT];
    r.user_row = d_user; r.item_row = d_item; r.hist = d_hist;
    r.dense = 0; r.nvalid = B;
    r.n_emb = (int)std::min<int64_t>(h->tab_rows[CTR_TABLE_ITEM_EMB], 0x7fffffff);
    r.n_user = (int)std::min<int64_t>(h->tab_rows[CTR_TABLE_USER_FEAT], 0x7fffffff);
    r.n_ifeat = (int)std::min<int64_t>(h->tab_rows[CTR_TABLE_ITEM_FEAT], 0x7fffffff);
    r.world = 1;
    return r;
}

// every table the configuration needs is uploaded with its width (this rank's shard of a row-sharded one)
int check_widths(const ctr_handle* h) {
    const ctr_config& c = h->cfg;
    if (!h->tab[CTR_TABLE_ITEM_EMB] || h->tab_width[CTR_TABLE_ITEM_EMB] != c.D)
        return set_err(h, CTR_ESTATE, "ITEM_EMB table not uploaded with width D=%d", c.D);
    if (c.uP > 0 && (!h->tab[CTR_TABLE_USER_FEAT] || h->tab_width[CTR_TABLE_USER_FEAT] != c.uP))
        return set_err(h, CTR_ESTATE, "USER_FEAT table not uploaded with width uP=%d", c.uP);
    if (c.cF > 0 && (!h->tab[CTR_TABLE_ITEM_FEAT] || h->tab_width[CTR_TABLE_ITEM_FEAT] != c.cF))
        return set_err(h, CTR_ESTATE, "ITEM_FEAT table not uploaded with width cF=%d", c.cF);
    return CTR_OK;
}

int check_tables(const ctr_handle* h) {
    RET(check_widths(h));
    if (h->comm.world > 1 && (h->tab_sharded[CTR_TABLE_ITEM_EMB] || h->tab_sharded[CTR_TABLE_ITEM_FEAT]))
        return set_err(h, CTR_ESTATE, "this entry point gathers locally: ITEM_EMB / ITEM_FEAT must both be replicated (or both sharded for the train / predict entry points)");
    return CTR_OK;
}

int stage_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row, const int32_t* hist, const float* label, int B) {
    const int S = h->cfg.S;
    CU(h, cudaMemcpyAsync(h->s_user, user_row, sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpyAsync(h->s_item, item_row, sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, h->stream));
    if (S > 0) CU(h, cudaMemcpyAsync(h->s_hist, hist, sizeof(int) * (size_t)B * S, cudaMemcpyHostToDevice, h->stream));
    if (label) CU(h, cudaMemcpyAsync(h->s_label, label, sizeof(float) * (size_t)B, cudaMemcpyHostToDevice, h->stream));
    return CTR_OK;
}

int read_cost(ctr_handle* h, int B, float* cost) {
    double s = 0;
    CU(h, cudaMemcpyAsync(&s, h->d_cost, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    *cost = -(float)(s / (double)B);         // -mean, cost.go:15
    if (h->comm.h_err && *h->comm.h_err) return set_err(h, CTR_ECOMM, "peer barrier timed out waiting for rank %d (a rank left the step loop?)", *h->comm.h_err - 1);
    return CTR_OK;
}

int dense_src(ctr_handle* h, const int32_t ranges[8], int32_t xcols, RowSrc* out) {
    const ctr_config& c = h->cfg;
    const int up0 = ranges[0], up1 = ranges[1], ub0 = ranges[2], ub1 = ranges[3], it0 = ranges[4], it1 = ranges[5], cx0 = ranges[6], cx1 = ranges[7];
    if (up1 - up0 != c.uP || ub1 - ub0 != c.S * c.D || it1 - it0 != c.D || cx1 - cx0 != c.cF)
        return set_err(h, CTR_EINVAL, "SampleInfo ranges do not match the model dims (uP=%d S*D=%d D=%d cF=%d)", c.uP, c.S * c.D, c.D, c.cF);
    for (int i = 0; i < 8; i++) if (ranges[i] < 0 || ranges[i] > xcols) return set_err(h, CTR_EINVAL, "SampleInfo range outside [0, xcols=%d]", xcols);
    RowSrc r{}; r.dense = 1; r.world = 1; r.ldx = xcols; r.up0 = up0; r.ub0 = ub0; r.it0 = it0; r.cx0 = cx0;
    *out = r;
    return CTR_OK;
}

int upload_dense(ctr_handle* h, const float* X, const float* Y, int64_t n, int32_t xcols) {
    size_t need = (size_t)n * xcols;
    RET(reserve(h, h->dXd, need, false));
    CU(h, cudaMemcpyAsync(h->dXd, X, need * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    if (Y) {
        RET(reserve(h, h->dYd, (size_t)n, false));
        CU(h, cudaMemcpyAsync(h->dYd, Y, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    }
    return CTR_OK;
}

void gaussian_fill(std::vector<float>& w, uint32_t seed, uint32_t stream) {
    for (size_t i = 0; i < w.size(); i++) {       // Box–Muller on the counter RNG
        uint64_t z = mix64(seed, stream, (uint64_t)i);
        double u1 = ((double)(z >> 40) + 1.0) * (1.0 / 16777217.0);
        double u2 = (double)((z >> 8) & 0xFFFFFFull) * (1.0 / 16777216.0);
        w[i] = (float)(std::sqrt(-2.0 * std::log(u1)) * std::cos(6.283185307179586 * u2));
    }
}

}  // namespace

#include "comm_impl.cuh"

// item2vec host plan: Huffman tree as dictionary.HuffnamTree builds it (huffman.go:23-57) and every word's
// root→leaf path as Node.GetPath(maxDepth) returns it (node.go:26-43), as a CSR of (inner node, child code).
// dictionary.HuffnamTree (huffman.go:23-57) over leaves already in stable count order (`leaves` = word ids sorted by
// count, ties in id order): merged nodes are created in non-decreasing value order and inserted before every queued
// node of equal value, so they win ties and equal-valued merged nodes pop newest-first.  O(V).
// parent / code are indexed by tree node (leaves [0,V), inner nodes V + creation index); node_val [V-1].
// Ids that never occur (count 0) are not dictionary words in the reference (the dictionary is built from the stream,
// dictionary.go:70-81).  Here they go through the literal procedure like every other leaf (they chain into a comb of
// zero-valued nodes below the lightest real word, which leaves every real word's path what the procedure gives it), but
// no PATH is built for them — they are never trained and walking a comb as deep as their number is quadratic.
// Returns the number of inner nodes created.
static int i2v_huffman_sorted(const int64_t* cnt_by_word, const int* leaves, int V, std::vector<int>& parent, std::vector<unsigned char>& code,
                              std::vector<long long>& node_val) {
    parent.assign((size_t)2 * V - 1, -1); code.assign((size_t)2 * V - 1, 0); node_val.assign((size_t)std::max(V - 1, 1), 0);
    const size_t first = 0;
    const int Vp = V;
    // merged queue as runs of equal value; inside a run the newest node pops first, runs are in non-decreasing value order
    std::vector<long long> run_val; std::vector<int> run_begin, run_top;      // run r holds ids mq[run_begin[r] .. run_top[r])
    std::vector<int> mq; mq.reserve((size_t)V);
    size_t rh = 0, lh = first; int next_id = V;
    for (int made = 0; made < Vp - 1; made++) {
        long long pv[2]; int pid[2];
        for (int k = 0; k < 2; k++) {
            while (rh + 1 < run_val.size() && run_top[rh] == run_begin[rh]) rh++;          // never step past the last run: it may refill
            const bool have_m = rh < run_val.size() && run_top[rh] > run_begin[rh];
            const bool use_m = have_m && (lh >= (size_t)V || run_val[rh] <= cnt_by_word[leaves[lh]]);
            if (use_m) { pv[k] = run_val[rh]; pid[k] = mq[(size_t)--run_top[rh]]; if (rh + 1 == run_val.size()) mq.resize((size_t)run_top[rh]); }
            else { pv[k] = cnt_by_word[leaves[lh]]; pid[k] = leaves[lh]; lh++; }
        }
        const long long val = pv[0] + pv[1]; const int id = next_id++;
        node_val[(size_t)(id - V)] = val;
        code[(size_t)pid[0]] = 0; code[(size_t)pid[1]] = 1; parent[(size_t)pid[0]] = id; parent[(size_t)pid[1]] = id;
        if (!run_val.empty() && run_val.back() == val && run_top.back() == (int)mq.size()) { mq.push_back(id); run_top.back() = (int)mq.size(); }
        else if (!run_val.empty() && run_top.back() == run_begin.back() && run_top.back() == (int)mq.size()) {      // reuse the emptied last run
            run_val.back() = val; mq.push_back(id); run_top.back() = (int)mq.size();
        } else { run_val.push_back(val); run_begin.push_back((int)mq.size()); mq.push_back(id); run_top.push_back((int)mq.size()); }
    }
    return std::max(Vp - 1, 0);
}

// item2vec host plan (CPU-only entry ctr_i2v_paths): Huffman tree + every word's root→leaf path as Node.GetPath(maxDepth)
// returns it (node.go:26-43), as a CSR of (inner node, child code).
static void i2v_build_paths(const std::vector<int64_t>& cnt, int V, int max_depth, std::vector<int64_t>& node_val,
                            std::vector<long long>& poff, std::vector<int>& pnode, std::vector<unsigned char>& pcode) {
    std::vector<int> leaves((size_t)V);
    for (int i = 0; i < V; i++) leaves[(size_t)i] = i;
    std::stable_sort(leaves.begin(), leaves.end(), [&](int x, int y) { return cnt[(size_t)x] < cnt[(size_t)y]; });
    std::vector<int> parent; std::vector<unsigned char> code; std::vector<long long> nv;
    i2v_huffman_sorted(cnt.data(), leaves.data(), V, parent, code, nv);
    node_val.assign(nv.begin(), nv.begin() + std::max(V - 1, 0));
    poff.assign((size_t)V + 1, 0); pnode.clear(); pcode.clear();
    std::vector<int> chain;
    for (int w = 0; w < V; w++) {                          // Node.GetPath(maxDepth), node.go:26-43
        if (cnt[(size_t)w] == 0) { poff[(size_t)w + 1] = (long long)pnode.size(); continue; }     // never occurs: no path
        chain.clear();
        for (int p = w; p != -1; p = parent[(size_t)p]) chain.push_back(p);
        const int len = (int)chain.size(), depth = std::min(max_depth, len);
        for (int i = 0; i < depth - 1; i++) { pnode.push_back(chain[(size_t)(len - 1 - i)] - V); pcode.push_back(code[(size_t)chain[(size_t)(len - 2 - i)]]); }
        poff[(size_t)w + 1] = (long long)pnode.size();
    }
}

// ---- ctr_knn_search (knn.cuh) ----------------------------------------------------------------------------------------
namespace {
struct KnnArgs {
    const double* qvec; const int* qrow; const int* excl; int nq, k; long rows_per_slice; int slices;
    double* sl_sim; int* sl_row;
};
template <int QT, bool ROWQ>
void knn_scan_launch(ctr_handle* h, const KnnArgs& a, size_t smem) {
    const int T = CTR_TABLE_ITEM_EMB;
    const bool sh = h->tab_sharded[T];            // this rank's shard: local row l is global row l·world + rank
    dim3 grid((a.nq + QT - 1) / QT, a.slices);
    knn::k_knn_scan<QT, ROWQ><<<grid, knn::kThreads, smem, h->stream>>>(h->tab[T], h->tab_ld[T], (long)h->tab_local_rows[T], sh ? h->comm.world : 1,
                                                                       sh ? h->comm.rank : 0, h->tab_width[T], a.qvec, a.qrow, a.excl, a.nq, a.k,
                                                                       a.rows_per_slice, a.sl_sim, a.sl_row);
}
template <int QT, bool ROWQ>
int knn_scan_occupancy(size_t smem) {
    cudaFuncSetAttribute(knn::k_knn_scan<QT, ROWQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, knn::k_knn_scan<QT, ROWQ>, knn::kThreads, smem);
    return std::max(n, 1);
}
// QT in {1, 2, 4, 8, 16}: the query-tile width the scan kernel was instantiated for
template <bool ROWQ>
int knn_scan_dispatch(ctr_handle* h, int QT, KnnArgs a, bool occupancy_only, size_t smem, int* occ) {
    switch (QT) {
        case 1:  if (occupancy_only) *occ = knn_scan_occupancy<1, ROWQ>(smem);  else knn_scan_launch<1, ROWQ>(h, a, smem);  break;
        case 2:  if (occupancy_only) *occ = knn_scan_occupancy<2, ROWQ>(smem);  else knn_scan_launch<2, ROWQ>(h, a, smem);  break;
        case 4:  if (occupancy_only) *occ = knn_scan_occupancy<4, ROWQ>(smem);  else knn_scan_launch<4, ROWQ>(h, a, smem);  break;
        case 8:  if (occupancy_only) *occ = knn_scan_occupancy<8, ROWQ>(smem);  else knn_scan_launch<8, ROWQ>(h, a, smem);  break;
        default: if (occupancy_only) *occ = knn_scan_occupancy<16, ROWQ>(smem); else knn_scan_launch<16, ROWQ>(h, a, smem); break;
    }
    return CTR_OK;
}

}  // namespace

// ---- live ubcache updates (ctr_ubcache_append / ctr_ubcache_set; kernels in ubcache.cuh)
namespace {
// bits needed to hold every value in [0, v]
int bits_for(unsigned long long v) { return v ? 64 - __builtin_clzll(v) : 0; }

// user rows an append / set may name: below the cache's user count, USER_FEAT's rows or the user id map's size
int64_t ub_row_bound(const ctr_handle* h) {
    return std::max({h->ub_off ? h->ub_users : (int64_t)0, h->tab_rows[CTR_TABLE_USER_FEAT], h->idm_keys[CTR_IDMAP_USER] ? h->idm_n[CTR_IDMAP_USER] : (int64_t)0});
}

// device workspace of one call, carved from a scratch slot in 256-byte pieces (pass base = nullptr to size it)
struct Carve {
    char* base; size_t used = 0;
    template <typename T> T* take(size_t n) { T* p = (T*)(base + used); used += (std::max<size_t>(n, 1) * sizeof(T) + 255) & ~(size_t)255; return p; }
};

// The batch of an append or set, as the touched users' segments (ubcache.cuh): T touched users, tuser / bb / bcnt / ob /
// oe [T], dcum [T+1], and the batch events bts / bit they index.
struct UbBatch {
    int T = 0; int64_t grow = 0;                      // grow: dcum[T], the change of the event count
    int *tuser = nullptr, *bb = nullptr, *bcnt = nullptr, *bit = nullptr;
    long long *ob = nullptr, *oe = nullptr, *dcum = nullptr, *bts = nullptr;
};

// the stored cache's user and event counts (0, 0 when none was uploaded)
void ub_stored(const ctr_handle* h, long long* n_users, long long* n) {
    *n_users = h->ub_off ? h->ub_users : 0; *n = h->ub_off ? h->ub_n : 0;
}

// append: the batch to the device, sorted by (user, ts desc, arrival desc) with CUB radix sort, run-length encoded by user
int ub_batch_append(ctr_handle* h, const int32_t* user_rows, const int64_t* ts, const int32_t* item_rows, int64_t m,
                    int32_t max_row, int64_t tmin, int64_t tmax, UbBatch* ub) {
    long long U, n; ub_stored(h, &U, &n);
    const int ubits = bits_for((unsigned long long)max_row), tbits = bits_for((unsigned long long)tmax - (unsigned long long)tmin);
    const bool two_pass = ubits + tbits > 64;
    size_t tmp = 0, t1 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t1, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, (int)m, 0, 64, h->stream); tmp = std::max(tmp, t1);
    cub::DeviceRadixSort::SortPairs(nullptr, t1, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, (int)m, 0, 32, h->stream); tmp = std::max(tmp, t1);
    cub::DeviceRunLengthEncode::Encode(nullptr, t1, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int)m, h->stream); tmp = std::max(tmp, t1);
    cub::DeviceScan::ExclusiveSum(nullptr, t1, (int*)nullptr, (int*)nullptr, (int)m, h->stream); tmp = std::max(tmp, t1);
    cub::DeviceScan::ExclusiveSum(nullptr, t1, (long long*)nullptr, (long long*)nullptr, (int)m + 1, h->stream); tmp = std::max(tmp, t1);
    auto carve = [&](char* base, UbBatch& b, int*& du, long long*& dts, int*& dit, unsigned long long*& ka, unsigned long long*& kb,
                     int*& ia, int*& ib, int*& nruns, long long*& delta, void*& ctmp) {
        Carve c{base};
        du = c.take<int>(m); dts = c.take<long long>(m); dit = c.take<int>(m);
        ka = c.take<unsigned long long>(m); kb = c.take<unsigned long long>(m); ia = c.take<int>(m); ib = c.take<int>(m);
        b.tuser = c.take<int>(m); b.bts = c.take<long long>(m); b.bit = c.take<int>(m);
        b.bb = c.take<int>(m); b.bcnt = c.take<int>(m); b.ob = c.take<long long>(m); b.oe = c.take<long long>(m);
        b.dcum = c.take<long long>(m + 1); delta = c.take<long long>(m + 1); nruns = c.take<int>(1);
        ctmp = c.take<char>(tmp);
        return c.used;
    };
    int *du, *dit, *ia, *ib, *nruns; long long *dts, *delta; unsigned long long *ka, *kb; void* ctmp; char* ws = nullptr;
    RET(scratch_get(h, 5, carve(nullptr, *ub, du, dts, dit, ka, kb, ia, ib, nruns, delta, ctmp), (void**)&ws));
    carve(ws, *ub, du, dts, dit, ka, kb, ia, ib, nruns, delta, ctmp);
    int* bu = ia;                                       // the sorted users reuse the first index buffer once it is read
    CU(h, cudaMemcpyAsync(du, user_rows, sizeof(int) * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpyAsync(dts, ts, sizeof(long long) * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpyAsync(dit, item_rows, sizeof(int) * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((m + 255) / 256, (int64_t)h->num_sms * 8));
    RET(launch(h, "ubcache_sort_keys", [&] { k_ub_sort_keys<<<grid, 256, 0, h->stream>>>(du, dts, m, tbits, tmax, two_pass, ka, ia); }));
    int* idx = ib;
    RET(launch(h, "ubcache_sort", [&] {
        cub::DeviceRadixSort::SortPairs(ctmp, tmp, ka, kb, ia, ib, (int)m, 0, std::max(1, two_pass ? tbits : ubits + tbits), h->stream);
    }));
    if (two_pass) {                                      // then by user row, stably
        RET(launch(h, "ubcache_user_keys", [&] { k_ub_user_keys<<<grid, 256, 0, h->stream>>>(du, ib, m, (unsigned*)ka); }));
        RET(launch(h, "ubcache_sort", [&] {
            cub::DeviceRadixSort::SortPairs(ctmp, tmp, (unsigned*)ka, (unsigned*)kb, ib, ia, (int)m, 0, std::max(1, ubits), h->stream);
        }));
        idx = ia; bu = ib;
    }
    RET(launch(h, "ubcache_gather", [&] { k_ub_gather_batch<<<grid, 256, 0, h->stream>>>(idx, du, dts, dit, m, bu, ub->bts, ub->bit); }));
    RET(launch(h, "ubcache_rle", [&] { cub::DeviceRunLengthEncode::Encode(ctmp, tmp, bu, ub->tuser, ub->bcnt, nruns, (int)m, h->stream); }));
    int T = 0;
    CU(h, cudaMemcpyAsync(&T, nruns, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    ub->T = T; ub->grow = m;
    RET(launch(h, "ubcache_scan", [&] { cub::DeviceScan::ExclusiveSum(ctmp, tmp, ub->bcnt, ub->bb, T, h->stream); }));
    RET(launch(h, "ubcache_touched", [&] {
        k_ub_touched<<<(T + 256) / 256, 256, 0, h->stream>>>(ub->tuser, nullptr, nullptr, T, h->ub_off, U, n, ub->bb, ub->bcnt, ub->ob, ub->oe, delta);
    }));
    return launch(h, "ubcache_scan", [&] { cub::DeviceScan::ExclusiveSum(ctmp, tmp, delta, ub->dcum, T + 1, h->stream); });
}

// set: the n_set sequences to the device, their users sorted (radix sort of (row, entry)); each touched user's new
// events stay where the caller put them
int ub_batch_set(ctr_handle* h, const int32_t* user_rows, const int64_t* offsets, const int64_t* ts, const int32_t* item_rows,
                 int64_t ns, int64_t m, int32_t max_row, UbBatch* ub) {
    long long U, n; ub_stored(h, &U, &n);
    const int ubits = bits_for((unsigned long long)max_row);
    size_t tmp = 0, t1 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t1, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, (int)ns, 0, 32, h->stream); tmp = std::max(tmp, t1);
    cub::DeviceScan::ExclusiveSum(nullptr, t1, (long long*)nullptr, (long long*)nullptr, (int)ns + 1, h->stream); tmp = std::max(tmp, t1);
    auto carve = [&](char* base, UbBatch& b, int*& du, long long*& soff, int*& iota, int*& perm, long long*& delta, void*& ctmp) {
        Carve c{base};
        du = c.take<int>(ns); soff = c.take<long long>(ns + 1); iota = c.take<int>(ns); perm = c.take<int>(ns);
        b.bts = c.take<long long>(m); b.bit = c.take<int>(m);
        b.tuser = c.take<int>(ns); b.bb = c.take<int>(ns); b.bcnt = c.take<int>(ns); b.ob = c.take<long long>(ns); b.oe = c.take<long long>(ns);
        b.dcum = c.take<long long>(ns + 1); delta = c.take<long long>(ns + 1);
        ctmp = c.take<char>(tmp);
        return c.used;
    };
    int *du, *iota, *perm; long long *soff, *delta; void* ctmp; char* ws = nullptr;
    RET(scratch_get(h, 5, carve(nullptr, *ub, du, soff, iota, perm, delta, ctmp), (void**)&ws));
    carve(ws, *ub, du, soff, iota, perm, delta, ctmp);
    std::vector<int> seq((size_t)ns);
    for (int64_t i = 0; i < ns; i++) seq[(size_t)i] = (int)i;
    CU(h, cudaMemcpyAsync(du, user_rows, sizeof(int) * (size_t)ns, cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpyAsync(soff, offsets, sizeof(long long) * (size_t)(ns + 1), cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpyAsync(iota, seq.data(), sizeof(int) * (size_t)ns, cudaMemcpyHostToDevice, h->stream));
    if (m > 0) {
        CU(h, cudaMemcpyAsync(ub->bts, ts, sizeof(long long) * (size_t)m, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(ub->bit, item_rows, sizeof(int) * (size_t)m, cudaMemcpyHostToDevice, h->stream));
    }
    RET(launch(h, "ubcache_sort", [&] {
        cub::DeviceRadixSort::SortPairs(ctmp, tmp, (unsigned*)du, (unsigned*)ub->tuser, iota, perm, (int)ns, 0, std::max(1, ubits), h->stream);
    }));
    const int T = (int)ns;
    RET(launch(h, "ubcache_touched", [&] {
        k_ub_touched<<<(T + 256) / 256, 256, 0, h->stream>>>(ub->tuser, perm, soff, T, h->ub_off, U, n, ub->bb, ub->bcnt, ub->ob, ub->oe, delta);
    }));
    RET(launch(h, "ubcache_scan", [&] { cub::DeviceScan::ExclusiveSum(ctmp, tmp, delta, ub->dcum, T + 1, h->stream); }));
    long long grow = 0;
    CU(h, cudaMemcpyAsync(&grow, ub->dcum + T, sizeof grow, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    ub->T = T; ub->grow = grow;
    return CTR_OK;
}

// the rewrite: offsets, stored events and new events into the spare CSR, then the swap.  It returns with the kernels
// still queued; the readers order themselves after them: engine-stream kernels by stream order, ctr_train_keys' windows
// by the window stream's wait on the engine stream at the start of that call.
int ub_rewrite(ctr_handle* h, const UbBatch& ub, bool replace, int64_t new_users) {
    long long U, n; ub_stored(h, &U, &n);
    const int64_t n_new = n + ub.grow;
    // The spare may still be read by work enqueued before the last swap: on the engine stream that is ordered before
    // this call's kernels; the window stream of ctr_train_keys is drained here.
    if (h->win_stream) CU(h, cudaStreamSynchronize(h->win_stream));
    // 1/8 slack, so steady growth rarely reallocates
    if (h->ubx_off.size() < (size_t)new_users + 1) RET(dalloc(h, h->ubx_off, (size_t)new_users + 1 + (size_t)new_users / 8, false));
    if (h->ubx_ts.size() < (size_t)n_new) RET(dalloc(h, h->ubx_ts, (size_t)n_new + (size_t)n_new / 8, false));
    if (h->ubx_items.size() < (size_t)n_new) RET(dalloc(h, h->ubx_items, (size_t)n_new + (size_t)n_new / 8, false));
    RET(launch(h, "ubcache_offsets", [&] {
        k_ub_offsets<<<(int)((new_users + kUbTile) / kUbTile), 256, 0, h->stream>>>(h->ub_off, U, n, ub.tuser, ub.T, ub.dcum, new_users, h->ubx_off);
    }));
    if (n > 0) RET(launch(h, "ubcache_move_stored", [&] {
        const int grid = (int)((n + kUbTile - 1) / kUbTile);
        if (replace) k_ub_move_stored<true><<<grid, 256, 0, h->stream>>>(h->ub_ts, h->ub_items, n, ub.ob, ub.oe, ub.dcum, ub.T, ub.bb, ub.bcnt, ub.bts, h->ubx_ts, h->ubx_items);
        else k_ub_move_stored<false><<<grid, 256, 0, h->stream>>>(h->ub_ts, h->ub_items, n, ub.ob, ub.oe, ub.dcum, ub.T, ub.bb, ub.bcnt, ub.bts, h->ubx_ts, h->ubx_items);
    }));
    if (ub.T > 0) RET(launch(h, "ubcache_place_new", [&] {
        const int grid = grid_for_warps(h, ub.T);
        if (replace) k_ub_place_new<true><<<grid, 256, 0, h->stream>>>(h->ub_ts, ub.ob, ub.oe, ub.dcum, ub.T, ub.bb, ub.bcnt, ub.bts, ub.bit, h->ubx_ts, h->ubx_items);
        else k_ub_place_new<false><<<grid, 256, 0, h->stream>>>(h->ub_ts, ub.ob, ub.oe, ub.dcum, ub.T, ub.bb, ub.bcnt, ub.bts, ub.bit, h->ubx_ts, h->ubx_items);
    }));
    std::swap(h->ub_off, h->ubx_off); std::swap(h->ub_ts, h->ubx_ts); std::swap(h->ub_items, h->ubx_items);
    h->ub_users = new_users; h->ub_n = n_new;
    return CTR_OK;
}
}  // namespace

// ---- whole-table top-k recommendation (ctr_recommend_topk / ctr_mlp_recommend_topk; kernels in rec.cuh)
namespace {
// the exclusion mode is one of CTR_EXCLUDE_*, and CTR_EXCLUDE_SEEN comes with its cuts
bool exclude_ok(int32_t exclude, const int64_t* max_ts) {
    return exclude >= CTR_EXCLUDE_NONE && exclude <= CTR_EXCLUDE_SEEN && (exclude != CTR_EXCLUDE_SEEN || max_ts);
}

// CTR_EXCLUDE_SEEN: the seen bitmap of one pass (k_ub_seen) over this rank's N local rows of the I global rows (local
// row l = global row l·world + rank), for user row u, cut max_ts and the window uh [S] on the device, from this rank's
// behaviour cache; profile key `key`
int rec_build_seen(ctr_handle* h, const char* key, unsigned* seen, int64_t I, int64_t N, int world, int rank, int u, long long max_ts,
                   const int* uh) {
    const int S = h->cfg.S;
    const int64_t ne = h->ub_off ? h->ub_n : 0;                         // an upper bound on the user's events
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((ne + S + 255) / 256, (int64_t)h->num_sms * 4));
    CU(h, cudaMemsetAsync(seen, 0, (size_t)(N + 31) / 32 * sizeof(unsigned), h->stream));
    return launch(h, key, [&] {
        k_ub_seen<<<grid, 256, 0, h->stream>>>(h->ub_off, h->ub_ts, h->ub_items, h->ub_off ? (long)h->ub_users : 0L, u, max_ts, uh, S, (long)I,
                                               world, rank, seen);
    });
}

// The ranks' lists [n][k] in ls / lr on a row-sharded table: all-gathered into gs / gr [world][n][k] and merged back
// into ls / lr (and their lengths into count, when given) under profile key `name`.  The selection order is total, so
// the result is that of one whole-table scan.
template <class K>
int merge_rank_lists(ctr_handle* h, const char* name, typename K::T* ls, int* lr, typename K::T* gs, int* gr, int n, int k, size_t msmem,
                     int* count) {
    const long nk = (long)n * k;
    RET(comm_gather_lists(h, ls, gs, sizeof(typename K::T), lr, gr, (size_t)nk));
    return launch(h, name, [&] { knn::k_knn_merge<K><<<n, knn::kThreads, msmem, h->stream>>>(gs, gr, h->comm.world, k, k, nk, lr, ls, count); });
}

// The selection over logits of key type K, on h's stream.  Per user, chunk by chunk, k_rec_scan writes the slices'
// lists behind the running list in sl[0, k); chunk 0 merges its slices only, later chunks merge the running list with
// theirs, in place, and the last chunk writes the user's row of ls / lr.
template <class K>
struct RecTopk {
    using T = typename K::T;
    ctr_handle* h; const char* pre;         // profile keys <pre>_topk, <pre>_merge, <pre>_merge_ranks, <pre>_finish and <pre>_seen
    int k, nex, world, rank;                // nex exclusion rows per user; local row l is global row l·world + rank
    int64_t N; int Bc;                      // the items scored, per chunk
    bool by_seen = false;                   // CTR_EXCLUDE_SEEN (nex = 0): each user's seen bitmap over the local rows excludes
    int64_t I = N;                          // the global row count
    // selection slices of at least 4 steps and 8k rows: merging the slices' lists stays small against scanning them
    const int rps = round_up(std::max(4 * knn::kStep, 8 * k), knn::kStep);
    const size_t ssmem = rec::scan_smem_bytes<K>(k, nex), msmem = knn::smem_bytes<K>(1, 0, k);
    const std::string n_topk = std::string(pre) + "_topk", n_merge = std::string(pre) + "_merge", n_finish = std::string(pre) + "_finish",
                      n_seen = std::string(pre) + "_seen", n_ranks = std::string(pre) + "_merge_ranks";
    T *sl_s, *ls, *ol, *gs = nullptr; int *sl_r, *lr, *orow, *oc, *gr = nullptr; float* os; unsigned* seen = nullptr;

    // scratch slot `slot`: the caller's buffers (own(c)), then the running and slice lists, then [G][k] lists and
    // outputs, and on a row-sharded table the [world][G][k] gather of the ranks' lists
    template <class F>
    int setup(int slot, int64_t G, F&& own) {
        CU(h, cudaFuncSetAttribute(rec::k_rec_scan<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssmem));
        CU(h, cudaFuncSetAttribute(knn::k_knn_merge<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msmem));
        if (by_seen) {      // the (world, rank) form of the overloaded name
            void (*scan_seen)(const T*, int, int, int, int, int, const unsigned*, int, const T*, const int*, T*, int*) = rec::k_rec_scan_seen<K>;
            CU(h, cudaFuncSetAttribute(scan_seen, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssmem));
        }
        const size_t sl = (size_t)(1 + (Bc + rps - 1) / rps) * k, gk = (size_t)G * k;
        auto carve = [&](char* base) {
            Carve c{base};
            own(c);
            sl_s = c.take<T>(sl); sl_r = c.take<int>(sl);
            ls = c.take<T>(gk); lr = c.take<int>(gk); orow = c.take<int>(gk); ol = c.take<T>(gk); os = c.take<float>(gk); oc = c.take<int>(G);
            if (by_seen) seen = c.take<unsigned>((size_t)(N + 31) / 32);
            if (world > 1) { gs = c.take<T>((size_t)world * gk); gr = c.take<int>((size_t)world * gk); }
            return c.used;
        };
        char* ws = nullptr;
        RET(scratch_get(h, slot, carve(nullptr), (void**)&ws));
        carve(ws);
        return CTR_OK;
    }
    // user j of the group, excluding excl[0, nex), or under by_seen the seen set of (user row u, cut max_ts, window
    // excl [S]): score(i0, nb) queues the logits of items [i0, i0 + nb) into z
    template <class F>
    int user(int j, const int* excl, const T* z, F&& score, int u = -1, long long max_ts = 0) {
        const int nchunks = (int)((N + Bc - 1) / Bc);
        T* us = ls + (size_t)j * k; int* ur = lr + (size_t)j * k;
        if (by_seen) RET(rec_build_seen(h, n_seen.c_str(), seen, I, N, world, rank, u, max_ts, excl));
        for (int c = 0; c < nchunks; c++) {
            const int i0 = c * Bc, nb = (int)std::min<int64_t>(Bc, N - i0);
            RET(score(i0, nb));
            const int slices = (nb + rps - 1) / rps;
            const bool first = c == 0, last = c == nchunks - 1;
            RET(launch(h, n_topk.c_str(), [&] {
                if (by_seen)
                    rec::k_rec_scan_seen<K><<<slices, knn::kThreads, ssmem, h->stream>>>(z, nb, i0, world, rank, rps, seen, k, first ? nullptr : sl_s,
                                                                                        first ? nullptr : sl_r, sl_s + k, sl_r + k);
                else
                    rec::k_rec_scan<K><<<slices, knn::kThreads, ssmem, h->stream>>>(z, nb, i0, world, rank, rps, excl, nex, k,
                                                                                   first ? nullptr : sl_s, first ? nullptr : sl_r, sl_s + k, sl_r + k);
            }));
            const int ns = first ? slices : slices + 1;
            RET(launch(h, n_merge.c_str(), [&] {
                knn::k_knn_merge<K><<<1, knn::kThreads, msmem, h->stream>>>(first ? sl_s + k : sl_s, first ? sl_r + k : sl_r, ns, k, (long)ns * k, k,
                                                                          last ? ur : sl_r, last ? us : sl_s, nullptr);
            }));
        }
        if (nchunks == 0)            // an empty table or shard: an empty list
            RET(launch(h, n_merge.c_str(), [&] { knn::k_knn_merge<K><<<1, knn::kThreads, msmem, h->stream>>>(sl_s, sl_r, 0, k, 0, 0, ur, us, nullptr); }));
        return CTR_OK;
    }
    // the lists of users [g0, g0 + ng), on a row-sharded table every rank's merged, → the caller's outputs; after(n)
    // runs under the same launch as k_rec_finish
    template <class F>
    int finish(int64_t g0, int ng, int32_t* out_rows, float* out_scores, T* out_logits, int32_t* out_count, F&& after) {
        const long n = (long)ng * k;
        if (world > 1) RET(merge_rank_lists<K>(h, n_ranks.c_str(), ls, lr, gs, gr, ng, k, msmem, nullptr));
        RET(launch(h, n_finish.c_str(), [&] {
            rec::k_rec_finish<K><<<(int)((n + 255) / 256), 256, 0, h->stream>>>(ls, lr, k, n, orow, ol, os, oc);
            after(n);
        }));
        CU(h, cudaMemcpyAsync(out_rows + g0 * k, orow, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaMemcpyAsync(out_scores + g0 * k, os, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        if (out_logits) CU(h, cudaMemcpyAsync(out_logits + g0 * k, ol, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaMemcpyAsync(out_count + g0, oc, (size_t)ng * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));          // the caller's per-group buffers and the lists are reused by the next group
        return CTR_OK;
    }
};

// The counting pass of the held-out ranks over logits of key type K, on h's stream (kernels in rec.cuh).  A pass is
// m <= kMaxK targets of one (user, window): the chunks that hold a target are scored first and their targets' logits
// copied out, then every chunk is scored and counted against the sorted targets.  On a row-sharded ITEM_EMB
// (world > 1; collective) each rank scores its own shard: the targets' logits are all-gathered from their owners
// before the sort, and the ranks' bins are summed before the ranks are read off.  Under CTR_EXCLUDE_SEEN each rank's
// bitmap covers its own rows, and a target's seen flag comes from its owner in the same all-gather as its logit.
template <class K>
struct RecRank {
    using T = typename K::T;
    ctr_handle* h; const char* pre;         // profile keys <pre>_target, <pre>_count and <pre>_seen
    int nex;                                // exclusion rows per pass
    int64_t N; int Bc;                      // the items this rank scores (its local rows), per chunk
    int world = 1, rank = 0;                // local row l is global row l·world + rank
    int64_t I = N;                          // the global row count
    bool by_seen = false;                   // CTR_EXCLUDE_SEEN (nex = 0): each pass's seen bitmap over the local rows excludes
    const std::string n_target = std::string(pre) + "_target", n_count = std::string(pre) + "_count", n_seen = std::string(pre) + "_seen";
    int *rows, *place, *nvalid, *sr; T *tl, *tlg, *ss, *ol; unsigned long long* bins; long long* orank;
    unsigned* seen = nullptr; int *flag = nullptr, *flagg = nullptr;      // by_seen: the bitmap, the targets' flags [m], [world][m]

    // scratch slot `slot`: the caller's buffers (own(c)), then one pass's target state
    template <class F>
    int setup(int slot, F&& own) {
        CU(h, cudaFuncSetAttribute(rec::k_rec_rank<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, std::max(nex, 1) * 4));
        const size_t M = knn::kMaxK;
        auto carve = [&](char* base) {
            Carve c{base};
            own(c);
            rows = c.take<int>(M); place = c.take<int>(M); nvalid = c.take<int>(1); sr = c.take<int>(M);
            tl = c.take<T>(M); ss = c.take<T>(M); ol = c.take<T>(M); bins = c.take<unsigned long long>(M + 1); orank = c.take<long long>(M);
            tlg = world > 1 ? c.take<T>((size_t)world * M) : tl;      // [world][m] the ranks' target logits
            if (by_seen) {
                seen = c.take<unsigned>((size_t)(N + 31) / 32);
                flag = c.take<int>(M);
                flagg = world > 1 ? c.take<int>((size_t)world * M) : flag;
            }
            return c.used;
        };
        char* ws = nullptr;
        RET(scratch_get(h, slot, carve(nullptr), (void**)&ws));
        carve(ws);
        return CTR_OK;
    }
    // targets trow[0, m) of one (user, window), excluding excl[0, nex), or under by_seen the seen set of (user row u,
    // cut max_ts, window excl [S]) as each row's owner holds it: score(i0, nb) queues the logits of items [i0, i0 + nb)
    // into z.  Ranks and logits go to out_rank / out_logit[0, m) (host) in stream order.
    template <class F>
    int pass(const int* trow, int m, const int* excl, const T* z, F&& score, int64_t* out_rank, T* out_logit, int u = -1, long long max_ts = 0) {
        std::vector<int64_t> chunks;                         // the local chunks that hold a target this rank owns, each once
        for (int j = 0; j < m; j++)
            if (trow[j] >= 0 && trow[j] < I && trow[j] % world == rank) chunks.push_back(trow[j] / world / Bc);
        std::sort(chunks.begin(), chunks.end());
        chunks.erase(std::unique(chunks.begin(), chunks.end()), chunks.end());
        CU(h, cudaMemcpyAsync(rows, trow, (size_t)m * sizeof(int), cudaMemcpyHostToDevice, h->stream));
        // the bitmap comes first: the owner's flags of its targets are written beside their logits
        if (by_seen) RET(rec_build_seen(h, n_seen.c_str(), seen, I, N, world, rank, u, max_ts, excl));
        for (const int64_t c : chunks) {
            const int i0 = (int)(c * Bc), nb = (int)std::min<int64_t>(Bc, N - i0);
            RET(score(i0, nb));
            RET(launch(h, n_target.c_str(), [&] {
                rec::k_rec_target_logits<T><<<(m + 255) / 256, 256, 0, h->stream>>>(z, nb, i0, world, rank, rows, m, tl, seen, flag);
            }));
        }
        // every rank's slot, bits as they are (a float sum would turn a -0 logit into +0), and its seen flags in the
        // same group; a rank owning no target sends a slot nobody reads
        if (world > 1) RET(comm_gather_lists(h, tl, tlg, sizeof(T), flag, flagg, (size_t)m));
        RET(launch(h, n_target.c_str(), [&] {
            if (by_seen) rec::k_rec_rank_sort_seen<K><<<1, knn::kMaxK, 0, h->stream>>>(rows, tlg, m, world, m, (long)I, flagg, place, nvalid, ss, sr, bins);
            else rec::k_rec_rank_sort<K><<<1, knn::kMaxK, 0, h->stream>>>(rows, tlg, m, world, m, (long)I, excl, nex, place, nvalid, ss, sr, bins);
        }));
        for (int64_t i0 = 0; i0 < N; i0 += Bc) {
            const int nb = (int)std::min<int64_t>(Bc, N - i0);
            const int grid = (nb + rec::kRankRows - 1) / rec::kRankRows;
            RET(score((int)i0, nb));
            RET(launch(h, n_count.c_str(), [&] {
                if (by_seen) rec::k_rec_rank_seen<K><<<grid, rec::kRankThreads, 0, h->stream>>>(z, nb, (int)i0, world, rank, seen, ss, sr, nvalid, bins);
                else rec::k_rec_rank<K><<<grid, rec::kRankThreads, (size_t)nex * 4, h->stream>>>(z, nb, (int)i0, world, rank, excl, nex, ss, sr, nvalid, bins);
            }));
        }
        // the ranks' counts: queued after this rank's last read of the shard, so it completes only once every rank
        // has finished reading, and a step queued after the call cannot change a row still being read
        if (world > 1) RET(comm_sum_u64(h, bins, (size_t)m + 1));
        RET(launch(h, n_count.c_str(), [&] {
            rec::k_rec_rank_finish<T><<<1, knn::kMaxK, 0, h->stream>>>(rows, tlg, m, world, place, m, (long)I, bins, orank, ol);
        }));
        static_assert(sizeof(long long) == sizeof(int64_t), "int64 ranks");
        CU(h, cudaMemcpyAsync(out_rank, orank, (size_t)m * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaMemcpyAsync(out_logit, ol, (size_t)m * sizeof(T), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));             // the next pass reuses the target state
        return CTR_OK;
    }
};

// Keys grouped into passes: keys with equal key(i) share a pass, groups in order of first appearance, at most kMaxK
// keys per pass.  Returns the passes as lists of key indices.
template <class F>
std::vector<std::vector<int64_t>> rank_passes(int64_t n, F&& key) {
    std::map<decltype(key(0)), size_t> seen;
    std::vector<std::vector<int64_t>> groups;
    for (int64_t i = 0; i < n; i++) {
        auto it = seen.emplace(key(i), groups.size()).first;
        if (it->second == groups.size()) groups.emplace_back();
        groups[it->second].push_back(i);
    }
    std::vector<std::vector<int64_t>> passes;
    for (auto& g : groups)
        for (size_t a = 0; a < g.size(); a += knn::kMaxK)
            passes.emplace_back(g.begin() + a, g.begin() + std::min(g.size(), a + (size_t)knn::kMaxK));
    return passes;
}

// a compensated (Neumaier) float64 sum in input order: the same terms give the same bits (ctr_rank_metrics)
struct NeumaierSum {
    double s = 0.0, c = 0.0;
    void add(double x) {
        const double t = s + x;
        c += std::fabs(s) >= std::fabs(x) ? (s - t) + x : (x - t) + s;
        s = t;
    }
    double value() const { return s + c; }
};

// ctr_recommend_topk's and ctr_rank_items' scoring pass over the item table on a single-GPU or row-sharded (coll)
// ITEM_EMB, in MlpRecScore's shape: chunk() leaves the logits of a chunk of items in z().  With the user kernel
// (k_attn_fwd_user, ugrid CTAs) the user's history rows are staged in shared memory; else index buffers of the repeated
// user and history feed the ordinary attention kernels.
struct AttnRecScore {
    ctr_handle* h;
    bool coll;
    bool user_kernel = false;
    int ugrid = 0;

    // the refusals of the handle's state, before anything is written
    int check() {
        const int T = CTR_TABLE_ITEM_EMB;
        if (!h->tab[T]) return set_err(h, CTR_ESTATE, "ITEM_EMB table not uploaded");
        RET(coll ? comm_check(h) : check_tables(h));
        const int64_t N = h->tab_rows[T];
        if (N > INT32_MAX) return set_err(h, CTR_ESTATE, "ITEM_EMB has %lld rows: row ids are int32", (long long)N);
        int optin = 0;
        CU(h, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->dev));
        user_kernel = attn_user_ok(h, (size_t)optin);
        if (coll && !user_kernel)
            return set_err(h, CTR_ESTATE, "recommendation on a row-sharded ITEM_EMB needs the user's %d history rows in shared memory (%zu bytes > %d)",
                           h->cfg.S, attn_user_smem(h), optin);
        return CTR_OK;
    }
    void prepare() { ugrid = user_kernel ? h->num_sms * attn_user_prepare(h, coll) : 0; }
    const float* z() const { return h->Z; }
    // the logits of (local) items [i0, i0 + nb) for (user, history uh on the device) into z()
    int chunk(int user, const int* uh, int i0, int nb) {
        const int S = h->cfg.S;
        StepOpts o;
        RowSrc r;
        if (user_kernel) {
            r = coll ? comm_src(h, nullptr, nullptr, nullptr, nb, false) : idx_src(h, nullptr, nullptr, nullptr, nb);
            RET(attn_forward_user(h, r, user, uh, i0, nb, ugrid));
            o.x0_ready = true;
        } else {
            const int fg = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)nb * std::max(S, 1) + 255) / 256, (int64_t)h->num_sms * 8));
            RET(launch(h, "rec_fill_idx", [&] { rec::k_rec_fill_idx<<<fg, 256, 0, h->stream>>>(user, uh, S, i0, nb, h->s_user, h->s_item, h->s_hist); }));
            r = idx_src(h, h->s_user, h->s_item, h->s_hist, nb);
        }
        return step_core(h, r, nb, o);
    }
};

}  // namespace

// =====================================================================================================
extern "C" {

int ctr_abi_version(void) { return CTR_B200_ABI_VERSION; }

void ctr_config_default(ctr_config* c, int model) {
    memset(c, 0, sizeof *c);
    c->model = model;
    c->uP = 52; c->S = 10; c->D = 16; c->cF = 53;          // example/movielens: feature.go:87-196, rcmd.go:22-24
    c->H0 = 200; c->H1 = 80;                                // din.go:17-18
    c->batch = 200; c->pred_batch = 100;                    // model_test.go:22, dinimpl_test.go
    c->lr = 0.01f; c->l2 = 1e-4f; c->beta1 = 0.9f; c->beta2 = 0.999f; c->eps = 1e-8f;   // model.go:88
    c->dropout0 = c->dropout1 = (model == CTR_MODEL_YOUTUBE) ? 0.003f : 0.005f;           // dnn.go:136-137, din.go:204-205
    c->seed = 0; c->table_opt = CTR_TABLE_FROZEN; c->table_lr = 0.0f; c->gemm = CTR_GEMM_AUTO;
    c->device = 0; c->rank = 0; c->world = 1;
}

const char* ctr_last_error(const ctr_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int ctr_create(const ctr_config* cfg, ctr_handle** out) {
    if (!cfg || !out) return set_err(nullptr, CTR_EINVAL, "null argument");
    *out = nullptr;
    const ctr_config& c = *cfg;
    if (c.model < 0 || c.model > 2) return set_err(nullptr, CTR_EINVAL, "unknown model %d", c.model);
    if (c.table_opt < CTR_TABLE_FROZEN || c.table_opt > CTR_TABLE_ADAM) return set_err(nullptr, CTR_EINVAL, "unknown table optimiser %d", c.table_opt);
    if (c.uP < 0 || c.cF < 0 || c.S < 1 || c.D < 1 || c.H0 < 1 || c.H1 < 1 || c.batch < 1 || c.pred_batch < 1)
        return set_err(nullptr, CTR_EINVAL, "bad dims");
    if (c.D > 32 * kGenAcc) return set_err(nullptr, CTR_EINVAL, "D=%d > %d unsupported", c.D, 32 * kGenAcc);
    if (c.H1 > 128) return set_err(nullptr, CTR_EINVAL, "H1=%d > 128 unsupported", c.H1);
    if (c.world < 1 || c.rank < 0 || c.rank >= c.world) return set_err(nullptr, CTR_EINVAL, "bad rank/world");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return set_err(nullptr, CTR_ENODEV, "no CUDA device: this engine has no CPU fallback"); }
    if (c.device < 0 || c.device >= ndev) return set_err(nullptr, CTR_ENODEV, "device %d of %d", c.device, ndev);
    cudaDeviceProp prop{};
    cudaGetDeviceProperties(&prop, c.device);
    if (prop.major != 9) return set_err(nullptr, CTR_ENODEV, "device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);

    ctr_handle* h = new ctr_handle();
    h->cfg = c; h->dev = c.device; h->num_sms = prop.multiProcessorCount;
    h->comm.rank = c.rank; h->comm.world = c.world;
#define CUC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_err(nullptr, CTR_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); ctr_destroy(h); return CTR_ECUDA; } } while (0)
#define RC(x) do { int r_ = (x); if (r_ != CTR_OK) { g_create_error = h->err; ctr_destroy(h); return r_; } } while (0)
    CUC(cudaSetDevice(h->dev));
    CUC(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true;
    CUC(h->ev0.create(cudaEventDefault)); CUC(h->ev1.create(cudaEventDefault));
    h->in = c.uP + 2 * c.D + c.cF;                      // din.go:187
    h->Kp = round_up(h->in, 32); h->H0p = round_up(c.H0, 32); h->H1p = round_up(c.H1, 32); h->Sp = round_up(c.S, 4);
    h->lddx = round_up(2 * c.D, 4);
    h->Bmax = std::max(c.batch, c.pred_batch);
    h->wsize[0] = (size_t)h->Kp * h->H0p; h->wsize[1] = (size_t)h->H0p * h->H1p; h->wsize[2] = h->H1p; h->wsize[3] = h->Sp;
    h->Gflat_n = h->wsize[0] + h->wsize[1] + h->wsize[2] + h->wsize[3];
    RC(dalloc(h, h->Gflat, h->Gflat_n));
    for (size_t i = 0, off = 0; i < 4; off += h->wsize[i], i++) h->G[i] = h->Gflat + off;
    for (int i = 0; i < 4; i++) { RC(dalloc(h, h->W[i], h->wsize[i])); RC(dalloc(h, h->Mo[i], h->wsize[i])); RC(dalloc(h, h->Vo[i], h->wsize[i])); }
    const size_t B = h->Bmax;
    RC(dalloc(h, h->X0, B * h->Kp)); RC(dalloc(h, h->H0d, B * h->H0p)); RC(dalloc(h, h->H1d, B * h->H1p));
    RC(dalloc(h, h->P, B)); RC(dalloc(h, h->Z, B));
    RC(dalloc(h, h->dZ1, B * h->H1p)); RC(dalloc(h, h->dZ0, B * h->H0p)); RC(dalloc(h, h->dX, B * h->lddx));
    RC(dalloc(h, h->d_cost, 1));
    RC(dalloc(h, h->s_user, B)); RC(dalloc(h, h->s_item, B)); RC(dalloc(h, h->s_hist, B * c.S)); RC(dalloc(h, h->s_label, B));
    RC(ctr_init_weights(h, c.seed));
    CUC(cudaStreamSynchronize(h->stream));
#undef CUC
#undef RC
    *out = h;
    return CTR_OK;
}

// the device buffers, events and library-created streams are members: they free themselves at `delete h`, with this
// handle's device current
void ctr_destroy(ctr_handle* h) {
    if (!h) return;
    cudaSetDevice(h->dev);
    if (h->stream) cudaStreamSynchronize(h->stream);
    comm_destroy(h);
    for (int i = 0; i < 3; i++) table_free(h, i);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

int ctr_set_weights(ctr_handle* h, const float* mlp0, const float* mlp1, const float* mlp2, const float* att0) {
    if (!h || !mlp0 || !mlp1 || !mlp2) return set_err(h, CTR_EINVAL, "null weights");
    std::lock_guard<std::mutex> lk(h->mu);
    const ctr_config& c = h->cfg;
    CU(h, cudaSetDevice(h->dev));
    for (int i = 0; i < 4; i++) {
        CU(h, cudaMemsetAsync(h->W[i], 0, h->wsize[i] * sizeof(float), h->stream));
        CU(h, cudaMemsetAsync(h->G[i], 0, h->wsize[i] * sizeof(float), h->stream));
        CU(h, cudaMemsetAsync(h->Mo[i], 0, h->wsize[i] * sizeof(float), h->stream));
        CU(h, cudaMemsetAsync(h->Vo[i], 0, h->wsize[i] * sizeof(float), h->stream));
    }
    CU(h, cudaMemcpy2DAsync(h->W[0], h->H0p * sizeof(float), mlp0, c.H0 * sizeof(float), c.H0 * sizeof(float), h->in, cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpy2DAsync(h->W[1], h->H1p * sizeof(float), mlp1, c.H1 * sizeof(float), c.H1 * sizeof(float), c.H0, cudaMemcpyHostToDevice, h->stream));
    CU(h, cudaMemcpyAsync(h->W[2], mlp2, c.H1 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    if (att0) CU(h, cudaMemcpyAsync(h->W[3], att0, c.S * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    else { std::vector<float> ones(c.S, 1.0f); CU(h, cudaMemcpyAsync(h->W[3], ones.data(), c.S * sizeof(float), cudaMemcpyHostToDevice, h->stream)); CU(h, cudaStreamSynchronize(h->stream)); }
    CU(h, cudaStreamSynchronize(h->stream));
    h->step = 0;
    h->um.dirty = true;
    return CTR_OK;
}

int ctr_init_weights(ctr_handle* h, uint32_t seed) {
    if (!h) return CTR_EINVAL;
    const ctr_config& c = h->cfg;
    std::vector<float> w0((size_t)h->in * c.H0), w1((size_t)c.H0 * c.H1), w2(c.H1), a(c.S, 1.0f);   // att0 = 1: din.go:181
    gaussian_fill(w0, seed, 0); gaussian_fill(w1, seed, 1); gaussian_fill(w2, seed, 2);
    return ctr_set_weights(h, w0.data(), w1.data(), w2.data(), a.data());
}

int ctr_get_weights(ctr_handle* h, float* mlp0, float* mlp1, float* mlp2, float* att0) {
    if (!h) return CTR_EINVAL;
    std::lock_guard<std::mutex> lk(h->mu);
    const ctr_config& c = h->cfg;
    CU(h, cudaSetDevice(h->dev));
    if (mlp0) CU(h, cudaMemcpy2DAsync(mlp0, c.H0 * sizeof(float), h->W[0], h->H0p * sizeof(float), c.H0 * sizeof(float), h->in, cudaMemcpyDeviceToHost, h->stream));
    if (mlp1) CU(h, cudaMemcpy2DAsync(mlp1, c.H1 * sizeof(float), h->W[1], h->H1p * sizeof(float), c.H1 * sizeof(float), c.H0, cudaMemcpyDeviceToHost, h->stream));
    if (mlp2) CU(h, cudaMemcpyAsync(mlp2, h->W[2], c.H1 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (att0) CU(h, cudaMemcpyAsync(att0, h->W[3], c.S * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

int ctr_table_upload(ctr_handle* h, int which, const float* rows, int64_t nrows, int32_t width) {
    if (!h || !rows || which < 0 || which > 2 || nrows < 1 || width < 1) return set_err(h, CTR_EINVAL, "bad table upload arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    const ctr_config& c = h->cfg;
    const int want = which == CTR_TABLE_USER_FEAT ? c.uP : which == CTR_TABLE_ITEM_FEAT ? c.cF : c.D;
    if (width != want) return set_err(h, CTR_EINVAL, "table %d width %d != model dim %d", which, width, want);
    CU(h, cudaSetDevice(h->dev));
    RET(table_alloc(h, which, nrows, width));
    const long ld = h->tab_ld[which]; const int64_t local = h->tab_local_rows[which];
    if (!h->tab_sharded[which]) {
        CU(h, cudaMemcpy2DAsync(h->tab[which], ld * sizeof(float), rows, (size_t)width * sizeof(float), (size_t)width * sizeof(float), (size_t)nrows, cudaMemcpyHostToDevice, h->stream));
    } else if (local > 0) {   // owner(row) = row % world; local row = row / world
        CU(h, cudaMemcpy2DAsync(h->tab[which], ld * sizeof(float), rows + (size_t)h->comm.rank * width, (size_t)width * h->comm.world * sizeof(float),
                                (size_t)width * sizeof(float), (size_t)local, cudaMemcpyHostToDevice, h->stream));
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

int ctr_table_fill(ctr_handle* h, int which, int64_t nrows, int32_t width, uint32_t seed, int32_t dist, float scale) {
    if (!h || which < 0 || which > 2 || nrows < 1 || width < 1) return set_err(h, CTR_EINVAL, "bad table fill arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    const ctr_config& c = h->cfg;
    const int want = which == CTR_TABLE_USER_FEAT ? c.uP : which == CTR_TABLE_ITEM_FEAT ? c.cF : c.D;
    if (width != want) return set_err(h, CTR_EINVAL, "table %d width %d != model dim %d", which, width, want);
    CU(h, cudaSetDevice(h->dev));
    RET(table_alloc(h, which, nrows, width));
    const bool shard = h->tab_sharded[which];
    RET(launch(h, "table_fill", [&] {
        k_table_fill<<<h->num_sms * 8, 256, 0, h->stream>>>(h->tab[which], h->tab_ld[which], (long)h->tab_local_rows[which], width, shard ? h->comm.world : 1,
                                                           shard ? h->comm.rank : 0, seed, (uint32_t)which, dist, scale);
    }));
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

int ctr_table_download(ctr_handle* h, int which, float* rows, int64_t nrows, int32_t width) {
    if (!h || !rows || which < 0 || which > 2) return set_err(h, CTR_EINVAL, "bad table download arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->tab[which] || nrows != h->tab_rows[which] || width != h->tab_width[which]) return set_err(h, CTR_EINVAL, "table %d shape mismatch", which);
    CU(h, cudaSetDevice(h->dev));
    const bool shard = h->tab_sharded[which];
    if (shard && which == CTR_TABLE_ITEM_EMB) RET(comm_hot_writeback(h));
    if (!shard) {
        CU(h, cudaMemcpy2DAsync(rows, (size_t)width * sizeof(float), h->tab[which], h->tab_ld[which] * sizeof(float), (size_t)width * sizeof(float), (size_t)nrows, cudaMemcpyDeviceToHost, h->stream));
    } else if (h->tab_local_rows[which] > 0) {   // fills only this rank's rows (row % world == rank)
        CU(h, cudaMemcpy2DAsync(rows + (size_t)h->comm.rank * width, (size_t)width * h->comm.world * sizeof(float), h->tab[which], h->tab_ld[which] * sizeof(float),
                                (size_t)width * sizeof(float), (size_t)h->tab_local_rows[which], cudaMemcpyDeviceToHost, h->stream));
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

int ctr_gather_rows(ctr_handle* h, const int32_t* user_row, const int32_t* item_row, const int32_t* hist, int64_t B, float* X) {
    if (!h || !user_row || !item_row || !hist || !X || B < 1) return set_err(h, CTR_EINVAL, "bad gather arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    RET(check_tables(h));
    CU(h, cudaSetDevice(h->dev));
    const ctr_config& c = h->cfg;
    const long xc = (long)c.uP + (long)c.S * c.D + c.D + c.cF;
    float* dout = nullptr;
    const int chunk = h->Bmax;
    RET(scratch_get(h, 0, (size_t)chunk * xc * sizeof(float), (void**)&dout));
    int rc = CTR_OK;
    for (int64_t s = 0; s < B && rc == CTR_OK; s += chunk) {
        int nb = (int)std::min<int64_t>(chunk, B - s);
        rc = stage_idx(h, user_row + s, item_row + s, hist + s * c.S, nullptr, nb);
        if (rc != CTR_OK) break;
        RowSrc r = idx_src(h, h->s_user, h->s_item, h->s_hist, nb);
        rc = launch(h, "gather_rows", [&] { k_gather_rows<<<grid_for_warps(h, nb), 256, 0, h->stream>>>(r, dims_of(h), dout, xc, nb, RowsAsIs{}); });
        if (rc != CTR_OK) break;
        if (cudaMemcpyAsync(X + s * xc, dout, (size_t)nb * xc * sizeof(float), cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
            cudaStreamSynchronize(h->stream) != cudaSuccess) rc = set_err(h, CTR_ECUDA, "gather D2H: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return rc;
}

int ctr_train_dense(ctr_handle* h, const float* X, const float* Y, int64_t n, int32_t xcols, const int32_t ranges[8],
                    int32_t epochs, int32_t early_stop, float* last_cost, int32_t* epochs_run) {
    if (!h || !X || !Y || !ranges || n < 1 || xcols < 1 || epochs < 0) return set_err(h, CTR_EINVAL, "bad train arguments");
    // the dense-X compatibility route has no gradient exchange: refusing beats training world replicas that silently diverge
    if (h->comm.world > 1) return set_err(h, CTR_ESTATE, "ctr_train_dense is single-GPU; with world=%d train through the index entry points", h->comm.world);
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    RowSrc base{};
    RET(dense_src(h, ranges, xcols, &base));
    RET(upload_dense(h, X, Y, n, xcols));
    const int B = h->cfg.batch;
    const int64_t batches = n / B + (n % B != 0);           // model.go:96-99
    float best = INFINITY, cost = 0.0f; int no_improve = 0, ep = 0;
    for (ep = 0; ep < epochs; ep++) {
        for (int64_t b = 0; b < batches; b++) {
            const int64_t start = b * B; int64_t end = start + B;
            if (start >= n) break;
            if (end > n) end = n;
            RowSrc r = base; r.X = h->dXd + start * xcols; r.nvalid = (int)(end - start);   // tail rows → zeros, label 0 (model.go:357-371)
            StepOpts o; o.training = true; o.update = true; o.d_label = h->dYd + start;
            RET(step_core(h, r, B, o));
        }
        RET(read_cost(h, B, &cost));                        // cost of the epoch's last batch, model.go:198
        if (cost < best) { best = cost; no_improve = 0; } else no_improve++;
        if (early_stop != 0 && no_improve >= early_stop) { ep++; break; }   // model.go:206-209
    }
    if (last_cost) *last_cost = cost;
    if (epochs_run) *epochs_run = ep;
    return CTR_OK;
}

int ctr_predict_dense(ctr_handle* h, const float* X, int64_t n, int32_t xcols, const int32_t ranges[8], float* out) {
    if (!h || !X || !ranges || !out || n < 1 || xcols < 1) return set_err(h, CTR_EINVAL, "bad predict arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    RowSrc base{};
    RET(dense_src(h, ranges, xcols, &base));
    RET(upload_dense(h, X, nullptr, n, xcols));
    const int B = h->cfg.pred_batch;
    const int64_t batches = n / B + (n % B != 0);
    for (int64_t b = 0; b < batches; b++) {
        const int64_t start = b * B; int64_t end = start + B;
        if (start >= n) break;
        if (end > n) end = n;
        RowSrc r = base; r.X = h->dXd + start * xcols; r.nvalid = (int)(end - start);
        StepOpts o;                                          // dropout off: din.go:133-145
        RET(step_core(h, r, B, o));
        CU(h, cudaMemcpyAsync(out + start, h->P, (size_t)(end - start) * sizeof(float), cudaMemcpyDeviceToHost, h->stream));   // model.go:344-347
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

namespace {
// options of one local-gather train step; with world > 1 (replicated ITEM_EMB) the row gradients go through
// comm.table_grad and everything is all-reduced before the update
int train_opts(ctr_handle* h, const float* d_label, int B, StepOpts* out) {
    StepOpts o; o.training = true; o.update = true; o.d_label = d_label;
    if (h->comm.world > 1) {
        Comm& cm = h->comm;
        const size_t n = (size_t)h->tab_rows[CTR_TABLE_ITEM_EMB] * h->tab_ld[CTR_TABLE_ITEM_EMB];
        if (cm.table_grad.size() != n) RET(dalloc(h, cm.table_grad, n));        // reallocated on any size change
        o.table_grad = cm.table_grad; o.table_grad_n = n; o.grad_scale = 1.0f / (float)cm.world; o.adam_batch = B * cm.world;
    }
    *out = o;
    return CTR_OK;
}

bool emb_sharded(const ctr_handle* h) { return h->comm.world > 1 && h->tab_sharded[CTR_TABLE_ITEM_EMB]; }

// one train step on device-resident ids; rows >= nvalid are the zero-padded tail trained as label 0 (model.go:357-371)
int train_step_dev(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, const float* d_label, int B, int nvalid) {
    if (emb_sharded(h)) return comm_train_step(h, d_user, d_item, d_hist, d_label, B, nvalid);
    RET(check_tables(h));
    RowSrc r = idx_src(h, d_user, d_item, d_hist, B);
    r.nvalid = nvalid;
    StepOpts o;
    RET(train_opts(h, d_label, B, &o));
    return step_core(h, r, B, o);
}
}  // namespace

int ctr_train_step_idx_dev(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, const float* d_label, int32_t B) {
    if (!h || !d_user || !d_item || !d_hist || !d_label) return set_err(h, CTR_EINVAL, "null argument");
    if (B != h->cfg.batch) return set_err(h, CTR_EINVAL, "B=%d != configured batch %d", B, h->cfg.batch);
    return train_step_dev(h, d_user, d_item, d_hist, d_label, B, B);
}

int ctr_train_step_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row, const int32_t* hist, const float* label, int32_t B, ctr_step_stats* stats) {
    if (!h || !user_row || !item_row || !hist || !label) return set_err(h, CTR_EINVAL, "null argument");
    if (B != h->cfg.batch) return set_err(h, CTR_EINVAL, "B=%d != configured batch %d", B, h->cfg.batch);
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    const int64_t l0 = h->launches;
    RET(stage_idx(h, user_row, item_row, hist, label, B));
    RET(ctr_train_step_idx_dev(h, h->s_user, h->s_item, h->s_hist, h->s_label, B));
    float cost = 0;
    RET(read_cost(h, B * h->comm.world, &cost));      // d_cost was summed over the ranks
    if (stats) { stats->cost = cost; stats->ms_device = 0; stats->launches = (int32_t)(h->launches - l0); stats->reserved = 0; }
    return CTR_OK;
}

namespace {
// lazily creates the pinned ring, the two device slots and the copy stream; slot size fits one idx batch.  Built
// into locals and moved into the handle once all of it exists.
int feed_init(ctr_handle* h) {
    if (h->copy_stream) return CTR_OK;
    const size_t B = (size_t)h->Bmax;
    size_t bytes = (B * (size_t)(h->cfg.S + 3) * 4 + 255) & ~(size_t)255;      // [user | item | hist | label] — also fits [uid | iid | ts | label] chunks
    bytes = std::max(bytes, (size_t)B * 28 + 256);
    Stream copy; Event copied[2], consumed[2], pin_free[ctr_handle::kPin];
    DevBuf<unsigned char> dev[2]; PinnedBuf<unsigned char> pin[ctr_handle::kPin];
    CU(h, copy.create());
    for (int i = 0; i < 2; i++) {
        CU(h, copied[i].create(cudaEventDisableTiming)); CU(h, consumed[i].create(cudaEventDisableTiming));
        CU(h, dev[i].alloc(bytes));
    }
    for (int i = 0; i < ctr_handle::kPin; i++) {
        CU(h, pin[i].alloc(bytes));
        CU(h, pin_free[i].create(cudaEventDisableTiming));
    }
    for (int i = 0; i < 2; i++) { h->ev_copied[i] = std::move(copied[i]); h->ev_consumed[i] = std::move(consumed[i]); h->feed_dev[i] = std::move(dev[i]); }
    for (int i = 0; i < ctr_handle::kPin; i++) { h->feed_pin[i] = std::move(pin[i]); h->pin_free[i] = std::move(pin_free[i]); }
    h->feed_bytes = bytes;
    h->pool = std::make_unique<CopyPool>(7);          // 7 workers + the caller: 8 memcpy streams, so a 14 MB batch is staged in parallel with the step
    h->copy_stream = std::move(copy);
    return CTR_OK;
}

// GetSample's assembly over sample keys (ctr_train_keys, ctr_mlp_fit_keys): the resident survivor arrays kt_* for cap
// samples, the flag / scan buffers of `chunk` keys and the survivor count, zeroed.  feed_init must have run.
int keys_prepare(ctr_handle* h, size_t cap, size_t chunk) {
    RET(reserve(h, h->kt_user, cap)); RET(reserve(h, h->kt_item, cap)); RET(reserve(h, h->kt_ts, cap)); RET(reserve(h, h->kt_label, cap));
    if (!h->kt_scan_tmp || h->kt_flag.size() < chunk + 1) {     // kt_scan_tmp is allocated last: it exists only with the other two
        h->kt_scan_tmp.reset();
        RET(dalloc(h, h->kt_flag, chunk + 1)); RET(dalloc(h, h->kt_pos, chunk + 1));
        size_t bytes = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, bytes, h->kt_flag.get(), h->kt_pos.get(), (int)(chunk + 1), h->stream);
        RET(dalloc(h, h->kt_scan_tmp, bytes, false));
    }
    if (!h->kt_count) RET(dalloc(h, h->kt_count, 1));
    CU(h, cudaMemsetAsync(h->kt_count, 0, sizeof(unsigned long long), h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

// keys [c·chunk, c·chunk + chunk) of n → (user row, item row, ts, label) appended to kt_* after the survivors of the
// earlier chunks; unresolvable samples dropped, order kept.  Caller memory → pinned ring (host threads) → device slot
// c & 1 → k_keys_rows, scan, k_keys_compact, count advance, all on stream rs.
int keys_resolve_chunk(ctr_handle* h, int64_t c, size_t chunk, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts,
                       const float* label, int64_t n, cudaStream_t rs) {
    const int slot = (int)(c & 1), ps = (int)(c % ctr_handle::kPin);
    const int64_t start = c * (int64_t)chunk; const size_t m = (size_t)std::min<int64_t>((int64_t)chunk, n - start);
    if (c >= ctr_handle::kPin) CU(h, cudaEventSynchronize(h->pin_free[ps]));
    unsigned char* pin = h->feed_pin[ps];
    h->pool->copy(pin, user_ids + start, m * 8); h->pool->copy(pin + m * 8, item_ids + start, m * 8);
    h->pool->copy(pin + m * 16, ts + start, m * 8); h->pool->copy(pin + m * 24, label + start, m * 4);
    CU(h, cudaMemcpyAsync(h->feed_dev[slot], pin, m * 28, cudaMemcpyHostToDevice, rs));     // after resolve(c-2), which read this slot (stream order)
    CU(h, cudaEventRecord(h->pin_free[ps], rs));
    const long long* dk = (const long long*)h->feed_dev[slot].get();
    const int grid = (int)std::max<size_t>(1, std::min<size_t>((m + 255) / 256, (size_t)h->num_sms * 8));
    RET(launch(h, "keys_rows", [&] {
        k_keys_rows<<<grid, 256, 0, rs>>>(h->idm_keys[0], h->idm_vals[0], h->idm_keys[0].size() - 1, h->idm_keys[1], h->idm_vals[1], h->idm_keys[1].size() - 1,
                                         dk, dk + m, (long)m, h->kt_flag);
    }));
    RET(launch(h, "cub_exclusive_scan", [&] { size_t tb = h->kt_scan_tmp.size(); cub::DeviceScan::ExclusiveSum(h->kt_scan_tmp, tb, h->kt_flag.get(), h->kt_pos.get(), (int)(m + 1), rs); }));
    RET(launch(h, "keys_compact", [&] {
        k_keys_compact<<<grid, 256, 0, rs>>>(h->idm_keys[0], h->idm_vals[0], h->idm_keys[0].size() - 1, h->idm_keys[1], h->idm_vals[1], h->idm_keys[1].size() - 1,
                                            dk, dk + m, dk + 2 * m, (const float*)(dk + 3 * m), (long)m, h->kt_flag, h->kt_pos, h->kt_count,
                                            h->kt_user, h->kt_item, h->kt_ts, h->kt_label);
    }));
    return launch(h, "keys_advance", [&] { k_keys_advance<<<1, 1, 0, rs>>>(h->kt_pos + m, h->kt_count); });
}

// GetUserBehavior(user row d_user[i], S, -1, d_ts[i]) into out[i·S, i·S + S) for i < n, on stream st, under profile key
// ubcache_window; no ubcache (no UserBehavior provider) → every history empty (rcmd.go:498,509)
int ub_windows(ctr_handle* h, cudaStream_t st, const int* d_user, const long long* d_ts, int n, int* out) {
    const int S = h->cfg.S;
    if (!h->ub_off) {
        CU(h, cudaMemsetAsync(out, 0xff, sizeof(int) * (size_t)n * S, st));
        return CTR_OK;
    }
    return launch(h, "ubcache_window", [&] {
        k_ub_window<<<grid_for_warps(h, n), 256, 0, st>>>(h->ub_off, h->ub_ts, h->ub_items, d_user, d_ts, n, S, (long)h->ub_users, out);
    });
}
}  // namespace

int ctr_train_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row, const int32_t* hist, const float* label,
                  int64_t n, float* costs) {
    if (!h || !user_row || !item_row || !hist || !label || n < 1) return set_err(h, CTR_EINVAL, "bad train arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    if (!emb_sharded(h)) RET(check_tables(h));
    const int B = h->cfg.batch, S = h->cfg.S;
    const int64_t nb = (n + B - 1) / B;                      // model.go:96-99
    RET(feed_init(h));
    RET(reserve(h, h->d_costs, (size_t)nb));
    const size_t o_item = (size_t)B * 4, o_hist = (size_t)B * 8, o_label = (size_t)B * (S + 2) * 4;
    CU(h, cudaStreamSynchronize(h->stream));                 // a device slot may still be in use by an earlier call
    for (int64_t b = 0; b < nb; b++) {
        const int slot = (int)(b & 1), ps = (int)(b % ctr_handle::kPin);
        const int64_t start = b * B; const size_t nv = (size_t)std::min<int64_t>(B, n - start);
        // caller memory → pinned slot (host threads; overlaps the GPU work already queued), then one DMA
        if (b >= ctr_handle::kPin) CU(h, cudaEventSynchronize(h->pin_free[ps]));
        unsigned char* pin = h->feed_pin[ps];
        memcpy(pin, user_row + start, nv * 4); memcpy(pin + o_item, item_row + start, nv * 4); memcpy(pin + o_label, label + start, nv * 4);
        h->pool->copy(pin + o_hist, hist + start * S, nv * S * 4);
        // H2D of batch b on the copy stream, after the compute that last used this device slot (batch b-2)
        if (b >= 2) CU(h, cudaStreamWaitEvent(h->copy_stream, h->ev_consumed[slot], 0));
        CU(h, cudaMemcpyAsync(h->feed_dev[slot], pin, o_label + (size_t)B * 4, cudaMemcpyHostToDevice, h->copy_stream));
        CU(h, cudaEventRecord(h->pin_free[ps], h->copy_stream));
        CU(h, cudaEventRecord(h->ev_copied[slot], h->copy_stream));
        // compute of batch b on the engine stream (overlaps the staging + H2D of batch b+1)
        CU(h, cudaStreamWaitEvent(h->stream, h->ev_copied[slot], 0));
        unsigned char* d = h->feed_dev[slot];
        RET(train_step_dev(h, (const int*)d, (const int*)(d + o_item), (const int*)(d + o_hist), (const float*)(d + o_label), B, (int)nv));   // ragged tail → zero rows with label 0 (model.go:357-371)
        CU(h, cudaMemcpyAsync(h->d_costs + b, h->d_cost, sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
        CU(h, cudaEventRecord(h->ev_consumed[slot], h->stream));
    }
    std::vector<double> hc((size_t)nb);
    CU(h, cudaMemcpyAsync(hc.data(), h->d_costs, sizeof(double) * (size_t)nb, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    CU(h, cudaStreamSynchronize(h->copy_stream));
    if (h->comm.h_err && *h->comm.h_err) return set_err(h, CTR_ECOMM, "peer barrier timed out waiting for rank %d", *h->comm.h_err - 1);
    if (costs) for (int64_t b = 0; b < nb; b++) costs[b] = -(float)(hc[(size_t)b] / ((double)B * h->comm.world));   // d_cost is summed over the ranks
    return CTR_OK;
}

// recommend.Train (rcmd.go:197-246) fed by sample keys: GetSample's assembly (rcmd.go:339-460) happens on the device —
// id maps resolve {UserId, ItemId}, samples whose user or item has no features are DROPPED as the reference's
// assembler skips them (rcmd.go:378-382), the survivors stay resident in HBM in input order, and every batch's
// history rows come from the device ubcache at the sample's timestamp (GetUserBehavior(uid, S, -1, ts),
// rcmd.go:509; prepare.go:13-38) right before its step — then model.Train's epoch loop (model.go:96-209).
int ctr_train_keys(ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label, int64_t n,
                   int32_t epochs, int32_t early_stop, float* last_cost, int32_t* epochs_run, int64_t* rows_used) {
    if (!h || !user_ids || !item_ids || !ts || !label || n < 1 || epochs < 0) return set_err(h, CTR_EINVAL, "bad train arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    if (!h->idm_keys[0] || !h->idm_keys[1]) return set_err(h, CTR_ESTATE, "ctr_train_keys needs both id maps (ctr_idmap_build)");
    if (!emb_sharded(h)) RET(check_tables(h));
    const int B = h->cfg.batch, S = h->cfg.S;
    RET(feed_init(h));
    // One GPU: the first epoch STREAMS — small chunks, and the steps over the samples already resident are queued while
    // the host stages the next chunk (the survivor count of chunk c-1 comes back through a pinned ring).  Several ranks:
    // every step is collective, so the ranks first agree on the batch count (resolve everything, then train).
    const bool streaming = epochs > 0 && h->comm.world == 1;
    const size_t chunk = std::min<size_t>((size_t)n, streaming ? std::min<size_t>(h->feed_bytes / 28, (size_t)2 * B) : h->feed_bytes / 28);   // keys per staging slot
    // ---- resident sample arrays (+B slack so a padded tail never indexes past the end)
    RET(keys_prepare(h, (size_t)n + (size_t)B, chunk));
    if (!h->kt_count_host) {            // the count ring and its events, moved into the handle together
        PinnedBuf<unsigned long long> ring; Event counted[ctr_handle::kCnt];
        CU(h, ring.alloc(ctr_handle::kCnt));
        for (int i = 0; i < ctr_handle::kCnt; i++) CU(h, counted[i].create(cudaEventDisableTiming));
        for (int i = 0; i < ctr_handle::kCnt; i++) h->kt_counted[i] = std::move(counted[i]);
        h->kt_count_host = std::move(ring);
    }
    if (!h->win_stream) {               // the window stream, its two buffers and their events, moved in together
        Stream ws; DevBuf<int> hist[2]; Event win[2], used[2], queued;
        CU(h, ws.create());
        for (int i = 0; i < 2; i++) {
            RET(dalloc(h, hist[i], (size_t)h->Bmax * S, false));
            CU(h, win[i].create(cudaEventDisableTiming)); CU(h, used[i].create(cudaEventDisableTiming));
        }
        CU(h, queued.create(cudaEventDisableTiming));
        for (int i = 0; i < 2; i++) { h->kt_hist[i] = std::move(hist[i]); h->kt_win[i] = std::move(win[i]); h->kt_used[i] = std::move(used[i]); }
        h->kt_queued = std::move(queued);
        h->win_stream = std::move(ws);
    }
    // The windows read the ubcache CSR, which an ubcache append / set rewrites on the engine stream without waiting for
    // it: every window of this call comes after the work already queued there.  (keys_prepare also drains the engine
    // stream from the host today; the windows' order does not rest on that.)
    CU(h, cudaEventRecord(h->kt_queued, h->stream));
    CU(h, cudaStreamWaitEvent(h->win_stream, h->kt_queued, 0));
    // one step of model.Train's loop over the resident samples [b*B, b*B + B) of which `have` exist so far.  The batch's
    // history windows (GetUserBehavior at the sample's timestamp) are cut on the window stream into one of two buffers,
    // so the window kernel of batch b+1 runs under the train step of batch b.
    int64_t nrun = 0;
    auto run_batch = [&](int64_t b, int64_t have) -> int {
        const int64_t start = std::min<int64_t>(b * B, have);
        const int nv = (int)std::max<int64_t>(0, std::min<int64_t>(B, have - start));
        const int k = (int)(nrun & 1);
        int* hist = h->kt_hist[k];
        if (nv > 0) {
            if (nrun >= 2) CU(h, cudaStreamWaitEvent(h->win_stream, h->kt_used[k], 0));         // the step two batches back has read this buffer
            RET(ub_windows(h, h->win_stream, h->kt_user + start, h->kt_ts + start, nv, hist));
            CU(h, cudaEventRecord(h->kt_win[k], h->win_stream));
            CU(h, cudaStreamWaitEvent(h->stream, h->kt_win[k], 0));
        }
        RET(train_step_dev(h, h->kt_user + start, h->kt_item + start, hist, h->kt_label + start, B, nv));
        CU(h, cudaEventRecord(h->kt_used[k], h->stream));
        nrun++;
        return CTR_OK;
    };
    // ---- keys → (user row, item row, ts, label), unresolvable samples dropped, order kept.  The resolve kernels of a
    // chunk follow its H2D on the COPY stream, so they (and the staging of the next chunk) overlap the train steps
    // running on the engine stream; the engine stream waits for a chunk's event before it reads that chunk's samples.
    cudaStream_t rs = h->copy_stream;
    int64_t nchunks = ((int64_t)n + (int64_t)chunk - 1) / (int64_t)chunk;
    int64_t queued = 0;                                       // first-epoch batches already on the engine stream (streaming)
    for (int64_t c = 0; c < nchunks; c++) {
        RET(keys_resolve_chunk(h, c, chunk, user_ids, item_ids, ts, label, n, rs));
        if (streaming) {
            const int cs = (int)(c % ctr_handle::kCnt);
            CU(h, cudaMemcpyAsync(h->kt_count_host + cs, h->kt_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, rs));
            CU(h, cudaEventRecord(h->kt_counted[cs], rs));
            if (c >= 1) {       // survivors up to chunk c-1: queue their full batches while chunk c resolves
                const int pc = (int)((c - 1) % ctr_handle::kCnt);
                CU(h, cudaEventSynchronize(h->kt_counted[pc]));
                const int64_t have = (int64_t)h->kt_count_host[pc];
                if ((queued + 1) * (int64_t)B <= have) CU(h, cudaStreamWaitEvent(h->stream, h->kt_counted[pc], 0));
                while ((queued + 1) * (int64_t)B <= have) { RET(run_batch(queued, have)); queued++; }
            }
        }
    }
    CU(h, cudaStreamSynchronize(rs));                          // every sample resolved; the engine stream may still be training
    unsigned long long used = 0;
    CU(h, cudaMemcpyAsync(&used, h->kt_count, sizeof used, cudaMemcpyDeviceToHost, rs));
    CU(h, cudaStreamSynchronize(rs));
    if (rows_used) *rows_used = (int64_t)used;
    // ---- model.Train's loop over the resident samples.  world > 1: every step is collective, so all ranks run the
    // batch count of the rank with the most samples (ranks that ran out train on all-padding batches)
    int64_t nmax = (int64_t)used;
    if (h->comm.world > 1) RET(comm_max_i64(h, &nmax));
    if (nmax == 0) return set_err(h, CTR_ENOTFOUND, "no sample resolved: every key has an unknown user or item");
    const int64_t batches = nmax / B + (nmax % B != 0);     // model.go:96-99
    float best = INFINITY, cost = 0.0f; int no_improve = 0, ep = 0;
    for (ep = 0; ep < epochs; ep++) {
        for (int64_t b = (ep == 0 ? queued : 0); b < batches; b++) RET(run_batch(b, (int64_t)used));
        RET(read_cost(h, B * h->comm.world, &cost));       // cost of the epoch's last batch, model.go:198
        if (cost < best) { best = cost; no_improve = 0; } else no_improve++;
        if (early_stop != 0 && no_improve >= early_stop) { ep++; break; }   // model.go:206-209
    }
    if (last_cost) *last_cost = cost;
    if (epochs_run) *epochs_run = ep;
    return CTR_OK;
}

int ctr_predict_idx_dev(ctr_handle* h, const int32_t* d_user, const int32_t* d_item, const int32_t* d_hist, int32_t B, float* d_out) {
    if (!h || !d_user || !d_item || !d_hist) return set_err(h, CTR_EINVAL, "null argument");
    if (B < 1 || B > h->Bmax) return set_err(h, CTR_EINVAL, "batch %d outside (0, %d]", B, h->Bmax);
    if (emb_sharded(h)) return comm_predict(h, d_user, d_item, d_hist, B, d_out);
    RET(check_tables(h));
    RowSrc r = idx_src(h, d_user, d_item, d_hist, B);
    StepOpts o;
    RET(step_core(h, r, B, o));
    if (d_out) CU(h, cudaMemcpyAsync(d_out, h->P, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    return CTR_OK;
}

int ctr_predict_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row, const int32_t* hist, int64_t n, float* out) {
    if (!h || !user_row || !item_row || !hist || !out || n < 1) return set_err(h, CTR_EINVAL, "bad predict arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    const int B = h->cfg.pred_batch, S = h->cfg.S;
    for (int64_t s = 0; s < n; s += B) {
        const int nb = (int)std::min<int64_t>(B, n - s);
        RET(stage_idx(h, user_row + s, item_row + s, hist + s * S, nullptr, nb));
        RET(ctr_predict_idx_dev(h, h->s_user, h->s_item, h->s_hist, nb, nullptr));
        CU(h, cudaMemcpyAsync(out + s, h->P, (size_t)nb * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));    // staging buffers are reused by the next chunk
    }
    return CTR_OK;
}

int ctr_last_cost(ctr_handle* h, float* cost) {
    if (!h || !cost) return CTR_EINVAL;
    CU(h, cudaSetDevice(h->dev));
    return read_cost(h, h->cfg.batch * h->comm.world, cost);
}

int ctr_sync(ctr_handle* h) {
    if (!h) return CTR_EINVAL;
    CU(h, cudaSetDevice(h->dev));
    CU(h, cudaStreamSynchronize(h->stream));
    if (h->comm.h_err && *h->comm.h_err) return set_err(h, CTR_ECOMM, "peer barrier timed out waiting for rank %d (a rank left the step loop?)", *h->comm.h_err - 1);
    return CTR_OK;
}

void* ctr_get_stream(ctr_handle* h) { return h ? (void*)h->stream : nullptr; }

int ctr_set_stream(ctr_handle* h, void* s) {
    if (!h) return CTR_EINVAL;
    CU(h, cudaStreamSynchronize(h->stream));
    if (h->own_stream) { cudaStreamDestroy(h->stream); h->own_stream = false; }
    h->stream = (cudaStream_t)s;
    return CTR_OK;
}

int64_t ctr_launch_count(const ctr_handle* h) { return h ? h->launches : 0; }

int ctr_profile_enable(ctr_handle* h, int on) { if (!h) return CTR_EINVAL; h->profiling = on != 0; return CTR_OK; }
int ctr_profile_reset(ctr_handle* h) { if (!h) return CTR_EINVAL; h->prof.clear(); return CTR_OK; }
int ctr_profile_get(ctr_handle* h, const char* kernel, double* ms, int64_t* n) {
    if (!h || !kernel) return CTR_EINVAL;
    auto it = h->prof.find(kernel);
    if (it == h->prof.end()) { if (ms) *ms = 0; if (n) *n = 0; return CTR_OK; }
    if (ms) *ms = it->second.ms; if (n) *n = it->second.n;
    return CTR_OK;
}
int ctr_profile_dump(ctr_handle* h, char* buf, int64_t len) {
    if (!h || !buf || len < 1) return CTR_EINVAL;
    std::string s;
    for (auto& kv : h->prof) { char line[256]; snprintf(line, sizeof line, "%s %.6f %ld\n", kv.first.c_str(), kv.second.ms, kv.second.n); s += line; }
    snprintf(buf, (size_t)len, "%s", s.c_str());
    return CTR_OK;
}

int ctr_debug_grads_idx(ctr_handle* h, const int32_t* user_row, const int32_t* item_row, const int32_t* hist, const float* label,
                        int32_t B, int32_t training, float* dmlp0, float* dmlp1, float* dmlp2, float* datt0,
                        float* dUb, float* dIt, float* p, float* logit, float* cost) {
    if (!h || !user_row || !item_row || !hist || !label) return set_err(h, CTR_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    RET(check_tables(h));
    const ctr_config& c = h->cfg;
    if (B < 1 || B > h->Bmax) return set_err(h, CTR_EINVAL, "batch %d outside (0, %d]", B, h->Bmax);
    RET(stage_idx(h, user_row, item_row, hist, label, B));
    RET(zero_grads(h));
    RowSrc r = idx_src(h, h->s_user, h->s_item, h->s_hist, B);
    StepOpts o; o.training = true; o.update = false; o.want_rows = true; o.d_label = h->s_label;
    ctr_config saved = h->cfg;
    if (!training) { h->cfg.dropout0 = 0; h->cfg.dropout1 = 0; }
    int rc = step_core(h, r, B, o);
    h->cfg = saved;
    RET(rc);
    if (dmlp0) CU(h, cudaMemcpy2DAsync(dmlp0, c.H0 * sizeof(float), h->G[0], h->H0p * sizeof(float), c.H0 * sizeof(float), h->in, cudaMemcpyDeviceToHost, h->stream));
    if (dmlp1) CU(h, cudaMemcpy2DAsync(dmlp1, c.H1 * sizeof(float), h->G[1], h->H1p * sizeof(float), c.H1 * sizeof(float), c.H0, cudaMemcpyDeviceToHost, h->stream));
    if (dmlp2) CU(h, cudaMemcpyAsync(dmlp2, h->G[2], c.H1 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (datt0) CU(h, cudaMemcpyAsync(datt0, h->G[3], c.S * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (dUb) CU(h, cudaMemcpyAsync(dUb, h->dUb, (size_t)B * c.S * c.D * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (dIt) CU(h, cudaMemcpyAsync(dIt, h->dIt, (size_t)B * c.D * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (p) CU(h, cudaMemcpyAsync(p, h->P, (size_t)B * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (logit) CU(h, cudaMemcpyAsync(logit, h->Z, (size_t)B * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    float cst = 0;
    RET(read_cost(h, B, &cst));
    if (cost) *cost = cst;
    RET(zero_grads(h));
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

int ctr_ubcache_upload(ctr_handle* h, const int64_t* offsets, const int64_t* ts, const int32_t* item_rows, int64_t n_users, int64_t n) {
    if (!h || !offsets || n_users < 1 || n < 0 || (n > 0 && (!ts || !item_rows))) return set_err(h, CTR_EINVAL, "bad ubcache arguments");
    if (offsets[0] != 0 || offsets[n_users] != n) return set_err(h, CTR_EINVAL, "ubcache offsets must run from 0 to n");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    h->ub_off.reset(); h->ub_ts.reset(); h->ub_items.reset();      // all three freed first; the spare (ubx_*) is kept
    RET(dalloc(h, h->ub_off, (size_t)n_users + 1, false)); RET(dalloc(h, h->ub_ts, (size_t)n, false)); RET(dalloc(h, h->ub_items, (size_t)n, false));
    CU(h, cudaMemcpyAsync(h->ub_off, offsets, sizeof(int64_t) * (size_t)(n_users + 1), cudaMemcpyHostToDevice, h->stream));
    if (n > 0) {
        CU(h, cudaMemcpyAsync(h->ub_ts, ts, sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(h->ub_items, item_rows, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
    }
    CU(h, cudaStreamSynchronize(h->stream));
    h->ub_users = n_users; h->ub_n = n;
    return CTR_OK;
}

int ctr_ubcache_window_dev(ctr_handle* h, const int32_t* d_user_row, const int64_t* d_max_ts, int32_t B, int32_t* d_hist_rows) {
    if (!h || !d_user_row || !d_max_ts || !d_hist_rows || B < 1) return set_err(h, CTR_EINVAL, "bad ubcache window arguments");
    if (!h->ub_off) return set_err(h, CTR_ESTATE, "ubcache not uploaded");
    CU(h, cudaSetDevice(h->dev));
    return ub_windows(h, h->stream, d_user_row, (const long long*)d_max_ts, B, d_hist_rows);
}

int ctr_ubcache_window(ctr_handle* h, const int32_t* user_row, const int64_t* max_ts, int32_t B, int32_t* hist_rows) {
    if (!h || !user_row || !max_ts || !hist_rows || B < 1) return set_err(h, CTR_EINVAL, "bad ubcache window arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    int* du = nullptr; long long* dt = nullptr; int* dh = nullptr;
    int rc = CTR_OK;
    RET(scratch_get(h, 0, sizeof(int) * (size_t)B, (void**)&du)); RET(scratch_get(h, 1, sizeof(long long) * (size_t)B, (void**)&dt));
    RET(scratch_get(h, 2, sizeof(int) * (size_t)B * h->cfg.S, (void**)&dh));
    {
        cudaMemcpyAsync(du, user_row, sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, h->stream);
        cudaMemcpyAsync(dt, max_ts, sizeof(long long) * (size_t)B, cudaMemcpyHostToDevice, h->stream);
        rc = ctr_ubcache_window_dev(h, du, (const int64_t*)dt, B, dh);
        if (rc == CTR_OK && (cudaMemcpyAsync(hist_rows, dh, sizeof(int) * (size_t)B * h->cfg.S, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
                             cudaStreamSynchronize(h->stream) != cudaSuccess)) rc = set_err(h, CTR_ECUDA, "ubcache window copy: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return rc;
}

int ctr_ubcache_append(ctr_handle* h, const int32_t* user_rows, const int64_t* ts, const int32_t* item_rows, int64_t n) {
    if (!h || n < 0 || n > INT32_MAX || (n > 0 && (!user_rows || !ts || !item_rows))) return set_err(h, CTR_EINVAL, "bad ubcache append arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (n == 0) return CTR_OK;
    const int64_t bound = ub_row_bound(h);
    int32_t max_row = 0; int64_t tmin = INT64_MAX, tmax = INT64_MIN;
    for (int64_t i = 0; i < n; i++) {
        if (user_rows[i] < 0 || user_rows[i] >= bound)
            return set_err(h, CTR_EINVAL, "ubcache append: user row %d of event %lld outside [0, %lld)", user_rows[i], (long long)i, (long long)bound);
        max_row = std::max(max_row, user_rows[i]); tmin = std::min(tmin, ts[i]); tmax = std::max(tmax, ts[i]);
    }
    CU(h, cudaSetDevice(h->dev));
    UbBatch ub;
    RET(ub_batch_append(h, user_rows, ts, item_rows, n, max_row, tmin, tmax, &ub));
    return ub_rewrite(h, ub, false, std::max<int64_t>(h->ub_off ? h->ub_users : 0, (int64_t)max_row + 1));
}

int ctr_ubcache_set(ctr_handle* h, const int32_t* user_rows, const int64_t* offsets, const int64_t* ts, const int32_t* item_rows, int64_t n_set, int64_t n) {
    if (!h || n_set < 0 || n < 0 || n_set > INT32_MAX || n > INT32_MAX || (n_set > 0 && (!user_rows || !offsets)) || (n > 0 && (!ts || !item_rows)))
        return set_err(h, CTR_EINVAL, "bad ubcache set arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (n_set == 0) return n == 0 ? CTR_OK : set_err(h, CTR_EINVAL, "ubcache set: %lld events for no user", (long long)n);
    if (offsets[0] != 0 || offsets[n_set] != n) return set_err(h, CTR_EINVAL, "ubcache set: offsets must run from 0 to n");
    const int64_t bound = ub_row_bound(h);
    int32_t max_row = 0;
    for (int64_t k = 0; k < n_set; k++) {
        if (user_rows[k] < 0 || user_rows[k] >= bound)
            return set_err(h, CTR_EINVAL, "ubcache set: user row %d outside [0, %lld)", user_rows[k], (long long)bound);
        if (offsets[k + 1] < offsets[k] || offsets[k + 1] > n) return set_err(h, CTR_EINVAL, "ubcache set: offsets must not decrease nor pass n (entry %lld)", (long long)k);
        for (int64_t e = offsets[k] + 1; e < offsets[k + 1]; e++)
            if (ts[e] > ts[e - 1]) return set_err(h, CTR_EINVAL, "ubcache set: the sequence of user row %d is not time-descending", user_rows[k]);
        max_row = std::max(max_row, user_rows[k]);
    }
    std::vector<int32_t> sorted(user_rows, user_rows + n_set);
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return set_err(h, CTR_EINVAL, "ubcache set: user row %d appears twice", *std::adjacent_find(sorted.begin(), sorted.end()));
    CU(h, cudaSetDevice(h->dev));
    UbBatch ub;
    RET(ub_batch_set(h, user_rows, offsets, ts, item_rows, n_set, n, max_row, &ub));
    return ub_rewrite(h, ub, true, std::max<int64_t>(h->ub_off ? h->ub_users : 0, (int64_t)max_row + 1));
}

int ctr_ubcache_download(ctr_handle* h, int64_t* offsets, int64_t* ts, int32_t* item_rows, int64_t cap_users, int64_t cap_events, int64_t* n_users, int64_t* n) {
    if (!h || !n_users || !n) return set_err(h, CTR_EINVAL, "bad ubcache download arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->ub_off) return set_err(h, CTR_ESTATE, "ubcache not uploaded");
    *n_users = h->ub_users; *n = h->ub_n;
    if ((offsets && cap_users < h->ub_users) || ((ts || item_rows) && cap_events < h->ub_n))
        return set_err(h, CTR_EINVAL, "ubcache download: the cache holds %lld users and %lld events", (long long)h->ub_users, (long long)h->ub_n);
    CU(h, cudaSetDevice(h->dev));
    if (offsets) CU(h, cudaMemcpyAsync(offsets, h->ub_off, sizeof(int64_t) * (size_t)(h->ub_users + 1), cudaMemcpyDeviceToHost, h->stream));
    if (ts && h->ub_n) CU(h, cudaMemcpyAsync(ts, h->ub_ts, sizeof(int64_t) * (size_t)h->ub_n, cudaMemcpyDeviceToHost, h->stream));
    if (item_rows && h->ub_n) CU(h, cudaMemcpyAsync(item_rows, h->ub_items, sizeof(int32_t) * (size_t)h->ub_n, cudaMemcpyDeviceToHost, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return CTR_OK;
}

// ---- sparse ids, serving keys, checkpoint (rows f3 / f4) -------------------------------------------------
int ctr_idmap_build(ctr_handle* h, int which, const int64_t* ids, int64_t n) {
    if (!h || !ids || which < 0 || which > 1 || n < 1 || n > 0x7fffffff) return set_err(h, CTR_EINVAL, "bad idmap arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    h->idm_keys[which].reset(); h->idm_vals[which].reset(); h->idm_n[which] = 0;
    unsigned long long cap = 64;
    while (cap < 2ull * (unsigned long long)n) cap <<= 1;                 // load factor <= 0.5
    RET(dalloc(h, h->idm_keys[which], (size_t)cap, false)); RET(dalloc(h, h->idm_vals[which], (size_t)cap, false));
    if (!h->k_flags) RET(dalloc(h, h->k_flags, 1));
    DevBuf<long long> d_ids;
    CU(h, d_ids.alloc((size_t)n));
    int flags = 0, rc = CTR_OK;
    cudaMemcpyAsync(d_ids, ids, sizeof(long long) * (size_t)n, cudaMemcpyHostToDevice, h->stream);
    cudaMemsetAsync(h->k_flags, 0, sizeof(int), h->stream);
    rc = launch(h, "idmap_clear", [&] { k_idmap_clear<<<h->num_sms * 8, 256, 0, h->stream>>>(h->idm_keys[which], h->idm_vals[which], cap); });
    if (rc == CTR_OK) rc = launch(h, "idmap_insert", [&] {
        k_idmap_insert<<<h->num_sms * 8, 256, 0, h->stream>>>(h->idm_keys[which], h->idm_vals[which], cap - 1, d_ids, (long)n, h->k_flags, 0);
    });
    if (rc == CTR_OK && (cudaMemcpyAsync(&flags, h->k_flags, sizeof(int), cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
                         cudaStreamSynchronize(h->stream) != cudaSuccess)) rc = set_err(h, CTR_ECUDA, "idmap build: %s", cudaGetErrorString(cudaGetLastError()));
    RET(rc);
    if (flags) {
        h->idm_keys[which].reset(); h->idm_vals[which].reset();
        return set_err(h, CTR_EINVAL, flags & 2 ? "idmap: id INT64_MIN is reserved" : "idmap: duplicate ids");
    }
    h->idm_n[which] = n;
    return CTR_OK;
}

int ctr_idmap_lookup_dev(ctr_handle* h, int which, const int64_t* d_ids, int64_t n, int32_t* d_rows) {
    if (!h || !d_ids || !d_rows || which < 0 || which > 1 || n < 1) return set_err(h, CTR_EINVAL, "bad idmap lookup arguments");
    if (!h->idm_keys[which]) return set_err(h, CTR_ESTATE, "idmap %d not built", which);
    CU(h, cudaSetDevice(h->dev));
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, h->num_sms * 8));
    return launch(h, "idmap_lookup", [&] {
        k_idmap_lookup<<<grid, 256, 0, h->stream>>>(h->idm_keys[which], h->idm_vals[which], h->idm_keys[which].size() - 1, (const long long*)d_ids, (long)n, d_rows);
    });
}

int ctr_idmap_lookup(ctr_handle* h, int which, const int64_t* ids, int64_t n, int32_t* rows) {
    if (!h || !ids || !rows || which < 0 || which > 1 || n < 1) return set_err(h, CTR_EINVAL, "bad idmap lookup arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    long long* d_ids = nullptr; int* d_rows = nullptr;
    int rc = CTR_OK;
    RET(scratch_get(h, 0, sizeof(long long) * (size_t)n, (void**)&d_ids)); RET(scratch_get(h, 1, sizeof(int) * (size_t)n, (void**)&d_rows));
    {
        cudaMemcpyAsync(d_ids, ids, sizeof(long long) * (size_t)n, cudaMemcpyHostToDevice, h->stream);
        rc = ctr_idmap_lookup_dev(h, which, (const int64_t*)d_ids, n, d_rows);
        if (rc == CTR_OK && (cudaMemcpyAsync(rows, d_rows, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
                             cudaStreamSynchronize(h->stream) != cudaSuccess)) rc = set_err(h, CTR_ECUDA, "idmap lookup copy: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return rc;
}

namespace {
// staging of the key-fed predict calls, moved in together: device [user ids | item ids | ts] of one pred_batch chunk and
// pinned host [keys | scores | first user row]
int keys_stage_init(ctr_handle* h) {
    if (h->k_keys) return CTR_OK;
    const int B = h->cfg.pred_batch;
    DevBuf<long long> keys; PinnedBuf<unsigned char> host;
    RET(dalloc(h, keys, (size_t)3 * B, false));
    CU(h, host.alloc(sizeof(long long) * (size_t)3 * B + sizeof(float) * (size_t)B + 16));
    h->k_host = std::move(host); h->k_keys = std::move(keys);
    return CTR_OK;
}
}  // namespace

int ctr_batch_predict_keys(ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n, float* scores) {
    if (!h || !user_ids || !item_ids || !ts || !scores || n < 1) return set_err(h, CTR_EINVAL, "bad batch predict arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    if (!h->idm_keys[0] || !h->idm_keys[1]) return set_err(h, CTR_ESTATE, "batch predict needs both id maps (ctr_idmap_build)");
    const int B = h->cfg.pred_batch, S = h->cfg.S;
    RET(keys_stage_init(h));
    long long* hk = (long long*)h->k_host.get();
    float* hs = (float*)(hk + (size_t)3 * B);
    int* hfirst = (int*)(hs + B);
    for (int64_t s = 0; s < n; s += B) {
        const int nb = (int)std::min<int64_t>(B, n - s);
        memcpy(hk, user_ids + s, sizeof(long long) * (size_t)nb);
        memcpy(hk + nb, item_ids + s, sizeof(long long) * (size_t)nb);
        memcpy(hk + 2 * (size_t)nb, ts + s, sizeof(long long) * (size_t)nb);
        CU(h, cudaMemcpyAsync(h->k_keys, hk, sizeof(long long) * (size_t)3 * nb, cudaMemcpyHostToDevice, h->stream));
        RET(launch(h, "keys_resolve", [&] {
            k_keys_resolve<<<grid_for_warps(h, nb), 256, 0, h->stream>>>(h->idm_keys[0], h->idm_vals[0], h->idm_keys[0].size() - 1, h->idm_keys[1], h->idm_vals[1], h->idm_keys[1].size() - 1,
                                                                    h->ub_off, h->ub_ts, h->ub_items, (long)h->ub_users, h->k_keys, nb, S, h->s_user, h->s_item, h->s_hist);
        }));
        if (s == 0) CU(h, cudaMemcpyAsync(hfirst, h->s_user, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        RET(ctr_predict_idx_dev(h, h->s_user, h->s_item, h->s_hist, nb, nullptr));
        CU(h, cudaMemcpyAsync(hs, h->P, (size_t)nb * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        // rcmd.go:300-303: an unresolvable FIRST key is an error, later ones become zero rows
        if (s == 0 && *hfirst < 0) return set_err(h, CTR_ENOTFOUND, "get sample vector error: user %lld or item %lld has no features", (long long)user_ids[0], (long long)item_ids[0]);
        memcpy(scores + s, hs, sizeof(float) * (size_t)nb);
    }
    return CTR_OK;
}

namespace {
struct CkptHeader {
    char magic[8];                 // "CTRB200\0"
    int32_t version, model, uP, S, D, cF, H0, H1, rank, world;
    uint32_t step;
    int32_t has_table[3];
    int64_t tab_rows[3], tab_local_rows[3];
    int32_t tab_width[3];
    int32_t replicated;            // ITEM_EMB placement under world > 1 (1 = every rank holds the whole table)
    int32_t has_moments;           // ITEM_EMB Adam moments follow the tables (CTR_TABLE_ADAM)
};
constexpr size_t kCkptChunk = 32u << 20;

// device [rows, ld] → file as compact [rows, width], through a pinned bounce buffer
int ckpt_write_2d(ctr_handle* h, FILE* f, const float* d, long ld, int64_t rows, int width, float* bounce) {
    const int64_t per = std::max<int64_t>(1, (int64_t)(kCkptChunk / sizeof(float)) / width);
    for (int64_t r = 0; r < rows; r += per) {
        const int64_t nr = std::min(per, rows - r);
        CU(h, cudaMemcpy2DAsync(bounce, (size_t)width * sizeof(float), d + (size_t)r * ld, (size_t)ld * sizeof(float), (size_t)width * sizeof(float), (size_t)nr, cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        if (fwrite(bounce, sizeof(float), (size_t)nr * width, f) != (size_t)nr * width) return set_err(h, CTR_EIO, "checkpoint: short write");
    }
    return CTR_OK;
}
int ckpt_read_2d(ctr_handle* h, FILE* f, float* d, long ld, int64_t rows, int width, float* bounce) {
    const int64_t per = std::max<int64_t>(1, (int64_t)(kCkptChunk / sizeof(float)) / width);
    for (int64_t r = 0; r < rows; r += per) {
        const int64_t nr = std::min(per, rows - r);
        if (fread(bounce, sizeof(float), (size_t)nr * width, f) != (size_t)nr * width) return set_err(h, CTR_EIO, "checkpoint: truncated file");
        CU(h, cudaMemcpy2DAsync(d + (size_t)r * ld, (size_t)ld * sizeof(float), bounce, (size_t)width * sizeof(float), (size_t)width * sizeof(float), (size_t)nr, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    }
    return CTR_OK;
}
// the four learnable tensors in their logical (reference JSON) shapes
void dense_shape(const ctr_handle* h, int i, int64_t* rows, int* width, long* ld) {
    const ctr_config& c = h->cfg;
    if (i == 0) { *rows = h->in; *width = c.H0; *ld = h->H0p; }
    else if (i == 1) { *rows = c.H0; *width = c.H1; *ld = h->H1p; }
    else if (i == 2) { *rows = 1; *width = c.H1; *ld = h->H1p; }
    else { *rows = 1; *width = c.S; *ld = h->Sp; }
}
}  // namespace

int ctr_checkpoint_save(ctr_handle* h, const char* path) {
    if (!h || !path) return set_err(h, CTR_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    if (h->tab_sharded[CTR_TABLE_ITEM_EMB]) RET(comm_hot_writeback(h));
    CU(h, cudaStreamSynchronize(h->stream));
    FILE* f = fopen(path, "wb");
    if (!f) return set_err(h, CTR_EIO, "checkpoint: cannot open %s for writing", path);
    PinnedBuf<float> bounce;
    if (bounce.alloc(kCkptChunk / sizeof(float)) != cudaSuccess) { fclose(f); return set_err(h, CTR_ENOMEM, "checkpoint bounce buffer"); }
    const ctr_config& c = h->cfg;
    CkptHeader hd{};
    memcpy(hd.magic, "CTRB200", 8);
    hd.version = 2; hd.model = c.model; hd.uP = c.uP; hd.S = c.S; hd.D = c.D; hd.cF = c.cF; hd.H0 = c.H0; hd.H1 = c.H1;
    hd.rank = h->comm.rank; hd.world = h->comm.world; hd.step = h->step; hd.replicated = h->comm.replicate ? 1 : 0;
    hd.has_moments = (h->emb_m && h->tab[CTR_TABLE_ITEM_EMB]) ? 1 : 0;
    for (int t = 0; t < 3; t++) { hd.has_table[t] = h->tab[t] != nullptr; hd.tab_rows[t] = h->tab_rows[t]; hd.tab_local_rows[t] = h->tab_local_rows[t]; hd.tab_width[t] = h->tab_width[t]; }
    int rc = fwrite(&hd, sizeof hd, 1, f) == 1 ? CTR_OK : set_err(h, CTR_EIO, "checkpoint: short write");
    for (int i = 0; i < 4 && rc == CTR_OK; i++) {
        int64_t rows; int width; long ld; dense_shape(h, i, &rows, &width, &ld);
        for (float* src : {h->W[i].get(), h->Mo[i].get(), h->Vo[i].get()}) if (rc == CTR_OK) rc = ckpt_write_2d(h, f, src, ld, rows, width, bounce);
    }
    for (int t = 0; t < 3 && rc == CTR_OK; t++)
        if (h->tab[t]) rc = ckpt_write_2d(h, f, h->tab[t], h->tab_ld[t], h->tab_local_rows[t], h->tab_width[t], bounce);
    if (hd.has_moments)
        for (float* src : {h->emb_m.get(), h->emb_v.get()})
            if (rc == CTR_OK) rc = ckpt_write_2d(h, f, src, h->tab_ld[CTR_TABLE_ITEM_EMB], h->tab_local_rows[CTR_TABLE_ITEM_EMB], h->tab_width[CTR_TABLE_ITEM_EMB], bounce);
    if (fclose(f) != 0 && rc == CTR_OK) rc = set_err(h, CTR_EIO, "checkpoint: close failed");
    return rc;
}

int ctr_checkpoint_load(ctr_handle* h, const char* path) {
    if (!h || !path) return set_err(h, CTR_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    FILE* f = fopen(path, "rb");
    if (!f) return set_err(h, CTR_EIO, "checkpoint: cannot open %s", path);
    CkptHeader hd{};
    const ctr_config& c = h->cfg;
    int rc = CTR_OK;
    if (fread(&hd, sizeof hd, 1, f) != 1 || memcmp(hd.magic, "CTRB200", 8) != 0 || hd.version != 2) rc = set_err(h, CTR_EIO, "checkpoint: %s is not a version-2 ctr-b200 snapshot", path);
    else if (hd.model != c.model || hd.uP != c.uP || hd.S != c.S || hd.D != c.D || hd.cF != c.cF || hd.H0 != c.H0 || hd.H1 != c.H1)
        rc = set_err(h, CTR_EINVAL, "checkpoint: model dims differ from this handle");
    else if (hd.rank != h->comm.rank || hd.world != h->comm.world) rc = set_err(h, CTR_EINVAL, "checkpoint: written by rank %d/%d, this handle is %d/%d", hd.rank, hd.world, h->comm.rank, h->comm.world);
    PinnedBuf<float> bounce;
    if (rc == CTR_OK && bounce.alloc(kCkptChunk / sizeof(float)) != cudaSuccess) rc = set_err(h, CTR_ENOMEM, "checkpoint bounce buffer");
    for (int i = 0; i < 4 && rc == CTR_OK; i++) {
        int64_t rows; int width; long ld; dense_shape(h, i, &rows, &width, &ld);
        for (float* dst : {h->W[i].get(), h->Mo[i].get(), h->Vo[i].get()}) if (rc == CTR_OK) rc = ckpt_read_2d(h, f, dst, ld, rows, width, bounce);
    }
    for (int t = 0; t < 3 && rc == CTR_OK; t++) {
        if (!hd.has_table[t]) continue;
        const int want = t == CTR_TABLE_USER_FEAT ? c.uP : t == CTR_TABLE_ITEM_FEAT ? c.cF : c.D;
        if (hd.tab_width[t] != want || hd.tab_rows[t] < 1 || hd.tab_local_rows[t] < 0) { rc = set_err(h, CTR_EIO, "checkpoint: bad table %d header", t); break; }
        const long ld = round_up(hd.tab_width[t], 4);
        const size_t bytes = (size_t)std::max<int64_t>(hd.tab_local_rows[t], 1) * ld * sizeof(float);
        // placement travels with the snapshot: a shard holds fewer rows than the logical table
        h->tab_sharded[t] = h->comm.world > 1 && t != CTR_TABLE_USER_FEAT && (t == CTR_TABLE_ITEM_EMB ? hd.replicated != 1 : hd.tab_local_rows[t] != hd.tab_rows[t]);
        rc = table_mem(h, t, h->tab_sharded[t], bytes);
        if (rc != CTR_OK) break;
        h->tab_ld[t] = ld; h->tab_rows[t] = hd.tab_rows[t]; h->tab_local_rows[t] = hd.tab_local_rows[t]; h->tab_width[t] = hd.tab_width[t];
        if (t == CTR_TABLE_ITEM_EMB) h->comm.replicate = h->comm.world > 1 && hd.replicated == 1;
        if (t != CTR_TABLE_USER_FEAT) h->tab_gen++;
        rc = ckpt_read_2d(h, f, h->tab[t], ld, hd.tab_local_rows[t], hd.tab_width[t], bounce);
        if (t == CTR_TABLE_ITEM_EMB && h->hot_acc) { h->hot_acc.reset(); h->hot_rows = 0; }
    }
    h->emb_m.reset(); h->emb_v.reset();
    if (rc == CTR_OK && hd.has_moments) {
        rc = ensure_moments(h);
        for (float* dst : {h->emb_m.get(), h->emb_v.get()})
            if (rc == CTR_OK) rc = ckpt_read_2d(h, f, dst, h->tab_ld[CTR_TABLE_ITEM_EMB], h->tab_local_rows[CTR_TABLE_ITEM_EMB], h->tab_width[CTR_TABLE_ITEM_EMB], bounce);
    }
    fclose(f);
    if (rc == CTR_OK) { h->step = hd.step; h->um.dirty = true; cudaStreamSynchronize(h->stream); }
    return rc;
}

int ctr_roc_auc(ctr_handle* h, const float* pred, const float* y, int64_t n, double* auc) {
    if (!h || !pred || !y || !auc || n < 1 || n > 0x7fffffff) return set_err(h, CTR_EINVAL, "bad auc arguments (n must be in [1, 2^31))");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    { cudaError_t e = auc_run(h->stream, pred, y, (long)n, auc); if (e != cudaSuccess) return set_err(h, CTR_ECUDA, "auc: %s", cudaGetErrorString(e)); return CTR_OK; }
}

namespace {

// the engine's launch() in the shape the shared drivers of auc.cuh take
auto profiled(ctr_handle* h) { return [h](const char* name, auto&& f) { return launch(h, name, f); }; }

// The fold of ctr_group_auc and ctr_group_auc_dist over the groups in uniq / agg (*d_runs of them; room for the per-group
// outputs of `room`), then the results: a non-null out_* array with cap < the group count is CTR_EINVAL with nothing
// written.
int gauc_fold(ctr_handle* h, const unsigned long long* uniq, const GaucAgg* agg, const int* d_runs, size_t room, int64_t cap, double* gauc,
              int64_t* n_groups, int64_t* n_used, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc) {
    cudaStream_t st = h->stream;
    DevBuf<GaucPart> part; DevBuf<GaucResult> res;
    DevBuf<long long> o_group; DevBuf<int> o_n, o_pos; DevBuf<double> o_auc;
    CU(h, part.alloc(kGaucParts)); CU(h, res.alloc(1));
    if (out_group) CU(h, o_group.alloc(room));
    if (out_n) CU(h, o_n.alloc(room));
    if (out_pos) CU(h, o_pos.alloc(room));
    if (out_auc) CU(h, o_auc.alloc(room));
    RET(gauc_fold_groups(profiled(h), uniq, agg, d_runs, o_group, o_n, o_pos, o_auc, part, res, st));
    GaucResult r{};
    CU(h, cudaMemcpyAsync(&r, res, sizeof r, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if ((out_group || out_n || out_pos || out_auc) && r.groups > cap)
        return set_err(h, CTR_EINVAL, "group auc: %lld groups do not fit the per-group arrays (cap %lld)", (long long)r.groups, (long long)cap);
    const size_t R = (size_t)r.groups;
    if (out_group) CU(h, cudaMemcpyAsync(out_group, o_group, R * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    if (out_n) CU(h, cudaMemcpyAsync(out_n, o_n, R * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (out_pos) CU(h, cudaMemcpyAsync(out_pos, o_pos, R * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (out_auc) CU(h, cudaMemcpyAsync(out_auc, o_auc, R * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    *gauc = r.gauc;
    if (n_groups) *n_groups = r.groups;
    if (n_used) *n_used = r.used;
    return CTR_OK;
}

// ctr_group_auc on the engine stream: (group, score) order by two stable radix passes, one scan, one reduce-by-key,
// then the per-group AUCs and their weighted mean on the device (auc.cuh); only the result, and the per-group arrays
// when asked for, come back
int gauc_run(ctr_handle* h, const float* pred_h, const float* y_h, const int64_t* group_h, long n, double* gauc,
             int64_t* n_groups, int64_t* n_used, int64_t cap, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc) {
    cudaStream_t st = h->stream;
    const size_t N = (size_t)n;
    const int grid = (int)std::min<long>((n + 255) / 256, (long)h->num_sms * 8);
    DevBuf<float> d_pred, d_y; DevBuf<long long> d_group;
    DevBuf<unsigned> k0, k1; DevBuf<int> i0, i1, d_runs;
    DevBuf<unsigned long long> g0, g1, v0, v1;
    DevBuf<GaucScan> scan; DevBuf<GaucAgg> val, agg;
    DevBuf<unsigned char> tmp;
    CU(h, d_pred.alloc(N)); CU(h, d_y.alloc(N)); CU(h, d_group.alloc(N));
    CU(h, k0.alloc(N)); CU(h, k1.alloc(N)); CU(h, i0.alloc(N)); CU(h, i1.alloc(N));
    CU(h, g0.alloc(N)); CU(h, g1.alloc(N)); CU(h, v0.alloc(N)); CU(h, v1.alloc(N));
    CU(h, scan.alloc(N)); CU(h, val.alloc(N)); CU(h, agg.alloc(N));
    CU(h, d_runs.alloc(1));
    unsigned long long* uniq = g0.get();     // free once the group pass has read it
    size_t b[4] = {0, 0, 0, 0};
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b[0], k0.get(), k1.get(), i0.get(), i1.get(), (int)n, 0, 32, st));
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b[1], g0.get(), g1.get(), v0.get(), v1.get(), (int)n, 0, 64, st));
    CU(h, cub::DeviceScan::InclusiveScan(nullptr, b[2], scan.get(), scan.get(), GaucScanOp(), (int)n, st));
    CU(h, cub::DeviceReduce::ReduceByKey(nullptr, b[3], g1.get(), uniq, val.get(), agg.get(), d_runs.get(), GaucAggOp(), (int)n, st));
    size_t bytes = std::max(std::max(b[0], b[1]), std::max(b[2], b[3]));
    CU(h, tmp.alloc(std::max<size_t>(bytes, 1)));
    CU(h, cudaMemcpyAsync(d_pred, pred_h, N * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_y, y_h, N * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_group, group_h, N * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    RET(launch(h, "gauc_keys", [&] { k_gauc_keys<<<grid, 256, 0, st>>>(d_pred, n, k0, i0); }));
    RET(launch(h, "gauc_sort_score", [&] {
        cub::DeviceRadixSort::SortPairs(tmp.get(), bytes, k0.get(), k1.get(), i0.get(), i1.get(), (int)n, 0, 32, st); }));
    RET(launch(h, "gauc_gather", [&] { k_gauc_gather<<<grid, 256, 0, st>>>(k1, i1, d_group, d_y, n, g0, v0); }));
    RET(launch(h, "gauc_sort_group", [&] {
        cub::DeviceRadixSort::SortPairs(tmp.get(), bytes, g0.get(), g1.get(), v0.get(), v1.get(), (int)n, 0, 64, st); }));
    RET(gauc_group_terms(profiled(h), g1, v1, n, scan, val, uniq, agg, d_runs, tmp, bytes, grid, st));
    return gauc_fold(h, uniq, agg, d_runs, N, cap, gauc, n_groups, n_used, out_group, out_n, out_pos, out_auc);
}

}  // namespace

int ctr_group_auc(ctr_handle* h, const float* pred, const float* y, const int64_t* group, int64_t n, double* gauc,
                  int64_t* n_groups, int64_t* n_used, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc) {
    if (!h || !pred || !y || !group || !gauc || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad group auc arguments (n must be in [1, 2^31); pred, y, group and gauc non-null)");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return gauc_run(h, pred, y, group, (long)n, gauc, n_groups, n_used, n, out_group, out_n, out_pos, out_auc);
}

namespace {

// The agreement of the two evaluation calls on world > 1: mode tells the calls apart, so that ranks in different calls
// refuse together; every rank's sample count comes back in shares and their total is checked here.
int eval_agree(ctr_handle* h, int mode, int verdict, int64_t n, int64_t* shares, int64_t* total) {
    CommHdr hd{};
    hd.mode = mode; hd.share = n;
    RET(comm_agree(h, hd, verdict, shares));
    *total = 0;
    for (int j = 0; j < h->comm.world; j++) *total += shares[j];
    if (*total < 1 || *total > (int64_t)0xffffffffll)
        return set_err(h, CTR_EINVAL, "the ranks pass %lld samples in all; the total must be in [1, 2^32)", (long long)*total);
    return CTR_OK;
}

// The exchange plan of a range partition: this rank's sorted keys are cut at the splitters of every rank's samples
// (smp: this rank's samples on the device, off: the cut on the device), the send counts all-gathered, and the receive
// counts and offsets derived.  Every rank computes the same matrix, so a receive over 2^31 - 1 is refused everywhere.
// keys: unsigned (wide = false) or unsigned long long (wide = true)
int dist_plan(ctr_handle* h, const char* key_part, const void* keys, bool wide, const int* d_u, long long* smp, unsigned long long* spl, long long* off,
              std::vector<int64_t>& scnt, std::vector<int64_t>& soff, std::vector<int64_t>& rcnt, std::vector<int64_t>& roff, int64_t* recv) {
    const int W = h->comm.world, me = h->comm.rank;
    cudaStream_t st = h->stream;
    int64_t mine[kDistSamples + 1], all[(kDistSamples + 1) * kMaxPeers];
    RET(launch(h, key_part, [&] {
        if (wide) dist_samples((const unsigned long long*)keys, d_u, smp, st); else dist_samples((const unsigned*)keys, d_u, smp, st); }));
    CU(h, cudaMemcpyAsync(mine, smp, sizeof mine, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    RET(comm_gather_i64(h, mine, kDistSamples + 1, all));
    unsigned long long hs[kMaxPeers];
    dist_splitters(all, W, hs);
    CU(h, cudaMemcpyAsync(spl, hs, sizeof(unsigned long long) * (size_t)(W - 1), cudaMemcpyHostToDevice, st));
    RET(launch(h, key_part, [&] {
        if (wide) dist_part((const unsigned long long*)keys, d_u, spl, W, off, st); else dist_part((const unsigned*)keys, d_u, spl, W, off, st); }));
    int64_t o[kMaxPeers + 1];
    CU(h, cudaMemcpyAsync(o, off, sizeof(int64_t) * (size_t)(W + 1), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    scnt.assign((size_t)W, 0); soff.assign((size_t)W, 0); rcnt.assign((size_t)W, 0); roff.assign((size_t)W, 0);
    for (int k = 0; k < W; k++) { soff[(size_t)k] = o[k]; scnt[(size_t)k] = o[k + 1] - o[k]; }
    int64_t mat[kMaxPeers * kMaxPeers];
    RET(comm_gather_i64(h, scnt.data(), W, mat));            // mat[j·W + k]: what rank j sends rank k
    *recv = 0;
    for (int k = 0; k < W; k++) {
        int64_t in = 0;
        for (int j = 0; j < W; j++) in += mat[j * W + k];
        if (in > 0x7fffffffll)
            return set_err(h, CTR_EINVAL, "rank %d would receive %lld entries of one key range; a rank takes at most 2^31 - 1", k, (long long)in);
    }
    for (int j = 0; j < W; j++) { roff[(size_t)j] = *recv; rcnt[(size_t)j] = mat[j * W + me]; *recv += rcnt[(size_t)j]; }
    return CTR_OK;
}

// ctr_roc_auc_dist on world > 1 after the agreement: local runs, range partition, runs to their owners, merge, the
// positives below each rank, integer area summed over the ranks
int auc_dist_ranks(ctr_handle* h, const float* pred_h, const float* y_h, long n, double* auc) {
    cudaStream_t st = h->stream;
    const int W = h->comm.world;
    const size_t N = (size_t)std::max<long>(n, 1);
    DevBuf<float> d_pred, d_y; DevBuf<unsigned> k0, ks, uk; DevBuf<unsigned long long> c0, cs, uc, spl, acc;
    DevBuf<long long> smp, off; DevBuf<int> d_u; DevBuf<unsigned char> tmp;
    CU(h, d_pred.alloc(N)); CU(h, d_y.alloc(N)); CU(h, k0.alloc(N)); CU(h, ks.alloc(N)); CU(h, uk.alloc(N));
    CU(h, c0.alloc(N)); CU(h, cs.alloc(N)); CU(h, uc.alloc(N));
    CU(h, spl.alloc(kMaxPeers)); CU(h, acc.alloc(1)); CU(h, smp.alloc(kDistSamples + 1)); CU(h, off.alloc(kMaxPeers + 1)); CU(h, d_u.alloc(1));
    size_t bytes = auc_dist_rle_bytes((long)N, st);
    CU(h, tmp.alloc(bytes));
    if (n > 0) {
        CU(h, cudaMemcpyAsync(d_pred, pred_h, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
        CU(h, cudaMemcpyAsync(d_y, y_h, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    cudaError_t e = cudaSuccess;
    RET(launch(h, "auc_dist_rle", [&] { e = auc_dist_local(d_pred, d_y, n, k0, c0, ks, cs, uk, uc, d_u, tmp, bytes, st); }));
    CU(h, e);
    d_pred.reset(); d_y.reset(); k0.reset(); c0.reset(); ks.reset(); cs.reset();
    std::vector<int64_t> scnt, soff, rcnt, roff;
    int64_t M = 0;
    RET(dist_plan(h, "auc_dist_part", uk, false, d_u, smp, spl, off, scnt, soff, rcnt, roff, &M));
    const size_t MM = (size_t)std::max<int64_t>(M, 1);
    DevBuf<unsigned> rk, mk; DevBuf<unsigned long long> rc, mc, inc;
    CU(h, rk.alloc(MM)); CU(h, rc.alloc(MM));
    int rcode = CTR_OK;
    RET(launch(h, "auc_dist_ranks", [&] {
        rcode = comm_route(h, uk, scnt.data(), soff.data(), rk, rcnt.data(), roff.data(), sizeof(unsigned));
        if (rcode == CTR_OK) rcode = comm_route(h, uc, scnt.data(), soff.data(), rc, rcnt.data(), roff.data(), sizeof(unsigned long long)); }));
    RET(rcode);
    CU(h, ks.alloc(MM)); CU(h, cs.alloc(MM)); CU(h, mk.alloc(MM)); CU(h, mc.alloc(MM)); CU(h, inc.alloc(MM));
    if ((size_t)M > N) { bytes = auc_dist_rle_bytes((long)M, st); CU(h, tmp.alloc(bytes)); }
    RET(launch(h, "auc_dist_merge", [&] { e = auc_dist_rle(rk, rc, (long)M, ks, cs, mk, mc, d_u, tmp, bytes, st); }));
    CU(h, e);
    int m = 0;
    CU(h, cudaMemcpyAsync(&m, d_u, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    unsigned long long pn[2];
    RET(launch(h, "auc_dist_area", [&] { e = auc_dist_totals(mc, m, inc, tmp, bytes, &pn[0], &pn[1], st); }));
    CU(h, e);
    int64_t mine[2] = {(int64_t)pn[0], (int64_t)pn[1]}, all[2 * kMaxPeers];
    RET(comm_gather_i64(h, mine, 2, all));
    unsigned long long base = 0, P = 0, Nn = 0;
    for (int j = 0; j < W; j++) {
        if (j < h->comm.rank) base += (unsigned long long)all[2 * j];
        P += (unsigned long long)all[2 * j]; Nn += (unsigned long long)all[2 * j + 1];
    }
    RET(launch(h, "auc_dist_area", [&] { e = auc_dist_area(mc, inc, m, base, acc, st); }));
    CU(h, e);
    RET(launch(h, "auc_dist_ranks", [&] { rcode = comm_sum_u64(h, acc, 1); }));
    RET(rcode);
    unsigned long long area2 = 0;
    CU(h, cudaMemcpyAsync(&area2, acc, sizeof area2, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    *auc = auc_dist_value(area2, P, Nn);
    return CTR_OK;
}

// ctr_group_auc_dist on world > 1 after the agreement: records sorted by group, range partition, records to their
// owners, the grouped driver on each rank's groups, the groups' terms concatenated in rank order (ascending groups) and
// folded on every rank as ctr_group_auc folds them
int gauc_dist_ranks(ctr_handle* h, const float* pred_h, const float* y_h, const int64_t* group_h, long n, double* gauc, int64_t* n_groups,
                    int64_t* n_used, int64_t cap, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc) {
    cudaStream_t st = h->stream;
    const int W = h->comm.world, me = h->comm.rank;
    const size_t N = (size_t)std::max<long>(n, 1);
    DevBuf<float> d_pred, d_y; DevBuf<long long> d_group, smp, off;
    DevBuf<unsigned long long> g0, v0, g1, v1, spl; DevBuf<int> d_u; DevBuf<unsigned char> tmp;
    CU(h, d_pred.alloc(N)); CU(h, d_y.alloc(N)); CU(h, d_group.alloc(N));
    CU(h, g0.alloc(N)); CU(h, v0.alloc(N)); CU(h, g1.alloc(N)); CU(h, v1.alloc(N));
    CU(h, spl.alloc(kMaxPeers)); CU(h, smp.alloc(kDistSamples + 1)); CU(h, off.alloc(kMaxPeers + 1)); CU(h, d_u.alloc(1));
    size_t bytes = gauc_dist_bytes((long)N, st);
    CU(h, tmp.alloc(bytes));
    const int un = (int)n;
    CU(h, cudaMemcpyAsync(d_u, &un, sizeof(int), cudaMemcpyHostToDevice, st));
    cudaError_t e = cudaSuccess;
    if (n > 0) {
        CU(h, cudaMemcpyAsync(d_pred, pred_h, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
        CU(h, cudaMemcpyAsync(d_y, y_h, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, st));
        CU(h, cudaMemcpyAsync(d_group, group_h, (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, st));
        RET(launch(h, "gauc_dist_sort", [&] { e = gauc_dist_sort(d_pred, d_y, d_group, n, g0, v0, g1, v1, tmp, bytes, st); }));
        CU(h, e);
    }
    CU(h, cudaStreamSynchronize(st));          // the pageable copies have read the caller's arrays
    d_pred.reset(); d_y.reset(); d_group.reset(); g0.reset(); v0.reset();
    std::vector<int64_t> scnt, soff, rcnt, roff;
    int64_t M = 0;
    RET(dist_plan(h, "gauc_dist_part", g1, true, d_u, smp, spl, off, scnt, soff, rcnt, roff, &M));
    const size_t MM = (size_t)std::max<int64_t>(M, 1);
    DevBuf<unsigned long long> rg, rv;
    CU(h, rg.alloc(MM)); CU(h, rv.alloc(MM));
    int rcode = CTR_OK;
    RET(launch(h, "gauc_dist_ranks", [&] {
        rcode = comm_route(h, g1, scnt.data(), soff.data(), rg, rcnt.data(), roff.data(), sizeof(unsigned long long));
        if (rcode == CTR_OK) rcode = comm_route(h, v1, scnt.data(), soff.data(), rv, rcnt.data(), roff.data(), sizeof(unsigned long long)); }));
    RET(rcode);
    CU(h, cudaStreamSynchronize(st));
    g1.reset(); v1.reset();
    DevBuf<unsigned long long> uniq; DevBuf<GaucAgg> agg;
    int R = 0;
    if (M > 0) {
        DevBuf<GaucScan> scan; DevBuf<GaucAgg> val;
        CU(h, g0.alloc(MM)); CU(h, v0.alloc(MM)); CU(h, g1.alloc(MM)); CU(h, v1.alloc(MM));
        CU(h, scan.alloc(MM)); CU(h, val.alloc(MM)); CU(h, uniq.alloc(MM)); CU(h, agg.alloc(MM));
        if ((size_t)M > N) { bytes = gauc_dist_bytes((long)M, st); CU(h, tmp.alloc(bytes)); }
        RET(launch(h, "gauc_dist_order", [&] { e = gauc_dist_order(rg, rv, (long)M, g0, v0, g1, v1, tmp, bytes, st); }));
        CU(h, e);
        rg.reset(); rv.reset();
        RET(gauc_group_terms(profiled(h), g1, v1, (long)M, scan, val, uniq, agg, d_u, tmp, bytes, dist_grid((long)M), st));
        CU(h, cudaMemcpyAsync(&R, d_u, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(h, cudaStreamSynchronize(st));
    }
    int64_t mine = R, cnt[kMaxPeers], goff[kMaxPeers];
    RET(comm_gather_i64(h, &mine, 1, cnt));
    int64_t G = 0;
    for (int j = 0; j < W; j++) { goff[j] = G; G += cnt[j]; }
    if (G > 0x7fffffffll) return set_err(h, CTR_EINVAL, "group auc: %lld groups; at most 2^31 - 1", (long long)G);
    if ((out_group || out_n || out_pos || out_auc) && G > cap)
        return set_err(h, CTR_EINVAL, "group auc: %lld groups do not fit the per-group arrays (cap %lld)", (long long)G, (long long)cap);
    DevBuf<unsigned long long> all_uniq; DevBuf<GaucAgg> all_agg;
    CU(h, all_uniq.alloc((size_t)G)); CU(h, all_agg.alloc((size_t)G));
    if (R > 0) {
        CU(h, cudaMemcpyAsync(all_uniq.get() + goff[me], uniq, sizeof(unsigned long long) * (size_t)R, cudaMemcpyDeviceToDevice, st));
        CU(h, cudaMemcpyAsync(all_agg.get() + goff[me], agg, sizeof(GaucAgg) * (size_t)R, cudaMemcpyDeviceToDevice, st));
    }
    RET(launch(h, "gauc_dist_ranks", [&] {
        rcode = comm_concat(h, all_uniq, sizeof(unsigned long long), cnt, goff);
        if (rcode == CTR_OK) rcode = comm_concat(h, all_agg, sizeof(GaucAgg), cnt, goff); }));
    RET(rcode);
    const int g32 = (int)G;
    CU(h, cudaMemcpyAsync(d_u, &g32, sizeof(int), cudaMemcpyHostToDevice, st));
    return gauc_fold(h, all_uniq, all_agg, d_u, (size_t)G, cap, gauc, n_groups, n_used, out_group, out_n, out_pos, out_auc);
}

}  // namespace

// On world > 1 a rank whose arguments are bad still takes part in the agreement with its refusal, so that no rank is
// left waiting; a null handle is refused before anything else.
int ctr_roc_auc_dist(ctr_handle* h, const float* pred, const float* y, int64_t n, double* auc) {
    if (!h) return set_err(h, CTR_EINVAL, "bad auc arguments (null handle)");
    if (h->comm.world == 1) return ctr_roc_auc(h, pred, y, n, auc);
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    h->err.clear();
    const bool ok = auc && n >= 0 && n <= 0x7fffffff && (n == 0 || (pred && y));
    const int verdict = ok ? CTR_OK : set_err(h, CTR_EINVAL, "bad auc_dist arguments (n in [0, 2^31), pred and y non-null when n > 0, auc non-null)");
    int64_t shares[kMaxPeers], total = 0;
    RET(eval_agree(h, 1, verdict, n, shares, &total));
    return auc_dist_ranks(h, pred, y, (long)n, auc);
}

int ctr_group_auc_dist(ctr_handle* h, const float* pred, const float* y, const int64_t* group, int64_t n, double* gauc, int64_t* n_groups,
                       int64_t* n_used, int64_t cap, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_auc) {
    if (!h) return set_err(h, CTR_EINVAL, "bad group auc arguments (null handle)");
    const bool outs = out_group || out_n || out_pos || out_auc;
    if (h->comm.world == 1) {
        if (!pred || !y || !group || !gauc || n < 1 || n > 0x7fffffff)
            return set_err(h, CTR_EINVAL, "bad group auc arguments (n must be in [1, 2^31); pred, y, group and gauc non-null)");
        if (outs && cap < 0) return set_err(h, CTR_EINVAL, "bad group auc arguments (cap %lld < 0)", (long long)cap);
        std::lock_guard<std::mutex> lk(h->mu);
        CU(h, cudaSetDevice(h->dev));
        return gauc_run(h, pred, y, group, (long)n, gauc, n_groups, n_used, cap, out_group, out_n, out_pos, out_auc);
    }
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    h->err.clear();
    const bool ok = gauc && n >= 0 && n <= 0x7fffffff && (n == 0 || (pred && y && group)) && (!outs || cap >= 0);
    const int verdict = ok ? CTR_OK : set_err(h, CTR_EINVAL, "bad group_auc_dist arguments (n in [0, 2^31), pred, y and group non-null when n > 0, "
                                                             "gauc non-null, cap >= 0 with per-group arrays)");
    int64_t shares[kMaxPeers], total = 0;
    RET(eval_agree(h, 2, verdict, n, shares, &total));
    return gauc_dist_ranks(h, pred, y, group, (long)n, gauc, n_groups, n_used, cap, out_group, out_n, out_pos, out_auc);
}
namespace {

// binaryClfCurve on the engine stream (auc.cuh): with check_labels the labels' range and binariness first, then
// ctr_roc_auc's key sort and positive-count scan, the threshold-group ends selected and turned into points.  Leaves
// the points and the summary on the device and the summary in *s.
struct ClfCurve { DevBuf<ClfPoint> pts; DevBuf<ClfSummary> sum; };
int clf_build(ctr_handle* h, const float* pred_h, const float* y_h, long n, double pos_label, bool check_labels,
              ClfCurve& c, ClfSummary* s) {
    cudaStream_t st = h->stream;
    const size_t N = (size_t)n;
    const int grid = (int)std::min<long>((n + 255) / 256, (long)h->num_sms * 8);
    DevBuf<float> d_pred, d_y; DevBuf<unsigned> k0, k1; DevBuf<int> f0, f1, tp, d_m;
    DevBuf<unsigned char> tmp;
    CU(h, d_pred.alloc(N)); CU(h, d_y.alloc(N));
    CU(h, k0.alloc(N)); CU(h, k1.alloc(N)); CU(h, f0.alloc(N)); CU(h, f1.alloc(N)); CU(h, tp.alloc(N));
    CU(h, d_m.alloc(1)); CU(h, c.pts.alloc(N)); CU(h, c.sum.alloc(1));
    int* ends = f0.get();                     // free once the sort has read it
    size_t b[3] = {0, 0, 0};
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b[0], k0.get(), k1.get(), f0.get(), f1.get(), (int)n, 0, 32, st));
    CU(h, cub::DeviceScan::InclusiveSum(nullptr, b[1], f1.get(), tp.get(), (int)n, st));
    CU(h, cub::DeviceSelect::If(nullptr, b[2], thrust::counting_iterator<int>(0), ends, d_m.get(), (int)n, ClfIsEnd{k1.get(), n}, st));
    size_t bytes = std::max(std::max(b[0], b[1]), b[2]);
    CU(h, tmp.alloc(std::max<size_t>(bytes, 1)));
    const ClfSummary init{0, 0, 0, 0, 0, 0, 0xffffffffu, 0u, 0};
    CU(h, cudaMemcpyAsync(c.sum, &init, sizeof init, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_pred, pred_h, N * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_y, y_h, N * sizeof(float), cudaMemcpyHostToDevice, st));
    if (check_labels) {
        RET(launch(h, "ap_label_range", [&] { k_clf_label_range<<<grid, 256, 0, st>>>(d_y, n, c.sum); }));
        RET(launch(h, "ap_label_check", [&] { k_clf_label_check<<<grid, 256, 0, st>>>(d_y, n, c.sum, 0); }));
    }
    RET(launch(h, "clf_keys", [&] { k_clf_keys<<<grid, 256, 0, st>>>(d_pred, d_y, n, pos_label, k0, f0); }));
    RET(launch(h, "clf_sort", [&] {
        cub::DeviceRadixSort::SortPairs(tmp.get(), bytes, k0.get(), k1.get(), f0.get(), f1.get(), (int)n, 0, 32, st); }));
    RET(launch(h, "clf_scan", [&] { cub::DeviceScan::InclusiveSum(tmp.get(), bytes, f1.get(), tp.get(), (int)n, st); }));
    RET(launch(h, "clf_ends", [&] {
        cub::DeviceSelect::If(tmp.get(), bytes, thrust::counting_iterator<int>(0), ends, d_m.get(), (int)n, ClfIsEnd{k1.get(), n}, st); }));
    RET(launch(h, "clf_points", [&] { k_clf_points<<<grid, 256, 0, st>>>(k1, tp, ends, d_m, n, c.pts, c.sum); }));
    CU(h, cudaMemcpyAsync(s, c.sum, sizeof *s, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}

// ctr_roc_curve (roc) or ctr_pr_curve: the points turned into the three arrays on the device; the arrays the caller
// passed come back, and nothing is written when the curve needs more than cap points (*npoints says how many)
int clf_curve_run(ctr_handle* h, bool roc, const float* pred, const float* y, long n, double pos_label,
                  double* a_h, double* b_h, double* thr_h, int64_t cap, int64_t* npoints) {
    ClfCurve c; ClfSummary s{};
    RET(clf_build(h, pred, y, n, pos_label, false, c, &s));
    const long np_ = roc ? (long)s.m + (s.fp0 != 0 ? 1 : 0) : (long)s.last_ind + 2;
    *npoints = np_;
    if (np_ > cap)
        return set_err(h, CTR_EINVAL, "%s curve needs %ld points, cap is %lld", roc ? "roc" : "pr", np_, (long long)cap);
    cudaStream_t st = h->stream;
    const int grid = (int)std::min<long>((np_ + 255) / 256, (long)h->num_sms * 8);
    DevBuf<double> a, b, t;
    CU(h, a.alloc((size_t)np_)); CU(h, b.alloc((size_t)np_)); CU(h, t.alloc((size_t)np_));
    if (roc) RET(launch(h, "clf_roc", [&] { k_clf_roc<<<grid, 256, 0, st>>>(c.pts, c.sum, a, b, t); }));
    else RET(launch(h, "clf_pr", [&] { k_clf_pr<<<grid, 256, 0, st>>>(c.pts, c.sum, a, b, t); }));
    const size_t nt = (size_t)(roc ? np_ : np_ - 1);
    if (a_h) CU(h, cudaMemcpyAsync(a_h, a, (size_t)np_ * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (b_h) CU(h, cudaMemcpyAsync(b_h, b, (size_t)np_ * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (thr_h) CU(h, cudaMemcpyAsync(thr_h, t, nt * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}

}  // namespace

int ctr_roc_curve(ctr_handle* h, const float* pred, const float* y, int64_t n, double pos_label, double* fpr, double* tpr,
                  double* thresholds, int64_t cap, int64_t* npoints) {
    if (!h || !pred || !y || !npoints || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad roc curve arguments (n must be in [1, 2^31); pred, y and npoints non-null)");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return clf_curve_run(h, true, pred, y, (long)n, pos_label, fpr, tpr, thresholds, cap, npoints);
}

int ctr_pr_curve(ctr_handle* h, const float* pred, const float* y, int64_t n, double pos_label, double* precision,
                 double* recall, double* thresholds, int64_t cap, int64_t* npoints) {
    if (!h || !pred || !y || !npoints || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad pr curve arguments (n must be in [1, 2^31); pred, y and npoints non-null)");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return clf_curve_run(h, false, pred, y, (long)n, pos_label, precision, recall, thresholds, cap, npoints);
}

int ctr_average_precision(ctr_handle* h, const float* pred, const float* y, int64_t n, double* ap) {
    if (!h || !pred || !y || !ap || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad average precision arguments (n must be in [1, 2^31); pred, y and ap non-null)");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    ClfCurve c; ClfSummary s{};
    RET(clf_build(h, pred, y, (long)n, 1.0, true, c, &s));
    if (s.other) return set_err(h, CTR_EINVAL, "average precision needs binary labels (every label the lowest or the highest, no NaN)");
    cudaStream_t st = h->stream;
    const int gparts = h->num_sms * 2;
    DevBuf<GaucPart> part; DevBuf<double> d_ap;
    CU(h, part.alloc(gparts)); CU(h, d_ap.alloc(1));
    RET(launch(h, "ap_terms", [&] { k_ap_terms<<<gparts, 256, 0, st>>>(c.pts, c.sum, part); }));
    RET(launch(h, "ap_final", [&] { k_ap_final<<<1, 256, 0, st>>>(part, gparts, c.sum, d_ap); }));
    double r = 0;
    CU(h, cudaMemcpyAsync(&r, d_ap, sizeof r, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    *ap = r;
    return CTR_OK;
}

namespace {

// ctr_group_average_precision: the label check (labels rewritten to pos_label = 1), GAUC's (group, score) order, heads
// and scan, each group's positives, the AP terms, one reduce-by-key of (double-double sum, n, positives) over the
// sorted group keys, then the per-group AP and their mean; only the result and the arrays asked for come back
int gap_run(ctr_handle* h, const float* pred_h, const float* y_h, const int64_t* group_h, long n, double* map,
            int64_t* n_groups, int64_t* n_used, int64_t* out_group, int32_t* out_n, int32_t* out_pos, double* out_ap) {
    cudaStream_t st = h->stream;
    const size_t N = (size_t)n;
    const int grid = (int)std::min<long>((n + 255) / 256, (long)h->num_sms * 8), gparts = h->num_sms * 2;
    DevBuf<float> d_pred, d_y; DevBuf<long long> d_group;
    DevBuf<unsigned> k0, k1; DevBuf<int> i0, i1, d_runs;
    DevBuf<unsigned long long> g0, g1, v0, v1;
    DevBuf<GaucScan> scan; DevBuf<GapAgg> val, agg; DevBuf<GaucPart> part; DevBuf<GaucResult> res; DevBuf<ClfSummary> lab;
    DevBuf<long long> o_group; DevBuf<int> o_n, o_pos; DevBuf<double> o_ap;
    DevBuf<unsigned char> tmp;
    CU(h, d_pred.alloc(N)); CU(h, d_y.alloc(N)); CU(h, d_group.alloc(N));
    CU(h, k0.alloc(N)); CU(h, k1.alloc(N)); CU(h, i0.alloc(N)); CU(h, i1.alloc(N));
    CU(h, g0.alloc(N)); CU(h, g1.alloc(N)); CU(h, v0.alloc(N)); CU(h, v1.alloc(N));
    CU(h, scan.alloc(N)); CU(h, val.alloc(N)); CU(h, agg.alloc(N));
    CU(h, d_runs.alloc(1)); CU(h, part.alloc(gparts)); CU(h, res.alloc(1)); CU(h, lab.alloc(1));
    if (out_group) CU(h, o_group.alloc(N));
    if (out_n) CU(h, o_n.alloc(N));
    if (out_pos) CU(h, o_pos.alloc(N));
    if (out_ap) CU(h, o_ap.alloc(N));
    unsigned long long* uniq = g0.get();     // free once the group pass has read it
    int* gpos = i0.get();                    // free once the score pass has read it
    size_t b[4] = {0, 0, 0, 0};
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b[0], k0.get(), k1.get(), i0.get(), i1.get(), (int)n, 0, 32, st));
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b[1], g0.get(), g1.get(), v0.get(), v1.get(), (int)n, 0, 64, st));
    CU(h, cub::DeviceScan::InclusiveScan(nullptr, b[2], scan.get(), scan.get(), GaucScanOp(), (int)n, st));
    CU(h, cub::DeviceReduce::ReduceByKey(nullptr, b[3], g1.get(), uniq, val.get(), agg.get(), d_runs.get(), GapAggOp(), (int)n, st));
    size_t bytes = std::max(std::max(b[0], b[1]), std::max(b[2], b[3]));
    CU(h, tmp.alloc(std::max<size_t>(bytes, 1)));
    const ClfSummary init{0, 0, 0, 0, 0, 0, 0xffffffffu, 0u, 0};
    CU(h, cudaMemcpyAsync(lab, &init, sizeof init, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_pred, pred_h, N * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_y, y_h, N * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(d_group, group_h, N * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    RET(launch(h, "gap_label_range", [&] { k_clf_label_range<<<grid, 256, 0, st>>>(d_y, n, lab); }));
    RET(launch(h, "gap_label_check", [&] { k_clf_label_check<<<grid, 256, 0, st>>>(d_y, n, lab, 1); }));
    RET(launch(h, "gap_keys", [&] { k_gauc_keys<<<grid, 256, 0, st>>>(d_pred, n, k0, i0); }));
    RET(launch(h, "gap_sort_score", [&] {
        cub::DeviceRadixSort::SortPairs(tmp.get(), bytes, k0.get(), k1.get(), i0.get(), i1.get(), (int)n, 0, 32, st); }));
    RET(launch(h, "gap_gather", [&] { k_gauc_gather<<<grid, 256, 0, st>>>(k1, i1, d_group, d_y, n, g0, v0); }));
    RET(launch(h, "gap_sort_group", [&] {
        cub::DeviceRadixSort::SortPairs(tmp.get(), bytes, g0.get(), g1.get(), v0.get(), v1.get(), (int)n, 0, 64, st); }));
    RET(launch(h, "gap_heads", [&] { k_gauc_heads<<<grid, 256, 0, st>>>(g1, v1, n, scan); }));
    RET(launch(h, "gap_scan", [&] {
        cub::DeviceScan::InclusiveScan(tmp.get(), bytes, scan.get(), scan.get(), GaucScanOp(), (int)n, st); }));
    RET(launch(h, "gap_pos", [&] { k_gap_pos<<<grid, 256, 0, st>>>(g1, scan, n, gpos); }));
    RET(launch(h, "gap_terms", [&] { k_gap_terms<<<grid, 256, 0, st>>>(g1, v1, scan, gpos, n, val); }));
    RET(launch(h, "gap_reduce", [&] {
        cub::DeviceReduce::ReduceByKey(tmp.get(), bytes, g1.get(), uniq, val.get(), agg.get(), d_runs.get(), GapAggOp(), (int)n, st); }));
    RET(launch(h, "gap_groups", [&] { k_gap_groups<<<gparts, 256, 0, st>>>(uniq, agg, d_runs, o_group, o_n, o_pos, o_ap, part); }));
    RET(launch(h, "gap_final", [&] { k_gauc_final<<<1, 256, 0, st>>>(part, gparts, d_runs, res); }));
    GaucResult r{}; ClfSummary ls{};
    CU(h, cudaMemcpyAsync(&r, res, sizeof r, cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(&ls, lab, sizeof ls, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if (ls.other)
        return set_err(h, CTR_EINVAL, "group average precision needs binary labels (every label the lowest or the highest, no NaN)");
    const size_t R = (size_t)r.groups;
    if (out_group) CU(h, cudaMemcpyAsync(out_group, o_group, R * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    if (out_n) CU(h, cudaMemcpyAsync(out_n, o_n, R * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (out_pos) CU(h, cudaMemcpyAsync(out_pos, o_pos, R * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (out_ap) CU(h, cudaMemcpyAsync(out_ap, o_ap, R * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    *map = r.gauc;
    if (n_groups) *n_groups = r.groups;
    if (n_used) *n_used = r.used;
    return CTR_OK;
}

}  // namespace

int ctr_group_average_precision(ctr_handle* h, const float* pred, const float* y, const int64_t* group, int64_t n, double* map,
                                int64_t* n_groups, int64_t* n_used, int64_t* out_group, int32_t* out_n, int32_t* out_pos,
                                double* out_ap) {
    if (!h || !pred || !y || !group || !map || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad group average precision arguments (n must be in [1, 2^31); pred, y, group and map non-null)");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return gap_run(h, pred, y, group, (long)n, map, n_groups, n_used, out_group, out_n, out_pos, out_ap);
}

// ---- nn/metrics classification.go and regression.go (metrics.cuh) -----------------------------------------------
namespace {

int met_grid(const ctr_handle* h, long work) { return (int)std::max<long>(1, std::min<long>((work + 255) / 256, (long)h->num_sms * 8)); }
int met_bits(unsigned long long max_key) { return max_key ? 64 - __builtin_clzll(max_key) : 1; }
constexpr unsigned long long kMetNone = ~0ull;

// The per-class outputs of ctr_precision_recall_fscore (null for ctr_confusion_matrix)
struct MetPrf { double beta; int average, pos_label; double *p, *r, *f, *support, *per_class; };

// ConfusionMatrix and PrecisionRecallFScoreSupport on the engine stream, one pipeline: the classes of y_true
// (class_sort_unique), both label vectors encoded and counted (k_met_encode), with weights the sorted segment sums
// (k_met_seg_*), then the matrix or the scores.  Every refusal comes before any output except *n_classes.
int met_class_run(ctr_handle* h, const char* what, const double* yt_h, const double* yp_h, const double* w_h, long n,
                  double* classes_h, double* cm_h, int64_t cap, int32_t* n_classes, const MetPrf* prf) {
    cudaStream_t st = h->stream;
    const size_t N = (size_t)n;
    const int grid = met_grid(h, n);
    DevBuf<double> yt, yp, w, key0, key1, classes; DevBuf<long> p0, p1, d_count; DevBuf<MetFlags> fl;
    DevBuf<unsigned char> tmp;
    CU(h, yt.alloc(N)); CU(h, yp.alloc(N)); if (w_h) CU(h, w.alloc(N));
    CU(h, key0.alloc(N)); CU(h, key1.alloc(N)); CU(h, p0.alloc(N)); CU(h, p1.alloc(N));
    CU(h, classes.alloc(N)); CU(h, d_count.alloc(1)); CU(h, fl.alloc(1));
    size_t bytes = 0;
    CU(h, class_sort_unique<double>(nullptr, &bytes, nullptr, nullptr, nullptr, nullptr, nullptr, n, st));
    CU(h, tmp.alloc(bytes));
    CU(h, cudaMemcpyAsync(yt, yt_h, N * sizeof(double), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(yp, yp_h, N * sizeof(double), cudaMemcpyHostToDevice, st));
    if (w_h) CU(h, cudaMemcpyAsync(w, w_h, N * sizeof(double), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemsetAsync(fl, 0xff, sizeof(MetFlags), st));
    RET(launch(h, "met_keys", [&] { k_met_keys<<<grid, 256, 0, st>>>(yt, yp, w, n, key0, p0, fl); }));
    RET(launch(h, "met_classes", [&] { class_sort_unique<double>(tmp.get(), &bytes, key0.get(), key1.get(), p0.get(), p1.get(), d_count.get(), n, st); }));
    RET(launch(h, "met_class_values", [&] { k_class_values<double><<<grid, 256, 0, st>>>(yt, p0, d_count, LONG_MAX, classes); }));
    MetFlags f{}; long C = 0;
    CU(h, cudaMemcpyAsync(&f, fl, sizeof f, cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(&C, d_count, sizeof C, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if (f.nan_true != kMetNone) return set_err(h, CTR_EINVAL, "%s: y_true[%llu] is NaN: the classes would be ill-defined", what, f.nan_true);
    *n_classes = (int32_t)C;
    if (f.nan_pred != kMetNone) return set_err(h, CTR_EINVAL, "%s: y_pred[%llu] is NaN", what, f.nan_pred);
    if (f.bad_weight != kMetNone) return set_err(h, CTR_EINVAL, "%s: weight[%llu] = %g is not finite", what, f.bad_weight, w_h[f.bad_weight]);
    if (prf && prf->pos_label >= C) return set_err(h, CTR_EINVAL, "%s: pos_label %d, but y_true has %ld classes", what, prf->pos_label, C);
    if (!prf && C * C > cap) return set_err(h, CTR_EINVAL, "%s: %ld classes need %ld cells, cap is %lld", what, C, C * C, (long long)cap);
    if (prf && prf->per_class && C > cap) return set_err(h, CTR_EINVAL, "%s: %ld classes, cap is %lld", what, C, (long long)cap);
    // LabelEncoder.Transform of both vectors and the unweighted counts
    const long cmc = !prf && cm_h ? C * C : 0;
    DevBuf<unsigned long long> cell, pcls, cm_u, cls_u;
    CU(h, cell.alloc(N)); CU(h, pcls.alloc(N)); CU(h, cls_u.alloc(3 * (size_t)C));
    if (cmc) CU(h, cm_u.alloc((size_t)cmc));
    CU(h, cudaMemsetAsync(cls_u, 0, 3 * (size_t)C * sizeof(unsigned long long), st));
    if (cmc) CU(h, cudaMemsetAsync(cm_u, 0, (size_t)cmc * sizeof(unsigned long long), st));
    const bool sh_cls = C <= kMetSmemClasses, sh_cnt = cmc + 3 * C <= kMetSmemCounts;
    const size_t smem = (sh_cls ? (size_t)C * sizeof(double) : 0) + (sh_cnt ? (size_t)(cmc + 3 * C) * sizeof(unsigned long long) : 0);
    const int Ci = (int)C;
    RET(launch(h, "met_encode", [&] {
        auto k = sh_cls ? (sh_cnt ? k_met_encode<true, true> : k_met_encode<true, false>) : (sh_cnt ? k_met_encode<false, true> : k_met_encode<false, false>);
        k<<<grid, 256, smem, st>>>(yt, yp, n, classes, Ci, cell, pcls, cm_u, cls_u, fl); }));
    CU(h, cudaMemcpyAsync(&f, fl, sizeof f, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if (f.above != kMetNone)
        return set_err(h, CTR_EINVAL, "%s: y_pred[%llu] = %g is above the largest class (the reference writes outside the row)", what, f.above, yp_h[f.above]);
    // weighted sums: (key, weight) sorted, then each segment summed in array order (k_met_seg_*)
    DevBuf<double> cm_w, tp_w, true_w, pred_w;
    if (w_h) {
        DevBuf<unsigned long long> ks; DevBuf<double> ws; DevBuf<double2> piece; DevBuf<long> heads; DevBuf<int> nheads;
        DevBuf<unsigned char> tmp2;
        CU(h, ks.alloc(N)); CU(h, ws.alloc(N)); CU(h, piece.alloc(N)); CU(h, heads.alloc(N)); CU(h, nheads.alloc(1));
        size_t b[2] = {0, 0};
        CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b[0], cell.get(), ks.get(), w.get(), ws.get(), (int)n, 0, 64, st));
        CU(h, cub::DeviceSelect::If(nullptr, b[1], thrust::counting_iterator<long>(0), heads.get(), nheads.get(), (int)n, MetSegHead{ks.get(), 1}, st));
        size_t b2 = std::max<size_t>(std::max(b[0], b[1]), 1);
        CU(h, tmp2.alloc(b2));
        auto seg = [&](unsigned long long div, double* out, double* diag) -> int {
            RET(launch(h, "met_seg_piece", [&] { k_met_seg_piece<<<grid, 256, 0, st>>>(ks, div, ws, n, piece); }));
            RET(launch(h, "met_seg_heads", [&] {
                cub::DeviceSelect::If(tmp2.get(), b2, thrust::counting_iterator<long>(0), heads.get(), nheads.get(), (int)n, MetSegHead{ks.get(), div}, st); }));
            return launch(h, "met_seg_total", [&] { k_met_seg_total<<<grid, 256, 0, st>>>(ks, div, heads, nheads, n, piece, Ci, out, diag); });
        };
        RET(launch(h, "met_sort_cells", [&] {
            cub::DeviceRadixSort::SortPairs(tmp2.get(), b2, cell.get(), ks.get(), w.get(), ws.get(), (int)n, 0, met_bits((unsigned long long)C * C - 1), st); }));
        if (cmc) {
            CU(h, cm_w.alloc((size_t)cmc)); CU(h, cudaMemsetAsync(cm_w, 0, (size_t)cmc * sizeof(double), st));
            RET(seg(1, cm_w, nullptr));
        }
        if (prf) {
            CU(h, tp_w.alloc((size_t)C)); CU(h, true_w.alloc((size_t)C)); CU(h, pred_w.alloc((size_t)C));
            for (double* a : {tp_w.get(), true_w.get(), pred_w.get()}) CU(h, cudaMemsetAsync(a, 0, (size_t)C * sizeof(double), st));
            RET(seg(1, nullptr, tp_w));
            RET(seg((unsigned long long)C, true_w, nullptr));
            RET(launch(h, "met_sort_cols", [&] {
                cub::DeviceRadixSort::SortPairs(tmp2.get(), b2, pcls.get(), ks.get(), w.get(), ws.get(), (int)n, 0, met_bits((unsigned long long)C - 1), st); }));
            RET(seg(1, pred_w, nullptr));
        }
    }
    double r4[4] = {0, 0, 0, 0};
    DevBuf<double> out4, pc;
    if (!prf) {
        if (cmc && !w_h) {
            CU(h, cm_w.alloc((size_t)cmc));
            RET(launch(h, "met_cm", [&] { k_met_cm_f64<<<met_grid(h, cmc), 256, 0, st>>>(cm_u, cmc, cm_w); }));
        }
        if (cmc) CU(h, cudaMemcpyAsync(cm_h, cm_w, (size_t)cmc * sizeof(double), cudaMemcpyDeviceToHost, st));
    } else {
        CU(h, out4.alloc(4));
        if (prf->per_class) CU(h, pc.alloc(4 * (size_t)C));
        RET(launch(h, "met_prf", [&] {
            k_met_prf<<<1, 256, 0, st>>>(cls_u, tp_w, true_w, pred_w, Ci, prf->beta, prf->pos_label, prf->average, pc, out4); }));
        CU(h, cudaMemcpyAsync(r4, out4, sizeof r4, cudaMemcpyDeviceToHost, st));
        if (prf->per_class) CU(h, cudaMemcpyAsync(prf->per_class, pc, 4 * (size_t)C * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    if (classes_h) CU(h, cudaMemcpyAsync(classes_h, classes, (size_t)C * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if (prf) {
        if (prf->p) *prf->p = r4[0];
        if (prf->r) *prf->r = r4[1];
        if (prf->f) *prf->f = r4[2];
        if (prf->support) *prf->support = r4[3];
    }
    return CTR_OK;
}

// R2Score (kind < 0) or MeanSquaredError / MeanAbsoluteError on the engine stream: k_mlp64_r2_part / k_mlp64_r2_fold
// over the [n, no] host matrices; out receives no values (RAW) or one
int met_regression_run(ctr_handle* h, const double* yt_h, const double* yp_h, const double* w_h, long n, int no, int kind,
                       int multioutput, double* out_h) {
    cudaStream_t st = h->stream;
    const size_t NN = (size_t)n * (size_t)no;
    DevBuf<double> yt, yp, w, mean, r, res; DevBuf<double2> part;
    CU(h, yt.alloc(NN)); CU(h, yp.alloc(NN)); if (w_h) CU(h, w.alloc((size_t)n));
    CU(h, mean.alloc((size_t)no)); CU(h, r.alloc(2 * (size_t)no)); CU(h, res.alloc(3)); CU(h, part.alloc((size_t)no * kR2Parts));
    CU(h, cudaMemcpyAsync(yt, yt_h, NN * sizeof(double), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(yp, yp_h, NN * sizeof(double), cudaMemcpyHostToDevice, st));
    if (w_h) CU(h, cudaMemcpyAsync(w, w_h, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
    const dim3 g(kR2Parts, no);
    const double* raw = mean;
    if (kind < 0) {
        RET(launch(h, "r2_mean", [&] { k_mlp64_r2_part<double><<<g, 256, 0, st>>>(nullptr, yt, w, n, no, kR2Mean, nullptr, part); }));
        RET(launch(h, "r2_mean_fold", [&] { k_mlp64_r2_fold<<<1, 256, 0, st>>>(part, no, 0.0, mean, nullptr, nullptr); }));
        RET(launch(h, "r2_sums", [&] { k_mlp64_r2_part<double><<<g, 256, 0, st>>>(yp, yt, w, n, no, kR2Sums, mean, part); }));
        RET(launch(h, "r2_fold", [&] { k_mlp64_r2_fold<<<1, 256, 0, st>>>(part, no, 1e-20, mean, r, res); }));
        raw = r;
    } else {
        const int k = kind == CTR_ERROR_SQUARED ? kErrSquared : kErrAbsolute;
        RET(launch(h, "err_sums", [&] { k_mlp64_r2_part<double><<<g, 256, 0, st>>>(yp, yt, nullptr, n, no, k, nullptr, part); }));
        RET(launch(h, "err_fold", [&] { k_mlp64_r2_fold<<<1, 256, 0, st>>>(part, no, 0.0, mean, nullptr, res); }));
    }
    if (multioutput == CTR_MULTIOUTPUT_RAW) CU(h, cudaMemcpyAsync(out_h, raw, (size_t)no * sizeof(double), cudaMemcpyDeviceToHost, st));
    else CU(h, cudaMemcpyAsync(out_h, res.get() + (multioutput == CTR_MULTIOUTPUT_UNIFORM ? 0 : 2), sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}

}  // namespace

// The arguments are checked before the handle, so each refusal's message is readable through ctr_last_error(h), or
// ctr_last_error(NULL) when h is null.
int ctr_accuracy_score(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, int32_t n_out, const double* weight,
                       int32_t normalize, double* score) {
    if (!y_true || !y_pred || !score || n < 1 || n > 0x7fffffff || n_out < 1 || n_out > 1024)
        return set_err(h, CTR_EINVAL, "bad accuracy arguments (n in [1, 2^31), n_out in [1, 1024]; y_true, y_pred and score non-null)");
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    cudaStream_t st = h->stream;
    const size_t NN = (size_t)n * (size_t)n_out;
    DevBuf<double> yt, yp, w, out; DevBuf<MetAccPart> part;
    CU(h, yt.alloc(NN)); CU(h, yp.alloc(NN)); if (weight) CU(h, w.alloc((size_t)n));
    CU(h, out.alloc(2)); CU(h, part.alloc(kMetParts));
    CU(h, cudaMemcpyAsync(yt, y_true, NN * sizeof(double), cudaMemcpyHostToDevice, st));
    CU(h, cudaMemcpyAsync(yp, y_pred, NN * sizeof(double), cudaMemcpyHostToDevice, st));
    if (weight) CU(h, cudaMemcpyAsync(w, weight, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
    RET(launch(h, "acc_part", [&] { k_met_acc_part<<<kMetParts, 256, 0, st>>>(yt, yp, w, (long)n, n_out, part); }));
    RET(launch(h, "acc_final", [&] { k_met_acc_final<<<1, 256, 0, st>>>(part, (long)n, weight != nullptr, normalize, out); }));
    double r[2] = {0, 0};
    CU(h, cudaMemcpyAsync(r, out, sizeof r, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if (r[1] != 0.0) return set_err(h, CTR_EINVAL, "accuracy: a weight is NaN or infinite");
    *score = r[0];
    return CTR_OK;
}

int ctr_confusion_matrix(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, const double* weight, double* classes,
                         double* cm, int64_t cap, int32_t* n_classes) {
    if (!y_true || !y_pred || !n_classes || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad confusion matrix arguments (n in [1, 2^31); y_true, y_pred and n_classes non-null)");
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return met_class_run(h, "confusion matrix", y_true, y_pred, weight, (long)n, classes, cm, cap, n_classes, nullptr);
}

int ctr_precision_recall_fscore(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, const double* weight, double beta,
                                int32_t average, int32_t pos_label, double* p, double* r, double* f, double* support,
                                double* per_class, int64_t cap, int32_t* n_classes) {
    if (!y_true || !y_pred || !n_classes || n < 1 || n > 0x7fffffff)
        return set_err(h, CTR_EINVAL, "bad precision/recall arguments (n in [1, 2^31); y_true, y_pred and n_classes non-null)");
    if (average != CTR_AVERAGE_MACRO && average != CTR_AVERAGE_MICRO && average != CTR_AVERAGE_WEIGHTED)
        return set_err(h, CTR_EINVAL, "average %d: macro (%d), micro (%d) or weighted (%d)", average, CTR_AVERAGE_MACRO, CTR_AVERAGE_MICRO, CTR_AVERAGE_WEIGHTED);
    if (!std::isfinite(beta)) return set_err(h, CTR_EINVAL, "beta %g must be finite", beta);
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    const MetPrf prf{beta, average, pos_label < 0 ? -1 : pos_label, p, r, f, support, per_class};
    return met_class_run(h, "precision/recall", y_true, y_pred, weight, (long)n, nullptr, nullptr, cap, n_classes, &prf);
}

int ctr_r2_score(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, int32_t n_out, const double* weight,
                 int32_t multioutput, double* out) {
    if (!y_true || !y_pred || !out || n < 1 || n > 0x7fffffff || n_out < 1 || n_out > 1024)
        return set_err(h, CTR_EINVAL, "bad r2 arguments (n in [1, 2^31), n_out in [1, 1024]; y_true, y_pred and out non-null)");
    if (multioutput != CTR_MULTIOUTPUT_RAW && multioutput != CTR_MULTIOUTPUT_UNIFORM && multioutput != CTR_MULTIOUTPUT_VARIANCE_WEIGHTED)
        return set_err(h, CTR_EINVAL, "multioutput %d: raw (%d), uniform (%d) or variance weighted (%d)", multioutput,
                       CTR_MULTIOUTPUT_RAW, CTR_MULTIOUTPUT_UNIFORM, CTR_MULTIOUTPUT_VARIANCE_WEIGHTED);
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return met_regression_run(h, y_true, y_pred, weight, (long)n, n_out, -1, multioutput, out);
}

int ctr_mean_error(ctr_handle* h, const double* y_true, const double* y_pred, int64_t n, int32_t n_out, int32_t kind,
                   int32_t multioutput, double* out) {
    if (!y_true || !y_pred || !out || n < 1 || n > 0x7fffffff || n_out < 1 || n_out > 1024)
        return set_err(h, CTR_EINVAL, "bad mean error arguments (n in [1, 2^31), n_out in [1, 1024]; y_true, y_pred and out non-null)");
    if (kind != CTR_ERROR_SQUARED && kind != CTR_ERROR_ABSOLUTE)
        return set_err(h, CTR_EINVAL, "kind %d: squared (%d) or absolute (%d)", kind, CTR_ERROR_SQUARED, CTR_ERROR_ABSOLUTE);
    if (multioutput != CTR_MULTIOUTPUT_RAW && multioutput != CTR_MULTIOUTPUT_UNIFORM)
        return set_err(h, CTR_EINVAL, "multioutput %d: raw (%d) or uniform (%d); the mean errors have no variance weighting", multioutput,
                       CTR_MULTIOUTPUT_RAW, CTR_MULTIOUTPUT_UNIFORM);
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return met_regression_run(h, y_true, y_pred, nullptr, (long)n, n_out, kind, multioutput, out);
}

int ctr_knn_search(ctr_handle* h, const double* queries, const int32_t* query_rows, int64_t nq, int32_t k,
                   int32_t* out_rows, double* out_sim, int32_t* out_count) {
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    const int T = CTR_TABLE_ITEM_EMB;
    // a row-sharded ITEM_EMB makes the call collective: every rank scans its shard, the ranks' lists are merged
    const bool coll = emb_sharded(h);
    const int W = coll ? h->comm.world : 1;
    const bool by_row = queries == nullptr;
    CU(h, cudaSetDevice(h->dev));        // before any CUDA call, the agreement's lazy staging buffer included
    const bool args_ok = !(k < 1 || k > knn::kMaxK || nq < 1 || (!queries && !query_rows) || !out_rows || !out_sim || !out_count);
    const int verdict = [&]() -> int {
        if (!args_ok)
            return set_err(h, CTR_EINVAL, "bad knn arguments (k in [1, %d], nq >= 1, queries or query_rows, non-null outputs)", knn::kMaxK);
        if (!h->tab[T]) return set_err(h, CTR_ESTATE, "ITEM_EMB table not uploaded");
        if (coll) RET(comm_check_emb(h));
        const int64_t N = h->tab_rows[T];
        if (N > INT32_MAX) return set_err(h, CTR_ESTATE, "ITEM_EMB has %lld rows: row ids are int32", (long long)N);
        if (query_rows) for (int64_t i = 0; i < nq; i++) {
            const int32_t r = query_rows[i];
            if (by_row && (r < 0 || r >= N)) return set_err(h, CTR_ENOTFOUND, "%d is not found in searcher", r);     // search.go:75-77
            if (!by_row && (r < -1 || r >= N)) return set_err(h, CTR_EINVAL, "excluded row %d of query %lld outside [-1, %lld)", r, (long long)i, (long long)N);
        }
        return CTR_OK;
    }();
    // the call's header: the arguments are hashed whenever they are well-formed, whatever this rank's state, so a rank
    // whose state check fails still agrees with the others and its verdict reaches them
    CommHdr hd{};
    hd.n = nq; hd.k = k; hd.mode = (queries ? 1 : 0) | (query_rows ? 2 : 0);
    if (coll && args_ok) {
        if (queries) hd.hash[0] = comm_hash(queries, (size_t)nq * h->cfg.D * sizeof(double));
        if (query_rows) hd.hash[1] = comm_hash(query_rows, (size_t)nq * sizeof(int32_t));
    }
    const int64_t N = h->tab_local_rows[T];   // the rows this rank scans
    const int D = h->tab_width[T], Dp = (D + 3) & ~3;
    // Row queries on a shard: the query rows are gathered (hot rows from the replica, the others from their owners)
    // and widened to float64, then scanned as vector queries that exclude their own row.  A product of two widened
    // floats is exact in float64, so the unfused sums of the vector instantiation equal the fused ones of ROWQ bit for bit.
    const bool rowq = by_row && !coll;
    const int gw = coll ? W : 0;
    const size_t msmem = knn::smem_bytes<knn::SimKey>(1, 0, k);
    // the plan, made only when this rank's checks passed (the agreement reads it only when every rank's did)
    int QT = 16, slices = 1;
    int64_t chunk = 0;
    long rps = 0;
    size_t smem = 0;
    if (verdict == CTR_OK) {
        // query tile: as wide as the batch needs, narrower when k's lists would not fit shared memory
        while (QT > 1 && (QT / 2 >= nq || knn::kTileBytes + knn::smem_bytes<knn::SimKey>(QT, Dp, k) > ((size_t)200 << 10))) QT /= 2;
        smem = knn::kTileBytes + knn::smem_bytes<knn::SimKey>(QT, Dp, k);
        int occ = 1;      // also sets the instantiation's shared-memory limit
        if (rowq) knn_scan_dispatch<true>(h, QT, KnnArgs{}, true, smem, &occ); else knn_scan_dispatch<false>(h, QT, KnnArgs{}, true, smem, &occ);
        // row slices: enough CTAs to fill the GPU with the least idle tail (whole waves of resident CTAs); queries are
        // chunked so that the slices' lists (and on a sharded table the ranks' gathered lists) stay within 256 MB of scratch
        // On a shard the plan is made for the largest shard (rank 0's), so that every rank picks the same query chunk and
        // the ranks' all-gathers match.
        const int64_t Nplan = coll ? (h->tab_rows[T] + W - 1) / W : N;
        const long steps = std::max<long>(1, (long)((Nplan + knn::kStep - 1) / knn::kStep));
        const long wave = (long)h->num_sms * occ;
        chunk = std::min<int64_t>(nq, 1024);
        for (;;) {
            const long tiles = (long)((chunk + QT - 1) / QT);
            double best = -1;
            for (long m = 1; m <= 8; m++) {
                const long s = std::max<long>(1, std::min<long>({(m * wave + tiles - 1) / tiles, steps, 4096}));
                const double w = (double)(s * tiles) / wave, eff = w / std::ceil(w);
                if (eff > best + 0.02) { best = eff; slices = (int)s; }
            }
            if (chunk == 1 || (size_t)chunk * (slices + gw) * k * 12 <= ((size_t)256 << 20)) break;
            chunk = (chunk + 1) / 2;
        }
        rps = (steps + slices - 1) / slices * knn::kStep;
        slices = (int)std::max<int64_t>(1, (N + rps - 1) / rps);     // an empty shard still writes (empty) lists
    }
    if (!coll) RET(verdict);
    else {
        hd.plan = chunk;                 // the number of list all-gathers follows from it: checked, not assumed equal
        RET(comm_serve_enter(h, hd, verdict));
    }

    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t b_q = al((size_t)chunk * D * 8), b_r = al((size_t)chunk * 4), b_ls = al((size_t)chunk * slices * k * 8),
                 b_lr = al((size_t)chunk * slices * k * 4), b_os = al((size_t)chunk * k * 8), b_or = al((size_t)chunk * k * 4), b_oc = al((size_t)chunk * 4),
                 b_gs = al((size_t)chunk * gw * k * 8), b_gr = al((size_t)chunk * gw * k * 4);
    char* base = nullptr;
    RET(scratch_get(h, 3, b_q + b_r + b_ls + b_lr + b_os + b_or + b_oc + b_gs + b_gr, (void**)&base));
    double* d_q = (double*)base; int* d_r = (int*)(base + b_q);
    double* d_ls = (double*)(base + b_q + b_r); int* d_lr = (int*)(base + b_q + b_r + b_ls);
    double* d_os = (double*)(base + b_q + b_r + b_ls + b_lr); int* d_or = (int*)(base + b_q + b_r + b_ls + b_lr + b_os);
    int* d_oc = (int*)(base + b_q + b_r + b_ls + b_lr + b_os + b_or);
    double* d_gs = (double*)(base + b_q + b_r + b_ls + b_lr + b_os + b_or + b_oc);      // [W][n][k] the ranks' lists
    int* d_gr = (int*)(base + b_q + b_r + b_ls + b_lr + b_os + b_or + b_oc + b_gs);

    for (int64_t s = 0; s < nq; s += chunk) {
        const int n = (int)std::min<int64_t>(chunk, nq - s);
        if (!by_row) CU(h, cudaMemcpyAsync(d_q, queries + s * D, (size_t)n * D * sizeof(double), cudaMemcpyHostToDevice, h->stream));
        if (query_rows) CU(h, cudaMemcpyAsync(d_r, query_rows + s, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
        if (by_row && coll) {
            const RowSrc src = comm_src(h, nullptr, nullptr, nullptr, 0, false);
            const int gg = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)n * D + 255) / 256, (int64_t)h->num_sms * 4));
            RET(launch(h, "knn_gather_rows", [&] { k_gather_rows_f64<<<gg, 256, 0, h->stream>>>(src, d_r, n, D, d_q); }));
        }
        const KnnArgs a{rowq ? nullptr : d_q, rowq ? d_r : nullptr, (!rowq && query_rows) ? d_r : nullptr, n, k, rps, slices, d_ls, d_lr};
        RET(launch(h, "knn_scan", [&] {
            int unused = 0;
            if (rowq) knn_scan_dispatch<true>(h, QT, a, false, smem, &unused); else knn_scan_dispatch<false>(h, QT, a, false, smem, &unused);
        }));
        const long sk = (long)slices * k;
        // this rank's lists, then on a shard every rank's
        RET(launch(h, "knn_merge", [&] {
            knn::k_knn_merge<knn::SimKey><<<n, knn::kThreads, msmem, h->stream>>>(d_ls, d_lr, slices, k, sk, k, d_or, d_os, coll ? nullptr : d_oc);
        }));
        if (coll) RET(merge_rank_lists<knn::SimKey>(h, "knn_merge_ranks", d_os, d_or, d_gs, d_gr, n, k, msmem, d_oc));
        CU(h, cudaMemcpyAsync(out_rows + s * k, d_or, (size_t)n * k * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaMemcpyAsync(out_sim + s * k, d_os, (size_t)n * k * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaMemcpyAsync(out_count + s, d_oc, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    }
    return CTR_OK;
}

int ctr_recommend_topk(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, int64_t nu, int32_t k, int32_t exclude_history,
                       int32_t* out_rows, float* out_scores, float* out_logits, int32_t* out_count) {
    return ctr_recommend_topk_ex(h, user_rows, hist_rows, nullptr, nu, k, exclude_history ? CTR_EXCLUDE_WINDOW : CTR_EXCLUDE_NONE, out_rows, out_scores,
                                 out_logits, out_count);
}

int ctr_recommend_topk_ex(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, const int64_t* max_ts, int64_t nu, int32_t k,
                          int32_t exclude, int32_t* out_rows, float* out_scores, float* out_logits, int32_t* out_count) {
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    const int T = CTR_TABLE_ITEM_EMB;
    // a row-sharded ITEM_EMB makes the call collective: every rank scores its shard, the ranks' lists are merged
    const bool coll = emb_sharded(h);
    const int W = coll ? h->comm.world : 1;
    const int S = h->cfg.S, Bc = h->Bmax;
    AttnRecScore sc{h, coll};
    CU(h, cudaSetDevice(h->dev));        // before any CUDA call, the agreement's lazy staging buffer included
    const bool args_ok = !(k < 1 || k > knn::kMaxK || nu < 1 || !user_rows || !hist_rows || !out_rows || !out_scores || !out_count) &&
                         exclude_ok(exclude, max_ts);
    const int verdict = args_ok ? sc.check()
                                : set_err(h, CTR_EINVAL, "bad recommend arguments (k in [1, %d], nu >= 1, user and history rows, non-null outputs, "
                                                         "exclude in [0, 2], max_ts under CTR_EXCLUDE_SEEN)", knn::kMaxK);
    if (!coll) RET(verdict);
    else {
        // the arguments are hashed whenever they are well-formed, whatever this rank's state (see ctr_knn_search)
        CommHdr hd{};
        hd.n = nu; hd.k = k; hd.flag = exclude;
        if (args_ok) {
            hd.hash[0] = comm_hash(user_rows, (size_t)nu * sizeof(int32_t));
            hd.hash[1] = comm_hash(hist_rows, (size_t)nu * S * sizeof(int32_t));
            if (exclude == CTR_EXCLUDE_SEEN) hd.hash[2] = comm_hash(max_ts, (size_t)nu * sizeof(int64_t));
            hd.plan = std::min<int64_t>(nu, 256);      // users per list all-gather (G below)
        }
        RET(comm_serve_enter(h, hd, verdict));
    }
    const int64_t N = h->tab_local_rows[T];   // the items this rank scores
    sc.prepare();
    const bool seen = exclude == CTR_EXCLUDE_SEEN;
    RecTopk<knn::LogitKey> sel{h, "rec", k, exclude == CTR_EXCLUDE_WINDOW ? S : 0, W, coll ? h->comm.rank : 0, N, Bc, seen, h->tab_rows[T]};
    const int64_t G = std::min<int64_t>(nu, 256);          // users per result copy
    int* d_hist;
    RET(sel.setup(4, G, [&](Carve& c) { d_hist = c.take<int>((size_t)G * S); }));
    for (int64_t g0 = 0; g0 < nu; g0 += G) {
        const int ng = (int)std::min<int64_t>(G, nu - g0);
        if (S > 0) CU(h, cudaMemcpyAsync(d_hist, hist_rows + g0 * S, (size_t)ng * S * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
        for (int j = 0; j < ng; j++) {
            const int user = user_rows[g0 + j];
            const int* uh = d_hist + (size_t)j * S;
            RET(sel.user(j, uh, sc.z(), [&](int i0, int nb) { return sc.chunk(user, uh, i0, nb); }, user, seen ? max_ts[g0 + j] : 0));
        }
        RET(sel.finish(g0, ng, out_rows, out_scores, out_logits, out_count, [](long) {}));
    }
    return CTR_OK;
}

int ctr_rank_items(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, const int32_t* item_rows, int64_t n,
                   int32_t exclude_history, int64_t* out_rank, float* out_logit) {
    return ctr_rank_items_ex(h, user_rows, hist_rows, nullptr, item_rows, n, exclude_history ? CTR_EXCLUDE_WINDOW : CTR_EXCLUDE_NONE, out_rank, out_logit);
}

int ctr_rank_items_ex(ctr_handle* h, const int32_t* user_rows, const int32_t* hist_rows, const int64_t* max_ts, const int32_t* item_rows, int64_t n,
                      int32_t exclude, int64_t* out_rank, float* out_logit) {
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    std::lock_guard<std::mutex> lk(h->mu);
    const int T = CTR_TABLE_ITEM_EMB;
    // a row-sharded ITEM_EMB makes the call collective: every rank counts its shard, the ranks' counts are summed
    const bool coll = emb_sharded(h);
    const int W = coll ? h->comm.world : 1;
    const int S = h->cfg.S, Bc = h->Bmax;
    AttnRecScore sc{h, coll};
    CU(h, cudaSetDevice(h->dev));        // before any CUDA call, the agreement's lazy staging buffer included
    const bool args_ok = !(n < 1 || !user_rows || !hist_rows || !item_rows || !out_rank) && exclude_ok(exclude, max_ts);
    const bool seen = exclude == CTR_EXCLUDE_SEEN;
    const int verdict = args_ok ? sc.check()
                                : set_err(h, CTR_EINVAL, "bad rank arguments (n >= 1, user, history and item rows, non-null out_rank, exclude in [0, 2], "
                                                         "max_ts under CTR_EXCLUDE_SEEN)");
    // keys with the same user row and window (and under CTR_EXCLUDE_SEEN the same cut) share a pass
    std::vector<std::vector<int64_t>> passes;
    if (args_ok)
        passes = rank_passes(n, [&](int64_t i) {
            std::vector<int> k(hist_rows + i * S, hist_rows + (i + 1) * S);
            k.push_back(user_rows[i]);
            return std::make_pair(k, seen ? max_ts[i] : (int64_t)0);
        });
    if (!coll) RET(verdict);
    else {
        // the arguments are hashed whenever they are well-formed, whatever this rank's state (see ctr_knn_search)
        CommHdr hd{};
        hd.n = n; hd.flag = exclude;
        if (args_ok) {
            hd.hash[0] = comm_hash(user_rows, (size_t)n * sizeof(int32_t));
            hd.hash[1] = comm_hash(hist_rows, (size_t)n * S * sizeof(int32_t));
            hd.hash[2] = comm_hash(item_rows, (size_t)n * sizeof(int32_t));
            if (seen) hd.hash[2] = comm_hash(max_ts, (size_t)n * sizeof(int64_t), hd.hash[2]);      // the cuts, chained
            hd.plan = (int64_t)passes.size();            // two collectives per pass
        }
        RET(comm_serve_enter(h, hd, verdict));
    }
    const int64_t N = h->tab_local_rows[T];   // the items this rank scores
    sc.prepare();
    RecRank<knn::LogitKey> rk{h, "rank", exclude == CTR_EXCLUDE_WINDOW ? S : 0, N, Bc, W, coll ? h->comm.rank : 0, h->tab_rows[T], seen};
    int* d_hist;
    RET(rk.setup(4, [&](Carve& c) { d_hist = c.take<int>((size_t)S); }));
    std::vector<int64_t> rank((size_t)n); std::vector<float> logit((size_t)n), pl(knn::kMaxK);
    std::vector<int> trow(knn::kMaxK); std::vector<int64_t> pr(knn::kMaxK);
    for (const auto& p : passes) {
        const int64_t i = p[0];
        const int user = user_rows[i], m = (int)p.size();
        for (int j = 0; j < m; j++) trow[j] = item_rows[p[j]];
        if (S > 0) CU(h, cudaMemcpyAsync(d_hist, hist_rows + i * S, (size_t)S * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
        RET(rk.pass(trow.data(), m, d_hist, sc.z(), [&](int i0, int nb) { return sc.chunk(user, d_hist, i0, nb); }, pr.data(), pl.data(), user,
                    seen ? max_ts[i] : 0));
        for (int j = 0; j < m; j++) { rank[(size_t)p[j]] = pr[j]; logit[(size_t)p[j]] = pl[j]; }
    }
    memcpy(out_rank, rank.data(), sizeof(int64_t) * (size_t)n);
    if (out_logit) memcpy(out_logit, logit.data(), sizeof(float) * (size_t)n);
    return CTR_OK;
}

int ctr_rank_metrics(const int64_t* rank, const int64_t* group, int64_t n, const int32_t* ks, int32_t nks,
                     double* hit, double* recall, double* ndcg, double* mrr) {
    if (!rank || !group || !ks || n < 1 || nks < 1) return set_err(nullptr, CTR_EINVAL, "bad rank metric arguments (n >= 1, nks >= 1, non-null rank, group and ks)");
    for (int a = 0; a < nks; a++)
        if (ks[a] < 1) return set_err(nullptr, CTR_EINVAL, "k = %d: every k must be >= 1", ks[a]);
    for (int64_t i = 0; i < n; i++)
        if (rank[i] == 0 || rank[i] < -1) return set_err(nullptr, CTR_EINVAL, "rank[%lld] = %lld: a rank is >= 1, or -1 for a miss", (long long)i, (long long)rank[i]);
    // groups in order of first appearance, their keys in input order
    std::map<int64_t, size_t> gid;
    std::vector<std::vector<int64_t>> gk;
    for (int64_t i = 0; i < n; i++) {
        auto it = gid.emplace(group[i], gk.size()).first;
        if (it->second == gk.size()) gk.emplace_back();
        gk[it->second].push_back(rank[i]);
    }
    const double G = (double)gk.size();
    for (int a = 0; a < nks; a++) {
        const int64_t k = ks[a];
        NeumaierSum h_sum, r_sum, n_sum;
        for (const auto& g : gk) {
            NeumaierSum dcg, idcg;
            int64_t hits = 0;
            for (const int64_t r : g)
                if (r > 0 && r <= k) { hits++; dcg.add(1.0 / std::log2((double)r + 1.0)); }
            for (int64_t j = 1; j <= std::min<int64_t>((int64_t)g.size(), k); j++) idcg.add(1.0 / std::log2((double)j + 1.0));
            h_sum.add((double)hits);
            r_sum.add((double)hits / (double)g.size());
            n_sum.add(dcg.value() / idcg.value());
        }
        if (hit) hit[a] = h_sum.value() / (double)n;
        if (recall) recall[a] = r_sum.value() / G;
        if (ndcg) ndcg[a] = n_sum.value() / G;
    }
    if (mrr) {
        NeumaierSum s;
        for (int64_t i = 0; i < n; i++)
            if (rank[i] > 0) s.add(1.0 / (double)rank[i]);
        *mrr = s.value() / (double)n;
    }
    return CTR_OK;
}

int ctr_i2v_paths(const int64_t* count, int32_t V, int32_t max_depth, int64_t* path_off, int32_t* path_node, uint8_t* path_code, int64_t cap) {
    if (!count || !path_off || V < 2 || max_depth < 2) return set_err(nullptr, CTR_EINVAL, "bad item2vec path arguments");
    std::vector<int64_t> cnt(count, count + V), node_val; std::vector<long long> poff; std::vector<int> pnode; std::vector<unsigned char> pcode;
    i2v_build_paths(cnt, V, max_depth, node_val, poff, pnode, pcode);
    for (int i = 0; i <= V; i++) path_off[i] = poff[(size_t)i];
    if ((int64_t)pnode.size() > cap) return set_err(nullptr, CTR_EINVAL, "path buffers too small: need %lld", (long long)pnode.size());
    if (path_node) memcpy(path_node, pnode.data(), sizeof(int) * pnode.size());
    if (path_code) memcpy(path_code, pcode.data(), pcode.size());
    return CTR_OK;
}

void ctr_i2v_config_default(ctr_i2v_config* c) {
    memset(c, 0, sizeof *c);
    c->dim = 16; c->window = 5; c->iter = 1;                  // rcmd.go:22-26, 543
    c->min_count = 5; c->max_depth = 100;                      // options.go:47-48
    c->init_lr = 0.025f; c->min_lr = 0.025f * 1.0e-4f; c->subsample = 1.0e-3f; c->update_lr_batch = 100000;
    c->seed = 0; c->device = 0;
}

namespace {
// Large transfers between PAGEABLE caller memory and the device (item2vec: the token stream in, the vector table out):
// two pinned bounce buffers, host-side memcpy by the copy pool overlapping the DMA of the other buffer.
cudaError_t big_copy(void* dst, const void* src, size_t bytes, bool to_device, cudaStream_t st) {
    const size_t kChunk = (size_t)32 << 20;
    if (bytes < ((size_t)8 << 20)) { cudaError_t e = cudaMemcpyAsync(dst, src, bytes, to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, st); return e != cudaSuccess ? e : cudaStreamSynchronize(st); }
    PinnedBuf<unsigned char> pin[2]; Event ev[2];
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 2 && e == cudaSuccess; i++) { e = pin[i].alloc(kChunk); if (e == cudaSuccess) e = ev[i].create(cudaEventDisableTiming); }
    if (e == cudaSuccess) {
        CopyPool pool(7);
        const size_t nchunks = (bytes + kChunk - 1) / kChunk;
        if (to_device) {
            for (size_t c = 0; c < nchunks && e == cudaSuccess; c++) {
                const int b = (int)(c & 1); const size_t off = c * kChunk, m = std::min(kChunk, bytes - off);
                if (c >= 2) e = cudaEventSynchronize(ev[b]);
                pool.copy(pin[b], (const char*)src + off, m);
                if (e == cudaSuccess) e = cudaMemcpyAsync((char*)dst + off, pin[b], m, cudaMemcpyHostToDevice, st);
                if (e == cudaSuccess) e = cudaEventRecord(ev[b], st);
            }
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        } else {
            // DMA chunk c+1 while the pool copies chunk c out of its bounce buffer
            if (nchunks > 0) { e = cudaMemcpyAsync(pin[0], src, std::min(kChunk, bytes), cudaMemcpyDeviceToHost, st); if (e == cudaSuccess) e = cudaEventRecord(ev[0], st); }
            for (size_t c = 0; c < nchunks && e == cudaSuccess; c++) {
                const int b = (int)(c & 1); const size_t off = c * kChunk, m = std::min(kChunk, bytes - off);
                if (c + 1 < nchunks) {
                    const size_t off2 = (c + 1) * kChunk, m2 = std::min(kChunk, bytes - off2);
                    e = cudaMemcpyAsync(pin[b ^ 1], (const char*)src + off2, m2, cudaMemcpyDeviceToHost, st);
                    if (e == cudaSuccess) e = cudaEventRecord(ev[b ^ 1], st);
                }
                if (e == cudaSuccess) e = cudaEventSynchronize(ev[b]);
                if (e == cudaSuccess) pool.copy((char*)dst + off, pin[b], m);
            }
        }
    }
    return e;
}

struct I2vDist { int rank = 0, world = 1; void* nccl = nullptr; long sync_every = 0; };

// embedding.TrainEmbedding on the device.  Stream-proportional work (dictionary counts, MinCount filter) and the
// per-word Huffman paths are built on the GPU; the host only runs the O(V) two-queue Huffman merge over the
// count-sorted leaves.  dist (world > 1): every rank trains on its own shard of the stream with a full replica of
// both vector tables; dictionary counts are all-reduced (identical tree everywhere) and the replicas are averaged
// every sync_every positions (local SGD / model averaging — the reference's own trainer is Hogwild over goroutines,
// word2vec.go:165-169; across GPUs the racy shared memory becomes periodic averaging).
int i2v_check_cfg(const ctr_i2v_config& c, const ctr_handle* eh) {
    if (c.dim < 4 || c.dim > 128 || (c.dim & (c.dim - 1)) || c.window < 1 || c.iter < 1 || c.max_depth < 2 || c.update_lr_batch < 1)
        return set_err(eh, CTR_EINVAL, "item2vec: dim must be a power of two in [4,128], window/iter >= 1");
    return CTR_OK;
}

// The trainer proper, from a device-resident word-id document d_tok [n] (ids in [0, V), corpus order) on stream st:
// leaves the trained float32 syn0 [V, D] in d_syn0 on the device.  The same document trains the same whether it came
// from the host (ctr_i2v_train) or was numbered on the device (ctr_item_emb_train).  Errors are reported on eh
// (nullptr: the stand-alone entry points).
int i2v_train_dev(const ctr_i2v_config& c, const int* d_tok, int64_t n, int32_t V, int num_sms, cudaStream_t st, DevBuf<float>& d_syn0,
                  ctr_i2v_stats* stats, I2vDist* dist, const ctr_handle* eh) {
    const int D = c.dim, W = c.window;
    const int world = dist ? dist->world : 1;
    const bool seq = c.reserved[0] == 1;
#define CI(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return set_err(eh, CTR_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)
#define CN(call) do { int r_ = (call); if (r_ != 0) return set_err(eh, CTR_ECOMM, "%s: %s", #call, g_nccl.GetErrorString(r_)); } while (0)
    // declared first, destroyed last: every buffer below is freed before the events
    Event e0, e1;
    DevBuf<int> d_doc, d_pnode, d_sid, d_sid2, d_parent, d_bad;
    DevBuf<unsigned long long> d_cnt64, d_skey, d_skey2, d_ctr, d_misc;
    DevBuf<unsigned char> d_keep, d_pcode, d_code, d_tmp;
    DevBuf<long long> d_poff, d_nval; DevBuf<long> d_nd;
    DevBuf<double> d_z; DevBuf<float> d_syn1, d_lr, d_nsc, d_wsc;
    size_t tmp_bytes = 0;
    float ms_total = 0; int launches = 0; unsigned long long hc[3] = {0, 0, 0};
    const int G = num_sms * 8;
    CI(e0.create(cudaEventDefault)); CI(e1.create(cudaEventDefault));
    // ---- dictionary counts over the whole stream (dictionary.go:70-81), on the device
    CI(d_doc.alloc((size_t)n)); CI(d_keep.alloc((size_t)n));
    CI(d_cnt64.alloc((size_t)V)); CI(d_bad.alloc(1)); CI(d_nd.alloc(1));
    CI(d_misc.alloc(4));
    CI(cudaMemsetAsync(d_cnt64, 0, sizeof(unsigned long long) * (size_t)V, st)); CI(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    k_i2v_count<<<G, 256, 0, st>>>(d_tok, (long)n, V, d_cnt64, d_bad); launches++;
    unsigned long long n_global = (unsigned long long)n;
    long nd_max_global = 0;
    if (world > 1) {
        CN(g_nccl.AllReduce(d_cnt64, d_cnt64, (size_t)V, kNcclUint64, kNcclSum, dist->nccl, st));
        CI(cudaMemcpyAsync(d_misc, &n_global, sizeof n_global, cudaMemcpyHostToDevice, st));
        CN(g_nccl.AllReduce(d_misc, d_misc, 1, kNcclUint64, kNcclSum, dist->nccl, st));
        CI(cudaMemcpyAsync(&n_global, d_misc, sizeof n_global, cudaMemcpyDeviceToHost, st));
    }
    // ---- the training document: words rarer than MinCount are dropped (memory.go:53-62), order kept
    k_i2v_keep<<<G, 256, 0, st>>>(d_tok, (long)n, d_cnt64, c.min_count, d_keep); launches++;
    cub::DeviceSelect::Flagged(nullptr, tmp_bytes, d_tok, d_keep.get(), d_doc.get(), d_nd.get(), (int)n, st);
    {
        size_t b2 = 0, b3 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, b2, d_skey.get(), d_skey2.get(), d_sid.get(), d_sid2.get(), V, 0, 64, st);
        cub::DeviceScan::ExclusiveSum(nullptr, b3, d_poff.get(), d_poff.get(), V + 1, st);
        tmp_bytes = std::max(tmp_bytes, std::max(b2, b3));
    }
    CI(d_tmp.alloc(tmp_bytes));
    { size_t tb = tmp_bytes; cub::DeviceSelect::Flagged(d_tmp, tb, d_tok, d_keep.get(), d_doc.get(), d_nd.get(), (int)n, st); launches++; }
    long nd = 0; int bad = 0;
    CI(cudaMemcpyAsync(&nd, d_nd, sizeof nd, cudaMemcpyDeviceToHost, st)); CI(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, st));
    CI(cudaStreamSynchronize(st));
    if (bad) return set_err(eh, CTR_EINVAL, "a token lies outside [0, vocab)");
    nd_max_global = nd;
    if (world > 1) {
        unsigned long long v = (unsigned long long)nd;
        CI(cudaMemcpyAsync(d_misc, &v, sizeof v, cudaMemcpyHostToDevice, st));
        CN(g_nccl.AllReduce(d_misc, d_misc, 1, kNcclUint64, kNcclMax, dist->nccl, st));
        CI(cudaMemcpyAsync(&v, d_misc, sizeof v, cudaMemcpyDeviceToHost, st)); CI(cudaStreamSynchronize(st));
        nd_max_global = (long)v;
    }
    // concurrency: (centre, context) pairs in flight ~ vocabulary / 4, at most the whole machine
    const int rpw = 32 / (D / 4);
    const long max_warps = (long)num_sms * 8 * 8;
    const long warps = std::max<long>(1, std::min<long>(std::min<long>(max_warps, (std::max<long>(nd, 1) + 63) / 64), std::max<long>(1, (long)V / 4 / rpw)));
    const int grid = (int)((warps + 7) / 8);
    const double Ceff = (double)grid * 8 * rpw;
    // ---- per-word tables + count-sorted leaves (stable: ties stay in id order, like the reference's sort)
    CI(d_z.alloc((size_t)V)); CI(d_wsc.alloc((size_t)V));
    CI(d_skey.alloc((size_t)V)); CI(d_skey2.alloc((size_t)V));
    CI(d_sid.alloc((size_t)V)); CI(d_sid2.alloc((size_t)V));
    k_i2v_word_tables<<<G, 256, 0, st>>>(d_cnt64, V, (double)c.subsample, Ceff, (double)n_global, d_z, d_wsc, d_skey, d_sid); launches++;
    { size_t tb = tmp_bytes; cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_skey.get(), d_skey2.get(), d_sid.get(), d_sid2.get(), V, 0, 64, st); launches++; }
    std::vector<int64_t> cnt((size_t)V); std::vector<int> leaves((size_t)V);
    CI(cudaMemcpyAsync(cnt.data(), d_cnt64, sizeof(int64_t) * (size_t)V, cudaMemcpyDeviceToHost, st));
    CI(cudaMemcpyAsync(leaves.data(), d_sid2, sizeof(int) * (size_t)V, cudaMemcpyDeviceToHost, st));
    CI(cudaStreamSynchronize(st));
    // ---- host: the Huffman merge (huffman.go:23-57), O(V)
    std::vector<int> parent; std::vector<unsigned char> code; std::vector<long long> node_val;
    const int n_inner = i2v_huffman_sorted(cnt.data(), leaves.data(), V, parent, code, node_val);
    if (n_inner < 1) return set_err(eh, CTR_EINVAL, "item2vec needs at least two distinct words in the stream");
    // ---- paths (node.go:26-43) on the device
    CI(d_parent.alloc(parent.size())); CI(d_code.alloc(code.size())); CI(d_nval.alloc(node_val.size()));
    CI(d_poff.alloc((size_t)V + 1)); CI(d_nsc.alloc(node_val.size()));
    CI(cudaMemcpyAsync(d_parent, parent.data(), sizeof(int) * parent.size(), cudaMemcpyHostToDevice, st));
    CI(cudaMemcpyAsync(d_code, code.data(), code.size(), cudaMemcpyHostToDevice, st));
    CI(cudaMemcpyAsync(d_nval, node_val.data(), sizeof(long long) * node_val.size(), cudaMemcpyHostToDevice, st));
    CI(cudaMemsetAsync(d_poff, 0, sizeof(long long) * ((size_t)V + 1), st));
    k_i2v_paths<<<G, 256, 0, st>>>(d_parent, d_code, d_cnt64, V, c.max_depth, 0, d_poff, nullptr, nullptr); launches++;
    { size_t tb = tmp_bytes; cub::DeviceScan::ExclusiveSum(d_tmp, tb, d_poff.get(), d_poff.get(), V + 1, st); launches++; }
    long long nsteps = 0;
    CI(cudaMemcpyAsync(&nsteps, d_poff + V, sizeof nsteps, cudaMemcpyDeviceToHost, st)); CI(cudaStreamSynchronize(st));
    CI(d_pnode.alloc((size_t)std::max<long long>(nsteps, 1))); CI(d_pcode.alloc((size_t)std::max<long long>(nsteps, 1)));
    k_i2v_paths<<<G, 256, 0, st>>>(d_parent, d_code, d_cnt64, V, c.max_depth, 1, d_poff, d_pnode, d_pcode); launches++;
    k_i2v_node_scale<<<G, 256, 0, st>>>(d_nval, V - 1, Ceff, (double)n_global, d_nsc); launches++;
    CI(d_ctr.alloc(3)); CI(cudaMemsetAsync(d_ctr, 0, 3 * sizeof(unsigned long long), st));
    if (seq) {
        // sequential float64 parity mode (item2vec.cuh): one warp, the reference's single-goroutine order
        DevBuf<double> d64_0, d64_1, d_lut64;
        std::vector<double> lut64(1000);
        for (int i = 0; i < 1000; i++) { double e = std::exp(((double)i / 1000.0 * 2.0 - 1.0) * 6.0); lut64[(size_t)i] = e / (e + 1.0); }   // sigmoid_table.go:28-45
        cudaError_t e1_ = d64_0.alloc((size_t)V * D), e2_ = d64_1.alloc((size_t)std::max(V - 1, 1) * D),
                    e3_ = d_lut64.alloc(1000), e4_ = d_syn0.alloc((size_t)V * D);
        if (e1_ != cudaSuccess || e2_ != cudaSuccess || e3_ != cudaSuccess || e4_ != cudaSuccess) return set_err(eh, CTR_ENOMEM, "item2vec float64 tables");
        cudaMemcpyAsync(d_lut64, lut64.data(), sizeof(double) * 1000, cudaMemcpyHostToDevice, st);
        cudaMemsetAsync(d64_1, 0, sizeof(double) * (size_t)std::max(V - 1, 1) * D, st);
        k_i2v_init64<<<G, 256, 0, st>>>(d64_0, (long)V * D, D, c.seed); launches++;
        I2vSeqArgs sa{}; sa.doc = d_doc; sa.nd = nd; sa.n_stream = (long)n; sa.z = d_z; sa.poff = d_poff; sa.pnode = d_pnode; sa.pcode = d_pcode;
        sa.syn0 = d64_0; sa.syn1 = d64_1; sa.lut = d_lut64; sa.D = D; sa.W = W; sa.upd = c.update_lr_batch; sa.iters = c.iter;
        sa.init_lr = (double)c.init_lr; sa.min_lr = (double)c.min_lr; sa.seed = c.seed; sa.counters = d_ctr;
        cudaEventRecord(e0, st);
        k_i2v_seq_f64<<<1, 32, 0, st>>>(sa); launches++;
        cudaEventRecord(e1, st);
        k_f64_to_f32_i2v<<<G, 256, 0, st>>>(d64_0, d_syn0, (long)V * D); launches++;
        cudaMemcpyAsync(hc, d_ctr, sizeof hc, cudaMemcpyDeviceToHost, st);
        if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess) return set_err(eh, CTR_ECUDA, "item2vec sequential mode: %s", cudaGetErrorString(cudaGetLastError()));
        cudaEventElapsedTime(&ms_total, e0, e1);
        if (stats) {
            stats->doc_len = nd; stats->trained_positions = (int64_t)hc[0]; stats->pairs = (int64_t)hc[1]; stats->node_visits = (int64_t)hc[2];
            stats->algorithmic_bytes = 2.0 * D * 8.0 * ((double)hc[1] + (double)hc[2]); stats->ms_device = ms_total; stats->launches = launches;
        }
        return CTR_OK;
    }
    // ---- vector tables: syn0 = (U-0.5)/dim (word2vec.go:103-111), inner nodes zero (huffman.go:40)
    std::vector<float> lut(1000);
    for (int i = 0; i < 1000; i++) { double e = std::exp(((double)i / 1000.0 * 2.0 - 1.0) * 6.0); lut[(size_t)i] = (float)(e / (e + 1.0)); }
    CI(cudaMemcpyToSymbolAsync(c_i2v_lut, lut.data(), sizeof(float) * 1000, 0, cudaMemcpyHostToDevice, st));
    CI(d_syn0.alloc((size_t)V * D)); CI(d_syn1.alloc((size_t)(V - 1) * D));
    CI(cudaMemsetAsync(d_syn1, 0, sizeof(float) * (size_t)(V - 1) * D, st));
    k_i2v_init<<<G, 256, 0, st>>>(d_syn0, (long)V * D, D, c.seed); launches++;
    const long nchunks = nd_max_global / c.update_lr_batch + 2;
    CI(d_lr.alloc((size_t)nchunks));
    std::vector<float> lr_tab((size_t)nchunks);
    double lr = c.init_lr;                                                           // w.currentlr persists across iterations
    // segments: one per iteration on a single GPU; every sync_every positions when replicas have to be averaged
    const long seg = (world > 1 && dist->sync_every > 0) ? dist->sync_every : std::max<long>(nd_max_global, 1);
    for (int it = 0; it < c.iter; it++) {
        for (long k = 0; k < nchunks; k++) {                                         // observe(), word2vec.go:223-233 (positions of all ranks advance together)
            lr_tab[(size_t)k] = (float)lr;
            const double seen = (double)(k + 1) * c.update_lr_batch * world;
            if ((double)(k + 1) * c.update_lr_batch <= (double)nd_max_global) lr = lr < (double)c.min_lr ? (double)c.min_lr : (double)c.init_lr * (1.0 - seen / (double)n_global);
        }
        CI(cudaMemcpyAsync(d_lr, lr_tab.data(), sizeof(float) * (size_t)nchunks, cudaMemcpyHostToDevice, st));
        I2vArgs a{}; a.doc = d_doc; a.nd = nd; a.z = d_z; a.poff = d_poff; a.pnode = d_pnode; a.pcode = d_pcode; a.syn0 = d_syn0; a.syn1 = d_syn1;
        a.D = D; a.W = W; a.lr_tab = d_lr; a.upd = c.update_lr_batch; a.seed = c.seed; a.iter = it; a.counters = d_ctr;
        a.node_scale = d_nsc; a.word_scale = d_wsc;
        a.hot_n = std::min(kI2vHot, n_inner); a.hot_base = n_inner - a.hot_n;      // the last nodes created = the top of the tree
        const size_t sm = (size_t)std::max(a.hot_n, 1) * D * sizeof(float);
        CI(cudaEventRecord(e0, st));
        for (long p0 = 0; p0 < std::max<long>(nd_max_global, 1); p0 += seg) {
            a.pos_begin = p0; a.pos_end = std::min<long>(nd, p0 + seg);
            if (a.pos_end > a.pos_begin) {
                switch (D / 4) {
                    case 1: k_i2v_skipgram_hs<1><<<grid, 256, sm, st>>>(a); break;   case 2: k_i2v_skipgram_hs<2><<<grid, 256, sm, st>>>(a); break;
                    case 4: k_i2v_skipgram_hs<4><<<grid, 256, sm, st>>>(a); break;   case 8: k_i2v_skipgram_hs<8><<<grid, 256, sm, st>>>(a); break;
                    case 16: k_i2v_skipgram_hs<16><<<grid, 256, sm, st>>>(a); break; default: k_i2v_skipgram_hs<32><<<grid, 256, sm, st>>>(a); break;
                }
                launches++;
            }
            if (world > 1) {      // model averaging: every replica continues from the mean of all replicas
                CN(g_nccl.GroupStart());
                CN(g_nccl.AllReduce(d_syn0, d_syn0, (size_t)V * D, kNcclFloat32, kNcclSum, dist->nccl, st));
                CN(g_nccl.AllReduce(d_syn1, d_syn1, (size_t)(V - 1) * D, kNcclFloat32, kNcclSum, dist->nccl, st));
                CN(g_nccl.GroupEnd());
                k_i2v_scale<<<G, 256, 0, st>>>(d_syn0, (long)V * D, 1.0f / (float)world);
                k_i2v_scale<<<G, 256, 0, st>>>(d_syn1, (long)(V - 1) * D, 1.0f / (float)world);
                launches += 3;
            }
        }
        CI(cudaGetLastError());
        CI(cudaEventRecord(e1, st)); CI(cudaStreamSynchronize(st));                   // lr_tab is reused by the next iteration
        float ms = 0; CI(cudaEventElapsedTime(&ms, e0, e1)); ms_total += ms;
    }
    CI(cudaMemcpyAsync(hc, d_ctr, sizeof hc, cudaMemcpyDeviceToHost, st));
    CI(cudaStreamSynchronize(st));
    if (stats) {
        stats->doc_len = nd; stats->trained_positions = (int64_t)hc[0]; stats->pairs = (int64_t)hc[1]; stats->node_visits = (int64_t)hc[2];
        stats->algorithmic_bytes = 2.0 * D * 4.0 * ((double)hc[1] + (double)hc[2]); stats->ms_device = ms_total; stats->launches = launches;
    }
#undef CI
#undef CN
    return CTR_OK;
}

// ctr_i2v_train / ctr_i2v_train_dist: the word-id stream from the caller's host memory, the table back to it
int i2v_train_impl(const ctr_i2v_config* cfg, const int32_t* tokens, int64_t n, int32_t V, float* emb_out, ctr_i2v_stats* stats, I2vDist* dist) {
    if (!cfg || !tokens || (!emb_out && !dist) || n < 1 || V < 2 || n > 0x7fffffffLL) return set_err(nullptr, CTR_EINVAL, "bad item2vec arguments");
    const ctr_i2v_config& c = *cfg;
    RET(i2v_check_cfg(c, nullptr));
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return set_err(nullptr, CTR_ENODEV, "no CUDA device: this engine has no CPU fallback"); }
    if (c.reserved[0] == 1 && dist && dist->world > 1) return set_err(nullptr, CTR_EINVAL, "the sequential float64 mode is single-GPU");
#define CI(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return set_err(nullptr, CTR_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)
    // declared first, destroyed last: both buffers are freed before the stream
    Stream st;
    DevBuf<int> d_tok; DevBuf<float> d_syn0;
    CI(cudaSetDevice(c.device));
    cudaDeviceProp prop{}; CI(cudaGetDeviceProperties(&prop, c.device));
    if (prop.major != 9) return set_err(nullptr, CTR_ENODEV, "device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
    CI(st.create());
    CI(d_tok.alloc((size_t)n));
    CI(big_copy(d_tok, tokens, sizeof(int) * (size_t)n, true, st));
    RET(i2v_train_dev(c, d_tok, n, V, prop.multiProcessorCount, st, d_syn0, stats, dist, nullptr));
    if (emb_out) CI(big_copy(emb_out, d_syn0, sizeof(float) * (size_t)V * c.dim, false, st));
#undef CI
    return CTR_OK;
}
}  // namespace

int ctr_i2v_train(const ctr_i2v_config* cfg, const int32_t* tokens, int64_t n, int32_t V, float* emb_out, ctr_i2v_stats* stats) {
    return i2v_train_impl(cfg, tokens, n, V, emb_out, stats, nullptr);
}

// BASELINE configs[4] (item2vec over 8 GPUs): one process per GPU, each with its own shard of the item stream.
int ctr_i2v_train_dist(const ctr_i2v_config* cfg, const int32_t* tokens_shard, int64_t n_shard, int32_t V, float* emb_out, ctr_i2v_stats* stats,
                       int32_t rank, int32_t world, const void* nccl_id, int32_t id_bytes, int64_t sync_every) {
    if (world < 1 || rank < 0 || rank >= world) return set_err(nullptr, CTR_EINVAL, "bad rank/world");
    if (world == 1) return i2v_train_impl(cfg, tokens_shard, n_shard, V, emb_out, stats, nullptr);
    if (!nccl_id || id_bytes != 128 || !cfg) return set_err(nullptr, CTR_EINVAL, "unique id must be 128 bytes");
    std::string err;
    if (!nccl_load(&err)) return set_err(nullptr, CTR_ECOMM, "%s", err.c_str());
    if (cudaSetDevice(cfg->device) != cudaSuccess) return set_err(nullptr, CTR_ECUDA, "cudaSetDevice(%d)", cfg->device);
    I2vDist d; d.rank = rank; d.world = world; d.sync_every = sync_every > 0 ? (long)sync_every : 4L << 20;
    Uid u; memcpy(&u, nccl_id, 128);
    int r = g_nccl.CommInitRank(&d.nccl, world, u, rank);
    if (r != 0) return set_err(nullptr, CTR_ECOMM, "ncclCommInitRank: %s", g_nccl.GetErrorString(r));
    const int rc = i2v_train_impl(cfg, tokens_shard, n_shard, V, emb_out, stats, &d);
    g_nccl.CommDestroy(d.nccl);
    return rc;
}

// recommend.Train's embedding stage (rcmd.go:207-213, 538-545) into the handle's ITEM_EMB: first-appearance numbering of
// the item-id stream on the device (item2vec.cuh, idmap.cuh), the trainer on that document, one scatter into the rows.
// With world > 1 every rank numbers its own shard of the stream against the words of the ranks' streams concatenated in
// rank order (the first-occurrence tags of i2v_dict_ranks), trains its shard with model averaging and writes its rows.
namespace {
// world > 1: every rank's verdict, the configuration (device aside), ITEM_EMB's shape and placement, the item map (its
// size and digest, compared once every rank is valid) and every rank's token count, in one agreement
int item_emb_agree(ctr_handle* h, const ctr_i2v_config* cfg, const int64_t* item_ids, int64_t n, int64_t cap, int64_t* total) {
    const int W = h->comm.world;
    int verdict = CTR_OK;
    if (!cfg || n < 0 || n > 0x7fffffffLL || (n > 0 && !item_ids) || cap < 0) verdict = set_err(h, CTR_EINVAL, "bad item embedding arguments");
    else if (cfg->dim != h->cfg.D) verdict = set_err(h, CTR_EINVAL, "item2vec dim %d != model dim D=%d", cfg->dim, h->cfg.D);
    else if ((verdict = i2v_check_cfg(*cfg, h)) != CTR_OK) {}
    else if (cfg->reserved[0] == 1) verdict = set_err(h, CTR_EINVAL, "the sequential float64 mode is single-GPU");
    else if (!h->idm_keys[CTR_IDMAP_ITEM]) verdict = set_err(h, CTR_ESTATE, "ctr_item_emb_train needs the item id map (ctr_idmap_build)");
    else if (W > kMaxPeers) verdict = set_err(h, CTR_EINVAL, "ctr_item_emb_train supports at most %d ranks, got %d", kMaxPeers, W);
    CommHdr hd{};
    if (cfg) { ctr_i2v_config cc = *cfg; cc.device = 0; hd.hash[0] = comm_hash(&cc, sizeof cc); }
    const int T = CTR_TABLE_ITEM_EMB;
    const int64_t tab[4] = {h->tab[T] ? 1 : 0, h->tab_rows[T], h->tab_width[T], h->tab_sharded[T] ? 1 : 0};
    hd.hash[1] = comm_hash(tab, sizeof tab);
    hd.share = verdict == CTR_OK ? n : 0;
    if (h->idm_keys[CTR_IDMAP_ITEM]) {
        unsigned long long* d_dig = nullptr;
        RET(scratch_get(h, 2, sizeof(unsigned long long), (void**)&d_dig));
        CU(h, cudaMemsetAsync(d_dig, 0, sizeof(unsigned long long), h->stream));
        RET(launch(h, "idmap_digest", [&] {
            k_idmap_digest<<<h->num_sms * 8, 256, 0, h->stream>>>(h->idm_keys[CTR_IDMAP_ITEM], h->idm_vals[CTR_IDMAP_ITEM], h->idm_keys[CTR_IDMAP_ITEM].size(), d_dig);
        }));
        uint64_t map[2] = {(uint64_t)h->idm_n[CTR_IDMAP_ITEM], 0};
        CU(h, cudaMemcpyAsync(&map[1], d_dig, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        hd.rows = comm_hash(map, sizeof map);
    }
    std::vector<int64_t> shares((size_t)W);
    RET(comm_agree(h, hd, verdict, shares.data()));
    *total = 0;
    for (int64_t v : shares) *total += v;
    if (*total == 0) return set_err(h, CTR_EINVAL, "ctr_item_emb_train: every rank's stream is empty");
    return CTR_OK;
}
}  // namespace

int ctr_item_emb_train(ctr_handle* h, const ctr_i2v_config* cfg, const int64_t* item_ids, int64_t n, int64_t* vocab_ids, int64_t cap,
                       int32_t* vocab, ctr_i2v_stats* stats) {
    if (!h) return set_err(nullptr, CTR_EINVAL, "null handle");
    Comm& cm = h->comm;
    const int W = cm.world;
    std::lock_guard<std::mutex> lk(h->mu);
    std::vector<int64_t>().swap(h->emb_vocab);
    if (W == 1 && (!cfg || !item_ids || n < 1 || n > 0x7fffffffLL || cap < 0)) return set_err(h, CTR_EINVAL, "bad item embedding arguments");
    if (W > 1) {
        int64_t total = 0;
        RET(item_emb_agree(h, cfg, item_ids, n, cap, &total));
    } else {
        if (cfg->dim != h->cfg.D) return set_err(h, CTR_EINVAL, "item2vec dim %d != model dim D=%d", cfg->dim, h->cfg.D);
        RET(i2v_check_cfg(*cfg, h));
        if (!h->idm_keys[CTR_IDMAP_ITEM]) return set_err(h, CTR_ESTATE, "ctr_item_emb_train needs the item id map (ctr_idmap_build)");
    }
    const ctr_i2v_config& c = *cfg;
    CU(h, cudaSetDevice(h->dev));
    cudaStream_t st = h->stream;
    const long R = (long)h->idm_n[CTR_IDMAP_ITEM];
    const int G = h->num_sms * 8;
    const unsigned long long* mkeys = h->idm_keys[CTR_IDMAP_ITEM]; const int* mvals = h->idm_vals[CTR_IDMAP_ITEM];
    const unsigned long long mcap = h->idm_keys[CTR_IDMAP_ITEM].size();
    // the numbering across ranks runs under its own profile key; on one GPU its steps keep the keys of the steps they extend
    const char* across_side = W > 1 ? "i2v_dict_ranks" : "i2v_dict_side";
    const char* across_rows = W > 1 ? "i2v_dict_ranks" : "i2v_dict_rank";
    // kept to the end: the word-id document, row -> word, the vocabulary's item ids, the trained vectors
    DevBuf<int> d_doc, d_word_row; DevBuf<long long> d_vocab; DevBuf<float> d_syn0;
    int V = 0;
    {
        DevBuf<long long> d_ids; DevBuf<unsigned> d_first; DevBuf<unsigned long long> d_cnt, d_row_tag;
        CU(h, d_ids.alloc((size_t)n)); CU(h, d_doc.alloc((size_t)n));
        CU(h, d_first.alloc((size_t)R)); CU(h, d_row_tag.alloc((size_t)R)); CU(h, d_word_row.alloc((size_t)R)); CU(h, d_cnt.alloc(2));
        if (n > 0) CU(h, big_copy(d_ids, item_ids, sizeof(int64_t) * (size_t)n, true, st));
        CU(h, cudaMemsetAsync(d_first, 0xff, sizeof(unsigned) * (size_t)R, st));
        CU(h, cudaMemsetAsync(d_word_row, 0xff, sizeof(int) * (size_t)R, st));
        CU(h, cudaMemsetAsync(d_cnt, 0, 2 * sizeof(unsigned long long), st));
        // 1. every token through the item map; first position per row; tokens without an entry counted
        RET(launch(h, "i2v_dict_resolve", [&] { k_idmap_first_pos<<<G, 256, 0, st>>>(mkeys, mvals, mcap - 1, d_ids, (long)n, d_doc, d_first, d_cnt); }));
        unsigned long long m = 0;
        CU(h, cudaMemcpyAsync(&m, d_cnt, sizeof m, cudaMemcpyDeviceToHost, st)); CU(h, cudaStreamSynchronize(st));
        //    each row's first occurrence in the concatenation: this rank's tags, at their minimum over the ranks
        int rc = CTR_OK;
        RET(launch(h, across_rows, [&] {
            i2v_first_tags(d_first, R, cm.rank, d_row_tag, G, st);
            if (W > 1 && R > 0) rc = comm_min_u64(h, d_row_tag, (size_t)R);
        }));
        RET(rc);
        // 2. this rank's side list: distinct unmapped ids (ascending as uint64) and the first position of each
        DevBuf<unsigned long long> k0, k1; DevBuf<int> p0, p1, d_u; DevBuf<unsigned char> tmp;
        int ur = 0;
        if (m > 0) {
            CU(h, k0.alloc(m)); CU(h, k1.alloc(m)); CU(h, p0.alloc(m)); CU(h, p1.alloc(m)); CU(h, d_u.alloc(1));
            CU(h, tmp.alloc(i2v_dict_side_tmp_bytes((int)m, st)));
            cudaError_t e = cudaSuccess;
            RET(launch(h, "i2v_dict_side", [&] { e = i2v_dict_side_list(d_doc, d_ids, (long)n, (int)m, k0, k1, p0, p1, d_cnt + 1, d_u, tmp, tmp.size(), G, st, &ur); }));
            CU(h, e);
        }
        //    the side words of the concatenation: the ranks' lists all-gathered (counts, then the lists padded to the longest),
        //    reduced to the distinct ids ascending with the tag of each one's first occurrence
        RankLists L{};
        long stride = ur;
        const unsigned long long* g_ids = k0; const int* g_pos = p0;
        DevBuf<unsigned long long> sid, gid; DevBuf<int> spos, gpos;
        L.cnt[0] = ur; L.off[1] = ur;
        if (W > 1) {
            int64_t all[kMaxPeers] = {};
            const int64_t mine = ur;
            RET(comm_gather_i64(h, &mine, 1, all));
            stride = 0;
            for (int j = 0; j < W; j++) { L.cnt[j] = (int)all[j]; L.off[j + 1] = L.off[j] + all[j]; stride = std::max<long>(stride, (long)all[j]); }
            if (L.off[W] > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "ctr_item_emb_train: the ranks' side ids (%lld) exceed INT32_MAX", (long long)L.off[W]);
            if (stride > 0) {
                CU(h, sid.alloc((size_t)stride)); CU(h, spos.alloc((size_t)stride));
                CU(h, gid.alloc((size_t)stride * W)); CU(h, gpos.alloc((size_t)stride * W));
                if (ur > 0) {
                    CU(h, cudaMemcpyAsync(sid, k0, sizeof(unsigned long long) * (size_t)ur, cudaMemcpyDeviceToDevice, st));
                    CU(h, cudaMemcpyAsync(spos, p0, sizeof(int) * (size_t)ur, cudaMemcpyDeviceToDevice, st));
                }
                RET(launch(h, "i2v_dict_ranks", [&] {
                    rc = comm_gather_lists(h, spos, gpos, sizeof(int), nullptr, nullptr, (size_t)stride);
                    if (rc == CTR_OK) rc = comm_gather_lists(h, sid, gid, sizeof(unsigned long long), nullptr, nullptr, (size_t)stride);
                }));
                RET(rc);
            }
            g_ids = gid; g_pos = gpos;
        }
        const int64_t mt = L.off[W];
        DevBuf<unsigned long long> side_id, side_tag, key1, tag1; DevBuf<int> d_word_side, d_us; DevBuf<unsigned char> mtmp;
        int u = 0;
        if (mt > 0) {
            CU(h, side_id.alloc((size_t)mt)); CU(h, side_tag.alloc((size_t)mt)); CU(h, key1.alloc((size_t)mt)); CU(h, tag1.alloc((size_t)mt)); CU(h, d_us.alloc(1));
            const size_t tb = idmap_merge_tmp_bytes((int)mt, st);
            CU(h, mtmp.alloc(std::max<size_t>(tb, 1)));
            cudaError_t e = cudaSuccess;
            RET(launch(h, across_side, [&] { e = idmap_merge_min(g_ids, g_pos, stride, L, W, side_id, key1, side_tag, tag1, d_us, mtmp, tb, G, st, &u); }));
            CU(h, e);
            CU(h, d_word_side.alloc((size_t)u));
        }
        // 3. rows and side words ordered by first occurrence: the rank is the word id
        {
            const long N = R + u;
            DevBuf<unsigned long long> rk0, rk1; DevBuf<int> rv0, rv1, d_V; DevBuf<long long> d_row_id; DevBuf<unsigned char> otmp;
            CU(h, rk0.alloc((size_t)N)); CU(h, rk1.alloc((size_t)N)); CU(h, rv0.alloc((size_t)N)); CU(h, rv1.alloc((size_t)N));
            CU(h, d_row_id.alloc((size_t)R)); CU(h, d_vocab.alloc((size_t)N)); CU(h, d_V.alloc(1));
            const size_t tb = i2v_dict_order_tmp_bytes(N, st);
            CU(h, otmp.alloc(std::max<size_t>(tb, 1)));
            cudaError_t e = cudaSuccess;
            RET(launch(h, "i2v_dict_rank", [&] {
                e = i2v_dict_order(mkeys, mvals, mcap, d_row_tag, R, side_id, side_tag, u, W, d_row_id, rk0, rk1, rv0, rv1, otmp, tb,
                                   d_word_row, d_word_side, d_vocab, d_V, G, st, &V);
            }));
            CU(h, e);
        }
        // 4. this rank's int32 word-id document, in place over its resolved rows
        RET(launch(h, "i2v_dict_doc", [&] { k_i2v_dict_doc<<<G, 256, 0, st>>>(d_doc, d_ids, (long)n, d_word_row, side_id, u, d_word_side); }));
        CU(h, cudaStreamSynchronize(st));
    }
    if (vocab) *vocab = V;
    if (vocab_ids && cap > 0) {
        CU(h, cudaMemcpyAsync(vocab_ids, d_vocab, sizeof(int64_t) * (size_t)std::min<int64_t>(cap, V), cudaMemcpyDeviceToHost, st));
        CU(h, cudaStreamSynchronize(st));
    }
    if (vocab_ids && cap < V) {          // the rest stays readable (ctr_item_emb_vocab): a rank cannot size vocab_ids for
        h->emb_vocab.resize((size_t)V);  // the unmapped ids of the other ranks' streams
        CU(h, cudaMemcpyAsync(h->emb_vocab.data(), d_vocab, sizeof(int64_t) * (size_t)V, cudaMemcpyDeviceToHost, st));
        CU(h, cudaStreamSynchronize(st));
    }
    if (V < 2) return set_err(h, CTR_EINVAL, "item2vec needs at least two distinct words in the stream (%d)", V);
    d_vocab.reset();
    ctr_i2v_stats s{};
    I2vDist dist;
    if (W > 1) { dist.rank = cm.rank; dist.world = W; dist.nccl = cm.nccl; dist.sync_every = c.reserved[1] > 0 ? (long)c.reserved[1] : 4L << 20; }
    RET(i2v_train_dev(c, d_doc, n, V, h->num_sms, st, d_syn0, &s, W > 1 ? &dist : nullptr, h));
    d_doc.reset();
    // ITEM_EMB [R, D]: as ctr_table_upload of the remapped table would leave it
    const int D = c.dim;
    const int T = CTR_TABLE_ITEM_EMB;
    if (h->tab[T] && h->tab_rows[T] == R && h->tab_width[T] == D) table_new_state(h, T);
    else RET(table_alloc(h, T, R, D));
    // A row-sharded table: this rank writes the rows it owns from its own replica (the replicas are equal after the final
    // averaging).  No peer still reads or writes this shard: the call's first collective (the agreement's all-gather on
    // the engine stream) completed on this rank only once every rank had reached it in its own stream order, behind every
    // earlier read or red.add of this shard it queued (a sharded step, a serving call); and tab_gen is bumped, so a peer's
    // next collective call republishes the mappings and pulls the hot rows only after an exchange with this rank, which
    // makes it after this write.
    const bool sh = h->tab_sharded[T];
    float* tab = h->tab[T];
    RET(launch(h, "i2v_emb_scatter", [&] { k_i2v_emb_scatter<<<G, 256, 0, st>>>(d_syn0, d_word_row, R, D, sh ? W : 1, sh ? cm.rank : 0, tab); }));
    CU(h, cudaStreamSynchronize(st));
    if (stats) *stats = s;
    return CTR_OK;
}

int ctr_item_emb_vocab(ctr_handle* h, int64_t* vocab_ids, int64_t cap, int32_t* vocab) {
    if (!h || !vocab || cap < 0 || (cap > 0 && !vocab_ids)) return set_err(h, CTR_EINVAL, "bad item embedding vocabulary arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (h->emb_vocab.empty()) return set_err(h, CTR_ESTATE, "no item embedding vocabulary kept: the last ctr_item_emb_train returned all of it, or none");
    *vocab = (int32_t)h->emb_vocab.size();
    if (cap > 0) memcpy(vocab_ids, h->emb_vocab.data(), sizeof(int64_t) * (size_t)std::min<int64_t>(cap, (int64_t)h->emb_vocab.size()));
    return CTR_OK;
}

// ---- live id maps and tables: new users and items on a running handle (row f3) -----------------------------------
namespace {
unsigned long long idmap_cap_for(int64_t n) {
    unsigned long long cap = 64;
    while (cap < 2ull * (unsigned long long)n) cap <<= 1;                 // load factor <= 0.5, as ctr_idmap_build
    return cap;
}

// The ids of d_ids [n] the map lacks, numbered as ctr_item_emb_train numbers its side words: the probe
// (k_idmap_first_pos) marks them, k_i2v_dict_side + a radix sort + ReduceByKey(MinPos) give each distinct one its first
// position.  k0 / p0 [u]: the distinct missing ids (ascending as uint64) and their first positions; d_rows [n]: the row of
// every id the map holds, -1 for the others; m: the ids without a row.  tmp also fits the sort by position of u entries.
struct IdmapSide {
    DevBuf<unsigned long long> k0, k1; DevBuf<int> p0, p1, d_u; DevBuf<unsigned char> tmp;
    unsigned long long m = 0; int u = 0;
};
int idmap_number(ctr_handle* h, int which, const long long* d_ids, int64_t n, int* d_rows, unsigned long long* d_cnt, IdmapSide* s) {
    cudaStream_t st = h->stream;
    const int G = h->num_sms * 8;
    s->m = (unsigned long long)n;
    if (h->idm_keys[which]) {
        RET(launch(h, "idmap_probe", [&] {
            k_idmap_first_pos<<<G, 256, 0, st>>>(h->idm_keys[which], h->idm_vals[which], h->idm_keys[which].size() - 1, d_ids, (long)n, d_rows, nullptr, d_cnt);
        }));
        CU(h, cudaMemcpyAsync(&s->m, d_cnt, sizeof s->m, cudaMemcpyDeviceToHost, st));
    } else CU(h, cudaMemsetAsync(d_rows, 0xff, sizeof(int) * (size_t)n, st));
    CU(h, cudaStreamSynchronize(st));
    if (s->m == 0) return CTR_OK;
    const unsigned long long m = s->m;
    CU(h, s->k0.alloc(m)); CU(h, s->k1.alloc(m)); CU(h, s->p0.alloc(m)); CU(h, s->p1.alloc(m)); CU(h, s->d_u.alloc(1));
    size_t b1 = 0, b2 = 0, b3 = 0;
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b1, s->k0.get(), s->k1.get(), s->p0.get(), s->p1.get(), (int)m, 0, 64, st));
    CU(h, cub::DeviceReduce::ReduceByKey(nullptr, b2, s->k1.get(), s->k0.get(), s->p1.get(), s->p0.get(), s->d_u.get(), MinPos{}, (int)m, st));
    CU(h, cub::DeviceRadixSort::SortPairs(nullptr, b3, s->p0.get(), s->p1.get(), s->k0.get(), s->k1.get(), (int)m, 0, 32, st));
    CU(h, s->tmp.alloc(std::max(b1, std::max(b2, b3))));
    RET(launch(h, "idmap_number", [&] { k_i2v_dict_side<<<G, 256, 0, st>>>(d_rows, d_ids, (long)n, s->k0, s->p0, d_cnt + 1); }));
    RET(launch(h, "idmap_number", [&] { size_t tb = s->tmp.size(); cub::DeviceRadixSort::SortPairs(s->tmp.get(), tb, s->k0.get(), s->k1.get(), s->p0.get(), s->p1.get(), (int)m, 0, 64, st); }));
    RET(launch(h, "idmap_number", [&] { size_t tb = s->tmp.size(); cub::DeviceReduce::ReduceByKey(s->tmp.get(), tb, s->k1.get(), s->k0.get(), s->p1.get(), s->p0.get(), s->d_u.get(), MinPos{}, (int)m, st); }));
    CU(h, cudaMemcpyAsync(&s->u, s->d_u, sizeof s->u, cudaMemcpyDeviceToHost, st)); CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}

// fresh [u] (ids the map lacks, distinct, in row order) get rows R, R + 1, ...: a table at the capacity ctr_idmap_build
// picks for the new count (the old entries rehashed into it, then swapped), the inserts, and d_rows [n] looked up again
// when `lookup`
int idmap_add(ctr_handle* h, int which, const unsigned long long* fresh, int u, const long long* d_ids, int64_t n, int* d_rows, bool lookup) {
    cudaStream_t st = h->stream;
    const int G = h->num_sms * 8;
    const int64_t R = h->idm_n[which];
    const bool have = (bool)h->idm_keys[which];
    const unsigned long long cap = idmap_cap_for(R + u), old_cap = have ? h->idm_keys[which].size() : 0;
    if (cap > old_cap) {
        DevBuf<unsigned long long> nk; DevBuf<int> nv;
        RET(dalloc(h, nk, (size_t)cap, false)); RET(dalloc(h, nv, (size_t)cap, false));
        RET(launch(h, "idmap_clear", [&] { k_idmap_clear<<<G, 256, 0, st>>>(nk, nv, cap); }));
        if (have) RET(launch(h, "idmap_rehash", [&] { k_idmap_rehash<<<G, 256, 0, st>>>(h->idm_keys[which], h->idm_vals[which], old_cap, nk, nv, cap - 1); }));
        h->idm_keys[which] = std::move(nk); h->idm_vals[which] = std::move(nv);        // cudaFree of the old table waits for the rehash
    }
    RET(launch(h, "idmap_insert", [&] {
        k_idmap_insert<<<G, 256, 0, st>>>(h->idm_keys[which], h->idm_vals[which], h->idm_keys[which].size() - 1, (const long long*)fresh, (long)u, h->k_flags, (int)R);
    }));
    h->idm_n[which] = R + u;
    if (lookup) RET(launch(h, "idmap_lookup", [&] {
        k_idmap_lookup<<<G, 256, 0, st>>>(h->idm_keys[which], h->idm_vals[which], h->idm_keys[which].size() - 1, d_ids, (long)n, d_rows);
    }));
    return CTR_OK;
}

// World > 1: every rank numbers its own missing ids, the ranks all-gather their lists (counts, then the lists padded to
// the longest) and each runs the same merge (idmap_merge_ranks, idmap.cuh) and inserts its result, so every map ends as
// the single-GPU insert of the ranks' ids concatenated in rank order.  Before any write the ranks agree on the arguments'
// verdicts and on the map they start from: its id count and the order-independent digest of its (id, row) pairs.
int idmap_insert_ranks(ctr_handle* h, int which, const int64_t* ids, int64_t n, int32_t* rows) {
    Comm& cm = h->comm;
    const int W = cm.world;
    CU(h, cudaSetDevice(h->dev));
    cudaStream_t st = h->stream;
    const bool args_ok = !(which < 0 || which > 1 || n < 0 || n > 0x7fffffffLL || (n > 0 && !ids));
    int verdict = args_ok ? CTR_OK : set_err(h, CTR_EINVAL, "bad idmap insert arguments");
    for (int64_t i = 0; verdict == CTR_OK && i < n; i++)
        if ((unsigned long long)ids[i] == kIdEmpty) verdict = set_err(h, CTR_EINVAL, "idmap insert: id INT64_MIN is reserved (position %lld of rank %d)", (long long)i, cm.rank);
    unsigned long long* d_cnt = nullptr;                 // [0] ids without a row, [1] side counter, [2] map digest
    RET(scratch_get(h, 2, 3 * sizeof(unsigned long long), (void**)&d_cnt));
    CommHdr hd{};
    if (args_ok) {
        hd.k = which; hd.n = h->idm_n[which]; hd.mode = h->idm_keys[which] ? 1 : 0;
        if (h->idm_keys[which]) {
            CU(h, cudaMemsetAsync(d_cnt + 2, 0, sizeof(unsigned long long), st));
            RET(launch(h, "idmap_digest", [&] {
                k_idmap_digest<<<h->num_sms * 8, 256, 0, st>>>(h->idm_keys[which], h->idm_vals[which], h->idm_keys[which].size(), d_cnt + 2);
            }));
            CU(h, cudaMemcpyAsync(&hd.hash[0], d_cnt + 2, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            CU(h, cudaStreamSynchronize(st));
        }
    }
    {
        const int rc = comm_agree(h, hd, verdict);
        if (rc != CTR_OK) return rc;
    }
    const int64_t R = h->idm_n[which];
    const int G = h->num_sms * 8;
    long long* d_ids = nullptr; int* d_rows = nullptr;
    RET(scratch_get(h, 0, sizeof(long long) * (size_t)std::max<int64_t>(n, 1), (void**)&d_ids));
    RET(scratch_get(h, 1, sizeof(int) * (size_t)std::max<int64_t>(n, 1), (void**)&d_rows));
    if (!h->k_flags) RET(dalloc(h, h->k_flags, 1));
    if (n > 0) CU(h, big_copy(d_ids, ids, sizeof(int64_t) * (size_t)n, true, st));
    CU(h, cudaMemsetAsync(d_cnt, 0, 2 * sizeof(unsigned long long), st));
    IdmapSide s;
    RET(idmap_number(h, which, d_ids, n, d_rows, d_cnt, &s));
    // the ranks' counts, then their lists padded to the longest
    int64_t all[2 * kMaxPeers] = {};
    const int64_t mine[2] = {s.u, n};
    RET(comm_gather_i64(h, mine, 2, all));
    RankLists L{};
    int64_t stride = 0, total = 0;
    for (int j = 0; j < W; j++) { L.cnt[j] = (int)all[2 * j]; L.off[j + 1] = L.off[j] + all[2 * j]; stride = std::max(stride, all[2 * j]); total += all[2 * j + 1]; }
    // one GPU refuses a concatenation of more than INT32_MAX ids: so do the ranks, all of them, before any write
    if (total > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "idmap insert: the ranks pass %lld ids in all (more than INT32_MAX)", (long long)total);
    if (stride > 0) {
        const int64_t m = L.off[W];
        if (m > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "idmap insert: the ranks' new ids (%lld) exceed INT32_MAX", (long long)m);
        DevBuf<unsigned long long> sid, gid, key0, key1, tag0, tag1; DevBuf<int> spos, gpos, d_u; DevBuf<unsigned char> tmp;
        CU(h, sid.alloc((size_t)stride)); CU(h, spos.alloc((size_t)stride));
        CU(h, gid.alloc((size_t)stride * W)); CU(h, gpos.alloc((size_t)stride * W));
        CU(h, key0.alloc((size_t)m)); CU(h, key1.alloc((size_t)m)); CU(h, tag0.alloc((size_t)m)); CU(h, tag1.alloc((size_t)m)); CU(h, d_u.alloc(1));
        const size_t tb = idmap_merge_tmp_bytes((int)m, st);
        CU(h, tmp.alloc(std::max<size_t>(tb, 1)));
        if (s.u > 0) {
            CU(h, cudaMemcpyAsync(sid, s.k0, sizeof(unsigned long long) * (size_t)s.u, cudaMemcpyDeviceToDevice, st));
            CU(h, cudaMemcpyAsync(spos, s.p0, sizeof(int) * (size_t)s.u, cudaMemcpyDeviceToDevice, st));
        }
        int rc = CTR_OK;
        RET(launch(h, "idmap_gather_ranks", [&] { rc = comm_gather_lists(h, spos, gpos, sizeof(int), nullptr, nullptr, (size_t)stride); }));
        RET(rc);
        RET(launch(h, "idmap_gather_ranks", [&] { rc = comm_gather_lists(h, sid, gid, sizeof(unsigned long long), nullptr, nullptr, (size_t)stride); }));
        RET(rc);
        int u = 0;
        cudaError_t e = cudaSuccess;
        RET(launch(h, "idmap_merge_ranks", [&] { e = idmap_merge_ranks(gid, gpos, (long)stride, L, W, key0, key1, tag0, tag1, d_u, tmp, tb, G, st, &u); }));
        CU(h, e);
        if (R + u > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "idmap insert: %lld ids + %d new ones exceed INT32_MAX rows", (long long)R, u);
        RET(idmap_add(h, which, key1, u, d_ids, n, d_rows, rows && s.m > 0));
    }
    if (rows && n > 0) CU(h, cudaMemcpyAsync(rows, d_rows, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}
}  // namespace

// The ids the map lacks get rows idm_n, idm_n + 1, ... in order of first occurrence (idmap_number), a sort by first
// position being the order.  Only the missing ids are sorted.
int ctr_idmap_insert(ctr_handle* h, int which, const int64_t* ids, int64_t n, int32_t* rows) {
    if (!h) return set_err(h, CTR_EINVAL, "bad idmap insert arguments");
    if (h->comm.world > 1) {
        std::lock_guard<std::mutex> lk(h->mu);
        return idmap_insert_ranks(h, which, ids, n, rows);
    }
    if (!ids || which < 0 || which > 1 || n < 1 || n > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "bad idmap insert arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    for (int64_t i = 0; i < n; i++)
        if ((unsigned long long)ids[i] == kIdEmpty) return set_err(h, CTR_EINVAL, "idmap insert: id INT64_MIN is reserved (position %lld)", (long long)i);
    CU(h, cudaSetDevice(h->dev));
    cudaStream_t st = h->stream;
    const int64_t R = h->idm_n[which];
    long long* d_ids = nullptr; int* d_rows = nullptr; unsigned long long* d_cnt = nullptr;
    RET(scratch_get(h, 0, sizeof(long long) * (size_t)n, (void**)&d_ids)); RET(scratch_get(h, 1, sizeof(int) * (size_t)n, (void**)&d_rows));
    RET(scratch_get(h, 2, 2 * sizeof(unsigned long long), (void**)&d_cnt));
    if (!h->k_flags) RET(dalloc(h, h->k_flags, 1));
    CU(h, big_copy(d_ids, ids, sizeof(int64_t) * (size_t)n, true, st));
    CU(h, cudaMemsetAsync(d_cnt, 0, 2 * sizeof(unsigned long long), st));
    IdmapSide s;
    RET(idmap_number(h, which, d_ids, n, d_rows, d_cnt, &s));
    if (s.m > 0) {
        const int u = s.u;
        if (R + u > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "idmap insert: %lld ids + %d new ones exceed INT32_MAX rows", (long long)R, u);
        // ordered by first position: k1[j] gets row R + j
        RET(launch(h, "idmap_number", [&] { size_t tb = s.tmp.size(); cub::DeviceRadixSort::SortPairs(s.tmp.get(), tb, s.p0.get(), s.p1.get(), s.k0.get(), s.k1.get(), u, 0, 32, st); }));
        RET(idmap_add(h, which, s.k1, u, d_ids, n, d_rows, rows != nullptr));
    }
    if (rows) CU(h, cudaMemcpyAsync(rows, d_rows, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}

int ctr_idmap_download(ctr_handle* h, int which, int64_t* ids, int64_t cap, int64_t* n) {
    if (!h || !n || which < 0 || which > 1) return set_err(h, CTR_EINVAL, "bad idmap download arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    if (!h->idm_keys[which]) return set_err(h, CTR_ESTATE, "idmap %d not built", which);
    *n = h->idm_n[which];
    if (!ids) return CTR_OK;
    if (cap < h->idm_n[which]) return set_err(h, CTR_EINVAL, "idmap download: the map holds %lld ids", (long long)h->idm_n[which]);
    CU(h, cudaSetDevice(h->dev));
    DevBuf<long long> d;
    CU(h, d.alloc((size_t)h->idm_n[which]));
    RET(launch(h, "idmap_download", [&] {
        k_idmap_dump<<<h->num_sms * 8, 256, 0, h->stream>>>(h->idm_keys[which], h->idm_vals[which], h->idm_keys[which].size(), d);
    }));
    CU(h, big_copy(ids, d, sizeof(int64_t) * (size_t)h->idm_n[which], false, h->stream));
    return CTR_OK;
}

namespace {
// A table in growable memory (and ITEM_EMB's moments) grown to nrows rows in place, the new rows zero.  Every buffer is
// mapped first; the row count changes only once all of them hold the new rows.
int table_grow(ctr_handle* h, int which, int64_t nrows) {
    cudaStream_t st = h->stream;
    const int64_t old = h->tab_rows[which];
    const long ld = h->tab_ld[which];
    const bool mom = which == CTR_TABLE_ITEM_EMB && h->emb_m;
    int rc = CTR_OK;
    RET(launch(h, "table_grow", [&] {
        for (GrowBuf<float>* b : {&h->tab_mem[which], mom ? &h->emb_m : nullptr, mom ? &h->emb_v : nullptr})
            if (b && rc == CTR_OK && (rc = grow_buf(h, *b, (size_t)nrows * ld)) == CTR_OK)
                cudaMemsetAsync(b->get() + (size_t)old * ld, 0, (size_t)(nrows - old) * ld * sizeof(float), st);
    }));
    RET(rc);
    h->tab[which] = h->tab_mem[which].get();
    h->tab_rows[which] = h->tab_local_rows[which] = nrows;
    return CTR_OK;
}

// A row-sharded table grown to nrows logical rows: the shard by vmm_grow_rows (vmm.cuh: reallocated at twice its live
// rows when the new ones do not fit, the new rows zero), ITEM_EMB's row-Adam moments in their growable memory.  tab_gen
// is bumped either way (the row count fixes the hot rows and the row-Adam gradient layout), so the next collective call
// republishes the mappings; ITEM_EMB's hot rows are written back into their owners' shards first, whichever table
// grows, since that republish pulls them from there.
int shard_grow(ctr_handle* h, int which, int64_t nrows) {
    Comm& cm = h->comm;
    cudaStream_t st = h->stream;
    RET(comm_hot_writeback(h));        // any table's growth bumps tab_gen, and the republish re-pulls ITEM_EMB's hot rows
    const long ld = h->tab_ld[which];
    const size_t row_b = (size_t)ld * sizeof(float);
    const int64_t old = h->tab_local_rows[which];
    const int64_t local = (nrows - cm.rank + cm.world - 1) / cm.world;
    int rc = CTR_OK;
    RET(launch(h, "table_shard_grow", [&] {
        std::string err;
        if (!vmm_grow_rows(&h->tab_vmm[which], (size_t)old, (size_t)local, row_b, h->dev, st, &err)) { rc = set_err(h, CTR_ENOMEM, "table %d shard (%lld rows): %s", which, (long long)local, err.c_str()); return; }
        h->tab[which] = (float*)h->tab_vmm[which].ptr;
        if (which == CTR_TABLE_ITEM_EMB && h->emb_m && local > old)
            for (GrowBuf<float>* b : {&h->emb_m, &h->emb_v})
                if (rc == CTR_OK && (rc = grow_buf(h, *b, (size_t)local * ld)) == CTR_OK)
                    cudaMemsetAsync(b->get() + (size_t)old * ld, 0, (size_t)(local - old) * row_b, st);
    }));
    RET(rc);
    h->tab_rows[which] = nrows; h->tab_local_rows[which] = local;
    h->tab_gen++;
    return CTR_OK;
}

// World > 1: the result is the single-GPU write of the ranks' (rows, data) concatenated in rank order.  Row ids are
// concatenated on every rank (one broadcast per rank, grouped) and checked for duplicates with the device sort.  A
// replicated table concatenates the data the same way and every rank writes every row; a row-sharded table routes each
// (row, data) to its owner by grouped send / recv, and a row below hot_k (the replicated hot rows of ITEM_EMB) to every
// rank as well.
int table_write_ranks(ctr_handle* h, int which, const int32_t* rows, const float* data, int64_t n, int32_t width) {
    Comm& cm = h->comm;
    const int W = cm.world, me = cm.rank;
    CU(h, cudaSetDevice(h->dev));
    cudaStream_t st = h->stream;
    const int G = h->num_sms * 8;
    const ctr_config& c = h->cfg;
    const bool args_ok = !(which < 0 || which > 2 || n < 0 || n > 0x7fffffffLL || (n > 0 && (!rows || !data)));
    int verdict = args_ok ? CTR_OK : set_err(h, CTR_EINVAL, "bad table write arguments");
    int32_t top = -1;
    if (verdict == CTR_OK) {
        const int want = which == CTR_TABLE_USER_FEAT ? c.uP : which == CTR_TABLE_ITEM_FEAT ? c.cF : c.D;
        if (width != want || width < 1) verdict = set_err(h, CTR_EINVAL, "table %d width %d != model dim %d (rank %d)", which, width, want, me);
    }
    for (int64_t i = 0; verdict == CTR_OK && i < n; i++) {
        if (rows[i] < 0 || rows[i] == 0x7fffffff) verdict = set_err(h, CTR_EINVAL, "table write: row %d outside [0, INT32_MAX) at position %lld of rank %d", rows[i], (long long)i, me);
        top = std::max(top, rows[i]);
    }
    // the table this call starts from must be the same everywhere: rows, width and placement
    CommHdr hd{};
    if (args_ok) { hd.k = which; hd.n = h->tab_rows[which]; hd.mode = h->tab_width[which]; hd.flag = (h->tab[which] ? 1 : 0) | (h->tab_sharded[which] ? 2 : 0); }
    {
        const int rc = comm_agree(h, hd, verdict);
        if (rc != CTR_OK) return rc;
    }
    int64_t all[2 * kMaxPeers];
    const int64_t mine[2] = {n, top};
    RET(comm_gather_i64(h, mine, 2, all));
    int64_t cnt[kMaxPeers], off[kMaxPeers + 1] = {0};
    int64_t gtop = -1;
    for (int j = 0; j < W; j++) { cnt[j] = all[2 * j]; off[j + 1] = off[j] + cnt[j]; gtop = std::max(gtop, all[2 * j + 1]); }
    const int64_t N = off[W];
    if (N == 0) return CTR_OK;
    if (N > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "table write: the ranks write %lld rows in all (more than INT32_MAX)", (long long)N);
    // every rank's row ids, concatenated; a row named twice anywhere is refused everywhere
    DevBuf<int> g_rows;
    CU(h, g_rows.alloc((size_t)N));
    if (n > 0) CU(h, cudaMemcpyAsync(g_rows.get() + off[me], rows, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, st));
    int rc = CTR_OK;
    RET(launch(h, "table_write_ranks", [&] { rc = comm_concat(h, g_rows, sizeof(int), cnt, off); }));
    RET(rc);
    if (N > 1) {
        DevBuf<int> sorted, d_dup; DevBuf<unsigned char> tmp;
        CU(h, sorted.alloc((size_t)N)); CU(h, d_dup.alloc(1));
        int bits = 1; while (bits < 31 && (gtop >> bits) != 0) bits++;
        size_t tb = 0;
        CU(h, cub::DeviceRadixSort::SortKeys(nullptr, tb, g_rows.get(), sorted.get(), (int)N, 0, bits, st));
        CU(h, tmp.alloc(tb));
        CU(h, cudaMemsetAsync(d_dup, 0, sizeof(int), st));
        RET(launch(h, "table_write_check", [&] { size_t b = tmp.size(); cub::DeviceRadixSort::SortKeys(tmp.get(), b, g_rows.get(), sorted.get(), (int)N, 0, bits, st); }));
        RET(launch(h, "table_write_check", [&] { k_rows_dup<<<G, 256, 0, st>>>(sorted, (long)N, d_dup); }));
        int dup = 0;
        CU(h, cudaMemcpyAsync(&dup, d_dup, sizeof dup, cudaMemcpyDeviceToHost, st)); CU(h, cudaStreamSynchronize(st));
        if (dup) return set_err(h, CTR_EINVAL, "table write: a row appears twice across the ranks' rows");
    }
    // growth: no table yet takes ctr_table_upload's placement for the size; a table keeps its placement when it grows
    const int64_t nrows = gtop + 1;
    if (!h->tab[which]) RET(table_alloc(h, which, nrows, width));
    else if (nrows > h->tab_rows[which]) RET(h->tab_sharded[which] ? shard_grow(h, which, nrows) : table_grow(h, which, nrows));
    const size_t row_b = (size_t)width * sizeof(float);
    float* mo = which == CTR_TABLE_ITEM_EMB && h->emb_m ? h->emb_m.get() : nullptr;
    float* vo = mo ? h->emb_v.get() : nullptr;
    if (!h->tab_sharded[which]) {
        DevBuf<float> g_data;
        CU(h, g_data.alloc((size_t)N * width));
        if (n > 0) CU(h, big_copy(g_data.get() + (size_t)off[me] * width, data, (size_t)n * row_b, true, st));
        RET(launch(h, "table_write_ranks", [&] { rc = comm_concat(h, g_data, row_b, cnt, off); }));
        RET(rc);
        RET(launch(h, "table_write_rows", [&] {
            k_table_write_rows<<<(int)std::min<int64_t>((N + 7) / 8, G), 256, 0, st>>>(h->tab[which], h->tab_ld[which], g_rows, g_data, (long)N, width, mo, vo);
        }));
        CU(h, cudaStreamSynchronize(st));
        return CTR_OK;
    }
    // row-sharded: this rank's rows by destination (the owner, and every rank for a hot row while the replica is live)
    const bool hot = which == CTR_TABLE_ITEM_EMB && cm.hot_k > 0 && cm.hot_tab && cm.published_gen == h->tab_gen;
    const int hot_k = hot ? cm.hot_k : 0;
    int64_t scnt[kMaxPeers] = {}, soff[kMaxPeers + 1] = {0};
    std::vector<int32_t> s_rows; std::vector<float> s_data;
    for (int k = 0; k < W; k++) {
        for (int64_t i = 0; i < n; i++)
            if (rows[i] % W == k || rows[i] < hot_k) {
                s_rows.push_back(rows[i]);
                s_data.insert(s_data.end(), data + (size_t)i * width, data + (size_t)(i + 1) * width);
                scnt[k]++;
            }
        soff[k + 1] = soff[k] + scnt[k];
    }
    int64_t allc[kMaxPeers * kMaxPeers];
    RET(comm_gather_i64(h, scnt, W, allc));             // allc[j·W + k]: what rank j sends rank k
    int64_t rcnt[kMaxPeers], roff[kMaxPeers + 1] = {0};
    for (int j = 0; j < W; j++) { rcnt[j] = allc[j * W + me]; roff[j + 1] = roff[j] + rcnt[j]; }
    const int64_t ns = soff[W], nr = roff[W];
    DevBuf<int> d_srows, d_rrows; DevBuf<float> d_sdata, d_rdata;
    CU(h, d_srows.alloc((size_t)std::max<int64_t>(ns, 1))); CU(h, d_sdata.alloc((size_t)std::max<int64_t>(ns, 1) * width));
    CU(h, d_rrows.alloc((size_t)std::max<int64_t>(nr, 1))); CU(h, d_rdata.alloc((size_t)std::max<int64_t>(nr, 1) * width));
    if (ns > 0) {
        CU(h, cudaMemcpyAsync(d_srows, s_rows.data(), sizeof(int32_t) * (size_t)ns, cudaMemcpyHostToDevice, st));
        CU(h, big_copy(d_sdata, s_data.data(), (size_t)ns * row_b, true, st));
    }
    RET(launch(h, "table_write_ranks", [&] {
        rc = comm_route(h, d_srows, scnt, soff, d_rrows, rcnt, roff, sizeof(int));
        if (rc == CTR_OK) rc = comm_route(h, d_sdata, scnt, soff, d_rdata, rcnt, roff, row_b);
    }));
    RET(rc);
    if (nr > 0) {
        float* hm = hot && cm.hot_m ? cm.hot_m.get() : nullptr;
        RET(launch(h, "table_write_shard", [&] {
            k_shard_write_rows<<<(int)std::min<int64_t>((nr + 7) / 8, G), 256, 0, st>>>(h->tab[which], h->tab_ld[which], d_rrows, d_rdata, (long)nr, width, W, me,
                                                                                      mo, vo, hot ? cm.hot_tab.get() : nullptr, hot_k, hm, hm ? cm.hot_v.get() : nullptr);
        }));
    }
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}
}  // namespace

// Rows are written in place; a row past the end grows the table (and ITEM_EMB's moments) in its growable memory, the
// gap zeroed.  Validation (ranges on the host, duplicates by a device sort) comes before any write to the table.
int ctr_table_write_rows(ctr_handle* h, int which, const int32_t* rows, const float* data, int64_t n, int32_t width) {
    if (!h) return set_err(h, CTR_EINVAL, "bad table write arguments");
    if (h->comm.world > 1) {
        std::lock_guard<std::mutex> lk(h->mu);
        return table_write_ranks(h, which, rows, data, n, width);
    }
    if (!rows || !data || which < 0 || which > 2 || n < 1 || n > 0x7fffffffLL) return set_err(h, CTR_EINVAL, "bad table write arguments");
    std::lock_guard<std::mutex> lk(h->mu);
    const ctr_config& c = h->cfg;
    const int want = which == CTR_TABLE_USER_FEAT ? c.uP : which == CTR_TABLE_ITEM_FEAT ? c.cF : c.D;
    if (width != want || width < 1) return set_err(h, CTR_EINVAL, "table %d width %d != model dim %d", which, width, want);
    int32_t top = -1;
    for (int64_t i = 0; i < n; i++) {
        if (rows[i] < 0 || rows[i] == 0x7fffffff) return set_err(h, CTR_EINVAL, "table write: row %d outside [0, INT32_MAX) at position %lld", rows[i], (long long)i);
        top = std::max(top, rows[i]);
    }
    CU(h, cudaSetDevice(h->dev));
    cudaStream_t st = h->stream;
    const int G = h->num_sms * 8;
    DevBuf<int> d_rows;
    CU(h, d_rows.alloc((size_t)n));
    CU(h, big_copy(d_rows, rows, sizeof(int32_t) * (size_t)n, true, st));
    if (n > 1) {
        DevBuf<int> sorted, d_dup; DevBuf<unsigned char> tmp;
        CU(h, sorted.alloc((size_t)n)); CU(h, d_dup.alloc(1));
        int bits = 1; while (bits < 31 && (top >> bits) != 0) bits++;
        size_t tb = 0;
        CU(h, cub::DeviceRadixSort::SortKeys(nullptr, tb, d_rows.get(), sorted.get(), (int)n, 0, bits, st));
        CU(h, tmp.alloc(tb));
        CU(h, cudaMemsetAsync(d_dup, 0, sizeof(int), st));
        RET(launch(h, "table_write_check", [&] { size_t b = tmp.size(); cub::DeviceRadixSort::SortKeys(tmp.get(), b, d_rows.get(), sorted.get(), (int)n, 0, bits, st); }));
        RET(launch(h, "table_write_check", [&] { k_rows_dup<<<G, 256, 0, st>>>(sorted, (long)n, d_dup); }));
        int dup = 0;
        CU(h, cudaMemcpyAsync(&dup, d_dup, sizeof dup, cudaMemcpyDeviceToHost, st)); CU(h, cudaStreamSynchronize(st));
        if (dup) return set_err(h, CTR_EINVAL, "table write: a row appears twice");
    }
    const int64_t nrows = (int64_t)top + 1;
    if (!h->tab[which]) RET(table_alloc(h, which, nrows, width));
    else if (nrows > h->tab_rows[which]) RET(table_grow(h, which, nrows));
    // host rows in chunks: through two pinned buffers (the caller's may be pageable) into two device slots
    const size_t row_b = (size_t)width * sizeof(float), total = (size_t)n * row_b;
    const size_t kChunk = (size_t)32 << 20;
    const int64_t per = (int64_t)std::max<size_t>(1, kChunk / row_b);
    const bool pinned = total >= ((size_t)8 << 20);
    const size_t slot = std::min<size_t>((size_t)per, (size_t)n) * row_b;
    PinnedBuf<unsigned char> pin[2]; DevBuf<unsigned char> stage[2]; Event ev[2];
    for (int b = 0; b < 2; b++) {
        CU(h, stage[b].alloc(slot)); CU(h, ev[b].create(cudaEventDisableTiming));
        if (pinned) CU(h, pin[b].alloc(slot));
    }
    std::unique_ptr<CopyPool> pool;
    if (pinned) pool.reset(new CopyPool(7));
    float* mo = which == CTR_TABLE_ITEM_EMB && h->emb_m ? h->emb_m.get() : nullptr;
    float* vo = mo ? h->emb_v.get() : nullptr;
    for (int64_t r0 = 0, k = 0; r0 < n; r0 += per, k++) {
        const int b = (int)(k & 1);
        const int64_t nr = std::min<int64_t>(per, n - r0);
        const char* src = (const char*)data + (size_t)r0 * row_b;
        if (k >= 2) CU(h, cudaEventSynchronize(ev[b]));
        if (pinned) { pool->copy(pin[b], src, (size_t)nr * row_b); src = (const char*)pin[b].get(); }
        CU(h, cudaMemcpyAsync(stage[b], src, (size_t)nr * row_b, cudaMemcpyHostToDevice, st));
        RET(launch(h, "table_write_rows", [&] {
            k_table_write_rows<<<(int)std::min<int64_t>((nr + 7) / 8, G), 256, 0, st>>>(h->tab[which], h->tab_ld[which], d_rows.get() + r0,
                                                                                                   (const float*)stage[b].get(), (long)nr, width, mo, vo);
        }));
        CU(h, cudaEventRecord(ev[b], st));
    }
    CU(h, cudaStreamSynchronize(st));
    return CTR_OK;
}

// ---- model/mlp: the float64 MLP classifier and regressor (row a11) -------------------------------------------
struct ctr_mlp {
    ctr_mlp_config cfg{};
    ctr_mlp_options opts{};
    Mlp64Dims d{};
    long np = 0;
    int dev = 0, num_sms = 132;
    Stream stream;
    mutable std::string err;
    std::mutex mu;
    DevBuf<double> params, grads, ms, vs;                             // sgd keeps its velocities in ms
    DevBuf<double> act[kMlpMaxLayers], del[kMlpMaxLayers];           // [rows, units[l]]
    DevBuf<double> X64; DevBuf<float> Y32; DevBuf<long> idx;
    DevBuf<double> scal;                                              // [0] batch loss, [1] epoch accumulator
    // key-fed fit / predict: [rows, nin] float64 inputs a feature store gathers (two, so minibatch k+1 is gathered on the
    // store's stream while k trains); stage_free[s]: the minibatch that last read stage[s] is done; stage_full[s]: gathered
    DevBuf<double> stage[2]; Event stage_free[2], stage_full[2];
    // LabelBinarizer64.Classes (basemlp64.go:1294-1313): empty for labels all 0 or 1 (no binarizer, one logistic output).
    // Otherwise the output width is max(1, classes.size()) and predictions are class labels.  class_dev mirrors it.
    std::vector<double> classes;
    DevBuf<double> class_dev;                                         // [kMlpMaxClasses]
    DevBuf<int> cls;                                                  // [n] the class index of each sample of the last fit
    bool regressor = false;                                           // MLPRegressor: no labels, targets [n, units[L-1]]
    int out_kind = CTR_MLP_OUT_LOGISTIC;                              // OutActivation; d.out_act mirrors it
    double adam_calls = 0;                                           // AdamOptimizer64.t
    double t = 0;                                                     // BaseMultilayerPerceptron64.t: samples since initialize (:412,814)
    bool fitted = false;
};
namespace {
int mlp_err(const ctr_mlp* m, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (m) m->err = buf; else g_create_error = buf;
    return code;
}
#define MCU(m, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return mlp_err(m, e_ == cudaErrorMemoryAllocation ? CTR_ENOMEM : CTR_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)
int mlp_grid(const ctr_mlp* m, long work) { return (int)std::max<long>(1, std::min<long>((work + 255) / 256, (long)m->num_sms * 8)); }
// grow-only; every layer's pair is checked, so a failed growth is redone by the next call
int mlp_rows(ctr_mlp* m, long rows) {
    for (int l = 1; l < m->d.n_layers; l++) {
        const size_t n = (size_t)rows * m->d.units[l];
        if (m->act[l].size() < n) MCU(m, m->act[l].alloc(n));
        if (m->del[l].size() < n) MCU(m, m->del[l].alloc(n));
    }
    return CTR_OK;
}
// f32 host matrix → f64 device matrix (mlp.go:47-52 / :17-29), through a bounded f32 staging buffer
int mlp_upload_x(ctr_mlp* m, const float* X, int64_t n, int nin) {
    const size_t need = (size_t)n * nin;
    if (m->X64.size() < need) MCU(m, m->X64.alloc(need));
    const size_t chunk = std::min<size_t>(need, (size_t)16 << 20);
    DevBuf<float> st;
    MCU(m, st.alloc(chunk));
    int rc = CTR_OK;
    for (size_t o = 0; o < need && rc == CTR_OK; o += chunk) {
        const size_t c = std::min(chunk, need - o);
        if (cudaMemcpyAsync(st, X + o, c * sizeof(float), cudaMemcpyHostToDevice, m->stream) != cudaSuccess) { rc = mlp_err(m, CTR_ECUDA, "upload X: %s", cudaGetErrorString(cudaGetLastError())); break; }
        k_f32_to_f64<<<mlp_grid(m, (long)c), 256, 0, m->stream>>>(st, m->X64 + o, (long)c);
        if (cudaStreamSynchronize(m->stream) != cudaSuccess) rc = mlp_err(m, CTR_ECUDA, "upload X: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return rc;
}
// forwardPass (basemlp64.go:259-275) over m rows; layer 0 reads the [*, nin] matrix X through idx (may be null = identity).
// A softmax output keeps the output layer's pre-activations and normalises them after (:504-511).
void mlp_forward(ctr_mlp* m, const double* X, const long* idx, int rows) {
    const int L = m->d.n_layers, nin = m->d.units[0], no = m->d.units[L - 1];
    const bool softmax = m->out_kind == CTR_MLP_OUT_SOFTMAX;
    auto layer = softmax ? k_mlp64_layer<true> : k_mlp64_layer<false>;
    for (int l = 0; l + 1 < L; l++)
        layer<<<mlp_grid(m, (long)rows * m->d.units[l + 1]), 256, 0, m->stream>>>(m->params, m->d, l, X, nin, idx,
                                                                              l == 0 ? nullptr : m->act[l].get(), m->act[l + 1], rows);
    if (softmax) k_mlp64_softmax<<<mlp_grid(m, rows), 256, 0, m->stream>>>(m->act[L - 1], rows, no);
}
// the float32 answer of predict from the output layer: without classes the output layer itself, [rows, units[L-1]] (the
// probability of a binary classifier, a regressor's values), with classes the class label [rows] (:917-931)
void mlp_output(ctr_mlp* m, int rows, float* out) {
    const int L = m->d.n_layers;
    if (m->classes.empty()) k_f64_to_f32<<<mlp_grid(m, (long)rows * m->d.units[L - 1]), 256, 0, m->stream>>>(m->act[L - 1], out, (long)rows * m->d.units[L - 1]);
    else k_mlp64_predict_label<<<mlp_grid(m, rows), 256, 0, m->stream>>>(m->act[L - 1], rows, m->d.units[L - 1], m->class_dev, out);
}
void mlp_set_out(ctr_mlp* m, int kind) {
    m->out_kind = kind;
    m->d.out_act = kind == CTR_MLP_OUT_LOGISTIC ? MLP_ACT_LOGISTIC : MLP_ACT_IDENTITY;
}
// installs the classes (empty: binary) and the output width they imply; parameters, gradients and moments are
// reallocated, zero, when the width changes, and the model then counts as not fitted.  Nothing changes on a failure.
int mlp_set_head(ctr_mlp* m, const std::vector<double>& classes) {
    const int L = m->d.n_layers, no = std::max<int>(1, (int)classes.size());
    const long np = m->d.off[L - 2] + (long)(1 + m->d.units[L - 2]) * no;
    DevBuf<double> b[4];
    if (no != m->d.units[L - 1])
        for (DevBuf<double>& x : b) { MCU(m, x.alloc((size_t)np)); MCU(m, cudaMemsetAsync(x, 0, sizeof(double) * (size_t)np, m->stream)); }
    if (!classes.empty() && !m->class_dev) MCU(m, m->class_dev.alloc(kMlpMaxClasses));
    if (!classes.empty()) MCU(m, cudaMemcpyAsync(m->class_dev, classes.data(), sizeof(double) * classes.size(), cudaMemcpyHostToDevice, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    if (no != m->d.units[L - 1]) {
        m->params = std::move(b[0]); m->grads = std::move(b[1]); m->ms = std::move(b[2]); m->vs = std::move(b[3]);
        m->d.units[L - 1] = no;
        m->np = np;
        m->fitted = false;
    }
    m->classes = classes;
    mlp_set_out(m, classes.size() > 1 ? CTR_MLP_OUT_SOFTMAX : CTR_MLP_OUT_LOGISTIC);
    return CTR_OK;
}
// BaseMultilayerPerceptron64.Fit's label handling (basemlp64.go:578-598) over the n labels Y of a fit, on the device:
// isBinarized64 (:1378-1388) and LabelBinarizer64.Fit (:1294-1313).  At a cold initialise the head follows the labels;
// a warm start keeps it and refuses labels whose class set differs.  With classes, *cls = each sample's class index
// (m->cls), else null.  The host reads the class count back once.  A refusal changes nothing.
int mlp_labels(ctr_mlp* m, const float* Y, long n, const int** cls) {
    *cls = nullptr;
    size_t t_tmp = 0;
    MCU(m, class_sort_unique<float>(nullptr, &t_tmp, nullptr, nullptr, nullptr, nullptr, nullptr, n, m->stream));
    DevBuf<float> k0, k1; DevBuf<long> p0, p1; DevBuf<char> tmp; DevBuf<Mlp64Classes> res;
    MCU(m, k0.alloc((size_t)n)); MCU(m, k1.alloc((size_t)n)); MCU(m, p0.alloc((size_t)n)); MCU(m, p1.alloc((size_t)n));
    MCU(m, tmp.alloc(t_tmp)); MCU(m, res.alloc(1));
    MCU(m, cudaMemsetAsync(res, 0, sizeof(Mlp64Classes), m->stream));
    k_mlp64_label_keys<<<mlp_grid(m, n), 256, 0, m->stream>>>(Y, n, k0, p0, res);
    // the stable sort leaves each class's first position at the head of its run; the unique keys go to k0, their positions to p0
    MCU(m, class_sort_unique<float>(tmp.get(), &t_tmp, k0.get(), k1.get(), p0.get(), p1.get(), &res.get()->count, n, m->stream));
    k_class_values<float><<<kMlpMaxClasses / 256, 256, 0, m->stream>>>(Y, p0, &res.get()->count, kMlpMaxClasses, res.get()->value);
    std::unique_ptr<Mlp64Classes> r(new Mlp64Classes);
    MCU(m, cudaMemcpyAsync(r.get(), res, sizeof(Mlp64Classes), cudaMemcpyDeviceToHost, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    MCU(m, cudaGetLastError());
    if (r->nan) return mlp_err(m, CTR_EINVAL, "a label is NaN: the classes would be ill-defined (DESIGN.md §2)");
    if (r->count > kMlpMaxClasses) return mlp_err(m, CTR_EINVAL, "%ld distinct labels: at most %d classes", r->count, kMlpMaxClasses);
    std::vector<double> classes(r->value, r->value + r->count);
    if (std::all_of(classes.begin(), classes.end(), [](double v) { return v == 0.0 || v == 1.0; })) classes.clear();   // isBinarized64
    if (m->cfg.warm_start && m->fitted) {                                // the head is kept; the binarizer is refitted (:592-597)
        const bool same = classes.size() == m->classes.size() && std::equal(classes.begin(), classes.end(), m->classes.begin());
        if (!same) return mlp_err(m, CTR_EINVAL, "warm start: the labels have %zu classes%s, the fitted model %zu (0 = labels in {0, 1}); the classes must match",
                                  classes.size(), classes.size() == m->classes.size() ? " of other values" : "", m->classes.size());
    }
    if (!classes.empty() && m->cls.size() < (size_t)n) MCU(m, m->cls.alloc((size_t)n));
    RET(mlp_set_head(m, classes));
    if (classes.empty()) return CTR_OK;
    k_mlp64_class_index<<<mlp_grid(m, n), 256, 0, m->stream>>>(Y, n, m->class_dev, (int)classes.size(), m->cls);
    *cls = m->cls;
    return CTR_OK;
}
// MLPRegressor.Fit's targets (basemlp64.go:495-511): Y [n·no] on the device, one pass that flags a target not 0 or 1
// and a non-finite one; the host reads back the two flags.  A cold initialise decides the output from them; a warm start
// of a fitted model keeps its output.  A NaN or ±inf target is refused and changes nothing (DESIGN.md §2).
int mlp_targets(ctr_mlp* m, const float* Y, long n) {
    DevBuf<int> fl;
    MCU(m, fl.alloc(2));
    MCU(m, cudaMemsetAsync(fl, 0, 2 * sizeof(int), m->stream));
    k_mlp64_target_flags<<<mlp_grid(m, n), 256, 0, m->stream>>>(Y, n, fl);
    int f[2] = {0, 0};
    MCU(m, cudaMemcpyAsync(f, fl, sizeof f, cudaMemcpyDeviceToHost, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    MCU(m, cudaGetLastError());
    if (f[1]) return mlp_err(m, CTR_EINVAL, "a target is NaN or infinite (DESIGN.md §2)");
    if (m->cfg.warm_start && m->fitted) return CTR_OK;
    const int no = m->d.units[m->d.n_layers - 1];
    mlp_set_out(m, f[0] ? CTR_MLP_OUT_IDENTITY : no == 1 ? CTR_MLP_OUT_LOGISTIC : CTR_MLP_OUT_SOFTMAX);
    return CTR_OK;
}
// the two [rows, nin] staging buffers and their events of the key-fed entry points (grow-only; events made once)
int mlp_stage(ctr_mlp* m, long rows) {
    const size_t n = (size_t)rows * m->d.units[0];
    for (int s = 0; s < 2; s++) if (m->stage[s].size() < n) MCU(m, m->stage[s].alloc(n));
    if (!m->stage_full[1]) {
        Event fr[2], fu[2];
        for (int s = 0; s < 2; s++) { MCU(m, fr[s].create(cudaEventDisableTiming)); MCU(m, fu[s].create(cudaEventDisableTiming)); }
        for (int s = 0; s < 2; s++) { m->stage_free[s] = std::move(fr[s]); m->stage_full[s] = std::move(fu[s]); }
    }
    return CTR_OK;
}
// initialize, basemlp64.go:459-476, unless a warm start keeps the fitted parameters
int mlp_init_params(ctr_mlp* m) {
    const ctr_mlp_config& c = m->cfg;
    if (c.warm_start && m->fitted) return CTR_OK;
    // every packed element (intercepts too) = U[0,1)·sqrt(f/(fi+fo)), f = 6, or 2 for a logistic hidden activation —
    // non-negative; counter RNG instead of the reference's time-seeded source
    std::vector<double> p((size_t)m->np);
    long pos = 0;
    for (int l = 0; l + 1 < m->d.n_layers; l++) {
        const int fi = m->d.units[l], fo = m->d.units[l + 1];
        const double bound = std::sqrt((c.hidden_act == CTR_MLP_LOGISTIC ? 2.0 : 6.0) / (double)(fi + fo));
        const long end = pos + (long)(1 + fi) * fo;
        for (; pos < end; pos++) p[(size_t)pos] = (double)(mix64(c.seed, 7, (uint64_t)pos) >> 11) * (1.0 / 9007199254740992.0) * bound;
    }
    MCU(m, cudaMemcpyAsync(m->params, p.data(), sizeof(double) * (size_t)m->np, cudaMemcpyHostToDevice, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    m->t = 0;                                                            // :412
    return CTR_OK;
}
// Layer 0's input of minibatch k (0-based within the epoch), whose samples are bi[0, rows): *X = a [rows, nin] matrix
// read row by row, or left null to read X64 through bi (ctr_mlp_fit).
using MlpInput = std::function<int(long k, const long* bi, int rows, const double** X)>;
// fitStochastic (basemlp64.go:729-857) over n samples with the device targets Y [n, units[L-1]] (binary labels or a
// regressor's targets) or class indices cls [n] (mlp_labels; cls non-null), in minibatches of bs: a fresh optimizer,
// the per-epoch shuffle, the solvers, weight decay, the stopping rules and the t carry.  Only layer 0's input differs
// between the callers (input may be empty).  m->idx holds n entries and the activations bs rows.
int mlp_epochs(ctr_mlp* m, long n, long bs, const float* Y, const int* cls, const MlpInput& input, int32_t* n_iter, double* loss_curve) {
    const ctr_mlp_config& c = m->cfg;
    const int nin = m->d.units[0];
    const ctr_mlp_options& o = m->opts;
    const bool sgd = o.solver == CTR_MLP_SOLVER_SGD;
    MCU(m, cudaMemsetAsync(m->ms, 0, sizeof(double) * (size_t)m->np, m->stream));        // a fresh optimizer per fit (:731-752)
    MCU(m, cudaMemsetAsync(m->vs, 0, sizeof(double) * (size_t)m->np, m->stream));
    m->adam_calls = 0;
    double sgd_lr = c.lr_init;                                           // SGDOptimizer64.LearningRate
    std::vector<long> idx((size_t)n);
    for (long i = 0; i < n; i++) idx[(size_t)i] = i;
    double lr_init = c.lr_init, lr_last = c.lr_init, best = INFINITY;
    int no_improve = 0, it = 0;
    const int L = m->d.n_layers;
    for (it = 0; it < c.max_iter;) {
        if (c.shuffle) {                                                 // rand.Shuffle (:788): Fisher–Yates from the top
            for (long i = n - 1; i > 0; i--) { const long j = (long)(mix64(c.seed, 100u + (uint32_t)it, (uint64_t)i) % (uint64_t)(i + 1)); std::swap(idx[(size_t)i], idx[(size_t)j]); }
        }
        MCU(m, cudaMemcpyAsync(m->idx, idx.data(), sizeof(long) * (size_t)n, cudaMemcpyHostToDevice, m->stream));
        MCU(m, cudaMemsetAsync(m->scal, 0, 2 * sizeof(double), m->stream));
        for (long b0 = 0; b0 < n; b0 += bs) {                            // :791-808
            const int rows = (int)std::min<long>(bs, n - b0);
            const long* bi = m->idx + b0;
            const double* X0 = nullptr;
            if (input) RET(input(b0 / bs, bi, rows, &X0));
            const long* xi = X0 ? nullptr : bi;
            if (!X0) X0 = m->X64;
            if (o.weight_decay > 0.0)                                    // backprop :342-346
                k_mlp64_decay<<<mlp_grid(m, m->np), 256, 0, m->stream>>>(m->params, m->np, 1.0 - o.weight_decay);
            mlp_forward(m, X0, xi, rows);
            if (cls) k_mlp64_loss_cls<<<1, 256, 0, m->stream>>>(m->params, m->d, m->act[L - 1], cls, bi, rows, c.alpha, m->del[L - 1], m->scal, m->scal + 1);
            else if (m->out_kind == CTR_MLP_OUT_LOGISTIC) k_mlp64_loss<<<1, 256, 0, m->stream>>>(m->params, m->d, m->act[L - 1], Y, bi, rows, c.alpha, m->del[L - 1], m->scal, m->scal + 1);
            else k_mlp64_loss_dense<<<1, 256, 0, m->stream>>>(m->params, m->d, m->act[L - 1], Y, bi, rows, c.alpha, m->out_kind == CTR_MLP_OUT_IDENTITY,
                                                              m->del[L - 1], m->scal, m->scal + 1);
            for (int l = L - 2; l >= 0; l--) {                           // backprop :382-402
                k_mlp64_grads<<<mlp_grid(m, (long)(m->d.units[l] + 1) * m->d.units[l + 1]), 256, 0, m->stream>>>(
                    m->params, m->grads, m->d, l, X0, nin, xi, l == 0 ? nullptr : m->act[l].get(), m->del[l + 1], rows, c.alpha);
                if (l >= 1) k_mlp64_delta<<<mlp_grid(m, (long)rows * m->d.units[l]), 256, 0, m->stream>>>(m->params, m->d, l, m->act[l], m->del[l + 1], m->del[l], rows);
            }
            if (sgd) {
                k_mlp64_sgd<<<mlp_grid(m, m->np), 256, 0, m->stream>>>(m->params, m->grads, m->ms, m->np, sgd_lr, o.momentum, o.nesterov);
            } else {
                k_mlp64_adam<<<mlp_grid(m, m->np), 256, 0, m->stream>>>(m->params, m->grads, m->ms, m->vs, m->np, m->adam_calls, lr_init, c.beta1, c.beta2, c.eps);
                m->adam_calls += 1;
            }
        }
        it++;
        double sc[2] = {0, 0};
        MCU(m, cudaMemcpyAsync(sc, m->scal, sizeof sc, cudaMemcpyDeviceToHost, m->stream));
        MCU(m, cudaStreamSynchronize(m->stream));
        MCU(m, cudaGetLastError());
        const double loss = sc[1] / (double)n;                           // :810-811
        m->t += (double)n;                                               // :814
        if (loss_curve) loss_curve[it - 1] = loss;
        if (!sgd) {   // the learning rate the optimizer last used (:1088): decides "adaptive" stopping (:1059-1064)
            const double e = m->adam_calls * (double)m->np;
            lr_last = lr_init * std::sqrt(1.0 - std::pow(c.beta2, e)) / (1.0 - std::pow(c.beta1, e));
        }
        if (loss > best - c.tol) no_improve++; else no_improve = 0;      // :886-892
        if (loss < best) best = loss;
        if (sgd && o.lr_schedule == CTR_MLP_LR_INVSCALING)               // iterationEnds :999-1003 (Adam's is a no-op, :1053)
            sgd_lr = c.lr_init / std::pow(m->t + 1.0, o.power_t);
        if (no_improve > c.n_iter_no_change) {                           // :826-840
            if (o.lr_schedule != CTR_MLP_LR_ADAPTIVE) break;             // triggerStopping :1005-1011, :1054-1060
            if ((sgd ? sgd_lr : lr_last) <= 1e-6) break;                 // :1012-1017, :1061-1066
            if (sgd) sgd_lr *= .8;                                       // :1018 — the current rate
            else lr_init *= .8;                                          // :1067 — the base rate
            no_improve = 0;
        }
    }
    if (n_iter) *n_iter = it;
    m->fitted = true;
    return CTR_OK;
}
long mlp_batch(const ctr_mlp* m, long n) {
    long bs = m->cfg.batch;
    if (bs <= 0) bs = n < 200 ? n : 200; else if (bs > n) bs = n;       // basemlp64.go:517-527
    return bs;
}
}  // namespace

void ctr_mlp_options_default(ctr_mlp_options* o) {
    memset(o, 0, sizeof *o);
    o->solver = CTR_MLP_SOLVER_ADAM; o->lr_schedule = CTR_MLP_LR_CONSTANT; o->nesterov = 1;     // :229-256
    o->power_t = 0.5; o->momentum = 0.9; o->weight_decay = 0.0;
}
void ctr_mlp_config_default(ctr_mlp_config* c, int32_t n_features) {
    memset(c, 0, sizeof *c);
    c->n_layers = 3; c->units[0] = n_features; c->units[1] = 100; c->units[2] = 1;      // HiddenLayerSizes {100}, basemlp64.go:239
    c->hidden_act = CTR_MLP_RELU; c->batch = 200; c->max_iter = 200; c->n_iter_no_change = 10; c->shuffle = 1;   // :229-254
    c->adaptive = 0; c->warm_start = 0; c->seed = 0; c->device = 0;
    c->alpha = 1e-4; c->lr_init = 1e-3; c->beta1 = 0.9; c->beta2 = 0.999; c->eps = 1e-8; c->tol = 1e-4;
}
const char* ctr_mlp_last_error(const ctr_mlp* m) { return m ? m->err.c_str() : g_create_error.c_str(); }

int ctr_mlp_create(const ctr_mlp_config* cfg, ctr_mlp** out) { return ctr_mlp_create_ex(cfg, nullptr, out); }

namespace {
// NewMLPClassifier / NewMLPRegressor: every argument is checked before the device is looked for
int mlp_create(const ctr_mlp_config* cfg, const ctr_mlp_options* opts, bool regressor, ctr_mlp** out) {
    if (!cfg || !out) return mlp_err(nullptr, CTR_EINVAL, "null argument");
    *out = nullptr;
    const ctr_mlp_config& c = *cfg;
    if (c.n_layers < 2 || c.n_layers > kMlpMaxLayers) return mlp_err(nullptr, CTR_EINVAL, "n_layers must be in [2, %d]", kMlpMaxLayers);
    for (int i = 0; i < c.n_layers; i++) if (c.units[i] < 1) return mlp_err(nullptr, CTR_EINVAL, "layer %d has %d units", i, c.units[i]);
    const int no = c.units[c.n_layers - 1];
    if (regressor && no > kMlpMaxClasses) return mlp_err(nullptr, CTR_EINVAL, "regressor: %d targets, at most %d", no, kMlpMaxClasses);
    if (!regressor && no != 1) return mlp_err(nullptr, CTR_EINVAL, "binary classifier: one output unit (basemlp64.go:423-425)");
    if (c.hidden_act < CTR_MLP_RELU || c.hidden_act > CTR_MLP_TANH || c.max_iter < 1) return mlp_err(nullptr, CTR_EINVAL, "bad activation / max_iter");
    ctr_mlp_options o;
    ctr_mlp_options_default(&o);
    if (opts) o = *opts;
    else if (c.adaptive) o.lr_schedule = CTR_MLP_LR_ADAPTIVE;
    if (o.solver != CTR_MLP_SOLVER_ADAM && o.solver != CTR_MLP_SOLVER_SGD)
        return mlp_err(nullptr, CTR_EINVAL, "solver %d: adam (%d) or sgd (%d); lbfgs is not built", o.solver, CTR_MLP_SOLVER_ADAM, CTR_MLP_SOLVER_SGD);
    if (o.lr_schedule < CTR_MLP_LR_CONSTANT || o.lr_schedule > CTR_MLP_LR_ADAPTIVE)
        return mlp_err(nullptr, CTR_EINVAL, "lr_schedule %d: constant (0), invscaling (1) or adaptive (2)", o.lr_schedule);
    if (c.adaptive && o.lr_schedule != CTR_MLP_LR_ADAPTIVE)
        return mlp_err(nullptr, CTR_EINVAL, "cfg.adaptive is set but the options' lr_schedule is %d, not adaptive", o.lr_schedule);
    if (!(o.momentum >= 0.0 && o.momentum <= 1.0)) return mlp_err(nullptr, CTR_EINVAL, "momentum %g must be in [0, 1] (basemlp64.go:635)", o.momentum);
    if (!(o.weight_decay >= 0.0 && o.weight_decay < 1.0)) return mlp_err(nullptr, CTR_EINVAL, "weight_decay %g must be in [0, 1)", o.weight_decay);
    if (!std::isfinite(o.power_t)) return mlp_err(nullptr, CTR_EINVAL, "power_t must be finite");
    if (o.nesterov != 0 && o.nesterov != 1) return mlp_err(nullptr, CTR_EINVAL, "nesterov must be 0 or 1");
    if (o.reserved0) return mlp_err(nullptr, CTR_EINVAL, "ctr_mlp_options.reserved0 must be 0");
    for (double r : o.reserved) if (r != 0.0) return mlp_err(nullptr, CTR_EINVAL, "ctr_mlp_options.reserved must be 0");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return mlp_err(nullptr, CTR_ENODEV, "no CUDA device: this engine has no CPU fallback"); }
    if (c.device < 0 || c.device >= ndev) return mlp_err(nullptr, CTR_ENODEV, "device %d of %d", c.device, ndev);
    cudaDeviceProp prop{}; cudaGetDeviceProperties(&prop, c.device);
    if (prop.major != 9) return mlp_err(nullptr, CTR_ENODEV, "device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
    ctr_mlp* m = new ctr_mlp();
    m->cfg = c; m->opts = o; m->dev = c.device; m->num_sms = prop.multiProcessorCount;
    m->d.n_layers = c.n_layers; m->d.hidden_act = c.hidden_act;
    m->regressor = regressor;
    mlp_set_out(m, regressor ? CTR_MLP_OUT_IDENTITY : CTR_MLP_OUT_LOGISTIC);
    long off = 0;
    for (int l = 0; l < c.n_layers; l++) { m->d.units[l] = c.units[l]; if (l + 1 < c.n_layers) { m->d.off[l] = off; off += (long)(1 + c.units[l]) * c.units[l + 1]; } }
    m->np = off;
    bool ok = cudaSetDevice(m->dev) == cudaSuccess && m->stream.create() == cudaSuccess;
    for (DevBuf<double>* p : {&m->params, &m->grads, &m->ms, &m->vs}) ok = ok && p->alloc((size_t)m->np) == cudaSuccess && cudaMemset(*p, 0, sizeof(double) * (size_t)m->np) == cudaSuccess;
    ok = ok && m->scal.alloc(2) == cudaSuccess;
    if (!ok) { mlp_err(nullptr, CTR_ECUDA, "ctr_mlp_create: %s", cudaGetErrorString(cudaGetLastError())); ctr_mlp_destroy(m); return CTR_ECUDA; }
    *out = m;
    return CTR_OK;
}
}  // namespace

int ctr_mlp_create_ex(const ctr_mlp_config* cfg, const ctr_mlp_options* opts, ctr_mlp** out) { return mlp_create(cfg, opts, false, out); }
int ctr_mlp_regressor_create(const ctr_mlp_config* cfg, const ctr_mlp_options* opts, ctr_mlp** out) { return mlp_create(cfg, opts, true, out); }

void ctr_mlp_destroy(ctr_mlp* m) {
    if (!m) return;
    cudaSetDevice(m->dev);
    if (m->stream) cudaStreamSynchronize(m->stream);
    delete m;                                         // the members free themselves, this device current
}

int ctr_mlp_get_params(ctr_mlp* m, double* params, int64_t cap, int64_t* np) {
    if (!m) return CTR_EINVAL;
    std::lock_guard<std::mutex> lk(m->mu);
    if (np) *np = m->np;
    if (!params) return CTR_OK;
    if (cap < m->np) return mlp_err(m, CTR_EINVAL, "parameter buffer too small: need %ld", m->np);
    MCU(m, cudaSetDevice(m->dev));
    MCU(m, cudaMemcpyAsync(params, m->params, sizeof(double) * (size_t)m->np, cudaMemcpyDeviceToHost, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    return CTR_OK;
}
int ctr_mlp_set_params(ctr_mlp* m, const double* params, int64_t np) {
    if (!m || !params) return CTR_EINVAL;
    std::lock_guard<std::mutex> lk(m->mu);
    if (np != m->np) return mlp_err(m, CTR_EINVAL, "expected %ld packed parameters, got %lld", m->np, (long long)np);
    MCU(m, cudaSetDevice(m->dev));
    MCU(m, cudaMemcpyAsync(m->params, params, sizeof(double) * (size_t)m->np, cudaMemcpyHostToDevice, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    m->fitted = true;
    return CTR_OK;
}

int ctr_mlp_get_classes(ctr_mlp* m, double* classes, int32_t cap, int32_t* n) {
    if (!m) return CTR_EINVAL;
    std::lock_guard<std::mutex> lk(m->mu);
    const int32_t c = (int32_t)m->classes.size();
    if (n) *n = c;
    if (!classes) return CTR_OK;
    if (cap < c) return mlp_err(m, CTR_EINVAL, "class buffer too small: need %d", c);
    std::copy(m->classes.begin(), m->classes.end(), classes);
    return CTR_OK;
}
// the arguments are checked before the handle, so a refusal's message is readable through ctr_mlp_last_error(m) (or
// ctr_mlp_last_error(NULL) when m is null)
int ctr_mlp_set_classes(ctr_mlp* m, const double* classes, int32_t n) {
    if (n < 0 || n > kMlpMaxClasses || (n > 0 && !classes)) return mlp_err(m, CTR_EINVAL, "n = %d classes: in [0, %d], non-null when n > 0", n, kMlpMaxClasses);
    for (int32_t i = 0; i < n; i++) {
        if (std::isnan(classes[i])) return mlp_err(m, CTR_EINVAL, "class %d is NaN", i);
        if (i > 0 && !(classes[i - 1] < classes[i])) return mlp_err(m, CTR_EINVAL, "the classes must be strictly ascending (class %d)", i);
    }
    if (!m) return mlp_err(nullptr, CTR_EINVAL, "null classifier");
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->regressor) return mlp_err(m, CTR_ESTATE, "a regressor has no classes");
    MCU(m, cudaSetDevice(m->dev));
    RET(mlp_set_head(m, std::vector<double>(classes, classes + n)));
    m->fitted = false;
    return CTR_OK;
}

int ctr_mlp_fit(ctr_mlp* m, const float* X, const float* Y, int64_t n, int32_t xcols, int32_t* n_iter, double* loss_curve) {
    if (!m || !X || !Y || n < 1) return mlp_err(m, CTR_EINVAL, "bad fit arguments");
    std::lock_guard<std::mutex> lk(m->mu);
    const int nin = m->d.units[0];
    if (xcols != nin) return mlp_err(m, CTR_EINVAL, "X has %d columns, the network %d inputs", xcols, nin);
    MCU(m, cudaSetDevice(m->dev));
    const long bs = mlp_batch(m, n);
    const size_t ny = (size_t)n * (m->regressor ? m->d.units[m->d.n_layers - 1] : 1);      // Y [n, no] for a regressor
    RET(mlp_upload_x(m, X, n, nin));
    if (m->Y32.size() < ny) MCU(m, m->Y32.alloc(ny));
    if (m->idx.size() < (size_t)n) MCU(m, m->idx.alloc((size_t)n));
    MCU(m, cudaMemcpyAsync(m->Y32, Y, sizeof(float) * ny, cudaMemcpyHostToDevice, m->stream));
    const int* cls = nullptr;
    if (m->regressor) RET(mlp_targets(m, m->Y32, (long)ny));
    else RET(mlp_labels(m, m->Y32, n, &cls));
    RET(mlp_rows(m, bs));
    RET(mlp_init_params(m));
    return mlp_epochs(m, n, bs, m->Y32, cls, MlpInput(), n_iter, loss_curve);
}

int ctr_mlp_predict(ctr_mlp* m, const float* X, int64_t n, int32_t xcols, float* out) {
    if (!m || !X || !out || n < 1) return mlp_err(m, CTR_EINVAL, "bad predict arguments");
    std::lock_guard<std::mutex> lk(m->mu);
    if (!m->fitted) return mlp_err(m, CTR_ESTATE, "predict before fit");
    const int nin = m->d.units[0];
    if (xcols != nin) return mlp_err(m, CTR_EINVAL, "X has %d columns, the network %d inputs", xcols, nin);
    MCU(m, cudaSetDevice(m->dev));
    RET(mlp_upload_x(m, X, n, nin));
    const long chunk = 8192;
    const int ow = m->classes.empty() ? m->d.units[m->d.n_layers - 1] : 1;   // floats per row of out
    RET(mlp_rows(m, std::min<long>(chunk, n)));
    DevBuf<float> d_out;
    MCU(m, d_out.alloc((size_t)std::min<long>(chunk, n) * ow));
    int rc = CTR_OK;
    for (long r0 = 0; r0 < n && rc == CTR_OK; r0 += chunk) {            // predict :917-931: raw outputs for the f64 class, or class labels
        const int rows = (int)std::min<long>(chunk, n - r0);
        mlp_forward(m, m->X64 + r0 * nin, nullptr, rows);
        mlp_output(m, rows, d_out);
        if (cudaMemcpyAsync(out + r0 * ow, d_out, sizeof(float) * (size_t)rows * ow, cudaMemcpyDeviceToHost, m->stream) != cudaSuccess ||
            cudaStreamSynchronize(m->stream) != cudaSuccess) rc = mlp_err(m, CTR_ECUDA, "predict: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return rc;
}

namespace {
// the float64 output layer [n, units[L-1]] of X, written to out (host or device memory), in chunks of 8192 rows
int mlp_output64(ctr_mlp* m, const float* X, int64_t n, double* out) {
    const int L = m->d.n_layers, nin = m->d.units[0], no = m->d.units[L - 1];
    RET(mlp_upload_x(m, X, n, nin));
    const long chunk = 8192;
    RET(mlp_rows(m, std::min<long>(chunk, n)));
    for (long r0 = 0; r0 < n; r0 += chunk) {
        const int rows = (int)std::min<long>(chunk, n - r0);
        mlp_forward(m, m->X64 + r0 * nin, nullptr, rows);
        MCU(m, cudaMemcpyAsync(out + r0 * no, m->act[L - 1], sizeof(double) * (size_t)rows * no, cudaMemcpyDefault, m->stream));
    }
    MCU(m, cudaStreamSynchronize(m->stream));
    return CTR_OK;
}
}  // namespace

int ctr_mlp_predict_f64(ctr_mlp* m, const float* X, int64_t n, int32_t xcols, double* out) {
    if (!m || !X || !out || n < 1) return mlp_err(m, CTR_EINVAL, "bad predict arguments");
    std::lock_guard<std::mutex> lk(m->mu);
    if (!m->fitted) return mlp_err(m, CTR_ESTATE, "predict before fit");
    if (xcols != m->d.units[0]) return mlp_err(m, CTR_EINVAL, "X has %d columns, the network %d inputs", xcols, m->d.units[0]);
    MCU(m, cudaSetDevice(m->dev));
    return mlp_output64(m, X, n, out);
}

int ctr_mlp_score(ctr_mlp* m, const float* X, const float* Y, int64_t n, int32_t xcols, double* r2) {
    if (!m || !X || !Y || !r2 || n < 1) return mlp_err(m, CTR_EINVAL, "bad score arguments");
    std::lock_guard<std::mutex> lk(m->mu);
    if (!m->regressor) return mlp_err(m, CTR_ESTATE, "score is the regressor's R²; a classifier's accuracy score is ctr_mlp_accuracy");
    if (!m->fitted) return mlp_err(m, CTR_ESTATE, "score before fit");
    if (xcols != m->d.units[0]) return mlp_err(m, CTR_EINVAL, "X has %d columns, the network %d inputs", xcols, m->d.units[0]);
    MCU(m, cudaSetDevice(m->dev));
    const int no = m->d.units[m->d.n_layers - 1];
    const size_t ny = (size_t)n * no;
    DevBuf<double> pred, mean, r, res; DevBuf<float> y; DevBuf<double2> part;
    MCU(m, pred.alloc(ny)); MCU(m, y.alloc(ny)); MCU(m, part.alloc((size_t)no * kR2Parts));
    MCU(m, mean.alloc((size_t)no)); MCU(m, r.alloc(2 * (size_t)no)); MCU(m, res.alloc(3));
    MCU(m, cudaMemcpyAsync(y, Y, sizeof(float) * ny, cudaMemcpyHostToDevice, m->stream));
    RET(mlp_output64(m, X, n, pred));                                     // MLPRegressor.Score → Predict (:64-70)
    k_mlp64_r2_part<float><<<dim3(kR2Parts, no), 256, 0, m->stream>>>(nullptr, y, nullptr, (long)n, no, kR2Mean, nullptr, part);
    k_mlp64_r2_fold<<<1, 256, 0, m->stream>>>(part, no, 0.0, mean, nullptr, nullptr);
    k_mlp64_r2_part<float><<<dim3(kR2Parts, no), 256, 0, m->stream>>>(pred, y, nullptr, (long)n, no, kR2Sums, mean, part);
    k_mlp64_r2_fold<<<1, 256, 0, m->stream>>>(part, no, 0.0, mean, r, res);
    double h[2] = {0, 0};
    MCU(m, cudaMemcpyAsync(h, res, sizeof h, cudaMemcpyDeviceToHost, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    MCU(m, cudaGetLastError());
    if (h[1] >= 0.0) return mlp_err(m, CTR_EINVAL, "target column %d is constant: R² divides by 0 (the reference panics)", (int)h[1]);
    *r2 = h[0];
    return CTR_OK;
}

int ctr_mlp_accuracy(ctr_mlp* m, const float* X, const float* Y, int64_t n, int32_t xcols, double* acc) {
    if (!m || !X || !Y || !acc || n < 1) return mlp_err(m, CTR_EINVAL, "bad accuracy arguments");
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->regressor) return mlp_err(m, CTR_ESTATE, "a regressor's score is R² (ctr_mlp_score)");
    if (!m->fitted) return mlp_err(m, CTR_ESTATE, "accuracy before fit");
    const int L = m->d.n_layers, nin = m->d.units[0], no = m->d.units[L - 1];
    if (xcols != nin) return mlp_err(m, CTR_EINVAL, "X has %d columns, the network %d inputs", xcols, nin);
    MCU(m, cudaSetDevice(m->dev));
    RET(mlp_upload_x(m, X, n, nin));
    DevBuf<float> y; DevBuf<unsigned long long> hits;
    MCU(m, y.alloc((size_t)n)); MCU(m, hits.alloc(1));
    MCU(m, cudaMemcpyAsync(y, Y, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, m->stream));
    MCU(m, cudaMemsetAsync(hits, 0, sizeof(unsigned long long), m->stream));
    const long chunk = 8192;
    RET(mlp_rows(m, std::min<long>(chunk, n)));
    const double* cls = m->classes.empty() ? nullptr : m->class_dev.get();
    for (long r0 = 0; r0 < n; r0 += chunk) {                             // Score → Predict (:127-133), in chunks as ctr_mlp_predict
        const int rows = (int)std::min<long>(chunk, n - r0);
        mlp_forward(m, m->X64 + r0 * nin, nullptr, rows);
        k_mlp64_acc_count<<<mlp_grid(m, rows), 256, 0, m->stream>>>(m->act[L - 1], rows, no, cls, y + r0, hits);
    }
    unsigned long long c = 0;
    MCU(m, cudaMemcpyAsync(&c, hits, sizeof c, cudaMemcpyDeviceToHost, m->stream));
    MCU(m, cudaStreamSynchronize(m->stream));
    MCU(m, cudaGetLastError());
    *acc = (double)c / (double)n;                                         // AccuracyScore64 :1143-1155
    return CTR_OK;
}

int ctr_mlp_get_output(ctr_mlp* m, int32_t* kind) {
    if (!m || !kind) return CTR_EINVAL;
    std::lock_guard<std::mutex> lk(m->mu);
    *kind = m->out_kind;
    return CTR_OK;
}
int ctr_mlp_set_output(ctr_mlp* m, int32_t kind) {
    if (!m) return mlp_err(nullptr, CTR_EINVAL, "null model");
    std::lock_guard<std::mutex> lk(m->mu);
    if (!m->regressor) return mlp_err(m, CTR_ESTATE, "a classifier's output follows its classes (ctr_mlp_set_classes)");
    const int no = m->d.units[m->d.n_layers - 1];
    if (kind != CTR_MLP_OUT_IDENTITY && kind != CTR_MLP_OUT_LOGISTIC && kind != CTR_MLP_OUT_SOFTMAX)
        return mlp_err(m, CTR_EINVAL, "output kind %d: identity (0), logistic (1) or softmax (2)", kind);
    if ((kind == CTR_MLP_OUT_LOGISTIC) != (no == 1) && kind != CTR_MLP_OUT_IDENTITY)
        return mlp_err(m, CTR_EINVAL, "%d targets: 0/1 targets make a logistic output for one target and a softmax for more (basemlp64.go:502-511)", no);
    mlp_set_out(m, kind);
    m->fitted = false;
    return CTR_OK;
}

// ---- the MLP fed by sample keys from a feature store (ctr_mlp_fit_keys / ctr_mlp_predict_keys) -------------
namespace {
// the refusals shared by every key-fed call; h->mu and m->mu are held, m's device is made current.  First this rank's
// own objects, then the feature store's tables: with ITEM_EMB and ITEM_FEAT both replicated (or one GPU) this GPU's
// tables serve alone; a row-sharded ITEM_EMB needs this rank's shard and the communicator (ITEM_FEAT sharded or
// replicated); a replicated ITEM_EMB beside a sharded ITEM_FEAT is refused (check_tables)
int mlp_keys_check(ctr_mlp* m, ctr_handle* h) {
    const ctr_config& c = h->cfg;
    const long width = (long)c.uP + (long)c.S * c.D + c.D + c.cF;
    if (m->dev != h->dev) return mlp_err(m, CTR_EINVAL, "the classifier is on device %d, the feature store on device %d", m->dev, h->dev);
    if (m->d.units[0] != width)
        return mlp_err(m, CTR_EINVAL, "the network has %d inputs, the feature store's samples uP + S*D + D + cF = %ld columns", m->d.units[0], width);
    if (!h->idm_keys[0] || !h->idm_keys[1]) return mlp_err(m, CTR_ESTATE, "the key-fed MLP needs both id maps of the feature store (ctr_idmap_build)");
    MCU(m, cudaSetDevice(m->dev));
    if (!emb_sharded(h)) return check_tables(h);
    RET(comm_check_emb(h));
    return check_widths(h);
}
// the entry of a collective key-fed call (comm_serve_enter on a row-sharded ITEM_EMB, else the agreement alone): a rank
// whose checks failed takes part with its message, and every rank returns the same verdict
int mlp_agree(ctr_mlp* m, ctr_handle* h, CommHdr hd, int verdict) {
    if (verdict != CTR_OK && h->err.empty()) h->err = m->err;
    CU(h, cudaSetDevice(h->dev));        // the checks may have stopped before making it current
    const int rc = emb_sharded(h) ? comm_serve_enter(h, hd, verdict) : comm_agree(h, hd, verdict);
    if (rc != CTR_OK) m->err = h->err;
    return rc;
}
// every exit of a key-fed call: no work of m may still read h's buffers, and the message is readable from both objects
int mlp_keys_done(ctr_mlp* m, ctr_handle* h, int rc) {
    if (m->dev == h->dev) {
        cudaSetDevice(m->dev);
        const cudaError_t e1 = cudaStreamSynchronize(m->stream), e2 = cudaStreamSynchronize(h->stream);
        if (rc == CTR_OK && (e1 != cudaSuccess || e2 != cudaSuccess))
            rc = mlp_err(m, CTR_ECUDA, "key-fed MLP: %s", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
    }
    if (rc != CTR_OK) { if (m->err.empty()) m->err = h->err; else h->err = m->err; }
    return rc;
}
// h's stream has queued what m's stream must see: m's stream waits for it (no host round trip)
int mlp_after_store(ctr_mlp* m, ctr_handle* h, int slot) {
    MCU(m, cudaEventRecord(m->stage_full[slot], h->stream));
    MCU(m, cudaStreamWaitEvent(m->stream, m->stage_full[slot], 0));
    return CTR_OK;
}

// a sample key carries one label: a regressor fed by keys has one target
int mlp_keys_width(ctr_mlp* m) {
    const int no = m->d.units[m->d.n_layers - 1];
    if (m->regressor && no != 1) return mlp_err(m, CTR_EINVAL, "a key-fed regressor has one target, this one %d", no);
    return CTR_OK;
}

// GetSample's resolution of n >= 1 keys, as in ctr_train_keys: the survivors resident in kt_* (input order kept) and,
// when there are any, each one's history GetUserBehavior(uid, S, -1, ts) in kt_hist_all, cut once (h->mu is held, so
// the cache stays as it is).  *used = the survivor count.
int mlp_keys_resolve(ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label, int64_t n,
                     long* used) {
    RET(feed_init(h));
    const size_t chunk = std::min<size_t>((size_t)n, h->feed_bytes / 28);
    RET(keys_prepare(h, (size_t)n, chunk));
    cudaStream_t rs = h->copy_stream;
    const int64_t nchunks = (n + (int64_t)chunk - 1) / (int64_t)chunk;
    for (int64_t c = 0; c < nchunks; c++) RET(keys_resolve_chunk(h, c, chunk, user_ids, item_ids, ts, label, n, rs));
    unsigned long long cnt = 0;
    CU(h, cudaMemcpyAsync(&cnt, h->kt_count, sizeof cnt, cudaMemcpyDeviceToHost, rs));
    CU(h, cudaStreamSynchronize(rs));
    *used = (long)cnt;
    if (cnt == 0) return CTR_OK;
    RET(reserve(h, h->kt_hist_all, (size_t)cnt * h->cfg.S, false));
    return ub_windows(h, h->stream, h->kt_user, h->kt_ts, (int)cnt, h->kt_hist_all);
}

// The classifier over ns resolved samples (user / item rows [ns], history rows [ns, S], labels [ns], on h's device, queued
// on h's stream): minibatch k's rows are gathered on h's stream into stage[k & 1] while minibatch k-1 trains.  peer: a
// row-sharded ITEM_EMB, read through r = comm_src (the mappings published); else r reads this GPU's tables.
int mlp_keys_train(ctr_mlp* m, ctr_handle* h, const RowSrc& r, bool peer, const float* label, long ns, int32_t* n_iter, double* loss_curve) {
    const long bs = mlp_batch(m, ns);
    if (m->idx.size() < (size_t)ns) MCU(m, m->idx.alloc((size_t)ns));
    RET(mlp_stage(m, bs));
    RET(mlp_after_store(m, h, 0));                                     // labels and windows before the first loss
    const int* cls = nullptr;
    if (m->regressor) RET(mlp_targets(m, label, ns));                   // the survivors' labels are their targets
    else RET(mlp_labels(m, label, ns, &cls));                           // the survivors' labels
    RET(mlp_rows(m, bs));
    RET(mlp_init_params(m));
    const int nin = m->d.units[0];
    auto input = [&](long k, const long* bi, int rows, const double** X) -> int {
        const int s = (int)(k & 1);
        // stage[(k+1) & 1] was last read by minibatch k-1, the last one queued on m's stream; at k == 0 both buffers are
        // free once the epoch's index upload is done
        if (k == 0) MCU(m, cudaEventRecord(m->stage_free[0], m->stream));
        MCU(m, cudaEventRecord(m->stage_free[(k + 1) & 1], m->stream));
        MCU(m, cudaStreamWaitEvent(h->stream, m->stage_free[s], 0));
        // the PEER form reads the hot rows from this rank's replica and the rest from their owners: the same float32
        // rows, so the same float64 ones, as the local gather over the whole table
        RET(launch(h, peer ? "mlp_fit_gather_peer" : "mlp_gather", [&] {
            if (peer) k_gather_rows<double, RowsByIdx, true><<<grid_for_warps(h, rows), 256, 0, h->stream>>>(r, dims_of(h), m->stage[s].get(), (long)nin, rows, RowsByIdx{bi});
            else k_gather_rows<<<grid_for_warps(h, rows), 256, 0, h->stream>>>(r, dims_of(h), m->stage[s].get(), (long)nin, rows, RowsByIdx{bi});
        }));
        RET(mlp_after_store(m, h, s));
        *X = m->stage[s];
        return CTR_OK;
    };
    return mlp_epochs(m, ns, bs, label, cls, input, n_iter, loss_curve);
}

int mlp_fit_keys(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label, int64_t n,
                 int32_t* n_iter, double* loss_curve, int64_t* rows_used) {
    RET(mlp_keys_width(m));
    long ns = 0;
    RET(mlp_keys_resolve(h, user_ids, item_ids, ts, label, n, &ns));
    if (rows_used) *rows_used = (int64_t)ns;
    if (ns == 0) return mlp_err(m, CTR_ENOTFOUND, "no sample resolved: every key has an unknown user or item");
    const RowSrc r = idx_src(h, h->kt_user, h->kt_item, h->kt_hist_all, (int)ns);
    return mlp_keys_train(m, h, r, false, h->kt_label, ns, n_iter, loss_curve);
}

// A 64-bit digest of what must be equal on every rank before ctr_mlp_fit_keys_dist trains: the configuration (its device
// aside; the unused units slots zeroed) and the options, the model kind and, on a warm start, whether the model is fitted
// and, if so, its output kind, classes, t and packed parameters.  m's device is current.
int mlp_fit_digest(ctr_mlp* m, uint64_t* out) {
    ctr_mlp_config c = m->cfg;
    c.device = 0;
    for (int i = c.n_layers; i < 8; i++) c.units[i] = 0;
    uint64_t d = comm_hash(&c, sizeof c);
    d = comm_hash(&m->opts, sizeof m->opts, d);
    const int64_t kind[3] = {m->regressor ? 1 : 0, c.warm_start ? 1 : 0, c.warm_start && m->fitted ? 1 : 0};
    d = comm_hash(kind, sizeof kind, d);
    if (c.warm_start && m->fitted) {
        std::vector<double> p((size_t)m->np);
        MCU(m, cudaMemcpyAsync(p.data(), m->params, sizeof(double) * (size_t)m->np, cudaMemcpyDeviceToHost, m->stream));
        MCU(m, cudaStreamSynchronize(m->stream));
        const int64_t out_kind = m->out_kind;
        d = comm_hash(&out_kind, sizeof out_kind, d);
        d = comm_hash(&m->t, sizeof m->t, d);
        d = comm_hash(m->classes.data(), sizeof(double) * m->classes.size(), d);
        d = comm_hash(p.data(), sizeof(double) * p.size(), d);
    }
    *out = d;
    return CTR_OK;
}

// ctr_mlp_fit_keys_dist on world > 1 (see the header): every rank resolves and windows its own keys, the ranks agree on
// their verdicts, the model and the placement, all-gather the survivor counts and then the survivor records in rank
// order, and every rank runs the single-GPU fit over the same records.  args: CTR_OK or this rank's argument refusal.
int mlp_fit_keys_ranks(ctr_mlp* m, ctr_handle* h, int args, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label,
                       int64_t n, int32_t* n_iter, double* loss_curve, int64_t* rows_used) {
    const int W = h->comm.world, me = h->comm.rank, S = h->cfg.S;
    // the counts' exchange holds kMaxPeers ranks; world is the same everywhere, so every rank refuses alike
    if (W > kMaxPeers) return mlp_err(m, CTR_EINVAL, "fit_keys_dist: world %d, at most %d", W, kMaxPeers);
    const bool sh = emb_sharded(h);
    CommHdr hd{};
    hd.flag = (h->tab_sharded[CTR_TABLE_ITEM_EMB] ? 1 : 0) | (h->tab_sharded[CTR_TABLE_ITEM_FEAT] ? 2 : 0);
    // the digest whatever this rank's verdict, so that a refusal reaches the other ranks as itself
    const cudaError_t de = cudaSetDevice(m->dev);
    const int dg = de != cudaSuccess ? mlp_err(m, CTR_ECUDA, "cudaSetDevice(%d): %s", m->dev, cudaGetErrorString(de)) : mlp_fit_digest(m, &hd.hash[0]);
    long ns = 0;
    const int verdict = args != CTR_OK ? args : dg != CTR_OK ? dg : [&]() -> int {
        RET(mlp_keys_check(m, h));
        RET(mlp_keys_width(m));
        CU(h, cudaSetDevice(h->dev));
        return n > 0 ? mlp_keys_resolve(h, user_ids, item_ids, ts, label, n, &ns) : CTR_OK;
    }();
    RET(mlp_agree(m, h, hd, verdict));
    // ---- the counts (keys and survivors of every rank), then the records, concatenated in rank order on every rank
    int64_t all[2 * kMaxPeers] = {};
    const int64_t mine[2] = {n, ns};
    RET(comm_gather_i64(h, mine, 2, all));
    int64_t keys = 0, cnt[kMaxPeers], off[kMaxPeers + 1] = {0};
    for (int j = 0; j < W; j++) { keys += all[2 * j]; cnt[j] = all[2 * j + 1]; off[j + 1] = off[j] + cnt[j]; }
    // one GPU refuses a concatenation of more than INT32_MAX keys: so do the ranks, all of them, before any write
    if (keys > INT32_MAX) return mlp_err(m, CTR_EINVAL, "fit_keys_dist: the ranks pass %lld keys in all (more than INT32_MAX)", (long long)keys);
    const int64_t T = off[W];
    if (rows_used) *rows_used = T;
    if (T == 0) return mlp_err(m, CTR_ENOTFOUND, "no sample resolved on any rank: every key has an unknown user or item");
    DevBuf<int> g_user, g_item, g_hist; DevBuf<float> g_label;
    CU(h, g_user.alloc((size_t)T)); CU(h, g_item.alloc((size_t)T)); CU(h, g_label.alloc((size_t)T));
    CU(h, g_hist.alloc((size_t)std::max<int64_t>(T * S, 1)));
    cudaStream_t st = h->stream;
    if (ns > 0) {                                                    // this rank's segment in place (the windows are on st)
        CU(h, cudaMemcpyAsync(g_user.get() + off[me], h->kt_user, sizeof(int) * (size_t)ns, cudaMemcpyDeviceToDevice, st));
        CU(h, cudaMemcpyAsync(g_item.get() + off[me], h->kt_item, sizeof(int) * (size_t)ns, cudaMemcpyDeviceToDevice, st));
        CU(h, cudaMemcpyAsync(g_label.get() + off[me], h->kt_label, sizeof(float) * (size_t)ns, cudaMemcpyDeviceToDevice, st));
        if (S > 0) CU(h, cudaMemcpyAsync(g_hist.get() + off[me] * S, h->kt_hist_all, sizeof(int) * (size_t)ns * S, cudaMemcpyDeviceToDevice, st));
    }
    int rc = CTR_OK;
    RET(launch(h, "mlp_fit_gather_ranks", [&] {
        if (rc == CTR_OK) rc = comm_concat(h, g_user, sizeof(int), cnt, off);
        if (rc == CTR_OK) rc = comm_concat(h, g_item, sizeof(int), cnt, off);
        if (rc == CTR_OK) rc = comm_concat(h, g_label, sizeof(float), cnt, off);
        if (rc == CTR_OK && S > 0) rc = comm_concat(h, g_hist, sizeof(int) * (size_t)S, cnt, off);
    }));
    RET(rc);
    const RowSrc r = sh ? comm_src(h, g_user, g_item, g_hist, (int)T, false) : idx_src(h, g_user, g_item, g_hist, (int)T);
    return mlp_keys_train(m, h, r, sh, g_label, (long)T, n_iter, loss_curve);
}

int mlp_predict_keys(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n, float* scores) {
    if (!m->fitted) return mlp_err(m, CTR_ESTATE, "predict before fit");
    RET(mlp_keys_width(m));
    const int B = h->cfg.pred_batch, S = h->cfg.S, nin = m->d.units[0];
    // a row-sharded ITEM_EMB: each rank scores its own keys and reads the rows from their owners, as comm_predict does
    // (the publish after a table change is collective; training and prediction are kept apart by the caller)
    const bool sh = emb_sharded(h);
    if (sh) RET(comm_ensure(h, false));
    RET(keys_stage_init(h));
    RET(mlp_rows(m, B));
    RET(mlp_stage(m, B));
    DevBuf<float> d_out;
    MCU(m, d_out.alloc((size_t)B));
    long long* hk = (long long*)h->k_host.get();
    float* hs = (float*)(hk + (size_t)3 * B);
    int* hfirst = (int*)(hs + B);
    for (int64_t s = 0; s < n; s += B) {
        const int nb = (int)std::min<int64_t>(B, n - s);
        memcpy(hk, user_ids + s, sizeof(long long) * (size_t)nb);
        memcpy(hk + nb, item_ids + s, sizeof(long long) * (size_t)nb);
        memcpy(hk + 2 * (size_t)nb, ts + s, sizeof(long long) * (size_t)nb);
        CU(h, cudaMemcpyAsync(h->k_keys, hk, sizeof(long long) * (size_t)3 * nb, cudaMemcpyHostToDevice, h->stream));
        // BatchPredict's resolution (rcmd.go:277-337): an unknown key → user, item and history rows -1 → an all-zero X row
        RET(launch(h, "keys_resolve", [&] {
            k_keys_resolve<<<grid_for_warps(h, nb), 256, 0, h->stream>>>(h->idm_keys[0], h->idm_vals[0], h->idm_keys[0].size() - 1, h->idm_keys[1], h->idm_vals[1], h->idm_keys[1].size() - 1,
                                                                    h->ub_off, h->ub_ts, h->ub_items, (long)h->ub_users, h->k_keys, nb, S, h->s_user, h->s_item, h->s_hist);
        }));
        if (s == 0) CU(h, cudaMemcpyAsync(hfirst, h->s_user, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        const RowSrc r = sh ? comm_src(h, h->s_user, h->s_item, h->s_hist, nb, false) : idx_src(h, h->s_user, h->s_item, h->s_hist, nb);
        RET(launch(h, "mlp_gather", [&] {
            if (sh) k_gather_rows<double, RowsAsIs, true><<<grid_for_warps(h, nb), 256, 0, h->stream>>>(r, dims_of(h), m->stage[0].get(), (long)nin, nb, RowsAsIs{});
            else k_gather_rows<<<grid_for_warps(h, nb), 256, 0, h->stream>>>(r, dims_of(h), m->stage[0].get(), (long)nin, nb, RowsAsIs{});
        }));
        RET(mlp_after_store(m, h, 0));
        mlp_forward(m, m->stage[0], nullptr, nb);
        mlp_output(m, nb, d_out);
        MCU(m, cudaMemcpyAsync(hs, d_out, sizeof(float) * (size_t)nb, cudaMemcpyDeviceToHost, m->stream));
        MCU(m, cudaStreamSynchronize(m->stream));                      // the next chunk's gather overwrites stage[0]
        CU(h, cudaStreamSynchronize(h->stream));
        // rcmd.go:300-303: an unresolvable FIRST key is an error, later ones become zero rows
        if (s == 0 && *hfirst < 0)
            return mlp_err(m, CTR_ENOTFOUND, "get sample vector error: user %lld or item %lld has no features", (long long)user_ids[0], (long long)item_ids[0]);
        memcpy(scores + s, hs, sizeof(float) * (size_t)nb);
    }
    return CTR_OK;
}

// The float64 MLP's scoring pass over the item table (ctr_mlp_recommend_topk, ctr_mlp_rank_items; see mlp64.cuh), on
// h's stream: per user, the prefix of layer 0 once (prefix); per chunk of items, layer 0 from it and the later layers
// (chunk), which leave the chunk's logits in z().  On a row-sharded ITEM_EMB the chunks are this rank's local rows and
// the prefix reads the window's rows from their owners (k_mlp64_prefix<true>); each item's chain is the same as on one
// GPU, so its logit is too, whatever the chunk size.
struct MlpRecScore {
    ctr_mlp* m; ctr_handle* h;
    int L = 0, H = 0, pcols = 0, Bc = 0, l0_ctas = 0;
    int64_t N = 0, NL = 0;                  // ITEM_EMB's rows, the rows this GPU scores
    bool coll = false;                      // a row-sharded ITEM_EMB
    bool smem_w = false; size_t l0smem = 0;
    RowSrc src{};

    // the refusals, before anything is written
    int check() {
        if (!m->fitted) return mlp_err(m, CTR_ESTATE, "recommend before fit");
        if (!m->classes.empty())
            return mlp_err(m, CTR_ESTATE, "the classifier predicts %zu class labels: there is no click probability to rank items by", m->classes.size());
        MCU(m, cudaStreamSynchronize(m->stream));                        // h's stream reads the parameters
        L = m->d.n_layers; H = m->d.units[1];
        if (m->d.units[L - 1] != 1) return mlp_err(m, CTR_ESTATE, "recommendation ranks one output unit, the network has %d", m->d.units[L - 1]);
        coll = emb_sharded(h);
        N = h->tab_rows[CTR_TABLE_ITEM_EMB];
        NL = coll ? h->tab_local_rows[CTR_TABLE_ITEM_EMB] : N;
        if (N > INT32_MAX) return mlp_err(m, CTR_ESTATE, "ITEM_EMB has %lld rows: row ids are int32", (long long)N);
        const ctr_config& c = h->cfg;
        const int T = c.D + c.cF;
        pcols = c.uP + c.S * c.D;
        int optin = 0;
        MCU(m, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, m->dev));
        // W0's item rows stay in shared memory when they fit beside the item tile; else they are read through L1
        smem_w = rec_layer0_smem(T, H, true) <= (size_t)optin;
        l0smem = rec_layer0_smem(T, H, smem_w);
        if (l0smem > (size_t)optin)
            return mlp_err(m, CTR_ESTATE, "D + cF = %d item columns: a tile of %d items needs %zu bytes of shared memory (> %d)", T, kRecTile, l0smem, optin);
        // items per chunk: pred_batch in whole tiles, at most the table.  The chunk's activations take
        // Bc · (units[1] + … + units[L-1]) · 8 bytes of the classifier's buffers: a large catalogue wants a large pred_batch.
        auto tiles = [](int64_t x) { return std::max<int64_t>((x + kRecTile - 1) / kRecTile, 1) * kRecTile; };
        Bc = (int)std::min(tiles(c.pred_batch), tiles(NL));
        return CTR_OK;
    }
    // the classifier's activation buffers for one chunk (the last holds the logits) and layer 0's launch shape; on a
    // row-sharded ITEM_EMB before the agreement, so that a rank which cannot allocate them says so in its verdict
    int prepare() {
        for (int l = 1; l < L; l++) {
            const size_t need = (size_t)Bc * m->d.units[l];
            if (m->act[l].size() < need) MCU(m, m->act[l].alloc(need));
        }
        CU(h, cudaFuncSetAttribute(l0(), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l0smem));
        int l0_per_sm = 0;
        CU(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&l0_per_sm, l0(), 256, l0smem));
        l0_ctas = m->num_sms * std::max(1, l0_per_sm);
        return CTR_OK;
    }
    // the rows the prefix reads; on a row-sharded ITEM_EMB after the agreement has published the peer mappings
    void bind_rows() { src = coll ? comm_src(h, nullptr, nullptr, nullptr, 0, false) : idx_src(h, nullptr, nullptr, nullptr, 0); }
    decltype(&k_mlp64_rec_layer0<true>) l0() const { return smem_w ? k_mlp64_rec_layer0<true> : k_mlp64_rec_layer0<false>; }
    const double* z() const { return m->act[L - 1]; }
    // user row u with window uh (device): layer 0's user columns into d_pre [H]
    int prefix(int u, const int* uh, double* d_pre) {
        const ctr_config& c = h->cfg;
        const float* up = (c.uP > 0 && u < h->tab_rows[CTR_TABLE_USER_FEAT]) ? h->tab[CTR_TABLE_USER_FEAT] + (long)u * h->tab_ld[CTR_TABLE_USER_FEAT] : nullptr;
        return launch(h, "mlp_rec_prefix", [&] {
            if (coll) k_mlp64_prefix<true><<<(H + 127) / 128, 128, 0, h->stream>>>(m->params, m->d, up, c.uP, src, uh, c.S, c.D, d_pre);
            else k_mlp64_prefix<false><<<(H + 127) / 128, 128, 0, h->stream>>>(m->params, m->d, up, c.uP, src, uh, c.S, c.D, d_pre);
        });
    }
    // the logits of (local) items [i0, i0 + nb) from d_pre into z()
    int chunk(const double* d_pre, int i0, int nb) {
        const ctr_config& c = h->cfg;
        const int F = CTR_TABLE_ITEM_FEAT;
        const int ctas = std::min(l0_ctas, (nb + kRecTile - 1) / kRecTile);
        // ITEM_FEAT beside a row-sharded ITEM_EMB: sharded alike (local rows), or replicated (global rows)
        const bool fsh = coll && h->tab_sharded[F];
        const int fworld = coll && !fsh ? h->comm.world : 1, frank = coll && !fsh ? h->comm.rank : 0;
        RET(launch(h, "mlp_rec_layer0", [&] {
            l0()<<<ctas, 256, l0smem, h->stream>>>(m->params, m->d, d_pre, pcols, h->tab[CTR_TABLE_ITEM_EMB], h->tab_ld[CTR_TABLE_ITEM_EMB], h->tab[F],
                                                  h->tab_ld[F], (long)(fsh ? h->tab_local_rows[F] : h->tab_rows[F]), fworld, frank, c.D, c.cF, (long)i0, nb,
                                                  m->act[1]);
        }));
        for (int l = 1; l + 1 < L; l++)
            RET(launch(h, "mlp_rec_layers", [&] {
                k_mlp64_layer<true><<<mlp_grid(m, (long)nb * m->d.units[l + 1]), 256, 0, h->stream>>>(m->params, m->d, l, nullptr, 0, nullptr,
                                                                                                  m->act[l], m->act[l + 1], nb);
            }));
        return CTR_OK;
    }
};

// ctr_mlp_recommend_topk (see mlp64.cuh): per user, the prefix of layer 0 once; per chunk of items, layer 0 from it,
// the later layers, and the selection of rec.cuh on the float64 logits.  Everything runs on h's stream.  On a row-sharded
// ITEM_EMB the call is collective (ctr_recommend_topk_ex's rule): every rank checks the call and resolves the user ids
// with its own id map, the ranks agree, then each scores its shard for the windows rank 0's cache cuts, and the ranks'
// lists of each group are all-gathered and merged: the same total order over the same logits, so one GPU's result.
// args: CTR_OK, or the refusal of the caller's arguments (a collective call still takes part in the agreement).
int mlp_recommend(ctr_mlp* m, ctr_handle* h, int args, const int64_t* user_ids, const int64_t* ts, int64_t nu, int32_t k, int32_t exclude,
                  int32_t* out_rows, float* out_scores, double* out_logits, int32_t* out_count) {
    MlpRecScore sc{m, h};
    const bool coll = emb_sharded(h);
    const int W = coll ? h->comm.world : 1, S = h->cfg.S;
    const int vcheck = args != CTR_OK ? args : [&]() -> int { RET(mlp_keys_check(m, h)); return sc.check(); }();

    // ---- every user id, resolved before anything is written
    const int64_t G = std::min<int64_t>(nu, 256);                        // users per result copy (and list all-gather)
    const bool seen = exclude == CTR_EXCLUDE_SEEN;
    RecTopk<knn::Logit64Key> sel{h, "mlp_rec", k, exclude == CTR_EXCLUDE_WINDOW ? S : 0, W, coll ? h->comm.rank : 0, sc.NL, sc.Bc, seen, sc.N};
    long long *d_ids, *d_ts; int *d_urow, *d_hist; double* d_pre;
    std::vector<int> urow;
    const int verdict = vcheck != CTR_OK ? vcheck : [&]() -> int {
        RET(sel.setup(6, G, [&](Carve& cv) {
            d_ids = cv.take<long long>(nu); d_urow = cv.take<int>(nu); d_ts = cv.take<long long>(G); d_hist = cv.take<int>((size_t)G * S);
            d_pre = cv.take<double>(sc.H);
        }));
        CU(h, cudaMemcpyAsync(d_ids, user_ids, (size_t)nu * 8, cudaMemcpyHostToDevice, h->stream));
        RET(launch(h, "mlp_rec_resolve", [&] {
            k_idmap_lookup<<<mlp_grid(m, (long)nu), 256, 0, h->stream>>>(h->idm_keys[0], h->idm_vals[0], h->idm_keys[0].size() - 1, d_ids, (long)nu, d_urow);
        }));
        urow.resize((size_t)nu);
        CU(h, cudaMemcpyAsync(urow.data(), d_urow, (size_t)nu * 4, cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        for (int64_t u = 0; u < nu; u++)                                 // serving.Recommend's rule: the first unknown user
            if (urow[(size_t)u] < 0) return mlp_err(m, CTR_ENOTFOUND, "user %lld is not found", (long long)user_ids[u]);
        return sc.prepare();
    }();
    if (!coll) RET(verdict);
    else {
        CommHdr hd{};
        hd.n = nu; hd.k = k; hd.flag = exclude;
        if (args == CTR_OK) {
            hd.hash[0] = comm_hash(user_ids, (size_t)nu * sizeof(int64_t));
            hd.hash[1] = comm_hash(ts, (size_t)nu * sizeof(int64_t));
            hd.plan = G;                                                 // users per list all-gather
        }
        if (verdict == CTR_OK) hd.rows = comm_hash(urow.data(), (size_t)nu * sizeof(int));
        RET(mlp_agree(m, h, hd, verdict));
    }

    sc.bind_rows();
    for (int64_t g0 = 0; g0 < nu; g0 += G) {
        const int ng = (int)std::min<int64_t>(G, nu - g0);
        // GetUserBehavior(uid, S, -1, ts) from the device ubcache; no ubcache → an empty history (ctr_mlp_predict_keys).
        // On a shard every rank takes rank 0's windows, so every rank scores for the same ones.
        if (h->ub_off) CU(h, cudaMemcpyAsync(d_ts, ts + g0, sizeof(long long) * (size_t)ng, cudaMemcpyHostToDevice, h->stream));
        RET(ub_windows(h, h->stream, d_urow + g0, d_ts, ng, d_hist));
        if (coll && S > 0) RET(comm_bcast0(h, d_hist, sizeof(int) * (size_t)ng * S));
        for (int j = 0; j < ng; j++) {
            const int* uh = d_hist + (size_t)j * S;
            RET(sc.prefix(urow[(size_t)(g0 + j)], uh, d_pre));
            RET(sel.user(j, uh, sc.z(), [&](int i0, int nb) { return sc.chunk(d_pre, i0, nb); }, urow[(size_t)(g0 + j)], ts[g0 + j]));
        }
        RET(sel.finish(g0, ng, out_rows, out_scores, out_logits, out_count, [&](long n) {
            // an identity output's score is the predicted value itself, as ctr_mlp_predict_keys returns it
            if (m->out_kind == CTR_MLP_OUT_IDENTITY) k_f64_to_f32<<<(int)((n + 255) / 256), 256, 0, h->stream>>>(sel.ol, sel.os, n);
        }));
    }
    return CTR_OK;
}

// ctr_mlp_rank_items: mlp_recommend's scoring pass, counted by rec.cuh's rank kernels.  Keys with the same user row and
// ts share a pass, and so a window.  On a row-sharded ITEM_EMB the call is collective (ctr_rank_items_ex's rule), with
// mlp_recommend's agreement and rank 0's windows; each rank counts its shard and RecRank sums the counts.
int mlp_rank_items(ctr_mlp* m, ctr_handle* h, int args, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n,
                   int32_t exclude, int64_t* out_rank, double* out_logit) {
    MlpRecScore sc{m, h};
    const bool coll = emb_sharded(h);
    const int S = h->cfg.S;
    const int vcheck = args != CTR_OK ? args : [&]() -> int { RET(mlp_keys_check(m, h)); return sc.check(); }();
    RecRank<knn::Logit64Key> rk{h, "mlp_rank", exclude == CTR_EXCLUDE_WINDOW ? S : 0, sc.NL, sc.Bc, coll ? h->comm.world : 1, coll ? h->comm.rank : 0,
                                sc.N, exclude == CTR_EXCLUDE_SEEN};
    long long *d_ids, *d_ts; int *d_rows, *d_urow, *d_hist; double* d_pre;
    std::vector<int> rows;
    std::vector<std::vector<int64_t>> passes;
    // ---- user and item ids → rows; every user resolved before anything is written
    const int verdict = vcheck != CTR_OK ? vcheck : [&]() -> int {
        RET(rk.setup(6, [&](Carve& cv) {
            d_ids = cv.take<long long>((size_t)2 * n); d_rows = cv.take<int>((size_t)2 * n); d_ts = cv.take<long long>(n); d_urow = cv.take<int>(n);
            d_hist = cv.take<int>((size_t)n * S); d_pre = cv.take<double>(sc.H);
        }));
        CU(h, cudaMemcpyAsync(d_ids, user_ids, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(d_ids + n, item_ids, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
        RET(launch(h, "mlp_rank_resolve", [&] {
            for (int w = 0; w < 2; w++)
                k_idmap_lookup<<<mlp_grid(m, (long)n), 256, 0, h->stream>>>(h->idm_keys[w], h->idm_vals[w], h->idm_keys[w].size() - 1, d_ids + w * n, (long)n, d_rows + w * n);
        }));
        rows.resize((size_t)2 * n);
        CU(h, cudaMemcpyAsync(rows.data(), d_rows, (size_t)n * 8, cudaMemcpyDeviceToHost, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
        for (int64_t i = 0; i < n; i++)
            if (rows[(size_t)i] < 0) return mlp_err(m, CTR_ENOTFOUND, "user %lld is not found", (long long)user_ids[i]);
        passes = rank_passes(n, [&](int64_t i) { return std::make_pair(rows[(size_t)i], ts[i]); });
        return sc.prepare();
    }();
    if (!coll) RET(verdict);
    else {
        CommHdr hd{};
        hd.n = n; hd.flag = exclude;
        if (args == CTR_OK) {
            hd.hash[0] = comm_hash(user_ids, (size_t)n * sizeof(int64_t));
            hd.hash[1] = comm_hash(ts, (size_t)n * sizeof(int64_t));
            hd.hash[2] = comm_hash(item_ids, (size_t)n * sizeof(int64_t));
        }
        if (verdict == CTR_OK) {
            hd.rows = comm_hash(rows.data(), (size_t)2 * n * sizeof(int));   // the user rows, then the item rows
            hd.plan = (int64_t)passes.size();                                // two collectives per pass
        }
        RET(mlp_agree(m, h, hd, verdict));
    }
    const int* urow = rows.data(); const int* irow = rows.data() + n;

    // ---- one window per (user row, ts): GetUserBehavior(uid, S, -1, ts) from the device ubcache, empty without one;
    // on a shard rank 0's
    std::vector<int> pu; std::vector<long long> pts;           // the distinct (user, ts) in pass order, each once
    std::vector<size_t> win(passes.size());
    for (size_t p = 0; p < passes.size(); p++) {
        const int64_t i = passes[p][0];
        if (p > 0 && urow[passes[p - 1][0]] == urow[i] && ts[passes[p - 1][0]] == ts[i]) { win[p] = win[p - 1]; continue; }
        win[p] = pu.size(); pu.push_back(urow[i]); pts.push_back(ts[i]);
    }
    const int nw = (int)pu.size();
    if (h->ub_off) {
        CU(h, cudaMemcpyAsync(d_urow, pu.data(), sizeof(int) * (size_t)nw, cudaMemcpyHostToDevice, h->stream));
        CU(h, cudaMemcpyAsync(d_ts, pts.data(), sizeof(long long) * (size_t)nw, cudaMemcpyHostToDevice, h->stream));
    }
    RET(ub_windows(h, h->stream, d_urow, d_ts, nw, d_hist));
    if (coll && S > 0) RET(comm_bcast0(h, d_hist, sizeof(int) * (size_t)nw * S));

    sc.bind_rows();
    std::vector<int64_t> rank((size_t)n); std::vector<double> logit((size_t)n), pl(knn::kMaxK);
    std::vector<int> trow(knn::kMaxK); std::vector<int64_t> pr(knn::kMaxK);
    for (size_t p = 0; p < passes.size(); p++) {
        const auto& keys = passes[p];
        const int m_ = (int)keys.size();
        const int* uh = d_hist + win[p] * S;
        for (int j = 0; j < m_; j++) trow[j] = irow[keys[j]];
        RET(sc.prefix(urow[keys[0]], uh, d_pre));
        RET(rk.pass(trow.data(), m_, uh, sc.z(), [&](int i0, int nb) { return sc.chunk(d_pre, i0, nb); }, pr.data(), pl.data(),
                    urow[keys[0]], ts[keys[0]]));
        for (int j = 0; j < m_; j++) { rank[(size_t)keys[j]] = pr[j]; logit[(size_t)keys[j]] = pl[j]; }
    }
    memcpy(out_rank, rank.data(), sizeof(int64_t) * (size_t)n);
    if (out_logit) memcpy(out_logit, logit.data(), sizeof(double) * (size_t)n);
    return CTR_OK;
}
}  // namespace

int ctr_mlp_fit_keys(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label,
                     int64_t n, int32_t* n_iter, double* loss_curve, int64_t* rows_used) {
    if (!m) return CTR_EINVAL;
    if (!h || !user_ids || !item_ids || !ts || !label || n < 1 || n > INT32_MAX)
        return mlp_err(m, CTR_EINVAL, "bad fit_keys arguments (n in [1, 2^31))");
    std::lock_guard<std::mutex> lh(h->mu);                           // the feature store first, then the classifier
    std::lock_guard<std::mutex> lm(m->mu);
    m->err.clear(); h->err.clear();
    int rc = h->comm.world > 1 ? mlp_err(m, CTR_ESTATE, "ctr_mlp_fit_keys trains on one GPU (world=%d): data-parallel float64 training would "
                                                        "not keep fit's bit-for-bit result; fit on one GPU and serve the parameters on every rank "
                                                        "through ctr_mlp_set_params", h->comm.world)
                               : mlp_keys_check(m, h);
    if (rc == CTR_OK) rc = mlp_fit_keys(m, h, user_ids, item_ids, ts, label, n, n_iter, loss_curve, rows_used);
    return mlp_keys_done(m, h, rc);
}

// The arguments are checked before either object is touched; on world > 1 a rank whose arguments are bad still takes
// part in the agreement with its refusal, so that no rank is left waiting.
int ctr_mlp_fit_keys_dist(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, const float* label,
                          int64_t n, int32_t* n_iter, double* loss_curve, int64_t* rows_used) {
    const bool args_ok = n >= 0 && n <= INT32_MAX && (n == 0 || (user_ids && item_ids && ts && label));
    if (!m || !h)
        return mlp_err(m, CTR_EINVAL, args_ok ? "fit_keys_dist: null model or feature store"
                                              : "bad fit_keys_dist arguments (n in [0, 2^31), the arrays non-null when n > 0)");
    if (h->comm.world == 1) return ctr_mlp_fit_keys(m, h, user_ids, item_ids, ts, label, n, n_iter, loss_curve, rows_used);
    std::lock_guard<std::mutex> lh(h->mu);                           // the feature store first, then the classifier
    std::lock_guard<std::mutex> lm(m->mu);
    m->err.clear(); h->err.clear();
    const int args = args_ok ? CTR_OK : mlp_err(m, CTR_EINVAL, "bad fit_keys_dist arguments (n in [0, 2^31), the arrays non-null when n > 0)");
    return mlp_keys_done(m, h, mlp_fit_keys_ranks(m, h, args, user_ids, item_ids, ts, label, n, n_iter, loss_curve, rows_used));
}

int ctr_mlp_predict_keys(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n, float* scores) {
    if (!m) return CTR_EINVAL;
    if (!h || !user_ids || !item_ids || !ts || !scores || n < 1) return mlp_err(m, CTR_EINVAL, "bad predict_keys arguments");
    std::lock_guard<std::mutex> lh(h->mu);
    std::lock_guard<std::mutex> lm(m->mu);
    m->err.clear(); h->err.clear();
    int rc = mlp_keys_check(m, h);
    if (rc == CTR_OK) rc = mlp_predict_keys(m, h, user_ids, item_ids, ts, n, scores);
    return mlp_keys_done(m, h, rc);
}

int ctr_mlp_recommend_topk(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* ts, int64_t nu, int32_t k, int32_t exclude_history,
                           int32_t* out_rows, float* out_scores, double* out_logits, int32_t* out_count) {
    return ctr_mlp_recommend_topk_ex(m, h, user_ids, ts, nu, k, exclude_history ? CTR_EXCLUDE_WINDOW : CTR_EXCLUDE_NONE, out_rows, out_scores,
                                     out_logits, out_count);
}

int ctr_mlp_recommend_topk_ex(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* ts, int64_t nu, int32_t k, int32_t exclude,
                              int32_t* out_rows, float* out_scores, double* out_logits, int32_t* out_count) {
    if (!m) return CTR_EINVAL;
    auto args = [&]() -> int {
        if (!h || !user_ids || !ts || !out_rows || !out_scores || !out_count || nu < 1 || k < 1 || k > knn::kMaxK)
            return mlp_err(m, CTR_EINVAL, "bad recommend arguments (k in [1, %d], nu >= 1, user ids and ts, non-null outputs)", knn::kMaxK);
        if (!exclude_ok(exclude, ts)) return mlp_err(m, CTR_EINVAL, "bad exclusion mode %d (CTR_EXCLUDE_NONE, _WINDOW or _SEEN)", exclude);
        return CTR_OK;
    };
    if (!h) return args();
    std::lock_guard<std::mutex> lh(h->mu);
    std::lock_guard<std::mutex> lm(m->mu);
    if (!emb_sharded(h)) RET(args());    // a collective call: a rank with bad arguments still takes part in the agreement
    m->err.clear(); h->err.clear();
    const int rc = mlp_recommend(m, h, args(), user_ids, ts, nu, k, exclude, out_rows, out_scores, out_logits, out_count);
    return mlp_keys_done(m, h, rc);
}

int ctr_mlp_rank_items(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n,
                       int32_t exclude_history, int64_t* out_rank, double* out_logit) {
    return ctr_mlp_rank_items_ex(m, h, user_ids, item_ids, ts, n, exclude_history ? CTR_EXCLUDE_WINDOW : CTR_EXCLUDE_NONE, out_rank, out_logit);
}

int ctr_mlp_rank_items_ex(ctr_mlp* m, ctr_handle* h, const int64_t* user_ids, const int64_t* item_ids, const int64_t* ts, int64_t n,
                          int32_t exclude, int64_t* out_rank, double* out_logit) {
    if (!m) return CTR_EINVAL;
    auto args = [&]() -> int {
        if (!h || !user_ids || !item_ids || !ts || !out_rank || n < 1 || n > INT32_MAX)
            return mlp_err(m, CTR_EINVAL, "bad rank arguments (n in [1, 2^31), user ids, item ids and ts, non-null out_rank)");
        if (!exclude_ok(exclude, ts)) return mlp_err(m, CTR_EINVAL, "bad exclusion mode %d (CTR_EXCLUDE_NONE, _WINDOW or _SEEN)", exclude);
        return CTR_OK;
    };
    if (!h) return args();
    std::lock_guard<std::mutex> lh(h->mu);
    std::lock_guard<std::mutex> lm(m->mu);
    if (!emb_sharded(h)) RET(args());    // a collective call: a rank with bad arguments still takes part in the agreement
    m->err.clear(); h->err.clear();
    const int rc = mlp_rank_items(m, h, args(), user_ids, item_ids, ts, n, exclude, out_rank, out_logit);
    return mlp_keys_done(m, h, rc);
}

int ctr_comm_unique_id(void* id_out, int32_t* id_bytes) { return comm_unique_id(id_out, id_bytes); }
int ctr_comm_init(ctr_handle* h, const void* id, int32_t id_bytes) {
    if (!h || !id) return set_err(h, CTR_EINVAL, "null argument");
    std::lock_guard<std::mutex> lk(h->mu);
    CU(h, cudaSetDevice(h->dev));
    return comm_init(h, id, id_bytes);
}

}  // extern "C"
