// shard_probe.cu — test-only entry points that launch the row-sharded kernels of go-ctr_b200/csrc/attn.cuh, knn.cuh and
// rec.cuh on device buffers the caller owns (tests/test_gpu_shard_probe.py through ctypes, tests/shard_probe.py).  The
// headers are included, not copied, and the attention kernels are instantiated from attn.cuh's lane-map table, so what
// runs here is what the engine launches for the same (model, D, PEER).
//
// The kernels of a row-sharded step need nothing from the other ranks but addresses: RowSrc::peer_emb[j], the owners'
// gradient buffers BwdOut::peer_adam[j] and the hot-row buffers are plain device pointers, and the system-scope atomics
// work on local memory.  So W shards allocated separately on one device act, for these kernels, as W ranks; the caller
// runs the ranks one after another on one stream.  Nothing here waits on another rank: no barrier kernel, no spin-wait,
// no collective.  Every entry point synchronises the device and returns 0, or -1 with shard_probe_error() set.
// Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libshard_probe.so tests/cuda/shard_probe.cu
#include "attn.cuh"
#include "knn.cuh"
#include "rec.cuh"
#include <algorithm>
#include <cstdio>

using namespace ctr;

namespace {
char g_err[256] = "";
int fail(const char* what, cudaError_t e = cudaSuccess) {
    if (e != cudaSuccess) snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    else snprintf(g_err, sizeof g_err, "%s", what);
    return -1;
}
#define PC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(#call, e_); } while (0)
int done() { PC(cudaGetLastError()); PC(cudaDeviceSynchronize()); return 0; }
int num_sms() {
    int dev = 0, n = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}
template <typename T> T* P(long long a) { return reinterpret_cast<T*>(a); }
}  // namespace

// What a RowSrc is built from: device addresses as integers (torch data_ptr()).  ctypes mirror: tests/shard_probe.py Rows.
struct ProbeRows {
    long long emb, ufeat, ifeat, user_row, item_row, hist, rows_cache, hot_tab;
    long long peer_emb[kMaxPeers], peer_ifeat[kMaxPeers];
    long long lde, ldu, ldi;
    int nvalid, n_emb, n_user, n_ifeat, world, ifeat_sharded, hot_k, pad;
};
// the owner-side row-Adam state of one rank's BwdOut
struct ProbeAdam {
    long long peer_adam[kMaxPeers];
    long long rows;             // the largest shard's local rows: shard_grad_layout(rows, lde)
    long long hot_touch;
};
struct ProbeRowAdam { float lr, b1, b2, eps, c1, c2, inv_batch; };

namespace {
RowSrc row_src(const ProbeRows& p) {
    RowSrc r{};
    r.emb = P<const float>(p.emb); r.lde = (long)p.lde;
    r.ufeat = P<const float>(p.ufeat); r.ldu = (long)p.ldu;
    r.ifeat = P<const float>(p.ifeat); r.ldi = (long)p.ldi;
    r.user_row = P<const int>(p.user_row); r.item_row = P<const int>(p.item_row); r.hist = P<const int>(p.hist);
    r.nvalid = p.nvalid; r.n_emb = p.n_emb; r.n_user = p.n_user; r.n_ifeat = p.n_ifeat;
    r.world = p.world; r.wmask = p.world - 1; r.wshift = 0;
    while ((1 << r.wshift) < p.world) r.wshift++;
    r.ifeat_sharded = p.ifeat_sharded;
    for (int j = 0; j < kMaxPeers; j++) { r.peer_emb[j] = P<float>(p.peer_emb[j]); r.peer_ifeat[j] = P<const float>(p.peer_ifeat[j]); }
    r.rows_cache = P<float>(p.rows_cache);
    r.hot_k = p.hot_k; r.hot_tab = P<const float>(p.hot_tab);
    return r;
}
RowAdam row_adam(const ProbeRowAdam& a) { return RowAdam{a.lr, a.b1, a.b2, a.eps, a.c1, a.c2, a.inv_batch}; }
bool shape_ok(int model, int D, int S, int world) {
    return model >= MODEL_YOUTUBE && model <= MODEL_DIN_EUC && (D == 16 || D == 32 || D == 64 || D == 128) && S >= 1 && S <= 64 &&
           world >= 1 && world <= kMaxPeers && (world & (world - 1)) == 0;
}
}  // namespace

extern "C" const char* shard_probe_error() { return g_err; }
extern "C" int shard_probe_num_sms() { return num_sms(); }
// LPR and VPL of the engine's lane map [bwd][peer][log2(D) - 4]
extern "C" int shard_probe_lanes(int bwd, int peer, int D, int* lpr, int* vpl) {
    const int i = D == 16 ? 0 : D == 32 ? 1 : D == 64 ? 2 : D == 128 ? 3 : -1;
    if (i < 0) return fail("D outside {16, 32, 64, 128}");
    *lpr = kLanes[bwd ? 1 : 0][peer ? 1 : 0][i].lpr; *vpl = kLanes[bwd ? 1 : 0][peer ? 1 : 0][i].vpl;
    return 0;
}
// offsets of ShardGrad for a shard of `rows` local rows: flag_off, list_off, grad_off, bytes
extern "C" void shard_probe_grad_layout(long long rows, long long lde, long long* out) {
    const ShardGrad s = shard_grad_layout((long)rows, (long)lde);
    out[0] = s.flag_off; out[1] = s.list_off; out[2] = s.grad_off; out[3] = s.bytes;
}

// k_attn_fwd_idx<lanes of (forward, lane_peer, D), model, peer> over B samples, X0 [B, ldx0]; grid as the engine's.
// peer takes the PEER lane map; lane_peer without peer is its single-table twin (same lane map, same arithmetic).
extern "C" int shard_probe_fwd_idx(const ProbeRows* p, int model, int uP, int S, int D, int cF, const float* att, float* X0, long ldx0,
                                   int Kp, int B, int peer, int lane_peer) {
    if (!shape_ok(model, D, S, p->world) || uP % 4 || (Kp - 2 * D) / 4 > 32 || B < 1) return fail("bad shape");
    if (peer && !lane_peer) return fail("the engine launches the PEER forward only with the PEER lane map");
    const RowSrc r = row_src(*p);
    const Dims d{uP, S, D, cF, uP + 2 * D + cF};
    const int g = attn_grid(num_sms(), B);
    with_model(model, [&](auto m) {
        constexpr int M = decltype(m)::value;
        auto run = [&](auto pk, auto lk) {
            constexpr bool PK = decltype(pk)::value, LK = decltype(lk)::value;
            with_lanes<false, LK>(D, [&](auto l) {
                using L = decltype(l);
                k_attn_fwd_idx<L::LPR, L::VPL, M, PK><<<g, kAttnThreads>>>(r, d, att, X0, ldx0, Kp, B);
            });
        };
        if (peer) run(std::true_type{}, std::true_type{});
        else if (lane_peer) run(std::false_type{}, std::true_type{});        // the single-table twin of the PEER kernel
        else run(std::false_type{}, std::false_type{});
    });
    return done();
}

// k_attn_bwd_idx<lanes of (backward, peer, D), model, FUSED = PEER = peer>.
//   peer: BwdOut as the engine fills it for a sharded step — sgd = 1, neg_lr (−lr/world for SGD, 1/world for row Adam),
//         the hot-row replica accumulators [hot_reps, hot_rows, D], and under row Adam (adam->peer_adam[0] != 0) the
//         owners' gradient buffers with shard_grad_layout(adam->rows, lde) and the hot rows' touch marks;
//   else: the single-table twin, gradients written to dUb [B, S, D] and dIt [B, D].
extern "C" int shard_probe_bwd_idx(const ProbeRows* p, int model, int uP, int S, int D, int cF, const float* att, const float* dX, long lddx,
                                   int B, int peer, float* datt, float* dUb, float* dIt, float neg_lr, float* hot_acc, int hot_rows,
                                   int hot_reps, const ProbeAdam* adam) {
    if (!shape_ok(model, D, S, p->world) || B < 1 || (hot_rows > 0 && hot_reps < 1)) return fail("bad shape");
    const RowSrc r = row_src(*p);
    const Dims d{uP, S, D, cF, uP + 2 * D + cF};
    BwdOut o{};
    o.datt = datt;
    if (peer) {
        o.sgd = 1; o.neg_lr = neg_lr;
        o.hot_acc = hot_acc; o.hot_rows = hot_rows; o.hot_reps = hot_reps;
        if (adam && adam->peer_adam[0]) {
            for (int j = 0; j < kMaxPeers; j++) o.peer_adam[j] = P<unsigned char>(adam->peer_adam[j]);
            o.adam = shard_grad_layout((long)adam->rows, r.lde);
            o.hot_touch = P<float>(adam->hot_touch);
        }
    } else { o.dUb = dUb; o.dIt = dIt; }
    const int g = attn_grid(num_sms(), B);
    with_model(model, [&](auto m) {
        constexpr int M = decltype(m)::value;
        if (peer) with_lanes<true, true>(D, [&](auto l) {
            using L = decltype(l);
            k_attn_bwd_idx<L::LPR, L::VPL, M, true, true><<<g, kAttnThreads>>>(r, d, att, dX, lddx, o, B);
        });
        else with_lanes<true, false>(D, [&](auto l) {
            using L = decltype(l);
            k_attn_bwd_idx<L::LPR, L::VPL, M, false, false><<<g, kAttnThreads>>>(r, d, att, dX, lddx, o, B);
        });
    });
    return done();
}

// the hot rows' replica accumulators folded into this rank's gradient sum: hot_sum[hot_k, D] += Σ_rep acc; acc = 0
extern "C" int shard_probe_hot_fold(float* hot_sum, float* hot_acc, int hot_k, int hot_reps, int D) {
    k_hot_apply<<<num_sms() * 4, 256>>>(hot_sum, D, hot_acc, hot_k, hot_reps, D, 1.0f);
    return done();
}
// SGD on the replicated hot rows: hot_tab += hot_sum (the all-reduced −lr/world sums); hot_sum = 0
extern "C" int shard_probe_hot_apply_sgd(float* hot_tab, float* hot_sum, long long n) {
    if (n % 4) return fail("n must be a multiple of 4");
    k_apply_table_grad<<<num_sms() * 8, 256>>>(hot_tab, hot_sum, (long)(n / 4));
    return done();
}
extern "C" int shard_probe_hot_adam(float* hot_tab, float* sum, float* touch, float* mo, float* vo, int hot_k, int D, const ProbeRowAdam* a) {
    k_hot_adam<<<num_sms() * 8, 256>>>(hot_tab, sum, touch, mo, vo, hot_k, D, row_adam(*a));
    return done();
}
// the owner's update of its touched rows; gbuf laid out by shard_grad_layout(rows, lde)
extern "C" int shard_probe_shard_adam(unsigned char* gbuf, long long rows, float* tab, float* mo, float* vo, long long lde, int D, const ProbeRowAdam* a) {
    k_shard_adam<<<num_sms() * 8, 256>>>(gbuf, shard_grad_layout((long)rows, (long)lde), tab, mo, vo, (long)lde, D, row_adam(*a));
    return done();
}
extern "C" int shard_probe_hot_pull(const ProbeRows* p, float* hot_tab, int hot_k, int D) {
    k_hot_pull<<<num_sms() * 4, 256>>>(row_src(*p), hot_tab, hot_k, D);
    return done();
}
extern "C" int shard_probe_hot_writeback(float* shard, long long lde, const float* hot_tab, int hot_k, int D, int world, int rank) {
    k_hot_writeback<<<num_sms() * 4, 256>>>(shard, (long)lde, hot_tab, hot_k, D, world, rank);
    return done();
}
extern "C" int shard_probe_hot_own(float* hot, const float* shard, long long lde, int hot_k, int D, int world, int rank) {
    k_hot_own<<<num_sms() * 4, 256>>>(hot, shard, (long)lde, hot_k, D, world, rank);
    return done();
}

// k_attn_fwd_user<lanes of (forward, non-PEER, D), model, peer>: X0 rows of (user, item i0 + b, hist) for b < B; on a
// shard (peer) the items are the rank's local rows.  One wave of resident CTAs, as attn_forward_user launches it.
extern "C" int shard_probe_fwd_user(const ProbeRows* p, int model, int uP, int S, int D, int cF, const float* att, int user, const int* hist,
                                    int i0, int rank, float* X0, long ldx0, int Kp, int B, int peer) {
    if (!shape_ok(model, D, S, p->world) || B < 1) return fail("bad shape");
    const RowSrc r = row_src(*p);
    const Dims d{uP, S, D, cF, uP + 2 * D + cF};
    const size_t smem = user_smem_floats(S, D, Kp) * sizeof(float);
    int rc = 0;
    with_model(model, [&](auto m) {
        constexpr int M = decltype(m)::value;
        with_lanes<false, false>(D, [&](auto l) {
            using L = decltype(l);
            auto launch = [&](auto kern) {
                int occ = 1;
                if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
                    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kAttnThreads, smem) != cudaSuccess) { rc = -1; return; }
                const int grid = std::min(num_sms() * std::max(occ, 1), attn_grid(num_sms(), B));
                kern<<<grid, kAttnThreads, smem>>>(r, d, att, user, hist, i0, rank, X0, ldx0, Kp, B);
            };
            if (peer) launch(k_attn_fwd_user<L::LPR, L::VPL, M, true>); else launch(k_attn_fwd_user<L::LPR, L::VPL, M, false>);
        });
    });
    if (rc) return fail("fwd_user: shared-memory attribute or occupancy query failed", cudaGetLastError());
    return done();
}
// out [n, D] = ITEM_EMB rows rows[0, n) widened to float64 (hot rows from the replica, the others from their owners)
extern "C" int shard_probe_gather_rows_f64(const ProbeRows* p, const int* rows, int n, int D, double* out) {
    const int gg = (int)std::max<long>(1, std::min<long>(((long)n * D + 255) / 256, (long)num_sms() * 4));
    k_gather_rows_f64<<<gg, 256>>>(row_src(*p), rows, n, D, out);
    return done();
}

// k_knn_scan<QT, rowq>: the table tab [nrows, ld] (local row l is global row l·world + rank) against nq queries — table
// rows qrow (rowq) or float64 vectors qvec with excluded rows excl — in `slices` slices of rows_per_slice rows;
// out [nq][slices][k].  QT as ctr_knn_search picks it.
extern "C" int shard_probe_knn_scan(const float* tab, long long ld, long long nrows, int world, int rank, int D, const double* qvec, const int* qrow,
                                    const int* excl, int nq, int k, long long rows_per_slice, int slices, double* out_sim, int* out_row, int rowq) {
    if (k < 1 || k > knn::kMaxK || nq < 1 || slices < 1 || rows_per_slice % knn::kStep) return fail("bad knn arguments");
    const int Dp = (D + 3) & ~3;
    int QT = 16;
    while (QT > 1 && (QT / 2 >= nq || knn::kTileBytes + knn::smem_bytes<knn::SimKey>(QT, Dp, k) > ((size_t)200 << 10))) QT /= 2;
    const size_t smem = knn::kTileBytes + knn::smem_bytes<knn::SimKey>(QT, Dp, k);
    auto go = [&](auto kern, int qt) {
        PC(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<dim3((nq + qt - 1) / qt, slices), knn::kThreads, smem>>>(tab, (long)ld, (long)nrows, world, rank, D, qvec, qrow, excl, nq, k,
                                                                        (long)rows_per_slice, out_sim, out_row);
        return 0;
    };
    int rc;
    if (rowq) {
        switch (QT) {
            case 1: rc = go(knn::k_knn_scan<1, true>, 1); break;   case 2: rc = go(knn::k_knn_scan<2, true>, 2); break;
            case 4: rc = go(knn::k_knn_scan<4, true>, 4); break;   case 8: rc = go(knn::k_knn_scan<8, true>, 8); break;
            default: rc = go(knn::k_knn_scan<16, true>, 16); break;
        }
    } else {
        switch (QT) {
            case 1: rc = go(knn::k_knn_scan<1, false>, 1); break;  case 2: rc = go(knn::k_knn_scan<2, false>, 2); break;
            case 4: rc = go(knn::k_knn_scan<4, false>, 4); break;  case 8: rc = go(knn::k_knn_scan<8, false>, 8); break;
            default: rc = go(knn::k_knn_scan<16, false>, 16); break;
        }
    }
    if (rc) return rc;
    return done();
}
// k_knn_merge over n queries: list s of query g starts at element g·qstride + s·sstride.  key 0: SimKey (float64
// similarities), 1: LogitKey (float32 logits).  out_count == nullptr writes the lists as they stand (empty entries too).
extern "C" int shard_probe_knn_merge(int key, const void* in_sim, const int* in_row, int slices, int k, long long qstride, long long sstride, int n,
                                     int* out_row, void* out_sim, int* out_count) {
    if (k < 1 || k > knn::kMaxK || n < 1) return fail("bad merge arguments");
    if (key == 0)
        knn::k_knn_merge<knn::SimKey><<<n, knn::kThreads, knn::smem_bytes<knn::SimKey>(1, 0, k)>>>(
            static_cast<const double*>(in_sim), in_row, slices, k, (long)qstride, (long)sstride, out_row, static_cast<double*>(out_sim), out_count);
    else
        knn::k_knn_merge<knn::LogitKey><<<n, knn::kThreads, knn::smem_bytes<knn::LogitKey>(1, 0, k)>>>(
            static_cast<const float*>(in_sim), in_row, slices, k, (long)qstride, (long)sstride, out_row, static_cast<float*>(out_sim), out_count);
    return done();
}
// k_rec_scan<LogitKey>: z [n] logits of local rows row0 + b (global (row0 + b)·world + rank), excluded global rows
// excl[0, nex); out [slices][k] with slices = ceil(n / rows_per_slice)
extern "C" int shard_probe_rec_scan(const float* z, int n, int row0, int world, int rank, int rows_per_slice, const int* excl, int nex, int k,
                                    const float* run_s, const int* run_r, float* out_s, int* out_row) {
    if (k < 1 || k > knn::kMaxK || n < 1 || rows_per_slice < 1) return fail("bad rec arguments");
    const size_t smem = rec::scan_smem_bytes<knn::LogitKey>(k, nex);
    PC(cudaFuncSetAttribute(rec::k_rec_scan<knn::LogitKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rec::k_rec_scan<knn::LogitKey><<<(n + rows_per_slice - 1) / rows_per_slice, knn::kThreads, smem>>>(z, n, row0, world, rank, rows_per_slice, excl, nex, k,
                                                                                                     run_s, run_r, out_s, out_row);
    return done();
}
