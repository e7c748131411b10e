// shard_mlp_probe.cu — test-only entry points that launch the float64 MLP's serving kernels of go-ctr_b200/csrc/attn.cuh,
// mlp64.cuh and rec.cuh on device buffers the caller owns (tests/test_gpu_shard_mlp_probe.py through ctypes,
// tests/shard_mlp_probe.py), one launch each, as mlp_predict_keys, MlpRecScore, RecTopk and RecRank launch them.  The
// headers are included, not copies.
//
// On a row-sharded ITEM_EMB the key-fed gather and the prefix read rows through RowSrc::peer_emb[j] and the hot-row
// replica; layer 0 scores one rank's local rows; the selection and rank kernels run over Logit64Key at (world, rank).
// None of them needs anything from the other ranks but addresses and the caller's buffers, so W shards of one device
// act as W ranks.  Every entry point synchronises the device and returns 0, or -1 with shard_mlp_probe_error() set.
// Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libshard_mlp_probe.so tests/cuda/shard_mlp_probe.cu
#include "attn.cuh"
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
template <typename T> T* P(long long a) { return reinterpret_cast<T*>(a); }
using K = knn::Logit64Key;
}  // namespace

// What a RowSrc is built from (tests/shard_probe.py Rows, the layout of shard_probe.cu's ProbeRows)
struct ProbeRows {
    long long emb, ufeat, ifeat, user_row, item_row, hist, rows_cache, hot_tab;
    long long peer_emb[kMaxPeers], peer_ifeat[kMaxPeers];
    long long lde, ldu, ldi;
    int nvalid, n_emb, n_user, n_ifeat, world, ifeat_sharded, hot_k, pad;
};

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
    r.hot_k = p.hot_k; r.hot_tab = P<const float>(p.hot_tab);
    return r;
}
// the packed layout of the engine's parameters: per layer [intercepts (fo) | coefs (fi x fo)]
Mlp64Dims dims(int n_layers, const int* units, int hidden_act, int out_act) {
    Mlp64Dims d{};
    d.n_layers = n_layers; d.hidden_act = hidden_act; d.out_act = out_act;
    long off = 0;
    for (int l = 0; l < n_layers; l++) {
        d.units[l] = units[l];
        if (l + 1 < n_layers) { d.off[l] = off; off += (long)units[l + 1] * (1 + units[l]); }
    }
    return d;
}
}  // namespace

extern "C" const char* shard_mlp_probe_error() { return g_err; }

// k_gather_rows<double, RowsAsIs, peer>: X [B][ldx] of samples 0 .. B-1
extern "C" int shard_mlp_probe_gather(const ProbeRows* p, int peer, int uP, int S, int D, int cF, double* X, long long ldx, int B) {
    if (B < 1 || (peer && p->world < 2) || (!peer && p->world != 1)) return fail("bad gather arguments");
    const RowSrc r = row_src(*p);
    const Dims d{uP, S, D, cF, uP + S * D + D + cF};
    const int grid = (B + 7) / 8;
    if (peer) k_gather_rows<double, RowsAsIs, true><<<grid, 256>>>(r, d, X, (long)ldx, B, RowsAsIs{});
    else k_gather_rows<<<grid, 256>>>(r, d, X, (long)ldx, B, RowsAsIs{});
    return done();
}

// k_mlp64_prefix<peer>: pre [units[1]]
extern "C" int shard_mlp_probe_prefix(int peer, const double* params, int n_layers, const int* units, int hidden_act, int out_act, const float* urow,
                                      int uP, const ProbeRows* p, const int* hist, int S, int D, double* pre) {
    if (n_layers < 2 || n_layers > kMlpMaxLayers) return fail("bad prefix arguments");
    const Mlp64Dims d = dims(n_layers, units, hidden_act, out_act);
    const RowSrc r = row_src(*p);
    const int H = units[1];
    if (peer) k_mlp64_prefix<true><<<(H + 127) / 128, 128>>>(params, d, urow, uP, r, hist, S, D, pre);
    else k_mlp64_prefix<false><<<(H + 127) / 128, 128>>>(params, d, urow, uP, r, hist, S, D, pre);
    return done();
}

// k_mlp64_rec_layer0<smem_w> over items row0 .. row0 + n - 1 of emb, ctas CTAs, then k_mlp64_layer<true> for the later
// layers: the logits of the n items into z [n] (acts: [n][units[1] + ... ] float64 scratch)
extern "C" int shard_mlp_probe_score(int smem_w, const double* params, int n_layers, const int* units, int hidden_act, int out_act, const double* pre,
                                     int pcols, const float* emb, long long lde, const float* ifeat, long long ldi, long long n_ifeat, int fworld,
                                     int frank, int D, int cF, long long row0, int n, int ctas, double* acts, double* z) {
    if (n_layers < 2 || n_layers > kMlpMaxLayers || n < 1 || ctas < 1) return fail("bad score arguments");
    const Mlp64Dims d = dims(n_layers, units, hidden_act, out_act);
    const int T = D + cF, H = units[1];
    const size_t smem = rec_layer0_smem(T, H, smem_w != 0);
    double* act[kMlpMaxLayers] = {};
    size_t o = 0;
    for (int l = 1; l < n_layers; l++) { act[l] = l + 1 == n_layers ? z : acts + o; o += (size_t)n * units[l]; }
    auto l0 = smem_w ? k_mlp64_rec_layer0<true> : k_mlp64_rec_layer0<false>;
    PC(cudaFuncSetAttribute(l0, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    l0<<<ctas, 256, smem>>>(params, d, pre, pcols, emb, (long)lde, ifeat, (long)ldi, (long)n_ifeat, fworld, frank, D, cF, (long)row0, n, act[1]);
    for (int l = 1; l + 1 < n_layers; l++) {
        const long work = (long)n * units[l + 1];
        k_mlp64_layer<true><<<(int)std::min<long>((work + 255) / 256, 1024), 256>>>(params, d, l, nullptr, 0, nullptr, act[l], act[l + 1], n);
    }
    return done();
}

// k_rec_scan<Logit64Key> (seen == nullptr: the exclusion rows excl [nex]) or k_rec_scan_seen<Logit64Key> (world, rank)
extern "C" int shard_mlp_probe_scan(const double* z, int n, int row0, int world, int rank, int rows_per_slice, const int* excl, int nex,
                                    const unsigned* seen, int k, const double* run_s, const int* run_r, double* out_s, int* out_row) {
    if (k < 1 || k > knn::kMaxK || n < 1 || rows_per_slice < 1 || world < 1 || rank < 0 || rank >= world) return fail("bad scan arguments");
    const size_t smem = rec::scan_smem_bytes<K>(k, seen ? 0 : nex);
    const int slices = (n + rows_per_slice - 1) / rows_per_slice;
    if (seen) {
        void (*f)(const double*, int, int, int, int, int, const unsigned*, int, const double*, const int*, double*, int*) = rec::k_rec_scan_seen<K>;
        PC(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        f<<<slices, knn::kThreads, smem>>>(z, n, row0, world, rank, rows_per_slice, seen, k, run_s, run_r, out_s, out_row);
    } else {
        PC(cudaFuncSetAttribute(rec::k_rec_scan<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rec::k_rec_scan<K><<<slices, knn::kThreads, smem>>>(z, n, row0, world, rank, rows_per_slice, excl, nex, k, run_s, run_r, out_s, out_row);
    }
    return done();
}

// k_knn_merge<Logit64Key> over n list groups: list s of group g starts at g·qstride + s·sstride
extern "C" int shard_mlp_probe_merge(const double* in_s, const int* in_row, int slices, int k, long long qstride, long long sstride, int n,
                                     int* out_row, double* out_s, int* out_count) {
    if (k < 1 || k > knn::kMaxK || n < 1 || slices < 0) return fail("bad merge arguments");
    const size_t smem = knn::smem_bytes<K>(1, 0, k);
    PC(cudaFuncSetAttribute(knn::k_knn_merge<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    knn::k_knn_merge<K><<<n, knn::kThreads, smem>>>(in_s, in_row, slices, k, (long)qstride, (long)sstride, out_row, out_s, out_count);
    return done();
}

extern "C" int shard_mlp_probe_target_logits(const double* z, int n, int row0, int world, int rank, const int* rows, int m, double* tl,
                                             const unsigned* seen, int* flag) {
    if (m < 1 || m > knn::kMaxK || n < 0 || world < 1 || rank < 0 || rank >= world) return fail("bad target arguments");
    rec::k_rec_target_logits<double><<<(m + 255) / 256, 256>>>(z, n, row0, world, rank, rows, m, tl, seen, flag);
    return done();
}

// k_rec_rank_sort<Logit64Key> (flag == nullptr: the exclusion rows) or k_rec_rank_sort_seen<Logit64Key> (the owners' flags)
extern "C" int shard_mlp_probe_sort(const int* rows, const double* tl, int tls, int world, int m, long long n_items, const int* excl, int nex,
                                    const int* flag, int* place, int* nvalid, double* ss, int* sr, unsigned long long* bins) {
    if (m < 1 || m > knn::kMaxK || tls < m || world < 1) return fail("bad sort arguments");
    if (flag) rec::k_rec_rank_sort_seen<K><<<1, knn::kMaxK>>>(rows, tl, tls, world, m, (long)n_items, flag, place, nvalid, ss, sr, bins);
    else rec::k_rec_rank_sort<K><<<1, knn::kMaxK>>>(rows, tl, tls, world, m, (long)n_items, excl, nex, place, nvalid, ss, sr, bins);
    return done();
}

// k_rec_rank<Logit64Key> (seen == nullptr) or k_rec_rank_seen<Logit64Key>, (world, rank) forms
extern "C" int shard_mlp_probe_count(const double* z, int n, int row0, int world, int rank, const int* excl, int nex, const unsigned* seen,
                                     const double* ss, const int* sr, const int* nvalid, unsigned long long* bins) {
    if (n < 1 || world < 1 || rank < 0 || rank >= world) return fail("bad count arguments");
    const int grid = (n + rec::kRankRows - 1) / rec::kRankRows;
    if (seen) rec::k_rec_rank_seen<K><<<grid, rec::kRankThreads>>>(z, n, row0, world, rank, seen, ss, sr, nvalid, bins);
    else {
        PC(cudaFuncSetAttribute(rec::k_rec_rank<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, std::max(nex, 1) * 4));
        rec::k_rec_rank<K><<<grid, rec::kRankThreads, (size_t)nex * 4>>>(z, n, row0, world, rank, excl, nex, ss, sr, nvalid, bins);
    }
    return done();
}

extern "C" int shard_mlp_probe_finish(const int* rows, const double* tl, int tls, int world, const int* place, int m, long long n_items,
                                      const unsigned long long* bins, long long* out_rank, double* out_logit) {
    if (m < 1 || m > knn::kMaxK || tls < m || world < 1) return fail("bad finish arguments");
    rec::k_rec_rank_finish<double><<<1, knn::kMaxK>>>(rows, tl, tls, world, place, m, (long)n_items, bins, out_rank, out_logit);
    return done();
}
