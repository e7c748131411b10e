// mlp_fit_probe.cu — a test-only entry point that launches the key-fed fit's minibatch gather of go-ctr_b200/csrc/attn.cuh
// on device buffers the caller owns (tests/test_gpu_mlp_fit_probe.py through ctypes, tests/mlp_fit_probe.py), one launch
// per minibatch, as mlp_keys_train launches it.  The header is included, not copied.
//
// ctr_mlp_fit_keys_dist on a row-sharded ITEM_EMB gathers minibatch k's rows with k_gather_rows<double, RowsByIdx, true>:
// the survivors in the shuffled order bi, ITEM_EMB rows through RowSrc::peer_emb[j] and the hot-row replica, ITEM_FEAT
// rows sharded or replicated.  The kernel needs nothing from the other ranks but addresses, so W shards of one device act
// as W ranks.  The entry point synchronises the device and returns 0, or -1 with mlp_fit_probe_error() set.
// Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libmlp_fit_probe.so tests/cuda/mlp_fit_probe.cu
#include "attn.cuh"
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
template <typename T> T* P(long long a) { return reinterpret_cast<T*>(a); }
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
}  // namespace

extern "C" const char* mlp_fit_probe_error() { return g_err; }

// k_gather_rows<double, RowsByIdx, peer>: X [rows][ldx] of the samples bi[0 .. rows-1] (a minibatch of the shuffled
// survivor order), on the engine's launch shape (grid_for_warps: 8 samples per CTA, at most num_sms · 8 CTAs)
extern "C" int mlp_fit_probe_gather(const ProbeRows* p, int peer, int uP, int S, int D, int cF, const long long* bi, double* X, long long ldx,
                                    int rows) {
    if (rows < 1 || !bi || (peer && p->world < 2) || (!peer && p->world != 1)) return fail("bad gather arguments");
    int dev = 0, sms = 0;
    PC(cudaGetDevice(&dev));
    PC(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const RowSrc r = row_src(*p);
    const Dims d{uP, S, D, cF, uP + S * D + D + cF};
    const RowsByIdx by{reinterpret_cast<const long*>(bi)};
    const int grid = std::max(1, std::min((rows + 7) / 8, sms * 8));
    if (peer) k_gather_rows<double, RowsByIdx, true><<<grid, 256>>>(r, d, X, (long)ldx, rows, by);
    else k_gather_rows<double, RowsByIdx, false><<<grid, 256>>>(r, d, X, (long)ldx, rows, by);
    PC(cudaGetLastError());
    PC(cudaDeviceSynchronize());
    return 0;
}
