// auc_dist_probe.cu — a test-only entry point that runs the per-rank steps of ctr_roc_auc_dist and ctr_group_auc_dist
// (go-ctr_b200/csrc/auc.cuh, included, not copied) for W ranks emulated as W shards of one device
// (tests/test_gpu_auc_dist_probe.py through ctypes, tests/auc_dist_probe.py).
//
// Rank r's samples are [cuts[r], cuts[r + 1]) of device arrays the caller owns.  Every step the engine runs on a rank
// runs here on that rank's buffers, in the engine's order; the exchanges the engine does with NCCL (the sample
// all-gather, the count all-gather, the routes of runs or records, the all-gather of the ranks' totals or group terms,
// the all-reduce of the area) are device copies in rank order and host sums.  The entry points synchronise the device
// and return 0, or -1 with auc_dist_probe_error() set.
// Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libauc_dist_probe.so tests/cuda/auc_dist_probe.cu
#include "auc.cuh"
#include <cstdio>
#include <vector>

using namespace ctr;

namespace {
char g_err[256] = "";
int fail(const char* what, cudaError_t e = cudaSuccess) {
    if (e != cudaSuccess) snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    else snprintf(g_err, sizeof g_err, "%s", what);
    return -1;
}
#define PC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(#call, e_); } while (0)
typedef unsigned long long u64;

// one rank's range-partition plan over its sorted keys: samples, splitters of every rank's samples, send offsets
struct Plan { std::vector<int64_t> off; };
template <typename K>
int plans(int W, const std::vector<const K*>& keys, const std::vector<int*>& d_u, std::vector<Plan>& out) {
    std::vector<int64_t> all((size_t)W * (kDistSamples + 1));
    DevBuf<long long> smp; DevBuf<u64> spl; DevBuf<long long> off;
    PC(smp.alloc(kDistSamples + 1)); PC(spl.alloc(kMaxPeers)); PC(off.alloc(kMaxPeers + 1));
    for (int r = 0; r < W; r++) {
        PC(dist_samples<K>(keys[r], d_u[r], smp, 0));
        PC(cudaMemcpy(&all[(size_t)r * (kDistSamples + 1)], smp, sizeof(int64_t) * (kDistSamples + 1), cudaMemcpyDeviceToHost));
    }
    u64 hs[kMaxPeers];
    dist_splitters(all.data(), W, hs);
    PC(cudaMemcpy(spl, hs, sizeof(u64) * (size_t)(W - 1), cudaMemcpyHostToDevice));
    out.assign((size_t)W, Plan{});
    for (int r = 0; r < W; r++) {
        PC(dist_part<K>(keys[r], d_u[r], spl, W, off, 0));
        out[r].off.resize((size_t)W + 1);
        PC(cudaMemcpy(out[r].off.data(), off, sizeof(int64_t) * (size_t)(W + 1), cudaMemcpyDeviceToHost));
    }
    return 0;
}
// the route: rank d receives rank 0's part for d, then rank 1's, ... into recv[d] (device, sized here)
template <typename T>
int route(int W, const std::vector<Plan>& p, const std::vector<const T*>& send, std::vector<DevBuf<T>>& recv, std::vector<long>& m) {
    recv.resize((size_t)W); m.assign((size_t)W, 0);
    for (int d = 0; d < W; d++) {
        for (int r = 0; r < W; r++) m[d] += (long)(p[r].off[d + 1] - p[r].off[d]);
        PC(recv[d].alloc((size_t)std::max<long>(m[d], 1)));
        long at = 0;
        for (int r = 0; r < W; r++) {
            const long c = (long)(p[r].off[d + 1] - p[r].off[d]);
            if (c > 0) PC(cudaMemcpy(recv[d].get() + at, send[r] + p[r].off[d], sizeof(T) * (size_t)c, cudaMemcpyDeviceToDevice));
            at += c;
        }
    }
    return 0;
}
int count(const int* d_u) { int u = 0; return cudaMemcpy(&u, d_u, sizeof u, cudaMemcpyDeviceToHost) == cudaSuccess ? u : -1; }
auto plain = [](const char*, auto&& f) { f(); return cudaGetLastError() == cudaSuccess ? 0 : -1; };
}  // namespace

extern "C" const char* auc_dist_probe_error() { return g_err; }

// ctr_roc_auc_dist over W emulated ranks: *auc, and stats[0 .. W) the runs each rank sends, stats[W .. 2W) the merged
// runs each rank owns, stats[2W] area2, stats[2W + 1] P, stats[2W + 2] N
extern "C" int auc_dist_probe_roc(const float* pred, const float* y, const long long* cuts, int W, double* auc, unsigned long long* stats) {
    if (W < 1 || W > kMaxPeers) return fail("bad world");
    std::vector<DevBuf<unsigned>> uk((size_t)W); std::vector<DevBuf<u64>> uc((size_t)W); std::vector<DevBuf<int>> du((size_t)W);
    for (int r = 0; r < W; r++) {
        const long n = (long)(cuts[r + 1] - cuts[r]), N = std::max<long>(n, 1);
        DevBuf<unsigned> k0, ks; DevBuf<u64> c0, cs; DevBuf<unsigned char> tmp;
        const size_t bytes = auc_dist_rle_bytes(N, 0);
        PC(k0.alloc(N)); PC(ks.alloc(N)); PC(c0.alloc(N)); PC(cs.alloc(N)); PC(tmp.alloc(bytes));
        PC(uk[r].alloc(N)); PC(uc[r].alloc(N)); PC(du[r].alloc(1));
        PC(auc_dist_local(pred + cuts[r], y + cuts[r], n, k0, c0, ks, cs, uk[r], uc[r], du[r], tmp, bytes, 0));
        PC(cudaDeviceSynchronize());
        stats[r] = (u64)count(du[r]);
    }
    std::vector<Plan> p;
    std::vector<const unsigned*> kp; std::vector<const u64*> cp; std::vector<int*> dp;
    for (int r = 0; r < W; r++) { kp.push_back(uk[r]); cp.push_back(uc[r]); dp.push_back(du[r]); }
    if (plans<unsigned>(W, kp, dp, p)) return -1;
    std::vector<DevBuf<unsigned>> rk; std::vector<DevBuf<u64>> rc; std::vector<long> m;
    if (route<unsigned>(W, p, kp, rk, m) || route<u64>(W, p, cp, rc, m)) return -1;
    std::vector<DevBuf<unsigned>> mk((size_t)W); std::vector<DevBuf<u64>> mc((size_t)W), inc((size_t)W);
    std::vector<u64> pos((size_t)W), neg((size_t)W); std::vector<int> mm((size_t)W);
    for (int d = 0; d < W; d++) {
        const long M = std::max<long>(m[d], 1);
        DevBuf<unsigned> ks; DevBuf<u64> cs; DevBuf<unsigned char> tmp;
        const size_t bytes = auc_dist_rle_bytes(M, 0);
        PC(ks.alloc(M)); PC(cs.alloc(M)); PC(mk[d].alloc(M)); PC(mc[d].alloc(M)); PC(inc[d].alloc(M)); PC(tmp.alloc(bytes));
        PC(auc_dist_rle(rk[d], rc[d], m[d], ks, cs, mk[d], mc[d], du[d], tmp, bytes, 0));
        PC(cudaDeviceSynchronize());
        mm[d] = count(du[d]);
        PC(auc_dist_totals(mc[d], mm[d], inc[d], tmp, bytes, &pos[d], &neg[d], 0));
        stats[W + d] = (u64)mm[d];
    }
    u64 base = 0, area2 = 0, P = 0, N = 0;
    DevBuf<u64> acc; PC(acc.alloc(1));
    for (int d = 0; d < W; d++) {
        PC(auc_dist_area(mc[d], inc[d], mm[d], base, acc, 0));
        u64 a = 0; PC(cudaMemcpy(&a, acc, sizeof a, cudaMemcpyDeviceToHost));
        area2 += a; base += pos[d]; P += pos[d]; N += neg[d];
    }
    stats[2 * W] = area2; stats[2 * W + 1] = P; stats[2 * W + 2] = N;
    *auc = auc_dist_value(area2, P, N);
    PC(cudaDeviceSynchronize());
    return 0;
}

// ctr_group_auc_dist over W emulated ranks: the result, and the per-group arrays (device, room for every group; each may
// be null); recv[0 .. W) the samples each rank owns after the route
extern "C" int auc_dist_probe_gauc(const float* pred, const float* y, const long long* group, const long long* cuts, int W, double* gauc,
                                   long long* n_groups, long long* n_used, long long* out_group, int* out_n, int* out_pos, double* out_auc,
                                   long long* recv) {
    if (W < 1 || W > kMaxPeers) return fail("bad world");
    std::vector<DevBuf<u64>> g1((size_t)W), v1((size_t)W); std::vector<DevBuf<int>> du((size_t)W);
    for (int r = 0; r < W; r++) {
        const long n = (long)(cuts[r + 1] - cuts[r]), N = std::max<long>(n, 1);
        DevBuf<u64> g0, v0; DevBuf<unsigned char> tmp;
        const size_t bytes = gauc_dist_bytes(N, 0);
        PC(g0.alloc(N)); PC(v0.alloc(N)); PC(g1[r].alloc(N)); PC(v1[r].alloc(N)); PC(du[r].alloc(1)); PC(tmp.alloc(bytes));
        const int un = (int)n;
        PC(cudaMemcpy(du[r], &un, sizeof un, cudaMemcpyHostToDevice));
        if (n > 0) PC(gauc_dist_sort(pred + cuts[r], y + cuts[r], group + cuts[r], n, g0, v0, g1[r], v1[r], tmp, bytes, 0));
        PC(cudaDeviceSynchronize());
    }
    std::vector<Plan> p;
    std::vector<const u64*> gp, vp; std::vector<int*> dp;
    for (int r = 0; r < W; r++) { gp.push_back(g1[r]); vp.push_back(v1[r]); dp.push_back(du[r]); }
    if (plans<u64>(W, gp, dp, p)) return -1;
    std::vector<DevBuf<u64>> rg, rv; std::vector<long> m;
    if (route<u64>(W, p, gp, rg, m) || route<u64>(W, p, vp, rv, m)) return -1;
    std::vector<DevBuf<u64>> uniq((size_t)W); std::vector<DevBuf<GaucAgg>> agg((size_t)W); std::vector<int> R((size_t)W, 0);
    for (int d = 0; d < W; d++) {
        recv[d] = m[d];
        if (m[d] == 0) continue;
        const long M = m[d];
        DevBuf<u64> a0, b0, a1, b1; DevBuf<GaucScan> scan; DevBuf<GaucAgg> val; DevBuf<unsigned char> tmp;
        const size_t bytes = gauc_dist_bytes(M, 0);
        PC(a0.alloc(M)); PC(b0.alloc(M)); PC(a1.alloc(M)); PC(b1.alloc(M)); PC(scan.alloc(M)); PC(val.alloc(M));
        PC(uniq[d].alloc(M)); PC(agg[d].alloc(M)); PC(tmp.alloc(bytes));
        PC(gauc_dist_order(rg[d], rv[d], M, a0, b0, a1, b1, tmp, bytes, 0));
        if (gauc_group_terms(plain, a1.get(), b1.get(), M, scan.get(), val.get(), uniq[d].get(), agg[d].get(), du[d].get(), tmp.get(), bytes,
                             dist_grid(M), (cudaStream_t)0))
            return fail("gauc_group_terms", cudaGetLastError());
        PC(cudaDeviceSynchronize());
        R[d] = count(du[d]);
    }
    long G = 0;
    for (int d = 0; d < W; d++) G += R[d];
    DevBuf<u64> all_uniq; DevBuf<GaucAgg> all_agg; DevBuf<GaucPart> part; DevBuf<GaucResult> res; DevBuf<int> d_runs;
    PC(all_uniq.alloc(std::max<long>(G, 1))); PC(all_agg.alloc(std::max<long>(G, 1))); PC(part.alloc(kGaucParts)); PC(res.alloc(1)); PC(d_runs.alloc(1));
    long at = 0;
    for (int d = 0; d < W; d++) {
        if (R[d] > 0) {
            PC(cudaMemcpy(all_uniq.get() + at, uniq[d], sizeof(u64) * (size_t)R[d], cudaMemcpyDeviceToDevice));
            PC(cudaMemcpy(all_agg.get() + at, agg[d], sizeof(GaucAgg) * (size_t)R[d], cudaMemcpyDeviceToDevice));
        }
        at += R[d];
    }
    const int g32 = (int)G;
    PC(cudaMemcpy(d_runs, &g32, sizeof g32, cudaMemcpyHostToDevice));
    if (gauc_fold_groups(plain, all_uniq.get(), all_agg.get(), d_runs.get(), out_group, out_n, out_pos, out_auc, part.get(), res.get(), (cudaStream_t)0))
        return fail("gauc_fold_groups", cudaGetLastError());
    GaucResult r{};
    PC(cudaMemcpy(&r, res, sizeof r, cudaMemcpyDeviceToHost));
    *gauc = r.gauc; *n_groups = r.groups; *n_used = r.used;
    PC(cudaDeviceSynchronize());
    return 0;
}
