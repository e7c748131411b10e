// shard_rank_probe.cu — test-only entry points that launch the rank kernels of go-ctr_b200/csrc/rec.cuh (ctr_rank_items)
// over LogitKey on device buffers the caller owns (tests/test_gpu_shard_rank_probe.py through ctypes,
// tests/shard_rank_probe.py), one launch each, as RecRank::pass launches them.  The header is included, not copied.
//
// On a row-sharded ITEM_EMB z holds one rank's logits of local rows row0 + b (global (row0 + b)·world + rank); tl
// [world][tls] is the ranks' gathered target logits, target j read from slot rows[j] % world; excl holds global rows.
// The kernels need nothing from the other ranks but these buffers, so W ranks are emulated on one device by the caller:
// nothing here waits on another rank.  Every entry point synchronises the device and returns 0, or -1 with
// shard_rank_probe_error() set.  Not linked into libctr_b200.so and not part of include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libshard_rank_probe.so tests/cuda/shard_rank_probe.cu
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
}  // namespace

extern "C" const char* shard_rank_probe_error() { return g_err; }

extern "C" int shard_rank_probe_target_logits(const float* z, int n, int row0, int world, int rank, const int* rows, int m, float* tl) {
    if (m < 1 || m > knn::kMaxK || n < 0 || world < 1 || rank < 0 || rank >= world) return fail("bad rank target arguments");
    rec::k_rec_target_logits<float><<<(m + 255) / 256, 256>>>(z, n, row0, world, rank, rows, m, tl);
    return done();
}
extern "C" int shard_rank_probe_sort(const int* rows, const float* tl, int tls, int world, int m, long long n_items, const int* excl, int nex,
                                     int* place, int* nvalid, float* ss, int* sr, unsigned long long* bins) {
    if (m < 1 || m > knn::kMaxK || tls < m || world < 1) return fail("bad rank sort arguments");
    rec::k_rec_rank_sort<knn::LogitKey><<<1, knn::kMaxK>>>(rows, tl, tls, world, m, (long)n_items, excl, nex, place, nvalid, ss, sr, bins);
    return done();
}
extern "C" int shard_rank_probe_count(const float* z, int n, int row0, int world, int rank, const int* excl, int nex, const float* ss, const int* sr,
                                      const int* nvalid, unsigned long long* bins) {
    if (n < 1 || world < 1 || rank < 0 || rank >= world) return fail("bad rank count arguments");
    PC(cudaFuncSetAttribute(rec::k_rec_rank<knn::LogitKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, std::max(nex, 1) * 4));
    rec::k_rec_rank<knn::LogitKey><<<(n + rec::kRankRows - 1) / rec::kRankRows, rec::kRankThreads, (size_t)nex * 4>>>(z, n, row0, world, rank, excl, nex,
                                                                                                                 ss, sr, nvalid, bins);
    return done();
}
extern "C" int shard_rank_probe_finish(const int* rows, const float* tl, int tls, int world, const int* place, int m, long long n_items,
                                       const unsigned long long* bins, long long* out_rank, float* out_logit) {
    if (m < 1 || m > knn::kMaxK || tls < m || world < 1) return fail("bad rank finish arguments");
    rec::k_rec_rank_finish<float><<<1, knn::kMaxK>>>(rows, tl, tls, world, place, m, (long)n_items, bins, out_rank, out_logit);
    return done();
}
