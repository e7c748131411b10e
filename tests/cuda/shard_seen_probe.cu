// shard_seen_probe.cu — test-only entry points that launch the CTR_EXCLUDE_SEEN kernels of go-ctr_b200/csrc/ubcache.cuh
// and rec.cuh over LogitKey on device buffers the caller owns (tests/test_gpu_shard_seen_probe.py through ctypes,
// tests/shard_seen_probe.py), one launch each, as RecTopk::user and RecRank::pass launch them.  The headers are
// included, not copied.
//
// On a row-sharded ITEM_EMB each rank builds a bitmap over its own local rows from its own behaviour cache (global row
// g is local row g / world of rank g % world); z holds one rank's logits of local rows row0 + b; tl and flag [world][tls]
// are the ranks' gathered target logits and seen flags, target j read from slot rows[j] % world.  The kernels need
// nothing from the other ranks but these buffers, so W ranks are emulated on one device by the caller.  The _one entry
// points launch the single-table forms (world = 1, a bitmap over the global rows).  Every entry point synchronises
// the device and returns 0, or -1 with shard_seen_probe_error() set.  Not linked into libctr_b200.so and not part of
// include/ctr_b200.h.
// Build: nvcc <flags of go-ctr_b200/build.py> -I go-ctr_b200/csrc -o tests/cuda/_build/libshard_seen_probe.so tests/cuda/shard_seen_probe.cu
#include "rec.cuh"
#include "ubcache.cuh"
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
using K = knn::LogitKey;
}  // namespace

extern "C" const char* shard_seen_probe_error() { return g_err; }

// rec_build_seen: seen [⌈n_local / 32⌉] zeroed, then k_ub_seen over the cache (off == nullptr: none) of n_users users and
// ne events, for user u, cut max_ts and the window hist [S]
extern "C" int shard_seen_probe_build(const long long* off, const long long* ts, const int* items, long long n_users, long long ne, int u,
                                      long long max_ts, const int* hist, int S, long long n_items, int world, int rank, long long n_local,
                                      unsigned* seen) {
    if (world < 1 || rank < 0 || rank >= world || n_local < 0 || S < 0) return fail("bad seen arguments");
    int dev = 0, sms = 0;
    PC(cudaGetDevice(&dev));
    PC(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long grid = std::max<long long>(1, std::min<long long>((ne + S + 255) / 256, (long long)sms * 4));
    PC(cudaMemset(seen, 0, (size_t)(n_local + 31) / 32 * sizeof(unsigned)));
    k_ub_seen<<<(int)grid, 256>>>(off, ts, items, off ? (long)n_users : 0L, u, max_ts, hist, S, (long)n_items, world, rank, seen);
    return done();
}

// k_rec_scan_seen: out [slices][k] with slices = ceil(n / rows_per_slice); one == 1: the single-table form
extern "C" int shard_seen_probe_scan(int one, const float* z, int n, int row0, int world, int rank, int rows_per_slice, const unsigned* seen, int k,
                                     const float* run_s, const int* run_r, float* out_s, int* out_row) {
    if (k < 1 || k > knn::kMaxK || n < 1 || rows_per_slice < 1 || world < 1 || rank < 0 || rank >= world || (one && world != 1))
        return fail("bad scan arguments");
    const size_t smem = rec::scan_smem_bytes<K>(k, 0);
    const int slices = (n + rows_per_slice - 1) / rows_per_slice;
    void (*sharded)(const float*, int, int, int, int, int, const unsigned*, int, const float*, const int*, float*, int*) = rec::k_rec_scan_seen<K>;
    void (*single)(const float*, int, int, int, const unsigned*, int, const float*, const int*, float*, int*) = rec::k_rec_scan_seen<K>;
    if (one) {
        PC(cudaFuncSetAttribute(single, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        single<<<slices, knn::kThreads, smem>>>(z, n, row0, rows_per_slice, seen, k, run_s, run_r, out_s, out_row);
    } else {
        PC(cudaFuncSetAttribute(sharded, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        sharded<<<slices, knn::kThreads, smem>>>(z, n, row0, world, rank, rows_per_slice, seen, k, run_s, run_r, out_s, out_row);
    }
    return done();
}

// k_knn_merge<LogitKey> over n lists groups: list s of group g starts at element g·qstride + s·sstride; out_count ==
// nullptr writes the lists as they stand (empty entries too)
extern "C" int shard_seen_probe_merge(const float* in_s, const int* in_row, int slices, int k, long long qstride, long long sstride, int n,
                                      int* out_row, float* out_s, int* out_count) {
    if (k < 1 || k > knn::kMaxK || n < 1 || slices < 0) return fail("bad merge arguments");
    const size_t smem = knn::smem_bytes<K>(1, 0, k);
    PC(cudaFuncSetAttribute(knn::k_knn_merge<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    knn::k_knn_merge<K><<<n, knn::kThreads, smem>>>(in_s, in_row, slices, k, (long)qstride, (long)sstride, out_row, out_s, out_count);
    return done();
}

extern "C" int shard_seen_probe_target_logits(const float* z, int n, int row0, int world, int rank, const int* rows, int m, float* tl,
                                              const unsigned* seen, int* flag) {
    if (m < 1 || m > knn::kMaxK || n < 0 || world < 1 || rank < 0 || rank >= world) return fail("bad target arguments");
    rec::k_rec_target_logits<float><<<(m + 255) / 256, 256>>>(z, n, row0, world, rank, rows, m, tl, seen, flag);
    return done();
}

// k_rec_rank_sort_seen: one == 0 reads the owners' flags [world][tls]; one == 1 the single-table form, which tests the
// bitmap seen over the global rows (tl [m])
extern "C" int shard_seen_probe_sort(int one, const int* rows, const float* tl, int tls, int world, int m, long long n_items, const int* flag,
                                     const unsigned* seen, int* place, int* nvalid, float* ss, int* sr, unsigned long long* bins) {
    if (m < 1 || m > knn::kMaxK || tls < m || world < 1 || (one && world != 1)) return fail("bad sort arguments");
    if (one) rec::k_rec_rank_sort_seen<K><<<1, knn::kMaxK>>>(rows, tl, m, (long)n_items, seen, place, nvalid, ss, sr, bins);
    else rec::k_rec_rank_sort_seen<K><<<1, knn::kMaxK>>>(rows, tl, tls, world, m, (long)n_items, flag, place, nvalid, ss, sr, bins);
    return done();
}

extern "C" int shard_seen_probe_count(int one, const float* z, int n, int row0, int world, int rank, const unsigned* seen, const float* ss,
                                      const int* sr, const int* nvalid, unsigned long long* bins) {
    if (n < 1 || world < 1 || rank < 0 || rank >= world || (one && world != 1)) return fail("bad count arguments");
    const int grid = (n + rec::kRankRows - 1) / rec::kRankRows;
    if (one) rec::k_rec_rank_seen<K><<<grid, rec::kRankThreads>>>(z, n, row0, seen, ss, sr, nvalid, bins);
    else rec::k_rec_rank_seen<K><<<grid, rec::kRankThreads>>>(z, n, row0, world, rank, seen, ss, sr, nvalid, bins);
    return done();
}

extern "C" int shard_seen_probe_finish(const int* rows, const float* tl, int tls, int world, const int* place, int m, long long n_items,
                                       const unsigned long long* bins, long long* out_rank, float* out_logit) {
    if (m < 1 || m > knn::kMaxK || tls < m || world < 1) return fail("bad finish arguments");
    rec::k_rec_rank_finish<float><<<1, knn::kMaxK>>>(rows, tl, tls, world, place, m, (long)n_items, bins, out_rank, out_logit);
    return done();
}
